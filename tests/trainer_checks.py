"""Shared by the trainer tests: a restatement of the reference's online training loop, written from
trainer/online_trainer.py (not copied), and comparisons of logs and buffer contents."""
import torch

TIME_FIELDS = ("elapsed_time", "steps_per_second")


def reference_online(cfg, env, agent, buffer):
    """A restatement of the reference's OnlineTrainer.train (trainer/online_trainer.py:74-127) with its to_td (:54-72),
    eval (:28-52) and common_metrics (:18-26, the time fields left out).  Returns the logged (category, dict) list."""
    logs, metrics = [], {}
    step, ep_idx, done, eval_next, info, rows = 0, 0, True, False, None, None
    seed = cfg.seed_steps

    def first_row(o):                    # :61-65 -- rand_act() is called for the NaN action's shape
        nan = torch.tensor(float("nan"))
        return o, torch.full_like(env.rand_act(), float("nan")), nan, nan

    def run_eval():                      # :30-52
        rewards, successes, lengths = [], [], []
        for _ in range(cfg.eval_episodes):
            o, d, total, t = env.reset(), False, 0, 0
            while not d:
                a = agent.act(o, t0=t == 0, eval_mode=True)
                o, r, d, inf = env.step(a)
                total, t = total + r, t + 1
            rewards.append(float(total))
            successes.append(inf["success"])
            lengths.append(t)
        n = len(rewards)
        return dict(episode_reward=sum(rewards) / n, episode_success=sum(successes) / n, episode_length=sum(lengths) / n)

    while step <= cfg.steps:             # :77
        if step % cfg.eval_freq == 0:    # :79-80
            eval_next = True
        if done:
            if eval_next:                # :84-88
                m = run_eval()
                m.update(step=step, episode=ep_idx)
                logs.append(("eval", m))
                eval_next = False
            if step > 0:                 # :90-101
                if info["terminated"] and not cfg.episodic:
                    raise ValueError("termination outside episodic mode")
                metrics.update(episode_reward=torch.tensor([r[2] for r in rows[1:]]).sum(),
                               episode_success=info["success"], episode_length=len(rows),
                               episode_terminated=info["terminated"], step=step, episode=ep_idx)
                logs.append(("train", dict(metrics)))
                ep_idx = buffer.add({"obs": torch.stack([r[0] for r in rows]), "action": torch.stack([r[1] for r in rows]),
                                     "reward": torch.stack([r[2] for r in rows]),
                                     "terminated": torch.stack([r[3] for r in rows])})
            obs = env.reset()            # :103-104
            rows = [first_row(obs)]
        action = agent.act(obs, t0=len(rows) == 1) if step > seed else env.rand_act()      # :107-110
        obs, reward, done, info = env.step(action)                                          # :111-112
        rows.append((obs, action, reward, info["terminated"]))
        if step >= seed:                 # :115-123
            for _ in range(seed if step == seed else 1):
                out = agent.update(buffer)
            metrics.update(out)
        step += 1
    return logs


def normal(logs):
    return [(c, {k: (v.item() if torch.is_tensor(v) else v) for k, v in d.items() if k not in TIME_FIELDS})
            for c, d in logs]


def stored(buf):
    """Every live trajectory's rows, oldest first."""
    cap = buf.capacity
    return [{k: st[(s + torch.arange(n)) % cap] for k, st in buf._storage.items()} for s, n in buf._table]


def same(a, b):
    """Equal dtype, shape and bits, NaN in the same places."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if not a.is_floating_point():
        return torch.equal(a, b)
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(nan=0.0), b.nan_to_num(nan=0.0))
