"""tdmpc2_b200/trainer.py on the host: a recording fake agent, scripted environments and the real Buffer (add / load run
on the host; the fake agent's update never samples).  At E = 1 OnlineTrainer is held call for call to a restatement of
the reference's OnlineTrainer (written below from trainer/online_trainer.py); at E > 1 to the lock-step rules of its
docstring; OfflineTrainer to the log / eval / checkpoint iterations of trainer/offline_trainer.py."""
import pytest
import torch

from tdmpc2_b200.buffer import Buffer
from tdmpc2_b200.config import Config, make_cfg
from tdmpc2_b200.trainer import MemoryLogger, OfflineTrainer, OnlineTrainer, seed_steps, set_seed
from trainer_checks import normal, reference_online, same, stored

OBS_DIM, A, H = 4, 2, 3


class Recorder(list):
    """One call log shared by the agent and the environments of a run."""


class ToyEnv:
    """Reference-wrapper surface (envs/wrappers/tensor.py).  obs = (env id, episode, t, 1); episode e of environment k
    lasts 6 + (e + k) % 4 steps, or when `terminate` ends early at step 3 + (e % 3) of every second episode.  Rewards
    are multiples of 1/8, so fp32 and float64 sums agree exactly.  rand_act draws from the environment's own
    generator."""

    def __init__(self, rec, k=0, terminate=False, seed=0):
        self.rec, self.k, self.terminate = rec, k, terminate
        self.g = torch.Generator().manual_seed(100 + seed + k)
        self.episode, self.t = -1, 0
        self.actions = []

    def _obs(self):
        return torch.tensor([self.k, self.episode, self.t, 1.0], dtype=torch.float32)

    def reset(self, task_idx=None):
        self.rec.append(("reset", self.k))
        self.episode, self.t = self.episode + 1, 0
        self.length = 6 + (self.episode + self.k) % 4
        self.term_at = 3 + self.episode % 3 if self.terminate and self.episode % 2 == 1 else None
        return self._obs()

    def rand_act(self):
        a = torch.rand(A, generator=self.g) * 2 - 1
        self.rec.append(("rand_act", self.k, a.tolist()))
        return a

    def step(self, action):
        assert torch.is_tensor(action) and action.shape == (A,) and action.device.type == "cpu"
        self.rec.append(("step", self.k, action.tolist()))
        self.actions.append((self.episode, self.t, action.clone()))
        self.t += 1
        term = self.term_at is not None and self.t == self.term_at
        reward = torch.tensor(0.125 * ((self.t + self.episode + self.k) % 5) + 0.5 * float(action[0] > 0))
        info = {"terminated": torch.tensor(float(term)), "success": float(self.t % 2 == 0)}
        return self._obs(), reward, term or self.t >= self.length, info


class FakeAgent:
    """act() is a pure function of (obs, t0, eval_mode) and of a call counter it writes into _prev_mean; update()
    returns its own count.  Every call goes to the shared log in one normal form ([E, obs] rows, t0 per row) so that the
    reference's unbatched calls and the trainer's batched ones compare equal."""

    def __init__(self, rec, num_envs=1, cfg=None):
        self.rec, self.num_envs = rec, num_envs
        self.cfg = cfg_for(num_envs) if cfg is None else cfg          # evaluate() reads the task names
        self._prev_mean = torch.zeros(*(() if num_envs == 1 else (num_envs,)), H, A)
        self.updates, self.acts = 0, []
        self.saved = []

    def act(self, obs, t0=False, eval_mode=False, task=None):
        rows = obs.reshape(-1, OBS_DIM)
        t0s = [bool(x) for x in torch.as_tensor(t0).reshape(-1)]
        t0s = t0s * rows.shape[0] if len(t0s) == 1 else t0s
        entry = self._prev_mean.clone()
        self.rec.append(("act", rows.tolist(), t0s, bool(eval_mode)))
        a = torch.stack([torch.tensor([0.25 * r[1] - 0.5 + (1.0 if t else 0.0), 0.125 * r[2] - 0.25]) for r, t in zip(rows, t0s)])
        self._prev_mean.fill_(float(len(self.acts)))
        self.acts.append((bool(eval_mode), entry, self._prev_mean.clone(), rows.clone(), t0s))
        return a[0] if obs.ndim == 1 else a

    def update(self, buffer):
        self.updates += 1
        self.rec.append(("update",))
        return {"total_loss": torch.tensor(float(self.updates)), "grad_norm": torch.tensor(0.5)}

    def save(self, fp):
        self.saved.append(str(fp))
        torch.save({"model": {"n": torch.tensor(self.updates)}}, fp)


class RecordingBuffer(Buffer):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.added = []

    def add(self, td):
        self.added.append({k: v.clone() for k, v in td.items()})
        return super().add(td)


def cfg_for(E=1, **kw):
    kw.setdefault("steps", 60)
    kw.setdefault("eval_episodes", 2)
    return make_cfg(obs_dim=OBS_DIM, action_dim=A, model_size=None, task="toy", episode_length=9, num_envs=E,
                    horizon=H, **kw)


def first_length(terminate):
    env = ToyEnv(Recorder(), terminate=terminate)
    env.reset()
    return env.length


@pytest.mark.parametrize("seed_case,eval_freq,episodic", [
    ("below", 5, False), ("equal", 5, False), ("above", 5, False),
    ("equal", 10, False), ("above", 7, True), ("below", 4, True), ("above", 13, True),
])
def test_one_environment_matches_the_reference_call_for_call(seed_case, eval_freq, episodic):
    L = first_length(episodic)
    seed = {"below": L - 3, "equal": L, "above": L + 5}[seed_case]
    cfg = cfg_for(seed_steps=seed, eval_freq=eval_freq, episodic=episodic)
    runs = []
    for trainer in (False, True):
        rec = Recorder()
        env, agent, buf = ToyEnv(rec, terminate=episodic), FakeAgent(rec), RecordingBuffer(cfg)
        if trainer:
            logger = MemoryLogger()
            OnlineTrainer(cfg, [env], agent, buf, logger=logger).train()
            logs = normal(logger.logs)
        else:
            logs = normal(reference_online(cfg, env, agent, buf))
        runs.append((rec, logs, buf))
    (want_rec, want_logs, want_buf), (got_rec, got_logs, got_buf) = runs
    assert got_rec == want_rec                       # act (with t0, eval_mode) / rand_act / step / reset / update, in order
    assert got_logs == want_logs
    assert any(c == "eval" for c, _ in got_logs) and sum(c == "train" for c, _ in got_logs) >= 4
    if episodic:
        assert any(d["episode_terminated"] == 1.0 for c, d in got_logs if c == "train")
    assert len(got_buf.added) == len(want_buf.added) == got_buf.num_eps
    for g, w in zip(got_buf.added, want_buf.added):
        assert set(g) == set(w) and all(same(g[k], w[k]) for k in g)
        assert torch.isnan(g["action"][0]).all() and torch.isnan(g["reward"][0]) and torch.isnan(g["terminated"][0])
        assert not torch.isnan(g["action"][1:]).any() and not torch.isnan(g["reward"][1:]).any()
    assert got_buf._table == want_buf._table and got_buf._cursor == want_buf._cursor
    for g, w in zip(stored(got_buf), stored(want_buf)):
        assert all(same(g[k], w[k]) for k in g)


class EvalWatch(OnlineTrainer):
    """Records, at each evaluation, how many act calls came before it and which training slots were in mid-episode."""

    def eval(self):
        mid = [0 < env.t < (env.term_at or env.length) for env in self.envs]
        self.mid_at_eval = getattr(self, "mid_at_eval", []) + [(len(self.agent.acts), mid)]
        return super().eval()


def run_lockstep(E, seed=11, steps=70, eval_freq=9, episodic=True):
    cfg = cfg_for(E, seed_steps=seed, steps=steps, eval_freq=eval_freq, episodic=episodic)
    rec = Recorder()
    envs = [ToyEnv(rec, k, terminate=episodic and k % 2 == 0, seed=E) for k in range(E)]
    eval_envs = [ToyEnv(Recorder(), 50 + k) for k in range(E)]
    agent, buf, logger = FakeAgent(rec, E), RecordingBuffer(cfg), MemoryLogger()
    trainer = EvalWatch(cfg, envs, agent, buf, logger=logger, eval_envs=eval_envs)
    trainer.train()
    return trainer, rec, envs, agent, buf, logger


@pytest.mark.parametrize("E", [2, 3, 5])
def test_lockstep_invariants(E):
    seed, steps, eval_freq = 11, 70, 9
    trainer, rec, envs, agent, buf, logger = run_lockstep(E, seed, steps, eval_freq)
    K = steps // E + 1                                         # vector steps: the last one covers cfg.steps
    J = K * E
    assert sum(env.episode + 1 for env in envs) >= E + 2 and sum(len(env.actions) for env in envs) == J

    # every stored episode is one slot's whole episode, each slot's in order
    seen = {k: [] for k in range(E)}
    for ep in buf.added:
        o = ep["obs"]
        k, e = int(o[0, 0]), int(o[0, 1])
        assert (o[:, 0] == k).all() and (o[:, 1] == e).all()
        assert torch.equal(o[:, 2], torch.arange(o.shape[0], dtype=torch.float32))
        assert torch.isnan(ep["action"][0]).all() and torch.isnan(ep["reward"][0]) and torch.isnan(ep["terminated"][0])
        taken = [a for (ee, _, a) in envs[k].actions if ee == e]
        assert len(taken) == o.shape[0] - 1 and torch.equal(ep["action"][1:], torch.stack(taken))
        T = o.shape[0] - 1
        env = ToyEnv(Recorder(), k, terminate=envs[k].terminate)
        for _ in range(e + 1):
            env.reset()
        assert T == (env.term_at or env.length) and float(ep["terminated"][-1]) == float(env.term_at is not None)
        seen[k].append(e)
    for k in range(E):
        assert seen[k] == list(range(len(seen[k]))) and len(seen[k]) == envs[k].episode  # all but the running one

    # updates: the reference's count over the covered env steps
    assert agent.updates == sum(seed if j == seed else int(j > seed) for j in range(J))

    # act: one per vector step with a covered j > seed_steps, none while every slot seeds; t0 on first steps only
    train_acts = [a for a in agent.acts if not a[0]]
    assert len(train_acts) == sum(1 for k in range(K) if k * E + E - 1 > seed)
    steps_done = 0
    for entry in rec:
        if entry[0] == "step":
            steps_done += 1
        elif entry[0] == "act" and not entry[3]:
            assert steps_done % E == 0 and steps_done + E - 1 > seed, "act() while every slot was seeding"
    for _, _, _, rows, t0s in train_acts:
        assert t0s == [float(r[2]) == 0.0 for r in rows]
    # a slot that is seeding takes its own rand_act in that vector step: the env steps' actions tell them apart
    rand_steps = sum(1 for e in rec if e[0] == "rand_act") - sum(env.episode + 1 for env in envs)
    assert rand_steps == min(J, seed + 1)

    # evaluations: the flag rule, and the warm starts of the slots in mid-episode put back
    evals = [d for c, d in logger.logs if c == "eval"]
    assert len(evals) >= 2 and evals[0]["step"] == 0
    checked = 0
    for n, mid in trainer.mid_at_eval:
        before = [a for a in agent.acts[:n] if not a[0]]
        after = [a for a in agent.acts[n:] if not a[0]]
        assert any(a[0] for a in agent.acts[n:]), "the evaluation made no act"
        if not before or not after or not any(mid):
            continue
        for i in range(E):
            if mid[i]:
                assert torch.equal(after[0][1][i], before[-1][2][i]), "a slot in mid-episode lost its warm start"
                checked += 1
    assert checked >= 1


def test_errors():
    cfg = cfg_for(seed_steps=3, eval_freq=5)
    rec = Recorder()
    env = ToyEnv(rec, terminate=True)
    with pytest.raises(ValueError, match="episodic"):
        OnlineTrainer(cfg, [env], FakeAgent(rec), Buffer(cfg)).train()
    with pytest.raises(ValueError, match="num_envs"):
        OnlineTrainer(cfg, [ToyEnv(rec), ToyEnv(rec, 1)], FakeAgent(rec), Buffer(cfg))
    cfg2 = cfg_for(2, seed_steps=3, eval_freq=5)
    with pytest.raises(ValueError, match="eval_envs"):
        OnlineTrainer(cfg2, [ToyEnv(rec), ToyEnv(rec, 1)], FakeAgent(rec, 2), Buffer(cfg2))
    with pytest.raises(ValueError, match="eval_envs"):
        OnlineTrainer(cfg2, [ToyEnv(rec), ToyEnv(rec, 1)], FakeAgent(rec, 2), Buffer(cfg2), eval_envs=[ToyEnv(rec)])
    with pytest.raises(ValueError, match="multi-task"):
        OfflineTrainer(cfg, FakeAgent(rec), ["x.pt"], [ToyEnv(rec)])
    mt = mt_cfg()
    with pytest.raises(ValueError, match="single-task"):
        OnlineTrainer(mt, [ToyEnv(rec)], FakeAgent(rec), Buffer(mt))


def test_defaults_and_seed_steps_rule():
    cfg = Config()
    assert cfg.eval_episodes == 10 and cfg.eval_freq == 50_000 and cfg.seed_steps is None
    assert seed_steps(cfg_for()) == 1000                                  # max(1000, 5 * 9)
    assert seed_steps(cfg_for().replace(episode_length=500)) == 2500
    assert seed_steps(cfg_for(seed_steps=7)) == 7
    assert OnlineTrainer(cfg_for(), [ToyEnv(Recorder())], FakeAgent(Recorder()), None).seed_steps == 1000
    set_seed(5)
    a = torch.rand(3)
    set_seed(5)
    assert torch.equal(a, torch.rand(3))


# ------------------------------------------------------------------------------------------------ offline
class TaskEnv(ToyEnv):
    def reset(self, task_idx=None):
        assert task_idx is not None
        return super().reset()


def mt_cfg(**kw):
    kw.setdefault("task", "toy-mt")
    return make_cfg(obs_dim=OBS_DIM, action_dim=A, model_size=None, tasks=["a", "b"], episode_length=8,
                    horizon=H, num_envs=1, task_dim=4, **kw)


def write_data(path, n_eps, T, seed):
    g = torch.Generator().manual_seed(seed)
    torch.save({"obs": torch.randn(n_eps, T, OBS_DIM, generator=g), "action": torch.rand(n_eps, T, A, generator=g),
                "reward": torch.rand(n_eps, T, generator=g), "task": torch.randint(0, 2, (n_eps, T), generator=g),
                "episode": torch.zeros(n_eps, T, dtype=torch.int64)}, path)


def test_offline_log_eval_and_checkpoint_positions(tmp_path):
    cfg = mt_cfg(steps=25, eval_freq=10, eval_episodes=1, buffer_size=90)
    files = [tmp_path / "a.pt", tmp_path / "b.pt"]
    write_data(files[0], 3, 9, 1)
    write_data(files[1], 4, 9, 2)
    rec = Recorder()
    agent, logger = FakeAgent(rec, cfg=cfg), MemoryLogger(tmp_path / "ckpt")
    tr = OfflineTrainer(cfg, agent, files, [TaskEnv(Recorder())], logger=logger)
    with pytest.warns(UserWarning, match="7 episodes"):                 # 90 // 9 = 10 expected
        tr.train()
    assert tr.buffer.num_eps == 7 and tr.buffer.capacity == 90 and agent.updates == 25
    assert set(tr.buffer._storage) == {"obs", "action", "reward", "task"}
    logs = [(c, d) for c, d in logger.logs]
    assert [c for c, _ in logs] == ["pretrain"] * 3 and [d["iteration"] for _, d in logs] == [0, 10, 20]
    for _, d in logs:
        assert d["total_loss"].item() == d["iteration"] + 1                 # the update of that iteration
        assert {"episode_reward+a", "episode_success+a", "episode_reward+b", "episode_success+b"} <= set(d)
    updates_before_eval = []
    n = 0
    for e in rec:
        n += e[0] == "update"
        if e[0] == "act" and e[3] and (not updates_before_eval or updates_before_eval[-1] != n):
            updates_before_eval.append(n)
    assert updates_before_eval == [1, 11, 21]
    assert [p.rsplit("/", 1)[1] for p in agent.saved] == ["10.pt", "20.pt", "final.pt"]
    assert all((tmp_path / "ckpt" / f).exists() for f in ("10.pt", "20.pt", "final.pt"))


def test_offline_episode_length_is_checked(tmp_path):
    cfg = mt_cfg(steps=2, eval_freq=10, eval_episodes=1, buffer_size=90)
    write_data(tmp_path / "a.pt", 2, 9, 1)
    write_data(tmp_path / "b.pt", 2, 7, 2)
    tr = OfflineTrainer(cfg, FakeAgent(Recorder(), cfg=cfg), [tmp_path / "a.pt", tmp_path / "b.pt"], [TaskEnv(Recorder())])
    with pytest.raises(ValueError, match="7 rows"):
        tr.train()
    assert OfflineTrainer(mt_cfg(task="mt80"), FakeAgent(Recorder()), ["x"], [TaskEnv(Recorder())]).dataset_shape() \
        == (101, 550_450_000)
    assert OfflineTrainer(mt_cfg(task="mt30"), FakeAgent(Recorder()), ["x"], [TaskEnv(Recorder())]).dataset_shape() \
        == (501, 345_690_000)
