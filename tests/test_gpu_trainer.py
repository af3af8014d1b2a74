"""OnlineTrainer / OfflineTrainer on the H100 kernels (tiny presets, seeded generators): bit-identical to a restated
reference loop on a twin agent at E = 1 and offline, whole episodes and warm starts kept at E = 4 in lock-step, uint8
frames through a pixel model, and a tiny agent that learns a toy reach task."""
import math

import pytest
import torch

from tdmpc2_b200.buffer import Buffer
from tdmpc2_b200.config import workload
from tdmpc2_b200.evaluate import evaluate
from tdmpc2_b200.tdmpc2 import TDMPC2
from tdmpc2_b200.trainer import MemoryLogger, OfflineTrainer, OnlineTrainer, set_seed
from trainer_checks import normal, reference_online, same, stored

pytestmark = pytest.mark.gpu
DEV = "cuda"


class ReachEnv:
    """Toy reach task: obs = (position, target) in [-1, 1]^2 each; the action moves the position by 0.2 * action
    (clipped to the box); reward = 1 - mean |position - target|; `length`-step episodes.  With `terminate`, an episode
    ends early, terminated, once the position is within 0.05 of the target after step 5 (episodic models).  Start,
    target and rand_act come from the environment's own generator."""

    def __init__(self, seed, length=50, terminate=False, A=2, obs_dim=4):
        self.g = torch.Generator().manual_seed(seed)
        self.length, self.terminate, self.A, self.obs_dim = length, terminate, A, obs_dim
        self.t = 0

    def _obs(self):
        o = torch.zeros(self.obs_dim)
        o[:4] = torch.cat([self.pos, self.target])
        return o

    def reset(self, task_idx=None):
        self.pos = torch.rand(2, generator=self.g) * 2 - 1
        self.target = torch.rand(2, generator=self.g) * 2 - 1
        self.t, self.done = 0, False
        return self._obs()

    def rand_act(self):
        return torch.rand(self.A, generator=self.g) * 2 - 1

    def step(self, action):
        a = torch.as_tensor(action, dtype=torch.float32).reshape(-1)[:2]
        self.pos = (self.pos + 0.2 * a.clamp(-1, 1)).clamp(-1, 1)
        self.t += 1
        dist = (self.pos - self.target).abs().mean()
        term = self.terminate and self.t > 5 and float(dist) < 0.05
        self.done = term or self.t >= self.length
        info = {"terminated": torch.tensor(float(term)), "success": float(float(dist) < 0.05)}
        return self._obs(), (1 - dist).to(torch.float32), self.done, info


class PixelReachEnv(ReachEnv):
    """ReachEnv rendered as uint8 [6, 64, 64] frames: channels 0-2 mark the position with an 8 x 8 square, channels
    3-5 the target."""

    def __init__(self, seed, length=10, A=4):
        super().__init__(seed, length=length, A=A)

    def _obs(self):
        f = torch.full((6, 64, 64), 20, dtype=torch.uint8)
        for c, p in ((0, self.pos), (3, self.target)):
            x, y = (((p + 1) / 2) * 56).long().tolist()
            f[c:c + 3, y:y + 8, x:x + 8] = 235
        return f


def make_agent(cfg, seed, gen_seed):
    set_seed(seed)                                   # the world model's initial weights come from torch's global RNG
    agent = TDMPC2(cfg, device=DEV)
    agent.generator = torch.Generator(DEV).manual_seed(gen_seed)
    return agent


def make_buffer(cfg, seed):
    buf = Buffer(cfg)
    buf.generator = torch.Generator(DEV).manual_seed(seed)
    return buf


def tensors_equal(a, b, path=""):
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and same(a, b), path
    elif isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            tensors_equal(a[k], b[k], f"{path}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            tensors_equal(x, y, f"{path}[{i}]")
    else:
        assert a == b, path


def assert_twins(a, b):
    tensors_equal(a.model.state_dict(), b.model.state_dict(), "model")
    tensors_equal(a.optim.state_dict(), b.optim.state_dict(), "optim")
    tensors_equal(a.pi_optim.state_dict(), b.pi_optim.state_dict(), "pi_optim")
    assert same(a.scale.value, b.scale.value)
    assert same(a._prev_mean, b._prev_mean)


def losses(logs):
    return [(c, {k: v for k, v in d.items() if torch.is_tensor(v) and v.device.type == "cuda"}) for c, d in logs]


def test_twin_at_one_environment():
    """OnlineTrainer and the restated reference loop make the same calls with the same draws through real planning,
    updates and evaluations: every weight, optimiser moment, the Q scale, the buffer and the logged losses agree bit
    for bit."""
    cfg = workload("tiny", obs_dim=4, action_dim=2, num_envs=1, batch_size=64, episode_length=20, seed_steps=40,
                   steps=100, eval_freq=50, eval_episodes=2)
    logs, agents, bufs = [], [], []
    for trainer in (True, False):
        agent, buf, env = make_agent(cfg, 1, 2), make_buffer(cfg, 3), ReachEnv(4, length=20)
        if trainer:
            logger = MemoryLogger()
            OnlineTrainer(cfg, [env], agent, buf, logger=logger).train()
            logs.append(logger.logs)
        else:
            logs.append(reference_online(cfg, env, agent, buf))
        agents.append(agent)
        bufs.append(buf)
    got, want = logs
    assert [c for c, _ in got] == [c for c, _ in want] and sum(c == "eval" for c, _ in got) == 3
    lg, lw = losses(got), losses(want)
    assert any(d for _, d in lg) and all("total_loss" in d for c, d in lg[-3:] if c == "train")
    for (_, dg), (_, dw) in zip(lg, lw):
        tensors_equal(dg, dw, "losses")
    for (c, dg), (_, dw) in zip(normal(got), normal(want)):
        for k in dw:
            assert dg[k] == pytest.approx(dw[k], rel=1e-6, abs=1e-6), (c, k)
    assert_twins(*agents)
    assert bufs[0]._table == bufs[1]._table and bufs[0].num_eps == bufs[1].num_eps == 5
    for g, w in zip(stored(bufs[0]), stored(bufs[1])):
        assert all(same(g[k].cpu(), w[k].cpu()) for k in g)


class WatchedTrainer(OnlineTrainer):
    """At every evaluation, records agent._prev_mean and which training slots are in mid-episode; the next training
    act() checks that those slots' warm starts came back bit for bit."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.watched, self.pending = [], None
        act = self.agent.act

        def watched_act(obs, t0=False, eval_mode=False, task=None):
            if not eval_mode and self.pending is not None:
                before, mid = self.pending
                for i in range(len(mid)):
                    if mid[i]:
                        assert same(self.agent._prev_mean[i], before[i]), "a slot in mid-episode lost its warm start"
                self.watched.append((mid, bool(before.abs().sum() > 0)))
                self.pending = None
            return act(obs, t0=t0, eval_mode=eval_mode, task=task)
        self.agent.act = watched_act

    def eval(self):
        mid = [0 < env.t < env.length and not env.done for env in self.envs]
        self.pending = (self.agent._prev_mean.clone(), mid)
        return super().eval()


def test_lockstep_four_environments():
    E = 4
    cfg = workload("tiny", obs_dim=4, action_dim=2, num_envs=E, batch_size=64, episodic=True, seed_steps=60,
                   steps=240, eval_freq=100, eval_episodes=2, episode_length=30)
    agent, buf = make_agent(cfg, 5, 6), make_buffer(cfg, 7)
    envs = [ReachEnv(10 + k, length=15 + 4 * k, terminate=True) for k in range(E)]
    eval_envs = [ReachEnv(20 + k, length=12) for k in range(E)]
    logger = MemoryLogger()
    tr = WatchedTrainer(cfg, envs, agent, buf, logger=logger, eval_envs=eval_envs)
    tr.train()
    # an evaluation after acting began, with some slot in mid-episode
    assert any(any(mid) and acted for mid, acted in tr.watched)
    # whole episodes: every trajectory the buffer holds is a logged episode, reset row first (the oldest may have lost
    # its head to the storage's wrap)
    train = [d for c, d in logger.logs if c == "train"]
    st, lengths = stored(buf), [n for _, n in buf._table]
    assert buf.num_eps == len(train) >= 8
    assert lengths[1:] == [int(d["episode_length"]) for d in train][-(len(lengths) - 1):]
    for ep in st[1:]:
        a, r, term = ep["action"].cpu(), ep["reward"].cpu(), ep["terminated"].cpu()
        assert torch.isnan(a[0]).all() and torch.isnan(r[0]) and torch.isnan(term[0])
        assert not torch.isnan(a[1:]).any() and not torch.isnan(r[1:]).any() and not torch.isnan(term[1:]).any()
        assert (term[1:-1] == 0).all()
    for d in train:                                  # an episode ends at its environment's length or terminated
        assert float(d["episode_terminated"]) == 1.0 or int(d["episode_length"]) - 1 in {15, 19, 23, 27}
    finite = [float(v) for d in train for k, v in d.items() if k.endswith("loss")]
    assert finite and all(math.isfinite(x) for x in finite)


@pytest.mark.parametrize("E", [1, 2])
def test_pixel_model_trains_on_uint8_frames(E):
    cfg = workload("tiny-rgb", num_envs=E, batch_size=32, episode_length=10, seed_steps=20, steps=40, eval_freq=1000,
                   eval_episodes=1)
    agent, buf = make_agent(cfg, 8, 9), make_buffer(cfg, 10)
    envs = [PixelReachEnv(30 + k) for k in range(E)]
    logger = MemoryLogger()
    OnlineTrainer(cfg, envs, agent, buf, logger=logger,
                  eval_envs=None if E == 1 else [PixelReachEnv(40 + k) for k in range(E)]).train()
    assert buf._storage["obs"].dtype == torch.uint8 and tuple(buf._storage["obs"].shape[1:]) == (6, 64, 64)
    assert buf.num_eps >= 3
    row = stored(buf)[0]["obs"][1].cpu()
    assert row.max() == 235 and row.min() == 20
    train = [d for c, d in logger.logs if c == "train" and "total_loss" in d]
    assert train and all(math.isfinite(float(v)) for d in train for k, v in d.items() if k.endswith("loss"))


def random_reward(episodes=20, seed=99):
    env = ReachEnv(seed)
    total = 0.0
    for _ in range(episodes):
        env.reset()
        done = False
        while not done:
            _, r, done, _ = env.step(env.rand_act())
            total += float(r)
    return total / episodes


def test_tiny_agent_learns_to_reach():
    """About 1,000 env steps of online training on the reach task; the final evaluation (10 episodes, eval mode) must
    beat random actions by a margin."""
    cfg = workload("tiny", obs_dim=4, action_dim=2, num_envs=1, episode_length=50, seed_steps=200, steps=1000,
                   eval_freq=1000, eval_episodes=10)
    agent, buf = make_agent(cfg, 11, 12), make_buffer(cfg, 13)
    logger = MemoryLogger()
    OnlineTrainer(cfg, [ReachEnv(14)], agent, buf, logger=logger, eval_envs=[ReachEnv(15)]).train()
    evals = [d for c, d in logger.logs if c == "eval"]
    assert [d["step"] for d in evals] == [0, 1000]
    rand = random_reward()
    print(f"reach: random {rand:.2f}, eval at step 0 {evals[0]['episode_reward']:.2f}, "
          f"after 1000 steps {evals[-1]['episode_reward']:.2f}")
    # H100 80GB HBM3 (700 W): random 13.49, untrained agent 18.62, after 1,000 steps 38.80 per 50-step episode
    assert evals[-1]["episode_reward"] > rand + 15.0


def write_dataset(path, cfg, n_eps, T, seed):
    g = torch.Generator().manual_seed(seed)
    task = torch.randint(0, len(cfg.tasks), (n_eps,), generator=g)
    mask = torch.zeros(n_eps, cfg.action_dim)
    for i, t in enumerate(task.tolist()):
        mask[i, :cfg.action_dims[t]] = 1
    action = (torch.rand(n_eps, T, cfg.action_dim, generator=g) * 2 - 1) * mask[:, None]
    action[:, 0] = float("nan")
    reward = torch.rand(n_eps, T, generator=g)
    reward[:, 0] = float("nan")
    obs = torch.randn(n_eps, T, cfg.obs_shape["state"][0], generator=g)
    torch.save({"obs": obs, "action": action, "reward": reward, "task": task[:, None].expand(n_eps, T).clone()}, path)


class TaskReachEnv(ReachEnv):
    def __init__(self, seed, cfg):
        super().__init__(seed, length=8, A=cfg.action_dim, obs_dim=cfg.obs_shape["state"][0])

    def reset(self, task_idx=None):
        assert task_idx is not None
        return super().reset()


def test_offline_twin(tmp_path):
    cfg = workload("tiny-mt", num_envs=2, batch_size=32, episode_length=20, buffer_size=400, steps=25, eval_freq=10,
                   eval_episodes=1)
    files = [tmp_path / "d0.pt", tmp_path / "d1.pt"]
    write_dataset(files[0], cfg, 6, 21, 1)
    write_dataset(files[1], cfg, 5, 21, 2)

    agent = make_agent(cfg, 21, 22)
    set_seed(23)                                     # the trainer's buffer draws from torch's default CUDA generator
    logger = MemoryLogger(tmp_path / "ckpt")
    tr = OfflineTrainer(cfg, agent, files, [TaskReachEnv(24 + k, cfg) for k in range(2)], logger=logger)
    with pytest.warns(UserWarning, match="11 episodes"):
        tr.train()

    twin = make_agent(cfg, 21, 22)
    set_seed(23)
    buf = Buffer(cfg.replace(episode_length=21, buffer_size=400, steps=400))
    for f in files:
        buf.load(torch.load(f, weights_only=True))
    eval_envs = [TaskReachEnv(24 + k, cfg) for k in range(2)]
    snapshots, want = {}, []
    for i in range(cfg.steps):
        info = twin.update(buf)
        if i % cfg.eval_freq == 0:
            want.append((i, info, evaluate(twin, eval_envs, cfg.eval_episodes, eval_mode=True)))
            if i > 0:
                snapshots[i] = {k: v.clone() if torch.is_tensor(v) else v for k, v in twin.model.state_dict().items()}
    assert_twins(agent, twin)
    assert tr.buffer._table == buf._table
    for g, w in zip(stored(tr.buffer), stored(buf)):
        assert all(same(g[k].cpu(), w[k].cpu()) for k in g)
    got = logger.logs
    assert [(c, d["iteration"]) for c, d in got] == [("pretrain", 0), ("pretrain", 10), ("pretrain", 20)]
    for (_, d), (i, info, ev) in zip(got, want):
        for k, v in info.items():
            assert same(d[k], v), (i, k)
        for name, r in ev["tasks"].items():
            assert d[f"episode_reward+{name}"] == r.reward and d[f"episode_success+{name}"] == r.success
    for i in (10, 20):
        fp = tmp_path / "ckpt" / f"{i}.pt"
        assert fp.exists()
        loaded = TDMPC2(cfg, device=DEV)
        loaded.load(str(fp))
        tensors_equal(loaded.model.state_dict(), snapshots[i], f"checkpoint {i}")
    assert (tmp_path / "ckpt" / "final.pt").exists()
