"""The vectorised evaluation loop driving the real planner: E toy environments in lock-step, one batched act() per step
(CUDA-graph replay), slots out of phase with per-slot t0.  Run on an H100: pytest -m gpu."""
from collections import defaultdict

import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.evaluate import evaluate
from tdmpc2_b200.synth import synth_state_dict

pytestmark = pytest.mark.gpu


class ToyEnv:
    """Stable linear system; reward = -|x|^2-ish; episode length depends on the instance so that slots desynchronise."""

    def __init__(self, obs_dim, action_dim, length, seed):
        g = torch.Generator().manual_seed(seed)
        self.A = 0.9 * torch.eye(obs_dim) + 0.02 * torch.randn(obs_dim, obs_dim, generator=g)
        self.B = 0.1 * torch.randn(obs_dim, action_dim, generator=g)
        self.g, self.length, self.action_dim = g, length, action_dim

    def reset(self, task_idx=None):
        self.task, self.t = task_idx, 0
        self.x = torch.randn(self.A.shape[0], generator=self.g)
        return self.x.clone()

    def step(self, action):
        assert action.shape == (self.action_dim,) and action.device.type == "cpu"
        assert bool(torch.isfinite(action).all()) and float(action.abs().max()) <= 1.0          # tdmpc2.py:204 clamp
        self.x = self.A @ self.x + self.B @ action
        self.t += 1
        info = defaultdict(float, success=float(self.x.norm() < 3.0))
        return self.x.clone(), torch.tensor(-float(self.x.square().mean())), self.t >= self.length, info


@pytest.mark.parametrize("wl", ["tiny", "tiny-mt"])
def test_batched_evaluation_runs_the_planner(wl):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    E, episodes = 4, 3
    cfg = workload(wl, num_envs=E)
    agent = TDMPC2(cfg, device="cuda:0")
    agent.load(synth_state_dict(cfg, seed=21, perturb=True))
    agent.generator = torch.Generator(device="cuda").manual_seed(5)
    envs = [ToyEnv(cfg.obs_shape["state"][0], cfg.action_dim, 3 + i, 100 + i) for i in range(E)]
    out = evaluate(agent, envs, episodes)
    names = list(cfg.tasks) if cfg.multitask else [cfg.task]
    assert sorted(out["tasks"]) == sorted(names)
    for name in names:
        r = out["tasks"][name]
        assert len(r.episode_rewards) == episodes and all(3 <= n <= 3 + E - 1 for n in r.episode_lengths)
        assert all(x == x and x < 0 for x in r.episode_rewards) and 0.0 <= r.success <= 1.0
    assert out["env_steps"] == sum(sum(r.episode_lengths) for r in out["tasks"].values())
    assert out["act_calls"] < out["env_steps"]
    assert (out["normalized_score"] is None) == (not cfg.multitask)
    if cfg.multitask:                       # masked action dimensions of each task stay zero through the loop's routing
        a = agent.act(torch.randn(E, cfg.obs_shape["state"][0]), t0=True, task=torch.tensor([1, 3, 0, 2]))
        for e, t in enumerate([1, 3, 0, 2]):
            assert bool((a[e, cfg.action_dims[t]:] == 0).all())
