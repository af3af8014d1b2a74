"""Planning configuration for the H100 planner.

Restates the planning / architecture keys of the reference's Hydra config as a
plain attribute bag (hydra/omegaconf are not needed on the hot path):

  * planning block            -> reference tdmpc2/config.yaml:33-42
  * actor / critic constants  -> reference tdmpc2/config.yaml:44-52
  * architecture block        -> reference tdmpc2/config.yaml:54-64
  * model-size presets        -> reference tdmpc2/common/__init__.py:1-24
  * bin_size / task_dim rules -> reference tdmpc2/common/parser.py:59-77
  * discount heuristic        -> reference tdmpc2/tdmpc2.py:57-70

`Config` supports attribute access and `.get()` exactly like the dataclass the
reference builds in parser.py:12-26, so a reference-made cfg and this one are
interchangeable for `TDMPC2(cfg)`.

One new key exists: `num_envs` (E) -- the batch-of-environments axis this build
adds (the reference is E == 1, tdmpc2.py:111).
"""
from __future__ import annotations

import copy
from typing import Any, Dict, List, Optional

# reference tdmpc2/common/__init__.py:1-24 (restated, same numbers)
MODEL_SIZE: Dict[int, Dict[str, int]] = {
    1: dict(enc_dim=256, mlp_dim=384, latent_dim=128, num_enc_layers=2, num_q=2),
    5: dict(enc_dim=256, mlp_dim=512, latent_dim=512, num_enc_layers=2),
    19: dict(enc_dim=1024, mlp_dim=1024, latent_dim=768, num_enc_layers=3),
    48: dict(enc_dim=1792, mlp_dim=1792, latent_dim=768, num_enc_layers=4),
    317: dict(enc_dim=4096, mlp_dim=4096, latent_dim=1376, num_enc_layers=5, num_q=8),
}

_DEFAULTS: Dict[str, Any] = dict(
    # environment
    task="dog-run", obs="state", episodic=False,
    # planning (config.yaml:33-42)
    mpc=True, iterations=6, num_samples=512, num_elites=64, num_pi_trajs=24,
    horizon=3, min_std=0.05, max_std=2.0, temperature=0.5,
    # actor (config.yaml:44-47)
    log_std_min=-10.0, log_std_max=2.0, entropy_coef=1e-4,
    # critic (config.yaml:49-52)
    num_bins=101, vmin=-10.0, vmax=10.0,
    # architecture (config.yaml:54-64)
    model_size=None, num_enc_layers=2, enc_dim=256, num_channels=32, mlp_dim=512,
    latent_dim=512, task_dim=0, num_q=5, dropout=0.01, simnorm_dim=8,
    # discount heuristic (config.yaml:28-30)
    discount_denom=5, discount_min=0.95, discount_max=0.995,
    # training keys (config.yaml:10-22), read by agent._update / agent.update_pi
    reward_coef=0.1, value_coef=0.1, termination_coef=1, consistency_coef=20,
    lr=3e-4, enc_lr_scale=0.3, tau=0.01, rho=0.5, grad_clip_norm=20, batch_size=256, seed=1, compile=False,
    # filled in by make_cfg
    multitask=False, tasks=None, obs_shape=None, action_dim=None, action_dims=None,
    episode_length=None, episode_lengths=None, bin_size=None,
    # new in this build
    num_envs=1,
)


class Config:
    """Attribute bag with `.get()`; mirrors parser.py:12-26's dataclass surface."""

    def __init__(self, **kw: Any) -> None:
        d = copy.deepcopy(_DEFAULTS)
        d.update(kw)
        self.__dict__.update(d)

    def get(self, key: str, default: Any = None) -> Any:
        return getattr(self, key, default)

    def to_dict(self) -> Dict[str, Any]:
        return copy.deepcopy(self.__dict__)

    def replace(self, **kw: Any) -> "Config":
        d = self.to_dict()
        d.update(kw)
        return Config(**d)

    def __repr__(self) -> str:  # pragma: no cover - debugging aid
        keys = ("task", "model_size", "num_envs", "num_samples", "horizon", "iterations",
                "latent_dim", "mlp_dim", "action_dim", "task_dim", "num_q")
        return "Config(" + ", ".join(f"{k}={self.__dict__.get(k)!r}" for k in keys) + ")"


def get_discount(cfg: Config, episode_length: int) -> float:
    """reference tdmpc2/tdmpc2.py:57-70."""
    frac = episode_length / cfg.discount_denom
    return min(max((frac - 1) / frac, cfg.discount_min), cfg.discount_max)


def make_cfg(*, obs_dim: int = 0, action_dim: int, model_size: Optional[int] = 5,
             episode_length: int = 500, tasks: Optional[List[str]] = None,
             action_dims: Optional[List[int]] = None,
             episode_lengths: Optional[List[int]] = None,
             task_dim: Optional[int] = None, **overrides: Any) -> Config:
    """Build a Config the way parser.py:29-80 + envs/__init__.py:76-82 would.

    Single-task when `tasks` is None; multi-task otherwise (task_dim defaults to
    96, parser.py:75).  `overrides` win over the model-size preset, like Hydra
    command-line overrides do in the reference.
    """
    kw: Dict[str, Any] = {}
    if model_size is not None:
        assert model_size in MODEL_SIZE, f"Invalid model size {model_size}"
        kw.update(MODEL_SIZE[model_size])
    kw["model_size"] = model_size
    multitask = tasks is not None
    kw["multitask"] = multitask
    if multitask:
        kw["tasks"] = list(tasks)
        kw["task_dim"] = 96 if task_dim is None else task_dim
        kw["action_dims"] = list(action_dims) if action_dims is not None else [action_dim] * len(tasks)
        kw["episode_lengths"] = (list(episode_lengths) if episode_lengths is not None
                                 else [episode_length] * len(tasks))
        assert len(kw["action_dims"]) == len(tasks) == len(kw["episode_lengths"])
    else:
        kw["tasks"] = [overrides.get("task", "dog-run")]
        kw["task_dim"] = 0
    if overrides.get("obs", "state") == "rgb":       # envs/dmcontrol.py:108: 64 x 64 frames, 3 channels x frame stack
        kw["obs_shape"] = {"rgb": (int(overrides.pop("obs_channels", 9)), 64, 64)}
    else:
        kw["obs_shape"] = {"state": (obs_dim,)}
    kw["action_dim"] = action_dim
    kw["episode_length"] = episode_length
    kw.update(overrides)
    cfg = Config(**kw)
    cfg.bin_size = (cfg.vmax - cfg.vmin) / (cfg.num_bins - 1)  # parser.py:59
    return cfg


def _mt80_tasks() -> Dict[str, Any]:
    # SURVEY.md section 8(d): 80 tasks; tasks 0-29 are DMControl-like (6 action
    # dims, 500-step episodes -> gamma 0.99), 30-79 Meta-World-like (4 dims,
    # 100-step episodes -> gamma 0.95).
    tasks = [f"task-{i}" for i in range(80)]
    action_dims = [6] * 30 + [4] * 50
    episode_lengths = [500] * 30 + [100] * 50
    return dict(tasks=tasks, action_dims=action_dims, episode_lengths=episode_lengths)


def workload(name: str, **overrides: Any) -> Config:
    """The five BASELINE.json configurations as concrete synthetic workloads
    (SURVEY.md section 8(d)); `iterations` is the effective loop count."""
    if name in ("c1", "c2"):
        kw = dict(obs_dim=223, action_dim=38, model_size=5, task="dog-run",
                  num_envs=1 if name == "c1" else 256,
                  num_samples=512, horizon=3, iterations=6)
    elif name == "c3":
        kw = dict(obs_dim=67, action_dim=21, model_size=48, task="humanoid-walk",
                  num_envs=1024, num_samples=512, horizon=5, iterations=8)
    elif name in ("c4", "c5"):
        kw = dict(obs_dim=39, action_dim=6, model_size=317, task="mt80", **_mt80_tasks(),
                  num_envs=2048 if name == "c4" else 4096,
                  num_samples=512 if name == "c4" else 1024,
                  horizon=3 if name == "c4" else 8,
                  iterations=6 if name == "c4" else 10)
    elif name == "tiny":  # test-sized single-task model (not a BASELINE config)
        kw = dict(obs_dim=17, action_dim=6, model_size=None, task="tiny",
                  enc_dim=64, mlp_dim=64, latent_dim=64, num_enc_layers=2, num_q=3,
                  num_envs=2, num_samples=128, num_elites=16, num_pi_trajs=8,
                  horizon=3, iterations=3)
    elif name == "tiny-wide":  # test-sized model whose hidden layers are wider than 512 (640 columns)
        kw = dict(obs_dim=19, action_dim=7, model_size=None, task="tiny-wide",
                  enc_dim=96, mlp_dim=640, latent_dim=64, num_enc_layers=2, num_q=3,
                  num_envs=2, num_samples=128, num_elites=16, num_pi_trajs=8,
                  horizon=2, iterations=2)
    elif name == "tiny-wide2":  # wide hidden (2 full super-chunks + 128), wide SimNorm latent, wide encoder; 2 tiles per env
        kw = dict(obs_dim=19, action_dim=7, model_size=None, task="tiny-wide2",
                  enc_dim=640, mlp_dim=1152, latent_dim=576, num_enc_layers=2, num_q=2,
                  num_envs=2, num_samples=256, num_elites=16, num_pi_trajs=8,
                  horizon=2, iterations=2)
    elif name == "tiny-rgb":  # test-sized pixel-observation model: layers.conv encoder, latent = 16 * num_channels
        kw = dict(obs="rgb", obs_channels=6, action_dim=4, model_size=None, task="tiny-rgb",
                  num_channels=8, enc_dim=64, mlp_dim=128, latent_dim=128, num_enc_layers=2, num_q=3,
                  num_envs=2, num_samples=128, num_elites=16, num_pi_trajs=8,
                  horizon=3, iterations=3)
    elif name == "tiny-mt":  # test-sized multi-task model
        kw = dict(obs_dim=11, action_dim=5, model_size=None, task="tiny-mt",
                  tasks=[f"t{i}" for i in range(4)], action_dims=[5, 3, 4, 2],
                  episode_lengths=[500, 100, 500, 100], task_dim=16,
                  enc_dim=64, mlp_dim=96, latent_dim=64, num_enc_layers=3, num_q=4,
                  num_envs=3, num_samples=128, num_elites=16, num_pi_trajs=8,
                  horizon=4, iterations=3)
    else:
        raise KeyError(f"unknown workload {name!r}")
    kw.update(overrides)
    return make_cfg(**kw)


def flops_per_env(cfg: Config, heads_used: int = 2) -> float:
    """Algorithmic GEMM FLOPs of one plan() call for ONE environment
    (SURVEY.md section 8(d); 2 FLOP per MAC, only `heads_used` Q heads)."""
    L, M, A, T, B = cfg.latent_dim, cfg.mlp_dim, cfg.action_dim, cfg.task_dim, cfg.num_bins
    D = L + T + A
    w = lambda i, h, o: i * h + h * h + h * o
    dyn, rew, pi, q = w(D, M, L), w(D, M, B), w(L + T, M, 2 * A), w(D, M, B)
    H, N, P, I = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.iterations
    term = w(L + T, M, 1) if cfg.episodic else 0          # termination head on z_{t+1} (world_model.py:28)
    macs = I * N * (H * (rew + dyn + term) + pi + heads_used * q) + P * (H * pi + (H - 1) * dyn)
    enc_in = cfg.obs_shape["state"][0] + T
    n_hidden = max(cfg.num_enc_layers - 1, 1)
    enc = enc_in * cfg.enc_dim + (n_hidden - 1) * cfg.enc_dim ** 2 + cfg.enc_dim * L
    return 2.0 * (macs + enc)
