"""CPU oracle for the TD-MPC2 planning hot path -- TEST INFRASTRUCTURE ONLY.

This file is the parity checker, never the product: only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs may import it.  The shipped path (`tdmpc2_b200`) never imports `oracle/`.

It restates, in plain fp32 PyTorch-on-CPU, the algorithm of the reference
(nicklashansen/tdmpc2 @ e9f5932), with every random draw made explicit:

  plan_oracle        <- TDMPC2._plan              tdmpc2/tdmpc2.py:138-206
  estimate_value     <- TDMPC2._estimate_value    tdmpc2/tdmpc2.py:122-136
  OracleModel.encode <- WorldModel.encode         common/world_model.py:103-112  (obs 'rgb': layers.conv / ShiftAug /
                                                  PixelPreprocess, common/layers.py:36-71,136-150)
  OracleModel.task_emb <- WorldModel.task_emb     common/world_model.py:88-101  (nn.Embedding max_norm=1, :21)
  OracleModel.next   <- WorldModel.next           common/world_model.py:114-121
  OracleModel.reward <- WorldModel.reward         common/world_model.py:123-130
  OracleModel.pi     <- WorldModel.pi             common/world_model.py:144-184 (only `action` is used by the planner)
  OracleModel.Q      <- WorldModel.Q('avg')       common/world_model.py:186-216
  _mlp               <- layers.mlp/NormedLinear/SimNorm  common/layers.py:74-133
  two_hot_inv/symexp <- common/math.py:50-55,74-83
  log_std            <- common/math.py:12-13
  gumbel pick        <- math.gumbel_softmax_sample common/math.py:86-94

Third-party arithmetic: torch (reference pins torch==2.7.1 in
docker/environment.yaml:11; this image has 2.11 -- the ops used are stable).

Pinning: the reference ships NO tests or golden vectors (SURVEY.md section 4),
so the pins are minted here: `oracle/ref_harness.py` executes the reference's
own unmodified `_plan` on CPU (only possible where /root/reference exists) and
`oracle/make_golden.py` records its outputs under tests/golden/.
`tests/test_oracle_golden.py` checks this restatement against those fixtures.

The env-batched semantics (new in this build; the reference is E == 1): every
environment is an independent reference `_plan` call with its own obs, task,
t0 flag, `_prev_mean`, and noise stream.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- noise
@dataclass
class PlanNoise:
    """Every random number one batched plan() consumes, in reference draw order
    (SURVEY.md section 8(a), 'RNG draw order per _plan call').

    prior : [E, H, P, A]      randn_like in pi() for the P policy-prior trajectories   (world_model.py:156 via tdmpc2.py:158,160)
    r     : [E, I, H, N-P, A] randn for the sampled action sequences                   (tdmpc2.py:176)
    pi    : [E, I, N, A]      randn_like in the terminal pi()                          (world_model.py:156 via tdmpc2.py:135)
    qidx  : [E, I, 2] int64   randperm(num_q)[:2]                                      (world_model.py:212)
    expo  : [E, K]            exponential_() draws of the gumbel pick                  (math.py:90)
    final : [E, A]            randn added to the chosen action when not eval_mode      (tdmpc2.py:204)
    """
    prior: torch.Tensor
    r: torch.Tensor
    pi: torch.Tensor
    qidx: torch.Tensor
    expo: torch.Tensor
    final: torch.Tensor
    shift: Optional[torch.Tensor] = None   # [E, 2] pixel models only: ShiftAug's randint(0, 7) (x, y), layers.py:55 -- the FIRST draw

    def to(self, device) -> "PlanNoise":
        return PlanNoise(*(getattr(self, f).to(device) for f in ("prior", "r", "pi", "qidx", "expo", "final")),
                         None if self.shift is None else self.shift.to(device))

    def env(self, e: int) -> "PlanNoise":
        return PlanNoise(*(getattr(self, f)[e:e + 1] for f in ("prior", "r", "pi", "qidx", "expo", "final")),
                         None if self.shift is None else self.shift[e:e + 1])


def draw_noise(cfg, seed: int, num_envs: int, eval_mode: bool = False) -> PlanNoise:
    """Draw noise exactly as `num_envs` independent reference calls would, env e
    seeded with `seed + e` (CPU generator; identical stream to
    torch.manual_seed(seed + e) followed by the reference's own draws)."""
    H, N, P, A, I, K = (cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim,
                        cfg.iterations, cfg.num_elites)
    out: Dict[str, List[torch.Tensor]] = {k: [] for k in ("prior", "r", "pi", "qidx", "expo", "final")}
    rgb = cfg.get("obs", "state") == "rgb"
    shifts = []
    for e in range(num_envs):
        g = torch.Generator(device="cpu").manual_seed(seed + e)
        if rgb:      # ShiftAug.forward inside encode() (layers.py:55): same call, same dtype, n = 1
            shifts.append(torch.randint(0, 2 * 3 + 1, size=(1, 1, 1, 2), dtype=torch.float32, generator=g).view(2))
        prior = torch.zeros(H, P, A)
        if P > 0:
            for t in range(H):                       # H-1 loop draws + the final pi() (tdmpc2.py:157-160)
                prior[t] = torch.randn(P, A, generator=g)
        r, pi, qidx = [], [], []
        for _ in range(I):
            r.append(torch.randn(H, N - P, A, generator=g))
            pi.append(torch.randn(N, A, generator=g))
            qidx.append(torch.randperm(cfg.num_q, generator=g)[:2])
        expo = torch.empty(K).exponential_(generator=g)
        final = torch.zeros(A) if eval_mode else torch.randn(A, generator=g)
        for k, v in (("prior", prior), ("r", torch.stack(r)), ("pi", torch.stack(pi)),
                     ("qidx", torch.stack(qidx)), ("expo", expo), ("final", final)):
            out[k].append(v)
    return PlanNoise(**{k: torch.stack(v) for k, v in out.items()}, shift=torch.stack(shifts) if rgb else None)


# --------------------------------------------------------------------------- model
def symexp(x: torch.Tensor) -> torch.Tensor:
    return torch.sign(x) * (torch.exp(torch.abs(x)) - 1)           # math.py:50-55


def two_hot_inv(x: torch.Tensor, cfg) -> torch.Tensor:
    if cfg.num_bins == 0:
        return x
    if cfg.num_bins == 1:
        return symexp(x)
    bins = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, dtype=x.dtype)   # math.py:80
    x = F.softmax(x, dim=-1)
    x = torch.sum(x * bins, dim=-1, keepdim=True)
    return symexp(x)


class OracleModel:
    """Functional restatement of the reference WorldModel's planning methods."""

    def __init__(self, cfg, sd: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float32):
        """dtype: fp32 (the reference's arithmetic) or torch.float64 (an error yardstick for fp32 results)."""
        self.cfg = cfg
        self.dtype = dtype
        self.sd = {k: (v.detach().to(dtype).cpu() if isinstance(v, torch.Tensor) else v) for k, v in sd.items()}
        self.log_std_min = self.sd["log_std_min"]
        self.log_std_dif = self.sd["log_std_dif"]

    # layers.py:94-133
    def _mlp(self, prefix: str, x: torch.Tensor, last: str, head: Optional[int] = None) -> torch.Tensor:
        i = 0
        while f"{prefix}.{i}.weight" in self.sd:
            w, b = self.sd[f"{prefix}.{i}.weight"], self.sd[f"{prefix}.{i}.bias"]
            g = self.sd.get(f"{prefix}.{i}.ln.weight")
            beta = self.sd.get(f"{prefix}.{i}.ln.bias")
            if head is not None:
                w, b = w[head], b[head]
                g = g[head] if g is not None else None
                beta = beta[head] if beta is not None else None
            is_last = f"{prefix}.{i + 1}.weight" not in self.sd
            x = F.linear(x, w, b)
            if g is not None:
                x = F.layer_norm(x, (x.shape[-1],), g, beta, 1e-5)
                if is_last and last == "simnorm":
                    shp = x.shape                                   # layers.py:84-88
                    x = F.softmax(x.view(*shp[:-1], -1, self.cfg.simnorm_dim), dim=-1).view(*shp)
                else:
                    x = F.mish(x)
            i += 1
        return x

    def task_emb(self, x: torch.Tensor, task: int) -> torch.Tensor:
        w = self.sd["_task_emb.weight"][task]
        # nn.Embedding(max_norm=1) renormalises the looked-up row (world_model.py:21):
        # rows with ||w||_2 > 1 are scaled by 1 / (norm + 1e-7).
        n = torch.linalg.vector_norm(w)
        if float(n) > 1.0:
            w = w * (1.0 / (n + 1e-7))
        return torch.cat([x, w.unsqueeze(0).repeat(x.shape[0], 1)], dim=-1)

    def encode(self, obs: torch.Tensor, task: Optional[int], shift: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.cfg.get("obs", "state") == "rgb":
            return self.encode_rgb(obs, shift)
        if self.cfg.multitask:
            obs = self.task_emb(obs, task)
        return self._mlp("_encoder.state", obs, "simnorm")

    def encode_rgb(self, obs: torch.Tensor, shift: torch.Tensor) -> torch.Tensor:
        """layers.conv (layers.py:136-150) on obs [n, C, 64, 64]: ShiftAug (:36-59) with its randint made explicit
        (`shift` [n, 2], values 0..6), PixelPreprocess (:62-71), 4 x Conv2d (+ ReLU between), Flatten, SimNorm."""
        pad = 3
        x = obs.to(self.dtype)
        n, _, h, w = x.size()
        assert h == w == 64                                                          # layers.py:141
        x = F.pad(x, (pad,) * 4, "replicate")
        eps = 1.0 / (h + 2 * pad)
        arange = torch.linspace(-1.0 + eps, 1.0 - eps, h + 2 * pad, dtype=x.dtype)[:h]
        arange = arange.unsqueeze(0).repeat(h, 1).unsqueeze(2)
        base_grid = torch.cat([arange, arange.transpose(1, 0)], dim=2)
        base_grid = base_grid.unsqueeze(0).repeat(n, 1, 1, 1)
        sh = shift.to(x.dtype).view(n, 1, 1, 2).clone()
        sh *= 2.0 / (h + 2 * pad)
        x = F.grid_sample(x, base_grid + sh, padding_mode="zeros", align_corners=False)
        x = x.div(255.).sub(0.5)
        for i, (idx, stride) in enumerate(((2, 2), (4, 2), (6, 2), (8, 1))):
            x = F.conv2d(x, self.sd[f"_encoder.rgb.{idx}.weight"], self.sd[f"_encoder.rgb.{idx}.bias"], stride=stride)
            if i < 3:
                x = F.relu(x)
        x = x.flatten(1)
        shp = x.shape                                                                # SimNorm, layers.py:84-88
        return F.softmax(x.view(*shp[:-1], -1, self.cfg.simnorm_dim), dim=-1).view(*shp)

    def next(self, z, a, task):
        if self.cfg.multitask:
            z = self.task_emb(z, task)
        return self._mlp("_dynamics", torch.cat([z, a], dim=-1), "simnorm")

    def reward(self, z, a, task):
        if self.cfg.multitask:
            z = self.task_emb(z, task)
        return self._mlp("_reward", torch.cat([z, a], dim=-1), "none")

    def termination_logits(self, z, task):
        """world_model.py:132-141 with unnormalized=True; the reference asserts `task is None`."""
        assert task is None
        if self.cfg.multitask:
            z = self.task_emb(z, task)
        return self._mlp("_termination", z, "none")

    def termination(self, z, task):
        return torch.sigmoid(self.termination_logits(z, task))

    def pi(self, z, task, eps):
        """Planner-visible part of WorldModel.pi: the squashed sampled action."""
        if self.cfg.multitask:
            z = self.task_emb(z, task)
        mean, log_std = self._mlp("_pi", z, "none").chunk(2, dim=-1)
        log_std = self.log_std_min + 0.5 * self.log_std_dif * (torch.tanh(log_std) + 1)   # math.py:12-13
        if self.cfg.multitask:
            m = self.sd["_action_masks"][task]
            mean, log_std, eps = mean * m, log_std * m, eps * m
        action = mean + eps * log_std.exp()
        return torch.tanh(action)                                                           # math.py:23-29 (squash)

    def Q_avg(self, z, a, task, qidx):
        if self.cfg.multitask:
            z = self.task_emb(z, task)
        x = torch.cat([z, a], dim=-1)
        qs = torch.stack([two_hot_inv(self._mlp("_Qs.params", x, "none", head=int(h)), self.cfg) for h in qidx])
        return qs.sum(0) / 2                                                                 # world_model.py:216


# --------------------------------------------------------------------------- planner
def _discount(cfg, task: Optional[int], dtype: torch.dtype = torch.float32) -> float:
    frac_of = lambda ep: ep / cfg.discount_denom
    d = lambda ep: min(max((frac_of(ep) - 1) / frac_of(ep), cfg.discount_min), cfg.discount_max)
    if cfg.multitask:
        return torch.tensor([d(ep) for ep in cfg.episode_lengths], dtype=dtype)[task]
    return d(cfg.episode_length)


def estimate_value(model: OracleModel, z, actions, task, eps_pi, qidx, info: Optional[dict] = None):
    """tdmpc2.py:122-136.  `info` (test aid, not in the reference) receives `term_margin` [N]: the smallest
    |termination logit| a sample saw, so parity tests can skip samples that sit on the 0.5 decision boundary."""
    cfg, dt = model.cfg, model.dtype
    z, actions, eps_pi = z.to(dt), actions.to(dt), eps_pi.to(dt)
    G, discount = 0, 1
    termination = torch.zeros(z.shape[0], 1, dtype=dt)
    margin = torch.full((z.shape[0],), float("inf"), dtype=dt)
    gamma = _discount(cfg, task, dt)
    for t in range(cfg.horizon):
        reward = two_hot_inv(model.reward(z, actions[t], task), cfg)
        z = model.next(z, actions[t], task)
        G = G + discount * (1 - termination) * reward
        discount = discount * gamma
        if cfg.episodic:                                                                    # tdmpc2.py:133-134
            logits = model.termination_logits(z, task)
            termination = torch.clip(termination + (torch.sigmoid(logits) > 0.5).float(), max=1.)
            margin = torch.minimum(margin, logits.abs().squeeze(1))
    if info is not None:
        info["term_margin"] = margin
    action = model.pi(z, task, eps_pi)
    return G + discount * (1 - termination) * model.Q_avg(z, action, task, qidx)


@torch.no_grad()
def balance_termination(cfg, sd: Dict[str, torch.Tensor], seed: int = 0, rows: int = 256) -> float:
    """Test aid for synthetic episodic models: random-init termination logits all share the sign of one
    common offset, so every sample would (not) terminate at once.  Shifts `_termination.2.bias` in place so
    that the logits of `rows` probe states (one dynamics step from an encoded random observation) have
    median 0.3 sigma -- a mix of terminated and live samples at every step.  Returns the new bias."""
    model = OracleModel(cfg, sd)
    g = torch.Generator().manual_seed(seed)
    z = model.encode(torch.randn(1, cfg.obs_shape["state"][0], generator=g), None).repeat(rows, 1)
    z = model.next(z, torch.rand(rows, cfg.action_dim, generator=g) * 2 - 1, None)
    lg = model.termination_logits(z, None).squeeze(1)
    bias = float(sd["_termination.2.bias"].reshape(-1)[0] - lg.median() - 0.3 * lg.std())
    sd["_termination.2.bias"] = torch.full_like(sd["_termination.2.bias"], bias)
    return bias


@dataclass
class PlanTrace:
    action: torch.Tensor                 # [E, A]
    mean: torch.Tensor                   # [E, H, A]  (next call's _prev_mean)
    std: torch.Tensor                    # [E, H, A]
    z: torch.Tensor                      # [E, L]
    pi_actions: torch.Tensor             # [E, H, P, A]
    values: torch.Tensor                 # [E, I, N]   (after nan_to_num)
    elite_idx: torch.Tensor              # [E, I, K] int64, sorted by value desc
    iter_mean: torch.Tensor              # [E, I, H, A]
    iter_std: torch.Tensor               # [E, I, H, A]
    score: torch.Tensor                  # [E, K]      (last iteration, normalised)
    pick: torch.Tensor                   # [E] int64   elite position chosen by the gumbel pick
    term_margin: Optional[torch.Tensor] = None   # [E, I, N] episodic models only: min |termination logit| per sample
    extras: Dict[str, torch.Tensor] = field(default_factory=dict)


@torch.no_grad()
def plan_one(model: OracleModel, obs, task, t0: bool, prev_mean, noise: PlanNoise, eval_mode: bool):
    """One reference `_plan` call (tdmpc2.py:138-206) with explicit noise; E == 1.  Runs in `model.dtype`."""
    cfg, dt = model.cfg, model.dtype
    obs, prev_mean = obs.to(dt), prev_mean.to(dt)
    H, N, P, A, K = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.num_elites
    if cfg.get("obs", "state") == "rgb":
        z = model.encode(obs.unsqueeze(0), task, noise.shift[0:1])                   # tdmpc2.py:111 unsqueezes; :153 encodes
    else:
        z = model.encode(obs.view(1, -1), task)
    z0 = z
    pi_actions = torch.zeros(H, P, A, dtype=dt)
    if P > 0:
        _z = z.repeat(P, 1)
        for t in range(H - 1):
            pi_actions[t] = model.pi(_z, task, noise.prior[0, t].to(dt))
            _z = model.next(_z, pi_actions[t], task)
        pi_actions[-1] = model.pi(_z, task, noise.prior[0, H - 1].to(dt))
    z = z.repeat(N, 1)
    mean = torch.zeros(H, A, dtype=dt)
    std = torch.full((H, A), float(cfg.max_std), dtype=dt)
    if not t0:
        mean[:-1] = prev_mean[1:]
    actions = torch.empty(H, N, A, dtype=dt)
    if P > 0:
        actions[:, :P] = pi_actions
    mask = model.sd["_action_masks"][task] if cfg.multitask else None
    vals, idxs, means, stds, margins = [], [], [], [], []
    for it in range(cfg.iterations):
        r = noise.r[0, it].to(dt)
        actions_sample = mean.unsqueeze(1) + std.unsqueeze(1) * r
        actions_sample = actions_sample.clamp(-1, 1)
        actions[:, P:] = actions_sample
        if mask is not None:
            actions = actions * mask
        info = {}
        value = estimate_value(model, z, actions, task, noise.pi[0, it], noise.qidx[0, it], info).nan_to_num(0)
        margins.append(info["term_margin"])
        elite_idxs = torch.topk(value.squeeze(1), K, dim=0).indices
        elite_value, elite_actions = value[elite_idxs], actions[:, elite_idxs]
        max_value = elite_value.max(0).values
        score = torch.exp(cfg.temperature * (elite_value - max_value))
        score = score / score.sum(0)
        mean = (score.unsqueeze(0) * elite_actions).sum(dim=1) / (score.sum(0) + 1e-9)
        std = ((score.unsqueeze(0) * (elite_actions - mean.unsqueeze(1)) ** 2).sum(dim=1)
               / (score.sum(0) + 1e-9)).sqrt()
        std = std.clamp(cfg.min_std, cfg.max_std)
        if mask is not None:
            mean = mean * mask
            std = std * mask
        vals.append(value.squeeze(1)); idxs.append(elite_idxs); means.append(mean); stds.append(std)
    # gumbel pick, math.py:86-94 with the exponential draw made explicit
    logits = score.squeeze(1).log()
    gumbels = -noise.expo[0].to(dt).log()
    y_soft = ((logits + gumbels) / 1.0).softmax(0)
    rand_idx = y_soft.argmax(-1)
    a = elite_actions[0, rand_idx]
    if not eval_mode:
        a = a + std[0] * noise.final[0].to(dt)
    out = dict(action=a.clamp(-1, 1), mean=mean, std=std, z=z0[0], pi_actions=pi_actions,
               values=torch.stack(vals), elite_idx=torch.stack(idxs), iter_mean=torch.stack(means),
               iter_std=torch.stack(stds), score=score.squeeze(1), pick=rand_idx)
    if cfg.episodic:
        out["term_margin"] = torch.stack(margins)
    return out


@torch.no_grad()
def plan_oracle(cfg, sd, obs, task=None, t0=None, prev_mean=None, noise: PlanNoise = None,
                eval_mode: bool = False, dtype: torch.dtype = torch.float32) -> PlanTrace:
    """Env-batched planner: obs [E, obs_dim], task [E] or None, t0 [E] bool,
    prev_mean [E, H, A]; loops the E independent reference plans.  `dtype` applies when `sd` is a state dict; an
    OracleModel brings its own."""
    model = sd if isinstance(sd, OracleModel) else OracleModel(cfg, sd, dtype)
    obs = torch.as_tensor(obs, dtype=model.dtype)
    E = obs.shape[0]
    if t0 is None:
        t0 = [True] * E
    if prev_mean is None:
        prev_mean = torch.zeros(E, cfg.horizon, cfg.action_dim)
    outs = []
    for e in range(E):
        tk = int(task[e]) if (cfg.multitask and task is not None) else None
        outs.append(plan_one(model, obs[e], tk, bool(t0[e]), prev_mean[e], noise.env(e), eval_mode))
    return PlanTrace(**{k: torch.stack([o[k] for o in outs]) for k in outs[0]})
