"""Synthetic world-model weights in the reference's state-dict layout.

There is no network here for released checkpoints, so benchmarks and tests run
on random-init weights of the reference architecture.  Key names and shapes
follow `WorldModel.state_dict()` of the reference
(tdmpc2/common/world_model.py:17-53, layers.py:121-164; listed in SURVEY.md
section 8(b)); values follow `common/init.py:4-11` (trunc-normal sigma 0.02,
zero bias, LayerNorm 1/0, embedding U(-0.02, 0.02)) but WITHOUT the zero-init of
the reward / Q output layers (world_model.py:32) -- with those zeroed every
trajectory value ties at 0 and top-k parity is degenerate (SURVEY.md section 7).

`perturb=True` additionally randomises biases and LayerNorm affine parameters
so that parity tests exercise every parameter tensor.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from .config import Config

QS_PREFIXES = ("_Qs.params.", "_detach_Qs_params.", "_target_Qs_params.")


def mlp_dims(in_dim: int, hidden: List[int], out_dim: int) -> List[Tuple[int, int]]:
    dims = [in_dim] + list(hidden) + [out_dim]
    return [(dims[i], dims[i + 1]) for i in range(len(dims) - 1)]


def head_layout(cfg: Config) -> Dict[str, Dict]:
    """Per-head (in, out) layer dims and which layers carry a LayerNorm."""
    L, M, A, T, B = cfg.latent_dim, cfg.mlp_dim, cfg.action_dim, cfg.task_dim, max(cfg.num_bins, 1)
    D = L + A + T
    obs_dim = cfg.obs_shape["state"][0] if "state" in cfg.obs_shape else 1
    n_hidden = max(cfg.num_enc_layers - 1, 1)
    return {
        # layers.enc: every layer is a NormedLinear, last activation SimNorm (layers.py:157-159)
        "_encoder.state": dict(dims=mlp_dims(obs_dim + T, n_hidden * [cfg.enc_dim], L), ln_last=True),
        "_dynamics": dict(dims=mlp_dims(D, 2 * [M], L), ln_last=True),    # world_model.py:26
        "_reward": dict(dims=mlp_dims(D, 2 * [M], B), ln_last=False),      # world_model.py:27
        "_pi": dict(dims=mlp_dims(L + T, 2 * [M], 2 * A), ln_last=False),  # world_model.py:29
        "_Qs": dict(dims=mlp_dims(D, 2 * [M], B), ln_last=False),          # world_model.py:30
        "_termination": dict(dims=mlp_dims(L + T, 2 * [M], 1), ln_last=False),   # world_model.py:28 (cfg.episodic only)
    }


def _trunc_normal(shape, gen: torch.Generator, std: float = 0.02) -> torch.Tensor:
    # nn.init.trunc_normal_(std=0.02) truncates at +-2.0 absolute (100 sigma):
    # numerically a plain normal; resample the (never observed) outliers anyway.
    w = torch.randn(shape, generator=gen) * std
    return w.clamp_(-2.0, 2.0)


def synth_state_dict(cfg: Config, seed: int = 1, perturb: bool = False,
                     emb_scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """Deterministic (CPU generator) state dict with the reference's keys."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def fill(prefix: str, dims, ln_last: bool, lead=()):
        n = len(dims)
        for i, (fin, fout) in enumerate(dims):
            sd[f"{prefix}.{i}.weight"] = _trunc_normal(lead + (fout, fin), gen)
            b = torch.zeros(lead + (fout,))
            if perturb:
                b = torch.randn(lead + (fout,), generator=gen) * 0.02
            sd[f"{prefix}.{i}.bias"] = b
            if i < n - 1 or ln_last:
                g, beta = torch.ones(lead + (fout,)), torch.zeros(lead + (fout,))
                if perturb:
                    g = 1.0 + 0.1 * torch.randn(lead + (fout,), generator=gen)
                    beta = 0.1 * torch.randn(lead + (fout,), generator=gen)
                sd[f"{prefix}.{i}.ln.weight"] = g
                sd[f"{prefix}.{i}.ln.bias"] = beta

    if cfg.multitask:
        emb = (torch.rand(len(cfg.tasks), cfg.task_dim, generator=gen) * 0.04 - 0.02) * emb_scale
        sd["_task_emb.weight"] = emb
        masks = torch.zeros(len(cfg.tasks), cfg.action_dim)
        for i, a in enumerate(cfg.action_dims):
            masks[i, :a] = 1.0
        sd["_action_masks"] = masks  # world_model.py:22-24
    lay = head_layout(cfg)
    if cfg.get("obs", "state") == "rgb":
        # layers.conv (layers.py:136-150): Conv2d at Sequential indices 2, 4, 6, 8.  The reference leaves them at
        # nn.Conv2d's default init (init.weight_init does not touch Conv2d); synthetic values of that scale.
        C, nc = cfg.obs_shape["rgb"][0], cfg.num_channels
        for idx, (cin, k) in zip((2, 4, 6, 8), ((C, 7), (nc, 5), (nc, 3), (nc, 3))):
            bound = 1.0 / (cin * k * k) ** 0.5
            sd[f"_encoder.rgb.{idx}.weight"] = (torch.rand(nc, cin, k, k, generator=gen) * 2 - 1) * bound
            sd[f"_encoder.rgb.{idx}.bias"] = (torch.rand(nc, generator=gen) * 2 - 1) * bound
    else:
        fill("_encoder.state", lay["_encoder.state"]["dims"], lay["_encoder.state"]["ln_last"])
    for name in ("_dynamics", "_reward", "_pi"):
        fill(name, lay[name]["dims"], lay[name]["ln_last"])
    q: Dict[str, torch.Tensor] = {}
    _sd, sd = sd, q
    fill("Q", lay["_Qs"]["dims"], False, lead=(cfg.num_q,))
    sd = _sd
    for k, v in q.items():
        sub = k[len("Q."):]
        sd["_Qs.params." + sub] = v
        sd["_detach_Qs_params." + sub] = v            # shares storage (world_model.py:40)
        sd["_target_Qs_params." + sub] = v.clone()    # world_model.py:41
    if cfg.episodic:     # drawn last: an episodic model shares every other tensor with the non-episodic one of the same seed
        fill("_termination", lay["_termination"]["dims"], False)
        # sigma 0.16 instead of 0.02 on the single output row: with init-scale weights every logit has the sign of
        # the bias and all samples would (not) terminate together; this spreads them across the 0.5 boundary
        sd["_termination.2.weight"] = sd["_termination.2.weight"] * 8.0
    sd["log_std_min"] = torch.tensor(float(cfg.log_std_min))
    sd["log_std_dif"] = torch.tensor(float(cfg.log_std_max)) - sd["log_std_min"]
    return sd


# Logit spread (standard deviation over rows and bins, in units of the layer's fan-in-normalised scale) that each level
# targets at the reward / Q / termination outputs, and the pre-activation scale of the policy's mean and log-std.  The
# gains are divided by sigma(W) sqrt(fan_in), so that one level lands in the same regime on every preset: a plain
# gain that sharpens a 512-wide model leaves a 64-wide one near-uniform.
TRAINED_LEVELS = {
    #          two-hot heads, pi mean, pi log-std, termination
    "mid": dict(twohot=1.15, pi_mean=1.5, pi_log_std=1.5, term=20.0),
    "sharp": dict(twohot=8.0, pi_mean=12.0, pi_log_std=12.0, term=60.0),
}
# Per-preset (Config.task) two-hot spreads where the level's default does not land in its regime: how far trajectory
# values spread also depends on how much the latent varies between samples, which the fan-in normalisation misses.
TRAINED_TWOHOT = {("tiny", "mid"): 1.2, ("tiny-mt", "mid"): 3.5, ("tiny-mt", "sharp"): 12.0}
OUTLIERS_PER_MATRIX = 3


def trained_scale(cfg: Config, sd: Dict[str, torch.Tensor], level: str, seed: int) -> Dict[str, torch.Tensor]:
    """A deterministic transform of a synthetic state dict towards what a trained model looks like, for parity tests
    beyond the benign initialisation regime:

      * LayerNorm gamma ~ lognormal(0, 0.5), beta ~ N(0, 0.5^2);
      * reward / Q output layers scaled so that the two-hot softmax is peaked (values reach 1e3 - 1e4 at "sharp");
      * the policy's mean rows scaled so that tanh saturates, its log-std rows so that log-stds reach their clamp;
      * the termination output scaled so that logits reach +-20 (re-centre it with balance_termination afterwards);
      * OUTLIERS_PER_MATRIX entries of every weight matrix (per Q head) set to 30 - 60 x the matrix's sigma, which
        moves the power-of-two scale the packer gives the matrix by several binades.

    Q-ensemble tensors (online, detach, target) get the same draws, so the online / target difference of the input
    (e.g. a target blend made before this transform) is kept.  Returns a new dict; `sd` is not modified."""
    lv = dict(TRAINED_LEVELS[level])
    lv["twohot"] = TRAINED_TWOHOT.get((cfg.task, level), lv["twohot"])
    gen = torch.Generator(device="cpu").manual_seed(seed)
    out = dict(sd)
    A = cfg.action_dim

    def fan_in_gain(w: torch.Tensor, spread: float) -> float:
        return spread / (float(w.std()) * w.shape[-1] ** 0.5)

    def per_key(key: str):
        """Same transform for every copy of a Q-ensemble tensor."""
        for p in QS_PREFIXES:
            if key.startswith(p):
                return "_Qs.params." + key[len(p):]
        return key

    draws: Dict[str, object] = {}

    def draw(key, make):
        k = per_key(key)
        if k not in draws:
            draws[k] = make()
        return draws[k]

    for key in sorted(sd):
        v = sd[key]
        if not isinstance(v, torch.Tensor) or not v.is_floating_point() or key.startswith(("_task_emb", "_action_masks",
                                                                                           "log_std", "_encoder.rgb")):
            continue
        if key.endswith(".ln.weight"):
            out[key] = draw(key, lambda: torch.exp(0.5 * torch.randn(v.shape, generator=gen)))
        elif key.endswith(".ln.bias"):
            out[key] = draw(key, lambda: 0.5 * torch.randn(v.shape, generator=gen))
        elif key.endswith(".weight"):
            def outliers(v=v):
                w = v.reshape(-1, v.shape[-2] * v.shape[-1])           # one row per Q head
                pos = torch.stack([torch.randperm(w.shape[1], generator=gen)[:OUTLIERS_PER_MATRIX] for _ in range(w.shape[0])])
                mag = (30.0 + 30.0 * torch.rand(pos.shape, generator=gen)) * torch.where(
                    torch.rand(pos.shape, generator=gen) < 0.5, -1.0, 1.0)
                return pos, mag
            pos, mag = draw(key, outliers)
            w = v.detach().clone().reshape(-1, v.shape[-2] * v.shape[-1])
            sigma = w.std(dim=1, keepdim=True)
            w.scatter_(1, pos, mag * sigma)
            out[key] = w.reshape(v.shape)
    # output-layer gains (after the outliers, so that sigma(W) includes them as a trained matrix's would)
    def gain(prefix: str, spread: float, rows=slice(None)):
        w = out[prefix + ".weight"]
        heads = w.reshape(-1, *w.shape[-2:])
        g = torch.ones(heads.shape[:2])
        for h in range(heads.shape[0]):
            g[h, rows] = fan_in_gain(heads[h][rows], spread)
        g = g.reshape(w.shape[:-1])
        out[prefix + ".weight"] = w * g.unsqueeze(-1)
        out[prefix + ".bias"] = out[prefix + ".bias"] * g
    if cfg.num_bins > 1:
        gain("_reward.2", lv["twohot"])
        for p in ("_Qs.params.", "_target_Qs_params."):
            gain(p + "2", lv["twohot"])
    gain("_pi.2", lv["pi_mean"], slice(0, A))
    gain("_pi.2", lv["pi_log_std"], slice(A, 2 * A))
    if cfg.episodic:
        gain("_termination.2", lv["term"])
    for k in sd:
        if k.startswith("_detach_Qs_params."):          # shares the online tensors, as in the reference (world_model.py:40)
            out[k] = out["_Qs.params." + k[len("_detach_Qs_params."):]]
    return out


def state_dict_checksum(sd: Dict[str, torch.Tensor]) -> float:
    """Order-independent fingerprint used by golden fixtures to detect RNG drift."""
    tot = 0.0
    for k in sorted(sd):
        v = sd[k]
        if isinstance(v, torch.Tensor) and v.is_floating_point() and not k.startswith(("_detach", "_target")):
            tot += float(v.double().abs().sum()) + 3.0 * float(v.double().sum())
    return tot
