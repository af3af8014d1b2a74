"""The model file: what a plain C or C++ host loads to plan without Python (`tdmpc2_model_file_open` / `_upload` of
include/tdmpc2_b200.h, examples/c_act.c).

`export_model(state_dict, cfg, fp)` writes the safetensors layout -- an 8-byte little-endian header length, a JSON header,
then the raw little-endian data -- with `json` and `struct` only, so exporting needs neither the `safetensors` package nor
a GPU.  It holds what acting reads, as fp32 under the reference's state-dict keys:

  * `_encoder.state.*` (state observations) or `_encoder.rgb.{2,4,6,8}.*` (pixels), `_dynamics.*`, `_reward.*`, `_pi.*`,
    the stacked `_Qs.params.{0,1,2}.*` (leading [num_q]), `_termination.*` of episodic models, `_task_emb.weight` and
    `_action_masks` of multi-task models;
  * `tdmpc2.bins` (the two-hot bins the planner packs), `tdmpc2.discount` [num_tasks] as F64 (`get_discount` per task;
    the library raises it to the powers of its horizon) and, for pixel models, `tdmpc2.grid_base` [64] (ShiftAug's grid).

The `_detach_` / `_target_` copies and tensordict's metadata entries are left out: the file is for acting, `agent.save`
stays the checkpoint format.  `__metadata__` holds `format`, `version`, `obs`, every `tdmpc2_dims` field (as the planner
fills them; `num_envs` = cfg.num_envs, `iterations` the effective count) and, for pixel models, `pixel.in_channels`,
`pixel.num_channels` and `pixel.simnorm_dim`.  Floats are written so that strtod followed by a cast to float gives the
fp32 value the planner would use.
"""
from __future__ import annotations

import json
import math
import struct
from fractions import Fraction
from typing import Dict

import numpy as np
import torch

from .config import Config, get_discount

FORMAT, VERSION = "tdmpc2_b200.model", "1"
_PREFIXES = ("_encoder.state.", "_encoder.rgb.", "_dynamics.", "_reward.", "_pi.", "_Qs.params.")


def _f32(x: float) -> float:
    """x rounded to the nearest fp32 value, as a Python float (what a ctypes c_float field stores)."""
    return struct.unpack("<f", struct.pack("<f", float(x)))[0]


def _round_f32(x: Fraction) -> float:
    """The exact rational x rounded once to the nearest fp32 value (ties to even)."""
    c = float(np.float32(float(x)))
    lo, hi = float(np.nextafter(np.float32(c), np.float32(-np.inf))), float(np.nextafter(np.float32(c), np.float32(np.inf)))
    best = min((abs(Fraction(v) - x), int(np.float32(v).view(np.int32)) & 1, v) for v in (lo, c, hi))
    return best[2]


def linspace_f32(start: float, end: float, steps: int) -> torch.Tensor:
    """torch.linspace(start, end, steps) in fp32 as the CUDA kernel computes it, which is what the planner packs: step =
    (end - start) / (steps - 1) in fp32, then start + step i (one rounding) below steps // 2 and end - step (steps - 1 - i)
    above.  Computed here with exact rationals, so the values do not depend on this machine's torch build."""
    s, e = _f32(start), _f32(end)
    step = _round_f32(Fraction(_round_f32(Fraction(e) - Fraction(s))) / (steps - 1)) if steps > 1 else 0.0
    half = steps // 2
    vals = [_round_f32(Fraction(s) + Fraction(step) * i) if i < half else _round_f32(Fraction(e) - Fraction(step) * (steps - 1 - i))
            for i in range(steps)]
    return torch.tensor(vals, dtype=torch.float32)


def grid_base() -> torch.Tensor:
    """ShiftAug's base grid (layers.py:50-51): torch.linspace(-1 + 1/70, 1 - 1/70, 70)[:64]."""
    eps = 1.0 / (64 + 2 * 3)
    return linspace_f32(-1.0 + eps, 1.0 - eps, 64 + 2 * 3)[:64].contiguous()


def _float_str(x: float) -> str:
    """The shortest decimal of the fp32 value of x: strtod gives that value's double exactly, and its cast to float is
    the value itself."""
    v = _f32(x)
    if not math.isfinite(v):
        raise ValueError(f"cannot export the non-finite value {x}")
    return repr(v)


def effective_iterations(cfg: Config) -> int:
    """The CEM loop count the agent plans with: cfg.iterations after tdmpc2.py:34's += 2 for action_dim >= 20 (TDMPC2
    applies it once and marks cfg.iterations_effective)."""
    return int(cfg.iterations) + (0 if cfg.get("iterations_effective", False) else 2 * int(cfg.action_dim >= 20))


def model_metadata(cfg: Config) -> Dict[str, str]:
    """`__metadata__` of the model file for cfg: format, version, obs and the tdmpc2_dims the planner builds from cfg."""
    rgb = cfg.get("obs", "state") == "rgb"
    ints = dict(num_envs=int(cfg.get("num_envs", 1) or 1), num_samples=cfg.num_samples, num_pi_trajs=cfg.num_pi_trajs,
                num_elites=cfg.num_elites, horizon=cfg.horizon, iterations=effective_iterations(cfg),
                obs_dim=1 if rgb else cfg.obs_shape["state"][0], action_dim=cfg.action_dim, latent_dim=cfg.latent_dim,
                mlp_dim=cfg.mlp_dim, enc_dim=cfg.enc_dim, num_enc_layers=0 if rgb else cfg.num_enc_layers,
                task_dim=cfg.task_dim if cfg.multitask else 0, num_tasks=len(cfg.tasks) if cfg.multitask else 1,
                num_q=cfg.num_q, num_bins=cfg.num_bins, simnorm_dim=cfg.simnorm_dim, episodic=int(bool(cfg.episodic)))
    floats = dict(temperature=cfg.temperature, min_std=cfg.min_std, max_std=cfg.max_std, log_std_min=float(cfg.log_std_min),
                  log_std_dif=float(cfg.log_std_max) - float(cfg.log_std_min))
    meta = {"format": FORMAT, "version": VERSION, "obs": "rgb" if rgb else "state"}
    meta.update({k: str(int(v)) for k, v in ints.items()})
    meta.update({k: _float_str(v) for k, v in floats.items()})
    if rgb:
        meta.update({"pixel.in_channels": str(int(cfg.obs_shape["rgb"][0])), "pixel.num_channels": str(int(cfg.num_channels)),
                     "pixel.simnorm_dim": str(int(cfg.simnorm_dim))})
    return meta


def model_tensors(state_dict: Dict[str, torch.Tensor], cfg: Config) -> Dict[str, torch.Tensor]:
    """The tensors of the model file, by key, as contiguous CPU tensors (fp32; tdmpc2.discount fp64)."""
    keep = lambda k: (k.startswith(_PREFIXES) or (cfg.episodic and k.startswith("_termination."))
                      or (cfg.multitask and k in ("_task_emb.weight", "_action_masks")))
    out = {}
    for k, v in state_dict.items():
        if keep(k) and torch.is_tensor(v) and not k.endswith(("__batch_size", "__device")):
            out[k] = v.detach().to("cpu", torch.float32).contiguous()
    out["tdmpc2.bins"] = linspace_f32(cfg.vmin, cfg.vmax, cfg.num_bins)            # math.py:80
    gammas = [get_discount(cfg, ep) for ep in cfg.episode_lengths] if cfg.multitask else [get_discount(cfg, cfg.episode_length)]
    out["tdmpc2.discount"] = torch.tensor(gammas, dtype=torch.float64)
    if cfg.get("obs", "state") == "rgb":
        out["tdmpc2.grid_base"] = grid_base()
    return out


def export_model(state_dict: Dict[str, torch.Tensor], cfg: Config, fp) -> None:
    """Write the model file of a reference-layout state dict and its cfg to `fp` (a path or a binary file object)."""
    tensors = model_tensors(state_dict, cfg)
    header, blobs, off = {"__metadata__": model_metadata(cfg)}, [], 0
    for k in sorted(tensors):
        t = tensors[k]
        data = t.numpy().astype("<f8" if t.dtype == torch.float64 else "<f4", copy=False).tobytes()
        header[k] = {"dtype": "F64" if t.dtype == torch.float64 else "F32", "shape": list(t.shape), "data_offsets": [off, off + len(data)]}
        blobs.append(data)
        off += len(data)
    h = json.dumps(header, separators=(",", ":")).encode()
    h += b" " * (-len(h) % 8)                     # the data section starts 8-byte aligned
    if isinstance(fp, (str, bytes)) or hasattr(fp, "__fspath__"):
        with open(fp, "wb") as f:
            _write(f, h, blobs)
    else:
        _write(fp, h, blobs)


def _write(f, h: bytes, blobs) -> None:
    f.write(struct.pack("<Q", len(h)))
    f.write(h)
    for b in blobs:
        f.write(b)
