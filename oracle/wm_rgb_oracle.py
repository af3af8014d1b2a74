"""Golden fixtures of pixel models' `encode` on batches of frames -- TEST INFRASTRUCTURE ONLY.

The no-grad block of the reference's `_update` (tdmpc2.py:259-264) on pixel observations: its own `WorldModel.encode` on
[T, B, C, 64, 64] frames (common/world_model.py:103-112: one layers.conv call per slice t, each with its own ShiftAug
randint draw, layers.py:36-59,136-150) followed by its own `_td_target`.  The frames are regenerated from a seed and
guarded by a checksum; a fixture holds the recorded shifts, z, the td inputs' draws and td.  The oracle side is
OracleModel.encode_rgb (oracle/plan_oracle.py) and WMOracle.td_target (oracle/wm_oracle.py).

    python -m oracle.wm_rgb_oracle [names]      # mints tests/golden/<name>.npz from the reference's own methods
"""
from __future__ import annotations

import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.wm_oracle import attach_target_qs, with_target_blend   # noqa: E402


# --------------------------------------------------------------------------- pixel-model fixtures (cfg.obs == 'rgb')
# name -> (workload, overrides, weight seed, target-blend seed, T, B, call seed).  Kept out of CASES: their inputs are
# frames, not state vectors.  The frames are regenerated from the call seed and guarded by a checksum.
RGB_CASES = {
    "tiny_rgb_wm": ("tiny-rgb", {}, 26, 126, 3, 5, 650),
    "c1_rgb_wm": ("c1", {"obs": "rgb", "obs_channels": 9}, 27, 127, 3, 4, 660),   # nc = 32, latent 512
}


def rgb_case_model(name):
    """(cfg, state dict with a blended target ensemble) of a pixel fixture."""
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    wl, over, wseed, tseed, T, B, _ = RGB_CASES[name]
    cfg = workload(wl, **over)
    sd = synth_state_dict(cfg, seed=wseed, perturb=True)
    return cfg, with_target_blend(cfg, sd, tseed)


def rgb_case_inputs(cfg, T, B, seed):
    """frames [T, B, C, 64, 64] (fp32 values 0..255), reward / terminated [T, B, 1]."""
    g = torch.Generator().manual_seed(seed)
    frames = torch.randint(0, 256, (T, B) + tuple(cfg.obs_shape["rgb"]), generator=g).float()
    reward = torch.randn(T, B, 1, generator=g)
    terminated = (torch.rand(T, B, 1, generator=g) < 0.3).float()
    return frames, reward, terminated


def frames_checksum(frames: torch.Tensor) -> float:
    x = frames.double().flatten()
    return float(x.sum()) + float((x * torch.linspace(0.0, 1.0, x.numel(), dtype=torch.float64)).sum())


def _record_rgb(agent, frames, reward, terminated, seed):
    """The reference's own `encode` on pixel frames (ShiftAug draws inside), then `_td_target`, under
    torch.manual_seed(seed); the randint / randn_like / randperm draws they make are captured."""
    m = agent.model
    draws = {"shift": [], "eps": [], "qidx": []}
    real_randint, real_randn_like, real_randperm = torch.randint, torch.randn_like, torch.randperm

    def randint(*a_, **k):
        out = real_randint(*a_, **k)
        draws["shift"].append(out.clone().reshape(-1, 2))        # ShiftAug's (n, 1, 1, 2), layers.py:55
        return out

    def randn_like(x, *a_, **k):
        out = real_randn_like(x, *a_, **k)
        draws["eps"].append(out.clone())
        return out

    def randperm(n, *a_, **k):
        out = real_randperm(n, *a_, **k)
        draws["qidx"].append(out[:2].clone())
        return out

    torch.manual_seed(seed)
    torch.randint, torch.randn_like, torch.randperm = randint, randn_like, randperm
    try:
        with torch.no_grad():
            z = m.encode(frames, None)
            td = agent._td_target(z, reward, terminated, None)
    finally:
        torch.randint, torch.randn_like, torch.randperm = real_randint, real_randn_like, real_randperm
    lead = frames.shape[:-3]
    return dict(shift=torch.stack(draws["shift"]).reshape(*lead, 2), z=z, td_eps=draws["eps"][0], td_qidx=draws["qidx"][0],
                td=td)


def main(only=None):
    import numpy as np
    from oracle import ref_harness as rh
    from tdmpc2_b200.synth import state_dict_checksum
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, (wl, over, wseed, tseed, T, B, seed) in RGB_CASES.items():
        if only and name not in only:
            continue
        t = time.time()
        cfg, sd = rgb_case_model(name)
        agent = rh.build_agent(cfg, sd)
        attach_target_qs(agent, sd)
        frames, reward, terminated = rgb_case_inputs(cfg, T, B, seed)
        rec = dict(case=name, weight_checksum=state_dict_checksum(sd), frames_checksum=frames_checksum(frames),
                   torch_version=torch.__version__)
        # the [T, B] batch (T ShiftAug draws of (B, 2)) and one 4-D [1, C, 64, 64] row (one draw)
        for pfx, (f_, rw, te), s in (("b", (frames, reward, terminated), seed),
                                     ("r", (frames[0, :1], reward[0, :1], terminated[0, :1]), seed + 1)):
            for k, v in _record_rgb(agent, f_, rw, te, s).items():
                rec[f"{pfx}_{k}"] = v.numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **rec)
        print(f"{name}: {time.time() - t:.1f}s -> tests/golden/{name}.npz")


def load_rgb_case(name):
    """(cfg, sd, {"b": [T, B] batch record, "r": one 4-D row record}) of a pixel fixture, inputs included: frames,
    reward_in, terminated, and the recorded shift, z, td_eps, td_qidx, td."""
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    f = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
    cfg, sd = rgb_case_model(name)
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), "synthetic weights differ from the fixture's"
    wl, over, wseed, tseed, T, B, seed = RGB_CASES[name]
    frames, reward, terminated = rgb_case_inputs(cfg, T, B, seed)
    fchk = frames_checksum(frames)
    assert abs(fchk - float(f["frames_checksum"])) <= 1e-12 * abs(fchk), "regenerated frames differ from the fixture's"
    inputs = {"b": (frames, reward, terminated), "r": (frames[0, :1], reward[0, :1], terminated[0, :1])}
    recs = {}
    for pfx in ("b", "r"):
        d = {k[2:]: torch.from_numpy(f[k]) for k in f.files if k.startswith(pfx + "_")}
        d["frames"], d["reward_in"], d["terminated"] = inputs[pfx]
        recs[pfx] = d
    return cfg, sd, recs



if __name__ == "__main__":
    main(sys.argv[1:] or None)
