"""Pixel encoder (cfg.obs == 'rgb') throughput: the persistent conv-encoder kernel against batched eager fp32 PyTorch.

Model: c1 with obs="rgb", obs_channels=9 (num_channels 32, latent 512).  Arms:
  a  Planner.encode_pixel_rows (the kernel alone) at each frame count
  b  WorldModel.encode end to end: uint8 frames [T, 256, C, 64, 64], ShiftAug draws, fp32 conversion, one launch
  c  batched eager fp32 PyTorch: grid_sample + 4 x conv2d (cuDNN, TF32 off) + SimNorm
  d  Planner(cfg, E).encode_pixels, the planning prologue's call, at E in --envs
CUDA-event medians after warm-up; prints the GPU name and power limit, and FP32 TFLOP/s computed from the shapes.

    python scripts/bench_pixel_encode.py [--frames 768 8192] [--envs 1 256 768] [--arms abcd] [--dump DIR]

--dump DIR writes z of arm d on seeded frames and shifts (tiny-rgb and c1-rgb, every E of --envs) to DIR/pixel_z.npz,
so two builds can be compared byte for byte.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tdmpc2_b200.config import workload          # noqa: E402
from tdmpc2_b200.synth import synth_state_dict   # noqa: E402


def conv_flop_per_frame(C, nc):
    """2 x multiply-adds of the four convolutions (29^2, 13^2, 6^2, 4^2 outputs)."""
    return 2 * nc * (C * 49 * 841 + nc * 25 * 169 + nc * 9 * 36 + nc * 9 * 16)


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2]


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit_clock"] = out[0] if out else "?"
    except Exception as exc:                                  # noqa: BLE001
        info["power_limit_clock"] = f"? ({exc})"
    return info


def frames_and_shift(cfg, R, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    frames = torch.randint(0, 256, (R,) + tuple(cfg.obs_shape["rgb"]), generator=g, device="cuda").to(dtype)
    shift = torch.randint(0, 7, (R, 2), generator=g, device="cuda", dtype=torch.float32)
    return frames, shift


def eager_encode(sd, cfg, frames, shift):
    """layers.conv batched in eager PyTorch (ShiftAug with explicit shifts, PixelPreprocess, convs, SimNorm)."""
    n, _, h, _ = frames.shape
    x = F.pad(frames, (3, 3, 3, 3), "replicate")
    eps = 1.0 / (h + 6)
    ar = torch.linspace(-1.0 + eps, 1.0 - eps, h + 6, device=x.device)[:h]
    ar = ar.unsqueeze(0).repeat(h, 1).unsqueeze(2)
    grid = torch.cat([ar, ar.transpose(1, 0)], dim=2).unsqueeze(0) + (shift * (2.0 / (h + 6))).view(n, 1, 1, 2)
    x = F.grid_sample(x, grid, padding_mode="zeros", align_corners=False).div(255.).sub(0.5)
    for i, (idx, st) in enumerate(((2, 2), (4, 2), (6, 2), (8, 1))):
        x = F.conv2d(x, sd[f"_encoder.rgb.{idx}.weight"], sd[f"_encoder.rgb.{idx}.bias"], stride=st)
        if i < 3:
            x = F.relu(x)
    x = x.flatten(1)
    return F.softmax(x.view(n, -1, cfg.simnorm_dim), dim=-1).view(n, -1)


def dump(out_dir, envs):
    import numpy as np
    from tdmpc2_b200.planner import Planner
    rec = {}
    for tag, wl, over in (("tiny_rgb", "tiny-rgb", {}), ("c1_rgb", "c1", {"obs": "rgb", "obs_channels": 9})):
        for E in envs:
            cfg = workload(wl, num_envs=E, **over)
            sd = synth_state_dict(cfg, seed=41, perturb=True)
            pl = Planner(cfg, E, "cuda:0")
            pl.pack(sd)
            frames, shift = frames_and_shift(cfg, E, 1000 + E)
            rec[f"{tag}_E{E}"] = pl.encode_pixels(frames, shift).cpu().numpy()
    os.makedirs(out_dir, exist_ok=True)
    np.savez(os.path.join(out_dir, "pixel_z.npz"), **rec)
    print(json.dumps({"dump": os.path.join(out_dir, "pixel_z.npz"), "keys": sorted(rec)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[768, 8192])
    ap.add_argument("--envs", type=int, nargs="+", default=[1, 256, 768])
    ap.add_argument("--arms", default="abcd")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pixel_encode.py needs a CUDA device")
    if args.dump:
        dump(args.dump, args.envs)
        return
    from tdmpc2_b200.planner import Planner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    over = {"obs": "rgb", "obs_channels": 9}
    cfg = workload("c1", **over)
    C, nc = cfg.obs_shape["rgb"][0], cfg.num_channels
    sd = {k: v.cuda() for k, v in synth_state_dict(cfg, seed=41, perturb=True).items()}
    flop = conv_flop_per_frame(C, nc)
    res = {"tag": args.tag, **gpu_info(), "model": "c1 rgb C=9 nc=32", "mflop_per_frame": flop / 1e6}
    rate = lambda n, ms: round(n * flop / (ms * 1e-3) / 1e12, 2)

    if any(a in args.arms for a in "abc"):
        pl = Planner(cfg, 1, "cuda:0")
        pl.pack(sd)
        if "b" in args.arms:
            from tdmpc2_b200.world_model import WorldModel
            m = WorldModel(cfg).cuda()
            m.load_state_dict(sd)
        for R in args.frames:
            frames, shift = frames_and_shift(cfg, R, 7)
            if "a" in args.arms:
                ms = median_ms(lambda: pl.encode_pixel_rows(frames, shift), args.reps, args.warmup)
                res[f"a_rows_R{R}_ms"], res[f"a_rows_R{R}_tflops"] = round(ms, 4), rate(R, ms)
            if "b" in args.arms:
                T = R // 256
                f8 = frames.to(torch.uint8).view(T, 256, *cfg.obs_shape["rgb"])
                ms = median_ms(lambda: m.encode(f8, None), args.reps, args.warmup)
                res[f"b_model_encode_R{R}_ms"], res[f"b_model_encode_R{R}_tflops"] = round(ms, 4), rate(R, ms)
            if "c" in args.arms:
                ms = median_ms(lambda: eager_encode(sd, cfg, frames, shift), args.reps, args.warmup)
                res[f"c_eager_cudnn_R{R}_ms"], res[f"c_eager_cudnn_R{R}_tflops"] = round(ms, 4), rate(R, ms)
                if "a" in args.arms:
                    dz = (pl.encode_pixel_rows(frames, shift) - eager_encode(sd, cfg, frames, shift)).abs().max()
                    res[f"a_vs_c_R{R}_max_abs_dz"] = float(dz)
            del frames, shift
    if "d" in args.arms:
        for E in args.envs:
            cfgE = workload("c1", num_envs=E, **over)
            plE = Planner(cfgE, E, "cuda:0")
            plE.pack(sd)
            frames, shift = frames_and_shift(cfgE, E, 8)
            ms = median_ms(lambda: plE.encode_pixels(frames, shift), args.reps, args.warmup)
            res[f"d_prologue_E{E}_ms"], res[f"d_prologue_E{E}_tflops"] = round(ms, 4), rate(E, ms)
            del plE
    res["datasheet_fp32_bound_ms"] = {R: round(R * flop / 67e12 * 1e3, 3) for R in args.frames}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
