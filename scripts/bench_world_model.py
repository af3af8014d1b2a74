"""Time `encode` followed by `_td_target` (the no-grad first block of the reference's `_update`, tdmpc2.py:259-264)
on the row-mode kernels against batched eager fp32 PyTorch on the same GPU.

    python scripts/bench_world_model.py [--workload c1] [--rows 768 131072] [--repeats 20] [--warmup 5]

Rows: 768 = batch 256 x horizon 3 (the reference's training shape), ~131k = a dataset-relabelling batch.  The eager
baseline evaluates all num_q target heads and keeps two, as the reference does (world_model.py:207-213).  Prints one
JSON line per row count, after the GPU's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tdmpc2_b200.config import workload            # noqa: E402
from tdmpc2_b200.planner import discount_table     # noqa: E402
from tdmpc2_b200.synth import synth_state_dict     # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2              # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Eager:
    """The reference's math as batched fp32 torch ops (no per-head Python loop: the ensemble is one bmm per layer)."""

    def __init__(self, cfg, sd, dev):
        self.cfg = cfg
        self.sd = {k: v.to(dev, torch.float32) for k, v in sd.items() if torch.is_tensor(v)}
        self.bins = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, device=dev)
        self.disc = float(discount_table(cfg, "cpu")[0, 1])

    def mlp(self, pfx, x, n, last):
        for i in range(n):
            x = F.linear(x, self.sd[f"{pfx}.{i}.weight"], self.sd[f"{pfx}.{i}.bias"])
            if f"{pfx}.{i}.ln.weight" in self.sd:
                x = F.layer_norm(x, (x.shape[-1],), self.sd[f"{pfx}.{i}.ln.weight"], self.sd[f"{pfx}.{i}.ln.bias"])
                x = F.mish(x) if (i < n - 1 or last != "simnorm") else \
                    F.softmax(x.view(*x.shape[:-1], -1, 8), -1).view(x.shape)
        return x

    def ensemble(self, x):                              # all num_q heads: x [R, D] -> [num_q, R, B]
        x = x.unsqueeze(0).expand(self.cfg.num_q, -1, -1)
        for i in range(3):
            w, b = self.sd[f"_target_Qs_params.{i}.weight"], self.sd[f"_target_Qs_params.{i}.bias"]
            x = torch.baddbmm(b.unsqueeze(1), x, w.transpose(1, 2))
            if i < 2:
                g, beta = self.sd[f"_target_Qs_params.{i}.ln.weight"], self.sd[f"_target_Qs_params.{i}.ln.bias"]
                x = F.mish(F.layer_norm(x, (x.shape[-1],)) * g.unsqueeze(1) + beta.unsqueeze(1))
        return x

    def run(self, obs, reward, terminated, eps, qidx):
        n_enc = sum(1 for k in self.sd if k.startswith("_encoder.state.") and k.endswith(".weight") and ".ln." not in k)
        z = self.mlp("_encoder.state", obs, n_enc, "simnorm")
        mean, ls = self.mlp("_pi", z, 3, "none").chunk(2, -1)
        ls = self.sd["log_std_min"] + 0.5 * self.sd["log_std_dif"] * (torch.tanh(ls) + 1)
        a = torch.tanh(mean + eps * ls.exp())
        q = self.ensemble(torch.cat([z, a], -1))[qidx]
        q = torch.sum(F.softmax(q, -1) * self.bins, -1, keepdim=True)
        q = torch.sign(q) * (torch.exp(q.abs()) - 1)
        return reward + self.disc * (1 - terminated) * q.min(0).values


def events_ms(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c1")
    ap.add_argument("--rows", type=int, nargs="+", default=[768, 131072])
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_world_model.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    cfg = workload(args.workload)
    sd = synth_state_dict(cfg, seed=1)
    other = synth_state_dict(cfg, seed=2)
    for k in sd:                                        # target ensemble != online ensemble (a Polyak-style blend)
        if k.startswith("_target_Qs_params."):
            sd[k] = torch.lerp(sd[k], other["_Qs.params." + k[len("_target_Qs_params."):]], 0.3)
    agent = TDMPC2(cfg, device=dev)
    agent.model.load_state_dict(sd)
    eager = Eager(cfg, sd, dev)
    print(f"# GPU: {gpu_info()}")
    g = torch.Generator(device=dev).manual_seed(0)
    for R in args.rows:
        obs = torch.randn(R, cfg.obs_shape["state"][0], device=dev, generator=g)
        reward = torch.randn(R, 1, device=dev, generator=g)
        terminated = torch.zeros(R, 1, device=dev)
        eps = torch.randn(R, cfg.action_dim, device=dev, generator=g)
        qidx = torch.tensor([3, 1], device=dev)

        def kernels():
            z = agent.model.encode(obs, None)
            return agent._td_target(z, reward, terminated, None, eps=eps, qidx=qidx)

        def baseline():
            return eager.run(obs, reward, terminated, eps, qidx)

        diff = float((kernels() - baseline()).abs().max())
        k_med, k_min, k_max = events_ms(kernels, args.warmup, args.repeats)
        b_med, b_min, b_max = events_ms(baseline, args.warmup, args.repeats)
        print(json.dumps(dict(workload=args.workload, rows=R, kernels_ms=round(k_med, 4), kernels_range_ms=[round(k_min, 4), round(k_max, 4)],
                              eager_fp32_ms=round(b_med, 4), eager_range_ms=[round(b_min, 4), round(b_max, 4)],
                              speedup=round(b_med / k_med, 3), tiles=(R + 127) // 128,
                              sms=torch.cuda.get_device_properties(dev).multi_processor_count,
                              max_abs_diff_vs_eager=diff)))


if __name__ == "__main__":
    main()
