"""Time agent.update_pi (tdmpc2.py:208-239) on the kernels against the same computation as eager fp32 PyTorch autograd
with a capturable Adam on the same GPU (TF32 off), in alternating runs.

    python scripts/bench_update_pi.py [--workloads c1 c3] [--batch 256] [--horizon 3] [--repeats 20] [--warmup 5]

zs is [horizon + 1, batch, L] (T = 4 at the reference's defaults).  The eager arm evaluates all num_q Q heads (one bmm
per layer, as the reference's vmapped ensemble does) and keeps two, updates the running scale, back-propagates the loss
into the pi MLP, clips the gradient norm and steps Adam.  Prints the GPU's name and power limit, then one JSON line per
workload with the median and the range of the milliseconds per call of each arm.
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
from tdmpc2_b200.scale import RunningScale         # noqa: E402
from tdmpc2_b200.synth import synth_state_dict     # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2              # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Eager:
    """update_pi as eager fp32 torch ops with autograd (single-task workloads)."""

    def __init__(self, cfg, sd, dev):
        self.cfg, self.dev = cfg, dev
        self.sd = {k: v.to(dev, torch.float32).clone() for k, v in sd.items() if torch.is_tensor(v)}
        self.pi = [self.sd[f"_pi.{i}.{n}"].requires_grad_(True) for i in range(3)
                   for n in (("weight", "bias", "ln.weight", "ln.bias") if i < 2 else ("weight", "bias"))]
        self.opt = torch.optim.Adam(self.pi, lr=cfg.lr, eps=1e-5, capturable=True)
        self.scale = RunningScale(cfg, dev)
        self.bins = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, device=dev)

    def _layer(self, x, w, b, g, beta):
        return F.mish(F.layer_norm(F.linear(x, w, b), (w.shape[-2],), g, beta, 1e-5))

    def step(self, zs):
        cfg, sd = self.cfg, self.sd
        x = zs
        for i in range(2):
            x = self._layer(x, *(sd[f"_pi.{i}.{n}"] for n in ("weight", "bias", "ln.weight", "ln.bias")))
        mean, log_std = F.linear(x, sd["_pi.2.weight"], sd["_pi.2.bias"]).chunk(2, dim=-1)
        log_std = sd["log_std_min"] + 0.5 * sd["log_std_dif"] * (torch.tanh(log_std) + 1)
        eps = torch.randn_like(mean)
        log_prob = (-0.5 * eps.pow(2) - log_std - 0.9189385175704956).sum(-1, keepdim=True)
        action = torch.tanh(mean + eps * log_std.exp())
        log_pi = log_prob - torch.log(F.relu(1 - action.pow(2)) + 1e-6).sum(-1, keepdim=True)
        scaled_entropy = -log_pi * (log_prob * cfg.action_dim / (log_pi + 1e-8))
        T, B = zs.shape[:2]
        h = torch.cat([zs, action], -1).reshape(1, T * B, -1).expand(cfg.num_q, -1, -1)
        for i in range(3):
            w, b = sd[f"_Qs.params.{i}.weight"], sd[f"_Qs.params.{i}.bias"]
            h = torch.baddbmm(b.unsqueeze(1), h, w.transpose(1, 2))
            if i < 2:
                if i == 0:
                    h = F.dropout(h, cfg.dropout, training=True)
                h = F.mish(F.layer_norm(h, (h.shape[-1],)) * sd[f"_Qs.params.{i}.ln.weight"].unsqueeze(1)
                           + sd[f"_Qs.params.{i}.ln.bias"].unsqueeze(1))
        qi = torch.randperm(cfg.num_q, device=self.dev)[:2]
        p = F.softmax(h[qi], dim=-1)
        v = (p * self.bins).sum(-1, keepdim=True)
        q = (torch.sign(v) * (torch.exp(v.abs()) - 1)).mean(0).view(T, B, 1)
        self.scale.update(q[0])
        qs = self.scale(q)
        rho = torch.pow(cfg.rho, torch.arange(T, device=self.dev))
        loss = (-(cfg.entropy_coef * scaled_entropy + qs).mean(dim=(1, 2)) * rho).mean()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(self.pi, cfg.grad_clip_norm)
        self.opt.step()
        self.opt.zero_grad(set_to_none=True)


def time_arm(fn, zs, repeats, warmup):
    for _ in range(warmup):
        fn(zs)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
        fn(zs)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["c1", "c3"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--horizon", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update_pi.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    print(gpu_info())
    dev = torch.device("cuda")
    for wl in args.workloads:
        cfg = workload(wl, num_envs=1)
        sd = synth_state_dict(cfg, seed=1, perturb=True)
        agent = TDMPC2(cfg, device=dev)
        agent.model.load_state_dict(sd)
        agent.model.train()                                   # update_pi runs inside _update, in train mode
        eager = Eager(cfg, sd, dev)
        g = torch.Generator(device=dev).manual_seed(0)
        zs = torch.softmax(torch.randn(args.horizon + 1, args.batch, cfg.latent_dim // 8, 8, device=dev, generator=g), -1)
        zs = zs.reshape(args.horizon + 1, args.batch, -1)
        kern, eag = [], []
        for _ in range(args.rounds):                          # alternating runs of the two arms
            kern.append(time_arm(lambda z: agent.update_pi(z, None), zs, args.repeats, args.warmup))
            eag.append(time_arm(eager.step, zs, args.repeats, args.warmup))
        med = lambda v: sorted(v)[len(v) // 2]
        print(json.dumps({"workload": wl, "T": args.horizon + 1, "B": args.batch, "kernels_ms": round(med(kern), 4),
                          "kernels_ms_range": [round(min(kern), 4), round(max(kern), 4)], "eager_ms": round(med(eag), 4),
                          "eager_ms_range": [round(min(eag), 4), round(max(eag), 4)], "speedup": round(med(eag) / med(kern), 3)}))


if __name__ == "__main__":
    main()
