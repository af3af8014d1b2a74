"""Time agent._update (tdmpc2.py:259-333) on the kernels against the world model's loss step as eager fp32 PyTorch
autograd with a capturable Adam on the same GPU (TF32 off), in alternating rounds.

    python scripts/bench_update.py [--workloads c1 c3] [--batch 256] [--horizon 3] [--repeats 20] [--warmup 5]

The kernel arm is the whole _update: encode + TD target, the taped forward, the backward chain, the loss terms for the
info dict, clip_grad_norm_, Adam, update_pi and the target soft update.  It is also broken down into the taped forward
(tdmpc2_wm_loss_forward) and the backward chain (tdmpc2_wm_loss_backward) timed alone; the rest (no-grad targets,
re-packs, torch-side losses / clip / Adam, update_pi) is the difference.  The eager arm runs the world-model loss
(encoder, H dynamics steps, num_q Q heads with dropout, reward head), backward, clip and Adam on fp32 tensors, given the
TD targets (it does not run update_pi).  Prints the GPU's name and power limit, then one JSON line per workload.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.update_oracle import _net, soft_ce, wm_groups   # noqa: E402
from tdmpc2_b200.config import workload                     # noqa: E402
from tdmpc2_b200.synth import synth_state_dict              # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2                       # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, n):
    out = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["c1", "c3"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--horizon", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    print(gpu_info())
    for wl in args.workloads:
        cfg = workload(wl, horizon=args.horizon)
        sd = synth_state_dict(cfg, seed=5, perturb=True)
        H, B, A = args.horizon, args.batch, cfg.action_dim
        g = torch.Generator(device=dev).manual_seed(0)
        obs = torch.randn(H + 1, B, cfg.obs_shape["state"][0], device=dev, generator=g)
        action = torch.rand(H, B, A, device=dev, generator=g) * 2 - 1
        reward = torch.randn(H, B, 1, device=dev, generator=g)
        term = torch.zeros(H, B, 1, device=dev)
        agent = TDMPC2(cfg, device=dev)
        agent.model.load_state_dict(sd)

        # eager arm: fp32 leaves on the GPU
        P = {k: v.detach().to(dev, torch.float32).clone() for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}
        groups = wm_groups(cfg, list(sd.keys()))
        for grp in groups:
            for k in grp:
                P[k].requires_grad_(True)
        opt = torch.optim.Adam([{"params": [P[k] for k in groups[0]], "lr": cfg.lr * cfg.enc_lr_scale}]
                               + [{"params": [P[k] for k in gg]} for gg in groups[1:]], lr=cfg.lr, capturable=True)
        params = [P[k] for gg in groups for k in gg]
        with torch.no_grad():
            next_z = agent.model.encode(obs[1:], None)
            td = agent.model.td_target(next_z, reward, term, None)
        keep = 1.0 - cfg.dropout

        def eager():
            drop = torch.empty(cfg.num_q, H, B, cfg.mlp_dim, device=dev).bernoulli_(keep).div_(keep)
            z = _net(P, "_encoder.state", obs[0], "simnorm", V=cfg.simnorm_dim)
            zs, cons = [z], 0
            for t in range(H):
                z = _net(P, "_dynamics", torch.cat([z, action[t]], -1), "simnorm", V=cfg.simnorm_dim)
                cons = cons + F.mse_loss(z, next_z[t]) * cfg.rho ** t
                zs.append(z)
            x = torch.cat([torch.stack(zs)[:-1], action], -1)
            qs = torch.stack([_net(P, "_Qs.params", x, "none", head=h, drop=drop[h]) for h in range(cfg.num_q)])
            rp = _net(P, "_reward", x, "none")
            rho = torch.pow(cfg.rho, torch.arange(H, device=dev, dtype=torch.float32))
            rl = (soft_ce(rp, reward, cfg).mean(dim=(1, 2)) * rho).sum() / H
            vl = (soft_ce(qs, td.unsqueeze(0).expand(cfg.num_q, H, B, 1), cfg).mean(dim=(2, 3)) * rho).sum() / (H * cfg.num_q)
            loss = cfg.consistency_coef * cons / H + cfg.reward_coef * rl + cfg.value_coef * vl
            loss.backward()
            torch.nn.utils.clip_grad_norm_(params, cfg.grad_clip_norm)
            opt.step()
            opt.zero_grad(set_to_none=True)

        def kernels():
            agent._update(obs, action, reward, term)

        pl = agent.planner
        act_rows = action.reshape(H * B, A).contiguous()
        drop_rows = torch.ones(cfg.num_q, H * B, cfg.mlp_dim, device=dev)
        fwd_out = {}

        def fwd():
            fwd_out["o"] = pl.wm_loss_forward(obs[0].contiguous(), act_rows, None, drop_rows, H, B)

        fwd()
        grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in agent._wm_keys}

        def bwd():
            tape, zs, ql, rl, tl = fwd_out["o"]
            pl.wm_loss_backward(agent.model.tensor, tape, obs[0].contiguous(), act_rows, None, drop_rows, H, B, zs, ql, rl, tl,
                                next_z.contiguous(), reward.contiguous(), td.contiguous(), term.contiguous(), grads)

        for f in (eager, kernels, fwd, bwd):
            timed(f, args.warmup)
        n0 = agent.planner.launches
        kernels()
        torch.cuda.synchronize()
        launches = agent.planner.launches - n0
        res = {"eager": [], "kernels": [], "forward": [], "backward": []}
        for _ in range(args.rounds):
            res["eager"] += timed(eager, args.repeats)
            res["kernels"] += timed(kernels, args.repeats)
            res["forward"] += timed(fwd, args.repeats)
            res["backward"] += timed(bwd, args.repeats)
        summ = {k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
                for k, v in res.items()}
        print(json.dumps({"workload": wl, "batch": B, "horizon": H, "planner_row_launches_per_update": launches, **summ}))


if __name__ == "__main__":
    main()
