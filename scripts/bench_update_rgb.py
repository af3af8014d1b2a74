"""Time agent._update of a pixel model (cfg.obs = 'rgb') on the kernels against the world model's loss step as eager fp32
PyTorch autograd (cuDNN convolutions, TF32 off) with a capturable Adam on the same GPU, in alternating rounds.

    python scripts/bench_update_rgb.py [--batch 256] [--horizon 3] [--channels 9] [--repeats 10] [--warmup 3]

The workload is c1 with pixel observations (C = 9 stacked channels, num_channels = 32, latent 512).  The kernel arm is
the whole _update: encode(obs[1:]) + TD target, the taped conv forward of obs[0], the latent world-model loss forward and
backward, the conv backward chain, clip_grad_norm_, Adam, update_pi and the target soft update.  It is broken down into
the taped conv forward (tdmpc2_pixel_encode_taped) and the conv backward chain (tdmpc2_pixel_encode_backward) timed
alone; the rest is the difference.  The eager arm runs the world-model loss (ShiftAug + conv encoder of obs[0], H
dynamics steps, num_q Q heads with dropout, reward head), backward, clip and Adam, given the TD targets (it does not run
update_pi).  Prints the GPU's name and power limit, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.update_oracle import _net, soft_ce, wm_groups               # noqa: E402
from scripts.bench_update import gpu_info, timed                       # noqa: E402
from tdmpc2_b200.config import workload                                # noqa: E402
from tdmpc2_b200.planner import draw_shifts                            # noqa: E402
from tdmpc2_b200.synth import synth_state_dict                         # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2                                  # noqa: E402


def eager_encode(cfg, P, frames, shift):
    """layers.conv (layers.py:36-59,136-150) in eager fp32 on the frames' device: ShiftAug with explicit shifts,
    PixelPreprocess, 4 x Conv2d (cuDNN) with ReLU between, Flatten, SimNorm."""
    n = frames.shape[0]
    x = F.pad(frames, (3,) * 4, "replicate")
    ar = torch.linspace(-1.0 + 1 / 70, 1.0 - 1 / 70, 70, device=frames.device)[:64].unsqueeze(0).repeat(64, 1).unsqueeze(2)
    base = torch.cat([ar, ar.transpose(1, 0)], dim=2).unsqueeze(0).repeat(n, 1, 1, 1)
    x = F.grid_sample(x, base + shift.view(n, 1, 1, 2) * (2.0 / 70), padding_mode="zeros", align_corners=False)
    x = x.div(255.).sub(0.5)
    for i, (idx, stride) in enumerate(((2, 2), (4, 2), (6, 2), (8, 1))):
        x = F.conv2d(x, P[f"_encoder.rgb.{idx}.weight"], P[f"_encoder.rgb.{idx}.bias"], stride=stride)
        x = F.relu(x) if i < 3 else x
    x = x.flatten(1)
    return F.softmax(x.view(n, -1, cfg.simnorm_dim), dim=-1).view(n, -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--horizon", type=int, default=3)
    ap.add_argument("--channels", type=int, default=9)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    print(gpu_info())
    cfg = workload("c1", obs="rgb", obs_channels=args.channels, horizon=args.horizon, batch_size=args.batch)
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    H, B, A = args.horizon, args.batch, cfg.action_dim
    g = torch.Generator(device=dev).manual_seed(0)
    obs = torch.randint(0, 256, (H + 1, B) + tuple(cfg.obs_shape["rgb"]), device=dev, generator=g, dtype=torch.uint8)
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
    frames0 = obs[0].float()
    with torch.no_grad():
        next_z = agent.model.encode(obs[1:], None)
        td = agent.model.td_target(next_z, reward, term, None)
    keep = 1.0 - cfg.dropout

    def eager():
        drop = torch.empty(cfg.num_q, H, B, cfg.mlp_dim, device=dev).bernoulli_(keep).div_(keep)
        z = eager_encode(cfg, P, frames0, draw_shifts((B,), dev))
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
    shift0 = draw_shifts((B,), dev)
    out = {}

    def conv_fwd():
        out["z"], out["tape"] = pl.encode_pixel_rows_taped(frames0, shift0)

    conv_fwd()
    grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in agent._wm_keys if k.startswith("_encoder.rgb.")}
    dz = torch.randn(B, cfg.latent_dim, device=dev, generator=g) * 1e-3

    def conv_bwd():
        pl.pixel_encode_backward(agent.model.tensor, out["tape"], frames0, shift0, out["z"], dz, grads)

    for f in (eager, kernels, conv_fwd, conv_bwd):
        timed(f, args.warmup)
    res = {"eager": [], "kernels": [], "conv_forward_taped": [], "conv_backward": []}
    for _ in range(args.rounds):
        res["eager"] += timed(eager, args.repeats)
        res["kernels"] += timed(kernels, args.repeats)
        res["conv_forward_taped"] += timed(conv_fwd, args.repeats)
        res["conv_backward"] += timed(conv_bwd, args.repeats)
    summ = {k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for k, v in res.items()}
    rest = statistics.median(res["kernels"]) - statistics.median(res["conv_forward_taped"]) - statistics.median(res["conv_backward"])
    print(json.dumps({"workload": "c1-rgb", "channels": args.channels, "num_channels": cfg.num_channels, "batch": B,
                      "horizon": H, **summ, "rest_median_ms": round(rest, 3)}))


if __name__ == "__main__":
    main()
