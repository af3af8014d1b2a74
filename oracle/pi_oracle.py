"""CPU oracle and golden fixtures of agent.update_pi -- TEST INFRASTRUCTURE ONLY.

`update_pi_oracle` restates TDMPC2.update_pi (reference tdmpc2/tdmpc2.py:208-239) on the world model's state dict with
every draw explicit (pi's eps, the dropout scale of Q layer 0 per head, the two Q heads) and takes its gradients from
torch autograd on the CPU, in fp32 (the reference's arithmetic) or float64 (an error yardstick for fp32 results):

    pi(zs) -> Q 'avg' of the detached online heads -> RunningScale update -> loss -> backward -> clip_grad_norm_ -> Adam

    python -m oracle.pi_oracle [names]     # mints tests/golden/<name>_pi.npz from the reference's own update_pi

The fixtures run the reference's update_pi through oracle/ref_harness.py with Adam(capturable=False) on the CPU (the
reference uses capturable=True on its GPU; the step's arithmetic is the same) and, for dropout cases, a Q ensemble
that applies the case's recorded masks.
"""
from __future__ import annotations

import os
import sys
import time
from typing import Dict

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PI_KEYS = [f"_pi.{i}.{n}" for i in range(3) for n in (("weight", "bias", "ln.weight", "ln.bias") if i < 2 else ("weight", "bias"))]


def percentile_scale(x: torch.Tensor, value: torch.Tensor, tau: float) -> torch.Tensor:
    """RunningScale.update (common/scale.py) on x [B, 1]: value lerped towards max(p95 - p5, 1) by tau."""
    n = x.shape[0]
    xs = torch.sort(x.flatten(1), dim=0).values
    pos = torch.tensor([5.0, 95.0], dtype=torch.float32) * (n - 1) / 100
    lo = torch.floor(pos)
    hi = torch.clamp(lo + 1, max=n - 1)
    w = (pos - lo).unsqueeze(1)
    p = (xs[lo.long()] * (1.0 - w) + xs[hi.long()] * w).to(x.dtype)
    return torch.lerp(value, torch.clamp(p[1] - p[0], min=1.0).to(value.dtype), tau)


def _mlp(P, prefix, x, head=None, drop=None):
    for i in range(3):
        w, b = P[f"{prefix}.{i}.weight"], P[f"{prefix}.{i}.bias"]
        g = P.get(f"{prefix}.{i}.ln.weight")
        beta = P.get(f"{prefix}.{i}.ln.bias")
        if head is not None:
            w, b = w[head], b[head]
            g, beta = (None, None) if g is None else (g[head], beta[head])
        x = F.linear(x, w, b)
        if g is not None:
            if i == 0 and drop is not None:
                x = x * drop                                       # nn.Dropout: x * (mask / (1 - p))
            x = F.mish(F.layer_norm(x, (x.shape[-1],), g, beta, 1e-5))
    return x


def update_pi_oracle(cfg, sd: Dict[str, torch.Tensor], zs, task, eps, qidx, drop=None, scale_value=1.0,
                     dtype=torch.float32, steps_state=None):
    """One update_pi.  zs [T, B, L]; task [B] or None; eps [T, B, A]; qidx [2]; drop [num_q, T, B, M] or None;
    scale_value: RunningScale.value before the call.  Returns a dict: loss, grads (by key, before clipping; "_task_emb.weight"
    for multi-task models), grad_norm, scale (after), params (the `_pi.*` tensors after one Adam step), entropy,
    scaled_entropy, q.  `steps_state`: an Adam state dict to continue from (successive steps)."""
    from oracle.plan_oracle import two_hot_inv
    P = {k: (v.detach().to(dtype).clone() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}
    for k in PI_KEYS:
        P[k].requires_grad_(True)
    zs, eps = zs.to(dtype), eps.to(dtype)
    T, B = zs.shape[:2]
    x = zs
    if cfg.multitask:
        W = P["_task_emb.weight"].requires_grad_(True)
        with torch.no_grad():                                      # nn.Embedding(max_norm=1): renormalised rows
            n = torch.linalg.vector_norm(W, dim=-1, keepdim=True)
            Wr = torch.where(n > 1, W * (1.0 / (n + 1e-7)), W)
        emb = (W + (Wr - W).detach())[task.long()].unsqueeze(0).expand(T, B, -1)
        x = torch.cat([zs, emb], dim=-1)
    mean, log_std = _mlp(P, "_pi", x).chunk(2, dim=-1)
    log_std = P["log_std_min"] + 0.5 * P["log_std_dif"] * (torch.tanh(log_std) + 1)
    if cfg.multitask:
        m = P["_action_masks"][task.long()].unsqueeze(0)
        mean, log_std, eps = mean * m, log_std * m, eps * m
        size = P["_action_masks"].sum(-1)[task.long()].view(1, B, 1)
    else:
        size = eps.shape[-1]
    log_prob = (-0.5 * eps.pow(2) - log_std - 0.9189385175704956).sum(-1, keepdim=True)
    scaled_log_prob = log_prob * size
    action = torch.tanh(mean + eps * log_std.exp())
    log_pi = log_prob - torch.log(F.relu(1 - action.pow(2)) + 1e-6).sum(-1, keepdim=True)
    scaled_entropy = -log_pi * (scaled_log_prob / (log_pi + 1e-8))
    xq = torch.cat([x, action], dim=-1)
    heads = [int(h) for h in qidx]
    Qs = [two_hot_inv(_mlp(P, "_Qs.params", xq, head=h, drop=None if drop is None else drop[h].to(dtype)), cfg) for h in heads]
    q = (Qs[0] + Qs[1]) / 2
    value = torch.as_tensor(scale_value, dtype=torch.float32).reshape(1)
    new_value = percentile_scale(q[0].detach().float(), value, cfg.tau)
    qs = q / new_value.to(dtype)
    rho = torch.pow(cfg.rho, torch.arange(T)).to(dtype)
    loss = (-(cfg.entropy_coef * scaled_entropy + qs).mean(dim=(1, 2)) * rho).mean()
    loss.backward()
    params = [P[k] for k in PI_KEYS]
    grads = {k: P[k].grad.detach().clone() for k in PI_KEYS}
    if cfg.multitask:
        grads["_task_emb.weight"] = P["_task_emb.weight"].grad.detach().clone()
    norm = torch.nn.utils.clip_grad_norm_(params, cfg.grad_clip_norm)
    opt = torch.optim.Adam(params, lr=cfg.lr, eps=1e-5, capturable=False)
    if steps_state is not None:
        opt.load_state_dict(steps_state)
    opt.step()
    return dict(loss=loss.detach(), grads=grads, grad_norm=norm.detach(), scale=new_value,
                params={k: P[k].detach().clone() for k in PI_KEYS}, entropy=(-log_pi).detach(),
                scaled_entropy=scaled_entropy.detach(), q=q.detach(), action=action.detach(), adam=opt.state_dict())


# --------------------------------------------------------------------------- golden fixtures
# name -> (workload, overrides, weight seed, emb_scale, T, B, input seed, dropout)
CASES = {
    "tiny_pi": ("tiny", {}, 31, 1.0, 3, 40, 700, False),
    "tiny_mt_pi": ("tiny-mt", {}, 32, 60.0, 3, 40, 710, False),          # per-row tasks: masks and the embedding gradient
    "c1_dog5m_pi": ("c1", {}, 33, 1.0, 2, 16, 720, False),
    "tiny_dropout_pi": ("tiny", {}, 34, 1.0, 3, 40, 730, True),           # train-mode dropout on Q layer 0
    "tiny_mt_t5_pi": ("tiny-mt", {"task_dim": 5, "action_dims": [5, 1, 4, 2]}, 35, 60.0, 2, 12, 740, False),
    "tiny_wide_heads_pi": ("tiny", {"action_dim": 128, "num_bins": 256, "latent_dim": 8}, 36, 1.0, 2, 6, 750, False),
}

SUB_NUMEL, SUB_ROWS = 65536, 32     # larger tensors are recorded for rows [0, SUB_ROWS) to keep the fixtures small


def case_model(name):
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    wl, over, wseed, emb_scale = CASES[name][:4]
    cfg = workload(wl, **over)
    return cfg, synth_state_dict(cfg, seed=wseed, perturb=True, emb_scale=emb_scale)


def case_inputs(cfg, name):
    """zs [T, B, L] (SimNorm-like latents), task [B] or None, dropout scale [num_q, T, B, M] or None, scale before."""
    *_, T, B, seed, dropout = CASES[name]
    g = torch.Generator().manual_seed(seed)
    zs = F.softmax(torch.randn(T, B, cfg.latent_dim // 8, 8, generator=g) * 3, dim=-1).reshape(T, B, -1)
    task = torch.randint(0, len(cfg.tasks), (B,), generator=g) if cfg.multitask else None
    drop = None
    if dropout:
        keep = 1.0 - cfg.dropout
        drop = (torch.rand(cfg.num_q, T, B, cfg.mlp_dim, generator=g) < keep).float() / keep
    scale0 = torch.tensor([1.0 + 3.0 * float(torch.rand(1, generator=g))])
    return zs, task, drop, scale0


def _reference_update_pi(cfg, sd, zs, task, drop, scale0, seed):
    """The reference's own update_pi on the harness agent; returns its info, the draws, grads before clipping and
    the parameters after the step."""
    from oracle import ref_harness as rh
    layers, init, WorldModel, ref = rh._import_reference()
    sys.path.insert(0, rh.REF_DIR)
    try:
        from common.scale import RunningScale
    finally:
        sys.path.remove(rh.REF_DIR)
    agent = rh.build_agent(cfg, sd)
    if drop is not None:                                   # a Q ensemble that applies the case's masks, head by head
        ens = agent.model._Qs

        class MaskedEnsemble(nn.Module):
            def __init__(self):
                super().__init__()
                self.p = ens.p

            def forward(self, x):
                outs = []
                for h in range(cfg.num_q):
                    params = {k.replace("/", "."): v[h] for k, v in self.p.items()}
                    mask = drop[h]
                    lin = lambda xx, w, b: F.linear(xx, w, b)
                    y = lin(x, params["0.weight"], params["0.bias"]) * mask
                    y = F.mish(F.layer_norm(y, (y.shape[-1],), params["0.ln.weight"], params["0.ln.bias"], 1e-5))
                    y = F.mish(F.layer_norm(lin(y, params["1.weight"], params["1.bias"]), (y.shape[-1],),
                                            params["1.ln.weight"], params["1.ln.bias"], 1e-5))
                    outs.append(lin(y, params["2.weight"], params["2.bias"]))
                return torch.stack(outs)
        agent.model._Qs = MaskedEnsemble()
    agent.model._detach_Qs = agent.model._Qs
    scale = RunningScale.__new__(RunningScale)                 # its __init__ places the buffers on cuda:0
    nn.Module.__init__(scale)
    scale.cfg = cfg
    scale.value = torch.nn.Buffer(scale0.clone())
    scale._percentiles = torch.nn.Buffer(torch.tensor([5, 95], dtype=torch.float32))
    agent.scale = scale
    agent.pi_optim = torch.optim.Adam(agent.model._pi.parameters(), lr=cfg.lr, eps=1e-5, capturable=False)
    grads = {}
    real_clip = torch.nn.utils.clip_grad_norm_

    def clip(params, max_norm, *a, **k):
        params = list(params)
        for i, p in enumerate(params):
            grads[i] = p.grad.detach().clone()
        return real_clip(params, max_norm, *a, **k)
    draws = {"eps": [], "qidx": []}
    real_randn_like, real_randperm = torch.randn_like, torch.randperm

    def randn_like(x, *a_, **k):
        out = real_randn_like(x, *a_, **k)
        draws["eps"].append(out.clone())
        return out

    def randperm(n, *a_, **k):
        out = real_randperm(n, *a_, **k)
        draws["qidx"].append(out[:2].clone())
        return out
    torch.manual_seed(seed)
    torch.randn_like, torch.randperm, torch.nn.utils.clip_grad_norm_ = randn_like, randperm, clip
    try:
        info = agent.update_pi(zs, task)
    finally:
        torch.randn_like, torch.randperm, torch.nn.utils.clip_grad_norm_ = real_randn_like, real_randperm, real_clip
    names = [n for n, _ in agent.model._pi.named_parameters()]
    emb_grad = agent.model._task_emb.weight.grad if cfg.multitask else None
    return dict(info=info, eps=draws["eps"][0], qidx=draws["qidx"][0],
                grads={"_pi." + n: grads[i] for i, n in enumerate(names)},
                params={"_pi." + n: p.detach().clone() for n, p in agent.model._pi.named_parameters()}, emb_grad=emb_grad)


def main(only=None):
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name in CASES:
        if only and name not in only:
            continue
        t = time.time()
        cfg, sd = case_model(name)
        zs, task, drop, scale0 = case_inputs(cfg, name)
        r = _reference_update_pi(cfg, sd, zs, task, drop, scale0, CASES[name][6] + 1)
        rec = dict(case=name, weight_checksum=state_dict_checksum(sd), torch_version=torch.__version__,
                   adam_capturable=False, eps=r["eps"].numpy(), qidx=r["qidx"].numpy(), scale_before=scale0.numpy(),
                   scale_after=r["info"]["pi_scale"].detach().numpy(), loss=r["info"]["pi_loss"].detach().numpy(),
                   grad_norm=r["info"]["pi_grad_norm"].detach().numpy(),
                   entropy=r["info"]["pi_entropy"].detach().numpy(),
                   scaled_entropy=r["info"]["pi_scaled_entropy"].detach().numpy())
        for k, v in r["grads"].items():
            rec["grad/" + k] = v[:SUB_ROWS].numpy() if v.numel() > SUB_NUMEL else v.numpy()
        for k, v in r["params"].items():
            rec["param/" + k] = v[:SUB_ROWS].numpy() if v.numel() > SUB_NUMEL else v.numpy()
        if r["emb_grad"] is not None:
            rec["grad/_task_emb.weight"] = r["emb_grad"].numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **rec)
        print(f"{name}: {time.time() - t:.1f}s -> tests/golden/{name}.npz")


def load_case(name):
    """(cfg, sd, inputs dict, fixture dict of tensors)."""
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    f = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
    cfg, sd = case_model(name)
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), "synthetic weights differ from the fixture's"
    zs, task, drop, scale0 = case_inputs(cfg, name)
    want = {k: torch.from_numpy(f[k]) for k in f.files if k not in ("case", "torch_version")}
    return cfg, sd, dict(zs=zs, task=task, drop=drop, scale0=scale0, eps=want["eps"], qidx=want["qidx"]), want


if __name__ == "__main__":
    main(sys.argv[1:] or None)
