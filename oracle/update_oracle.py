"""CPU oracle of agent._update (the world model's training step) -- TEST INFRASTRUCTURE ONLY.

`update_oracle` restates TDMPC2._update (reference tdmpc2/tdmpc2.py:259-333) on the world model's state dict with every
draw explicit (the TD target's pi noise and Q pair, the dropout scale of Q layer 0 per head, update_pi's draws) and takes
its gradients from torch autograd on the CPU, in fp32 (the reference's arithmetic) or float64 (an error yardstick):

    encode(obs[1:]) -> _td_target (no grad) -> encode(obs[0]) -> H x next -> Q 'all' (dropout) / reward / termination
    -> consistency, reward, value, termination losses -> backward -> clip_grad_norm_ -> Adam
    -> update_pi(zs.detach()) (oracle/pi_oracle.py) -> soft_update_target_Q

The task embedding follows nn.Embedding(max_norm=1): the looked-up rows are renormalised in place at the step's first
lookup and again at update_pi's, and the embedding gradient the previous update_pi left (`emb_grad`) is added to before
clipping, as in the reference, whose pi_optim does not own the embedding.
"""
from __future__ import annotations

import os
import sys
from typing import Dict, Optional

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.pi_oracle import update_pi_oracle          # noqa: E402
from oracle.wm_oracle import QS, TARGET, WMOracle      # noqa: E402


def wm_groups(cfg, keys):
    """The reference's optim groups (tdmpc2.py:22-30) as state-dict keys: encoder, dynamics, reward, termination, Qs,
    task embedding."""
    grp = lambda pfx: [k for k in keys if k.startswith(pfx)]
    return [grp("_encoder."), grp("_dynamics."), grp("_reward."), grp("_termination.") if cfg.episodic else [],
            grp(QS), ["_task_emb.weight"] if cfg.multitask else []]


@torch.no_grad()
def renorm_rows(W: torch.Tensor, task: torch.Tensor) -> None:
    """nn.Embedding(max_norm=1)'s in-place renormalisation of the looked-up rows."""
    idx = torch.unique(task.long())
    n = torch.linalg.vector_norm(W[idx], dim=-1, keepdim=True)
    W[idx] = torch.where(n > 1, W[idx] * (1.0 / (n + 1e-7)), W[idx])


def _two_hot(x, cfg):
    x = torch.clamp(torch.sign(x) * torch.log(1 + torch.abs(x)), cfg.vmin, cfg.vmax).squeeze(-1)
    idx = torch.floor((x - cfg.vmin) / cfg.bin_size)
    off = ((x - cfg.vmin) / cfg.bin_size - idx).unsqueeze(-1)
    out = torch.zeros(*x.shape, cfg.num_bins, dtype=x.dtype, device=x.device)
    idx = idx.long().unsqueeze(-1)
    out = out.scatter(-1, idx, 1 - off)
    return out.scatter(-1, (idx + 1) % cfg.num_bins, off)


def soft_ce(pred, target, cfg):
    """math.py:5-9."""
    return -(_two_hot(target, cfg) * F.log_softmax(pred, dim=-1)).sum(-1, keepdim=True)


def split_act(x):
    """x as the kernels' forward stores a layer input: two fp16 planes hi = fp16(x), lo = fp16(x - hi); the gradient
    passes straight through."""
    hi = x.detach().half().to(x.dtype)
    return x + (hi + (x.detach() - hi).half().to(x.dtype) - x.detach())


def _net(P, prefix, x, last, head=None, drop=None, V=8, split=False):
    n = 0
    while f"{prefix}.{n}.weight" in P:
        n += 1
    for i in range(n):
        w, b = P[f"{prefix}.{i}.weight"], P[f"{prefix}.{i}.bias"]
        g, beta = P.get(f"{prefix}.{i}.ln.weight"), P.get(f"{prefix}.{i}.ln.bias")
        if head is not None:
            w, b = w[head], b[head]
            g, beta = (None, None) if g is None else (g[head], beta[head])
        x = F.linear(split_act(x) if split else x, w, b)
        if g is None:
            continue
        if i == 0 and drop is not None:
            x = x * drop
        x = F.layer_norm(x, (x.shape[-1],), g, beta, 1e-5)
        if i < n - 1:
            x = F.mish(x)
        else:
            assert last == "simnorm"
            shp = x.shape
            x = F.softmax(x.view(*shp[:-1], -1, V), dim=-1).view(shp)
    return x


def update_oracle(cfg, sd: Dict[str, torch.Tensor], obs, action, reward, terminated, task, td_eps, td_qidx, drop,
                  pi_eps, pi_qidx, pi_drop, scale_value=1.0, dtype=torch.float32, emb_grad=None, adam_state=None,
                  pi_adam_state=None, split=False):
    """One _update.  obs [H+1, B, obs_dim], action [H, B, A], reward / terminated [H, B, 1], task [B] or None;
    td_eps [H, B, A], td_qidx [2]; drop / pi_drop [num_q, H(+1), B, M] or None; pi_eps [H+1, B, A], pi_qidx [2].
    Returns a dict: the losses, grads (by key, before clipping), grad_norm, sd (the state dict after the step, the
    target soft update and update_pi), pi (update_pi_oracle's result), emb_grad (the embedding gradient update_pi
    leaves), adam / pi_adam states, zs.  `split`: every Linear of the world-model loss reads its input rounded as the
    kernels' forward stores it (split_act), for a yardstick on the kernels' rounded operands."""
    P = {k: (v.detach().to(dtype).clone() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}
    for k in list(P):
        if k.startswith("_detach_Qs_params."):
            P[k] = P[QS + k[len("_detach_Qs_params."):]]
    obs, action, reward, terminated = (x.to(dtype) for x in (obs, action, reward, terminated))
    H, B = action.shape[:2]
    mt = cfg.multitask
    if mt:
        renorm_rows(P["_task_emb.weight"], task)
    taskHB = task.long().unsqueeze(0).expand(H, B) if mt else None
    with torch.no_grad():
        wm = WMOracle(cfg, P, dtype)
        next_z = wm.encode(obs[1:], taskHB)
        td = wm.td_target(next_z, reward, terminated, taskHB, td_eps, td_qidx)

    keys = [k for g in wm_groups(cfg, list(sd.keys())) for k in g]
    for k in keys:
        P[k].requires_grad_(True)
    cat = (lambda x, t: torch.cat([x, P["_task_emb.weight"][t.long()]], dim=-1)) if mt else (lambda x, t: x)
    z = _net(P, "_encoder.state", cat(obs[0], task), "simnorm", V=cfg.simnorm_dim, split=split)
    zs, cons = [z], 0
    for t in range(H):
        z = _net(P, "_dynamics", torch.cat([cat(z, task), action[t]], dim=-1), "simnorm", V=cfg.simnorm_dim, split=split)
        cons = cons + F.mse_loss(z, next_z[t]) * cfg.rho ** t
        zs.append(z)
    Z = torch.stack(zs)
    x = torch.cat([cat(Z[:-1], taskHB), action], dim=-1)
    qs = torch.stack([_net(P, QS[:-1], x, "none", head=h, drop=None if drop is None else drop[h].to(dtype), split=split)
                      for h in range(cfg.num_q)])
    rp = _net(P, "_reward", x, "none", split=split)
    rew_loss, val_loss = 0, 0
    for t in range(H):
        rew_loss = rew_loss + soft_ce(rp[t], reward[t], cfg).mean() * cfg.rho ** t
        for h in range(cfg.num_q):
            val_loss = val_loss + soft_ce(qs[h, t], td[t], cfg).mean() * cfg.rho ** t
    cons, rew_loss, val_loss = cons / H, rew_loss / H, val_loss / (H * cfg.num_q)
    if cfg.episodic:
        term_pred = _net(P, "_termination", Z[1:], "none", split=split)
        term_loss = F.binary_cross_entropy_with_logits(term_pred, terminated)
    else:
        term_loss = torch.zeros((), dtype=dtype)
    total = (cfg.consistency_coef * cons + cfg.reward_coef * rew_loss + cfg.termination_coef * term_loss
             + cfg.value_coef * val_loss)
    total.backward()
    if mt and emb_grad is not None:
        P["_task_emb.weight"].grad += emb_grad.to(dtype)
    grads = {k: P[k].grad.detach().clone() for k in keys}
    params = [P[k] for k in keys]
    norm = torch.nn.utils.clip_grad_norm_(params, cfg.grad_clip_norm)
    groups = wm_groups(cfg, list(sd.keys()))
    opt = torch.optim.Adam([{"params": [P[k] for k in groups[0]], "lr": cfg.lr * cfg.enc_lr_scale}]
                           + [{"params": [P[k] for k in g]} for g in groups[1:]], lr=cfg.lr, capturable=False)
    if adam_state is not None:
        opt.load_state_dict(adam_state)
    opt.step()
    after = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in P.items()}
    if mt:
        renorm_rows(after["_task_emb.weight"], task)
    pi = update_pi_oracle(cfg, after, Z.detach(), task, pi_eps, pi_qidx, pi_drop, scale_value, dtype=dtype,
                          steps_state=pi_adam_state)
    after.update(pi["params"])
    with torch.no_grad():
        for k in sd:
            if k.startswith(TARGET):
                after[k] = torch.lerp(after[k], after[QS + k[len(TARGET):]], cfg.tau)
    out = dict(consistency_loss=cons.detach(), reward_loss=rew_loss.detach(), value_loss=val_loss.detach(),
               termination_loss=term_loss.detach(), total_loss=total.detach(), grad_norm=norm.detach(), grads=grads,
               sd=after, pi=pi, emb_grad=pi["grads"].get("_task_emb.weight"), adam=opt.state_dict(), pi_adam=pi["adam"],
               zs=Z.detach(), td=td.detach())
    if cfg.episodic:
        out["term_pred"] = term_pred.detach()
    return out


# --------------------------------------------------------------------------- cases
# name -> (workload, overrides, weight seed, emb_scale, H, B, input seed, dropout)
CASES = {
    "tiny_update": ("tiny", {}, 41, 1.0, 3, 40, 800, False),
    "tiny_mt_update": ("tiny-mt", {}, 42, 60.0, 3, 40, 810, False),       # per-row tasks; max_norm renormalises
    "tiny_episodic_update": ("tiny", {"episodic": True}, 43, 1.0, 3, 40, 820, False),
    "tiny_dropout_update": ("tiny", {}, 44, 1.0, 3, 40, 830, True),
    "c1_dog5m_update": ("c1", {}, 45, 1.0, 3, 16, 840, False),
    "tiny_corner_update": ("tiny", {"action_dim": 128, "num_bins": 256, "latent_dim": 8}, 46, 1.0, 2, 12, 850, False),
    "tiny_h1_update": ("tiny", {}, 47, 1.0, 1, 24, 860, False),
}


def case_model(name):
    from oracle.wm_oracle import with_target_blend
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    wl, over, wseed, emb_scale, H, B = CASES[name][:6]
    cfg = workload(wl, **over, horizon=H, batch_size=B)        # the reference's _update sizes zs by these
    sd = synth_state_dict(cfg, seed=wseed, perturb=True, emb_scale=emb_scale)
    if cfg.episodic:
        from oracle.plan_oracle import balance_termination
        balance_termination(cfg, sd)
    return cfg, with_target_blend(cfg, sd, wseed + 100)


def case_inputs(cfg, name, step=0):
    """Inputs and explicit draws of a case's step `step`.  Some rewards sit on bin centres, at +-symexp(vmax) and beyond
    the clamp, so that two_hot's floor, wrap and clamp are all reached."""
    *_, H, B, seed, dropout = CASES[name]
    g = torch.Generator().manual_seed(seed + 17 * step)
    A, M, nq = cfg.action_dim, cfg.mlp_dim, cfg.num_q
    obs = torch.randn(H + 1, B, cfg.obs_shape["state"][0], generator=g)
    action = torch.rand(H, B, A, generator=g) * 2 - 1
    reward = torch.randn(H, B, 1, generator=g) * 3
    centres = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins)
    sym = lambda v: torch.sign(v) * (torch.exp(torch.abs(v)) - 1)
    special = torch.cat([sym(centres[torch.randint(0, cfg.num_bins, (4,), generator=g)]),
                         sym(torch.tensor([cfg.vmax, cfg.vmin])), torch.tensor([1e6, -1e6, 0.0])])
    reward.view(-1)[:special.numel()] = special[: reward.numel()]
    terminated = (torch.rand(H, B, 1, generator=g) < 0.3).float() if cfg.episodic else torch.zeros(H, B, 1)
    task = torch.randint(0, len(cfg.tasks), (B,), generator=g) if cfg.multitask else None
    keep = 1.0 - cfg.dropout
    # train mode always applies Dropout(cfg.dropout) to Q layer 0: cases without dropout pass all-ones masks explicitly
    mask = lambda T: (torch.rand(nq, T, B, M, generator=g) < keep).float() / keep if dropout else torch.ones(nq, T, B, M)
    return dict(obs=obs, action=action, reward=reward, terminated=terminated, task=task,
                td_eps=torch.randn(H, B, A, generator=g), td_qidx=torch.randperm(nq, generator=g)[:2],
                drop=mask(H), pi_eps=torch.randn(H + 1, B, A, generator=g), pi_qidx=torch.randperm(nq, generator=g)[:2],
                pi_drop=mask(H + 1), scale0=torch.tensor([1.0 + 3.0 * float(torch.rand(1, generator=g))]))


def run_case(name, steps=1, dtype=torch.float32):
    """`steps` consecutive oracle steps of a case -> (cfg, sd before, list of (inputs, result))."""
    cfg, sd = case_model(name)
    cur, emb_grad, adam, pi_adam, scale = sd, None, None, None, None
    out = []
    for s in range(steps):
        inp = case_inputs(cfg, name, s)
        scale = inp["scale0"] if scale is None else scale
        r = update_oracle(cfg, cur, inp["obs"], inp["action"], inp["reward"], inp["terminated"], inp["task"],
                          inp["td_eps"], inp["td_qidx"], inp["drop"], inp["pi_eps"], inp["pi_qidx"], inp["pi_drop"],
                          scale_value=scale, dtype=dtype, emb_grad=emb_grad, adam_state=adam, pi_adam_state=pi_adam)
        out.append((inp, r))
        cur, emb_grad, adam, pi_adam, scale = r["sd"], r["emb_grad"], r["adam"], r["pi_adam"], r["pi"]["scale"]
    return cfg, sd, out


# --------------------------------------------------------------------------- golden fixtures from the reference
# name -> (case, steps): consecutive steps on one agent -- the embedding gradient update_pi leaves, both renormalisations
MULTI_STEP = {"tiny_mt_update_3steps": ("tiny_mt_update", 3)}
SUB_NUMEL = 2048       # tensors are recorded as their first SUB_NUMEL elements (flattened) to keep the fixtures small
INFO_KEYS = ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss", "grad_norm", "pi_loss",
             "pi_grad_norm", "pi_entropy", "pi_scaled_entropy", "pi_scale")


def _ref_key(name: str) -> str:
    """A harness parameter name -> the state-dict key (`_Qs.p.0/weight` -> `_Qs.params.0.weight`)."""
    if name.startswith("_Qs.p."):
        return QS + name[len("_Qs.p."):].replace("/", ".")
    return name


def reference_update(cfg, sd, xs):
    """Consecutive steps of the reference's own _update on one harness agent (oracle/ref_harness.py), one per inputs
    dict in `xs`, with the case's draws: its randn_like / randperm calls return td_eps, td_qidx, pi_eps, pi_qidx in the
    reference's order, and the Q ensemble applies the recorded dropout masks ("drop" for the value loss, "pi_drop" for
    update_pi).  Returns the info dict of every step, the last step's gradients before clipping, the state after the
    last step (target Q included) and the embedding gradient left behind."""
    x = xs[0]
    import torch.nn as nn
    from oracle import ref_harness as rh
    from oracle.wm_oracle import attach_target_qs
    rh._import_reference()
    sys.path.insert(0, rh.REF_DIR)
    try:
        from common.scale import RunningScale
    finally:
        sys.path.remove(rh.REF_DIR)
    agent = rh.build_agent(cfg, sd)
    attach_target_qs(agent, sd)                                     # the target ensemble the TD target reads
    ens = agent.model._Qs
    masks = [m_ for xx in xs for m_ in (xx["drop"], xx["pi_drop"])]

    class MaskedEnsemble(nn.Module):                                 # Q layer 0's train-mode dropout, recorded masks
        def __init__(self, detach):
            super().__init__()
            self.p, self.detach = ens.p, detach

        def forward(self, xx):
            mask = masks.pop(0)
            outs = []
            for h in range(cfg.num_q):
                P = {k.replace("/", "."): (v.detach() if self.detach else v)[h] for k, v in self.p.items()}
                y = F.linear(xx, P["0.weight"], P["0.bias"]) * mask[h]
                y = F.mish(F.layer_norm(y, (y.shape[-1],), P["0.ln.weight"], P["0.ln.bias"], 1e-5))
                y = F.mish(F.layer_norm(F.linear(y, P["1.weight"], P["1.bias"]), (y.shape[-1],), P["1.ln.weight"],
                                        P["1.ln.bias"], 1e-5))
                outs.append(F.linear(y, P["2.weight"], P["2.bias"]))
            return torch.stack(outs)
    m = agent.model
    m._Qs = MaskedEnsemble(False)
    m._detach_Qs = MaskedEnsemble(True)
    tq = m._target_Qs

    @torch.no_grad()
    def soft_update_target_Q():                                      # stands in for the tensordict lerp_ (world_model.py:86)
        for k, p in tq.p.items():
            p.lerp_(ens.p[k].detach(), cfg.tau)
    m.soft_update_target_Q = soft_update_target_Q
    scale = RunningScale.__new__(RunningScale)                       # its __init__ places the buffers on cuda:0
    nn.Module.__init__(scale)
    scale.cfg = cfg
    scale.value = torch.nn.Buffer(x["scale0"].clone())
    scale._percentiles = torch.nn.Buffer(torch.tensor([5, 95], dtype=torch.float32))
    agent.scale = scale
    agent.optim = torch.optim.Adam([                                 # tdmpc2.py:22-30, capturable=False on the CPU
        {"params": m._encoder.parameters(), "lr": cfg.lr * cfg.enc_lr_scale},
        {"params": m._dynamics.parameters()},
        {"params": m._reward.parameters()},
        {"params": m._termination.parameters() if cfg.episodic else []},
        {"params": m._Qs.parameters()},
        {"params": m._task_emb.parameters() if cfg.multitask else []}], lr=cfg.lr, capturable=False)
    agent.pi_optim = torch.optim.Adam(m._pi.parameters(), lr=cfg.lr, eps=1e-5, capturable=False)
    names = {id(p): _ref_key(n) for n, p in m.named_parameters()}
    grads = {}
    real_clip, real_randn_like, real_randperm = torch.nn.utils.clip_grad_norm_, torch.randn_like, torch.randperm
    eps_q = [e for xx in xs for e in (xx["td_eps"], xx["pi_eps"])]
    qidx_q = [q for xx in xs for q in (xx["td_qidx"], xx["pi_qidx"])]
    ncalls = []

    def clip(params, max_norm, *a, **k):
        params = list(params)
        ncalls.append(1)
        if len(ncalls) == 2 * len(xs) - 1:                           # the last step's first call clips the world model
            for p in params:
                if p.grad is not None:
                    grads[names[id(p)]] = p.grad.detach().clone()
        return real_clip(params, max_norm, *a, **k)

    def randn_like(t, *a_, **k):
        out = eps_q.pop(0)
        assert out.shape == t.shape
        return out.clone().to(t.dtype)

    def randperm(n, *a_, **k):
        q = qidx_q.pop(0).long()
        rest = [i for i in range(n) if i not in q.tolist()]
        return torch.cat([q, torch.tensor(rest, dtype=torch.long)])
    torch.randn_like, torch.randperm, torch.nn.utils.clip_grad_norm_ = randn_like, randperm, clip
    try:
        infos = [agent._update(xx["obs"], xx["action"], xx["reward"], xx["terminated"], xx["task"]) for xx in xs]
    finally:
        torch.randn_like, torch.randperm, torch.nn.utils.clip_grad_norm_ = real_randn_like, real_randperm, real_clip
    assert not masks and not eps_q and not qidx_q, "the reference made a different number of draws"
    params = {_ref_key(n): p.detach().clone() for n, p in m.named_parameters() if not n.startswith("_target_Qs.")}
    params.update({TARGET + k.replace("/", "."): p.detach().clone() for k, p in tq.p.items()})
    emb_grad = m._task_emb.weight.grad.detach().clone() if cfg.multitask else None
    return infos, grads, params, emb_grad


def _cut(v):
    return v.reshape(-1)[:SUB_NUMEL].numpy()


def main(only=None):
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name in list(CASES) + list(MULTI_STEP):
        if only and name not in only:
            continue
        base, steps = MULTI_STEP.get(name, (name, 1))
        cfg, sd = case_model(base)
        infos, grads, params, emb_grad = reference_update(cfg, sd, [case_inputs(cfg, base, s) for s in range(steps)])
        rec = dict(case=name, weight_checksum=state_dict_checksum(sd), torch_version=torch.__version__, adam_capturable=False)
        for s, info in enumerate(infos):
            for k, v in info.items():
                rec[("info/" if s == 0 else f"info{s}/") + k] = v.detach().numpy()
        for k, v in grads.items():
            rec["grad/" + k] = _cut(v)
        for k, v in params.items():
            rec["param/" + k] = _cut(v)
        if emb_grad is not None:
            rec["emb_grad_after"] = emb_grad.numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **rec)
        print(f"{name} -> tests/golden/{name}.npz")


def load_case(name):
    """(cfg, sd, inputs, fixture dict of tensors) of a golden case."""
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    f = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
    cfg, sd = case_model(MULTI_STEP.get(name, (name, 1))[0])
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), "synthetic weights differ from the fixture's"
    want = {k: torch.from_numpy(f[k]) for k in f.files if k not in ("case", "torch_version")}
    return cfg, sd, case_inputs(cfg, MULTI_STEP.get(name, (name, 1))[0]), want


if __name__ == "__main__":
    main(sys.argv[1:] or None)
