"""CPU oracle of agent._update for pixel models (cfg.obs == 'rgb') -- TEST INFRASTRUCTURE ONLY.

`update_rgb_oracle` restates TDMPC2._update (reference tdmpc2/tdmpc2.py:259-333) on pixel observations like
oracle/update_oracle.py does on state observations, with every draw explicit and the gradients from torch autograd on
the CPU, in fp32 (the reference's arithmetic) or float64 (an error yardstick).  The encoder is the conv stack of
layers.conv (layers.py:36-59,136-150) under autograd (OracleModel.encode_rgb), with ShiftAug's shifts explicit: `shift`
[H+1, B, 2], shift[t] belonging to obs[t].  Pixel models are single-task in this build, so there is no task embedding.

    encode(obs[1:], shift[1:]) -> _td_target (no grad) -> encode(obs[0], shift[0]) -> H x next -> Q 'all' (dropout) /
    reward / termination -> the losses -> backward -> clip_grad_norm_ -> Adam -> update_pi(zs.detach()) -> soft update

    python -m oracle.update_rgb_oracle [names]      # mints tests/golden/<name>.npz from the reference's own _update
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace
from typing import Dict

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.pi_oracle import update_pi_oracle  # noqa: E402
from oracle.plan_oracle import OracleModel  # noqa: E402
from oracle.update_oracle import SUB_NUMEL, _net, reference_update, soft_ce, wm_groups  # noqa: E402
from oracle.wm_oracle import QS, TARGET, WMOracle  # noqa: E402


def encode_rgb(cfg, P, frames, shift, dtype):
    """layers.conv on frames [n, C, 64, 64] with explicit shifts [n, 2], differentiable in the conv parameters of P."""
    return OracleModel.encode_rgb(SimpleNamespace(cfg=cfg, sd=P, dtype=dtype), frames, shift)


def update_rgb_oracle(cfg, sd: Dict[str, torch.Tensor], obs, shift, action, reward, terminated, td_eps, td_qidx, drop,
                      pi_eps, pi_qidx, pi_drop, scale_value=1.0, dtype=torch.float32, adam_state=None, pi_adam_state=None,
                      split=False):
    """One _update of a pixel model.  obs [H+1, B, C, 64, 64] (values 0..255), shift [H+1, B, 2], action [H, B, A],
    reward / terminated [H, B, 1]; td_eps [H, B, A], td_qidx [2]; drop / pi_drop [num_q, H(+1), B, M] or None;
    pi_eps [H+1, B, A], pi_qidx [2].  Returns the dict of update_oracle.update_oracle.  `split`: every Linear reads its
    input rounded as the kernels' forward stores it (update_oracle.split_act); the conv layers read theirs unrounded,
    as the conv kernels are plain fp32."""
    P = {k: (v.detach().to(dtype).clone() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}
    for k in list(P):
        if k.startswith("_detach_Qs_params."):
            P[k] = P[QS + k[len("_detach_Qs_params."):]]
    obs, action, reward, terminated = (x.to(dtype) for x in (obs, action, reward, terminated))
    H, B = action.shape[:2]
    with torch.no_grad():
        wm = WMOracle(cfg, P, dtype)
        next_z = torch.stack([encode_rgb(cfg, P, obs[1 + t], shift[1 + t], dtype) for t in range(H)])
        td = wm.td_target(next_z, reward, terminated, None, td_eps, td_qidx)

    keys = [k for g in wm_groups(cfg, list(sd.keys())) for k in g]
    for k in keys:
        P[k].requires_grad_(True)
    z = encode_rgb(cfg, P, obs[0], shift[0], dtype)
    zs, cons = [z], 0
    for t in range(H):
        z = _net(P, "_dynamics", torch.cat([z, action[t]], dim=-1), "simnorm", V=cfg.simnorm_dim, split=split)
        cons = cons + F.mse_loss(z, next_z[t]) * cfg.rho ** t
        zs.append(z)
    Z = torch.stack(zs)
    x = torch.cat([Z[:-1], action], dim=-1)
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
    grads = {k: P[k].grad.detach().clone() for k in keys}
    norm = torch.nn.utils.clip_grad_norm_([P[k] for k in keys], cfg.grad_clip_norm)
    groups = wm_groups(cfg, list(sd.keys()))
    opt = torch.optim.Adam([{"params": [P[k] for k in groups[0]], "lr": cfg.lr * cfg.enc_lr_scale}]
                           + [{"params": [P[k] for k in g]} for g in groups[1:]], lr=cfg.lr, capturable=False)
    if adam_state is not None:
        opt.load_state_dict(adam_state)
    opt.step()
    after = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in P.items()}
    pi = update_pi_oracle(cfg, after, Z.detach(), None, pi_eps, pi_qidx, pi_drop, scale_value, dtype=dtype,
                          steps_state=pi_adam_state)
    after.update(pi["params"])
    with torch.no_grad():
        for k in sd:
            if k.startswith(TARGET):
                after[k] = torch.lerp(after[k], after[QS + k[len(TARGET):]], cfg.tau)
    out = dict(consistency_loss=cons.detach(), reward_loss=rew_loss.detach(), value_loss=val_loss.detach(),
               termination_loss=term_loss.detach(), total_loss=total.detach(), grad_norm=norm.detach(), grads=grads,
               sd=after, pi=pi, emb_grad=None, adam=opt.state_dict(), pi_adam=pi["adam"], zs=Z.detach(), td=td.detach())
    if cfg.episodic:
        out["term_pred"] = term_pred.detach()
    return out


# --------------------------------------------------------------------------- cases
# name -> (workload, overrides, weight seed, H, B, input seed, dropout).  The frames are regenerated from the input seed
# and guarded by a checksum.
RGB_CASES = {
    "tiny_rgb_update": ("tiny-rgb", {}, 48, 3, 6, 870, True),
    "tiny_rgb_episodic_update": ("tiny-rgb", {"episodic": True}, 49, 2, 5, 880, False),
    "c1_rgb_update": ("c1", {"obs": "rgb", "obs_channels": 9}, 50, 3, 4, 890, False),      # nc = 32, latent 512
}
# name -> (case, steps): consecutive steps on one agent -- Adam state of the conv parameters, re-packed conv weights
RGB_MULTI_STEP = {"tiny_rgb_update_2steps": ("tiny_rgb_update", 2)}


def frames_checksum(frames: torch.Tensor) -> float:
    x = frames.double().flatten()
    return float(x.sum()) + float((x * torch.linspace(0.0, 1.0, x.numel(), dtype=torch.float64)).sum())


def _balance_termination_rgb(cfg, sd, rows=64):
    """plan_oracle.balance_termination for pixel models: probe states one dynamics step from encoded random frames;
    shifts `_termination.2.bias` so that their logits mix terminated and live samples."""
    model = OracleModel(cfg, sd)
    g = torch.Generator().manual_seed(0)
    frames = torch.randint(0, 256, (rows,) + tuple(cfg.obs_shape["rgb"]), generator=g).float()
    z = model.encode_rgb(frames, torch.randint(0, 7, (rows, 2), generator=g))
    z = model.next(z, torch.rand(rows, cfg.action_dim, generator=g) * 2 - 1, None)
    lg = model.termination_logits(z, None).squeeze(1)
    bias = float(sd["_termination.2.bias"].reshape(-1)[0] - lg.median() - 0.3 * lg.std())
    sd["_termination.2.bias"] = torch.full_like(sd["_termination.2.bias"], bias)


def case_model(name):
    from oracle.wm_oracle import with_target_blend
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    wl, over, wseed, H, B = RGB_CASES[name][:5]
    cfg = workload(wl, **over, horizon=H, batch_size=B)        # the reference's _update sizes zs by these
    sd = synth_state_dict(cfg, seed=wseed, perturb=True)
    if cfg.episodic:
        _balance_termination_rgb(cfg, sd)
    return cfg, with_target_blend(cfg, sd, wseed + 100)


def case_inputs(cfg, name, step=0):
    """Inputs and explicit draws of a case's step `step`: frames obs [H+1, B, C, 64, 64] (fp32 values 0..255) and
    ShiftAug's shifts [H+1, B, 2].  Some rewards sit on bin centres, at +-symexp(vmax) and beyond the clamp."""
    *_, H, B, seed, dropout = RGB_CASES[name]
    g = torch.Generator().manual_seed(seed + 17 * step)
    A, M, nq = cfg.action_dim, cfg.mlp_dim, cfg.num_q
    obs = torch.randint(0, 256, (H + 1, B) + tuple(cfg.obs_shape["rgb"]), generator=g).float()
    action = torch.rand(H, B, A, generator=g) * 2 - 1
    reward = torch.randn(H, B, 1, generator=g) * 3
    centres = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins)
    sym = lambda v: torch.sign(v) * (torch.exp(torch.abs(v)) - 1)
    special = torch.cat([sym(centres[torch.randint(0, cfg.num_bins, (4,), generator=g)]),
                         sym(torch.tensor([cfg.vmax, cfg.vmin])), torch.tensor([1e6, -1e6, 0.0])])
    reward.view(-1)[:special.numel()] = special[: reward.numel()]
    terminated = (torch.rand(H, B, 1, generator=g) < 0.3).float() if cfg.episodic else torch.zeros(H, B, 1)
    keep = 1.0 - cfg.dropout
    # train mode always applies Dropout(cfg.dropout) to Q layer 0: cases without dropout pass all-ones masks explicitly
    mask = lambda T: (torch.rand(nq, T, B, M, generator=g) < keep).float() / keep if dropout else torch.ones(nq, T, B, M)
    return dict(obs=obs, action=action, reward=reward, terminated=terminated, task=None,
                td_eps=torch.randn(H, B, A, generator=g), td_qidx=torch.randperm(nq, generator=g)[:2],
                drop=mask(H), pi_eps=torch.randn(H + 1, B, A, generator=g), pi_qidx=torch.randperm(nq, generator=g)[:2],
                pi_drop=mask(H + 1), scale0=torch.tensor([1.0 + 3.0 * float(torch.rand(1, generator=g))]),
                shift=torch.randint(0, 7, (H + 1, B, 2), generator=g).float())


def run_case(name, steps=1, dtype=torch.float32):
    """`steps` consecutive oracle steps of a case -> (cfg, sd before, list of (inputs, result))."""
    cfg, sd = case_model(name)
    cur, adam, pi_adam, scale = sd, None, None, None
    out = []
    for s in range(steps):
        x = case_inputs(cfg, name, s)
        scale = x["scale0"] if scale is None else scale
        r = update_rgb_oracle(cfg, cur, x["obs"], x["shift"], x["action"], x["reward"], x["terminated"], x["td_eps"],
                              x["td_qidx"], x["drop"], x["pi_eps"], x["pi_qidx"], x["pi_drop"], scale_value=scale,
                              dtype=dtype, adam_state=adam, pi_adam_state=pi_adam)
        out.append((x, r))
        cur, adam, pi_adam, scale = r["sd"], r["adam"], r["pi_adam"], r["pi"]["scale"]
    return cfg, sd, out


# --------------------------------------------------------------------------- golden fixtures from the reference
def reference_update_rgb(cfg, sd, xs):
    """update_oracle.reference_update on pixel frames: ShiftAug's randint (layers.py:55) returns the case's shifts in the
    reference's order -- obs[1:]'s, one (B, 2) draw per t in order (world_model.py:110-111), then obs[0]'s -- and every
    recorded shift must be drawn."""
    queue = [sh for x in xs for sh in list(x["shift"][1:]) + [x["shift"][0]]]
    real_randint = torch.randint

    def randint(low, high, size, *a_, dtype=None, **k):
        sh = queue.pop(0)
        assert (low, high) == (0, 7) and tuple(size) == (sh.shape[0], 1, 1, 2), size
        return sh.view(size).to(dtype or torch.int64).clone()
    torch.randint = randint
    try:
        out = reference_update(cfg, sd, xs)
    finally:
        torch.randint = real_randint
    assert not queue, "the reference made a different number of ShiftAug draws"
    return out


def main(only=None):
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name in list(RGB_CASES) + list(RGB_MULTI_STEP):
        if only and name not in only:
            continue
        base, steps = RGB_MULTI_STEP.get(name, (name, 1))
        cfg, sd = case_model(base)
        xs = [case_inputs(cfg, base, s) for s in range(steps)]
        infos, grads, params, _ = reference_update_rgb(cfg, sd, xs)
        rec = dict(case=name, weight_checksum=state_dict_checksum(sd), torch_version=torch.__version__, adam_capturable=False,
                   frames_checksum=frames_checksum(torch.stack([x["obs"] for x in xs])))
        for s, info in enumerate(infos):
            for k, v in info.items():
                rec[("info/" if s == 0 else f"info{s}/") + k] = v.detach().numpy()
        for k, v in grads.items():
            rec["grad/" + k] = v.reshape(-1)[:SUB_NUMEL].numpy()
        for k, v in params.items():
            rec["param/" + k] = v.reshape(-1)[:SUB_NUMEL].numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **rec)
        print(f"{name} -> tests/golden/{name}.npz")


def load_case(name):
    """(cfg, sd, inputs of step 0, fixture dict of tensors) of a golden case; the regenerated frames are checked against
    the fixture's checksum."""
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    f = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
    base, steps = RGB_MULTI_STEP.get(name, (name, 1))
    cfg, sd = case_model(base)
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), "synthetic weights differ from the fixture's"
    fchk = frames_checksum(torch.stack([case_inputs(cfg, base, s)["obs"] for s in range(steps)]))
    assert abs(fchk - float(f["frames_checksum"])) <= 1e-12 * abs(fchk), "regenerated frames differ from the fixture's"
    want = {k: torch.from_numpy(f[k]) for k in f.files if k not in ("case", "torch_version")}
    return cfg, sd, case_inputs(cfg, base), want


if __name__ == "__main__":
    main(sys.argv[1:] or None)
