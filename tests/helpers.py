"""Shared helpers for parity tests (tolerances are written where they are used)."""
import ast
import os

import numpy as np
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict, state_dict_checksum

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    f = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    over = ast.literal_eval(str(f["overrides"]))  # repr() of a plain dict written by oracle/make_golden.py
    cfg = workload(str(f["workload"]), **over)
    sd = synth_state_dict(cfg, seed=int(f["weight_seed"]), perturb=bool(f["perturb"]),
                          emb_scale=float(f["emb_scale"]))
    if "trained_level" in f.files:  # trained-scale fixtures: the synth.trained_scale transform they were minted with
        from tdmpc2_b200.synth import trained_scale
        sd = trained_scale(cfg, sd, str(f["trained_level"]), int(f["trained_seed"]))
    if "term_bias" in f.files:      # episodic fixtures: the calibrated termination bias they were minted with
        sd["_termination.2.bias"] = torch.full_like(sd["_termination.2.bias"], float(f["term_bias"]))
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), \
        "synthetic weights differ from the ones the golden vectors were minted with (torch RNG drift?)"
    calls = []
    for i in range(int(f["n_calls"])):
        g = lambda k: f[f"c{i}_{k}"]
        task = int(g("task"))
        calls.append(dict(obs=torch.from_numpy(g("obs")), t0=bool(g("t0")), eval_mode=bool(g("eval_mode")),
                          task=None if task < 0 else task, seed=int(g("seed")),
                          prev_mean=torch.from_numpy(g("prev_mean")), action=torch.from_numpy(g("action")),
                          mean=torch.from_numpy(g("mean")), values=torch.from_numpy(g("values")),
                          elite_idx=torch.from_numpy(g("elite_idx"))))
    return cfg, sd, calls


OBS_SCALES = (1.0, 30.0, 1e3)
OBS_BIG = 6e4          # one observation column near the top of fp16's range (the kernels clamp activations to +-65000)


def trained_model(wl, level, seed, **over):
    """(cfg, state dict) of a trained-scale model: synthetic weights (seed), a blended target ensemble (seed + 100),
    synth.trained_scale(level, seed + 200) and, for episodic models, a re-centred termination bias."""
    from oracle.plan_oracle import balance_termination
    from oracle.wm_oracle import with_target_blend
    from tdmpc2_b200.synth import trained_scale
    cfg = workload(wl, **over)
    sd = synth_state_dict(cfg, seed=seed, perturb=True, emb_scale=60.0 if cfg.multitask else 1.0)
    sd = trained_scale(cfg, with_target_blend(cfg, sd, seed + 100), level, seed + 200)
    if cfg.episodic:
        balance_termination(cfg, sd)
    return cfg, sd


def trained_obs(cfg, rows, seed):
    """[rows, obs_dim] observations whose rows cycle through the scales OBS_SCALES and a fourth kind: scale 1 with
    column 0 near +-OBS_BIG (it dominates the encoder's first LayerNorm, so only one row in four carries it)."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(rows, cfg.obs_shape["state"][0], generator=g)
    kind = torch.arange(rows) % (len(OBS_SCALES) + 1)
    obs *= torch.tensor(OBS_SCALES + (1.0,))[kind].unsqueeze(1)
    big = OBS_BIG * (0.9 + 0.1 * torch.rand(rows, generator=g)) * torch.where(torch.rand(rows, generator=g) < 0.5, -1.0, 1.0)
    obs[:, 0] = torch.where(kind == len(OBS_SCALES), big, obs[:, 0])
    return obs


def refit_stats(cfg, tr):
    """Per (env, iteration) of an oracle PlanTrace: the largest normalised elite weight, and whether the refit clamped
    some std to min_std."""
    top = torch.gather(tr.values, -1, tr.elite_idx)                          # [E, I, K] elite values, sorted
    w = torch.softmax(cfg.temperature * (top - top[..., :1]).double(), -1)   # the refit's score
    live = torch.ones_like(tr.iter_std, dtype=torch.bool)
    if cfg.multitask:
        live = tr.iter_std > 0                                               # masked action dims are zeroed after the clamp
    clamped = ((tr.iter_std == torch.tensor(cfg.min_std, dtype=tr.iter_std.dtype)) & live).flatten(2).any(-1)
    return w.max(-1).values, clamped


def stable_positions(values, k, tol):
    """bool [..., k]: sorted-top-k positions whose value is further than `tol` from
    both neighbours in the sorted order (incl. the (k+1)-th value).  Only there is
    a bit-exact sorted top-k index well defined under fp32 re-association noise."""
    top = torch.topk(values, k + 1, dim=-1).values
    gaps = top[..., :-1] - top[..., 1:]                       # [..., k]; gaps[j] = v_j - v_{j+1}
    ok_next = gaps > tol
    ok_prev = torch.cat([torch.ones_like(ok_next[..., :1]), ok_next[..., :-1]], dim=-1)
    return ok_next & ok_prev


def boundary_separated(values, k, tol):
    """bool [...]: the k-th and (k+1)-th largest values differ by more than `tol`,
    i.e. the elite SET (hence the refit mean/std) is well defined."""
    top = torch.topk(values, k + 1, dim=-1).values
    return (top[..., k - 1] - top[..., k]) > tol


def mixed_noise(cfg, E, oracle_envs, seed, device="cuda", eval_mode=False):
    """Noise for a big batch on `device`: torch-drawn for every environment, with the environments in `oracle_envs`
    overwritten by oracle-drawn (reference-order, CPU generator) noise.  Returns (planner.Noise, oracle PlanNoise of
    just those environments, in the order given)."""
    from oracle.plan_oracle import draw_noise as oracle_noise
    from tdmpc2_b200.planner import draw_noise
    g = torch.Generator(device=device).manual_seed(seed)
    nz = draw_noise(cfg, E, device, eval_mode=eval_mode, generator=g, reference_order=False)
    on = oracle_noise(cfg, seed + 17, len(oracle_envs), eval_mode=eval_mode)
    for j, e in enumerate(oracle_envs):
        nz.prior[e] = on.prior[j].to(device)
        nz.r[:, e] = on.r[j].to(device)
        nz.pi[:, e] = on.pi[j].to(device)
        nz.qidx[:, e] = on.qidx[j].to(torch.int32).to(device)
        nz.expo[e] = on.expo[j].to(device)
        if not eval_mode:
            nz.final[e] = on.final[j].to(device)
    return nz, on


def slice_noise(nz, envs):
    """The planner.Noise of a subset of environments (contiguous copies)."""
    from tdmpc2_b200.planner import Noise
    idx = torch.as_tensor(envs, device=nz.prior.device)
    return Noise(nz.prior[idx].contiguous(), nz.r[:, idx].contiguous(), nz.pi[:, idx].contiguous(),
                 nz.qidx[:, idx].contiguous(), nz.expo[idx].contiguous(),
                 None if nz.final is None else nz.final[idx].contiguous())


def compare_with_oracle(cfg, tr, action, new_mean, want, on, envs, value_atol=5e-5, value_rtol=1e-5, gap=None):
    """Kernel trace of environments `envs` (rows of the big batch) against oracle rows 0..len(envs)-1.
    values: |got - want| <= value_atol + value_rtol * |want| (the tolerance of tests/test_gpu_parity.py: fp32 round-off
    level -- the fp32 oracle itself is only that close to float64); top-k indices exact where the oracle's sorted values
    are separated by > gap (default 2 x the value tolerance at that magnitude, at least 1e-4); refit mean/std and final
    action within 1e-4 (north-star tolerance) while the elite set is unambiguous.  Returns counters so that callers can
    assert that the comparisons really ran."""
    K = cfg.num_elites
    n = dict(values=0, topk=0, refit=0, actions=0, max_value_err=0.0)
    for j, e in enumerate(envs):
        clean = True
        for it in range(cfg.iterations):
            v_got, v_want = tr["values"][e, it].cpu(), want.values[j, it]
            err = float((v_got - v_want).abs().max())
            n["max_value_err"] = max(n["max_value_err"], err)
            assert torch.allclose(v_got, v_want, atol=value_atol, rtol=value_rtol), f"values env={e} it={it} err={err:.3e}"
            n["values"] += v_want.numel()
            gap_it = gap if gap is not None else max(1e-4, 2 * (value_atol + value_rtol * float(v_want.abs().max())))
            stable = stable_positions(v_want, K, gap_it)
            assert torch.equal(tr["elite_idx"][e, it].cpu()[stable], want.elite_idx[j, it][stable]), f"top-k env={e} it={it}"
            n["topk"] += int(stable.sum())
            if not bool(boundary_separated(v_want, K, gap_it)):
                clean = False
                break
            assert torch.allclose(tr["iter_mean"][e, it].cpu(), want.iter_mean[j, it], atol=1e-4, rtol=0), f"mean env={e} it={it}"
            assert torch.allclose(tr["iter_std"][e, it].cpu(), want.iter_std[j, it], atol=1e-4, rtol=0), f"std env={e} it={it}"
            n["refit"] += 1
        if clean:
            assert torch.allclose(new_mean[e].cpu(), want.mean[j], atol=1e-4, rtol=0)
            logits = want.score[j].log() - on.expo[j].log()
            top2 = torch.topk(logits, 2).values
            if float(top2[0] - top2[1]) > 1e-3:
                assert int(tr["pick"][e].cpu()) == int(want.pick[j])
                assert torch.allclose(action[e].cpu(), want.action[j], atol=1e-4, rtol=0), f"action env={e}"
                n["actions"] += 1
    return n
