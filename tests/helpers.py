"""Shared helpers for parity tests (tolerances are written where they are used)."""
import ast
import math
import os

import numpy as np
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import head_layout, synth_state_dict, state_dict_checksum

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


def _top_k_plus_one(values, k):
    """The k + 1 largest values, sorted; when every value is an elite (k == n) the (k+1)-th is -inf."""
    if values.shape[-1] == k:
        values = torch.cat([values, torch.full_like(values[..., :1], float("-inf"))], dim=-1)
    return torch.topk(values, k + 1, dim=-1).values


def stable_positions(values, k, tol):
    """bool [..., k]: sorted-top-k positions whose value is further than `tol` from
    both neighbours in the sorted order (incl. the (k+1)-th value).  Only there is
    a bit-exact sorted top-k index well defined under fp32 re-association noise."""
    top = _top_k_plus_one(values, k)
    gaps = top[..., :-1] - top[..., 1:]                       # [..., k]; gaps[j] = v_j - v_{j+1}
    ok_next = gaps > tol
    ok_prev = torch.cat([torch.ones_like(ok_next[..., :1]), ok_next[..., :-1]], dim=-1)
    return ok_next & ok_prev


def boundary_separated(values, k, tol):
    """bool [...]: the k-th and (k+1)-th largest values differ by more than `tol`,
    i.e. the elite SET (hence the refit mean/std) is well defined."""
    top = _top_k_plus_one(values, k)
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


# ------------------------------------------------------------------------------------------------- the ratio rule
# Every quantity computed by the kernel (k), the fp32 oracle (o32) and the float64 oracle (o64) obeys
#     max|k - o64| <= RATIO * max|o32 - o64| + FLOOR * max|o64|
# (tests/test_gpu_trained_scale.py explains why a fixed tolerance cannot serve both init and trained scale).
DEV = "cuda"
RATIO = 8.0
FLOOR = 2.0 ** -23
# A product of two operands whose fp16 hi and lo parts are both normal carries <= 2^-21 relative error (two 22-bit
# operands, the lo x lo term dropped) and each output sums 3K fp32-rounded terms plus the bias; the largest of ~10^5
# outputs of that rounding walk reaches 21 x 2^-22 sum|W||x| on the H100 (the fp32 oracle's own error is of the same
# size: the ratio rule holds), so the bound is c = 32, not the 4 a single product would suggest (DESIGN.md section 2).
# Declared limit: a weight below 2^-3 / 2^k (2^k the layer's packing scale, max|W| 2^k in [128, 256)) has a subnormal
# or zero lo part, good to 2^-25 / 2^k absolutely, not relatively; an activation x multiplies that error by |x|, and
# near the +-65000 clamp this reaches the size of the c-term.  The bound carries that term explicitly (SUBNORMAL_LO).
LINEAR_C = 32.0
SUBNORMAL_LO = 2.0 ** -25
TERM_MARGIN = 2e-5          # as tests/test_gpu_parity.py: a termination decision this close to 0.5 is not defined
OBSERVED = {}               # (quantity, case) -> [worst ratio, elements compared, elements excluded]


def print_ratio_table():
    if OBSERVED:
        print(f"\n{'quantity':18s} {'case':34s} {'ratio':>7s} {'compared':>9s} {'excluded':>9s}")
        for (q, case), (r, n, x) in sorted(OBSERVED.items(), key=lambda kv: (kv[0][1], kv[0][0])):
            print(f"{q:18s} {case:34s} {r:7.2f} {n:9d} {x:9d}")


def ratio_rule(q, case, k, o32, o64, keep=None, need=0.5):
    """Asserts the ratio rule on the elements `keep` (default: all; at least the fraction `need` of them) and records
    the observed ratio."""
    k, o32, o64 = (t.detach().double().cpu().reshape(-1) for t in (k, o32, o64))
    assert k.shape == o64.shape == o32.shape, q
    keep = torch.ones_like(o64, dtype=torch.bool) if keep is None else keep.reshape(-1).cpu()
    n, x = int(keep.sum()), int((~keep).sum())
    assert n >= max(1, need * keep.numel()), f"{q}: only {n} of {keep.numel()} elements comparable"
    e_k = float((k - o64).abs()[keep].max())
    e_32 = float((o32 - o64).abs()[keep].max())
    floor = FLOOR * float(o64.abs()[keep].max())
    ratio = e_k / max(e_32, floor, 1e-300)
    old = OBSERVED.get((q, case), [0.0, 0, 0])
    OBSERVED[(q, case)] = [max(old[0], ratio), old[1] + n, old[2] + x]
    assert e_k <= RATIO * e_32 + floor, f"{q} [{case}]: |k - o64| {e_k:.3e} > {RATIO} x |o32 - o64| {e_32:.3e} + {floor:.1e}"
    return RATIO * e_32 + floor


def level_model(wl, level, **over):
    """(cfg, state dict) of workload `wl` at `level`: "init" = the synthetic initialisation with a blended target
    ensemble, otherwise trained_model(level)."""
    from oracle.plan_oracle import balance_termination
    from oracle.wm_oracle import with_target_blend
    if level != "init":
        return trained_model(wl, level, 7, **over)
    cfg = workload(wl, **over)
    sd = synth_state_dict(cfg, seed=7, perturb=True, emb_scale=60.0 if cfg.multitask else 1.0)
    if cfg.episodic:
        balance_termination(cfg, sd)
    return cfg, with_target_blend(cfg, sd, 107)


def agent_for(cfg, sd, engine):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    return agent


def symlog(x):
    return torch.sign(x) * torch.log1p(x.abs())


def row_inputs(cfg, R, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(obs=trained_obs(cfg, R, seed),
                task=torch.randint(0, len(cfg.tasks), (R,), generator=g) if cfg.multitask else None,
                a=torch.rand(R, cfg.action_dim, generator=g) * 2 - 1, eps=torch.randn(R, cfg.action_dim, generator=g),
                rew=torch.randn(R, 1, generator=g) * 100, term=(torch.rand(R, 1, generator=g) < 0.3).float(),
                qidx=torch.randperm(cfg.num_q, generator=g)[:2])


def run_methods(cfg, m, x, z, kernel):
    """Every method on inputs x (the kernels' WorldModel if `kernel`, else an oracle); z is the latent the methods
    other than encode take, so that each is checked on its own layers."""
    dv = (lambda t: None if t is None else t.to(DEV)) if kernel else (lambda t: t)
    task, a, eps = dv(x["task"]), dv(x["a"]), dv(x["eps"])
    zz = dv(z)
    out = {"z": m.encode(dv(x["obs"]), task), "next": m.next(zz, a, task), "reward": m.reward(zz, a, task)}
    if kernel:
        act, info = m.pi(zz, task, eps=eps)
        qa = lambda rt, tgt, qi: m.Q(zz, a, task, return_type=rt, target=tgt, qidx=None if qi is None else dv(qi))
    else:
        act, info = m.pi(zz, task, eps)
        qa = lambda rt, tgt, qi: m.Q(zz, a, task, rt, target=tgt, qidx=qi)
    out.update(pi_action=act, pi_mean=info["mean"], pi_log_std=info["log_std"], pi_entropy=info["entropy"],
               pi_scaled_entropy=info["scaled_entropy"], q_all=qa("all", False, None), qt_all=qa("all", True, None),
               q_min=qa("min", False, x["qidx"]), q_avg=qa("avg", False, x["qidx"].flip(0)),
               qt_min=qa("min", True, x["qidx"]))
    if kernel:
        out["td"] = m.td_target(zz, dv(x["rew"]), dv(x["term"]), task, eps=eps, qidx=dv(x["qidx"]))
    else:
        out["td"] = m.td_target(zz, x["rew"], x["term"], task, eps, x["qidx"])
    if cfg.episodic:
        out["term_logit"] = m.termination(zz, None, unnormalized=True)
    return out


def row_mode_ratio_rule(cfg, sd, tag, level, R, engines, entropy_need=None):
    """Every WorldModel method and _td_target on R rows, on each engine, by the ratio rule (case = tag/engine).
    Two-hot values are compared in the symlog domain.  Excluded: entropy rows with min(1 - a^2) <= 1e-3 or
    |log_pi| < 1e-2 (the squash term and the entropy scale are ill-conditioned there).  `entropy_need`: the fraction
    of entropy rows that must remain (default: none at "sharp", 2 % otherwise)."""
    import oracle.wm_oracle as wm
    x = row_inputs(cfg, R, 11)
    o32, o64 = wm.WMOracle(cfg, sd), wm.WMOracle(cfg, sd, torch.float64)
    z_in = o64.encode(x["obs"], x["task"]).float()          # the latent every other method reads, rounded to fp32
    want32 = run_methods(cfg, o32, x, z_in, False)
    want64 = run_methods(cfg, o64, x, z_in, False)
    a64 = want64["pi_action"]
    ok_rows = ((1 - a64 ** 2).min(-1).values > 1e-3) & (want64["pi_entropy"].reshape(-1).abs() > 1e-2)
    for engine in engines:
        m = agent_for(cfg, sd, engine).model
        got = run_methods(cfg, m, x, z_in, True)
        case = f"{tag}/{engine}"
        for q in got:
            k, w32, w64 = got[q], want32[q], want64[q]
            keep, need = None, 0.5
            if q in ("q_min", "q_avg", "qt_min"):             # two-hot values: the symlog domain
                k, w32, w64 = symlog(k.double()), symlog(w32.double()), symlog(w64)
            if q in ("pi_entropy", "pi_scaled_entropy"):
                # a row with any saturated action dim is excluded: at "sharp" that is nearly every row (the counts are
                # printed); the mid and init levels keep the entropy under test
                keep = ok_rows.reshape(k.shape)
                need = entropy_need if entropy_need is not None else 0.0 if level == "sharp" else 0.02
                if need == 0.0 and not bool(keep.any()):
                    OBSERVED.setdefault((q, case), [0.0, 0, int(keep.numel())])
                    continue
            ratio_rule(q, case, k, w32, w64, keep, need)
        del m
        torch.cuda.empty_cache()


def layer_list(cfg):
    """(layer index, state-dict prefix, head | None, has_ln, last_is_simnorm) in the packer's order."""
    lay = head_layout(cfg)
    out, li = [], 0
    for name, n in (("_encoder.state", len(lay["_encoder.state"]["dims"])), ("_dynamics", 3),
                    ("_reward", 3), ("_pi", 3)):
        for i in range(n):
            ln = i < n - 1 or name in ("_encoder.state", "_dynamics")
            out.append((li, f"{name}.{i}", None, ln, ln and i == n - 1)); li += 1
    for h in range(cfg.num_q):
        for i in range(3):
            out.append((li, f"_Qs.params.{i}", h, i < 2, False)); li += 1
    return out


def fused_layer_ratio_rule(cfg, sd, engine, case):
    """Each packed layer of (cfg, sd) through Planner.debug_layer on inputs at scales 1, 30, 1e3 and with a column
    near 6e4.  The linear output obeys the component-wise forward-error bound
    |k - y64| <= c * 2^-22 * sum_k |W_nk| |x_k| + 2^-23 |b_n| + 2^-25 / 2^k * sum_{k: W_nk tiny} |x_k|
    (c = LINEAR_C; the last term is the declared subnormal-lo limit, SUBNORMAL_LO) and the ratio rule; LayerNorm + Mish /
    SimNorm outputs obey the ratio rule.  Returns the layers compared: (prefix, head, output width, epilogue)."""
    from tdmpc2_b200.planner import Planner
    F = torch.nn.functional
    pl = Planner(cfg, 2, DEV, engine=engine)
    pl.pack(sd)
    g = torch.Generator().manual_seed(0)
    compared = []
    for (li, prefix, head, has_ln, simnorm) in layer_list(cfg):
        W, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
        if head is not None:
            W, b = W[head], b[head]
        if W.shape[1] > cfg.latent_dim + cfg.action_dim + cfg.task_dim + 64 and not prefix.startswith("_encoder"):
            continue                                  # hidden-width inputs do not fit the X scratch debug_layer reads
        rows = 128                                    # debug_layer runs one tile
        x = torch.randn(rows, W.shape[1], generator=g) * torch.tensor([1.0, 30.0, 1e3])[torch.arange(rows) % 3].unsqueeze(1)
        x[::7, 0] = 6e4
        A = cfg.action_dim
        Apad = (A + 31) // 32 * 32
        n_out = Apad + A if prefix == "_pi.2" else W.shape[0]
        try:
            y = pl.debug_layer(li, 0, x.to(DEV), n_out).cpu().double()
        except Exception as e:
            if "wider than the X scratch" in str(e):
                continue
            raise
        if prefix == "_pi.2":
            y = torch.cat([y[:, :A], y[:, Apad:Apad + A]], dim=1)
        y64 = x.double() @ W.double().T + b.double()
        scale = 2.0 ** (8 - math.frexp(float(W.abs().max()))[1])          # the packer's power of two (api.cu)
        tiny = (W.double().abs() * scale < 2.0 ** -3).double()            # weights whose lo part is subnormal or 0
        bound = (LINEAR_C * 2.0 ** -22 * (x.double().abs() @ W.double().abs().T) + FLOOR * b.double().abs()
                 + SUBNORMAL_LO / scale * (x.double().abs() @ tiny.T))
        over = float(((y - y64).abs() / bound).max())
        old = OBSERVED.get(("linear/bound", case), [0.0, 0, 0])
        OBSERVED[("linear/bound", case)] = [max(old[0], over), old[1] + y.numel(), 0]
        assert over <= 1.0, f"{prefix} head={head}: linear error {over:.2f} x the forward-error bound"
        ratio_rule("linear", case, y, F.linear(x, W, b), y64)
        compared.append((prefix, head, W.shape[0], "simnorm" if simnorm else "ln+mish" if has_ln else "linear"))
        if has_ln:
            gw, gb = sd[prefix + ".ln.weight"], sd[prefix + ".ln.bias"]
            if head is not None:
                gw, gb = gw[head], gb[head]

            def act(dt):
                h = F.layer_norm(F.linear(x.to(dt), W.to(dt), b.to(dt)), (W.shape[0],), gw.to(dt), gb.to(dt), 1e-5)
                return torch.softmax(h.view(rows, -1, 8), -1).view(rows, -1) if simnorm else F.mish(h)
            got = pl.debug_layer(li, 2 if simnorm else 1, x.to(DEV), W.shape[0])
            ratio_rule("simnorm" if simnorm else "ln+mish", case, got, act(torch.float32), act(torch.float64))
    return compared


def to_gpu_noise(n):
    from tdmpc2_b200.planner import Noise
    return Noise.from_env_major(n.prior, n.r, n.pi, n.qidx, n.expo, n.final, device=DEV)


def plan_three_ways(cfg, sd, engine, E, seed, warm=False):
    """One plan() by the kernels and by the fp32 and float64 oracles on the same inputs and noise.  Every environment
    starts afresh (t0), or with `warm` the odd ones are warm-started from a random previous mean."""
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    from tdmpc2_b200.planner import Planner
    obs = trained_obs(cfg, E, seed)
    task = [(2 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    noise = oracle_noise(cfg, 40 + seed, E)
    t0 = torch.ones(E, dtype=torch.uint8)
    prev = torch.zeros(E, cfg.horizon, cfg.action_dim)
    if warm:
        t0[1::2] = 0
        prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=torch.Generator().manual_seed(seed))
    w32 = plan_oracle(cfg, sd, obs, task=task, t0=t0.bool().tolist(), prev_mean=prev, noise=noise)
    w64 = plan_oracle(cfg, sd, obs, task=task, t0=t0.bool().tolist(), prev_mean=prev, noise=noise, dtype=torch.float64)
    pl = Planner(cfg, E, DEV, engine=engine)
    pl.pack(sd)
    taskv = torch.tensor(task, dtype=torch.int32, device=DEV) if task is not None else None
    action, new_mean, tr = pl.plan(obs.to(DEV), taskv, t0.to(DEV), prev.to(DEV), to_gpu_noise(noise), trace=True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in tr.items()}, action.cpu(), new_mean.cpu(), w32, w64, noise


def compare_plans(cfg, case, tr, action, new_mean, w32, w64, noise, pool_envs=False):
    """Values by the ratio rule per (env, iteration); top-k indices exact where float64's sorted values are separated
    by more than twice the allowed value error; refit mean / std within 1e-4 plus the value error they inherit, and
    the action within 1e-4 plus what it inherits from the refits, while the elite set is unambiguous
    (helpers.compare_with_oracle's logic).  `pool_envs`: the ratio rule takes its maximum over every environment's
    values of an iteration at once (for a handful of samples per environment, where a maximum over one environment's
    values says nothing about fp32's error).  Returns counters."""
    E, K = tr["values"].shape[0], cfg.num_elites
    n = dict(values=0, topk=0, refit=0, clamped=0, dominated=0, actions=0)
    wmax, clamped = refit_stats(cfg, w64)
    keep_all = w64.term_margin > TERM_MARGIN if cfg.episodic else torch.ones_like(w64.values, dtype=torch.bool)
    pooled = [ratio_rule("plan values", case, tr["values"][:, it], w32.values[:, it], w64.values[:, it],
                         keep_all[:, it]) for it in range(cfg.iterations)] if pool_envs else None
    for e in range(E):
        clean = True
        stable = None
        tols = []
        for it in range(cfg.iterations):
            v64 = w64.values[e, it]
            keep = keep_all[e, it]
            if pooled:
                allowed = pooled[it]
            else:
                allowed = ratio_rule("plan values", case, tr["values"][e, it], w32.values[e, it], v64, keep)
            n["values"] += int(keep.sum())
            if not bool(keep.all()):
                clean = False                           # a flipped termination may change the elite set
                break
            gap = 2 * allowed
            stable = stable_positions(v64, K, gap)
            assert torch.equal(tr["elite_idx"][e, it][stable], w64.elite_idx[e, it][stable]), f"top-k {case} env={e} it={it}"
            n["topk"] += int(stable.sum())
            if not bool(boundary_separated(v64, K, gap)):
                clean = False
                break
            # The refit weights exp(T (v - v_max)) pass a value error dv on to the mean and the std as at most
            # T dv sigma (Cauchy-Schwarz with sum(w) = 1; sigma = the elites' std): on top of the 1e-4 north-star tolerance
            tol = 1e-4 + cfg.temperature * allowed * w64.iter_std[e, it]
            tols.append(float((tol - 1e-4).max()))
            for q in ("iter_mean", "iter_std"):
                err = (tr[q][e, it].double() - getattr(w64, q)[e, it]).abs()
                assert bool((err <= tol).all()), f"{q} {case} env={e} it={it}: {float(err.max()):.2e}"
            n["refit"] += 1
            n["clamped"] += int(clamped[e, it])
            n["dominated"] += int(wmax[e, it] > 0.9)
        if clean:
            assert bool(((new_mean[e].double() - w64.mean[e]).abs() <= tol).all())
            logits = w64.score[e].log() - noise.expo[e].double().log()
            top2 = _top_k_plus_one(logits, 1)               # one elite: its pick is never ambiguous
            # the pick is a position in the sorted elite list: it names the same sample only where that order is stable
            if float(top2[0] - top2[1]) > 1e-3 and bool(stable[int(w64.pick[e])]):
                assert int(tr["pick"][e]) == int(w64.pick[e])
                # The action is the picked elite's first action clamp(mu + sigma eps), drawn from the second-to-last
                # refit, plus sigma eps_final from the last refit: each refit's value-induced error reaches the action
                # scaled by the noise it meets (1e-4 alone when the values are exact)
                eps_r = float(noise.r[e, -1].abs().max()) if noise.r[e, -1].numel() else 0.0
                eps_f = float(noise.final[e].abs().max()) if noise.final is not None else 0.0
                tol_a = 1e-4 + (tols[-2] if len(tols) > 1 else 0.0) * (1 + eps_r) + tols[-1] * eps_f
                err = float((action[e].double() - w64.action[e]).abs().max())
                assert err <= tol_a, f"action {case} env={e}: {err:.2e} > {tol_a:.2e}"
                n["actions"] += 1
    return n


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
