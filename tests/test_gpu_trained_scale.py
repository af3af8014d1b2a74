"""The H100 kernels at trained scale (synth.trained_scale) and at init scale, held to an error budget set by fp32
itself: every quantity is computed by the kernel (k), the fp32 oracle (o32) and the float64 oracle (o64), and

    max|k - o64| <= R * max|o32 - o64| + 2^-23 * max|o64|          (the ratio rule, R = RATIO)

A fixed absolute tolerance cannot serve both regimes: at init scale it is ~100x the real error, at trained scale no
fp32 computation meets it.  Two-hot values (reward / Q min / avg) are compared in the symlog domain, where they are
well conditioned.  The observed ratios are printed as a table at the end of the module (pytest -s)."""
import functools

import pytest
import torch

from helpers import boundary_separated, refit_stats, stable_positions, trained_model, trained_obs
from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
from oracle.wm_oracle import WMOracle, with_target_blend
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import head_layout, synth_state_dict

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
DEV = "cuda"
RATIO = 8.0
FLOOR = 2.0 ** -23
TERM_MARGIN = 2e-5          # as tests/test_gpu_parity.py: a termination decision this close to 0.5 is not defined
# Each product carries <= 2^-21 relative error (two 22-bit operands, the lo x lo term dropped) and each output sums 3K
# fp32-rounded terms plus the bias; the largest of ~10^5 outputs of that rounding walk reaches 21 x 2^-22 sum|W||x| on
# the H100 (the fp32 oracle's own error is of the same size: the ratio rule holds), so the bound is c = 32, not the 4
# a single product would suggest (DESIGN.md section 2)
LINEAR_C = 32.0
OBSERVED = {}               # (quantity, case) -> [worst ratio, elements compared, elements excluded]


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    if OBSERVED:
        print(f"\n{'quantity':18s} {'case':34s} {'ratio':>7s} {'compared':>9s} {'excluded':>9s}")
        for (q, case), (r, n, x) in sorted(OBSERVED.items(), key=lambda kv: (kv[0][1], kv[0][0])):
            print(f"{q:18s} {case:34s} {r:7.2f} {n:9d} {x:9d}")


def symlog(x):
    return torch.sign(x) * torch.log1p(x.abs())


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


# ------------------------------------------------------------------------------------------------- models
PRESET = {"tiny": ("tiny", {}), "tiny-mt": ("tiny-mt", {}), "tiny-episodic": ("tiny", {"episodic": True}),
          "c1": ("c1", {}), "c3": ("c3", {"num_envs": 1}), "c4": ("c4", {"num_envs": 1})}


@functools.lru_cache(maxsize=1)
def model(preset, level, **extra):
    """(cfg, state dict) at `level` ("init" = the synthetic initialisation with a blended target ensemble)."""
    wl, over = PRESET[preset]
    over = dict(over, **extra)
    if level != "init":
        return trained_model(wl, level, 7, **over)
    cfg = workload(wl, **over)
    sd = synth_state_dict(cfg, seed=7, perturb=True, emb_scale=60.0 if cfg.multitask else 1.0)
    if cfg.episodic:
        from oracle.plan_oracle import balance_termination
        balance_termination(cfg, sd)
    return cfg, with_target_blend(cfg, sd, 107)


def agent_for(cfg, sd, engine):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    return agent


# ------------------------------------------------------------------------------------------------- one fused layer
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


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("wl", ["tiny", "tiny-mt", "c1"])
def test_fused_layer_error_bound(engine, wl):
    """Each packed layer with trained-scale weights (outliers move its packing scale by several binades) on inputs at
    scales 1, 30, 1e3 and with a column near 6e4.  The linear output obeys the component-wise forward-error bound
    |k - y64| <= c * 2^-22 * sum_k |W_nk| |x_k| + 2^-23 |b_n| (c = LINEAR_C) and the ratio rule; LayerNorm + Mish /
    SimNorm outputs obey the ratio rule."""
    from tdmpc2_b200.planner import Planner
    F = torch.nn.functional
    cfg, sd = model(wl, "sharp")
    pl = Planner(cfg, 2, DEV, engine=engine)
    pl.pack(sd)
    g = torch.Generator().manual_seed(0)
    case = f"{wl}/sharp/{engine}"
    n_layers = 0
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
        bound = LINEAR_C * 2.0 ** -22 * (x.double().abs() @ W.double().abs().T) + FLOOR * b.double().abs()
        over = float(((y - y64).abs() / bound).max())
        old = OBSERVED.get(("linear/bound", case), [0.0, 0, 0])
        OBSERVED[("linear/bound", case)] = [max(old[0], over), old[1] + y.numel(), 0]
        assert over <= 1.0, f"{prefix} head={head}: linear error {over:.2f} x the forward-error bound"
        ratio_rule("linear", case, y, F.linear(x, W, b), y64)
        n_layers += 1
        if has_ln:
            gw, gb = sd[prefix + ".ln.weight"], sd[prefix + ".ln.bias"]
            if head is not None:
                gw, gb = gw[head], gb[head]

            def act(dt):
                h = F.layer_norm(F.linear(x.to(dt), W.to(dt), b.to(dt)), (W.shape[0],), gw.to(dt), gb.to(dt), 1e-5)
                return torch.softmax(h.view(rows, -1, 8), -1).view(rows, -1) if simnorm else F.mish(h)
            got = pl.debug_layer(li, 2 if simnorm else 1, x.to(DEV), W.shape[0])
            ratio_rule("simnorm" if simnorm else "ln+mish", case, got, act(torch.float32), act(torch.float64))
    assert n_layers >= 10


# ------------------------------------------------------------------------------------------------- row mode
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


ROW_CASES = [(p, lv) for p in ("tiny", "tiny-mt", "c1", "c3", "c4") for lv in ("mid", "sharp")] + \
            [("tiny-episodic", "sharp"), ("tiny-mt", "init"), ("c1", "init")]


@pytest.mark.parametrize("preset,level", ROW_CASES)
def test_row_mode_ratio_rule(preset, level):
    """Every WorldModel method and _td_target on one tile plus a partial one (c3: 1792-wide rows, the strided
    LayerNorm path; c4: K = 4096, 80 tasks and the target blob).  Excluded: entropy rows with min(1 - a^2) <= 1e-3 or
    |log_pi| < 1e-2 (the squash term and the entropy scale are ill-conditioned there)."""
    cfg, sd = model(preset, level)
    R = 150 if preset in ("c3", "c4") else 300
    x = row_inputs(cfg, R, 11)
    o32, o64 = WMOracle(cfg, sd), WMOracle(cfg, sd, torch.float64)
    z_in = o64.encode(x["obs"], x["task"]).float()          # the latent every other method reads, rounded to fp32
    want32 = run_methods(cfg, o32, x, z_in, False)
    want64 = run_methods(cfg, o64, x, z_in, False)
    a64 = want64["pi_action"]
    ok_rows = ((1 - a64 ** 2).min(-1).values > 1e-3) & (want64["pi_entropy"].reshape(-1).abs() > 1e-2)
    for engine in ENGINES:
        m = agent_for(cfg, sd, engine).model
        got = run_methods(cfg, m, x, z_in, True)
        case = f"{preset}/{level}/{engine}"
        for q in got:
            k, w32, w64 = got[q], want32[q], want64[q]
            keep, need = None, 0.5
            if q in ("q_min", "q_avg", "qt_min"):             # two-hot values: the symlog domain
                k, w32, w64 = symlog(k.double()), symlog(w32.double()), symlog(w64)
            if q in ("pi_entropy", "pi_scaled_entropy"):
                # a row with any saturated action dim is excluded: at "sharp" that is nearly every row (the counts are
                # printed); the mid and init levels keep the entropy under test
                keep, need = ok_rows.reshape(k.shape), 0.0 if level == "sharp" else 0.02
                if level == "sharp" and not bool(keep.any()):
                    OBSERVED.setdefault((q, case), [0.0, 0, int(keep.numel())])
                    continue
            ratio_rule(q, case, k, w32, w64, keep, need)
        del m
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------- planning
def to_gpu_noise(n):
    from tdmpc2_b200.planner import Noise
    return Noise.from_env_major(n.prior, n.r, n.pi, n.qidx, n.expo, n.final, device=DEV)


def plan_three_ways(cfg, sd, engine, E, seed):
    from tdmpc2_b200.planner import Planner
    obs = trained_obs(cfg, E, seed)
    task = [(2 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    noise = oracle_noise(cfg, 40 + seed, E)
    w32 = plan_oracle(cfg, sd, obs, task=task, noise=noise)
    w64 = plan_oracle(cfg, sd, obs, task=task, noise=noise, dtype=torch.float64)
    pl = Planner(cfg, E, DEV, engine=engine)
    pl.pack(sd)
    taskv = torch.tensor(task, dtype=torch.int32, device=DEV) if task is not None else None
    action, new_mean, tr = pl.plan(obs.to(DEV), taskv, torch.ones(E, dtype=torch.uint8, device=DEV),
                                   torch.zeros(E, cfg.horizon, cfg.action_dim, device=DEV), to_gpu_noise(noise), trace=True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in tr.items()}, action.cpu(), new_mean.cpu(), w32, w64, noise


def compare_plans(cfg, case, tr, action, new_mean, w32, w64, noise):
    """Values by the ratio rule per (env, iteration); top-k indices exact where float64's sorted values are separated
    by more than twice the allowed value error; refit mean / std and the action within 1e-4 while the elite set is
    unambiguous (helpers.compare_with_oracle's logic).  Returns counters."""
    E, K = tr["values"].shape[0], cfg.num_elites
    n = dict(values=0, topk=0, refit=0, clamped=0, dominated=0, actions=0)
    wmax, clamped = refit_stats(cfg, w64)
    for e in range(E):
        clean = True
        stable = None
        for it in range(cfg.iterations):
            v64 = w64.values[e, it]
            keep = w64.term_margin[e, it] > TERM_MARGIN if cfg.episodic else torch.ones_like(v64, dtype=torch.bool)
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
            for q in ("iter_mean", "iter_std"):
                err = (tr[q][e, it].double() - getattr(w64, q)[e, it]).abs()
                assert bool((err <= tol).all()), f"{q} {case} env={e} it={it}: {float(err.max()):.2e}"
            n["refit"] += 1
            n["clamped"] += int(clamped[e, it])
            n["dominated"] += int(wmax[e, it] > 0.9)
        if clean:
            assert bool(((new_mean[e].double() - w64.mean[e]).abs() <= tol).all())
            logits = w64.score[e].log() - noise.expo[e].double().log()
            top2 = torch.topk(logits, 2).values
            # the pick is a position in the sorted elite list: it names the same sample only where that order is stable
            if float(top2[0] - top2[1]) > 1e-3 and bool(stable[int(w64.pick[e])]):
                assert int(tr["pick"][e]) == int(w64.pick[e])
                assert float((action[e].double() - w64.action[e]).abs().max()) <= 1e-4, f"action {case} env={e}"
                n["actions"] += 1
    return n


PLAN_CASES = [(p, lv) for p in ("tiny", "tiny-mt", "c1", "tiny-episodic") for lv in ("mid", "sharp")] + \
             [("tiny-mt", "init"), ("c1", "init")]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("preset,level", PLAN_CASES)
def test_plan_ratio_rule(engine, preset, level):
    cfg, sd = model(preset, level)
    E = 4
    cfg = cfg.replace(num_envs=E)
    tr, action, new_mean, w32, w64, noise = plan_three_ways(cfg, sd, engine, E, 1)
    case = f"{preset}/{level}/{engine}"
    n = compare_plans(cfg, case, tr, action, new_mean, w32, w64, noise)
    print(case, n)
    assert n["values"] > 0 and n["topk"] > 0 and n["refit"] > 0, n
    if level != "init":                       # the min_std clamp ran and was compared
        assert n["clamped"] > 0, n
    if level == "sharp":                      # and so did refits dominated by one elite
        assert n["dominated"] > 0, n


# ------------------------------------------------------------------------------------------------- refit edges
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("preset,level,over", [
    ("tiny", "init", dict(num_samples=4096, num_elites=64)),             # the API's largest sample count
    ("tiny", "mid", dict(num_samples=4096, num_elites=64)),
    ("tiny", "init", dict(num_samples=4096, num_elites=1024, horizon=6)),  # K H A = 36864 > 32768: elite actions unstaged
    ("tiny", "mid", dict(num_samples=4096, num_elites=1024, horizon=6)),
    ("c1", "init", dict(num_samples=1024, num_elites=512)),              # K H A = 58368
    ("c1", "mid", dict(num_samples=1024, num_elites=512)),
])
def test_refit_edges(engine, preset, level, over):
    """The largest num_samples, and elite sets too large for the refit's staged copy of their actions (refit_env then
    reads them through sample_action)."""
    cfg, sd = model(preset, level, **over)
    E = 2
    cfg = cfg.replace(num_envs=E)
    tr, action, new_mean, w32, w64, noise = plan_three_ways(cfg, sd, engine, E, 2)
    n = compare_plans(cfg, f"{preset}/{level}/N{cfg.num_samples}K{cfg.num_elites}H{cfg.horizon}/{engine}",
                      tr, action, new_mean, w32, w64, noise)
    print(n)
    assert n["values"] >= E * cfg.num_samples, n
    if level == "init":
        assert n["refit"] > 0, n
