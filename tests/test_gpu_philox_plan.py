"""The philox planning mode (cfg.rng = 'philox', tdmpc2_plan_iter_rng, tdmpc2_plan_draws, tdmpc2_act) against float64:

  (a) the generator: tdmpc2_debug_rng's normals against oracle/philox_oracle.py's float64 law, on iteration and draw
      streams, around the 2^32 group and plan-counter boundaries and at the pinned extreme groups;
  (b) tdmpc2_plan_draws element by element against the host law (qidx and shift exact, normals within the generator's
      bound, exponentials within 2 ulp), with sentinels where nothing may be written;
  (c) philox plans, traced, against the fp32 and float64 plan oracles fed the kernels' own noise (dumped, and checked
      against the host law first) by helpers.compare_plans, on shapes that reach each branch of the in-kernel noise;
  (d) tdmpc2_act against the float64 oracle over consecutive calls, every small draw regenerated on the host;
  (e) the Gumbel pick when an exponential draw is exactly 0.

The tensor-core engine only: the SIMT engine refuses in-kernel noise (tests/test_gpu_c_act.py).  Run on an H100:
pytest -m gpu tests/test_gpu_philox_plan.py -s (prints the ratio table and the generator's largest error)."""
import functools

import numpy as np
import pytest
import torch

from helpers import (DEV, FLOOR, RATIO, SENTINEL, boundary_separated, compare_plans, cuda_stream, draw_planner, level_model,
                     plan_draws, planner_for, stable_positions, trained_obs, _top_k_plus_one)
from helpers import ratio_table  # noqa: F401 (autouse: this module's ratio table)
from oracle import philox_oracle as ph
from test_gpu_shape_envelope import CASES as ENVELOPE, shape
from test_philox_oracle_cpu import PINNED, ZERO_EXPO
from tdmpc2_b200 import _cabi
from tdmpc2_b200.config import workload
from tdmpc2_b200.planner import alloc_noise

pytestmark = pytest.mark.gpu
SEED_HI = 0x1D872B41C9A5F3E7            # a seed >= 2^32 (below 2^63: Planner keeps 63 bits)
NORMAL_BOUND = 2.0 ** -21               # |device - float64| <= 2^-21 rho (rng_normal4's budget, DESIGN.md section 2)
GEN_ERR = {}                            # what -> largest |device - float64| in units of 2^-24 rho


@pytest.fixture(scope="module", autouse=True)
def generator_table():
    """The generator's largest errors, printed after the ratio table (pytest sets up a module's autouse fixtures in
    order of name, so this one before ratio_table, and tears them down in reverse)."""
    GEN_ERR.clear()
    yield
    if GEN_ERR:
        print(f"\n{'normals':44s} {'max |dev - f64| / (2^-24 rho)':>30s}")
        for k, v in sorted(GEN_ERR.items()):
            print(f"{k:44s} {v:30.3f}")


def _state(seed, plan):
    """The device state {seed, plan counter} the kernels read (both below 2^63 here)."""
    return torch.tensor([seed, plan], dtype=torch.int64, device=DEV)


def dump(state, stream, group0, ngroups):
    """tdmpc2_debug_rng: the normals of groups group0 .. group0 + ngroups - 1 -> float32 numpy [ngroups, 4]."""
    lib = _cabi.load()
    out = torch.empty(4 * ngroups, device=DEV, dtype=torch.float32)
    _cabi.check(lib.tdmpc2_debug_rng(state.data_ptr(), stream, group0, ngroups, out.data_ptr(), cuda_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(ngroups, 4)


def check_normals(what, dev, want, rho):
    """|dev - float64| <= 2^-21 rho element-wise (exact where rho = 0); records the largest error in 2^-24 rho."""
    dev, want, rho = (np.asarray(x, dtype=np.float64).reshape(-1) for x in (dev, want, rho))
    err = np.abs(dev - want)
    bad = err > NORMAL_BOUND * rho
    assert not bad.any(), f"{what}: {int(bad.sum())} normals off the float64 law, e.g. {dev[bad][:4]} vs {want[bad][:4]}"
    live = rho > 0
    if live.any():
        GEN_ERR[what] = max(GEN_ERR.get(what, 0.0), float((err[live] / (2.0 ** -24 * rho[live])).max()))


# ------------------------------------------------------------------------------------------------ (a) the generator
STREAMS = [0, 1, 2 * 6 - 1] + [0x80000000 + k for k in range(5)]
WINDOWS = [(0, 1 << 16), ((1 << 32) - 1024, 2048)]           # the second crosses 2^32: the group's high word is nonzero


@pytest.mark.parametrize("plan", [(1 << 32) - 1, 1 << 32, (1 << 32) + 1])
def test_generator_is_the_float64_law(plan):
    st = _state(SEED_HI, plan)
    for stream in STREAMS:
        for g0, n in WINDOWS:
            want, rho = ph.normal4(SEED_HI, plan, stream, np.arange(g0, g0 + n, dtype=np.uint64))
            check_normals(f"plan {plan:#x}", dump(st, stream, g0, n), want, rho)


@pytest.mark.parametrize("name", [k for k in PINNED if not k.startswith("expo")])
def test_generator_extremes(name):
    seed, plan, stream, group, comp = PINNED[name]
    got = dump(_state(seed, plan), stream, group, 1)[0]
    want, rho = ph.normal4(seed, plan, stream, group)
    check_normals(f"pinned {name}", got, want, rho)
    pair = slice(comp & ~1, (comp & ~1) + 2)
    if name == "u1=1":                                   # rho = 0: both normals of the pair are +-0
        assert np.array_equal(got[pair], [0.0, 0.0])
    elif name == "u1=2^-24":                             # the largest radius: the pair lies on the circle rho_max
        assert abs(float(np.hypot(*got[pair].astype(np.float64))) - ph.RHO_MAX) <= 2.0 ** -20 * ph.RHO_MAX
    else:                                                # sincospif is exact at multiples of pi / 2
        q = {"u2=0": 0, "u2=1/4": 1, "u2=1/2": 2, "u2=3/4": 3}[name]
        zero = comp if q % 2 == 0 else comp - 1         # sin at 0, pi; cos at pi / 2, 3 pi / 2
        assert got[zero] == 0.0, got


# ------------------------------------------------------------------------------------------------ (b) tdmpc2_plan_draws
def check_expo(what, dev, want):
    """Exponentials within 2 ulp (fp32, at the float64 value) of float64; an exact 0 stays exact."""
    dev, want = np.asarray(dev, dtype=np.float64).reshape(-1), np.asarray(want, dtype=np.float64).reshape(-1)
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    bad = np.abs(dev - want) > 2 * ulp
    assert not bad.any(), f"{what}: {dev[bad][:4]} vs {want[bad][:4]}"


# (num_q, eval_mode, P, pixel, (seed, plan counter)): draw counts E H P A = 3 2 7 5, E K = 3 9 are not multiples of 4
DRAW_CASES = [(2, False, 7, True, (5, 1)), (3, True, 7, False, (SEED_HI, 3)), (4, False, 0, True, (SEED_HI, 1 << 32)),
              (5, True, 0, False, (77, (1 << 32) + 1)), (8, False, 7, False, (2 ** 62 + 9, 17)), (10, False, 7, True, (SEED_HI, 2))]


@pytest.mark.parametrize("num_q,eval_mode,P,pixel,state", DRAW_CASES,
                         ids=[f"q{c[0]}-{'eval' if c[1] else 'explore'}-P{c[2]}-{'pixel' if c[3] else 'state'}" for c in DRAW_CASES])
def test_plan_draws_are_the_host_law(num_q, eval_mode, P, pixel, state):
    E, H, A, I, K, N = 3, 2, 5, 3, 9, 16
    lib, p, d = draw_planner(E, N, P, K, H, A, I, num_q)
    seed, plan = state
    try:
        prior, qidx, expo, final, shift = plan_draws(p, _state(seed, plan), d, eval_mode, pixel, sentinel=True)
    finally:
        lib.tdmpc2_planner_destroy(p)
    want = ph.plan_draws(seed, plan, E, H, P, A, I, K, num_q, eval_mode, pixel)
    assert np.array_equal(qidx.numpy(), want["qidx"]), (qidx, want["qidx"])
    check_expo("expo", expo.numpy(), want["expo"])
    if P > 0:
        check_normals("draws: prior", prior.numpy(), want["prior"], want["prior_rho"])
    else:
        assert bool((prior == SENTINEL).all()), "prior written with num_pi_trajs = 0"
    if eval_mode:
        assert bool((final == SENTINEL).all()), "final written in eval mode"
    else:
        check_normals("draws: final", final.numpy(), want["final"], want["final_rho"])
    if pixel:
        assert np.array_equal(shift.numpy(), want["shift"])


def test_expo_extremes():
    """The pinned exponential words: u = 0 gives exactly 0, u = 1 - 2^-24 gives 24 ln 2 (one draw of 6 x 2^20 elements)."""
    (seed, plan, _, g0, c0), (_, _, _, g1, c1) = PINNED["expo=0"], PINNED["expo=24ln2"]
    E, K = 65536, 96
    assert 4 * max(g0, g1) + 3 < E * K
    lib, p, d = draw_planner(E, K, 0, K, 1, 1, 1, 2)
    try:
        expo = plan_draws(p, _state(seed, plan), d, eval_mode=True)[2].numpy().reshape(-1)
    finally:
        lib.tdmpc2_planner_destroy(p)
    assert expo[4 * g0 + c0] == 0.0
    check_expo("expo extremes", expo[[4 * g0 + c0, 4 * g1 + c1]], [0.0, 24 * np.log(2.0)])
    check_expo("expo 6 x 2^20", expo, ph.expo(seed, plan, E * K))


# ------------------------------------------------------------------------------------------------ (c) philox plans
def _c1_reaches(s, cfg):
    return (s["A"] == 38 and (s["A"] + 3) // 4 == 10 and s["vector_pass"] and 8 * s["groups"] > s["A"]
            and s["N"] // 128 == 4 and cfg.iterations == 6)


# id -> (workload, overrides, eval_mode, what it reaches, check(shape, cfg), envs compared (None: all), rng state)
PLAN_CASES = {
    "c1": ("c1", dict(num_envs=2), False, "A4 = 10, the vector pass's last 8-column item ends in padding; 4 sample tiles "
           "per env; six iteration streams", _c1_reaches, None, None),
    "c1-eval": ("c1", dict(num_envs=2), True, "the same in eval mode: no final draw", _c1_reaches, None, None),
    "mt_t5": ("tiny-mt", dict(ENVELOPE["mt_t5"][1], num_envs=2, iterations=2), False, ENVELOPE["mt_t5"][2],
              lambda s, cfg: ENVELOPE["mt_t5"][3](s), None, None),
    "a1": ("tiny", dict(ENVELOPE["a1"][1], num_envs=2, iterations=2), False, "A4 = 1: the vector pass's second group "
           "belongs to the next sample", lambda s, cfg: ENVELOPE["a1"][3](s) and (s["A"] + 3) // 4 == 1 and s["vector_pass"],
           None, None),
    "a97": ("tiny", dict(ENVELOPE["a97"][1], num_envs=2, iterations=2), False, "a partial last group, 13 vector items",
            lambda s, cfg: ENVELOPE["a97"][3](s) and s["A"] % 4 != 0 and s["groups"] == 13 and s["vector_pass"], None, None),
    "nopi": ("tiny", dict(num_pi_trajs=0), False, "every sample from noise; prior not drawn",
             lambda s, cfg: s["P"] == 0, None, None),
    "pi_all": ("tiny", dict(ENVELOPE["pi_all"][1], num_envs=2, iterations=2), False, "P = N: stream 2 it is never read",
               lambda s, cfg: ENVELOPE["pi_all"][3](s), None, None),
    "episodic": ("tiny", dict(episodic=True), False, "the termination head",
                 lambda s, cfg: bool(cfg.episodic), None, None),
    "wide2": ("tiny-wide2", {}, False, "2 tiles per env on a 576-wide latent",
              lambda s, cfg: s["N"] // 128 == 2 and s["L"] == 576, None, None),
    "rgb": ("tiny-rgb", dict(num_envs=2), False, "ShiftAug's shift from the draws; the pixel encode",
            lambda s, cfg: cfg.get("obs", "state") == "rgb", None, None),
    "e130": ("tiny", dict(ENVELOPE["pi1_e130"][1], iterations=1), False, "environment indices >= 128 in the group arithmetic",
             lambda s, cfg: ENVELOPE["pi1_e130"][3](s), [0, 127, 128, 129], None),
    "counter-hi": ("tiny", {}, False, "the plan at counter 2^32: low word 0, high word folded into the key",
                   lambda s, cfg: True, None, (SEED_HI, (1 << 32) - 1)),
}


@functools.lru_cache(maxsize=1)
def plan_model(case):
    wl, over = PLAN_CASES[case][:2]
    return level_model(wl, "mid", **over)


def rgb_shape(cfg):
    return dict(N=cfg.num_samples, P=cfg.num_pi_trajs, L=cfg.latent_dim, A=cfg.action_dim)


def plan_inputs(cfg, E, seed):
    g = torch.Generator().manual_seed(seed)
    if cfg.get("obs", "state") == "rgb":
        obs = torch.randint(0, 256, (E, *cfg.obs_shape["rgb"]), generator=g).float()
    else:
        obs = trained_obs(cfg, E, seed)
    task = [(2 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    t0 = torch.ones(E, dtype=torch.uint8)
    t0[1::2] = 0
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    return obs, task, t0, prev


def iteration_noise(state, seed, plan, it, cfg, E):
    """Dumps of streams 2 it and 2 it + 1 over the groups the layout names, checked against the host law ->
    (r [E, H, N - P, A], pi [E, N, A]) as float32."""
    H, N, P, A = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim
    r = dump(state, 2 * it, 0, ph.r_groups(E, H, N, A))
    pi = dump(state, 2 * it + 1, 0, ph.pi_groups(E, N, A))
    want_r, rho_r = ph.noise_r(seed, plan, it, E, H, N, P, A)
    want_pi, rho_pi = ph.noise_pi(seed, plan, it, E, N, A)
    r, pi = ph.layout_r(r, E, H, N, P, A), ph.layout_pi(pi, E, N, A)
    check_normals("iteration noise", r, want_r, rho_r)
    check_normals("iteration noise", pi, want_pi, rho_pi)
    return r, pi


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_philox_plan_against_oracles(case):
    from oracle.plan_oracle import plan_oracle
    wl, over, eval_mode, what, check, envs, state0 = PLAN_CASES[case]
    cfg, sd = plan_model(case)
    seed = SEED_HI if state0 is None else state0[0]
    cfg = cfg.replace(rng="philox", rng_seed=seed)
    E, H, N, P, A, I, K = cfg.num_envs, cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.iterations, cfg.num_elites
    pixel = cfg.get("obs", "state") == "rgb"
    s = rgb_shape(cfg) if pixel else shape(cfg)
    assert check(s, cfg), f"{case} does not reach {what!r}: {s}"
    pl = planner_for(cfg, E, None, sd)
    assert pl.philox and int(pl.rng_state[0]) == seed
    if state0 is not None:
        pl.rng_state[1] = state0[1]
    plan = int(pl.rng_state[1]) + 1                                    # plan() advances the counter first
    state = _state(seed, plan)
    nz = alloc_noise(cfg, E, DEV, eval_mode)
    prior, qidx, expo, final, shift = plan_draws(pl.h, state, pl._dims, eval_mode, pixel)
    nz.qidx.copy_(qidx); nz.expo.copy_(expo)
    if P > 0:
        nz.prior.copy_(prior)
    if not eval_mode:
        nz.final.copy_(final)
    if pixel:
        nz.shift.copy_(shift)
    obs, task, t0, prev = plan_inputs(cfg, E, 2)
    taskv = None if task is None else torch.tensor(task, dtype=torch.int32, device=DEV)
    action, new_mean, tr = pl.plan(obs.to(DEV), taskv, t0.to(DEV), prev.to(DEV), nz, trace=True)
    torch.cuda.synchronize()
    assert int(pl.rng_state[1]) == plan
    tr = {k: v.cpu() for k, v in tr.items()}
    action, new_mean = action.cpu(), new_mean.cpu()
    rs, pis = zip(*(iteration_noise(state, seed, plan, it, cfg, E) for it in range(I)))
    if state0 is not None:                                             # counter 2^32 is not counter 0
        assert not np.array_equal(dump(_state(seed, 0), 0, 0, 64), dump(state, 0, 0, 64))
    sel = list(range(E)) if envs is None else envs
    noise = ph.plan_noise(np.stack(rs)[:, sel], np.stack(pis)[:, sel], None if P == 0 else prior[sel], qidx[:, sel],
                          expo[sel], None if eval_mode else final[sel], None if shift is None else shift[sel], H=H, A=A)
    args = dict(task=None if task is None else [task[e] for e in sel], t0=[bool(t0[e]) for e in sel], prev_mean=prev[sel],
                noise=noise, eval_mode=eval_mode)
    w32 = plan_oracle(cfg, sd, obs[sel], **args)
    w64 = plan_oracle(cfg, sd, obs[sel], dtype=torch.float64, **args)
    tr = {k: v[sel] for k, v in tr.items()}
    n = compare_plans(cfg, f"philox/{case}", tr, action[sel], new_mean[sel], w32, w64, noise)
    print(case, n)
    assert n["values"] >= len(sel) * N and n["topk"] > 0 and n["refit"] > 0, n
    if cfg.multitask:                                                  # masked action dims are exactly zero
        for j, e in enumerate(sel):
            adim = cfg.action_dims[task[e]]
            assert torch.all(action[e, adim:] == 0) and torch.all(new_mean[e, :, adim:] == 0)


# ------------------------------------------------------------------------------------------------ (d) tdmpc2_act
def final_step_ok(cfg, w32, w64, noise, e):
    """compare_plans' final-step tolerances decided on the oracles alone: (prev_mean tolerance, action tolerance or None)
    when float64's elite set is separated in every iteration by twice the value error the ratio rule allows, else None."""
    K, tols, stable = cfg.num_elites, [], None
    for it in range(cfg.iterations):
        v64 = w64.values[e, it]
        allowed = RATIO * float((w32.values[e, it].double() - v64).abs().max()) + FLOOR * float(v64.abs().max())
        if not bool(boundary_separated(v64, K, 2 * allowed)):
            return None
        stable = stable_positions(v64, K, 2 * allowed)
        tol = 1e-4 + cfg.temperature * allowed * w64.iter_std[e, it]
        tols.append((tol, float((tol - 1e-4).max())))
    mean_tol = tols[-1][0]
    logits = w64.score[e].log() - noise.expo[e].double().log()
    top2 = _top_k_plus_one(logits, 1)
    if not (float(top2[0] - top2[1]) > 1e-3 and bool(stable[int(w64.pick[e])])):
        return mean_tol, None
    eps_r = float(noise.r[e, -1].abs().max()) if noise.r[e, -1].numel() else 0.0
    eps_f = float(noise.final[e].abs().max())
    return mean_tol, 1e-4 + (tols[-2][1] if len(tols) > 1 else 0.0) * (1 + eps_r) + tols[-1][1] * eps_f


@pytest.mark.parametrize("case,E,eval_mode,calls", [("c1", 4, False, 3), ("tiny-rgb", 2, True, 2)])
def test_act_against_float64(case, E, eval_mode, calls, tmp_path):
    """tdmpc2_act over consecutive calls (t0 on the first only): every small draw regenerated on the host at the counter
    the call used, the iteration noise dumped, the oracles fed the kernel's prev_mean of the previous call."""
    from oracle.plan_oracle import plan_oracle
    from test_gpu_c_act import CModel, _inputs, _model
    seed = SEED_HI
    cfg, sd, path = _model(case, E, tmp_path)
    m = CModel(path, seed=seed)
    H, N, P, A, I, K = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.iterations, cfg.num_elites
    obs, task = _inputs(cfg, E, calls)
    compared = dict(mean=0, action=0)
    for k in range(calls):
        t0 = torch.full((E,), int(k == 0), dtype=torch.uint8, device=DEV)
        prev_in = m.prev_mean.clone().cpu()
        action, prev_out = m.act(obs[k], t0, task, eval_mode)
        torch.cuda.synchronize()
        plan = k + 1
        assert int(m.rng_state[1]) == plan
        d = ph.plan_draws(seed, plan, E, H, P, A, I, K, cfg.num_q, eval_mode, m.pixel)
        state = _state(seed, plan)
        rs, pis = zip(*(iteration_noise(state, seed, plan, it, cfg, E) for it in range(I)))
        noise = ph.plan_noise(np.stack(rs), np.stack(pis), d["prior"], d["qidx"], d["expo"], d["final"], d["shift"], H=H, A=A)
        args = dict(task=None if task is None else task.tolist(), t0=[k == 0] * E, prev_mean=prev_in, noise=noise,
                    eval_mode=eval_mode)
        w32 = plan_oracle(cfg, sd, obs[k].cpu(), **args)
        w64 = plan_oracle(cfg, sd, obs[k].cpu(), dtype=torch.float64, **args)
        for e in range(E):
            ok = final_step_ok(cfg, w32, w64, noise, e)
            if ok is None:
                continue
            mean_tol, tol_a = ok
            err = (prev_out[e].cpu().double() - w64.mean[e]).abs()
            assert bool((err <= mean_tol).all()), f"prev_mean call {k} env {e}: {float(err.max()):.2e}"
            compared["mean"] += 1
            if tol_a is not None:
                err = float((action[e].cpu().double() - w64.action[e]).abs().max())
                assert err <= tol_a, f"action call {k} env {e}: {err:.2e} > {tol_a:.2e}"
                compared["action"] += 1
    print(case, compared)
    assert compared["mean"] > 0 and compared["action"] > 0, compared


# ------------------------------------------------------------------------------------------------ (e) expo == 0
def test_pick_with_an_exact_zero_exponential():
    """An exponential draw of exactly 0 (u = 0: -log(1 - 0)) gives its elite a Gumbel logit of +inf: the pick is the
    argmax of log score - log expo with the first maximum winning ties, so that elite is picked -- the limit of the
    Gumbel-max rule.  (The oracle's softmax is NaN there and torch.argmax would return position 0.)"""
    seed, plan, elem = ZERO_EXPO
    cfg = workload("tiny", rng="philox", rng_seed=seed)
    from tdmpc2_b200.synth import synth_state_dict
    sd = synth_state_dict(cfg, seed=7, perturb=True)
    E, K = cfg.num_envs, cfg.num_elites
    assert (E, K) == (2, 16)
    pl = planner_for(cfg, E, None, sd)
    assert int(pl.rng_state[1]) == plan - 1
    nz = alloc_noise(cfg, E, DEV)
    prior, qidx, expo, final, _ = plan_draws(pl.h, _state(seed, plan), pl._dims)
    assert float(expo.reshape(-1)[elem]) == 0.0
    nz.prior.copy_(prior); nz.qidx.copy_(qidx); nz.expo.copy_(expo); nz.final.copy_(final)
    obs, _, t0, prev = plan_inputs(cfg, E, 4)
    action, _, tr = pl.plan(obs.to(DEV), None, t0.to(DEV), prev.to(DEV), nz, trace=True)
    torch.cuda.synchronize()
    score, pick = tr["score"].cpu().double(), tr["pick"].cpu()
    for e in range(E):
        logits = score[e].log() - expo[e].double().log()
        want = int(torch.nonzero(logits == logits.max())[0])          # the first maximum
        assert int(pick[e]) == want, (e, logits)
    e0, k0 = divmod(elem, K)
    assert float(score[e0, k0]) > 0 and int(pick[e0]) == k0
