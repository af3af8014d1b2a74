"""The kernels at the edges of the shape envelope tdmpc2_planner_create accepts (tests/test_shape_envelope_cpu.py pins
the envelope itself): the widest heads, odd and narrow latents, LayerNorm widths around the staged 512-column path,
scratch pitches set by the encoder, the deepest encoder, the planner's prior-tile and elite limits, and the two
MODEL_SIZE presets no other GPU test builds.  These are the shapes where a loop bound, a lane mask, a padding rule or a
pitch that is right for every preset goes wrong.

Each case names the branch or bound it reaches and asserts the shape arithmetic that gets it there (`reaches`).  Every
comparison is the ratio rule of tests/test_gpu_trained_scale.py against the fp32 and float64 oracles; the observed
ratios are printed as a table at the end of the module (pytest -s)."""
import functools

import pytest
import torch

from helpers import (DEV, OBSERVED, compare_plans, fused_layer_ratio_rule, level_model, mixed_noise, plan_three_ways,
                     print_ratio_table, row_mode_ratio_rule, slice_noise, trained_obs)

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
MAX_ENC_LAYERS = 8       # TDMPC2_MAX_ENC_LAYERS
HEAD_REG_COLS = 8        # kHeadRegCols: a head row is 8 register columns per lane (kMaxHeadCols = 256)
LN_STAGED = 512          # rows_ln_act's staged cp.async path: N == 32 * kLnRegCols


def pad(x, m):
    return (x + m - 1) // m * m


def shape(cfg):
    """The shape arithmetic of tdmpc2_planner_create (api.cu) and the planning kernel for `cfg`."""
    L, M, A, B = cfg.latent_dim, cfg.mlp_dim, cfg.action_dim, cfg.num_bins
    T = cfg.task_dim if cfg.multitask else 0
    obs, P = cfg.obs_shape["state"][0], cfg.num_pi_trajs
    D = L + T + A
    KpadX = max(pad(D, 64), pad(obs + T, 64))
    ng = (A + 7) // 8
    Ppad = 1
    while Ppad < P:
        Ppad *= 2
    return dict(L=L, M=M, A=A, B=B, T=T, obs=obs, D=D, Apad=pad(A, 32), pi_cols=pad(A, 32) + A,
                pi_npad=pad(pad(A, 32) + A, 128), bin_npad=pad(B, 128), lane_strides=(A + 31) // 32,
                KpadX=KpadX, KpadX_D=pad(D, 64), KpadX_obs=pad(obs + T, 64),
                KpadH=max(pad(M, 64), pad(cfg.enc_dim, 64)), n_enc=max(cfg.num_enc_layers - 1, 1) + 1,
                groups=ng, vector_pass=(L + T) % 8 == 0 and L + T + 8 * ng <= KpadX, Ppad=Ppad,
                envs_per_prior_tile=128 // Ppad, N=cfg.num_samples, P=P, K=cfg.num_elites, E=cfg.num_envs,
                Q=cfg.num_q, action_dims=tuple(cfg.action_dims or ()))


# id -> (workload, overrides, what it reaches, the shape arithmetic that proves it, what runs)
#   rows:   row-mode levels (every WorldModel method and _td_target)
#   layers: Planner.debug_layer on each fused layer (forward-error bound and ratio rule)
#   plan:   plan() at E = 2 (one t0, one warm start) against the fp32 / float64 oracles
#   envs:   plan() at E = 130, sampled environments against the oracles
HEAD = dict(rows=("init", "mid", "sharp"), plan=True)
ROWS = dict(rows=("init", "mid"), plan=True)
WIDTH = dict(rows=("init", "mid"), layers=True, plan=True)
PLAN = dict(plan=True)
CASES = {
    # ---- head columns: num_bins
    "bins2": ("tiny", dict(num_bins=2), "two-hot over two bins (the first register column only)",
              lambda s: s["B"] == 2, ROWS),
    "bins255": ("tiny", dict(num_bins=255), "the last head register column, lanes 0-30 live",
                lambda s: 32 * (HEAD_REG_COLS - 1) < s["B"] < 32 * HEAD_REG_COLS, HEAD),
    "bins256": ("tiny", dict(num_bins=256), "every lane of every head register column; Npad = 256 reward / Q heads "
                "(two 128-column GEMM blocks)", lambda s: s["B"] == 32 * HEAD_REG_COLS and s["bin_npad"] == 256, HEAD),
    # ---- head columns: action_dim
    "a1": ("tiny", dict(action_dim=1), "Apad = 32 with one live action column; one partial action group",
           lambda s: s["Apad"] == 32 and s["A"] == 1 and s["groups"] == 1, ROWS),
    "a32": ("tiny", dict(action_dim=32), "Apad = A: the log-std columns start right after the mean's",
            lambda s: s["Apad"] == s["A"] == 32 and s["pi_cols"] == 64, ROWS),
    "a33": ("tiny", dict(action_dim=33), "Apad = 64 with one column in its second block; a 97-column pi head",
            lambda s: s["Apad"] == 64 and s["pi_cols"] == 97 and s["lane_strides"] == 2, ROWS),
    "a97": ("tiny", dict(action_dim=97), "a 225-column pi head (Npad 256); rows_pi's fourth lane stride; a partial "
            "action group", lambda s: s["pi_cols"] == 225 and s["pi_npad"] == 256 and s["lane_strides"] == 4
            and s["A"] % 8 != 0, HEAD),
    "a128": ("tiny", dict(action_dim=128), "a 256-column pi head; rows_pi with 4 full lane strides; 16 action groups "
             "in the vector pass", lambda s: s["pi_cols"] == 256 and s["lane_strides"] == 4 and s["groups"] == 16
             and s["vector_pass"], HEAD),
    # ---- the scalar action pass and the shared-latent fold
    "mt_t5": ("tiny-mt", dict(task_dim=5, action_dims=[5, 1, 4, 2]), "the scalar action pass (L + T odd: mean + "
              "std noise, clamp, mask); the shared-latent fold at L + T = 69; a task with one action dim",
              lambda s: not s["vector_pass"] and (s["L"] + s["T"]) % 8 != 0 and (s["L"] + s["T"]) // 64 == 1
              and 1 in s["action_dims"], ROWS),
    # ---- LayerNorm widths around the staged 512-column path
    "mlp511": ("tiny", dict(mlp_dim=511), "LayerNorm rows one short of the staged 512 path, 31 lanes in the last "
               "column", lambda s: s["M"] == LN_STAGED - 1, WIDTH),
    "mlp513": ("tiny", dict(mlp_dim=513), "LayerNorm rows one past the staged 512 path", lambda s: s["M"] == LN_STAGED + 1,
               WIDTH),
    "mlp200": ("tiny", dict(mlp_dim=200), "LayerNorm rows with a partial last lane column",
               lambda s: s["M"] % 32 != 0 and s["M"] < LN_STAGED, WIDTH),
    # ---- latents
    "lat8": ("tiny", dict(latent_dim=8), "one SimNorm group: a latent narrower than a warp",
             lambda s: s["L"] == 8, WIDTH),
    "lat40": ("tiny", dict(latent_dim=40), "a latent that is not a multiple of 32: lanes of a group past N",
              lambda s: s["L"] % 32 != 0 and s["L"] > 32, WIDTH),
    "lat520": ("tiny", dict(latent_dim=520), "SimNorm rows just beyond 512 columns",
               lambda s: LN_STAGED < s["L"] < LN_STAGED + 32, WIDTH),
    # ---- scratch pitches
    "obs1": ("tiny", dict(obs_dim=1), "an encoder input of one column (63 zero K columns in its chunk)",
             lambda s: s["obs"] == 1 and s["KpadX_obs"] == 64, ROWS),
    "obs700": ("tiny", dict(obs_dim=700), "KpadX set by the encoder input obs_dim + T",
               lambda s: s["KpadX"] == s["KpadX_obs"] > s["KpadX_D"], ROWS),
    "enc600": ("tiny", dict(enc_dim=600), "KpadH set by the encoder (enc_dim > mlp_dim)",
               lambda s: s["KpadH"] == pad(600, 64) > pad(s["M"], 64), ROWS),
    "enc8": ("tiny", dict(num_enc_layers=8), "the encoder-table limit (7 hidden + 1 output layer)",
             lambda s: s["n_enc"] == MAX_ENC_LAYERS, ROWS),
    # ---- the planner's limits
    "pi128": ("tiny", dict(num_pi_trajs=128, num_samples=256), "a prior tile holding one environment of 128 "
              "trajectories", lambda s: s["Ppad"] == 128 and s["envs_per_prior_tile"] == 1, PLAN),
    "pi_all": ("tiny", dict(num_pi_trajs=96, num_samples=96), "every sample a policy-prior sample (no noise rows)",
               lambda s: s["P"] == s["N"], PLAN),
    "elite1": ("tiny", dict(num_elites=1), "a refit from one elite (std clamped to min_std) and a top-1",
               lambda s: s["K"] == 1 < s["N"], PLAN),
    "samples1": ("tiny", dict(num_samples=1, num_elites=1, num_pi_trajs=0), "one sample: top-k and refit of a single "
                 "value", lambda s: s["N"] == s["K"] == 1, PLAN),
    "pi1_e130": ("tiny", dict(num_pi_trajs=1, num_envs=130), "a prior tile holding 128 environments, and the tile "
                 "boundary at environment 128", lambda s: s["envs_per_prior_tile"] == 128 < s["E"] and s["P"] == 1,
                 dict(envs=True)),
    # ---- the Q ensemble
    "q2": ("tiny", dict(num_q=2), "num_q = 2: the Q pair is forced", lambda s: s["Q"] == 2, ROWS),
    "q10": ("tiny", dict(num_q=10), "ten heads: Q-all output offsets past the presets' 8", lambda s: s["Q"] == 10, ROWS),
    # ---- the presets no other GPU test builds
    "preset1": ("c1", dict(model_size=1), "MODEL_SIZE 1 (mlp 384, latent 128, num_q 2)",
                lambda s: (s["M"], s["L"]) == (384, 128), ROWS),
    "preset19": ("c1", dict(model_size=19), "MODEL_SIZE 19 (1024 / 1024 / 768, 3 encoder layers)",
                 lambda s: (s["M"], s["L"], s["n_enc"]) == (1024, 768, 3), ROWS),
}
# plan() runs every case with few iterations (the float64 oracle runs on the host); the presets also with fewer samples
PLAN_OVER = dict(iterations=2)
PRESET_PLAN_OVER = dict(num_samples=256, num_elites=32)
SATURATED_POLICY = ("a97", "a128", "preset19")


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    OBSERVED.clear()
    yield
    print_ratio_table()


@functools.lru_cache(maxsize=1)
def model(case, level, **extra):
    wl, over, _, _, _ = CASES[case]
    return level_model(wl, level, **dict(over, **extra))


def reaches(case, cfg):
    """Asserts that `cfg` reaches the branch the case names."""
    wl, over, what, check, _ = CASES[case]
    s = shape(cfg)
    assert check(s), f"{case} does not reach {what!r}: {s}"


def cases_with(key):
    return [c for c, v in CASES.items() if v[4].get(key)]


ROW_CASES = [(c, lv) for c, v in CASES.items() for lv in v[4].get("rows", ())]


@pytest.mark.parametrize("case,level", ROW_CASES, ids=[f"{c}-{lv}" for c, lv in ROW_CASES])
def test_row_mode(case, level):
    """Every WorldModel method and _td_target on one full tile plus a partial one (200 rows), both engines."""
    cfg, sd = model(case, level)
    reaches(case, cfg)
    # at mid a row with any saturated action dim leaves the entropy comparison; with 97-128 action dims and in the
    # 768-wide preset that is nearly every row (< 2 %), so there the entropy is held to the rule at init only
    need = 0.0 if case in SATURATED_POLICY and level == "mid" else None
    row_mode_ratio_rule(cfg, sd, f"{case}/{level}", level, 200, ENGINES, entropy_need=need)
    for engine in ENGINES:
        assert OBSERVED[("td", f"{case}/{level}/{engine}")][1] == 200


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", cases_with("layers"))
def test_fused_layers(case, engine):
    """Each fused layer through Planner.debug_layer at trained scale; the layers whose width the case is about (mlp:
    the LayerNorm + Mish rows; latent: the SimNorm rows) must be among those compared."""
    cfg, sd = model(case, "sharp")
    reaches(case, cfg)
    done = fused_layer_ratio_rule(cfg, sd, engine, f"{case}/sharp/{engine}")
    kinds = {(n, kind) for _, _, n, kind in done}
    if case.startswith("mlp"):
        assert (cfg.mlp_dim, "ln+mish") in kinds, kinds
    else:
        assert (cfg.latent_dim, "simnorm") in kinds, kinds
    assert len(done) >= 6, done


def plan_cfg(case, level):
    cfg, sd = model(case, level)
    over = dict(PLAN_OVER, **(PRESET_PLAN_OVER if CASES[case][0] == "c1" else {}))
    return cfg.replace(num_envs=2, **over), sd


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", cases_with("plan"))
def test_plan(case, engine):
    """plan() at E = 2 (environment 0 from t0, environment 1 warm-started): values by the ratio rule, top-k exact where
    separated, refit and action within the tolerances of tests/test_gpu_trained_scale.py.  One sample per environment
    (samples1): E = 128, and the ratio rule's maximum runs over all environments' values of an iteration (helpers'
    trained_obs cycles four observation scales 10^3 apart, so the largest kind alone contributes 32 values)."""
    cfg, sd = plan_cfg(case, "mid")
    E = 128 if cfg.num_samples == 1 else 2
    cfg = cfg.replace(num_envs=E)
    reaches(case, cfg)
    # seed 2: every case has an iteration whose elite set float64 separates (checked on the oracles alone)
    tr, action, new_mean, w32, w64, noise = plan_three_ways(cfg, sd, engine, E, 2, warm=True)
    n = compare_plans(cfg, f"{case}/mid/{engine}", tr, action, new_mean, w32, w64, noise, pool_envs=E > 2)
    print(case, engine, n)
    # an environment's comparison stops at the first iteration whose elite set is ambiguous: its first always runs
    assert n["values"] >= E * cfg.num_samples and n["topk"] > 0 and n["refit"] > 0, n
    if cfg.multitask:          # masked action dims are exactly zero
        for e in range(E):
            adim = cfg.action_dims[(2 * e + 1) % len(cfg.tasks)]
            assert torch.all(action[e, adim:] == 0) and torch.all(new_mean[e, :, adim:] == 0)


@pytest.mark.parametrize("engine", ENGINES)
def test_plan_prior_tile_boundary(engine):
    """num_pi_trajs = 1 at E = 130: one prior tile holds 128 environments, so environments 127 and 128 sit on either
    side of a prior-tile boundary.  Every environment of a two-iteration plan is bit-identical to a two-environment
    run of the same inputs and noise (pairs across and beside the boundary); the policy prior feeds the first
    iteration, which is held to the oracles on sampled environments (0, 127, 128, 129): values, top-k, refit and the
    action of a one-iteration plan.  (A later iteration samples from each implementation's own refit, so its values
    carry that refit's allowed difference times the value's slope in the actions as well as the arithmetic error.)"""
    from oracle.plan_oracle import plan_oracle
    from tdmpc2_b200.planner import Planner
    cfg, sd = model("pi1_e130", "mid")
    cfg = cfg.replace(**PLAN_OVER)
    reaches("pi1_e130", cfg)
    E = cfg.num_envs
    envs = [0, 127, 128, 129]
    obs = trained_obs(cfg, E, 5)
    t0 = torch.tensor([i % 2 == 0 for i in range(E)], dtype=torch.uint8)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=torch.Generator().manual_seed(5))
    nz, on = mixed_noise(cfg, E, envs, 500)
    pl = Planner(cfg, E, DEV, engine=engine)
    pl.pack(sd)
    action, new_mean, tr = pl.plan(obs.to(DEV), None, t0.to(DEV), prev.to(DEV), nz, trace=True)
    torch.cuda.synchronize()
    for pair in ([0, 1], [126, 127], [127, 128], [128, 129]):
        p2 = Planner(cfg.replace(num_envs=2), 2, DEV, engine=engine)
        p2.pack(sd)
        a2, m2, tr2 = p2.plan(obs[pair].to(DEV), None, t0[pair].to(DEV), prev[pair].to(DEV), slice_noise(nz, pair),
                              trace=True)
        torch.cuda.synchronize()
        for name, x, y in (("action", action[pair], a2), ("mean", new_mean[pair], m2)) + tuple(
                (k, tr[k][pair], tr2[k]) for k in ("values", "elite_idx", "iter_mean", "iter_std", "pick", "z")):
            assert torch.equal(x.cpu(), y.cpu()), f"envs {pair}: {name} differs from the two-environment run"
    del pl
    cfg = cfg.replace(iterations=1)
    nz, on = mixed_noise(cfg, E, envs, 500)
    pl = Planner(cfg, E, DEV, engine=engine)
    pl.pack(sd)
    action, new_mean, tr = pl.plan(obs.to(DEV), None, t0.to(DEV), prev.to(DEV), nz, trace=True)
    torch.cuda.synchronize()
    sel = torch.tensor(envs)
    tr = {k: v[sel].cpu() for k, v in tr.items()}
    args = dict(t0=[bool(t0[e]) for e in envs], prev_mean=prev[sel], noise=on)
    w32 = plan_oracle(cfg, sd, obs[sel], **args)
    w64 = plan_oracle(cfg, sd, obs[sel], dtype=torch.float64, **args)
    n = compare_plans(cfg, f"pi1_e130/mid/{engine}", tr, action[sel].cpu(), new_mean[sel].cpu(), w32, w64, on)
    print("pi1_e130", engine, n)
    assert n["values"] >= len(envs) * cfg.num_samples and n["topk"] > 0 and n["refit"] > 0, n
