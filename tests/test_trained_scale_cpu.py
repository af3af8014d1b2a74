"""Trained-scale synthetic weights (synth.trained_scale) and the float64 oracle, without a GPU.

The regime statistics are asserted here so that the GPU parity tests at these levels keep testing what they claim to:
peaked two-hot heads, a refit dominated by one elite, std clamped to min_std, saturated tanh and log-stds at their
bounds."""
import pytest
import torch

from helpers import refit_stats, trained_model, trained_obs
from oracle.plan_oracle import OracleModel, balance_termination, draw_noise, plan_oracle
from oracle.wm_oracle import WMOracle
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict, trained_scale

PRESETS = ["tiny", "tiny-mt", "c1"]
TASKS = [1, 3, 0, 2]


def plan_stats(wl, level, dtype=torch.float32):
    cfg, sd = trained_model(wl, level, 7)
    E = 4
    tr = plan_oracle(cfg, sd, trained_obs(cfg, E, 1), task=TASKS[:E] if cfg.multitask else None, t0=[True] * E,
                     noise=draw_noise(cfg, 40, E), dtype=dtype)
    return cfg, sd, tr


def policy_stats(cfg, sd, rows=256):
    """Fractions of live action dims with |a| > 0.999 and with log_std within 1e-3 of a bound."""
    o = WMOracle(cfg, sd)
    g = torch.Generator().manual_seed(5)
    task = torch.randint(0, len(cfg.tasks), (rows,), generator=g) if cfg.multitask else None
    z = o.encode(trained_obs(cfg, rows, 2), task)
    act, info = o.pi(z, task, torch.randn(rows, cfg.action_dim, generator=g))
    live = o.sd["_action_masks"][task] > 0 if cfg.multitask else torch.ones_like(act, dtype=torch.bool)
    ls = info["log_std"]
    at_bound = ((ls - cfg.log_std_min).abs() < 1e-3) | ((ls - cfg.log_std_max).abs() < 1e-3)
    return float((act.abs() > 0.999)[live].float().mean()), float(at_bound[live].float().mean())


@pytest.mark.parametrize("wl", PRESETS)
def test_mid_level_regime(wl):
    cfg, sd, tr = plan_stats(wl, "mid")
    wmax, clamped = refit_stats(cfg, tr)
    print(wl, f"median largest elite weight {float(wmax.median()):.3f}, min_std refits {float(clamped.float().mean()):.2f}")
    assert 0.1 <= float(wmax.median()) <= 0.6
    assert bool(clamped.any())


@pytest.mark.parametrize("wl", PRESETS)
def test_sharp_level_regime(wl):
    cfg, sd, tr = plan_stats(wl, "sharp")
    wmax, clamped = refit_stats(cfg, tr)
    sat, at_bound = policy_stats(cfg, sd)
    vmax = float(tr.values.abs().max())
    print(wl, f"median largest elite weight {float(wmax.median()):.3f}, min_std refits {float(clamped.float().mean()):.2f}, "
          f"max |value| {vmax:.0f}, |a| > 0.999: {sat:.2f}, log_std at a bound: {at_bound:.2f}")
    assert float(wmax.median()) >= 0.9                      # one elite dominates
    assert float(clamped.float().mean()) > 0.5
    assert 1e3 <= vmax <= 1e5
    assert sat >= 0.2 and at_bound >= 0.1


def test_termination_logits_reach_20_with_both_signs():
    cfg, sd = trained_model("tiny", "sharp", 7, episodic=True)
    o = WMOracle(cfg, sd)
    z = o.encode(trained_obs(cfg, 512, 3), None)
    z = o.next(z, torch.rand(512, cfg.action_dim, generator=torch.Generator().manual_seed(0)) * 2 - 1, None)
    lg = o.termination(z, unnormalized=True)
    assert float(lg.abs().max()) >= 20
    assert 0.05 < float((lg > 0).float().mean()) < 0.95


def test_trained_scale_is_deterministic_and_plants_outliers():
    cfg = workload("tiny-mt")
    base = synth_state_dict(cfg, seed=3, perturb=True)
    a, b = trained_scale(cfg, base, "sharp", 9), trained_scale(cfg, base, "sharp", 9)
    assert all(torch.equal(a[k], b[k]) for k in a if torch.is_tensor(a[k]))
    assert not torch.equal(a["_dynamics.0.weight"], trained_scale(cfg, base, "sharp", 10)["_dynamics.0.weight"])
    assert a["_detach_Qs_params.0.weight"] is a["_Qs.params.0.weight"]
    for k, w in a.items():
        if not k.endswith(".weight") or ".ln." in k or not k.startswith(("_encoder", "_dynamics", "_reward", "_pi", "_Qs")):
            continue
        for h in w.reshape(-1, *w.shape[-2:]):
            # the packer scales max|W| to [128, 256): the outliers move that power of two by >= 3 binades
            ratio = float(h.abs().max() / h.std())
            assert ratio > 15, (k, ratio)
        _, e_before = torch.frexp(base[k].abs().max())
        _, e_after = torch.frexp(w.abs().max())
        if not k.endswith(".2.weight"):                     # output layers are rescaled as a whole
            assert int(e_after) - int(e_before) >= 3, k


@pytest.mark.parametrize("wl", PRESETS)
def test_fp64_oracle_agrees_with_fp32_at_init_scale(wl):
    """The float64 port computes the same thing: at init scale (where fp32 is well conditioned) both oracles agree to
    fp32 round-off on the plan's values and refits and on every world-model method."""
    cfg = workload(wl, num_envs=2)
    sd = synth_state_dict(cfg, seed=7, perturb=True, emb_scale=60.0 if cfg.multitask else 1.0)
    g = torch.Generator().manual_seed(3)
    obs = torch.randn(2, cfg.obs_shape["state"][0], generator=g)
    task = [1, 2] if cfg.multitask else None
    noise = draw_noise(cfg, 40, 2)
    t32 = plan_oracle(cfg, sd, obs, task=task, noise=noise)
    t64 = plan_oracle(cfg, sd, obs, task=task, noise=noise, dtype=torch.float64)
    assert t64.values.dtype == torch.float64
    err = float((t32.values.double() - t64.values).abs().max())
    print(wl, f"plan values fp32 - fp64: {err:.2e}")
    assert err <= 1e-5 * max(1.0, float(t64.values.abs().max()))
    assert float((t32.iter_mean[:, 0].double() - t64.iter_mean[:, 0]).abs().max()) < 1e-4
    o32, o64 = WMOracle(cfg, sd), WMOracle(cfg, sd, torch.float64)
    R = 64
    x = torch.randn(R, cfg.obs_shape["state"][0], generator=g)
    tk = torch.randint(0, len(cfg.tasks), (R,), generator=g) if cfg.multitask else None
    a = torch.rand(R, cfg.action_dim, generator=g) * 2 - 1
    eps = torch.randn(R, cfg.action_dim, generator=g)
    qidx = torch.tensor([0, 1])
    for name, f in (("z", lambda o: o.encode(x, tk)), ("next", lambda o: o.next(o.encode(x, tk), a, tk)),
                    ("q_all", lambda o: o.Q(o.encode(x, tk), a, tk, "all")),
                    ("pi", lambda o: o.pi(o.encode(x, tk), tk, eps)[0]),
                    ("entropy", lambda o: o.pi(o.encode(x, tk), tk, eps)[1]["entropy"]),
                    ("td", lambda o: o.td_target(o.encode(x, tk), a[:, :1], (a[:, 1:2] > 0).float(), tk, eps, qidx))):
        y32, y64 = f(o32), f(o64)
        assert y64.dtype == torch.float64, name
        d = float((y32.double() - y64).abs().max())
        assert d <= 2e-6 * max(1.0, float(y64.abs().max())), (name, d)


def test_fp64_oracle_default_is_fp32():
    cfg = workload("tiny")
    sd = synth_state_dict(cfg, seed=1)
    assert OracleModel(cfg, sd).dtype == torch.float32 and OracleModel(cfg, sd).sd["_pi.0.weight"].dtype == torch.float32


# ------------------------------------------------------------------------------------------------- trained-scale goldens
def test_oracle_matches_reference_golden_at_trained_scale():
    """tests/golden/tiny_sharp.npz, minted from the reference's own _plan on trained-scale weights: the comparisons of
    tests/test_oracle_golden.py with the value tolerance scaled by |v| (values reach 1e3 - 1e4 here)."""
    from helpers import boundary_separated, load_golden, stable_positions
    cfg, sd, calls = load_golden("tiny_sharp")
    model = OracleModel(cfg, sd)
    n_clamped = n_dominated = 0
    for c in calls:
        noise = draw_noise(cfg, c["seed"], 1, eval_mode=c["eval_mode"])
        tr = plan_oracle(cfg, model, c["obs"][None], t0=[c["t0"]], prev_mean=c["prev_mean"][None], noise=noise,
                         eval_mode=c["eval_mode"])
        scale = max(1.0, float(c["values"].abs().max()))
        assert torch.allclose(tr.values[0], c["values"], atol=2e-5 * scale, rtol=0)
        stable = stable_positions(c["values"], cfg.num_elites, 5e-6 * scale)
        assert stable.float().mean() > 0.9
        assert torch.equal(tr.elite_idx[0][stable], c["elite_idx"][stable])
        assert boundary_separated(c["values"], cfg.num_elites, 5e-6 * scale).all() and stable.all()
        assert torch.allclose(tr.action[0], c["action"], atol=1e-5, rtol=0)
        assert torch.allclose(tr.mean[0], c["mean"], atol=1e-5, rtol=0)
        wmax, clamped = refit_stats(cfg, tr)
        n_clamped += int(clamped.sum())
        n_dominated += int((wmax > 0.9).sum())
    assert n_clamped > 0 and n_dominated > 0       # the fixture pins the clamp and the dominated refit


@pytest.mark.parametrize("batch", ["b", "r"])
def test_oracle_matches_reference_world_model_at_trained_scale(batch):
    """tests/golden/c1_sharp_wm.npz: every method and _td_target of the reference on trained-scale weights, against the
    oracle, relative above |v| = 1 as tests/test_world_model_cpu.py."""
    from oracle.wm_oracle import load_case
    cfg, sd, recs = load_case("c1_sharp_wm")
    o = WMOracle(cfg, sd)
    r = recs[batch]
    z, a = r["z"], r["a"]
    got = {"z": o.encode(r["obs"], None), "next": o.next(z, a, None), "reward": o.reward(z, a, None)}
    act, info = o.pi(z, None, r["pi_eps"])
    got["pi_action"] = act
    for k in ("mean", "log_std", "entropy", "scaled_entropy"):
        got["pi_" + k] = info[k]
    sub = (Ellipsis, slice(0, r["q_all"].shape[-2]), slice(None))
    got["q_all"] = o.Q(z, a, None, "all")[sub]
    got["qt_all"] = o.Q(z, a, None, "all", target=True)[sub]
    got["q_min"] = o.Q(z, a, None, "min", qidx=r["q_min_qidx"])
    got["q_avg"] = o.Q(z, a, None, "avg", qidx=r["q_avg_qidx"])
    got["qt_min"] = o.Q(z, a, None, "min", target=True, qidx=r["qt_min_qidx"])
    got["td"] = o.td_target(z, r["reward_in"], r["terminated"], None, r["td_eps"], r["td_qidx"])
    worst = {}
    for k, v in got.items():
        assert v.shape == r[k].shape, (k, v.shape, r[k].shape)
        worst[k] = float(((v - r[k]).abs() / r[k].abs().clamp(min=1.0)).max())
    print(batch, {k: f"{e:.1e}" for k, e in worst.items()})
    # Q logits of magnitude ~10 differ by a few ulp between the reference's batched ensemble and per-head F.linear; the
    # two-hot values amplify that by d symexp(y) / symexp(y) = dy with |y| ~ 10, and the entropy's squash term
    # log(1 - tanh^2 + 1e-6) is ill-conditioned once actions saturate
    tol = {"q_all": 2e-5, "qt_all": 2e-5, "q_min": 1e-4, "q_avg": 1e-4, "qt_min": 1e-4, "td": 1e-4,
           "pi_entropy": 1e-5, "pi_scaled_entropy": 1e-5}
    assert all(e <= tol.get(k, 2e-6) for k, e in worst.items()), worst
    assert float(r["q_min"].abs().max()) > 1e3 and float((r["pi_action"].abs() > 0.999).float().mean()) > 0.2
