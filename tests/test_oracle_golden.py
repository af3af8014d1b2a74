"""The CPU oracle (oracle/plan_oracle.py) against golden vectors minted from the
reference's own unmodified `_plan` (oracle/make_golden.py).  CPU only."""
import pytest
import torch

from oracle.plan_oracle import draw_noise, plan_oracle
from helpers import load_golden, stable_positions, boundary_separated

CASES = ["tiny", "tiny_mt", "c1_dog5m", "tiny_episodic", "c1_dog5m_episodic", "tiny_rgb", "tiny_nopi", "tiny_h1", "tiny_knobs",
         "tiny_mt_t5", "tiny_wide_heads", "tiny_odd_widths",
         pytest.param("c3_humanoid48m_e1", marks=pytest.mark.slow),
         pytest.param("c4_mt80_317m_e1", marks=pytest.mark.slow)]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    cfg, sd, calls = load_golden(name)
    from oracle.plan_oracle import OracleModel
    model = OracleModel(cfg, sd)
    for c in calls:
        noise = draw_noise(cfg, c["seed"], 1, eval_mode=c["eval_mode"])
        tr = plan_oracle(cfg, model, c["obs"][None], task=None if c["task"] is None else [c["task"]],
                         t0=[c["t0"]], prev_mean=c["prev_mean"][None], noise=noise, eval_mode=c["eval_mode"])
        # fp32: the oracle re-uses torch's own kernels, only the Q-ensemble goes through
        # per-head F.linear instead of vmap/bmm -> a few ulp.  Tolerance 2e-5 abs on
        # trajectory values (|v| ~ 1), 1e-5 on actions/means.
        assert torch.allclose(tr.values[0], c["values"], atol=2e-5, rtol=0)
        # observed |dv| <= 7e-7, so positions separated by > 5e-6 must agree bit-exactly
        stable = stable_positions(c["values"], cfg.num_elites, 5e-6)
        assert stable.float().mean() > 0.9
        assert torch.equal(tr.elite_idx[0][stable], c["elite_idx"][stable])      # bit-exact top-k indices
        if boundary_separated(c["values"], cfg.num_elites, 5e-6).all() and stable.all():
            assert torch.allclose(tr.action[0], c["action"], atol=1e-5, rtol=0)
            assert torch.allclose(tr.mean[0], c["mean"], atol=1e-5, rtol=0)


def test_noise_stream_is_the_reference_stream():
    """draw_noise(seed) reproduces torch.manual_seed(seed) + the reference's draw order."""
    cfg, _, _ = load_golden("tiny")
    n = draw_noise(cfg, 5, 1)
    torch.manual_seed(5)
    H, N, P, A = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim
    for t in range(H):
        assert torch.equal(torch.randn(P, A), n.prior[0, t])
    for it in range(cfg.iterations):
        assert torch.equal(torch.randn(H, N - P, A), n.r[0, it])
        assert torch.equal(torch.randn_like(torch.empty(N, A)), n.pi[0, it])
        assert torch.equal(torch.randperm(cfg.num_q)[:2], n.qidx[0, it])
    assert torch.equal(torch.empty(cfg.num_elites).exponential_(), n.expo[0])
    assert torch.equal(torch.randn(A), n.final[0])


def test_batched_oracle_is_independent_envs():
    cfg, sd, calls = load_golden("tiny_mt")
    E = 3
    g = torch.Generator().manual_seed(0)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    pm = torch.randn(E, cfg.horizon, cfg.action_dim, generator=g) * 0.2
    task, t0 = [0, 3, 1], [False, True, False]
    noise = draw_noise(cfg, 77, E)
    tr = plan_oracle(cfg, sd, obs, task=task, t0=t0, prev_mean=pm, noise=noise)
    for e in range(E):
        one = plan_oracle(cfg, sd, obs[e:e + 1], task=[task[e]], t0=[t0[e]], prev_mean=pm[e:e + 1],
                          noise=draw_noise(cfg, 77 + e, 1))
        assert torch.equal(one.action[0], tr.action[e])
    # masked action dims are exactly zero (world_model.py:158-162, tdmpc2.py:180-181,195-197)
    for e in range(E):
        a = cfg.action_dims[task[e]]
        assert torch.all(tr.action[e, a:] == 0) and torch.all(tr.mean[e, :, a:] == 0)


def test_episodic_oracle_properties():
    """cfg.episodic (tdmpc2.py:126-136): a never-terminating head reproduces the non-episodic values bit for bit,
    an always-terminating head leaves only the first discounted reward."""
    from oracle.plan_oracle import OracleModel, estimate_value, two_hot_inv
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    cfg_e, cfg_0 = workload("tiny", episodic=True), workload("tiny")
    sd = synth_state_dict(cfg_e, seed=4, perturb=True)
    g = torch.Generator().manual_seed(2)
    N = cfg_e.num_samples
    z = torch.softmax(torch.randn(N, cfg_e.latent_dim // 8, 8, generator=g), -1).view(N, -1)
    acts = torch.rand(cfg_e.horizon, N, cfg_e.action_dim, generator=g) * 2 - 1
    eps, qidx = torch.randn(N, cfg_e.action_dim, generator=g), torch.tensor([1, 0])
    base = estimate_value(OracleModel(cfg_0, sd), z, acts, None, eps, qidx)
    sd["_termination.2.bias"] = torch.full((1,), -50.0)
    assert torch.equal(estimate_value(OracleModel(cfg_e, sd), z, acts, None, eps, qidx), base)
    sd["_termination.2.bias"] = torch.full((1,), 50.0)
    m = OracleModel(cfg_e, sd)
    first = two_hot_inv(m.reward(z, acts[0], None), cfg_e)
    assert torch.equal(estimate_value(m, z, acts, None, eps, qidx), first)


def test_oracle_properties_t0_eval_mode_nan():
    """Properties SURVEY.md 8(c) lists for the reference planner, held on the oracle:
    t0=True ignores _prev_mean (tdmpc2.py:166-167); eval_mode skips the final exploration draw and returns the picked
    elite action itself (tdmpc2.py:203-204); NaN trajectory values count as 0 (tdmpc2.py:184)."""
    from oracle.plan_oracle import OracleModel
    cfg, sd, calls = load_golden("tiny")
    model = OracleModel(cfg, sd)
    obs = calls[0]["obs"][None]
    noise = draw_noise(cfg, 9, 1)
    pm_a = torch.zeros(1, cfg.horizon, cfg.action_dim)
    pm_b = torch.full((1, cfg.horizon, cfg.action_dim), 0.7)
    a = plan_oracle(cfg, model, obs, t0=[True], prev_mean=pm_a, noise=noise)
    b = plan_oracle(cfg, model, obs, t0=[True], prev_mean=pm_b, noise=noise)
    assert torch.equal(a.action, b.action) and torch.equal(a.values, b.values)
    c = plan_oracle(cfg, model, obs, t0=[False], prev_mean=pm_b, noise=noise)
    assert not torch.equal(a.values, c.values)                       # the warm start is used when t0 is False
    # eval_mode: same trajectory values, action == the picked elite's first action (no std * randn term)
    ev = plan_oracle(cfg, model, obs, t0=[True], prev_mean=pm_a, noise=noise, eval_mode=True)
    assert torch.equal(ev.values, a.values) and torch.equal(ev.pick, a.pick)
    assert not torch.equal(ev.action, a.action)
    assert float((a.action - (ev.action + a.std[:, 0] * noise.final).clamp(-1, 1)).abs().max()) < 1e-6
    # NaN observation -> every value NaN -> nan_to_num(0): all values exactly 0 (which K of the tied samples torch.topk
    # returns is implementation-defined; the kernels break ties towards the lower index)
    nan = plan_oracle(cfg, model, torch.full_like(obs, float("nan")), t0=[True], prev_mean=pm_a, noise=noise)
    assert torch.all(nan.values == 0)
