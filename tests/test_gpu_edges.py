"""Edge cases of the planning path on the GPU (through the C ABI / agent API) against the oracle:
ragged sample counts (N not a multiple of the 128-row tile), no policy-prior trajectories, horizon 1,
odd environment counts, single-env reference shapes, NaN guard, checkpoint round trip."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import stable_positions, boundary_separated

pytestmark = pytest.mark.gpu


def _run_and_compare(cfg, E, sd, seed=11, eval_mode=False, obs_scale=1.0, atol_v=5e-5):
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    from tdmpc2_b200.planner import Noise, Planner
    g = torch.Generator().manual_seed(seed)
    obs = obs_scale * torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [bool((i + 1) % 2) for i in range(E)]
    task = [(3 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    n = oracle_noise(cfg, 70 + seed, E, eval_mode=eval_mode)
    want = plan_oracle(cfg, sd, obs, task=task, t0=t0, prev_mean=prev, noise=n, eval_mode=eval_mode)
    pl = Planner(cfg, E, "cuda:0")
    pl.pack(sd)
    noise = Noise.from_env_major(n.prior, n.r, n.pi, n.qidx, n.expo, None if eval_mode else n.final, device="cuda")
    taskv = torch.tensor(task, dtype=torch.int32).cuda() if task is not None else None
    action, new_mean, tr = pl.plan(obs.cuda().contiguous(), taskv, torch.tensor(t0, dtype=torch.uint8).cuda(),
                                   prev.cuda().contiguous(), noise, trace=True)
    torch.cuda.synchronize()
    K, n_ok = cfg.num_elites, 0
    for e in range(E):
        clean = True
        for it in range(cfg.iterations):
            if not clean:
                break
            got, ref = tr["values"][e, it].cpu(), want.values[e, it]
            assert torch.allclose(got, ref, atol=atol_v, rtol=1e-5), f"env {e} it {it}: {(got - ref).abs().max():.3e}"
            st = stable_positions(ref, K, 1e-4) if K < cfg.num_samples else torch.zeros(K, dtype=torch.bool)
            assert torch.equal(tr["elite_idx"][e, it].cpu()[st], want.elite_idx[e, it][st])
            clean = bool(boundary_separated(ref, K, 1e-4)) if K < cfg.num_samples else True
        if clean:
            assert torch.allclose(new_mean[e].cpu(), want.mean[e], atol=1e-4, rtol=0)
            n_ok += 1
    assert n_ok > 0
    return action.cpu(), want


@pytest.mark.parametrize("over", [
    dict(num_samples=200, num_elites=24, num_pi_trajs=8),      # ragged: 2 tiles, second one 72 rows
    dict(num_samples=128, num_elites=16, num_pi_trajs=0),      # no policy-prior trajectories
    dict(num_samples=96, num_elites=96, num_pi_trajs=5),       # every sample is an elite; N < one tile
    dict(horizon=1, num_samples=128, num_elites=16),           # single-step rollout
    dict(num_q=2, iterations=1),                               # smallest ensemble, one iteration
])
def test_ragged_and_degenerate_shapes(over):
    cfg = workload("tiny", num_envs=3, **over)
    sd = synth_state_dict(cfg, seed=21, perturb=True)
    _run_and_compare(cfg, 3, sd)


def test_multitask_odd_env_count_eval_mode():
    cfg = workload("tiny-mt", num_envs=5, num_samples=160, num_elites=20)
    sd = synth_state_dict(cfg, seed=22, perturb=True, emb_scale=60.0)
    action, want = _run_and_compare(cfg, 5, sd, eval_mode=True)
    assert action.abs().max() <= 1.0


def test_nan_values_are_zeroed_like_nan_to_num():
    """Infinite observations make every trajectory value NaN; tdmpc2.py:184 turns them into 0."""
    from tdmpc2_b200.planner import Planner, draw_noise
    cfg = workload("tiny", num_envs=1)
    sd = synth_state_dict(cfg, seed=23, perturb=True)
    pl = Planner(cfg, 1, "cuda:0")
    pl.pack(sd)
    obs = torch.full((1, cfg.obs_shape["state"][0]), float("inf"), device="cuda")
    n = draw_noise(cfg, 1, "cuda:0")
    action, mean, tr = pl.plan(obs, None, torch.ones(1, dtype=torch.uint8, device="cuda"),
                               torch.zeros(1, cfg.horizon, cfg.action_dim, device="cuda"), n, trace=True)
    torch.cuda.synchronize()
    assert torch.all(tr["values"] == 0)
    # all-equal values: ties resolve to the lowest indices, like a stable descending sort
    assert torch.equal(tr["elite_idx"][0, 0].cpu(), torch.arange(cfg.num_elites))
    # (the policy-prior actions are NaN too and are among the tied elites, so the refit mean is NaN in the
    #  reference as well; only the value guard is specified behaviour)


def test_agent_api_shapes_state_and_checkpoint(tmp_path):
    """Reference-shaped surface: act() on CPU obs returns a CPU action in [-1,1]; _prev_mean is carried;
    save()/load() round-trips through the reference's {"model": state_dict} format."""
    from tdmpc2_b200.tdmpc2 import TDMPC2
    cfg = workload("tiny", num_envs=1)
    agent = TDMPC2(cfg, device="cuda:0")
    agent.load(synth_state_dict(cfg, seed=24, perturb=True))
    agent.generator = torch.Generator(device="cuda:0").manual_seed(5)
    obs = torch.randn(cfg.obs_shape["state"][0])
    a0 = agent.act(obs, t0=True)
    assert a0.device.type == "cpu" and a0.shape == (cfg.action_dim,) and a0.abs().max() <= 1
    pm = agent._prev_mean.clone()
    assert pm.shape == (cfg.horizon, cfg.action_dim) and pm.abs().sum() > 0
    a1 = agent.act(obs, t0=False, eval_mode=True)
    assert not torch.equal(agent._prev_mean, pm)
    fp = tmp_path / "agent.pt"
    agent.save(fp)
    other = TDMPC2(workload("tiny", num_envs=1), device="cuda:0")
    other.load(str(fp))
    other.generator = torch.Generator(device="cuda:0").manual_seed(5)
    agent.generator = torch.Generator(device="cuda:0").manual_seed(5)
    agent._prev_mean.zero_(); other._prev_mean.zero_()
    assert torch.equal(agent.act(obs, t0=True), other.act(obs, t0=True))
    # batched agent: [E, obs] in, [E, A] out, one _prev_mean per environment
    cfgb = workload("tiny", num_envs=4)
    b = TDMPC2(cfgb, device="cuda:0")
    b.load(synth_state_dict(cfgb, seed=24, perturb=True))
    out = b.act(torch.randn(4, cfgb.obs_shape["state"][0]), t0=torch.tensor([True, False, True, False]))
    assert out.shape == (4, cfgb.action_dim) and b._prev_mean.shape == (4, cfgb.horizon, cfgb.action_dim)
    with pytest.raises(ValueError):
        b.act(torch.randn(3, cfgb.obs_shape["state"][0]))


def test_non_mpc_act_runs_the_policy_through_the_kernels():
    """cfg.mpc = False (tdmpc2.py:116-120): act() = pi(encode(obs)) with noise, or tanh(mean) in eval_mode -- both come
    from the row-mode encode and pi launches and must match the oracle's encode/pi (1e-5, like the prior test)."""
    from oracle.plan_oracle import OracleModel
    from tdmpc2_b200.tdmpc2 import TDMPC2
    E = 3
    cfg = workload("tiny-mt", num_envs=E, mpc=False)
    sd = synth_state_dict(cfg, seed=25, perturb=True, emb_scale=60.0)
    agent = TDMPC2(cfg, device="cuda:0")
    agent.load(sd)
    g = torch.Generator().manual_seed(4)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    eps = torch.randn(E, cfg.action_dim, generator=g)
    task = [1, 3, 0]
    om = OracleModel(cfg, sd)
    want_eval = torch.stack([om.pi(om.encode(obs[e:e + 1], task[e]), task[e], torch.zeros(1, cfg.action_dim))[0] for e in range(E)])
    want_eps = torch.stack([om.pi(om.encode(obs[e:e + 1], task[e]), task[e], eps[e:e + 1])[0] for e in range(E)])
    got_eval = agent.act(obs, eval_mode=True, task=task)
    assert got_eval.device.type == "cpu" and got_eval.shape == (E, cfg.action_dim)
    assert torch.allclose(got_eval, want_eval, atol=1e-5, rtol=0), (got_eval - want_eval).abs().max()
    got_eps = agent._policy_action(obs.cuda(), eval_mode=False, task=task, eps=eps).cpu()
    assert torch.allclose(got_eps, want_eps, atol=1e-5, rtol=0), (got_eps - want_eps).abs().max()
    for e in range(E):                                     # masked action dims are exactly 0 (world_model.py:158-162)
        assert torch.all(got_eps[e, cfg.action_dims[task[e]]:] == 0)


@pytest.mark.parametrize("wl,engine", [("c1", "tcgen05x2"), ("c1", "tcgen05"), ("tiny-mt", "tcgen05x2"), ("tiny-mt", "simt")])
def test_shared_latent_fold_only_reorders_the_sum(wl, engine, monkeypatch):
    """At rollout step 0 every sample row of an environment carries the same [z | emb] (z.repeat(N), tdmpc2.py:163): the
    prologue folds its product with reward.0 / dynamics.0 into a per-environment bias (zbias_kernel) and the t = 0
    GEMMs cover the action columns only.  Same sum, different association: trajectory values with the fold on and off
    agree to fp32 round-off (2e-5), far inside the 5e-5 the oracle comparison allows."""
    from tdmpc2_b200.planner import Planner, draw_noise
    E = 3
    cfg = workload(wl, num_envs=E)
    sd = synth_state_dict(cfg, seed=11, perturb=True)
    g = torch.Generator().manual_seed(5)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g).cuda()
    prev = (0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)).cuda()
    t0 = torch.tensor([1, 0, 0], dtype=torch.uint8).cuda()
    task = torch.tensor([2, 0, 1], dtype=torch.int32).cuda() if cfg.multitask else None
    noise = draw_noise(cfg, E, "cuda", generator=torch.Generator(device="cuda").manual_seed(9), reference_order=False)
    vals = {}
    for fold in ("1", "0"):
        monkeypatch.setenv("TDMPC2_B200_ZFOLD", fold)
        pl = Planner(cfg, E, "cuda:0", engine=engine)
        pl.pack(sd)
        _, _, tr = pl.plan(obs, task, t0, prev, noise, trace=True)
        torch.cuda.synchronize()
        vals[fold] = tr["values"][:, 0].cpu()          # first iteration: identical inputs on both sides
    d = (vals["1"] - vals["0"]).abs().max().item()
    assert 0.0 < d < 2e-5, d                           # > 0: the fold really ran


@pytest.mark.parametrize("wl", ["tiny", "tiny-mt", "tiny-rgb"])
def test_one_environment_paths_agree_bit_for_bit(wl):
    """One environment per act() (the reference's call shape) has three host paths: draws interleaved with the launches
    (default), all draws then one CUDA-graph replay, all draws then eager launches.  Same generator, same kernels: the
    actions and the carried _prev_mean must be identical, call after call (t0, warm start, eval_mode)."""
    from tdmpc2_b200.tdmpc2 import TDMPC2
    sd = synth_state_dict(workload(wl, num_envs=1), seed=26, perturb=True)
    g = torch.Generator().manual_seed(12)
    base = workload(wl, num_envs=1)
    obs = [torch.randint(0, 256, tuple(base.obs_shape["rgb"]), generator=g).float() if base.get("obs", "state") == "rgb"
           else torch.randn(base.obs_shape["state"][0], generator=g) for _ in range(4)]
    task = 2 if base.multitask else None
    outs = {}
    for name, over in (("interleaved", {}), ("graph", dict(e1_interleaved=False)), ("eager", dict(cuda_graph=False))):
        agent = TDMPC2(workload(wl, num_envs=1, **over), device="cuda:0")
        agent.load(sd)
        agent.generator = torch.Generator(device="cuda:0").manual_seed(77)
        if name == "graph":                      # capture (which draws from the default generator) before the seeded stream starts
            agent.act(obs[0], t0=True, task=task); agent.act(obs[0], t0=True, eval_mode=True, task=task)
            agent.generator = torch.Generator(device="cuda:0").manual_seed(77)
            agent._prev_mean.zero_()
        seq = []
        for i, (t0, ev) in enumerate([(True, False), (False, False), (False, True), (False, False)]):
            a = agent.act(obs[i], t0=t0, eval_mode=ev, task=task)
            seq.append((a.clone(), agent._prev_mean.cpu().clone()))
        outs[name] = seq
        if name == "interleaved":
            assert agent.planner._e1_noise and not agent.planner._graphs
        if name == "graph":
            assert agent.planner._graphs and not agent.planner._e1_noise
    for other in ("graph", "eager"):
        for i, ((a, m), (b, n)) in enumerate(zip(outs["interleaved"], outs[other])):
            assert torch.equal(a, b) and torch.equal(m, n), f"{wl}: call {i} differs between interleaved and {other}"
