"""Edge cases of the planning path on the GPU (through the C ABI / agent API) against the oracle:
ragged sample counts (N not a multiple of the 128-row tile), no policy-prior trajectories, horizon 1,
odd environment counts, single-env reference shapes, NaN guard, checkpoint round trip."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import compare_with_oracle, planner_for, to_gpu_noise

pytestmark = pytest.mark.gpu


def _run_and_compare(cfg, E, sd, seed=11, eval_mode=False):
    """One plan() against the oracle (helpers.compare_with_oracle; top-k separated by 1e-4)."""
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [bool((i + 1) % 2) for i in range(E)]
    task = [(3 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    n = oracle_noise(cfg, 70 + seed, E, eval_mode=eval_mode)
    want = plan_oracle(cfg, sd, obs, task=task, t0=t0, prev_mean=prev, noise=n, eval_mode=eval_mode)
    pl = planner_for(cfg, E, None, sd)
    taskv = torch.tensor(task, dtype=torch.int32).cuda() if task is not None else None
    action, new_mean, tr = pl.plan(obs.cuda().contiguous(), taskv, torch.tensor(t0, dtype=torch.uint8).cuda(),
                                   prev.cuda().contiguous(), to_gpu_noise(n, eval_mode), trace=True)
    torch.cuda.synchronize()
    counts = compare_with_oracle(cfg, tr, action, new_mean, want, n, range(E), gap=1e-4)
    print(counts)
    assert counts["means"] > 0, counts
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
    from tdmpc2_b200.planner import draw_noise
    cfg = workload("tiny", num_envs=1)
    sd = synth_state_dict(cfg, seed=23, perturb=True)
    pl = planner_for(cfg, 1, None, sd)
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


@pytest.mark.parametrize("wl,engine", [("c1", "tcgen05"), ("tiny-mt", "tcgen05"), ("tiny-mt", "simt")])
def test_shared_latent_fold_only_reorders_the_sum(wl, engine, monkeypatch):
    """At rollout step 0 every sample row of an environment carries the same [z | emb] (z.repeat(N), tdmpc2.py:163): the
    prologue folds its product with reward.0 / dynamics.0 into a per-environment bias (zbias_kernel) and the t = 0
    GEMMs cover the action columns only.  Same sum, different association: trajectory values with the fold on and off
    agree to fp32 round-off (2e-5), far inside the 5e-5 the oracle comparison allows."""
    from tdmpc2_b200.planner import draw_noise
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
        pl = planner_for(cfg, E, engine, sd)
        _, _, tr = pl.plan(obs, task, t0, prev, noise, trace=True)
        torch.cuda.synchronize()
        vals[fold] = tr["values"][:, 0].cpu()          # first iteration: identical inputs on both sides
    d = (vals["1"] - vals["0"]).abs().max().item()
    assert 0.0 < d < 2e-5, d                           # > 0: the fold really ran


def test_only_the_two_engines_are_accepted():
    """"tcgen05" and "simt" (codes 0 and 1) are the engines; the names and codes of the removed Blackwell-era engines are
    errors, not aliases of "tcgen05"."""
    from tdmpc2_b200.planner import Planner
    cfg = workload("tiny", num_envs=1)
    for name in ("auto", "tcgen05x2", "tcgen05pp", "tcgen05x2pf"):
        with pytest.raises(ValueError, match="'tcgen05' and 'simt'"):
            Planner(cfg, 1, "cuda:0", engine=name)
    pl = Planner(cfg, 1, "cuda:0")
    assert pl.iter_engine == "tcgen05"
    for code in (2, 3, 4, 5):
        assert pl.lib.tdmpc2_planner_set_engine(pl.h, code) == -1         # TDMPC2_ERR_INVALID
    assert Planner(cfg, 1, "cuda:0", engine="simt").iter_engine == "simt"


def test_obs_or_latent_rules_of_prologue_and_world_model_loss():
    """The prologue takes exactly one of obs and z; the world-model loss backward takes dz0 exactly when obs0 is NULL.
    Both other combinations are TDMPC2_ERR_INVALID on every planner.  A pixel planner refuses obs (prologue:
    TDMPC2_ERR_STATE) and obs0 (loss forward and backward: TDMPC2_ERR_UNSUPPORTED).  Valid calls still return 0."""
    import ctypes as C
    from tdmpc2_b200.planner import _ptr
    from tdmpc2_b200.tdmpc2 import TDMPC2
    H, B = 2, 4
    for wl in ("tiny", "tiny-rgb"):
        cfg = workload(wl, num_envs=1)
        agent = TDMPC2(cfg, device="cuda:0")
        agent.model.load_state_dict(synth_state_dict(cfg, seed=27, perturb=True))
        pl, lib, rgb = agent.planner, agent.planner.lib, wl == "tiny-rgb"
        g = torch.Generator().manual_seed(8)
        obs_shape = tuple(cfg.obs_shape["rgb"]) if rgb else (cfg.obs_shape["state"][0],)
        obs = torch.rand(B, *obs_shape, generator=g).cuda()
        z = torch.softmax(torch.randn(B, cfg.latent_dim // cfg.simnorm_dim, cfg.simnorm_dim, generator=g), -1).reshape(B, -1).cuda()
        t0, prev = torch.ones(1, dtype=torch.uint8, device="cuda"), torch.zeros(1, cfg.horizon, cfg.action_dim, device="cuda")
        prior = torch.randn(1, cfg.horizon, cfg.num_pi_trajs, cfg.action_dim, generator=g).cuda()

        def prologue(o, zz):
            return lib.tdmpc2_plan_prologue(pl.h, _ptr(o), _ptr(zz), None, _ptr(t0), _ptr(prev), _ptr(prior), pl._stream())
        assert prologue(obs[:1], z[:1]) == -1 and prologue(None, None) == -1, wl
        assert b"exactly one of obs and z" in lib.tdmpc2_last_error()
        if rgb:
            assert prologue(obs[:1], None) == -4 and b"pass z, not obs" in lib.tdmpc2_last_error()
        assert prologue(None if rgb else obs[:1], z[:1] if rgb else None) == 0, wl

        act = (torch.rand(H * B, cfg.action_dim, generator=g) * 2 - 1).cuda()
        zs = torch.empty(H + 1, B, cfg.latent_dim, device="cuda")
        zs[0] = z
        tape, zs, ql, rl, tl = pl.wm_loss_forward(None if rgb else obs, act, None, None, H, B, zs=zs)
        next_z, rew, td, term = zs[1:].clone(), torch.rand(H * B, 1).cuda(), torch.rand(H * B, 1).cuda(), torch.zeros(H * B, 1).cuda()
        grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in agent._wm_keys}
        W, G, cf = pl._wm_loss_structs(agent.model.tensor, grads)
        ws = pl._scratch(lib.tdmpc2_wm_loss_workspace_bytes, pl.h, H, B)
        dz0 = torch.empty(B, cfg.latent_dim, device="cuda")

        def backward(o, d):
            return lib.tdmpc2_wm_loss_backward(pl.h, C.byref(W), _ptr(tape), _ptr(o), _ptr(act), None, None, H, B, _ptr(zs),
                                               _ptr(ql), _ptr(rl), _ptr(tl), _ptr(next_z), _ptr(rew), _ptr(td), _ptr(term),
                                               C.byref(cf), C.byref(G), _ptr(d), _ptr(ws), pl._stream())
        assert backward(None, None) == -1 and b"dz0 must be non-NULL exactly when obs0 is NULL" in lib.tdmpc2_last_error()
        if rgb:
            fwd = lib.tdmpc2_wm_loss_forward(pl.h, _ptr(obs), _ptr(act), None, None, H, B, _ptr(zs), _ptr(ql), _ptr(rl),
                                             _ptr(tl), _ptr(tape), pl._stream())
            assert fwd == -5 and b"no state encoder" in lib.tdmpc2_last_error()
            assert backward(obs, None) == -5 and backward(obs, dz0) == -5
        else:
            assert backward(obs, dz0) == -1 and b"dz0 must be non-NULL" in lib.tdmpc2_last_error()
            assert backward(obs, None) == 0
        assert backward(None, dz0) == 0, wl
        torch.cuda.synchronize()


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
