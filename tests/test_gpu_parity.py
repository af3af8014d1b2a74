"""GPU parity tests: the fused sm_90a kernels (through the C ABI) against the CPU
oracle on identical weights, inputs and noise.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import TERM_MARGIN, boundary_separated, compare_with_oracle, layer_list, planner_for, to_gpu_noise

pytestmark = pytest.mark.gpu

ENGINES = ["simt", "tcgen05"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("wl", ["tiny", "tiny-mt", "c1", "tiny-wide", "tiny-wide2", "tiny-episodic"])
def test_fused_layer_matches_fp64(engine, wl):
    """One packed layer (GEMM on split fp16 operands + bias + LN + Mish/SimNorm) vs float64.
    Tolerance: 1e-5 abs + 1e-5 rel -- fp32 round-off level (3-pass fp16 split carries ~22 bits)."""
    cfg = workload("tiny", episodic=True) if wl == "tiny-episodic" else workload(wl)
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    pl = planner_for(cfg, 2, engine, sd)
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    for (li, prefix, head, has_ln, simnorm) in layer_list(cfg):
        W, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
        if head is not None:
            W, b = W[head], b[head]
        if W.shape[1] > pl.cfg.latent_dim + pl.cfg.action_dim + pl.cfg.task_dim + 64 and not prefix.startswith("_encoder"):
            continue
        rows = 128 if li % 2 == 0 else 77
        x = torch.randn(rows, W.shape[1], generator=g)
        A = cfg.action_dim
        Apad = (A + 31) // 32 * 32
        n_out = Apad + A if prefix == "_pi.2" else W.shape[0]
        try:
            y_lin = pl.debug_layer(li, 0, x.cuda(), n_out).cpu().double()
        except Exception as e:
            if "wider than the X scratch" in str(e):
                continue
            raise
        ref = x.double() @ W.double().T + b.double()
        if prefix == "_pi.2":
            # the packer moves the log_std rows [A, 2A) to the 32-aligned column pad32(A)
            assert torch.all(y_lin[:, A:Apad] == 0)
            y_lin = torch.cat([y_lin[:, :A], y_lin[:, Apad:Apad + A]], dim=1)
        err = (y_lin - ref).abs().max().item()
        worst = max(worst, err)
        assert torch.allclose(y_lin, ref, atol=1e-5, rtol=1e-5), f"{prefix} head={head} linear err {err}"
        if has_ln:
            gw, gb = sd[prefix + ".ln.weight"], sd[prefix + ".ln.bias"]
            if head is not None:
                gw, gb = gw[head], gb[head]
            ln = torch.nn.functional.layer_norm(ref, (ref.shape[-1],), gw.double(), gb.double(), 1e-5)
            if simnorm:
                want = torch.softmax(ln.view(rows, -1, 8), -1).view(rows, -1)
            else:
                want = torch.nn.functional.mish(ln)
            got = pl.debug_layer(li, 2 if simnorm else 1, x.cuda(), W.shape[0]).cpu().double()
            assert torch.allclose(got, want, atol=1e-5, rtol=1e-5), \
                f"{prefix} head={head} ln/act err {(got - want).abs().max().item()}"
    print(f"[{engine}/{wl}] worst linear abs err {worst:.3e}")


CASES = [  # workload, E, perturb, emb_scale, eval_mode
    ("tiny", 2, True, 1.0, False),
    ("tiny-mt", 3, True, 60.0, False),
    ("tiny-mt", 3, True, 1.0, True),
    ("c1", 2, False, 1.0, False),
    ("tiny-wide", 2, True, 1.0, False),     # hidden width 640 > 512: five 128-column output blocks
    ("tiny-wide2", 2, True, 1.0, False),    # 1152-wide hidden (3 super-chunks), 576-wide SimNorm latent, 640-wide encoder
]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("wl,E,perturb,emb_scale,eval_mode", CASES)
def test_plan_matches_oracle(engine, wl, E, perturb, emb_scale, eval_mode):
    """Full plan(): prologue, every CEM iteration, epilogue -- kernel trace vs oracle trace.
    Tolerances: trajectory values 5e-5 abs (values are O(1); observed error ~1e-6);
    top-k indices bit-exact wherever the oracle's sorted values are separated by > 1e-4;
    means/stds/actions 1e-4 (the north-star tolerance) for environments whose elite set
    is well separated in every iteration."""
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    cfg = workload(wl, num_envs=E)
    sd = synth_state_dict(cfg, seed=7, perturb=perturb, emb_scale=emb_scale)
    g = torch.Generator().manual_seed(3)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [bool(i % 2) for i in range(E)]
    task = [(2 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None
    noise = oracle_noise(cfg, 40, E, eval_mode=eval_mode)
    want = plan_oracle(cfg, sd, obs, task=task, t0=t0, prev_mean=prev, noise=noise, eval_mode=eval_mode)

    pl = planner_for(cfg, E, engine, sd)
    taskv = torch.tensor(task, dtype=torch.int32).cuda() if task is not None else None
    action, new_mean, tr = pl.plan(obs.cuda().contiguous(), taskv, torch.tensor(t0, dtype=torch.uint8).cuda(),
                                   prev.cuda().contiguous(), to_gpu_noise(noise, eval_mode), trace=True)
    torch.cuda.synchronize()
    cpu = lambda t: t.detach().cpu()
    assert torch.allclose(cpu(tr["z"]), want.z, atol=2e-6, rtol=1e-5), "encode()"
    assert torch.allclose(cpu(tr["pi_actions"]), want.pi_actions, atol=1e-5, rtol=0), "policy-prior trajectories"
    n = compare_with_oracle(cfg, tr, action, new_mean, want, noise, range(E), gap=1e-4)
    print(wl, engine, n)
    assert n["topk"] > 0 and n["means"] > 0, f"test inputs too degenerate: nothing was compared: {n}"
    if cfg.multitask:
        for e in range(E):
            a = cfg.action_dims[task[e]]
            assert torch.all(cpu(action[e, a:]) == 0) and torch.all(cpu(new_mean[e, :, a:]) == 0)


@pytest.mark.parametrize("engine", ENGINES)
def test_estimate_value_matches_oracle(engine):
    from oracle.plan_oracle import OracleModel, estimate_value
    cfg = workload("tiny-mt", num_envs=2)
    sd = synth_state_dict(cfg, seed=9, perturb=True)
    E, N, H, A, L = 2, cfg.num_samples, cfg.horizon, cfg.action_dim, cfg.latent_dim
    g = torch.Generator().manual_seed(1)
    z = torch.softmax(torch.randn(E, N, L // 8, 8, generator=g), -1).view(E, N, L)
    actions = torch.rand(E, H, N, A, generator=g) * 2 - 1
    eps = torch.randn(E, N, A, generator=g)
    qidx = torch.tensor([[0, 2], [3, 1]])
    task = [1, 2]
    model = OracleModel(cfg, sd)
    want = torch.stack([estimate_value(model, z[e], actions[e], task[e], eps[e], qidx[e]).squeeze(1) for e in range(E)])
    pl = planner_for(cfg, E, engine, sd)
    got = pl.estimate_value(z.cuda().contiguous(), actions.cuda().contiguous(), torch.tensor(task, dtype=torch.int32).cuda(),
                            eps.cuda().contiguous(), qidx.to(torch.int32).cuda().contiguous()).cpu()
    assert torch.allclose(got, want, atol=5e-5, rtol=1e-5), (got - want).abs().max()


@pytest.mark.parametrize("perturb", [False, True])
def test_tensor_core_engine_matches_oracle_and_simt_engine(perturb):
    """The wgmma engine and the CUDA-core (SIMT) engine sum the same products in different orders, so they are checked
    to tolerance against each other and against the oracle: tensor-core values within 5e-5 + 1e-5 |v| of the oracle
    and of the SIMT engine, top-k indices exact on separated positions, refit mean/std, new mean and action 1e-4."""
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    E = 3
    cfg = workload("c1", num_envs=E)
    sd = synth_state_dict(cfg, seed=11, perturb=perturb)
    g = torch.Generator().manual_seed(6)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [True, False, False]
    noise = oracle_noise(cfg, 43, E)
    want = plan_oracle(cfg, sd, obs, task=None, t0=t0, prev_mean=prev, noise=noise)
    out = {}
    for engine in ("simt", "tcgen05"):
        pl = planner_for(cfg, E, engine, sd)
        a, m, tr = pl.plan(obs.cuda(), None, torch.tensor(t0, dtype=torch.uint8).cuda(), prev.cuda(),
                           to_gpu_noise(noise), trace=True)
        torch.cuda.synchronize()
        out[engine] = (a.cpu(), m.cpu(), {k: v.cpu() for k, v in tr.items()})
    action, new_mean, tr = out["tcgen05"]
    n = compare_with_oracle(cfg, tr, action, new_mean, want, noise, range(E), gap=1e-4)
    print(perturb, n)
    assert n["topk"] > 0, n
    v_simt = out["simt"][2]["values"]
    for e in range(E):                 # the engines' values agree for as long as the oracle's elite sets are separated
        for it in range(cfg.iterations):
            assert torch.allclose(tr["values"][e, it], v_simt[e, it], atol=5e-5, rtol=1e-5), f"tensor core vs simt env={e} it={it}"
            if not boundary_separated(want.values[e, it], cfg.num_elites, 1e-4):
                break


# ------------------------------------------------------------------------------------ cfg.episodic (termination head)
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("wl,E", [("tiny", 2), ("c1", 2)])
def test_episodic_plan_matches_oracle(engine, wl, E):
    """Episodic models run the termination head on z_{t+1} inside the fused rollout and carry the sticky
    (1 - termination) factor through the value (tdmpc2.py:126-136).  Values within 5e-5 (absolute); samples whose
    termination logit is within TERM_MARGIN (|logit| < 2e-5: the 0.5 decision is not well defined under ~1e-6 kernel
    error) of the decision boundary are excluded, and an environment stops being compared at the first iteration that
    contains such a sample; top-k, refit, pick and action as in the non-episodic test."""
    from oracle.plan_oracle import balance_termination, draw_noise as oracle_noise, plan_oracle
    cfg = workload(wl, num_envs=E, episodic=True)
    sd = synth_state_dict(cfg, seed=21, perturb=True)
    balance_termination(cfg, sd)
    g = torch.Generator().manual_seed(8)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [bool(i % 2) for i in range(E)]
    noise = oracle_noise(cfg, 44, E)
    want = plan_oracle(cfg, sd, obs, task=None, t0=t0, prev_mean=prev, noise=noise)
    assert 0.02 < float((want.values.abs() > 0).float().mean())             # sanity: not degenerate

    pl = planner_for(cfg, E, engine, sd)
    action, new_mean, tr = pl.plan(obs.cuda().contiguous(), None, torch.tensor(t0, dtype=torch.uint8).cuda(),
                                   prev.cuda().contiguous(), to_gpu_noise(noise), trace=True)
    torch.cuda.synchronize()
    cpu = lambda t: t.detach().cpu()
    n = compare_with_oracle(cfg, tr, action, new_mean, want, noise, range(E), value_atol=5e-5, value_rtol=0, gap=1e-4,
                            keep=want.term_margin > TERM_MARGIN)
    print(wl, engine, n)
    assert n["values"] > 0 and n["topk"] > 0 and n["refit"] > 0, n
    # the termination head really acted: a planner for the same weights without it gives different values
    cfg0 = workload(wl, num_envs=E)
    pl0 = planner_for(cfg0, E, engine, {k: v for k, v in sd.items() if not k.startswith("_termination")})
    _, _, tr0 = pl0.plan(obs.cuda().contiguous(), None, torch.tensor(t0, dtype=torch.uint8).cuda(), prev.cuda().contiguous(),
                         to_gpu_noise(noise), trace=True)
    torch.cuda.synchronize()
    assert float((cpu(tr0["values"][:, 0]) - cpu(tr["values"][:, 0])).abs().max()) > 1e-3


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_episodic_estimate_value_matches_oracle(engine):
    from oracle.plan_oracle import OracleModel, balance_termination, estimate_value
    cfg = workload("tiny", num_envs=2, episodic=True)
    sd = synth_state_dict(cfg, seed=9, perturb=True)
    balance_termination(cfg, sd)
    E, N, H, A, L = 2, cfg.num_samples, cfg.horizon, cfg.action_dim, cfg.latent_dim
    g = torch.Generator().manual_seed(1)
    z = torch.softmax(torch.randn(E, N, L // 8, 8, generator=g), -1).view(E, N, L)
    actions = torch.rand(E, H, N, A, generator=g) * 2 - 1
    eps = torch.randn(E, N, A, generator=g)
    qidx = torch.tensor([[0, 2], [1, 0]])
    model = OracleModel(cfg, sd)
    want, decided = [], []
    for e in range(E):
        info = {}
        want.append(estimate_value(model, z[e], actions[e], None, eps[e], qidx[e], info).squeeze(1))
        decided.append(info["term_margin"] > TERM_MARGIN)
    want, decided = torch.stack(want), torch.stack(decided)
    pl = planner_for(cfg, E, engine, sd)
    got = pl.estimate_value(z.cuda().contiguous(), actions.cuda().contiguous(), None, eps.cuda().contiguous(),
                            qidx.to(torch.int32).cuda().contiguous()).cpu()
    assert decided.float().mean() > 0.99
    assert float((got - want).abs()[decided].max()) < 5e-5
