"""Parity in the regime bench.py times: more tiles than persistent CTAs, so that every CTA runs SEVERAL trips of the tile
loop -- mbarrier phases / pipeline counters carried across tiles, operand smem reused as refit scratch between tiles,
the cross-CTA "last tile of this environment" hand-off with tiles of one environment finishing in different trips, CTAs
desynchronised by refits.  Checked two ways:

  * bit-identity: a row's arithmetic does not depend on which CTA / trip / batch it runs in, so every environment of a
    big batch must reproduce, bit for bit, a 2-environment run of the same inputs and noise (single trip);
  * the CPU oracle on sampled environments of the big batch (same tolerances as tests/test_gpu_parity.py).

Also: the c5 planner shape (N=1024, H=8, I=10 -> 8 tiles per environment, 57 layer steps per tile) on a 5M-sized model,
and the 48M / 317M presets (wide layers) at E > 1.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import mixed_noise, slice_noise, compare_with_oracle

pytestmark = pytest.mark.gpu


def _planner(cfg, E, engine, sd):
    from tdmpc2_b200.planner import Planner
    pl = Planner(cfg, E, "cuda:0", engine=engine)
    pl.pack(sd)
    return pl


def _inputs(cfg, E, seed):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = torch.tensor([int(i % 3 == 0) for i in range(E)], dtype=torch.uint8)
    task = (torch.arange(E) * 7 + 3) % len(cfg.tasks) if cfg.multitask else None
    return obs, prev, t0, task


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _two_plans(pl, obs, task, t0, prev, nz_a, nz_b):
    """plan() twice: the second call is warm-started from the first one's mean (pipeline counters mid-stream)."""
    dev = "cuda"
    taskv = None if task is None else task.to(torch.int32).to(dev)
    a1, m1, tr1 = pl.plan(obs.to(dev), taskv, t0.to(dev), prev.to(dev), nz_a, trace=True)
    a2, m2, tr2 = pl.plan(obs.to(dev), taskv, torch.zeros_like(t0).to(dev), m1, nz_b, trace=True)
    torch.cuda.synchronize()
    return (a1, m1, tr1), (a2, m2, tr2)


@pytest.mark.parametrize("engine", ["tcgen05", "simt"])
@pytest.mark.parametrize("E", [64, 256])
def test_many_trip_batch_is_bit_identical_to_small_runs_and_matches_oracle(E, engine):
    """c1 model (the bench's 5M dog-run net) on the tensor-core engine (the default) and on the CUDA-core engine:
    E=64 -> 256 tiles (1.9 trips/CTA on 132 SMs), E=256 -> 1024 tiles (7.8 trips/CTA; exactly bench.py's c2 schedule)."""
    from oracle.plan_oracle import plan_oracle
    cfg = workload("c1", num_envs=E)
    assert E * ((cfg.num_samples + 127) // 128) > _num_sms()
    sd = synth_state_dict(cfg, seed=7, perturb=True)
    obs, prev, t0, task = _inputs(cfg, E, 31)
    oracle_envs = [0, E // 3, E // 2 + 1, E - 1]
    nz_a, on_a = mixed_noise(cfg, E, oracle_envs, 100)
    nz_b, on_b = mixed_noise(cfg, E, oracle_envs, 200)
    pl = _planner(cfg, E, engine, sd)
    big1, big2 = _two_plans(pl, obs, task, t0, prev, nz_a, nz_b)
    del pl
    # ---- bit-identity against single-trip 2-environment runs of the same environments
    pairs = [(0, 1), (E // 3, E // 3 + 1), (E // 2, E // 2 + 1), (E - 2, E - 1), (E // 5, E - 7)]
    for envs in pairs:
        idx = list(envs)
        cfg2 = workload("c1", num_envs=2)
        pl2 = _planner(cfg2, 2, engine, sd)
        small1, small2 = _two_plans(pl2, obs[idx], None, t0[idx], prev[idx], slice_noise(nz_a, idx), slice_noise(nz_b, idx))
        for big, small, which in ((big1, small1, "first"), (big2, small2, "warm-started")):
            (ab, mb, trb), (as_, ms, trs) = big, small
            for name, x, y in (("action", ab[idx], as_), ("mean", mb[idx], ms), ("values", trb["values"][idx], trs["values"]),
                               ("elite_idx", trb["elite_idx"][idx], trs["elite_idx"]), ("iter_mean", trb["iter_mean"][idx], trs["iter_mean"]),
                               ("iter_std", trb["iter_std"][idx], trs["iter_std"]), ("pick", trb["pick"][idx], trs["pick"])):
                assert torch.equal(x.cpu(), y.cpu()), f"E={E} envs={envs} {which} plan: {name} differs from the 2-env run"
        del pl2
    # ---- the oracle on sampled environments of the big batch (first plan, and the warm-started second one)
    sel = torch.tensor(oracle_envs)
    want1 = plan_oracle(cfg, sd, obs[sel], t0=[bool(t0[e]) for e in oracle_envs], prev_mean=prev[sel], noise=on_a)
    n1 = compare_with_oracle(cfg, big1[2], big1[0], big1[1], want1, on_a, oracle_envs)
    # second plan: warm start from the KERNEL's first-plan mean (the oracle's is within 1e-4 of it where compared)
    want2 = plan_oracle(cfg, sd, obs[sel], t0=[False] * len(oracle_envs), prev_mean=big1[1][sel].cpu(), noise=on_b)
    n2 = compare_with_oracle(cfg, big2[2], big2[0], big2[1], want2, on_b, oracle_envs)
    for n in (n1, n2):
        assert n["topk"] > 0 and n["refit"] > 0, n
    print(f"[multitrip E={E}] first {n1} second {n2}")


def test_c5_planner_shape_on_5m_model():
    """N=1024, H=8, I=10 (BASELINE config c5's planner shape): 8 tiles per environment, 57 layer steps per tile, 20
    environments -> 160 tiles > 132 CTAs.  Tensor-core engine vs the oracle on 2 environments, and its first-iteration
    trajectory values within the parity tolerance of the CUDA-core engine on all of them (the first iteration's inputs do
    not depend on either engine's refit)."""
    from oracle.plan_oracle import plan_oracle
    E = 20
    cfg = workload("c1", num_envs=E, num_samples=1024, horizon=8, iterations=10)
    assert E * 8 > _num_sms()
    sd = synth_state_dict(cfg, seed=8, perturb=True)
    obs, prev, t0, task = _inputs(cfg, E, 32)
    oracle_envs = [3, E - 1]
    nz, on = mixed_noise(cfg, E, oracle_envs, 300)
    out = {}
    for engine in ("simt", "tcgen05"):
        pl = _planner(cfg, E, engine, sd)
        a, m, tr = pl.plan(obs.cuda(), None, t0.cuda(), prev.cuda(), nz, trace=True)
        torch.cuda.synchronize()
        out[engine] = (a, m, tr)
        del pl
    v_tc, v_simt = out["tcgen05"][2]["values"][:, 0].cpu(), out["simt"][2]["values"][:, 0].cpu()
    assert torch.allclose(v_tc, v_simt, atol=5e-5, rtol=1e-5), (v_tc - v_simt).abs().max()
    sel = torch.tensor(oracle_envs)
    want = plan_oracle(cfg, sd, obs[sel], t0=[bool(t0[e]) for e in oracle_envs], prev_mean=prev[sel], noise=on)
    a, m, tr = out["tcgen05"]
    n = compare_with_oracle(cfg, tr, a, m, want, on, oracle_envs)
    assert n["topk"] > 0 and n["refit"] > 0, n
    print(f"[c5-shape] {n}")


# The wide presets keep the tolerance of every other parity test (values: 5e-5 + 1e-5 |v|; their values reach 8 / 17).
# What makes that possible on tensor cores: the tensor core's internal accumulation is not round-to-nearest, a drift that
# would grow with the reduction length (K = 1792 / 4096 here); every 64-element K-chunk's partial sum is therefore added
# in fp32 with round-to-nearest (gemm_tc in plan_kernels.cuh).
@pytest.mark.parametrize("wl", ["c3", "c4"])
def test_wide_presets_multi_env(wl):
    """humanoid-walk 48M (M=1792) and mt80 317M (M=4096, multi-task) at E=3: 12 tiles on the wide-layer path, one
    environment checked against the oracle (the oracle needs 0.6 / 2.2 TFLOP per environment on the host)."""
    from oracle.plan_oracle import plan_oracle
    E = 3
    cfg = workload(wl, num_envs=E)
    sd = synth_state_dict(cfg, seed=9)
    obs, prev, t0, task = _inputs(cfg, E, 33)
    oracle_envs = [1]
    nz, on = mixed_noise(cfg, E, oracle_envs, 400)
    pl = _planner(cfg, E, None, sd)
    taskv = None if task is None else task.to(torch.int32).cuda()
    a, m, tr = pl.plan(obs.cuda(), taskv, t0.cuda(), prev.cuda(), nz, trace=True)
    torch.cuda.synchronize()
    sel = torch.tensor(oracle_envs)
    want = plan_oracle(cfg, sd, obs[sel], task=None if task is None else [int(task[e]) for e in oracle_envs],
                       t0=[bool(t0[e]) for e in oracle_envs], prev_mean=prev[sel], noise=on)
    n = compare_with_oracle(cfg, tr, a, m, want, on, oracle_envs)
    assert n["topk"] > 0 and n["refit"] > 0, f"{wl}: nothing beyond the values was compared: {n}"
    print(f"[{wl} E=3] {n}")
    if cfg.multitask:
        for e in range(E):
            adim = cfg.action_dims[int(task[e])]
            assert torch.all(a[e, adim:] == 0) and torch.all(m[e, :, adim:] == 0)
