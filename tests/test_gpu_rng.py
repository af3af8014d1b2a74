"""The DECLARED NON-PARITY throughput mode with in-kernel noise (tdmpc2_plan_iter_rng, csrc/rng.cuh): the generator's
statistics, and that every consumer of an element -- the per-step action pass and the MPPI refit that re-derives the elites'
actions -- regenerates the same value (the refit mean recomputed on the host from the dumped stream must match the kernel's).
There is no oracle comparison: the oracle consumes torch's draws.  Run on an H100: pytest -m gpu."""
import ctypes as C

import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict

pytestmark = pytest.mark.gpu


def _dump(lib, state, stream, group0, ngroups):
    out = torch.empty(4 * ngroups, device="cuda", dtype=torch.float32)
    from tdmpc2_b200 import _cabi
    _cabi.check(lib.tdmpc2_debug_rng(state.data_ptr(), stream, group0, ngroups, out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu()


def test_generator_statistics_and_determinism():
    from tdmpc2_b200 import _cabi
    lib = _cabi.load()
    st = torch.tensor([1234567, 3], dtype=torch.int64, device="cuda")
    n = 1 << 20
    x = _dump(lib, st, 4, 0, n // 4)
    assert torch.isfinite(x).all()
    assert abs(float(x.mean())) < 5.0 / n ** 0.5 and abs(float(x.var()) - 1.0) < 0.01
    assert abs(float((x ** 4).mean()) - 3.0) < 0.05 and abs(float((x ** 3).mean())) < 0.02       # kurtosis, skewness
    assert abs(float((x[:-1] * x[1:]).mean())) < 0.005                                             # lag-1 correlation
    assert float(x.abs().max()) > 4.0                                                              # tails are there
    assert torch.equal(x, _dump(lib, st, 4, 0, n // 4))                                            # deterministic
    assert torch.equal(x[4 * 1000:4 * 1010], _dump(lib, st, 4, 1000, 10))                          # random access by group
    for other in (torch.tensor([1234567, 4]), torch.tensor([1234568, 3])):                         # plan counter / seed
        y = _dump(lib, other.to(torch.int64).cuda(), 4, 0, n // 4)
        assert abs(float((x * y).mean())) < 0.005
    assert abs(float((x * _dump(lib, st, 5, 0, n // 4)).mean())) < 0.005                           # another stream


@pytest.mark.parametrize("wl,engine", [("c1", "tcgen05pp"), ("c1", "tcgen05x2"), ("tiny-mt", "tcgen05x2"), ("tiny-wide", "tcgen05x2")])
def test_in_kernel_noise_is_consistent_between_action_pass_and_refit(wl, engine):
    from tdmpc2_b200.planner import Planner, draw_noise
    E = 2
    cfg = workload(wl, num_envs=E, rng="philox", rng_seed=99)
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    H, N, P, A, K = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.num_elites
    g = torch.Generator().manual_seed(3)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g).cuda()
    prev = torch.zeros(E, H, A).cuda()
    t0 = torch.ones(E, dtype=torch.uint8).cuda()
    task = torch.tensor([1, 2], dtype=torch.int32).cuda() if cfg.multitask else None
    runs = []
    for rep in range(2):
        pl = Planner(cfg, E, "cuda:0", engine=engine)
        assert pl.philox and pl.rng_state is not None
        pl.pack(sd)
        noise = draw_noise(cfg, E, "cuda", generator=torch.Generator(device="cuda").manual_seed(7))
        assert noise.r is None and noise.pi is None                       # nothing large is drawn or stored
        action, new_mean, tr = pl.plan(obs, task, t0, prev, noise, trace=True)
        torch.cuda.synchronize()
        runs.append((action.cpu(), tr["values"].cpu(), tr["elite_idx"].cpu(), tr["iter_mean"].cpu(), tr["pi_actions"].cpu(),
                     pl.rng_state.clone()))
        assert int(pl.rng_state[1]) == 1
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][0], runs[1][0])      # same seed, same counter: same plan
    action, values, elite_idx, iter_mean, pi_actions, state = runs[0]
    assert torch.isfinite(values).all() and bool((action.abs() <= 1).all())
    # ---- first iteration recomputed on the host from the dumped stream (stream 0 = noise_r of iteration 0)
    A4 = (A + 3) // 4
    x = _dump(pl.lib, state, 0, 0, E * H * N * A4).view(E, H, N, A4 * 4)[..., :A]
    mask = torch.ones(E, 1, 1, A)
    if cfg.multitask:
        mask = sd["_action_masks"][task.cpu().long()].view(E, 1, 1, A)
    acts = (cfg.max_std * x).clamp(-1, 1)                                 # t0: mean 0, std max_std (tdmpc2.py:164-165,176-179)
    acts[:, :, :P] = pi_actions
    acts = acts * mask
    for e in range(E):
        idx = elite_idx[e, 0]
        ev = values[e, 0][idx]
        score = torch.exp(cfg.temperature * (ev - ev.max()))
        score = score / score.sum()
        mean = (score.view(1, K, 1) * acts[e][:, idx]).sum(1) / (score.sum() + 1e-9)
        assert torch.allclose(iter_mean[e, 0], mean, atol=2e-5, rtol=0), (iter_mean[e, 0] - mean).abs().max()
    # a second plan() draws a fresh stream
    a2, _, tr2 = pl.plan(obs, task, t0, prev, noise, trace=True)
    torch.cuda.synchronize()
    assert int(pl.rng_state[1]) == 2 and not torch.equal(tr2["values"].cpu(), values)
