"""The DECLARED NON-PARITY fast mode (tdmpc2_planner_set_passes(p, 1): one fp16 MMA per product instead of the three of
the fp32-parity path).  It is not held to the oracle's 5e-5: these tests pin down what it IS -- the same plan with
fp16-rounded operands (values within ~1e-2 of the oracle, far outside 5e-5, elite sets mostly but not exactly the
reference's) -- and that switching it on does not disturb the parity mode.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import planner_for, to_gpu_noise

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("wl,engine", [("c1", "tcgen05"), ("tiny-mt", "tcgen05"), ("tiny-wide", "tcgen05")])
def test_fast_mode_is_close_to_but_not_at_parity(wl, engine):
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    E = 2
    cfg = workload(wl, num_envs=E)
    sd = synth_state_dict(cfg, seed=13, perturb=True)
    g = torch.Generator().manual_seed(6)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0, task = [True, False], ([1, 3] if cfg.multitask else None)
    on = oracle_noise(cfg, 50, E)
    want = plan_oracle(cfg, sd, obs, task=task, t0=t0, prev_mean=prev, noise=on)
    noise = to_gpu_noise(on)
    taskv = None if task is None else torch.tensor(task, dtype=torch.int32).cuda()
    got = {}
    for passes in (3, 1, 3):                                   # parity, fast, parity again (the knob leaves no state behind)
        pl = planner_for(cfg.replace(passes=passes), E, engine, sd)
        assert pl.passes == passes
        _, _, tr = pl.plan(obs.cuda(), taskv, torch.tensor(t0, dtype=torch.uint8).cuda(), prev.cuda(), noise, trace=True)
        torch.cuda.synchronize()
        got.setdefault(passes, []).append((tr["values"][:, 0].cpu(), tr["elite_idx"][:, 0].cpu()))
    v3, v1 = got[3][0][0], got[1][0][0]
    assert torch.equal(v3, got[3][1][0])                       # parity mode is bit-reproducible around a fast-mode planner
    assert torch.allclose(v3, want.values[:, 0], atol=5e-5, rtol=1e-5)
    err1 = (v1 - want.values[:, 0]).abs().max().item()
    assert 5e-5 < err1 < 5e-2, err1                            # fp16 operands: visible, bounded
    K = cfg.num_elites
    same = sum(len(set(got[1][0][1][e].tolist()) & set(want.elite_idx[e, 0].tolist())) for e in range(E)) / (E * K)
    assert same > 0.5, same                                    # still the same search, not the same elites


def test_set_passes_rejects_other_values():
    from tdmpc2_b200 import _cabi
    from tdmpc2_b200.planner import Planner
    cfg = workload("tiny", num_envs=1)
    pl = Planner(cfg, 1, "cuda:0")
    with pytest.raises(_cabi.CabiError):
        _cabi.check(pl.lib.tdmpc2_planner_set_passes(pl.h, 2))
