"""Pixel observations (cfg.obs == 'rgb'): the conv encoder kernel (ShiftAug + PixelPreprocess + 4 x Conv2d + SimNorm,
reference common/layers.py:36-71,136-150) and the planner behind it, against the CPU oracle, whose pixel path is pinned to
a fixture minted from the reference's own `_plan` on pixel observations (tests/golden/tiny_rgb.npz; the full-plan golden
comparison is tests/test_gpu_golden.py::tiny_rgb).  Run on an H100: pytest -m gpu."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import compare_with_oracle, planner_for, to_gpu_noise

pytestmark = pytest.mark.gpu


def _frames(cfg, E, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (E,) + tuple(cfg.obs_shape["rgb"]), generator=g).float()


@pytest.mark.parametrize("E", [1, 5])
def test_encode_pixel_rows_matches_oracle(E):
    """z = encode(frames) for every shift pair the reference can draw on some environment: 1e-5 (the convolutions are exact
    fp32 products summed in a different order than ATen's; SimNorm outputs are <= 1)."""
    from oracle.plan_oracle import OracleModel
    cfg = workload("tiny-rgb", num_envs=E)
    sd = synth_state_dict(cfg, seed=14, perturb=True)
    frames = _frames(cfg, E, 3)
    shift = torch.tensor([[(3 * e) % 7, (5 * e + 6) % 7] for e in range(E)], dtype=torch.float32)
    want = OracleModel(cfg, sd).encode_rgb(frames, shift)
    pl = planner_for(cfg, E, None, sd)
    got = pl.encode_pixel_rows(frames.cuda(), shift.cuda(), out=pl.pix_z).cpu()
    torch.cuda.synchronize()
    assert got.shape == (E, cfg.latent_dim)
    assert torch.allclose(got, want, atol=1e-5, rtol=0), (got - want).abs().max()
    assert torch.allclose(got.view(E, -1, cfg.simnorm_dim).sum(-1), torch.ones(E, cfg.latent_dim // cfg.simnorm_dim), atol=1e-5)


def test_pixel_plan_matches_oracle_and_act_shapes():
    """Full plan() on pixel observations, E = 2, explicit noise (ShiftAug's draw included) vs the oracle; then the
    reference's call shape act(obs[C, 64, 64] on the host) -> action[A] on the host through the CUDA-graph path."""
    from oracle.plan_oracle import draw_noise as oracle_noise, plan_oracle
    from tdmpc2_b200.tdmpc2 import TDMPC2
    E = 2
    cfg = workload("tiny-rgb", num_envs=E)
    sd = synth_state_dict(cfg, seed=15, perturb=True)
    frames = _frames(cfg, E, 4)
    g = torch.Generator().manual_seed(9)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    t0 = [True, False]
    on = oracle_noise(cfg, 70, E)
    want = plan_oracle(cfg, sd, frames, t0=t0, prev_mean=prev, noise=on)
    pl = planner_for(cfg, E, None, sd)
    action, new_mean, tr = pl.plan(frames.cuda(), None, torch.tensor(t0, dtype=torch.uint8).cuda(), prev.cuda(),
                                   to_gpu_noise(on), trace=True)
    torch.cuda.synchronize()
    assert torch.allclose(tr["z"].cpu(), want.z, atol=1e-5, rtol=0)
    n = compare_with_oracle(cfg, tr, action, new_mean, want, on, range(E))
    print(n)
    assert n["topk"] > 0 and n["values"] > 0, n
    # reference-shaped agent: one environment, host observation in, host action out (graph replay from the 2nd call)
    cfg1 = workload("tiny-rgb", num_envs=1)
    agent = TDMPC2(cfg1, device="cuda:0")
    agent.load(sd)
    for i in range(3):
        a = agent.act(frames[0], t0=(i == 0))
        assert a.device.type == "cpu" and a.shape == (cfg1.action_dim,) and bool((a.abs() <= 1).all())
    a_eval = agent.act(frames[0].to(torch.uint8), eval_mode=True)          # uint8 frames as the env wrappers deliver them
    assert a_eval.shape == (cfg1.action_dim,)
