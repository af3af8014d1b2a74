"""`WorldModel.encode` on batches of pixel frames ([B, C, 64, 64] and [T, B, C, 64, 64], one launch of the persistent
conv-encoder kernel) against fixtures minted from the reference's own encode + _td_target (oracle/wm_rgb_oracle.py),
its ShiftAug draw order, its independence of how frames are spread over CTAs, and its agreement with the planner's
prologue.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from oracle.wm_rgb_oracle import RGB_CASES, load_rgb_case, rgb_case_model
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z_TOL = 1e-5                       # the bar of test_gpu_pixels.py: exact fp32 products, another summation order than ATen's
TD_TOL = (5e-5, 1e-5)              # "value" tolerance of the world-model goldens (test_gpu_world_model.py)


def agent_for(cfg, sd, engine="tcgen05"):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    return agent


def model_for(cfg, sd):
    from tdmpc2_b200.world_model import WorldModel
    m = WorldModel(cfg).to(DEV)
    m.load_state_dict(sd)
    return m


def frames_on_gpu(cfg, R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 256, (R,) + tuple(cfg.obs_shape["rgb"]), generator=g, device=DEV).float()


def shifts_on_gpu(R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 7, (R, 2), generator=g, device=DEV, dtype=torch.float32)


@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
@pytest.mark.parametrize("name", list(RGB_CASES))
def test_encode_and_td_target_match_reference_golden(name, engine):
    cfg, sd, recs = load_rgb_case(name)
    agent = agent_for(cfg, sd, engine)
    for pfx in ("b", "r"):           # [T, B, C, 64, 64] with T draws; one 4-D row
        r = recs[pfx]
        z = agent.model.encode(r["frames"].to(DEV), None, shift=r["shift"].to(DEV))
        assert z.shape == r["z"].shape
        zerr = float((z.cpu() - r["z"]).abs().max())
        assert zerr <= Z_TOL, (pfx, zerr)
        td = agent._td_target(z, r["reward_in"].to(DEV), r["terminated"].to(DEV), None, eps=r["td_eps"].to(DEV),
                              qidx=r["td_qidx"].to(DEV))
        err = (td.cpu() - r["td"]).abs()
        assert td.shape == r["td"].shape
        assert bool((err <= TD_TOL[0] + TD_TOL[1] * r["td"].abs()).all()), (pfx, float(err.max()))
        print(name, engine, pfx, f"|dz|={zerr:.1e} |dtd|={float(err.max()):.1e}")


@pytest.mark.parametrize("lead", [(4,), (3, 4)])
def test_draws_follow_the_reference_order(lead):
    """encode(frames) draws like the reference: one randint (B, 2) per leading slice t, from the agent's generator."""
    cfg, sd = rgb_case_model("tiny_rgb_wm")
    agent = agent_for(cfg, sd)
    frames = frames_on_gpu(cfg, int(torch.tensor(lead).prod()), 5).view(*lead, *cfg.obs_shape["rgb"])
    agent.generator = torch.Generator(device=DEV).manual_seed(77)
    z = agent.model.encode(frames, None)
    state = agent.generator.get_state()
    g = torch.Generator(device=DEV).manual_seed(77)
    B = lead[-1]
    S = torch.stack([torch.randint(0, 7, (B, 2), generator=g, device=DEV, dtype=torch.float32)
                     for _ in range(lead[0] if len(lead) == 2 else 1)]).view(*lead, 2)
    assert torch.equal(z, agent.model.encode(frames, None, shift=S))
    assert torch.equal(state, g.get_state())
    assert z.shape == lead + (cfg.latent_dim,)


def test_row_counts_bit_identical_to_single_frames():
    """Every row of a large call equals encoding its frame alone: the persistent CTAs reuse their smem and conv1 scratch
    slot from frame to frame and stride by the grid width."""
    cfg, sd = rgb_case_model("c1_rgb_wm")
    m = model_for(cfg, sd)
    pl = m._kernels()
    N = 8192
    frames, shift = frames_on_gpu(cfg, N, 11), shifts_on_gpu(N, 12)
    alone = torch.cat([pl.encode_pixel_rows(frames[i:i + 1], shift[i:i + 1]) for i in range(N)])
    for R in (1, 131, 132, 133, 1000, 8192):
        z = m.encode(frames[:R], None, shift=shift[:R])
        bad = (z != alone[:R]).any(-1).nonzero().flatten()
        assert bad.numel() == 0, (R, bad[:8].tolist())


@pytest.mark.parametrize("wl,over,E", [("tiny-rgb", {}, 5), ("c1", {"obs": "rgb", "obs_channels": 9}, 3)])
def test_encode_matches_planner_prologue(wl, over, E):
    """For the same frames and shifts, model.encode equals the z the planner's prologue computes (tdmpc2_pixel_encode)."""
    from tdmpc2_b200.planner import Planner, draw_noise
    cfg = workload(wl, num_envs=E, **over)
    sd = synth_state_dict(cfg, seed=31, perturb=True)
    pl = Planner(cfg, E, DEV)
    pl.pack(sd)
    frames = frames_on_gpu(cfg, E, 13)
    noise = draw_noise(cfg, E, DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    prev = torch.zeros(E, cfg.horizon, cfg.action_dim, device=DEV)
    t0 = torch.ones(E, dtype=torch.uint8, device=DEV)
    _, _, tr = pl.plan(frames, None, t0, prev, noise, trace=True)
    z = model_for(cfg, sd).encode(frames, None, shift=noise.shift)
    assert torch.equal(z, tr["z"])


@pytest.mark.parametrize("over", [{"num_channels": 64, "latent_dim": 1024},   # conv2-4 weights in output-channel chunks
                                  {"obs_channels": 14}])                       # conv1 in input-channel chunks
def test_weight_chunking_matches_oracle(over):
    from oracle.plan_oracle import OracleModel
    cfg = workload("tiny-rgb", **over)
    sd = synth_state_dict(cfg, seed=32, perturb=True)
    R = 140
    frames, shift = frames_on_gpu(cfg, R, 14), shifts_on_gpu(R, 15)
    z = model_for(cfg, sd).encode(frames, None, shift=shift).cpu()
    want = OracleModel(cfg, sd).encode_rgb(frames.cpu(), shift.cpu())
    err = float((z - want).abs().max())
    assert err <= Z_TOL, err


def test_errors_and_uint8_frames():
    cfg, sd = rgb_case_model("tiny_rgb_wm")
    m = model_for(cfg, sd)
    C = cfg.obs_shape["rgb"][0]
    for bad in (torch.zeros(C, 64, 64), torch.zeros(2, 2, 2, C, 64, 64), torch.zeros(2, C + 1, 64, 64),
                torch.zeros(2, C, 32, 32)):
        with pytest.raises(ValueError):
            m.encode(bad.to(DEV), None)
    with pytest.raises(ValueError):
        m.encode(torch.zeros(2, C, 64, 64, device=DEV), None, shift=torch.zeros(3, 2, device=DEV))
    frames, shift = frames_on_gpu(cfg, 6, 16).view(2, 3, C, 64, 64), shifts_on_gpu(6, 17).view(2, 3, 2)
    assert torch.equal(m.encode(frames.to(torch.uint8), None, shift=shift), m.encode(frames, None, shift=shift))
    assert torch.equal(m.encode(frames.to(torch.uint8).cpu(), None, shift=shift.cpu()), m.encode(frames, None, shift=shift))
