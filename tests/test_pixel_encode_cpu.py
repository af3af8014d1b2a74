"""Pixel-model `encode` on batches of frames without a GPU: the oracle against fixtures minted from the reference's own
`WorldModel.encode` on [T, B, C, 64, 64] frames followed by `_td_target` (oracle/wm_rgb_oracle.py), ShiftAug's
draw order, and the C entry point's no-device failure."""
import pytest
import torch

from oracle.wm_oracle import WMOracle
from oracle.wm_rgb_oracle import RGB_CASES, load_rgb_case

ORACLE_TOL = 7e-7          # relative above |v| = 1, as for the state-model fixtures (test_world_model_cpu.py)


@pytest.mark.parametrize("name", list(RGB_CASES))
@pytest.mark.parametrize("batch", ["b", "r"])
def test_oracle_matches_reference_pixel_encode(name, batch):
    cfg, sd, recs = load_rgb_case(name)
    r = recs[batch]
    o = WMOracle(cfg, sd)
    frames = r["frames"]
    lead = frames.shape[:-3]
    assert r["shift"].shape == lead + (2,)
    z = o.encode_rgb(frames.reshape(-1, *frames.shape[-3:]), r["shift"].reshape(-1, 2)).view(*lead, -1)
    # the same ATen convolutions on the same fp32 inputs: bit-identical
    assert torch.equal(z, r["z"])
    td = o.td_target(r["z"], r["reward_in"], r["terminated"], None, r["td_eps"], r["td_qidx"])
    assert td.shape == r["td"].shape
    assert float(((td - r["td"]).abs() / r["td"].abs().clamp(min=1.0)).max()) <= ORACLE_TOL


@pytest.mark.parametrize("name", list(RGB_CASES))
def test_draw_helper_reproduces_shiftaug_draws(name):
    """draw_shifts seeded like the mint gives the reference's ShiftAug draws: T successive (B, 2) draws for a 5-D batch,
    one draw for a 4-D one."""
    from tdmpc2_b200.planner import draw_shifts
    cfg, sd, recs = load_rgb_case(name)
    seed = RGB_CASES[name][-1]
    for batch, s in (("b", seed), ("r", seed + 1)):
        want = recs[batch]["shift"]
        got = draw_shifts(tuple(want.shape[:-1]), "cpu", torch.Generator().manual_seed(s))
        assert torch.equal(got, want), batch


def test_single_pixel_encode_call_exported():
    from tdmpc2_b200 import build, _cabi
    build.build()
    lib = _cabi.load()
    assert "tdmpc2_pixel_encode" in _cabi.SYMBOLS and hasattr(lib, "tdmpc2_pixel_encode")
    for old in ("tdmpc2_pixel_encode_rows", "tdmpc2_pixel_encode_taped"):     # ABI 8 merged them into tdmpc2_pixel_encode
        assert old not in _cabi.SYMBOLS and not hasattr(lib, old), old
    assert lib.tdmpc2_abi_version() == _cabi.ABI_VERSION == 9


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_single_pixel_encode_call_needs_a_device():
    from tdmpc2_b200 import build, _cabi
    build.build()
    lib = _cabi.load()
    assert lib.tdmpc2_pixel_encode(None, None, None, None, None, None, 1, None, None, None) == -2   # TDMPC2_ERR_NO_DEVICE
    assert b"no CUDA device" in lib.tdmpc2_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_pixel_world_model_encode_has_no_cpu_fallback():
    """The device check comes before the shape check: a CPU model raises NotImplementedError for any input."""
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.world_model import WorldModel
    m = WorldModel(workload("tiny-rgb"))
    for x in (torch.zeros(2, 6, 64, 64), torch.zeros(3, 2, 6, 64, 64), torch.zeros(6, 64, 64)):
        with pytest.raises(NotImplementedError, match="no CPU fallback"):
            m.encode(x, None)
