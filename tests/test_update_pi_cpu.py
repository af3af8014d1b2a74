"""agent.update_pi without a GPU: the oracle against fixtures minted from the reference's own update_pi, RunningScale
against the reference module, the training keys' defaults, and the CPU refusal."""
import os
import subprocess
import sys

import pytest
import torch

from oracle.pi_oracle import CASES, PI_KEYS, load_case, update_pi_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def close(got, want, rtol, atol_frac):
    """|got - want| <= rtol |want| + atol_frac max|want| (fp32 rounding of sums over rows and columns)"""
    got, want = got.double(), want.double()
    assert got.shape == want.shape
    tol = rtol * want.abs() + atol_frac * float(want.abs().max()) + 1e-30
    assert bool(((got - want).abs() <= tol).all()), float((got - want).abs().max())


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_fixture(name):
    cfg, sd, x, want = load_case(name)
    r = update_pi_oracle(cfg, sd, x["zs"], x["task"], x["eps"], x["qidx"], x["drop"], x["scale0"])
    close(r["loss"].reshape(1), want["loss"].reshape(1), 1e-5, 0)
    close(r["scale"], want["scale_after"], 1e-6, 0)
    close(r["grad_norm"].reshape(1), want["grad_norm"].reshape(1), 1e-4, 0)
    close(r["entropy"], want["entropy"], 1e-5, 1e-6)
    close(r["scaled_entropy"], want["scaled_entropy"], 1e-5, 1e-6)
    for k in PI_KEYS + (["_task_emb.weight"] if cfg.multitask else []):
        w = want["grad/" + k]
        close(r["grads"][k][:w.shape[0]], w, 1e-3, 1e-4)
    for k in PI_KEYS:
        w = want["param/" + k]
        close(r["params"][k][:w.shape[0]], w, 0, 1e-6)


def _reference_scale_cls():
    from oracle import ref_harness as rh
    if not rh.available():
        pytest.skip("reference modules not available")
    rh._import_reference()
    sys.path.insert(0, rh.REF_DIR)
    try:
        from common.scale import RunningScale
    finally:
        sys.path.remove(rh.REF_DIR)
    return RunningScale


@pytest.mark.parametrize("kind", ["random", "tied", "small"])
def test_running_scale_matches_reference(kind):
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.scale import RunningScale
    Ref = _reference_scale_cls()
    cfg = workload("tiny")
    ref = Ref.__new__(Ref)                      # its __init__ places the buffers on cuda:0
    torch.nn.Module.__init__(ref)
    ref.cfg = cfg
    ref.value = torch.nn.Buffer(torch.ones(1))
    ref._percentiles = torch.nn.Buffer(torch.tensor([5, 95], dtype=torch.float32))
    ours = RunningScale(cfg, "cpu")
    g = torch.Generator().manual_seed(3)
    for i in range(5):
        if kind == "random":
            x = torch.randn(256, 1, generator=g) * 10 ** i
        elif kind == "tied":
            x = torch.full((64, 1), 3.0)
            x[::7] = -2.0
        else:
            x = torch.randn(7, 1, generator=g) * 0.1
        ref.update(x)
        ours.update(x)
        assert torch.equal(ours.value, ref.value)
        assert torch.equal(ours(x), ref(x))
    assert set(ours.state_dict()) == {"value", "percentiles"}


def test_training_config_defaults():
    from tdmpc2_b200.config import make_cfg
    cfg = make_cfg(obs_dim=4, action_dim=2)
    assert (cfg.rho, cfg.grad_clip_norm, cfg.lr, cfg.tau, cfg.entropy_coef, cfg.dropout) == (0.5, 20, 3e-4, 0.01, 1e-4, 0.01)


def test_update_pi_refuses_cpu_before_shape_checks():
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(workload("tiny"), device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        agent.update_pi(torch.zeros(1), None)        # a wrong shape: the device is reported first


def test_product_does_not_import_oracle():
    code = ("import sys; import tdmpc2_b200.tdmpc2, tdmpc2_b200.scale; "
            "assert not [m for m in sys.modules if m.startswith('oracle')], 'oracle imported'")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)
