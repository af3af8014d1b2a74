"""agent._update of pixel models without a GPU: the oracle (conv encoder under autograd) against fixtures minted from the
reference's own _update, the fp32 oracle against float64, and the order of ShiftAug's draws in the reference."""
import pytest
import torch
import torch.nn.functional as F

from oracle.update_rgb_oracle import RGB_CASES, RGB_MULTI_STEP, case_inputs, case_model, load_case, run_case
from rgb_update_checks import check_state_rgb, fixture_info
from update_checks import check_info

FIXTURES = list(RGB_CASES) + list(RGB_MULTI_STEP)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_reference_fixture(name):
    base, steps = RGB_MULTI_STEP.get(name, (name, 1))
    cfg, sd, _, want = load_case(name)
    _, _, out = run_case(base, steps=steps)
    for s, (x, r) in enumerate(out):
        check_info(fixture_info(cfg, r, x), want, "info/" if s == 0 else f"info{s}/", rel=1e-5, gn_rel=1e-5)
    r = out[-1][1]
    assert sum(k.startswith("_encoder.rgb.") for k in r["grads"]) == 8
    # after one step the conv biases already differ by Adam-amplified rounding (rgb_update_checks), which moves the next
    # step's gradients by a few 1e-5 of their maximum
    zero = check_state_rgb(r["grads"], lambda k: r["sd"][k], r["emb_grad"], want, grad_rel=1e-5 if steps == 1 else 1e-4,
                           param_abs=1e-6)
    assert zero <= {"grad/_encoder.rgb.8.bias"}, zero


@pytest.mark.parametrize("name", list(RGB_CASES))
def test_oracle_fp32_against_float64(name):
    """The fp32 oracle's losses and gradients, conv gradients included, sit within fp32 error of float64."""
    _, _, o32 = run_case(name)
    _, _, o64 = run_case(name, dtype=torch.float64)
    a, b = o32[0][1], o64[0][1]
    for k in ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss", "grad_norm"):
        assert abs(float(a[k]) - float(b[k])) <= 1e-4 * abs(float(b[k])) + 1e-6, k
    conv = max(float(w.abs().max()) for k, w in b["grads"].items() if k.startswith("_encoder.rgb."))
    for k, w in b["grads"].items():
        bar = 1e-3 * conv if k == "_encoder.rgb.8.bias" else 1e-3 * float(w.abs().max()) + 1e-9   # zero up to rounding
        assert float((a["grads"][k].double() - w).abs().max()) <= bar, k


def test_reference_shift_draw_order():
    """The reference's _update makes H + 1 ShiftAug draws: one per obs[1 + t] in order of t (the no-grad targets), then
    obs[0]'s (the latent rollout), which is the order `shift` and the agent's own draws follow."""
    from oracle import ref_harness as rh
    from oracle.update_rgb_oracle import reference_update_rgb
    if not rh.available():
        pytest.skip("reference modules not available")
    name = "tiny_rgb_episodic_update"
    cfg, sd = case_model(name)
    x = case_inputs(cfg, name)
    H = x["action"].shape[0]
    seen = []
    real = F.grid_sample

    def spy(inp, grid, *a, **k):                 # ShiftAug samples right after its randint draw (layers.py:55-59)
        seen.append(inp[:, :, 3:-3, 3:-3].detach().clone())
        return real(inp, grid, *a, **k)
    F.grid_sample = spy
    try:
        reference_update_rgb(cfg, sd, [x])           # asserts that all H + 1 recorded shifts were drawn
    finally:
        F.grid_sample = real
    assert len(seen) == H + 1
    order = list(range(1, H + 1)) + [0]
    for got, t in zip(seen, order):
        assert torch.equal(got, x["obs"][t].float()), t
