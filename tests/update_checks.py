"""Comparison of one agent._update (or the oracle's) with a fixture minted from the reference's own _update
(oracle/update_oracle.py) -- shared by tests/test_update_cpu.py and tests/test_gpu_update.py."""
import torch

from oracle.update_oracle import MULTI_STEP, SUB_NUMEL

LOSSES = ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss")
PI_INFO = ("pi_loss", "pi_grad_norm", "pi_entropy", "pi_scaled_entropy", "pi_scale")


def steps_of(name):
    return MULTI_STEP.get(name, (name, 1))


def check_info(info, want, prefix, rel, gn_rel):
    """The info dict of one step (values reduced with .mean() like the reference's)."""
    for k in LOSSES + ("pi_loss", "pi_entropy", "pi_scaled_entropy", "pi_scale"):
        w = float(want[prefix + k])
        assert abs(float(info[k]) - w) <= rel * abs(w) + 1e-6, (prefix + k, float(info[k]), w)
    for k in ("grad_norm", "pi_grad_norm"):
        w = float(want[prefix + k])
        assert abs(float(info[k]) - w) <= gn_rel * w, (prefix + k, float(info[k]), w)
    if prefix + "termination_rate" in want:
        assert float(info["termination_rate"]) == float(want[prefix + "termination_rate"])
        assert abs(float(info["termination_f1"]) - float(want[prefix + "termination_f1"])) <= 1e-5


def check_state(grads, params, emb_grad, want, grad_rel, param_abs):
    """Gradients before clipping (the recorded leading elements of every tensor), the state after the step (target Q
    included) and the embedding gradient update_pi leaves."""
    gk = {k[len("grad/"):] for k in want if k.startswith("grad/")}
    assert gk == set(grads), gk ^ set(grads)
    for k in gk:
        w = want["grad/" + k].double()
        g = grads[k].detach().reshape(-1)[:SUB_NUMEL].double().cpu()
        assert float((g - w).abs().max()) <= grad_rel * float(w.abs().max()) + 1e-12, k
    for k in (k[len("param/"):] for k in want if k.startswith("param/")):
        w = want["param/" + k].double()
        got = params(k).detach().reshape(-1)[:SUB_NUMEL].double().cpu()
        assert float((got - w).abs().max()) <= param_abs, k
    if "emb_grad_after" in want:
        w = want["emb_grad_after"].double()
        assert float((emb_grad.detach().double().cpu() - w).abs().max()) <= grad_rel * float(w.abs().max()), "emb grad"
