"""Comparison of a pixel model's _update with a fixture: update_checks.check_state, except for gradients that are zero up
to rounding.  conv4's bias is one: SimNorm's groups (simnorm_dim = 8 consecutive values of the flattened [nc][4][4] map)
each lie inside one output channel, and softmax ignores a constant added to a group, so dL/db4 = 0 exactly; what the
reference records is rounding noise.  Those tensors are held to an absolute bar, `grad_rel` of the largest conv
gradient.  Other conv elements can have a true gradient near zero too (cancelling ReLU and SimNorm paths); Adam moves an
element by lr |g| / (|g| + eps), so where |g| is below eps = 1e-8 the step depends on its rounding.  The conv parameters
after the step are therefore held to `conv_param_abs`, set well below one Adam step of the encoder group
(lr * enc_lr_scale = 9e-5), so that a gradient of the wrong sign still fails."""
import torch

from oracle.update_oracle import SUB_NUMEL
from update_checks import check_state


def check_state_rgb(grads, params, emb_grad, want, grad_rel, param_abs, conv_param_abs=1e-5):
    conv = [float(want[k].abs().max()) for k in want if k.startswith("grad/_encoder.rgb.")]
    floor = grad_rel * max(conv)
    zero = {k for k in want if k.startswith("grad/") and float(want[k].abs().max()) < 1e-5 * max(conv)}
    for k in zero:
        g = grads[k[len("grad/"):]].detach().reshape(-1)[:SUB_NUMEL].double().cpu()
        assert float((g - want[k].double()).abs().max()) <= floor, k
    for k in (k for k in want if k.startswith("param/_encoder.rgb.")):
        got = params(k[len("param/"):]).detach().reshape(-1)[:SUB_NUMEL].double().cpu()
        assert float((got - want[k].double()).abs().max()) <= max(conv_param_abs, param_abs), k
    check_state({k: v for k, v in grads.items() if "grad/" + k not in zero}, params, emb_grad,
                {k: v for k, v in want.items() if k not in zero and not k.startswith("param/_encoder.rgb.")}, grad_rel,
                param_abs)
    return zero


def fixture_info(cfg, r, x):
    """The info dict of one oracle step, as the agent reports it."""
    info = {k: r[k] for k in ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss",
                              "grad_norm")}
    info.update(pi_loss=r["pi"]["loss"], pi_grad_norm=r["pi"]["grad_norm"], pi_scale=r["pi"]["scale"],
                pi_entropy=r["pi"]["entropy"].mean(), pi_scaled_entropy=r["pi"]["scaled_entropy"].mean())
    if cfg.episodic:
        from tdmpc2_b200.tdmpc2 import _termination_statistics
        info.update(_termination_statistics(torch.sigmoid(r["term_pred"][-1]), x["terminated"][-1]))
    return info
