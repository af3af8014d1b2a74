"""512-wide LayerNorm row phases (LN + Mish, LN + SimNorm) at their corners, on both engines, against float64:
constant rows (variance 0), rows poisoned by a NaN or an infinity, outputs far beyond the fp16 planes' +-65000 clamp,
and SimNorm groups dominated by one logit.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from helpers import agent_for, layer_list, ratio_rule

pytestmark = pytest.mark.gpu

ENGINES = ["simt", "tcgen05"]
F = torch.nn.functional


def _model():
    """c2's weights with dynamics.0 and dynamics.2 edited to reach the corners: a constant weight column 0 and a zero
    bias (an input e0 * s gives a constant pre-LayerNorm row), gamma 3e5 on every 16th column of dynamics.0 (Mish
    outputs near 1e6, clamped to +-65000 in the planes dynamics.1 reads) and beta 40 on the first column of every
    other SimNorm group of dynamics.2 (one dominant logit)."""
    cfg = workload("c2")
    sd = synth_state_dict(cfg, seed=3)
    for i in (0, 2):
        p = f"_dynamics.{i}"
        sd[p + ".weight"][:, 0] = 0.5
        sd[p + ".bias"].zero_()
    sd["_dynamics.0.ln.weight"][::16] = 3e5
    sd["_dynamics.2.ln.bias"][::16] = 40.0
    return cfg, sd


def _inputs(K, seed):
    """128 rows: row 0 constant pre-LayerNorm, rows 1-3 one NaN / +inf / -inf input, rows 4.. random at scales 1, 30,
    1e3."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(128, K, generator=g) * torch.tensor([1.0, 30.0, 1e3])[torch.arange(128) % 3].unsqueeze(1)
    x[0] = 0.0
    x[0, 0] = 4.0
    x[1, 5] = float("nan")
    x[2, 6] = float("inf")
    x[3, 7] = -float("inf")
    return x


def _ln_act(x, sd, prefix, simnorm, dt, clamp=False):
    h = F.linear(x.to(dt), sd[prefix + ".weight"].to(dt), sd[prefix + ".bias"].to(dt))
    h = F.layer_norm(h, (h.shape[-1],), sd[prefix + ".ln.weight"].to(dt), sd[prefix + ".ln.bias"].to(dt), 1e-5)
    if simnorm:
        return torch.softmax(h.view(h.shape[0], -1, 8), -1).view(h.shape[0], -1)
    h = F.mish(h)
    return h.clamp(-65000.0, 65000.0) if clamp else h


def _check_simnorm_sums(y):
    s = y.double().view(y.shape[0], -1, 8).sum(-1)
    assert float((s - 1).abs().max()) <= 8 * 2.0 ** -24, "a SimNorm group does not sum to 1"


@pytest.mark.parametrize("engine", ENGINES)
def test_ln_row_phase_corners_debug_layer(engine):
    from tdmpc2_b200.planner import Planner
    cfg, sd = _model()
    pl = Planner(cfg, 2, "cuda", engine=engine)
    pl.pack(sd)
    layers = {prefix: (li, simnorm) for (li, prefix, head, has_ln, simnorm) in layer_list(cfg)}
    for prefix in ("_dynamics.0", "_dynamics.2"):
        li, simnorm = layers[prefix]
        K = sd[prefix + ".weight"].shape[1]
        x = _inputs(K, 5)
        got = pl.debug_layer(li, 2 if simnorm else 1, x.cuda(), sd[prefix + ".weight"].shape[0]).cpu()
        assert got.shape[1] == 512
        o32, o64 = _ln_act(x, sd, prefix, simnorm, torch.float32), _ln_act(x, sd, prefix, simnorm, torch.float64)
        # a non-finite input poisons its own row and no other, as in float64
        assert bool(torch.isnan(got[1:4]).all()), f"{prefix}: a poisoned row is not all NaN"
        assert bool(torch.isnan(o64[1:4]).all())
        assert bool(torch.isfinite(got[4:]).all()) and bool(torch.isfinite(got[0]).all()), f"{prefix}: poison left its row"
        # variance 0: LayerNorm returns beta
        beta = sd[prefix + ".ln.bias"].double().unsqueeze(0)
        want0 = torch.softmax(beta.view(1, -1, 8), -1).view(1, -1) if simnorm else F.mish(beta)
        assert torch.allclose(got[0:1].double(), want0, rtol=1e-6, atol=1e-7), f"{prefix}: constant row"
        keep = torch.ones(128, dtype=torch.bool)
        keep[1:4] = False
        keep = keep.unsqueeze(1).expand_as(got)
        ratio_rule("simnorm" if simnorm else "ln+mish", f"row-phase/{prefix}/{engine}", got, o32, o64, keep, need=0.9)
        if simnorm:
            _check_simnorm_sums(got[keep[:, 0]])
            dom = got[4:].view(124, -1, 8)[:, ::2, 0]          # groups with the beta-40 logit
            assert float(dom.min()) > 1 - 1e-6
        else:
            assert float(got[4:].abs().max()) > 65000.0         # the pass reaches beyond the planes' clamp


@pytest.mark.parametrize("engine", ENGINES)
def test_ln_row_phase_corners_row_mode(engine):
    """WorldModel.next in row mode: dynamics.0 and .1 write the clamped fp16 planes the next GEMM reads, dynamics.2
    ends in SimNorm; float64 applies the same +-65000 clamp to the two hidden activations."""
    cfg, sd = _model()
    g = torch.Generator().manual_seed(9)
    R = 300                                                 # three tiles, the last one partly padding
    z = torch.softmax(torch.randn(R, cfg.latent_dim // 8, 8, generator=g) * 3, -1).view(R, -1)
    a = torch.rand(R, cfg.action_dim, generator=g) * 2 - 1
    z[0] = 0.0
    a[0] = 0.0
    z[0, 0] = 4.0                                           # a constant dynamics.0 row
    a[1, 3] = float("nan")

    def ref(dt):
        h = torch.cat([z, a], -1)
        h = _ln_act(h, sd, "_dynamics.0", False, dt, clamp=True)
        h = _ln_act(h, sd, "_dynamics.1", False, dt, clamp=True)
        return _ln_act(h, sd, "_dynamics.2", True, dt)

    m = agent_for(cfg, sd, engine).model
    got = m.next(z.cuda(), a.cuda(), None).cpu()
    o32, o64 = ref(torch.float32), ref(torch.float64)
    assert bool(torch.isnan(got[1]).all()) and bool(torch.isnan(o64[1]).all())
    ok = torch.ones(R, dtype=torch.bool)
    ok[1] = False
    assert bool(torch.isfinite(got[ok]).all()), "poison left its row"
    ratio_rule("next", f"row-phase/{engine}", got, o32, o64, ok.unsqueeze(1).expand_as(got), need=0.9)
    _check_simnorm_sums(got[ok])
