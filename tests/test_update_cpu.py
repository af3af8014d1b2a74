"""agent._update without a GPU: the oracle against fixtures minted from the reference's own _update, the config
defaults, the optimiser's groups against the reference's __init__, soft_update_target_Q, and the refusals."""
import os

import pytest
import torch

from oracle.update_oracle import CASES, MULTI_STEP, load_case, run_case, soft_ce
from tdmpc2_b200.config import workload
from update_checks import check_info, check_state, steps_of

FIXTURES = list(CASES) + list(MULTI_STEP)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_matches_reference_fixture(name):
    base, steps = steps_of(name)
    cfg, sd, _, want = load_case(name)
    _, _, out = run_case(base, steps=steps)
    for s, (_, r) in enumerate(out):
        info = {k: r[k] for k in ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss",
                                  "grad_norm")}
        info.update(pi_loss=r["pi"]["loss"], pi_grad_norm=r["pi"]["grad_norm"], pi_scale=r["pi"]["scale"],
                    pi_entropy=r["pi"]["entropy"].mean(), pi_scaled_entropy=r["pi"]["scaled_entropy"].mean())
        if cfg.episodic:
            from tdmpc2_b200.tdmpc2 import _termination_statistics
            x = out[s][0]
            info.update(_termination_statistics(torch.sigmoid(r["term_pred"][-1]), x["terminated"][-1]))
        check_info(info, want, "info/" if s == 0 else f"info{s}/", rel=1e-5, gn_rel=1e-5)
    r = out[-1][1]
    check_state(r["grads"], lambda k: r["sd"][k], r["emb_grad"], want, grad_rel=1e-5, param_abs=1e-6)


def test_config_defaults():
    cfg = workload("tiny")
    assert (cfg.reward_coef, cfg.value_coef, cfg.termination_coef, cfg.consistency_coef) == (0.1, 0.1, 1, 20)


@pytest.mark.parametrize("wl,over", [("tiny", {}), ("tiny-mt", {}), ("tiny", {"episodic": True})])
def test_optim_groups(wl, over):
    """agent.optim against the reference's own optimiser of tdmpc2.py:22-30, built on the reference's modules."""
    from oracle import ref_harness as rh
    from tdmpc2_b200.synth import synth_state_dict
    from tdmpc2_b200.tdmpc2 import TDMPC2
    if not rh.available():
        pytest.skip("reference modules not available")
    cfg = workload(wl, **over)
    agent = TDMPC2(cfg, device="cpu")
    ref = rh.build_agent(cfg, synth_state_dict(cfg, seed=1))
    rh._import_reference()
    # the reference's __init__ hard-codes cuda:0; its optimiser is rebuilt here by running those lines' source
    import inspect
    import textwrap
    src = inspect.getsource(type(ref).__init__)
    start = src.index("self.optim = torch.optim.Adam(")
    end = src.index("self.pi_optim")
    ns = {"self": ref, "torch": torch}
    exec(textwrap.dedent(src[start:end]), ns)
    want = ref.optim.param_groups
    names = {id(p): n for n, p in ref.model.named_parameters()}
    mine = {id(agent.model.tensor(k)): k for k in agent.model.keys() if not k.startswith("_detach_Qs_params.")}
    got = agent.optim.param_groups
    assert len(got) == len(want)
    for g, w in zip(got, want):
        gk = [mine[id(p)] for p in g["params"]]
        wk = [names[id(p)] for p in w["params"]]
        wk = ["_Qs.params." + n[len("_Qs.p."):].replace("/", ".") if n.startswith("_Qs.p.") else n for n in wk]
        if gk and gk[0].startswith("_Qs.params."):
            # the harness's stand-in for the tensordict ensemble orders its parameters its own way; Adam is elementwise
            assert sorted(gk) == sorted(wk)
        else:
            assert gk == wk
            assert [tuple(p.shape) for p in g["params"]] == [tuple(p.shape) for p in w["params"]]
        for key in ("lr", "eps", "betas", "weight_decay", "amsgrad"):
            assert g[key] == w[key], key
    assert ref.optim.defaults["capturable"] is True       # the reference's; this agent is capturable on CUDA devices only
    assert agent.optim.defaults["capturable"] is False


def test_soft_update_target_q():
    from tdmpc2_b200.tdmpc2 import TDMPC2
    cfg = workload("tiny")
    agent = TDMPC2(cfg, device="cpu")
    m = agent.model
    keys = [k for k in m.keys() if k.startswith("_target_Qs_params.")]
    before = {k: m.tensor(k).clone() for k in keys}
    for k in keys:
        m.tensor("_Qs.params." + k[len("_target_Qs_params."):]).data.add_(1.0)
    v = m._version
    m.soft_update_target_Q()
    assert m._version == v + 1
    for k in keys:
        online = m.tensor("_Qs.params." + k[len("_target_Qs_params."):])
        assert torch.equal(m.tensor(k), torch.lerp(before[k], online, cfg.tau))


def test_cpu_and_pixel_refusals():
    from tdmpc2_b200.tdmpc2 import TDMPC2
    cfg = workload("tiny")
    agent = TDMPC2(cfg, device="cpu")
    H, B, A = 2, 4, cfg.action_dim
    args = (torch.zeros(H + 1, B, cfg.obs_shape["state"][0]), torch.zeros(H, B, A), torch.zeros(H, B, 1), torch.zeros(H, B, 1))
    with pytest.raises(RuntimeError, match="CUDA"):
        agent._update(*args)
    rgb = workload("tiny", obs="rgb", num_channels=4, latent_dim=64)
    pix = TDMPC2(rgb, device="cpu")
    with pytest.raises(NotImplementedError, match="conv encoder"):
        pix._update(torch.zeros(H + 1, B, 3, 64, 64), *args[1:])


def test_soft_ce_two_hot_edges():
    cfg = workload("tiny")
    sym = lambda v: torch.sign(v) * (torch.exp(torch.abs(v)) - 1)
    # a target on a bin centre puts all its weight there; +-symexp(vmax) and beyond the clamp land on the end bins
    centres = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins)
    logits = torch.randn(4, cfg.num_bins)
    for i, tgt in ((37, sym(centres[37])), (cfg.num_bins - 1, sym(torch.tensor(cfg.vmax))), (0, torch.tensor(-1e6))):
        ce = soft_ce(logits[:1], tgt.view(1, 1), cfg)
        assert torch.allclose(ce, -torch.log_softmax(logits[:1], -1)[:, i:i + 1], atol=1e-4)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_fp32_against_float64(name):
    """The fp32 oracle's losses and gradients sit within fp32 error of its float64 restatement."""
    _, _, o32 = run_case(name)
    _, _, o64 = run_case(name, dtype=torch.float64)
    a, b = o32[0][1], o64[0][1]
    for k in ("consistency_loss", "reward_loss", "value_loss", "termination_loss", "total_loss", "grad_norm"):
        assert abs(float(a[k]) - float(b[k])) <= 1e-4 * abs(float(b[k])) + 1e-6, k
    for k, w in b["grads"].items():
        assert float((a["grads"][k].double() - w).abs().max()) <= 1e-3 * float(w.abs().max()) + 1e-9, k
