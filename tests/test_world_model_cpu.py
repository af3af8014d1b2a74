"""World-model methods without a GPU: the oracle (oracle/wm_oracle.py) against fixtures minted from the reference's own
WorldModel methods and _td_target, and the C entry points' no-device failure."""
import ctypes as C

import pytest
import torch

from oracle.wm_oracle import CASES, WMOracle, load_case

ORACLE_TOL = 7e-7


def rows_task(task, lead):
    return None if task is None else task.expand(*lead)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("batch", ["b", "r"])
def test_oracle_matches_reference_world_model(name, batch):
    cfg, sd, recs = load_case(name)
    o = WMOracle(cfg, sd)
    r = recs[batch]
    lead = r["obs"].shape[:-1]
    task = rows_task(r["task"], lead)
    z, a = r["z"], r["a"]
    got = {"z": o.encode(r["obs"], task), "next": o.next(z, a, task), "reward": o.reward(z, a, task)}
    act, info = o.pi(z, task, r["pi_eps"])
    got["pi_action"] = act
    for k in ("mean", "log_std", "entropy", "scaled_entropy"):
        got["pi_" + k] = info[k]
    sub = (Ellipsis, slice(0, r["q_all"].shape[-2]), slice(None))
    got["q_all"] = o.Q(z, a, task, "all")[sub]
    got["qt_all"] = o.Q(z, a, task, "all", target=True)[sub]
    got["q_min"] = o.Q(z, a, task, "min", qidx=r["q_min_qidx"])
    got["q_avg"] = o.Q(z, a, task, "avg", qidx=r["q_avg_qidx"])
    got["qt_min"] = o.Q(z, a, task, "min", target=True, qidx=r["qt_min_qidx"])
    if cfg.episodic:
        got["term"] = o.termination(z)
        got["term_logit"] = o.termination(z, unnormalized=True)
    got["td"] = o.td_target(z, r["reward_in"], r["terminated"], task, r["td_eps"], r["td_qidx"])
    worst = {}
    for k, v in got.items():
        assert v.shape == r[k].shape, (k, v.shape, r[k].shape)
        worst[k] = float(((v - r[k]).abs() / r[k].abs().clamp(min=1.0)).max())     # relative above |v| = 1
    print(name, batch, {k: f"{e:.1e}" for k, e in worst.items()})
    # entropies sum A log terms of magnitude up to ~10, and inherit the few-ulp difference of the renormalised task
    # embedding (nn.Embedding's in-place renorm vs its restatement): a relative 2e-6 there
    assert all(e <= (2e-6 if "entropy" in k else ORACLE_TOL) for k, e in worst.items()), worst
    # the target ensemble is not the online one
    assert not torch.equal(got["q_all"], got["qt_all"])


def test_td_target_discount_bits():
    """The kernels take the discount from the packer's table (planner.discount_table, column 1); reference
    _td_target multiplies with a Python float (single-task) or an fp32 tensor (multi-task, tdmpc2.py:35-37,256).
    Both give the same fp32 products."""
    from tdmpc2_b200.config import get_discount, workload
    from tdmpc2_b200.planner import discount_table
    x = torch.rand(4096) * 2 - 1
    for wl in ("tiny", "tiny-mt", "c1", "c4"):
        cfg = workload(wl)
        tab = discount_table(cfg, "cpu")[:, 1]
        if cfg.multitask:
            ref = torch.tensor([get_discount(cfg, ep) for ep in cfg.episode_lengths])
            assert torch.equal(tab, ref)
        else:
            d = get_discount(cfg, cfg.episode_length)
            assert torch.equal(d * x, tab[0] * x)


NEW_SYMBOLS = ["tdmpc2_planner_target_q_bytes", "tdmpc2_planner_bind_target_q", "tdmpc2_pack_target_q", "tdmpc2_wm_encode",
               "tdmpc2_wm_next", "tdmpc2_wm_reward", "tdmpc2_wm_termination", "tdmpc2_wm_pi", "tdmpc2_wm_q", "tdmpc2_td_target"]


@pytest.fixture(scope="module")
def lib():
    from tdmpc2_b200 import build, _cabi
    build.build()
    return _cabi.load()


def test_world_model_entry_points_exported(lib):
    from tdmpc2_b200 import _cabi
    assert _cabi.ABI_VERSION == 7 and lib.tdmpc2_abi_version() == 7
    for s in NEW_SYMBOLS:
        assert s in _cabi.SYMBOLS and hasattr(lib, s), s


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_world_model_entry_points_need_a_device(lib):
    nul = None
    calls = [lambda: lib.tdmpc2_wm_encode(nul, nul, nul, 1, nul, nul),
             lambda: lib.tdmpc2_wm_next(nul, nul, nul, nul, 1, nul, nul),
             lambda: lib.tdmpc2_wm_reward(nul, nul, nul, nul, 1, nul, nul),
             lambda: lib.tdmpc2_wm_termination(nul, nul, 1, 1, nul, nul),
             lambda: lib.tdmpc2_wm_pi(nul, nul, nul, nul, 1, nul, nul, nul, nul, nul),
             lambda: lib.tdmpc2_wm_q(nul, nul, nul, nul, 1, 0, 0, nul, nul, nul),
             lambda: lib.tdmpc2_td_target(nul, nul, nul, nul, nul, nul, nul, 1, nul, nul)]
    for f in calls:
        assert f() == -2 and b"no CUDA device" in lib.tdmpc2_last_error()     # TDMPC2_ERR_NO_DEVICE


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_world_model_methods_have_no_cpu_fallback():
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.world_model import WorldModel
    cfg = workload("tiny")
    m = WorldModel(cfg)
    z = torch.zeros(2, cfg.latent_dim)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.encode(torch.zeros(2, cfg.obs_shape["state"][0]), None)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.Q(z, torch.zeros(2, cfg.action_dim), None, target=True)
    with pytest.raises(NotImplementedError):
        WorldModel(workload("tiny-rgb")).encode(torch.zeros(1, 9, 64, 64), None)


def test_load_and_sync_mark_packed_weights_stale():
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.world_model import WorldModel
    m = WorldModel(workload("tiny"))
    v = m._version
    m.load_state_dict(m.state_dict())
    assert m._version == v + 1
    m.sync_weights()
    assert m._version == v + 2
