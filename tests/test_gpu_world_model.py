"""World-model methods and _td_target on the H100 kernels (plan_kernel's row mode) against fixtures minted from the
reference's own methods and against the CPU oracle (oracle/wm_oracle.py)."""
import pytest
import torch

from helpers import agent_for
from oracle.wm_oracle import CASES, WMOracle, case_model, load_case, with_target_blend

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
DEV = "cuda"

# |got - want| <= atol + rtol |want|
TOL = {"latent": (2e-6, 1e-5), "pi": (1e-5, 0.0), "value": (5e-5, 1e-5), "entropy": (1e-4, 1e-5)}
KIND = {"z": "latent", "next": "latent", "reward": "value", "pi_action": "pi", "pi_mean": "pi", "pi_log_std": "pi",
        "pi_entropy": "entropy", "pi_scaled_entropy": "entropy", "q_all": "value", "qt_all": "value", "q_min": "value",
        "q_avg": "value", "qt_min": "value", "term": "value", "term_logit": "value", "td": "value"}


def check(name, got, want, worst):
    atol, rtol = TOL[KIND[name]]
    got, want = got.detach().float().cpu(), want.float()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = (got - want).abs()
    worst[name] = max(worst.get(name, 0.0), float(err.max()))
    assert bool((err <= atol + rtol * want.abs()).all()), f"{name}: max err {float(err.max()):.3e}"


def run_all(m, r, cfg):
    """Every method through WorldModel's public surface with the fixture's draws."""
    dev = lambda t: None if t is None else t.to(DEV)
    task = dev(r["task"])
    z, a = dev(r["z"]), dev(r["a"])
    out = {"z": m.encode(dev(r["obs"]), task), "next": m.next(z, a, task), "reward": m.reward(z, a, task)}
    act, info = m.pi(z, task, eps=dev(r["pi_eps"]))
    out["pi_action"] = act
    for k in ("mean", "log_std", "entropy", "scaled_entropy"):
        out["pi_" + k] = info[k]
    sub = r["q_all"].shape[-2]
    out["q_all"] = m.Q(z, a, task, return_type="all")[..., :sub, :]
    out["qt_all"] = m.Q(z, a, task, return_type="all", target=True)[..., :sub, :]
    out["q_min"] = m.Q(z, a, task, qidx=dev(r["q_min_qidx"]))
    out["q_avg"] = m.Q(z, a, task, return_type="avg", detach=True, qidx=dev(r["q_avg_qidx"]))
    out["qt_min"] = m.Q(z, a, task, target=True, qidx=dev(r["qt_min_qidx"]))
    if cfg.episodic:
        out["term"] = m.termination(z, None)
        out["term_logit"] = m.termination(z, None, unnormalized=True)
    return out


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(CASES))
def test_methods_match_reference_golden(engine, name):
    cfg, sd, recs = load_case(name)
    agent = agent_for(cfg, sd, engine)
    worst = {}
    for pfx in ("b", "r"):          # [H, B, .] with task [B] (one full tile + a partial one); one 2-D row
        r = recs[pfx]
        out = run_all(agent.model, r, cfg)
        dev = lambda t: None if t is None else t.to(DEV)
        out["td"] = agent._td_target(dev(r["z"]), dev(r["reward_in"]), dev(r["terminated"]), dev(r["task"]),
                                     eps=dev(r["td_eps"]), qidx=dev(r["td_qidx"]))
        for k, v in out.items():
            check(k, v, r[k], worst)
    print(engine, name, {k: f"{e:.1e}" for k, e in worst.items()})


def oracle_rows(cfg, sd, R, seed):
    """Random inputs of R flat rows and the oracle's outputs for them."""
    g = torch.Generator().manual_seed(seed)
    o = WMOracle(cfg, sd)
    obs = torch.randn(R, cfg.obs_shape["state"][0], generator=g)
    task = torch.randint(0, len(cfg.tasks), (R,), generator=g) if cfg.multitask else None
    a = torch.rand(R, cfg.action_dim, generator=g) * 2 - 1
    eps = torch.randn(R, cfg.action_dim, generator=g)
    rew, term = torch.randn(R, 1, generator=g), (torch.rand(R, 1, generator=g) < 0.3).float()
    qidx = torch.randperm(cfg.num_q, generator=g)[:2]
    z = o.encode(obs, task)
    want = dict(z=z, next=o.next(z, a, task), q_all=o.Q(z, a, task, "all"),
                td=o.td_target(z, rew, term, task, eps, qidx))
    return dict(obs=obs, task=task, a=a, eps=eps, rew=rew, term=term, qidx=qidx), want


def kernel_rows(m, x, z=None):
    dev = lambda t: None if t is None else t.to(DEV)
    task = dev(x["task"])
    zz = m.encode(dev(x["obs"]), task) if z is None else z
    return dict(z=zz, next=m.next(zz, dev(x["a"]), task), q_all=m.Q(zz, dev(x["a"]), task, return_type="all"),
                td=m.td_target(zz, dev(x["rew"]), dev(x["term"]), task, eps=dev(x["eps"]), qidx=dev(x["qidx"])))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("wl", ["tiny-mt", "tiny-wide2"])
def test_row_counts_and_chunking(engine, wl):
    """Row counts 1, 127, 128, 129 and one past 132 x 128 (every CTA loops over several tiles) against the oracle; on
    the big batch every row is bit-identical to computing it in a small chunk.  tiny-wide2: multi-block columns."""
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    cfg = workload(wl)
    sd = with_target_blend(cfg, synth_state_dict(cfg, seed=31, perturb=True, emb_scale=60.0), 131)
    agent = agent_for(cfg, sd, engine)
    m = agent.model
    big = 132 * 128 + 77 if wl == "tiny-mt" else None       # the wide model's CPU oracle is too slow for the big batch
    worst = {}
    for R in (1, 127, 128, 129, 300) + ((big,) if big else ()):
        x, want = oracle_rows(cfg, sd, R, seed=R)
        got = kernel_rows(m, x)
        # z feeds the other methods; compare them on the oracle's z so that each checks its own layers
        got_on_want = kernel_rows(m, x, z=want["z"].to(DEV))
        check("z", got["z"], want["z"], worst)
        for k in ("next", "q_all", "td"):
            check(k, got_on_want[k], want[k], worst)
        if R == big:
            for lo in range(0, R, 1000):
                hi = min(R, lo + 1000)
                xc = {k: (v if k == "qidx" or v is None else v[lo:hi]) for k, v in x.items()}
                part = kernel_rows(m, xc)
                for k in ("z", "next", "td"):
                    assert torch.equal(part[k], got[k][lo:hi]), (k, lo)
                assert torch.equal(part["q_all"], got["q_all"][:, lo:hi])
    print(engine, wl, {k: f"{e:.1e}" for k, e in worst.items()})


@pytest.mark.parametrize("engine", ENGINES)
def test_target_and_online_weights(engine):
    """Target and online Q differ, each matches its own weights; sync_weights() after a Polyak-style update of the
    target ensemble re-packs it."""
    cfg, sd = case_model("tiny_mt_wm")
    agent = agent_for(cfg, sd, engine)
    x, _ = oracle_rows(cfg, sd, 300, seed=5)
    o = WMOracle(cfg, sd)
    z = o.encode(x["obs"], x["task"])
    dev = lambda t: t.to(DEV)
    m = agent.model
    q_on = m.Q(dev(z), dev(x["a"]), dev(x["task"]), return_type="all")
    q_tg = m.Q(dev(z), dev(x["a"]), dev(x["task"]), return_type="all", target=True)
    assert not torch.equal(q_on, q_tg)
    worst = {}
    check("q_all", q_on, o.Q(z, x["a"], x["task"], "all"), worst)
    check("qt_all", q_tg, o.Q(z, x["a"], x["task"], "all", target=True), worst)
    packed, ws = agent.planner.packed.numel(), agent.planner.workspace.numel()
    # Polyak update of the target ensemble, as a training loop does (world_model.py:76-80), then sync_weights()
    with torch.no_grad():
        for k in m.keys():
            if k.startswith("_target_Qs_params."):
                m.tensor(k).lerp_(m.tensor("_Qs.params." + k[len("_target_Qs_params."):]), 0.5)
    agent.sync_weights()
    sd2 = {k: v.detach().cpu() for k, v in m.state_dict().items() if torch.is_tensor(v)}
    q_tg2 = m.Q(dev(z), dev(x["a"]), dev(x["task"]), return_type="all", target=True)
    assert not torch.equal(q_tg2, q_tg)
    check("qt_all", q_tg2, WMOracle(cfg, sd2).Q(z, x["a"], x["task"], "all", target=True), worst)
    # the target blob is separate: the planner's own buffers keep their sizes
    assert agent.planner.packed.numel() == packed and agent.planner.workspace.numel() == ws
    print(engine, {k: f"{e:.1e}" for k, e in worst.items()})


def test_planner_without_target_keeps_its_memory():
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.planner import Planner
    cfg = workload("c2")
    pl = Planner(cfg, 4, DEV)
    packed, ws = pl.packed.numel(), pl.workspace.numel()
    assert pl.target_blob is None
    pl2 = Planner(cfg, 4, DEV)
    from tdmpc2_b200.synth import synth_state_dict
    sd = synth_state_dict(cfg, seed=1)
    pl2.pack(sd)
    pl2.pack_target_q(sd)
    assert pl2.packed.numel() == packed and pl2.workspace.numel() == ws and pl2.target_blob.numel() > 0


@pytest.mark.parametrize("engine", ENGINES)
def test_planner_state_is_not_disturbed(engine):
    """plan -> world-model calls -> plan gives the same actions, bit for bit, as plan -> plan, eagerly and through
    the captured graph."""
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.planner import draw_noise
    from tdmpc2_b200.synth import synth_state_dict
    cfg = workload("tiny-mt", num_envs=3)
    sd = with_target_blend(cfg, synth_state_dict(cfg, seed=41, perturb=True, emb_scale=60.0), 141)
    x, _ = oracle_rows(cfg, sd, 700, seed=7)
    dev = lambda t: t.to(DEV)

    def session(interleave, graphed):
        agent = agent_for(cfg, sd, engine)
        pl = agent.planner
        E = agent.num_envs
        g = torch.Generator().manual_seed(3)
        obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g).to(DEV)
        task = torch.tensor([0, 2, 1], dtype=torch.int32, device=DEV)
        t0 = torch.tensor([1, 0, 1], dtype=torch.uint8, device=DEV)
        prev = (torch.randn(E, cfg.horizon, cfg.action_dim, generator=g) * 0.3).to(DEV)
        gen = torch.Generator(device=DEV).manual_seed(11)
        acts = []
        for step in range(2):
            if graphed:
                a, prev = pl.plan_graphed(obs, task, t0, prev, generator=gen)
            else:
                nz = draw_noise(cfg, E, DEV, generator=gen, reference_order=False)
                a, prev, _ = pl.plan(obs, task, t0, prev, nz)
            acts.append(a.clone())
            if interleave and step == 0:
                m = agent.model
                z = m.encode(dev(x["obs"]), dev(x["task"]))
                m.next(z, dev(x["a"]), dev(x["task"]))
                m.pi(z, dev(x["task"]), eps=dev(x["eps"]))
                m.Q(z, dev(x["a"]), dev(x["task"]), return_type="all", target=True)
                agent._td_target(z, dev(x["rew"]), dev(x["term"]), dev(x["task"]), eps=dev(x["eps"]), qidx=dev(x["qidx"]))
        torch.cuda.synchronize()
        return acts

    for graphed in (False, True):
        base, mixed = session(False, graphed), session(True, graphed)
        for a, b in zip(base, mixed):
            assert torch.equal(a, b), f"graphed={graphed}"


def test_standalone_model_and_errors():
    """A WorldModel outside an agent creates its own one-environment planner; termination needs an episodic model."""
    from tdmpc2_b200 import _cabi
    from tdmpc2_b200.world_model import WorldModel
    cfg, sd, recs = load_case("tiny_episodic_wm")
    m = WorldModel(cfg).to(DEV)
    m.load_state_dict(sd)
    r = recs["b"]
    worst = {}
    check("z", m.encode(r["obs"].to(DEV), None), r["z"], worst)
    check("term", m.termination(r["z"].to(DEV), None), r["term"], worst)
    check("td", m.td_target(r["z"].to(DEV), r["reward_in"].to(DEV), r["terminated"].to(DEV), None,
                            eps=r["td_eps"].to(DEV), qidx=r["td_qidx"].to(DEV)), r["td"], worst)
    cfg2, sd2 = case_model("tiny_wm")
    m2 = WorldModel(cfg2).to(DEV)
    m2.load_state_dict(sd2)
    with pytest.raises(AttributeError):
        m2.termination(torch.zeros(2, cfg2.latent_dim, device=DEV), None)
    pl = m2._kernels()
    with pytest.raises(_cabi.CabiError, match=r"\(-5\)"):           # TDMPC2_ERR_UNSUPPORTED: no termination head
        pl.wm_termination(torch.zeros(2, cfg2.latent_dim, device=DEV), True)
    z, a = torch.zeros(2, cfg2.latent_dim, device=DEV), torch.zeros(2, cfg2.action_dim, device=DEV)
    q = torch.tensor([0, 1], dtype=torch.int32, device=DEV)
    with pytest.raises(_cabi.CabiError, match=r"\(-4\)"):           # TDMPC2_ERR_STATE: target blob not bound yet
        pl.wm_q(z, a, None, True, "min", q)
