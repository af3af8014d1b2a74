"""cfg.compile on the H100: `agent._update` / `agent.update(buffer)` as one CUDA-graph replay per step.

A compiled agent and an eager twin (same weights, same generator seeds, same buffer) take the same steps with act()
between them; every info dict and, at the end, the weights, both optimisers, the Q scale, the `.grad` pattern and the
next action agree bit for bit.  Also: a steady-state call is one cudaGraphLaunch and no host launch of the library,
without a host synchronisation; a new generator, set_engine, a rebound embedding gradient and an optimiser's
load_state_dict recapture, load() does not; explicit draws and a failed capture run eagerly; the trainers end as
their eager twins do."""
import pytest
import torch

from buffer_checks import episode
from test_gpu_trainer import ReachEnv, TaskReachEnv, assert_twins, losses, tensors_equal, write_dataset
from tdmpc2_b200.buffer import Buffer
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from tdmpc2_b200.tdmpc2 import TDMPC2
from tdmpc2_b200.trainer import MemoryLogger, OfflineTrainer, OnlineTrainer, set_seed
from trainer_checks import same, stored

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = {   # name: workload, overrides, engine
    "tiny-tcgen05": ("tiny", {}, "tcgen05"),
    "tiny-simt": ("tiny", {}, "simt"),
    "tiny-mt": ("tiny-mt", {}, "tcgen05"),
    "tiny-episodic": ("tiny", {"episodic": True}, "tcgen05"),
    "tiny-rgb": ("tiny-rgb", {}, "tcgen05"),
    "c1": ("c1", {"batch_size": 256}, "tcgen05"),
}


def twins(wl, over, engine=None, batch_size=32):
    """(compiled agent, eager agent, their buffers): same perturbed weights, generators, episodes and buffer draws."""
    cfg = workload(wl, **{"batch_size": batch_size, "buffer_size": 4000, **over})
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    rgb = cfg.get("obs", "state") == "rgb"
    obs_shape = cfg.obs_shape["rgb" if rgb else "state"]
    agents, bufs = [], []
    for compile_ in (True, False):
        set_seed(1)
        a = TDMPC2(cfg.replace(compile=compile_), device=DEV, engine=engine)
        a.model.load_state_dict(sd)
        a.generator = torch.Generator(DEV).manual_seed(2)
        buf = Buffer(cfg)
        for i in range(6):
            buf.add(episode(40, i, obs_shape=obs_shape, A=cfg.action_dim, terminated=True,
                            task=(i % len(cfg.tasks)) if cfg.multitask else None, seed=6))
        buf.generator = torch.Generator(DEV).manual_seed(3)
        agents.append(a)
        bufs.append(buf)
    return agents, bufs


def act_obs(cfg, i):
    """One act() input: [obs_dim] or [C, 64, 64] for one environment, [E, ...] for cfg.num_envs = E."""
    g = torch.Generator().manual_seed(100 + i)
    E = cfg.num_envs
    if cfg.get("obs", "state") == "rgb":
        obs = torch.randint(0, 256, (E, *cfg.obs_shape["rgb"]), generator=g, dtype=torch.uint8)
    else:
        obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    return obs[0] if E == 1 else obs


def act_both(agents, i):
    cfg = agents[0].cfg
    E = cfg.num_envs
    t0 = i % 2 == 0 if E == 1 else [(i + k) % 2 == 0 for k in range(E)]
    task = None
    if cfg.multitask:
        task = i % len(cfg.tasks) if E == 1 else [(i + k) % len(cfg.tasks) for k in range(E)]
    outs = [a.act(act_obs(cfg, i), t0=t0, task=task) for a in agents]
    assert same(*outs)


def grads(agent):
    return {k: agent.model.tensor(k).grad for k in agent.model._keys}


def assert_same_state(agents):
    assert_twins(*agents)
    tensors_equal(grads(agents[0]), grads(agents[1]), "grad")
    tensors_equal(agents[0].scale.state_dict(), agents[1].scale.state_dict(), "scale")


def step_both(agents, bufs):
    infos = [a.update(b) for a, b in zip(agents, bufs)]
    tensors_equal(infos[0], infos[1], "info")
    assert agents[1].update_path == "eager"
    return infos[0]


@pytest.mark.parametrize("case", list(CASES))
def test_twins_bit_for_bit(case):
    wl, over, engine = CASES[case]
    agents, bufs = twins(wl, over, engine, batch_size=over.get("batch_size", 32))
    paths = []
    for i in range(6):
        step_both(agents, bufs)
        paths.append(agents[0].update_path)
        act_both(agents, i)
    assert paths == ["eager", "captured", "replayed", "replayed", "replayed", "replayed"]
    assert_same_state(agents)
    act_both(agents, 99)


def test_one_graph_launch_per_step_without_host_sync():
    agents, bufs = twins("tiny", {})
    agent, buf = agents[0], bufs[0]
    for _ in range(3):
        agent.update(buf)
    pl = agent._planner
    (st,) = pl.update_graphs.values()
    assert st["launches"] > 0
    torch.cuda.synchronize()
    lib0, total0 = pl.lib.tdmpc2_planner_launch_count(pl.h), pl.launches
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        agent.update(buf)
        torch.cuda.synchronize()
    assert agent.update_path == "replayed"
    assert sum(e.name.startswith("cudaGraphLaunch") for e in prof.events()) == 1
    assert pl.lib.tdmpc2_planner_launch_count(pl.h) == lib0
    assert pl.launches == total0 + st["launches"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        agent.update(buf)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert agent.update_path == "replayed"


def change_generator(a):
    a.generator = torch.Generator(DEV).manual_seed(77)


def change_engine(a):
    a._planner.set_engine("simt")


def change_emb_grad(a):
    a.model.tensor("_task_emb.weight").grad = None


def change_optim(a):
    a.optim.load_state_dict(a.optim.state_dict())


def change_weights(a):
    a.load({"model": synth_state_dict(a.cfg, seed=9, perturb=True)})


INVALIDATIONS = {   # name: workload, change, whether the next call recaptures
    "generator": ("tiny", change_generator, True),
    "set_engine": ("tiny", change_engine, True),
    "emb_grad": ("tiny-mt", change_emb_grad, True),
    "optim_load_state_dict": ("tiny", change_optim, True),
    "load": ("tiny-mt", change_weights, False),
}


@pytest.mark.parametrize("name", list(INVALIDATIONS))
def test_invalidation(name):
    wl, change, recapture = INVALIDATIONS[name]
    agents, bufs = twins(wl, {})
    for i in range(3):
        step_both(agents, bufs)
        act_both(agents, i)
    assert agents[0].update_path == "replayed"
    for a in agents:
        change(a)
    paths = []
    for i in range(4):
        step_both(agents, bufs)
        paths.append(agents[0].update_path)
        act_both(agents, 10 + i)
    assert paths == (["eager", "captured", "replayed", "replayed"] if recapture else ["replayed"] * 4)
    assert_same_state(agents)


def test_explicit_draws_run_eagerly_and_info_dicts_stay():
    agents, bufs = twins("tiny", {})
    cfg = agents[0].cfg
    kept = []
    for i in range(4):
        info = step_both(agents, bufs)
        kept.append((info, {k: v.clone() for k, v in info.items()}))
    assert agents[0].update_path == "replayed"
    for info, copy in kept:                          # the dicts of earlier steps do not alias the graph's memory
        tensors_equal(info, copy, "kept info")
    H, B, A = cfg.horizon, cfg.batch_size, cfg.action_dim
    g = torch.Generator(DEV).manual_seed(8)
    draws = dict(td_eps=torch.randn(H, B, A, device=DEV, generator=g), td_qidx=torch.tensor([0, 1], device=DEV),
                 pi_eps=torch.randn(H + 1, B, A, device=DEV, generator=g))
    batch = bufs[0].sample()
    bufs[1].sample()
    infos = [a._update(*batch[:4], batch[4], **draws) for a in agents]
    assert [a.update_path for a in agents] == ["eager", "eager"]
    tensors_equal(infos[0], infos[1], "explicit-draw info")
    step_both(agents, bufs)
    assert agents[0].update_path == "replayed"        # the graph survives an explicit-draw call
    assert_same_state(agents)


def test_failed_capture_warns_and_runs_eagerly(monkeypatch):
    agents, bufs = twins("tiny", {})
    step_both(agents, bufs)

    class Refused:
        def __init__(self, *a, **k):
            pass

        def __enter__(self):
            raise RuntimeError("capture refused")

        def __exit__(self, *a):
            return False
    monkeypatch.setattr(torch.cuda, "graph", Refused)
    with pytest.warns(UserWarning, match="capture refused"):
        step_both(agents, bufs)
    monkeypatch.undo()
    assert agents[0].update_path == "eager" and not agents[0]._compile
    step_both(agents, bufs)
    assert agents[0].update_path == "eager"
    assert_same_state(agents)


@pytest.mark.parametrize("E", [1, 4])
def test_online_trainer_twins(E):
    cfg = workload("tiny", obs_dim=4, action_dim=2, num_envs=E, batch_size=64, episode_length=20, seed_steps=40 * E,
                   steps=100 * E, eval_freq=50 * E, eval_episodes=2, episodic=E > 1)
    logs, agents, bufs = [], [], []
    for compile_ in (True, False):
        set_seed(1)
        agent = TDMPC2(cfg.replace(compile=compile_), device=DEV)
        agent.generator = torch.Generator(DEV).manual_seed(2)
        buf = Buffer(cfg)
        buf.generator = torch.Generator(DEV).manual_seed(3)
        logger = MemoryLogger()
        envs = [ReachEnv(4 + k, length=20 - 2 * k, terminate=E > 1) for k in range(E)]
        eval_envs = None if E == 1 else [ReachEnv(20 + k, length=12) for k in range(E)]
        OnlineTrainer(cfg, envs, agent, buf, logger=logger, eval_envs=eval_envs).train()
        logs.append(logger.logs)
        agents.append(agent)
        bufs.append(buf)
    assert agents[0].update_path == "replayed" and agents[1].update_path == "eager"
    got, want = logs
    assert [c for c, _ in got] == [c for c, _ in want]
    for (_, dg), (_, dw) in zip(losses(got), losses(want)):
        tensors_equal(dg, dw, "losses")
    assert_twins(*agents)
    assert bufs[0]._table == bufs[1]._table
    for g, w in zip(stored(bufs[0]), stored(bufs[1])):
        assert all(same(g[k], w[k]) for k in g)


def test_offline_trainer_twins(tmp_path):
    cfg = workload("tiny-mt", num_envs=2, batch_size=32, episode_length=20, buffer_size=400, steps=25, eval_freq=10,
                   eval_episodes=1)
    files = [tmp_path / "d0.pt", tmp_path / "d1.pt"]
    write_dataset(files[0], cfg, 6, 21, 1)
    write_dataset(files[1], cfg, 5, 21, 2)
    logs, agents, bufs = [], [], []
    for compile_ in (True, False):
        set_seed(21)
        agent = TDMPC2(cfg.replace(compile=compile_), device=DEV)
        agent.generator = torch.Generator(DEV).manual_seed(22)
        set_seed(23)
        logger = MemoryLogger()
        tr = OfflineTrainer(cfg, agent, files, [TaskReachEnv(24 + k, cfg) for k in range(2)], logger=logger)
        with pytest.warns(UserWarning, match="11 episodes"):
            tr.train()
        logs.append(logger.logs)
        agents.append(agent)
        bufs.append(tr.buffer)
    assert agents[0].update_path == "replayed"
    assert_twins(*agents)
    assert bufs[0]._table == bufs[1]._table
    got, want = logs
    assert [(c, d["iteration"]) for c, d in got] == [(c, d["iteration"]) for c, d in want]
    for (_, dg), (_, dw) in zip(got, want):
        assert set(dg) == set(dw)
        for k in dw:
            if torch.is_tensor(dw[k]):
                assert same(dg[k], dw[k]), k
            elif k not in ("elapsed_time", "steps_per_second"):
                assert dg[k] == dw[k], k
