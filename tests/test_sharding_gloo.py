"""N > 1 path on CPU: environment-axis sharding + the single action all-gather, world_size 2 over gloo.
The per-rank planner is replaced by a deterministic stand-in (the kernels need a H100); what is under
test is the host logic bench.py and ShardedActor use: contiguous env blocks, rank-local planning,
all_gather_into_tensor of [E/G, A] actions in rank order."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tdmpc2_b200.sharded import ShardedActor, shard_range


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _fake_plan(obs, t0, task):
    """Stand-in for TDMPC2._plan on one shard: an action that depends on the env's obs and task only."""
    a = torch.tanh(obs[:, :4] * 0.5)
    if task is not None:
        a = a + 0.01 * task.to(a.dtype).unsqueeze(-1)
    return a


def _worker(rank, world, port, E, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)
        obs = torch.randn(E, 7, generator=g)                   # every rank holds the global batch (as bench.py does)
        task = torch.arange(E) % 3
        actor = ShardedActor(_fake_plan, E)
        assert (actor.lo, actor.hi) == shard_range(E, rank, world)
        out = actor.act(obs, t0=torch.zeros(E, dtype=torch.bool), task=task)
        want = _fake_plan(obs, None, task)
        ok = torch.equal(out, want)
        # scalar t0 / no task also pass through
        out2 = actor.act(obs, t0=True, task=None)
        ok = ok and torch.equal(out2, _fake_plan(obs, None, None))
        q.put((rank, bool(ok), tuple(out.shape)))
    finally:
        dist.destroy_process_group()


def test_env_sharding_all_gather_world2():
    world, E = 2, 12
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, E, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert sorted(r[0] for r in res) == [0, 1]
    assert all(r[1] for r in res), res
    assert all(r[2] == (E, 4) for r in res)


def test_shard_range_rejects_ragged():
    assert shard_range(256, 3, 8) == (96, 128)
    with pytest.raises(ValueError):
        shard_range(10, 0, 4)
