"""Time `agent.update(buffer)` issued launch by launch (cfg.compile = False) against one CUDA-graph replay per step
(cfg.compile = True), in alternating rounds in one process.

    python scripts/bench_update_graph.py [--models c1 c1-rgb 48M] [--batch 256] [--horizon 3] [--repeats 20]
                                         [--warmup 5] [--rounds 3]

Models: c1 (5M, state obs 223, A 38); c1's shapes with pixel observations (C = 9 stacked uint8 frames, num_channels 32,
as bench_update_rgb.py builds it); the 48M preset (c3's shapes, obs 67, A 21) at H = 3.  Both arms start from the same
weights and generator seeds and sample one device-storage Buffer with generators of the same seed, so they take the same
steps; CUDA events around each call.  After the timed rounds the two arms' state dicts, optimisers and Q scale must be
bit-identical.  A separate profiler pass over one replay of the graph counts its kernel nodes, the pack kernels among
them (absmax / split / pad / embedding renorm) and its memcpy / memset nodes.  The graph's memory is the growth of
torch's reserved memory over the capturing call.  Prints the GPU's name and power limit, then one JSON line per model.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_update import gpu_info, timed                       # noqa: E402
from tdmpc2_b200.buffer import Buffer                                  # noqa: E402
from tdmpc2_b200.config import workload                                # noqa: E402
from tdmpc2_b200.synth import synth_state_dict                         # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2                                  # noqa: E402

PACK_KERNELS = ("absmax_kernel", "split_weight_kernel", "pad_vector_kernel", "emb_renorm_kernel")


def model_cfg(name, H, B):
    if name == "c1":
        return workload("c1", horizon=H, batch_size=B, buffer_size=20_000)
    if name == "c1-rgb":
        return workload("c1", obs="rgb", obs_channels=9, horizon=H, batch_size=B, buffer_size=5_000)
    if name == "48M":
        return workload("c3", num_envs=1, horizon=H, batch_size=B, buffer_size=20_000)
    raise SystemExit(f"unknown model {name!r}: c1, c1-rgb or 48M")


def fill(cfg, buf, n_eps=24, T1=101):
    g = torch.Generator().manual_seed(0)
    rgb = cfg.get("obs", "state") == "rgb"
    for _ in range(n_eps):
        obs = (torch.randint(0, 256, (T1, *cfg.obs_shape["rgb"]), generator=g, dtype=torch.uint8) if rgb
               else torch.randn(T1, cfg.obs_shape["state"][0], generator=g))
        ep = {"obs": obs, "action": torch.rand(T1, cfg.action_dim, generator=g) * 2 - 1,
              "reward": torch.randn(T1, generator=g), "terminated": torch.zeros(T1)}
        for k in ("action", "reward", "terminated"):
            ep[k][0] = float("nan")
        buf.add(ep)


def same(a, b):
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    if isinstance(a, dict):
        return set(a) == set(b) and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return a == b


def graph_nodes(st):
    """Kernel / pack-kernel / memcpy / memset activities of one replay of a captured step (torch.profiler)."""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=acts) as prof:
        st["graph"].replay()
        torch.cuda.synchronize()
    dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    copies = [e for e in dev if "memcpy" in e.name.lower()]
    sets = [e for e in dev if "memset" in e.name.lower()]
    kernels = [e for e in dev if e not in copies and e not in sets]
    packs = [e for e in kernels if any(p in e.name for p in PACK_KERNELS)]
    names = {}
    for e in kernels:
        names[e.name[:60]] = names.get(e.name[:60], 0) + 1
    top = dict(sorted(names.items(), key=lambda kv: -kv[1])[:12])
    return {"kernels": len(kernels), "pack_kernels": len(packs), "memcpy": len(copies), "memset": len(sets),
            "most_frequent_kernels": top}


def bench(name, args):
    dev = torch.device("cuda")
    cfg = model_cfg(name, args.horizon, args.batch)
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    buf = Buffer(cfg)
    fill(cfg, buf)
    agents, gens = {}, {}
    for arm, compile_ in (("eager", False), ("graph", True)):
        a = TDMPC2(cfg.replace(compile=compile_), device=dev)
        a.model.load_state_dict(sd)
        a.generator = torch.Generator(dev).manual_seed(2)
        agents[arm], gens[arm] = a, torch.Generator(dev).manual_seed(3)

    def call(arm):
        def f():
            buf.generator = gens[arm]
            agents[arm].update(buf)
        return f

    fns = {arm: call(arm) for arm in agents}
    timed(fns["eager"], args.warmup)
    timed(fns["graph"], 1)                                 # eager: Adam state, target blob, tables
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r0 = torch.cuda.memory_reserved()
    capture_ms = timed(fns["graph"], 1)[0]                 # capture + first replay
    pool = torch.cuda.memory_reserved() - r0
    assert agents["graph"].update_path == "captured", agents["graph"].update_path
    timed(fns["graph"], args.warmup - 2)
    pl_e, pl_g = agents["eager"]._planner, agents["graph"]._planner
    n0 = pl_e.launches
    fns["eager"]()
    torch.cuda.synchronize()
    launches = pl_e.launches - n0
    res = {"eager": [], "graph": []}
    for _ in range(args.rounds):
        for arm in ("eager", "graph"):
            res[arm] += timed(fns[arm], args.repeats)
    fns["graph"]()                                         # the eager arm made one extra call for the launch count
    assert agents["graph"].update_path == "replayed"
    torch.cuda.synchronize()
    e, g = agents["eager"], agents["graph"]
    identical = (same(e.model.state_dict(), g.model.state_dict()) and same(e.optim.state_dict(), g.optim.state_dict())
                 and same(e.pi_optim.state_dict(), g.pi_optim.state_dict()) and same(e.scale.value, g.scale.value))
    (st,) = pl_g.update_graphs.values()
    nodes = graph_nodes(st)                                # after the comparison: this replay is one more step
    summ = {k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for k, v in res.items()}
    speedup = statistics.median(res["eager"]) / statistics.median(res["graph"])
    out = {"model": name, "batch": args.batch, "horizon": args.horizon, **summ, "speedup_median": round(speedup, 3),
           "capture_call_ms": round(capture_ms, 2), "library_launches_per_update": launches,
           "library_launches_in_graph": st["launches"], "graph_nodes": nodes, "graph_pool_mib": round(pool / 2 ** 20, 1),
           "final_state_bit_identical": identical}
    for a in agents.values():
        a._planner.update_graphs.clear()
    return out, identical


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["c1", "c1-rgb", "48M"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--horizon", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update_graph.py times the H100 kernels: no CUDA device")
    if args.warmup < 3:
        raise SystemExit("--warmup must cover the eager call, the capture and one replay (>= 3)")
    print(gpu_info())
    ok = True
    for name in args.models:
        out, identical = bench(name, args)
        ok &= identical
        print(json.dumps(out), flush=True)
    if not ok:
        raise SystemExit("the two arms' final states differ")


if __name__ == "__main__":
    main()
