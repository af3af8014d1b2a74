"""Act latency of a plain C host: examples/c_act.c (tdmpc2_act, every draw on the device) captured as one CUDA graph and
replayed, against the Python agent's `agent.act` on the same model.

    python scripts/bench_act_c.py [--replays-e1 500] [--replays-c2 50] [--calls 50] [--out DIR]

Builds the library and c_act (gcc against the CUDA runtime) in a temporary directory, exports the c1 model (dog-run 5M,
synthetic weights, I = 8 after tdmpc2.py:34) once, and runs

  * c_act at E = 1 and at the c2 shape (E = 256 on the same model): CUDA-event time per replay of one captured
    tdmpc2_act, back to back on one stream (device time; no host copies);
  * `agent.act` at E = 1 the way bench.py's act_latency_e1 times it: CPU observation in, CPU action out, median
    wall-clock of `--calls` calls (torch's draws in the reference's order, interleaved with the launches).

Prints the GPU's name, power limit and maximum SM clock, then one JSON line; `--out DIR` also writes it there.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tdmpc2_b200 import _cabi, build                 # noqa: E402
from tdmpc2_b200.config import workload              # noqa: E402
from tdmpc2_b200.export import export_model          # noqa: E402
from tdmpc2_b200.synth import synth_state_dict       # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2                # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def compile_c_act(tmp):
    gcc = shutil.which("gcc")
    if gcc is None:
        raise RuntimeError("gcc not found: c_act cannot be built")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(build.find_nvcc())))
    cudalib = next(p for p in (os.path.join(cuda, "lib64"), os.path.join(cuda, "targets", "x86_64-linux", "lib"))
                   if os.path.exists(os.path.join(p, "libcudart.so")))
    libdir = os.path.dirname(_cabi.LIB_PATH)
    exe = os.path.join(tmp, "c_act")
    subprocess.run([gcc, "-std=c11", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                    os.path.join(ROOT, "examples", "c_act.c"), "-L" + libdir, "-ltdmpc2_b200", "-L" + cudalib, "-lcudart",
                    "-Wl,-rpath," + libdir, "-Wl,-rpath," + cudalib, "-o", exe], check=True)
    return exe


def c_act_graph_ms(exe, model, tmp, E, obs_dim, replays):
    obs = os.path.join(tmp, f"obs_{E}.bin")
    np.random.default_rng(0).standard_normal(3 * E * obs_dim).astype("<f4").tofile(obs)
    res = subprocess.run([exe, model, obs, os.path.join(tmp, f"act_{E}.bin"), "--envs", str(E), "--steps", "3",
                          "--graph", str(replays)], capture_output=True, text=True, timeout=900)
    if res.returncode != 0:
        raise RuntimeError(res.stdout + res.stderr)
    m = re.search(r"graph: (\d+) replays, ([0-9.]+) ms per act", res.stdout)
    return float(m.group(2))


def agent_act_ms(sd, calls):
    cfg = workload("c1", num_envs=1)
    agent = TDMPC2(cfg, device="cuda:0")
    agent.load(sd)
    obs = torch.randn(cfg.obs_shape["state"][0]).pin_memory()
    agent.act(obs, t0=True)
    for _ in range(5):
        agent.act(obs)
    torch.cuda.synchronize()
    ts = []
    for _ in range(calls):
        t = time.perf_counter()
        agent.act(obs)
        ts.append(1e3 * (time.perf_counter() - t))
    return statistics.median(ts), min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays-e1", type=int, default=500)
    ap.add_argument("--replays-c2", type=int, default=50)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    build.build()
    gpu = gpu_info()
    print(gpu)
    cfg = workload("c1")
    sd = synth_state_dict(cfg, seed=1)
    with tempfile.TemporaryDirectory() as tmp:
        exe = compile_c_act(tmp)
        model = os.path.join(tmp, "c1.tdmpc2")
        export_model(sd, cfg, model)
        obs_dim = cfg.obs_shape["state"][0]
        e1 = c_act_graph_ms(exe, model, tmp, 1, obs_dim, args.replays_e1)
        c2 = c_act_graph_ms(exe, model, tmp, workload("c2").num_envs, obs_dim, args.replays_c2)
    act_med, act_min = agent_act_ms(sd, args.calls)
    line = {"gpu": gpu, "model": "c1 dog-run 5M (synthetic weights), N 512, H 3, I 8",
            "c_act_graph_ms_per_act": {"E1": e1, "E256": c2},
            "agent_act_e1_ms": {"median": act_med, "min": act_min, "calls": args.calls},
            "what": "c_act: CUDA-event time per replay of one captured tdmpc2_act (device draws), back to back; agent.act: "
                    "wall clock of TDMPC2.act(obs on host) -> action on host, torch draws"}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_act_c.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
