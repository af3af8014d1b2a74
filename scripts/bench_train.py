"""Online training throughput: OnlineTrainer on a toy environment with c1's shapes (state obs 223, A = 38, the 5M preset,
B = 256, H = 3), at E = 1 and E = 16 environments in lock-step.

    python scripts/bench_train.py [--envs 1 16] [--seed-steps 511] [--measure-steps 320] [--warm-acts 4] [--compile]

Each E runs twice from the same seeds.  With --compile, each E runs three times: untimed without and with cfg.compile
(every update a CUDA-graph replay after its first two calls), then split with cfg.compile.
  untimed  trainer.train() as a user runs it; the window opens at the `--warm-acts`-th training act() (the act graph and
           every update shape are warm by then) and closes when train() returns, each end behind a device synchronise.
           Reports env steps per second in the window.
  split    the same run with act(), env.step(), buffer.add() and update() each between host clocks that end in a
           device synchronise; reports milliseconds per env step in each part over the same window, and the rest
           (the trainer's own bookkeeping, stacking, and the synchronises themselves).
seed_steps = 511 is one less than a multiple of 16, so the vector step that runs the seed updates ends the seeding at
both E, and at E = 16 it gives each slot 32 steps: a whole 25-step episode is in the buffer when the updates start.
The toy environment is a fixed linear system on the host (x' = 0.95 x + 0.1 W a, reward -mean(x^2), 25-step
episodes), cheap beside the agent's calls.  Evaluation runs once, at step 0, before the window.  Prints the
GPU's name and power limit, then one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from time import perf_counter

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_update import gpu_info                              # noqa: E402
from tdmpc2_b200.buffer import Buffer                                  # noqa: E402
from tdmpc2_b200.config import workload                                # noqa: E402
from tdmpc2_b200.tdmpc2 import TDMPC2                                  # noqa: E402
from tdmpc2_b200.trainer import MemoryLogger, OnlineTrainer, set_seed  # noqa: E402

OBS, A, LENGTH = 223, 38, 25


class LinearEnv:
    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)
        self.W = torch.randn(OBS, A, generator=torch.Generator().manual_seed(0)) / A ** 0.5

    def reset(self, task_idx=None):
        self.x, self.t = torch.randn(OBS, generator=self.g), 0
        return self.x.clone()

    def rand_act(self):
        return torch.rand(A, generator=self.g) * 2 - 1

    def step(self, action):
        self.x = 0.95 * self.x + 0.1 * (self.W @ action)
        self.t += 1
        info = {"terminated": torch.tensor(0.0), "success": 0.0}
        return self.x.clone(), -(self.x ** 2).mean(), self.t >= LENGTH, info


class Clock:
    """Wraps the trainer's four calls.  `split`: each call between host clocks ending in a device synchronise.  The
    window opens at the warm_acts-th training act (behind a synchronise) and counts env steps from there."""

    PARTS = ("act", "env_step", "buffer_add", "update")

    def __init__(self, split, warm_acts):
        self.split, self.warm_acts = split, warm_acts
        self.acts = self.env_steps = 0
        self.start = None                     # (time, env steps) when the window opened
        self.time = dict.fromkeys(self.PARTS, 0.0)

    def wrap(self, part, fn, opens=False):
        def call(*a, **k):
            if opens and not k.get("eval_mode", False):       # evaluation's acts run before the window
                self.acts += 1
                if self.acts == self.warm_acts:
                    torch.cuda.synchronize()
                    self.start = (perf_counter(), self.env_steps)
            if part == "env_step":
                self.env_steps += 1
            if not (self.split and self.start is not None):
                return fn(*a, **k)
            torch.cuda.synchronize()
            t = perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            self.time[part] += perf_counter() - t
            return out
        return call


def run(E, split, args, compile_=False):
    cfg = workload("c1", num_envs=E, batch_size=256, horizon=3, episode_length=LENGTH, seed_steps=args.seed_steps,
                   steps=args.seed_steps + args.measure_steps, eval_freq=10 ** 9, eval_episodes=1, compile=compile_)
    set_seed(1)
    agent = TDMPC2(cfg, device="cuda")
    agent.generator = torch.Generator("cuda").manual_seed(2)
    buf = Buffer(cfg)
    buf.generator = torch.Generator("cuda").manual_seed(3)
    envs = [LinearEnv(10 + k) for k in range(E)]
    eval_envs = [LinearEnv(100 + k) for k in range(E)]
    clock = Clock(split, args.warm_acts)
    agent.act = clock.wrap("act", agent.act, opens=True)
    agent.update = clock.wrap("update", agent.update)
    buf.add = clock.wrap("buffer_add", buf.add)
    for env in envs:
        env.step = clock.wrap("env_step", env.step)
    trainer = OnlineTrainer(cfg, envs, agent, buf, logger=MemoryLogger(), eval_envs=eval_envs)
    trainer.train()
    torch.cuda.synchronize()
    t1 = perf_counter()
    t0, s0 = clock.start
    steps, seconds = clock.env_steps - s0, t1 - t0
    out = {"env_steps": steps, "seconds": round(seconds, 3), "env_steps_per_s": round(steps / seconds, 2)}
    if split:
        ms = {k: 1e3 * v / steps for k, v in clock.time.items()}
        ms["rest"] = 1e3 * seconds / steps - sum(ms.values())
        out["ms_per_env_step"] = {k: round(v, 4) for k, v in ms.items()}
    losses = [float(d["total_loss"]) for c, d in trainer.logger.logs if c == "train" and "total_loss" in d]
    out["last_total_loss"] = losses[-1] if losses else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--seed-steps", type=int, default=511)
    ap.add_argument("--measure-steps", type=int, default=320)
    ap.add_argument("--warm-acts", type=int, default=4)
    ap.add_argument("--compile", action="store_true", help="also run with cfg.compile (the update as a CUDA graph)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py times the H100 kernels: no CUDA device")
    info = gpu_info()
    print(info)
    out = {"gpu": info, "workload": "c1 shapes (obs 223, A 38, 5M), B 256, H 3", "seed_steps": args.seed_steps}
    for E in args.envs:
        if args.compile:
            res = {"untimed": run(E, False, args), "untimed_compile": run(E, False, args, True),
                   "split_compile": run(E, True, args, True)}
        else:
            res = {"untimed": run(E, False, args), "split": run(E, True, args)}
        print(f"E={E}: {res}", flush=True)
        out[f"E{E}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
