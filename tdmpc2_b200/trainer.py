"""Training loops with the reference's surface (tdmpc2/trainer/online_trainer.py, offline_trainer.py, common/seed.py),
on `TDMPC2.act` / `TDMPC2.update` and `Buffer`: no torchrl, tensordict or wandb.

* `OnlineTrainer(cfg, envs, agent, buffer).train()` collects experience from E = len(envs) environments in lock-step
  (E == agent.num_envs) and trains on it.  At E = 1 it makes the reference's calls in the reference's order
  (online_trainer.py:74-127).  At E > 1 vector step k covers env steps j = kE ... kE + E - 1, slot i taking j = kE + i,
  and every per-step rule of the reference is applied to the covered j:
    - a slot with j > seed_steps acts through ONE batched `agent.act(obs[E], t0[E])` per vector step, a slot with
      j <= seed_steps takes its own `rand_act()`; no act() is made while every slot is seeding;
    - the vector step runs sum over the covered j of (seed_steps if j == seed_steps, 1 if j > seed_steps, else 0)
      updates, the reference's one update per env step;
    - the evaluation flag is raised when a covered j is a multiple of eval_freq; the evaluation runs at the first vector
      step, this one included, at which some slot is at an episode end;
    - each slot's episode ends on its own: it is logged and added to the buffer (slots in ascending order), the slot's
      environment is reset and its t0 raised;
    - the loop ends after the vector step that covers cfg.steps.
  Draws: the agent's from `agent.generator`, the buffer's from `buffer.generator`, random actions (and the one
  `rand_act()` each episode's NaN first row takes its shape from, as the reference's `to_td` does) from each
  environment's own generator.
* `OfflineTrainer(cfg, agent, data_files, eval_envs).train()` loads the data files into a `Buffer` of the reference's
  dataset capacity and runs cfg.steps updates, logging, evaluating and checkpointing at the reference's iterations.
* Evaluation is `evaluate.evaluate(agent, eval_envs, cfg.eval_episodes, eval_mode=True)`.  The online trainer saves
  `agent._prev_mean` before it and restores the rows of the slots in mid-episode after it, so that they keep their warm
  starts; a slot at an episode end keeps what the evaluation left, as the reference's single environment does (at E = 1
  an evaluation only runs at an episode end, so nothing is restored).
* A logger is anything with the reference Logger's `log(metrics, category)`, `save_agent(agent, identifier)` and
  `finish(agent)`; `MemoryLogger` is the default.

Environments have the reference wrappers' surface (envs/wrappers/tensor.py): `reset()` -> obs tensor, `step(action)` ->
(obs, reward tensor, done, info) with info['terminated'] (tensor) and info['success'], `rand_act()` -> action tensor;
multi-task evaluation environments take `reset(task_idx=...)`.
"""
from __future__ import annotations

import copy
import random
import warnings
from pathlib import Path
from time import time
from typing import Any, List, Optional, Sequence

import numpy as np
import torch

from .buffer import Buffer
from .evaluate import evaluate

_DATASET_FIELDS = ("obs", "action", "reward", "terminated", "task")
# offline_trainer.py:53-55: rows per episode and capacity of the released multi-task datasets
_DATASETS = {"mt80": (101, 550_450_000), "mt30": (501, 345_690_000)}


def set_seed(seed: int) -> None:
    """Seed `random`, numpy, torch and every CUDA device (common/seed.py)."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


def seed_steps(cfg) -> int:
    """cfg.seed_steps, or when it is None max(1000, 5 * episode_length) (envs/__init__.py:82)."""
    s = cfg.get("seed_steps")
    return int(max(1000, 5 * cfg.episode_length) if s is None else s)


class MemoryLogger:
    """The reference Logger's three methods without wandb, CSV or video: `logs` keeps (category, metrics) in call order
    (a copy of each dict; values are kept as given, device tensors included), and with a `directory` `save_agent`
    writes `agent.save()` checkpoints there as `<identifier>.pt` (`finish` saves 'final')."""

    def __init__(self, directory=None):
        self.directory = None if directory is None else Path(directory)
        self.logs: List[tuple] = []
        self.saved: List[Path] = []

    def log(self, metrics, category="train"):
        self.logs.append((category, dict(metrics)))

    def save_agent(self, agent=None, identifier="final"):
        if self.directory is None or agent is None:
            return
        self.directory.mkdir(parents=True, exist_ok=True)
        fp = self.directory / f"{identifier}.pt"
        agent.save(fp)
        self.saved.append(fp)

    def finish(self, agent=None):
        self.save_agent(agent)


class _Episode:
    """One slot's running episode, one row per step as the reference's to_td builds it (online_trainer.py:54-72): the
    first row holds the reset observation with NaN action, reward and terminated."""

    def __init__(self, obs, action_like):
        nan = torch.tensor(float("nan"))
        self.obs, self.action = [obs], [torch.full_like(action_like, float("nan"))]
        self.reward, self.terminated = [nan], [nan]

    def __len__(self) -> int:
        return len(self.obs)

    def append(self, obs, action, reward, terminated) -> None:
        self.obs.append(obs)
        self.action.append(action)
        self.reward.append(torch.as_tensor(reward, dtype=torch.float32).reshape(()))
        self.terminated.append(torch.as_tensor(terminated, dtype=torch.float32).reshape(()))

    def stack(self) -> dict:
        return {"obs": torch.stack(self.obs), "action": torch.stack(self.action),
                "reward": torch.stack(self.reward), "terminated": torch.stack(self.terminated)}


class OnlineTrainer:
    """Single-task online training over E environments in lock-step (see the module docstring).  At E > 1 each slot
    has taken about seed_steps / E steps when the seed updates run, and only finished episodes are in the buffer, so
    seed_steps must cover a whole episode per slot (about E * (episode_length + 1) steps)."""

    def __init__(self, cfg, envs: Sequence[Any], agent, buffer, logger=None, eval_envs: Optional[Sequence[Any]] = None):
        envs = list(envs)
        E = len(envs)
        if cfg.multitask:
            raise ValueError("online training is single-task; multi-task models train offline (OfflineTrainer)")
        if E < 1 or E != int(agent.num_envs):
            raise ValueError(f"{E} environments for an agent built with cfg.num_envs={agent.num_envs}")
        if eval_envs is None:
            if E > 1:
                raise ValueError(f"training on {E} environments needs {E} separate eval_envs: an evaluation may start "
                                 f"while training episodes are in progress")
            eval_envs = envs
        eval_envs = list(eval_envs)
        if len(eval_envs) != E:
            raise ValueError(f"{len(eval_envs)} eval_envs for an agent built with cfg.num_envs={E}")
        self.cfg, self.envs, self.agent, self.buffer = cfg, envs, agent, buffer
        self.eval_envs = eval_envs
        self.logger = MemoryLogger() if logger is None else logger
        self.seed_steps = seed_steps(cfg)
        self._step = 0
        self._ep_idx = 0
        self._start_time = time()

    def common_metrics(self) -> dict:
        elapsed_time = time() - self._start_time
        return dict(step=self._step, episode=self._ep_idx, elapsed_time=elapsed_time,
                    steps_per_second=self._step / elapsed_time)

    def eval(self) -> dict:
        r = evaluate(self.agent, self.eval_envs, self.cfg.eval_episodes, eval_mode=True)["tasks"][self.cfg.task]
        return dict(episode_reward=r.reward, episode_success=r.success,
                    episode_length=sum(r.episode_lengths) / len(r.episode_lengths))

    def _end_episode(self, episode: _Episode, info, train_metrics: dict) -> None:
        if bool(info["terminated"]) and not self.cfg.episodic:
            raise ValueError("an environment reported a termination but cfg.episodic is false: set episodic=True to "
                             "train with terminations")
        ep = episode.stack()
        train_metrics.update(episode_reward=ep["reward"][1:].sum(), episode_success=info["success"],
                             episode_length=len(episode), episode_terminated=info["terminated"])
        train_metrics.update(self.common_metrics())
        self.logger.log(train_metrics, "train")
        self._ep_idx = self.buffer.add(ep)

    def train(self) -> None:
        cfg, agent, envs, E = self.cfg, self.agent, self.envs, len(self.envs)
        seed, eval_freq = self.seed_steps, int(cfg.eval_freq)
        train_metrics, eval_next = {}, False
        done: List[bool] = [True] * E
        obs: List[Any] = [None] * E
        info: List[Any] = [None] * E
        episodes: List[Optional[_Episode]] = [None] * E
        while self._step <= cfg.steps:
            js = range(self._step, self._step + E)                   # the env steps this vector step covers
            if any(j % eval_freq == 0 for j in js):
                eval_next = True
            if any(done):
                if eval_next:
                    mid = [i for i in range(E) if not done[i]]             # slots in mid-episode keep their warm starts
                    warm = agent._prev_mean.clone() if mid else None
                    eval_metrics = self.eval()
                    for i in mid:
                        agent._prev_mean.view(E, -1)[i].copy_(warm.view(E, -1)[i])
                    eval_metrics.update(self.common_metrics())
                    self.logger.log(eval_metrics, "eval")
                    eval_next = False
                for i in range(E):
                    if not done[i]:
                        continue
                    if episodes[i] is not None:
                        self._end_episode(episodes[i], info[i], train_metrics)
                    obs[i] = envs[i].reset()
                    episodes[i] = _Episode(obs[i], envs[i].rand_act())

            acting = [j > seed for j in js]
            if any(acting):
                t0 = torch.tensor([len(ep) == 1 for ep in episodes])
                planned = agent.act(torch.stack(obs), t0=t0).reshape(E, -1)
            actions = [planned[i] if acting[i] else envs[i].rand_act() for i in range(E)]
            for i in range(E):
                obs[i], reward, d, info[i] = envs[i].step(actions[i])
                done[i] = bool(d)
                episodes[i].append(obs[i], actions[i], reward, info[i]["terminated"])

            num_updates = sum(seed if j == seed else int(j > seed) for j in js)
            for _ in range(num_updates):
                update_metrics = agent.update(self.buffer)
            if num_updates:
                train_metrics.update(update_metrics)
            self._step += E
        self.logger.finish(agent)


class OfflineTrainer:
    """Multi-task offline training on a fixed dataset (offline_trainer.py).  `data_files` are `torch.save`d mappings of
    [N_eps, T, ...] tensors (obs, action, reward, task, optionally terminated), loaded in the order given."""

    def __init__(self, cfg, agent, data_files: Sequence[Any], eval_envs: Sequence[Any], logger=None):
        if not cfg.multitask:
            raise ValueError("offline training is multi-task: cfg.multitask must be true")
        self.data_files = [Path(f) for f in data_files]
        if not self.data_files:
            raise ValueError("no data files given")
        self.cfg, self.agent, self.eval_envs = cfg, agent, list(eval_envs)
        if len(self.eval_envs) != int(agent.num_envs):
            raise ValueError(f"{len(self.eval_envs)} eval_envs for an agent built with cfg.num_envs={agent.num_envs}")
        self.logger = MemoryLogger() if logger is None else logger
        self.buffer: Optional[Buffer] = None
        self._start_time = time()

    def dataset_shape(self) -> tuple:
        """(rows per episode, capacity): the released mt80 / mt30 datasets' (offline_trainer.py:53-55); for any other
        task set, episodes of cfg.episode_length steps (+1 reset row) in a buffer of cfg.buffer_size."""
        return _DATASETS.get(self.cfg.task, (int(self.cfg.episode_length) + 1, int(self.cfg.buffer_size)))

    def _load_dataset(self) -> None:
        T, capacity = self.dataset_shape()
        buffer_cfg = copy.deepcopy(self.cfg)
        buffer_cfg.episode_length, buffer_cfg.buffer_size, buffer_cfg.steps = T, capacity, capacity
        self.buffer = Buffer(buffer_cfg)
        for fp in self.data_files:
            data = torch.load(fp, weights_only=True)
            if data["reward"].shape[1] != T:
                raise ValueError(f"{fp}: episodes of {data['reward'].shape[1]} rows; the {self.cfg.task} task set "
                                 f"expects {T}")
            self.buffer.load({k: v for k, v in data.items() if k in _DATASET_FIELDS})
        expected = capacity // T
        if self.buffer.num_eps != expected:
            warnings.warn(f"the buffer holds {self.buffer.num_eps} episodes; the {self.cfg.task} task set has {expected}")

    def eval(self) -> dict:
        tasks = evaluate(self.agent, self.eval_envs, self.cfg.eval_episodes, eval_mode=True)["tasks"]
        out = {}
        for name in self.cfg.tasks:
            out[f"episode_reward+{name}"] = tasks[name].reward
            out[f"episode_success+{name}"] = tasks[name].success
        return out

    def train(self) -> None:
        cfg = self.cfg
        self._load_dataset()
        for i in range(cfg.steps):
            train_metrics = self.agent.update(self.buffer)
            if i % cfg.eval_freq == 0 or i % 10_000 == 0:
                metrics = {"iteration": i, "elapsed_time": time() - self._start_time}
                metrics.update(train_metrics)
                if i % cfg.eval_freq == 0:
                    metrics.update(self.eval())
                    if i > 0:
                        self.logger.save_agent(self.agent, identifier=f"{i}")
                self.logger.log(metrics, "pretrain")
        self.logger.finish(self.agent)
