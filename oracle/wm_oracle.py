"""CPU oracle and golden fixtures of the world model's inference methods -- TEST INFRASTRUCTURE ONLY.

Extends oracle/plan_oracle.py (whose planning restatement is unchanged) to the methods a training script calls:

  WMOracle.encode / next / reward   <- WorldModel.encode / next / reward   common/world_model.py:103-130
  WMOracle.termination              <- WorldModel.termination              common/world_model.py:132-141
  WMOracle.pi (action, info)        <- WorldModel.pi                       common/world_model.py:144-184, math.py:12-29
  WMOracle.Q (all / min / avg, target=)  <- WorldModel.Q                   common/world_model.py:186-216
  WMOracle.td_target                <- TDMPC2._td_target                   tdmpc2/tdmpc2.py:242-257

with every random draw explicit (pi's randn_like -> `eps`, Q's randperm(num_q)[:2] -> `qidx`) and a per-row task
(the broadcast of WorldModel.task_emb, world_model.py:88-101: `task` has the inputs' leading shape).

`with_target_blend` gives synthetic models target Q weights that differ from the online ones; `attach_target_qs`
lets the reference harness run the reference's own `Q(..., target=True)` and `_td_target` on them.

    python -m oracle.wm_oracle [names]      # mints tests/golden/<name>.npz from the reference's own methods
"""
from __future__ import annotations

import copy
import os
import sys
import time
from typing import Dict, Optional

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.plan_oracle import OracleModel, _discount, two_hot_inv   # noqa: E402

QS = "_Qs.params."
TARGET = "_target_Qs_params."


def with_target_blend(cfg, sd: Dict[str, torch.Tensor], seed: int, tau: float = 0.3) -> Dict[str, torch.Tensor]:
    """A copy of `sd` whose target Q ensemble is a Polyak-style blend (lerp, as soft_update_target_Q does,
    world_model.py:76-80) of the online ensemble towards the Q ensemble of a second synthetic model (`seed`)."""
    from tdmpc2_b200.synth import synth_state_dict
    other = synth_state_dict(cfg, seed=seed, perturb=True)
    out = dict(sd)
    for k in sd:
        if k.startswith(TARGET):
            sub = k[len(TARGET):]
            out[k] = torch.lerp(sd[QS + sub].float(), other[QS + sub].float(), tau)
    return out


def attach_target_qs(agent, sd: Dict[str, torch.Tensor]) -> None:
    """Give a reference-harness agent (oracle/ref_harness.build_agent) `_target_Qs` built from `_target_Qs_params.*`
    and `_detach_Qs` (the online ensemble, world_model.py:40), so that the reference's Q(target=True / detach=True)
    and _td_target run unmodified."""
    m = agent.model
    tq = copy.deepcopy(m._Qs)
    with torch.no_grad():
        for k, p in tq.p.items():
            p.copy_(sd[TARGET + k.replace("/", ".")].to(p.device, p.dtype))
    m._target_Qs = tq
    m._detach_Qs = m._Qs


class WMOracle(OracleModel):
    """Row-wise restatement of the reference WorldModel's inference methods (CPU; fp32 unless `dtype` says otherwise).
    Inputs are cast to the model's dtype."""

    def _emb(self, task: torch.Tensor) -> torch.Tensor:
        rows = [self.task_emb(torch.zeros(1, 0, dtype=self.dtype), t)[0] for t in range(self.sd["_task_emb.weight"].shape[0])]
        return torch.stack(rows)[task.long()]                  # nn.Embedding(max_norm=1) lookup, world_model.py:21

    def _cat(self, x, task):
        return torch.cat([x, self._emb(task)], dim=-1) if self.cfg.multitask else x

    def encode(self, obs, task):
        return self._mlp("_encoder.state", self._cat(obs.to(self.dtype), task), "simnorm")

    def next(self, z, a, task):
        return self._mlp("_dynamics", torch.cat([self._cat(z.to(self.dtype), task), a.to(self.dtype)], dim=-1), "simnorm")

    def reward(self, z, a, task):
        return self._mlp("_reward", torch.cat([self._cat(z.to(self.dtype), task), a.to(self.dtype)], dim=-1), "none")

    def termination(self, z, task=None, unnormalized=False):
        x = self._mlp("_termination", z.to(self.dtype), "none")
        return x if unnormalized else torch.sigmoid(x)

    def pi(self, z, task, eps):
        """world_model.py:144-184 -> (action, info)."""
        z, eps = z.to(self.dtype), eps.to(self.dtype)
        mean, log_std = self._mlp("_pi", self._cat(z, task), "none").chunk(2, dim=-1)
        log_std = self.log_std_min + 0.5 * self.log_std_dif * (torch.tanh(log_std) + 1)         # math.py:12-13
        if self.cfg.multitask:
            m = self.sd["_action_masks"][task.long()]
            mean, log_std, eps = mean * m, log_std * m, eps * m
            size = self.sd["_action_masks"].sum(-1)[task.long()].unsqueeze(-1)
        else:
            size = eps.shape[-1]
        log_prob = (-0.5 * eps.pow(2) - log_std - 0.9189385175704956).sum(-1, keepdim=True)    # math.py:16-20
        scaled_log_prob = log_prob * size
        action = mean + eps * log_std.exp()
        mean, action = torch.tanh(mean), torch.tanh(action)                                    # math.py:23-29
        log_prob = log_prob - torch.log(F.relu(1 - action.pow(2)) + 1e-6).sum(-1, keepdim=True)
        entropy_scale = scaled_log_prob / (log_prob + 1e-8)
        return action, dict(mean=mean, log_std=log_std, action_prob=1., entropy=-log_prob,
                            scaled_entropy=-log_prob * entropy_scale)

    def Q(self, z, a, task, return_type="min", target=False, qidx=None):
        """world_model.py:186-216; detach=True reads the online weights (same tensors)."""
        x = torch.cat([self._cat(z.to(self.dtype), task), a.to(self.dtype)], dim=-1)
        prefix = TARGET[:-1] if target else QS[:-1]
        out = torch.stack([self._mlp(prefix, x, "none", head=h) for h in range(self.cfg.num_q)])
        if return_type == "all":
            return out
        Q = two_hot_inv(out[torch.as_tensor(qidx).long()], self.cfg)
        return Q.min(0).values if return_type == "min" else Q.sum(0) / 2

    def td_target(self, next_z, reward, terminated, task, eps, qidx):
        """tdmpc2.py:255-257."""
        reward, terminated = reward.to(self.dtype), terminated.to(self.dtype)
        action, _ = self.pi(next_z, task, eps)
        discount = (_discount(self.cfg, task.long(), self.dtype).unsqueeze(-1) if self.cfg.multitask
                    else _discount(self.cfg, None))
        return reward + discount * (1 - terminated) * self.Q(next_z, action, task, "min", target=True, qidx=qidx)


# --------------------------------------------------------------------------- golden fixtures
# name -> (workload, overrides, weight seed, target-blend seed, emb_scale, H, B, call seed)
CASES = {
    "tiny_wm": ("tiny", {}, 21, 121, 1.0, 3, 50, 600),
    "tiny_mt_wm": ("tiny-mt", {}, 22, 122, 60.0, 3, 50, 610),     # per-row tasks; emb_scale 60 exercises max_norm
    "tiny_episodic_wm": ("tiny", {"episodic": True}, 23, 123, 1.0, 3, 50, 620),
    "c1_dog5m_wm": ("c1", {}, 24, 124, 1.0, 3, 10, 630),           # 512-wide rows: the register LayerNorm path
    # corners of the shape envelope: an odd L + T and a one-dimensional task action space; 256-column heads on a latent
    # of one SimNorm group (a few rows each: tests/test_gpu_shape_envelope.py compares 200-row batches with the oracle)
    "tiny_mt_t5_wm": ("tiny-mt", {"task_dim": 5, "action_dims": [5, 1, 4, 2]}, 26, 126, 60.0, 1, 6, 650),
    "tiny_wide_heads_wm": ("tiny", {"action_dim": 128, "num_bins": 256, "latent_dim": 8}, 27, 127, 1.0, 1, 2, 660),
}
# Trained-scale cases (same fields), kept apart from CASES because fixed fp32 tolerances do not apply to them:
# TRAINED gives the synth.trained_scale (level, seed) applied after the target blend -- peaked two-hot heads with values
# of 1e3 - 1e4, saturated tanh, log-stds at their bounds
TRAINED_CASES = {"c1_sharp_wm": ("c1", {}, 25, 125, 1.0, 3, 10, 640)}
TRAINED = {"c1_sharp_wm": ("sharp", 225)}
OBS_SCALE = {"c1_sharp_wm": 30.0}
SUB_B = 8            # 'all' logits are recorded for batch columns [0, SUB_B) to keep the fixtures small


def case_model(name):
    """(cfg, state dict with a blended target ensemble) of a golden case."""
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    wl, over, wseed, tseed, emb_scale, H, B, _ = {**CASES, **TRAINED_CASES}[name]
    cfg = workload(wl, **over)
    sd = synth_state_dict(cfg, seed=wseed, perturb=True, emb_scale=emb_scale)
    if cfg.episodic:
        from oracle.plan_oracle import balance_termination
        balance_termination(cfg, sd)
    sd = with_target_blend(cfg, sd, tseed)
    if name in TRAINED:
        from tdmpc2_b200.synth import trained_scale
        sd = trained_scale(cfg, sd, *TRAINED[name])
    return cfg, sd


def case_inputs(cfg, H, B, seed, obs_scale=1.0):
    """obs [H, B, obs_dim], a [H, B, A], reward / terminated [H, B, 1], task [B] int64 or None."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(H, B, cfg.obs_shape["state"][0], generator=g) * obs_scale
    a = torch.rand(H, B, cfg.action_dim, generator=g) * 2 - 1
    reward = torch.randn(H, B, 1, generator=g)
    terminated = (torch.rand(H, B, 1, generator=g) < 0.3).float()
    task = torch.randint(0, len(cfg.tasks), (B,), generator=g) if cfg.multitask else None
    return obs, a, reward, terminated, task


def _record(agent, cfg, obs, a, reward, terminated, task, seed):
    """Every method of the reference's own WorldModel (+ _td_target) under torch.manual_seed(seed); the randn_like /
    randperm draws they make are captured."""
    m = agent.model
    draws = {"eps": [], "qidx": []}
    real_randn_like, real_randperm = torch.randn_like, torch.randperm

    def randn_like(x, *a_, **k):
        out = real_randn_like(x, *a_, **k)
        draws["eps"].append(out.clone())
        return out

    def randperm(n, *a_, **k):
        out = real_randperm(n, *a_, **k)
        draws["qidx"].append(out[:2].clone())
        return out

    torch.manual_seed(seed)
    torch.randn_like, torch.randperm = randn_like, randperm
    try:
        with torch.no_grad():
            r = {}
            r["z"] = z = m.encode(obs, task)
            r["next"] = m.next(z, a, task)
            r["reward"] = m.reward(z, a, task)
            r["pi_action"], info = m.pi(z, task)
            for k in ("mean", "log_std", "entropy", "scaled_entropy"):
                r["pi_" + k] = info[k]
            r["q_all"] = m.Q(z, a, task, return_type="all")
            r["q_min"] = m.Q(z, a, task, return_type="min")
            r["q_avg"] = m.Q(z, a, task, return_type="avg", detach=True)
            r["qt_all"] = m.Q(z, a, task, return_type="all", target=True)
            r["qt_min"] = m.Q(z, a, task, return_type="min", target=True)
            if cfg.episodic:
                r["term"] = m.termination(z, None)
                r["term_logit"] = m.termination(z, None, unnormalized=True)
            r["td"] = agent._td_target(z, reward, terminated, task)
    finally:
        torch.randn_like, torch.randperm = real_randn_like, real_randperm
    r["pi_eps"], r["td_eps"] = draws["eps"]
    r["q_min_qidx"], r["q_avg_qidx"], r["qt_min_qidx"], r["td_qidx"] = draws["qidx"]
    return r


def main(only=None):
    import numpy as np
    from oracle import ref_harness as rh
    from tdmpc2_b200.synth import state_dict_checksum
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, (wl, over, wseed, tseed, emb_scale, H, B, seed) in {**CASES, **TRAINED_CASES}.items():
        if only and name not in only:
            continue
        t = time.time()
        cfg, sd = case_model(name)
        agent = rh.build_agent(cfg, sd)
        attach_target_qs(agent, sd)
        obs, a, reward, terminated, task = case_inputs(cfg, H, B, seed, OBS_SCALE.get(name, 1.0))
        rec = dict(case=name, weight_checksum=state_dict_checksum(sd), torch_version=torch.__version__)
        if name in TRAINED:
            rec["trained_level"], rec["trained_seed"] = TRAINED[name]
        # the [H, B] batch (one full 128-row tile and a partial one for B = 50) and one 2-D row
        one = (obs[0, :1], a[0, :1], reward[0, :1], terminated[0, :1], None if task is None else task[:1])
        for pfx, (o, a_, rw, te, tk), s in (("b", (obs, a, reward, terminated, task), seed), ("r", one, seed + 1)):
            r = _record(agent, cfg, o, a_, rw, te, tk, s)
            for k, v in r.items():
                if k in ("q_all", "qt_all"):
                    v = v[..., :SUB_B, :] if pfx == "b" else v
                rec[f"{pfx}_{k}"] = v.numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **rec)
        print(f"{name}: {time.time() - t:.1f}s -> tests/golden/{name}.npz")


def load_case(name):
    """(cfg, sd, {"b": batch record, "r": one-row record}) of a fixture, inputs included."""
    import numpy as np
    from tdmpc2_b200.synth import state_dict_checksum
    f = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
    cfg, sd = case_model(name)
    if name in TRAINED:
        assert (str(f["trained_level"]), int(f["trained_seed"])) == TRAINED[name], "fixture minted with another transform"
    chk = state_dict_checksum(sd)
    assert abs(chk - float(f["weight_checksum"])) <= 1e-9 * abs(chk), "synthetic weights differ from the fixture's"
    wl, over, wseed, tseed, emb_scale, H, B, seed = {**CASES, **TRAINED_CASES}[name]
    obs, a, reward, terminated, task = case_inputs(cfg, H, B, seed, OBS_SCALE.get(name, 1.0))
    inputs = {"b": (obs, a, reward, terminated, task),
              "r": (obs[0, :1], a[0, :1], reward[0, :1], terminated[0, :1], None if task is None else task[:1])}
    recs = {}
    for pfx in ("b", "r"):
        d = {k[2:]: torch.from_numpy(f[k]) for k in f.files if k.startswith(pfx + "_")}
        d["obs"], d["a"], d["reward_in"], d["terminated"], d["task"] = inputs[pfx]
        recs[pfx] = d
    return cfg, sd, recs


if __name__ == "__main__":
    main(sys.argv[1:] or None)
