"""`WorldModel`: the reference's checkpoint surface as a FLAT parameter container with kernel-backed methods.

The planner's kernels read the weights straight from `state_dict()` (tdmpc2_b200/planner.py packs them into the
kernel layout), so this class holds tensors, not a module tree.  Every forward of the planning path runs in the fused
sm_90a kernels, including the non-MPC `act()` branch (TDMPC2.act -> row-mode encode and pi).  The reference's
methods -- `encode`, `next`, `reward`, `termination`, `pi`, `Q` (common/world_model.py:103-216) -- exist with its
signatures and shapes and run on the kernels' row mode (one launch per call, any [..., .] batch); `td_target` is
TDMPC2._td_target's fused launch.  They use the owning agent's Planner, or a one-environment Planner of their own; the
packed copies are re-packed after `load_state_dict()` / `sync_weights()` (the target ensemble at its next use).  There
is no CPU fallback: on the CPU the methods raise.

What is kept, because reference checkpoints and `evaluate.py` depend on it (SURVEY.md section 8(b)):

  * `state_dict()` / `load_state_dict()` with exactly the reference's keys: `_encoder.state.{i}.*` (or, for pixel
    observations, `_encoder.rgb.{2,4,6,8}.{weight,bias}`: layers.conv, layers.py:136-150), `_dynamics.{i}.*`,
    `_reward.{i}.*`, `_pi.{i}.*`, `_termination.{i}.*` (episodic), the stacked `_Qs.params.{i}.*` with their
    `_detach_Qs_params.*` aliases (same storage) and `_target_Qs_params.*` copies, tensordict's `__batch_size` /
    `__device` metadata entries, `_task_emb.weight`, `_action_masks`, `log_std_min`, `log_std_dif`;
  * the reference's initial values (common/init.py:4-17: trunc-normal sigma 0.02, zero bias, LayerNorm 1/0, embedding
    U(-0.02, 0.02); reward / Q output layers zeroed, world_model.py:32), drawn from torch's global generator;
  * `convert_legacy_checkpoint` for pre-torch.compile-API checkpoints (behaviour of layers.api_model_conversion,
    layers.py:167-221).
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from .planner import Planner, draw_shifts
from .synth import QS_PREFIXES, synth_state_dict

_LAYER_PARAM_NAMES = ("weight", "bias", "ln.weight", "ln.bias")
_BUFFER_KEYS = ("_action_masks", "log_std_min", "log_std_dif")
_META = ("__batch_size", "__device")


def _slot(key: str) -> str:
    """Attribute name under which a state-dict key is registered (module attribute names cannot contain dots)."""
    return "t__" + key.replace(".", "__")


class WorldModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        if cfg.get("obs", "state") not in ("state", "rgb"):
            raise NotImplementedError(f"Encoder for observation type {cfg.get('obs')} not implemented.")   # layers.py:163
        if cfg.get("obs", "state") == "rgb":
            if cfg.multitask:
                raise NotImplementedError("pixel observations are single-task in this build")
            if 16 * cfg.num_channels != cfg.latent_dim:
                raise ValueError("layers.conv flattens [num_channels, 4, 4]: latent_dim must be 16 * num_channels")
        seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())          # consumes torch's global RNG like nn.init does
        init = synth_state_dict(cfg, seed=seed)
        init["_reward.2.weight"].zero_()                                 # world_model.py:32
        init["_Qs.params.2.weight"].zero_()
        init["_target_Qs_params.2.weight"].zero_()
        self._agent = None           # weakref to the owning TDMPC2: its Planner serves the forward methods
        self._planner: Optional[Planner] = None
        self._version = 0            # bumped by load_state_dict / sync_weights: packed copies compare against it
        self._keys: List[str] = []                                       # owned tensors, in state-dict order
        for key, val in init.items():
            if key.startswith("_detach_Qs_params."):
                continue                                                 # alias of _Qs.params.* (world_model.py:40): not stored twice
            self._keys.append(key)
            if key in _BUFFER_KEYS:
                self.register_buffer(_slot(key), val.clone())
            else:
                self.register_parameter(_slot(key), nn.Parameter(val.clone(), requires_grad=not key.startswith("_target_Qs_params.")))

    # ------------------------------------------------------------------ tensor access by reference key
    def tensor(self, key: str) -> torch.Tensor:
        if key.startswith("_detach_Qs_params."):
            key = "_Qs.params." + key[len("_detach_Qs_params."):]
        return getattr(self, _slot(key))

    def keys(self) -> List[str]:
        """Reference state-dict keys (without tensordict's metadata entries), aliases included."""
        out = []
        for k in self._keys:
            out.append(k)
            if k.startswith("_Qs.params."):
                out.append("_detach_Qs_params." + k[len("_Qs.params."):])
        return out

    @property
    def total_params(self) -> int:
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def __repr__(self):
        return f"TD-MPC2 World Model (H100 planner build, flat parameter container)\nLearnable parameters: {self.total_params:,}"

    # ------------------------------------------------------------------ (de)serialisation with the reference's keys
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for k in self.keys():
            t = self.tensor(k)
            destination[prefix + k] = t if keep_vars else t.detach()
        dev = self.tensor(self._keys[0]).device
        for pfx in QS_PREFIXES:                                          # what tensordict's TensorDictParams serialises
            destination[prefix + pfx + "__batch_size"] = torch.Size([self.cfg.num_q])
            destination[prefix + pfx + "__device"] = dev

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        known = set()
        for k in self.keys():
            key = prefix + k
            known.add(key)
            if key not in state_dict:
                # the alias may be absent when its source is present (and the other way round): same storage
                twin = None
                if k.startswith("_detach_Qs_params."):
                    twin = prefix + "_Qs.params." + k[len("_detach_Qs_params."):]
                if twin is None or twin not in state_dict:
                    if strict:
                        missing_keys.append(key)
                continue
            if k.startswith("_detach_Qs_params.") and (prefix + "_Qs.params." + k[len("_detach_Qs_params."):]) in state_dict:
                continue                                                 # loaded through its source key
            src, dst = state_dict[key], self.tensor(k)
            if tuple(src.shape) != tuple(dst.shape):
                error_msgs.append(f"size mismatch for {key}: checkpoint {tuple(src.shape)} vs model {tuple(dst.shape)}")
                continue
            with torch.no_grad():
                dst.copy_(src)
        known |= {prefix + p + m for p in QS_PREFIXES for m in _META}
        if strict:
            unexpected_keys.extend(k for k in state_dict if k.startswith(prefix) and k not in known)
        self._version += 1                                               # packed copies are stale

    # ------------------------------------------------------------------ forward methods on the kernels
    def sync_weights(self) -> None:
        """Call after modifying parameters in place (an optimiser step, the Polyak update of `_target_Qs_params.*`):
        the kernels' packed copies are re-packed before the next call that reads them."""
        self._version += 1

    @torch.no_grad()
    def soft_update_target_Q(self) -> None:
        """world_model.py:82-86: Polyak-average `_target_Qs_params.*` towards the online `_Qs.params.*` by cfg.tau, in
        place, then mark the packed copies stale."""
        for k in self._keys:
            if k.startswith("_target_Qs_params."):
                self.tensor(k).lerp_(self.tensor("_Qs.params." + k[len("_target_Qs_params."):]), self.cfg.tau)
        self.sync_weights()

    def _kernels(self) -> Planner:
        """The Planner whose packed weights these methods run on: the owning agent's, or a one-environment planner of
        this model's own (created on first use; CUDA only -- there is no CPU fallback)."""
        agent = self._agent() if self._agent is not None else None
        if agent is not None:
            return agent.planner
        dev = self.tensor(self._keys[0]).device
        if dev.type != "cuda":
            raise RuntimeError("WorldModel's forward methods run on the sm_90a kernels: move the model to a CUDA device "
                               "(there is no CPU fallback)")
        if self._planner is None or self._planner.device != dev:
            self._planner = Planner(self.cfg, 1, dev)
        if self._planner.weights_version != self._version:
            self._planner.pack(self.state_dict())
            self._planner.weights_version = self._version
        return self._planner

    def _target_kernels(self) -> Planner:
        pl = self._kernels()
        if pl.target_version != self._version:
            pl.pack_target_q(self.state_dict())
            pl.target_version = self._version
        return pl

    def _generator(self) -> Optional[torch.Generator]:
        agent = self._agent() if self._agent is not None else None
        return agent.generator if agent is not None else None

    def _rows(self, pl: Planner, x) -> torch.Tensor:
        return x.to(pl.device, torch.float32).reshape(-1, x.shape[-1]).contiguous()

    def _task_rows(self, pl: Planner, task, lead) -> Optional[torch.Tensor]:
        """Per-row int32 task of a batch with leading shape `lead`: an int or [1] applies to every row, a [B] task to
        the rows of each leading [.., B] slice (task_emb's broadcast, world_model.py:88-101)."""
        if not self.cfg.multitask:
            return None
        t = torch.as_tensor(task, device=pl.device).reshape(-1).to(torch.int32)
        return t.expand(*lead).reshape(-1).contiguous()

    def encode(self, obs, task, *, shift: Optional[torch.Tensor] = None):
        """world_model.py:103-112: obs [..., obs_dim] -> z [..., L].  Pixel models (layers.py:36-59,136-150): frames
        [B, C, 64, 64] -> z [B, L], or [T, B, C, 64, 64] -> z [T, B, L] in one launch; `shift` [..., 2] (x, y) (default:
        ShiftAug's randint draws from the agent's generator, one (B, 2) draw per t, like the reference's slice loop)."""
        if self.cfg.get("obs", "state") == "rgb":
            return self._encode_rgb(obs, shift)
        pl = self._kernels()
        lead = obs.shape[:-1]
        return pl.wm_encode(self._rows(pl, obs), self._task_rows(pl, task, lead)).view(*lead, -1)

    def _encode_rgb(self, obs, shift):
        agent = self._agent() if self._agent is not None else None
        if agent is None and self.tensor(self._keys[0]).device.type != "cuda":
            raise NotImplementedError("pixel encoding runs on the sm_90a conv-encoder kernel: move the model to a CUDA "
                                      "device (there is no CPU fallback)")
        C_in = self.cfg.obs_shape["rgb"][0]
        if obs.ndim not in (4, 5) or tuple(obs.shape[-3:]) != (C_in, 64, 64):
            raise ValueError(f"pixel obs must be [B, {C_in}, 64, 64] or [T, B, {C_in}, 64, 64]; got {tuple(obs.shape)}")
        pl = self._kernels()
        lead = tuple(obs.shape[:-3])
        shift = draw_shifts(lead, pl.device, self._generator()) if shift is None else torch.as_tensor(shift)
        if tuple(shift.shape) != lead + (2,):
            raise ValueError(f"shift must be {list(lead) + [2]}; got {tuple(shift.shape)}")
        return pl.encode_pixel_rows(obs.reshape(-1, C_in, 64, 64), shift.reshape(-1, 2)).view(*lead, -1)

    def next(self, z, a, task):
        """world_model.py:114-121: z [..., L], a [..., A] -> z' [..., L]."""
        pl = self._kernels()
        lead = z.shape[:-1]
        return pl.wm_next(self._rows(pl, z), self._rows(pl, a), self._task_rows(pl, task, lead)).view(*lead, -1)

    def reward(self, z, a, task):
        """world_model.py:123-130: -> reward logits [..., num_bins]."""
        pl = self._kernels()
        lead = z.shape[:-1]
        return pl.wm_reward(self._rows(pl, z), self._rows(pl, a), self._task_rows(pl, task, lead)).view(*lead, -1)

    def termination(self, z, task, unnormalized=False):
        """world_model.py:132-141 (episodic models): -> sigmoid(logit), or the logit, [..., 1]."""
        assert task is None
        if not self.cfg.episodic:
            raise AttributeError("this model has no termination head (cfg.episodic is False)")
        pl = self._kernels()
        return pl.wm_termination(self._rows(pl, z), not unnormalized).view(*z.shape[:-1], 1)

    def pi(self, z, task, *, eps: Optional[torch.Tensor] = None):
        """world_model.py:144-184: -> (action [..., A], info).  `eps` (default: randn_like(mean) from the agent's
        generator, the reference's draw) is the policy noise."""
        pl = self._kernels()
        lead, A = z.shape[:-1], self.cfg.action_dim
        if eps is None:
            eps = torch.randn(*lead, A, device=pl.device, generator=self._generator())
        taskv = self._task_rows(pl, task, lead)
        act, mean, log_std, lp = pl.wm_pi(self._rows(pl, z), taskv, self._rows(pl, eps))
        log_prob, log_pi = lp[:, :1], lp[:, :1] - lp[:, 1:]                # gaussian log-prob; after squash (math.py:23-29)
        size = float(A) if taskv is None else self.tensor("_action_masks").sum(-1)[taskv.long()].unsqueeze(-1)
        entropy_scale = log_prob * size / (log_pi + 1e-8)
        info = {"mean": mean.view(*lead, A), "log_std": log_std.view(*lead, A), "action_prob": 1.,
                "entropy": (-log_pi).view(*lead, 1), "scaled_entropy": (-log_pi * entropy_scale).view(*lead, 1)}
        return act.view(*lead, A), info

    def _qidx(self, pl: Planner, qidx) -> torch.Tensor:
        if qidx is None:
            qidx = torch.randperm(self.cfg.num_q, device=pl.device, generator=self._generator())[:2]
        return torch.as_tensor(qidx, device=pl.device).reshape(2).to(torch.int32).contiguous()

    def Q(self, z, a, task, return_type='min', target=False, detach=False, *, qidx=None):
        """world_model.py:186-216: 'all' -> logits [num_q, ..., num_bins]; 'min' / 'avg' of two heads -> [..., 1].
        `detach` reads the online weights (the reference's _detach_Qs shares them); `qidx` (default:
        randperm(num_q)[:2] from the agent's generator) picks the two heads."""
        assert return_type in {'min', 'avg', 'all'}
        pl = self._target_kernels() if target else self._kernels()
        lead = z.shape[:-1]
        qi = None if return_type == 'all' else self._qidx(pl, qidx)
        out = pl.wm_q(self._rows(pl, z), self._rows(pl, a), self._task_rows(pl, task, lead), target, return_type, qi)
        return out.view(self.cfg.num_q, *lead, -1) if return_type == 'all' else out.view(*lead, 1)

    def td_target(self, next_z, reward, terminated, task, *, eps=None, qidx=None):
        """TDMPC2._td_target (tdmpc2.py:242-257) in one launch: reward + discount * (1 - terminated) *
        Q(next_z, pi(next_z), 'min', target=True).  Draws like the reference: pi's noise, then the Q heads."""
        pl = self._target_kernels()
        lead, A = next_z.shape[:-1], self.cfg.action_dim
        if eps is None:
            eps = torch.randn(*lead, A, device=pl.device, generator=self._generator())
        qi = self._qidx(pl, qidx)
        out = pl.td_target(self._rows(pl, next_z), self._rows(pl, reward), self._rows(pl, terminated),
                           self._task_rows(pl, task, lead), self._rows(pl, eps), qi)
        return out.view(*lead, 1)


def convert_legacy_checkpoint(target_state_dict, source_state_dict):
    """Accept checkpoints written by the reference's pre-torch.compile API
    (behaviour of layers.api_model_conversion, layers.py:167-221): there the Q
    ensemble was a ParameterList `_Qs.params.<n>` / `_target_Qs.params.<n>` with
    n = 4*layer + {0: weight, 1: bias, 2: ln.weight, 3: ln.bias}."""
    if "_detach_Qs_params.0.weight" in source_state_dict:
        return source_state_dict
    out = {}
    for key, val in source_state_dict.items():
        for old_prefix, new_prefixes in (("_Qs.params.", ("_Qs.params.", "_detach_Qs_params.")),
                                         ("_target_Qs.params.", ("_target_Qs_params.",))):
            if key.startswith(old_prefix):
                n = int(key[len(old_prefix):])
                name = f"{n // 4}.{_LAYER_PARAM_NAMES[n % 4]}"
                for npfx in new_prefixes:
                    out[npfx + name] = val
                break
        else:
            if "Qs" in key:
                raise AssertionError(f"key {key} contains 'Qs'")
            out[key] = val
    for pfx in QS_PREFIXES:
        for meta in _META:
            if pfx + meta in target_state_dict:
                out[pfx + meta] = target_state_dict[pfx + meta]
    for key in target_state_dict:
        if "Qs" in key and key not in out:
            raise AssertionError(f"key {key} not in converted checkpoint")
    for key in _BUFFER_KEYS:
        if key in target_state_dict:
            out[key] = target_state_dict[key]
    return out
