"""`WorldModel`: the reference's checkpoint surface as a FLAT parameter container.

The planner's kernels read the weights straight from `state_dict()` (tdmpc2_b200/planner.py packs them into the
kernel layout), so this class holds tensors, not a module tree: there are no eager forward methods here -- every
forward of the planning path (encode / next / reward / pi / Q / termination, reference common/world_model.py:103-216)
runs in the fused sm_90a kernels, including the non-MPC `act()` branch (TDMPC2.act -> the policy-prior kernel mode).

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

from typing import List

import torch
import torch.nn as nn

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
