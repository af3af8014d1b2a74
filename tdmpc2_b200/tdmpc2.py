"""TDMPC2 agent with the reference's inference surface, planning on the H100 kernels.

Drop-in for the inference half of the reference class `TDMPC2`
(tdmpc2/tdmpc2.py:10-206): `TDMPC2(cfg)`, `.model`, `.cfg`, `.device`,
`._prev_mean`, `.discount`, `.load()`, `.save()`, `.act()`, `.plan`, `._plan()`,
`._estimate_value()`, `._td_target()` keep their names, argument meaning and return shapes, so
`evaluate.py:57-80` of the reference runs unchanged on it (INTEGRATION.md), and so does the
no-grad block of `_update` (`model.encode` + `_td_target`, tdmpc2.py:259-264), and the policy update
`update_pi` (tdmpc2.py:208-239) with its `scale` (RunningScale) and `pi_optim`, and the whole training step
`update(buffer)` / `_update` (tdmpc2.py:259-346) with its `optim`, for state and pixel observations.  Call `sync_weights()` after
changing the model's parameters outside these methods.

New: an environments axis.  `obs [E, obs_dim]`, `t0 [E]`, `task [E]` plan E
independent environments in one call; E == 1 (1-D obs) is the reference API.
"""
from __future__ import annotations

import os
import weakref
from typing import Optional, Sequence, Union

import torch
import torch.nn.functional as F

from .config import Config, get_discount
from .planner import Noise, Planner, draw_noise, draw_shifts
from .scale import RunningScale
from .world_model import WorldModel, convert_legacy_checkpoint


class TDMPC2(torch.nn.Module):
    def __init__(self, cfg: Config, device: Union[str, torch.device, None] = None, engine: Optional[str] = None):
        super().__init__()
        self.cfg = cfg
        self.device = torch.device("cuda:0" if device is None else device)      # tdmpc2.py:20
        self.model = WorldModel(cfg).to(self.device)
        self.model.eval()                                                        # tdmpc2.py:32
        self.model._agent = weakref.ref(self)                                    # the model's methods share self.planner
        if not cfg.get("iterations_effective", False):
            self.cfg.iterations += 2 * int(cfg.action_dim >= 20)                # tdmpc2.py:34
            self.cfg.iterations_effective = True
        self.discount = torch.tensor(
            [get_discount(cfg, ep) for ep in cfg.episode_lengths], device=self.device
        ) if cfg.multitask else get_discount(cfg, cfg.episode_length)           # tdmpc2.py:35-37
        self.num_envs = int(cfg.get("num_envs", 1) or 1)
        shape = (cfg.horizon, cfg.action_dim) if self.num_envs == 1 else (self.num_envs, cfg.horizon, cfg.action_dim)
        self._prev_mean = torch.nn.Buffer(torch.zeros(*shape, device=self.device))   # tdmpc2.py:40
        self._engine = engine
        self._planner: Optional[Planner] = None
        self._weights_dirty = True
        self.generator: Optional[torch.Generator] = None     # None -> torch's default CUDA generator, like the reference
        self._use_graph = bool(cfg.get("cuda_graph", True))   # replay the launch chain as one CUDA graph (cfg.compile's role)
        # one environment: interleave the reference-order noise draws with the launches instead (TDMPC2_B200_E1_GRAPH=1: A/B knob)
        self._e1_interleaved = bool(cfg.get("e1_interleaved", True)) and os.environ.get("TDMPC2_B200_E1_GRAPH", "0") in ("", "0")
        # the policy update (tdmpc2.py:26-30,41): Adam over the `_pi.*` parameters, and the running Q scale
        self.scale = RunningScale(cfg, self.device)
        self._pi_keys = [k for k in self.model.keys() if k.startswith("_pi.")]
        self.pi_optim = torch.optim.Adam([self.model.tensor(k) for k in self._pi_keys], lr=cfg.lr, eps=1e-5,
                                         capturable=self.device.type == "cuda")
        # the world model's optimiser (tdmpc2.py:22-30): the reference's groups, in its order
        keys = self.model.keys()
        grp = lambda pfx: [k for k in keys if k.startswith(pfx)]
        self._wm_groups = [grp("_encoder."), grp("_dynamics."), grp("_reward."), grp("_termination.") if cfg.episodic else [],
                           grp("_Qs.params."), ["_task_emb.weight"] if cfg.multitask else []]
        self._wm_keys = [k for g in self._wm_groups for k in g]
        self.optim = torch.optim.Adam(
            [{"params": [self.model.tensor(k) for k in self._wm_groups[0]], "lr": cfg.lr * cfg.enc_lr_scale}]
            + [{"params": [self.model.tensor(k) for k in g]} for g in self._wm_groups[1:]],
            lr=cfg.lr, capturable=self.device.type == "cuda")

    # ------------------------------------------------------------------ planner plumbing
    @property
    def planner(self) -> Planner:
        if self._planner is None:
            self._planner = Planner(self.cfg, self.num_envs, self.device, engine=self._engine)
            self._weights_dirty = True
        if self._weights_dirty or self._planner.weights_version != self.model._version:
            self._planner.pack(self.model.state_dict())
            self._planner.weights_version = self.model._version
            self._weights_dirty = False
        return self._planner

    def sync_weights(self) -> None:
        """Call after modifying `self.model`'s parameters in place (an optimiser step, the Polyak update of the
        target Q ensemble): the online and target weights are re-packed before the next call that reads them."""
        self._weights_dirty = True
        self.model.sync_weights()

    @property
    def plan(self):
        # The reference wraps _plan in torch.compile(mode="reduce-overhead") (tdmpc2.py:45-55);
        # here the fused kernels are the compiled artefact, so `plan` is `_plan`.
        return self._plan

    def save(self, fp):
        torch.save({"model": self.model.state_dict()}, fp)                       # tdmpc2.py:72-79

    def load(self, fp):
        """tdmpc2.py:81-95: path or dict, optional {"model": ...} wrapper, legacy-key conversion."""
        if isinstance(fp, dict):
            state_dict = fp
        else:
            state_dict = torch.load(fp, map_location=self.device, weights_only=False)
        state_dict = state_dict["model"] if "model" in state_dict else state_dict
        state_dict = convert_legacy_checkpoint(self.model.state_dict(), dict(state_dict))
        self.model.load_state_dict(state_dict)
        self._weights_dirty = True

    # ------------------------------------------------------------------ inference API
    @torch.no_grad()
    def act(self, obs, t0=False, eval_mode=False, task=None):
        """tdmpc2.py:97-120.  obs [obs_dim] (CPU) -> action [A] (CPU); or batched
        obs [E, obs_dim], t0 bool | [E], task int | [E] -> [E, A]."""
        obs = obs.to(self.device, non_blocking=True)
        batched = obs.ndim == (4 if self.cfg.get("obs", "state") == "rgb" else 2)   # rgb: [C, 64, 64] per environment
        if not batched:
            obs = obs.unsqueeze(0)
        if task is not None and not torch.is_tensor(task):
            task = torch.tensor([task] if isinstance(task, int) else list(task), device=self.device)
        if self.cfg.mpc:
            out = self._plan(obs, t0=t0, eval_mode=eval_mode, task=task)
            return out.cpu()
        out = self._policy_action(obs, eval_mode=eval_mode, task=task)           # tdmpc2.py:116-120
        return (out if batched else out[0]).cpu()

    @torch.no_grad()
    def _policy_action(self, obs, eval_mode=False, task=None, eps: Optional[torch.Tensor] = None):
        """The non-MPC branch of act() (tdmpc2.py:116-120): a = pi(encode(obs)), or its mean in eval_mode
        (`info["mean"]` = tanh(mean), world_model.py:173).  Two row-mode launches, encode then pi with noise eps
        (zero noise gives the mean); the planner's state is not touched."""
        cfg, E, dev = self.cfg, self.num_envs, self.device
        rgb = cfg.get("obs", "state") == "rgb"
        obs = obs.to(dev, torch.float32)
        obs = (obs.reshape(E, *cfg.obs_shape["rgb"]) if rgb else obs.reshape(E, -1)).contiguous()
        taskv = None
        if cfg.multitask:
            if task is None:
                raise ValueError("multi-task model needs `task`")
            taskv = torch.as_tensor(task, device=dev).reshape(-1).to(torch.int32)
            taskv = taskv.expand(E).contiguous() if taskv.numel() == 1 else taskv.contiguous()
        pl = self.planner
        if rgb:                                                                     # ShiftAug's draw comes first (layers.py:55)
            shift = torch.randint(0, 7, (E, 2), device=dev, dtype=torch.float32, generator=self.generator)
            z = pl.encode_pixels(obs, shift)
        else:
            z = pl.wm_encode(obs, taskv)
        if eval_mode:
            eps = torch.zeros(E, cfg.action_dim, device=dev)
        elif eps is None:
            eps = torch.randn(E, cfg.action_dim, device=dev, generator=self.generator)
        else:
            eps = eps.to(dev, torch.float32).expand(E, cfg.action_dim).contiguous()
        return pl.wm_pi(z, taskv, eps)[0]

    @torch.no_grad()
    def _plan(self, obs, t0=False, eval_mode=False, task=None, noise: Optional[Noise] = None, return_trace=False):
        """tdmpc2.py:138-206 on the fused kernels.  obs [1|E, obs_dim] on self.device.
        Returns action [A] when planning a single environment (reference shape),
        else [E, A]."""
        cfg, E, dev = self.cfg, self.num_envs, self.device
        obs = obs.to(dev, torch.float32)
        if obs.ndim == (3 if cfg.get("obs", "state") == "rgb" else 1):
            obs = obs.unsqueeze(0)
        if obs.shape[0] != E:
            raise ValueError(f"obs has {obs.shape[0]} environments, agent was built for cfg.num_envs={E}")
        obs = obs.contiguous()
        if torch.is_tensor(t0):
            t0v = t0.to(dev).reshape(-1).to(torch.uint8)
            t0v = t0v.expand(E).contiguous() if t0v.numel() == 1 else t0v.contiguous()
        else:
            t0v = torch.full((E,), int(bool(t0)), dtype=torch.uint8, device=dev) if not isinstance(t0, (list, tuple)) \
                else torch.tensor([int(bool(x)) for x in t0], dtype=torch.uint8, device=dev)
        taskv = None
        if cfg.multitask:
            if task is None:
                raise ValueError("multi-task model needs `task`")
            taskv = torch.as_tensor(task, device=dev).reshape(-1).to(torch.int32)
            taskv = taskv.expand(E).contiguous() if taskv.numel() == 1 else taskv.contiguous()
        prev = self._prev_mean.reshape(E, cfg.horizon, cfg.action_dim).contiguous()
        trace = None
        if noise is None and not return_trace and self._use_graph:
            # steady state: replay the captured prologue -> I x iter -> epilogue chain (tdmpc2.py:45-55 replays a
            # `reduce-overhead` graph); noise is drawn into the graph's static buffers
            try:
                if E == 1 and self._e1_interleaved and not self.planner.philox:
                    # one environment draws in the reference's order (29 small launches for I = 8): issue each draw right
                    # before its consumer instead of all of them ahead of a graph replay (planner.plan_interleaved)
                    action, new_mean = self.planner.plan_interleaved(obs, taskv, t0v, prev, eval_mode=eval_mode,
                                                                     generator=self.generator)
                else:
                    action, new_mean = self.planner.plan_graphed(obs, taskv, t0v, prev, eval_mode=eval_mode,
                                                                 generator=self.generator)
            except RuntimeError as e:                      # capture unsupported here: keep the eager launch chain
                import warnings
                warnings.warn(f"CUDA-graph capture of the plan chain failed ({e}); launching eagerly")
                self._use_graph = False
                return self._plan(obs, t0=t0, eval_mode=eval_mode, task=task)
        else:
            if noise is None:
                noise = draw_noise(cfg, E, dev, eval_mode=eval_mode, generator=self.generator)
            elif eval_mode:
                noise = Noise(noise.prior, noise.r, noise.pi, noise.qidx, noise.expo, None, noise.shift)
            action, new_mean, trace = self.planner.plan(obs, taskv, t0v, prev, noise, trace=return_trace)
        self._prev_mean.copy_(new_mean.reshape(self._prev_mean.shape))           # tdmpc2.py:205
        out = action[0] if E == 1 else action
        return (out, trace) if return_trace else out

    def update_pi(self, zs, task, *, eps=None, qidx=None, dropout_mask=None):
        """tdmpc2.py:208-239 on the kernels: one forward launch (pi, then the online Q pair's average, writing a tape) and
        the backward chain of grad_kernels.cuh, which ADDS the gradients to `.grad` of the `_pi.*` parameters (and of
        `_task_emb.weight` in multi-task models) as autograd would; then torch's clip_grad_norm_ and pi_optim.step().
        zs [T, B, L] (detached), task [B] | int | None.  Draws from self.generator in the reference's order: eps
        ([T, B, A], pi's randn_like), then in train mode (`self.model.training`, as inside _update) the dropout masks of
        Q layer 0 -- one [T B, mlp_dim] draw per head for all num_q heads (the reference's vmap dropout stream is not
        replayed bit for bit) -- then qidx (randperm(num_q)[:2]).  `eps`, `qidx`, `dropout_mask` ([num_q, T, B,
        mlp_dim] of mask / (1 - p) values) pass them explicitly.  Returns the reference's info dict."""
        cfg, dev = self.cfg, self.device
        if dev.type != "cuda":
            raise RuntimeError("update_pi runs on the sm_90a kernels: the agent needs a CUDA device (there is no CPU fallback)")
        pl = self.planner
        if zs.ndim != 3 or zs.shape[-1] != cfg.latent_dim or zs.shape[0] < 1 or zs.shape[1] < 1:
            raise ValueError(f"zs must be [T, B, {cfg.latent_dim}]; got {tuple(zs.shape)}")
        if cfg.multitask and task is None:
            raise ValueError("multi-task model needs `task`")
        T, B = int(zs.shape[0]), int(zs.shape[1])
        R, A, M, g = T * B, cfg.action_dim, cfg.mlp_dim, self.generator
        z = zs.detach().to(dev, torch.float32).reshape(R, -1).contiguous()
        eps = (torch.randn(T, B, A, device=dev, generator=g) if eps is None else torch.as_tensor(eps, device=dev))
        if tuple(eps.shape) != (T, B, A):
            raise ValueError(f"eps must be [{T}, {B}, {A}]; got {tuple(eps.shape)}")
        eps = eps.to(torch.float32).reshape(R, A).contiguous()
        drop = None
        if dropout_mask is not None:
            drop = torch.as_tensor(dropout_mask, device=dev)
            if tuple(drop.shape) != (cfg.num_q, T, B, M):
                raise ValueError(f"dropout_mask must be [{cfg.num_q}, {T}, {B}, {M}]; got {tuple(drop.shape)}")
            drop = drop.to(torch.float32).contiguous()
        elif self.model.training and cfg.dropout > 0:       # nn.Dropout(cfg.dropout) of Q layer 0 (layers.py:104-108)
            keep = 1.0 - cfg.dropout
            drop = torch.empty(cfg.num_q, R, M, device=dev).bernoulli_(keep, generator=g).div_(keep)
        if qidx is None:
            qidx = torch.randperm(cfg.num_q, device=dev, generator=g)[:2]
        qidx = torch.as_tensor(qidx, device=dev).reshape(-1)
        if qidx.numel() != 2:
            raise ValueError(f"qidx must hold 2 head indices; got {qidx.numel()}")
        qidx = qidx.to(torch.int32).contiguous()
        taskv = self.model._task_rows(pl, task, (T, B))

        tape, _, q, lp = pl.pi_loss_forward(z, taskv, eps, qidx, drop)
        log_prob, log_pi = lp[:, :1], lp[:, :1] - lp[:, 1:]                 # world_model.py:166-176
        size = float(A) if taskv is None else self.model.tensor("_action_masks").sum(-1)[taskv.long()].unsqueeze(-1)
        entropy = (-log_pi).view(T, B, 1)
        scaled_entropy = (-log_pi * (log_prob * size / (log_pi + 1e-8))).view(T, B, 1)
        qs = q.view(T, B, 1)
        self.scale.update(qs[0])
        qs = self.scale(qs)
        rho = torch.pow(cfg.rho, torch.arange(T, device=dev))
        pi_loss = (-(cfg.entropy_coef * scaled_entropy + qs).mean(dim=(1, 2)) * rho).mean()

        params = [self.model.tensor(k) for k in self._pi_keys]
        for p in params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        emb = None
        if cfg.multitask:
            emb = self.model.tensor("_task_emb.weight")
            if emb.grad is None:
                emb.grad = torch.zeros_like(emb)
        pl.pi_loss_backward(self.model.tensor, tape, z, taskv, eps, qidx, drop, T, B, self.scale.value, cfg.entropy_coef,
                            cfg.rho, {k: p.grad for k, p in zip(self._pi_keys, params)}, None if emb is None else emb.grad)
        pi_grad_norm = torch.nn.utils.clip_grad_norm_(params, cfg.grad_clip_norm)
        self.pi_optim.step()
        self.pi_optim.zero_grad(set_to_none=True)
        self.sync_weights()
        return {"pi_loss": pi_loss.detach(), "pi_grad_norm": pi_grad_norm, "pi_entropy": entropy,
                "pi_scaled_entropy": scaled_entropy, "pi_scale": self.scale.value}

    @torch.no_grad()
    def _renorm_task_emb(self, taskv) -> None:
        """nn.Embedding(max_norm=1)'s lookup (world_model.py:21): the looked-up rows of `_task_emb.weight` with norm > 1
        are scaled by 1 / (norm + 1e-7) in place.  Device-side masks: no host synchronisation."""
        W = self.model.tensor("_task_emb.weight")
        n = torch.linalg.vector_norm(W, dim=-1, keepdim=True)
        hit = torch.zeros(W.shape[0], 1, dtype=torch.bool, device=W.device).index_fill_(0, taskv.long(), True)
        W.mul_(torch.where(hit & (n > 1), 1.0 / (n + 1e-7), torch.ones_like(n)))
        self.sync_weights()

    def update(self, buffer):
        """tdmpc2.py:335-346: one training step on `buffer.sample()` = (obs, action, reward, terminated, task)."""
        obs, action, reward, terminated, task = buffer.sample()
        kwargs = {}
        if task is not None:
            kwargs["task"] = task
        return self._update(obs, action, reward, terminated, **kwargs)

    def _update(self, obs, action, reward, terminated, task=None, *, td_eps=None, td_qidx=None, dropout_mask=None,
                pi_eps=None, pi_qidx=None, pi_dropout_mask=None, shift=None):
        """tdmpc2.py:259-333 on the kernels.  obs [H+1, B, obs_dim] (state) or [H+1, B, C, 64, 64] (pixels, any dtype,
        values 0..255), action [H, B, A], reward / terminated [H, B, 1], task [B] | None.  The latent rollout and the heads
        run as taped row launches (tdmpc2_wm_loss_forward), the backward chain of grad_kernels.cuh ADDS the gradients of
        the world-model loss to `.grad` as autograd would; then torch's clip_grad_norm_ and optim.step(), update_pi on the
        detached latents, and the Polyak update of the target Q ensemble.  Pixel models encode obs[0] with a taped conv
        forward into zs[0] (tdmpc2_pixel_encode_taped, tdmpc2_wm_loss_forward_latent), and dL/dz_0 runs through the conv
        backward of pixel_grad_kernels.cuh into `.grad` of `_encoder.rgb.*`.
        Draws from self.generator in the reference's order: pixel models' ShiftAug shifts of obs[1:] (H draws of (B, 2)),
        the TD target's pi noise and Q pair (`td_eps` [H, B, A], `td_qidx` [2]), pixel models' shift of obs[0], the
        dropout scale of Q layer 0 for the value loss (`dropout_mask` [num_q, H, B, mlp_dim] of mask / (1 - p) values;
        the reference's vmap dropout stream is not replayed bit for bit), then update_pi's own (`pi_eps`, `pi_qidx`,
        `pi_dropout_mask`, see update_pi).  `shift` [H+1, B, 2] passes the shifts explicitly, shift[t] belonging to
        obs[t].  Returns the reference's info dict."""
        cfg, dev = self.cfg, self.device
        rgb = cfg.get("obs", "state") == "rgb"
        if rgb and dev.type != "cuda":
            raise NotImplementedError("pixel `_update` runs on the sm_90a conv encoder kernels: no CPU fallback")
        if dev.type != "cuda":
            raise RuntimeError("_update runs on the sm_90a kernels: the agent needs a CUDA device (there is no CPU fallback)")
        A, L, M = cfg.action_dim, cfg.latent_dim, cfg.mlp_dim
        if rgb:
            C_in = cfg.obs_shape["rgb"][0]
            if obs.ndim != 5 or obs.shape[0] < 2 or obs.shape[1] < 1 or tuple(obs.shape[2:]) != (C_in, 64, 64):
                raise ValueError(f"obs must be [H + 1, B, {C_in}, 64, 64]; got {tuple(obs.shape)}")
        else:
            obs_dim = cfg.obs_shape["state"][0]
            if obs.ndim != 3 or obs.shape[0] < 2 or obs.shape[1] < 1 or obs.shape[2] != obs_dim:
                raise ValueError(f"obs must be [H + 1, B, {obs_dim}]; got {tuple(obs.shape)}")
        H, B = int(obs.shape[0]) - 1, int(obs.shape[1])
        for name, x, shape in (("action", action, (H, B, A)), ("reward", reward, (H, B, 1)), ("terminated", terminated, (H, B, 1))):
            if tuple(x.shape) != shape:
                raise ValueError(f"{name} must be {list(shape)}; got {tuple(x.shape)}")
            if not x.is_floating_point():
                raise ValueError(f"{name} must be a floating-point tensor; got {x.dtype}")
        if not rgb and not obs.is_floating_point():
            raise ValueError(f"obs must be a floating-point tensor; got {obs.dtype}")
        if shift is not None:
            if not rgb:
                raise ValueError("shift applies to pixel models (cfg.obs == 'rgb')")
            shift = torch.as_tensor(shift, device=dev)
            if tuple(shift.shape) != (H + 1, B, 2):
                raise ValueError(f"shift must be [{H + 1}, {B}, 2]; got {tuple(shift.shape)}")
            shift = shift.to(torch.float32)
        if cfg.multitask and task is None:
            raise ValueError("multi-task model needs `task`")
        drop = None
        if dropout_mask is not None:
            drop = torch.as_tensor(dropout_mask, device=dev)
            if tuple(drop.shape) != (cfg.num_q, H, B, M):
                raise ValueError(f"dropout_mask must be [{cfg.num_q}, {H}, {B}, {M}]; got {tuple(drop.shape)}")
        f32 = lambda x: x.detach().to(dev, torch.float32).contiguous()
        obs, action, reward, terminated = f32(obs), f32(action), f32(reward), f32(terminated)
        pl, g = self.planner, self.generator
        taskv = self.model._task_rows(pl, task, (H, B))
        if cfg.multitask:
            self._renorm_task_emb(taskv)                       # the first embedding lookup of the step

        # targets (tdmpc2.py:261-264)
        with torch.no_grad():
            if rgb:
                next_z = self.model.encode(obs[1:], task, shift=None if shift is None else shift[1:])
            else:
                next_z = self.model.encode(obs[1:], task)
            td_targets = self.model.td_target(next_z, reward, terminated, task, eps=td_eps, qidx=td_qidx)
        self.model.train()
        if rgb:                                              # ShiftAug's draw inside encode(obs[0]) (layers.py:55)
            shift0 = draw_shifts((B,), dev, g) if shift is None else shift[0]
        if drop is None and cfg.dropout > 0:                 # nn.Dropout(cfg.dropout) of Q layer 0 (layers.py:104-108)
            keep = 1.0 - cfg.dropout
            drop = torch.empty(cfg.num_q, H * B, M, device=dev).bernoulli_(keep, generator=g).div_(keep)
        elif drop is not None:
            drop = drop.to(torch.float32).reshape(cfg.num_q, H * B, M).contiguous()

        # latent rollout and heads (tdmpc2.py:269-285), on the kernels with a tape
        pl = self.planner
        act_rows = action.reshape(H * B, A)
        if rgb:
            zs = torch.empty(H + 1, B, L, device=dev, dtype=torch.float32)
            _, pix_tape = pl.encode_pixel_rows_taped(obs[0], shift0, out=zs[0])
            tape, zs, ql, rl, tl = pl.wm_loss_forward_latent(zs, act_rows, taskv, drop, H, B)
        else:
            tape, zs, ql, rl, tl = pl.wm_loss_forward(obs[0], act_rows, taskv, drop, H, B)
        rho = torch.pow(cfg.rho, torch.arange(H, device=dev, dtype=torch.float32))
        consistency_loss = (F.mse_loss(zs[1:], next_z, reduction="none").mean(dim=(1, 2)) * rho).sum() / H
        reward_loss = (_soft_ce(rl.view(H, B, -1), reward, cfg).mean(dim=(1, 2)) * rho).sum() / H
        value_loss = (_soft_ce(ql.view(cfg.num_q, H, B, -1), td_targets.unsqueeze(0).expand(cfg.num_q, H, B, 1), cfg)
                      .mean(dim=(2, 3)) * rho).sum() / (H * cfg.num_q)
        if cfg.episodic:
            termination_pred = tl.view(H, B, 1)
            termination_loss = F.binary_cross_entropy_with_logits(termination_pred, terminated)
        else:
            termination_loss = 0.
        total_loss = (cfg.consistency_coef * consistency_loss + cfg.reward_coef * reward_loss
                      + cfg.termination_coef * termination_loss + cfg.value_coef * value_loss)

        # backward, clip, step (tdmpc2.py:305-309); the embedding's .grad left by the previous update_pi is added to
        params = [self.model.tensor(k) for k in self._wm_keys]
        for p in params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        grads = {k: p.grad for k, p in zip(self._wm_keys, params)}
        if rgb:
            dz0 = pl.wm_loss_backward_latent(self.model.tensor, tape, act_rows, taskv, drop, H, B, zs, ql, rl, tl, next_z,
                                             reward, td_targets, terminated, grads)
            pl.pixel_encode_backward(self.model.tensor, pix_tape, obs[0], shift0, zs[0], dz0, grads)
        else:
            pl.wm_loss_backward(self.model.tensor, tape, obs[0], act_rows, taskv, drop, H, B, zs, ql, rl, tl, next_z, reward,
                                td_targets, terminated, grads)
        grad_norm = torch.nn.utils.clip_grad_norm_([p for p in self.model.parameters() if p.grad is not None],
                                                   cfg.grad_clip_norm)
        self.optim.step()
        self.optim.zero_grad(set_to_none=True)
        self.sync_weights()                                     # update_pi reads the stepped Q weights

        # policy update, target Q (tdmpc2.py:312-315)
        if cfg.multitask:
            self._renorm_task_emb(taskv)                       # update_pi's embedding lookup after the step
        pi_info = self.update_pi(zs.detach(), task, eps=pi_eps, qidx=pi_qidx, dropout_mask=pi_dropout_mask)
        self.model.soft_update_target_Q()
        self.model.eval()
        info = {"consistency_loss": consistency_loss, "reward_loss": reward_loss, "value_loss": value_loss,
                "termination_loss": termination_loss, "total_loss": total_loss, "grad_norm": grad_norm}
        if cfg.episodic:
            info.update(_termination_statistics(torch.sigmoid(termination_pred[-1]), terminated[-1]))
        info.update(pi_info)
        return {k: v.detach().mean() if isinstance(v, torch.Tensor) else torch.tensor(v) for k, v in info.items()}

    @torch.no_grad()
    def _td_target(self, next_z, reward, terminated, task, *, eps=None, qidx=None):
        """tdmpc2.py:242-257 as one fused launch: next_z [..., L], reward / terminated [..., 1] ->
        reward + discount * (1 - terminated) * Q(next_z, pi(next_z), 'min', target=True)  [..., 1].
        `eps` / `qidx` (default: drawn from self.generator in the reference's order) are pi's noise and the two heads."""
        return self.model.td_target(next_z, reward, terminated, task, eps=eps, qidx=qidx)

    @torch.no_grad()
    def _estimate_value(self, z, actions, task, eps_pi=None, qidx=None):
        """tdmpc2.py:122-136.  z [N, L], actions [H, N, A] -> [N, 1]  (E == 1), or
        z [E, N, L], actions [E, H, N, A] -> [E, N, 1]."""
        cfg, E, dev = self.cfg, self.num_envs, self.device
        single = z.ndim == 2
        zb = (z.unsqueeze(0) if single else z).to(dev, torch.float32).contiguous()
        ab = (actions.unsqueeze(0) if single else actions).to(dev, torch.float32).contiguous()
        if eps_pi is None:
            eps_pi = torch.randn(E, cfg.num_samples, cfg.action_dim, device=dev, generator=self.generator)
        if qidx is None:
            qidx = torch.rand(E, cfg.num_q, device=dev, generator=self.generator).argsort(-1)[:, :2]
        taskv = None
        if cfg.multitask:
            taskv = torch.as_tensor(task, device=dev).reshape(-1).to(torch.int32)
            taskv = taskv.expand(E).contiguous() if taskv.numel() == 1 else taskv.contiguous()
        v = self.planner.estimate_value(zb, ab, taskv, eps_pi.reshape(E, cfg.num_samples, cfg.action_dim).contiguous(),
                                        qidx.reshape(E, 2).to(torch.int32).contiguous())
        return v[0].unsqueeze(-1) if single else v.unsqueeze(-1)


def _two_hot(x, cfg):
    """math.py:58-71 on x [..., 1] -> [..., num_bins]."""
    x = torch.clamp(torch.sign(x) * torch.log(1 + torch.abs(x)), cfg.vmin, cfg.vmax).squeeze(-1)
    idx = torch.floor((x - cfg.vmin) / cfg.bin_size)
    off = ((x - cfg.vmin) / cfg.bin_size - idx).unsqueeze(-1)
    out = torch.zeros(*x.shape, cfg.num_bins, device=x.device, dtype=x.dtype)
    idx = idx.long().unsqueeze(-1)
    out = out.scatter(-1, idx, 1 - off)
    return out.scatter(-1, (idx + 1) % cfg.num_bins, off)


def _soft_ce(pred, target, cfg):
    """math.py:5-9: -(two_hot(target) . log_softmax(pred)) [..., 1]."""
    return -(_two_hot(target, cfg) * F.log_softmax(pred, dim=-1)).sum(-1, keepdim=True)


def _termination_statistics(pred, target, eps=1e-9):
    """math.py:97-109."""
    pred, target = pred.squeeze(-1), target.squeeze(-1)
    rate = target.sum() / len(target)
    tp = ((pred > 0.5) & (target == 1)).sum()
    fn = ((pred <= 0.5) & (target == 1)).sum()
    fp = ((pred > 0.5) & (target == 0)).sum()
    recall = tp / (tp + fn + eps)
    precision = tp / (tp + fp + eps)
    return {"termination_rate": rate, "termination_f1": 2 * (precision * recall) / (precision + recall + eps)}
