"""Python host of the fused H100 planner: owns the device buffers (torch tensors)
and drives the C ABI (include/tdmpc2_b200.h).  torch is plumbing here -- device
memory, streams, RNG -- the planning math runs in the sm_90a kernels.

Call sequence of one `plan()` (reference tdmpc2.py:138-206):
    prologue  -> encode, policy-prior trajectories, mean/std init
    I x iter  -> sample, H-step latent rollout, value, top-k, MPPI refit
    epilogue  -> gumbel pick, exploration noise, clamp, _prev_mean update
"""
from __future__ import annotations

import os

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from . import _cabi
from .config import Config, get_discount


# GEMM engine of the fused kernels (include/tdmpc2_b200.h, tdmpc2_engine); TDMPC2_B200_ENGINE overrides.  "tcgen05" is the
# TMA + wgmma engine, "simt" the CUDA-core fp32 engine the tests compare it against.
ENGINES = {"tcgen05": _cabi.ENGINE_TCGEN05, "simt": _cabi.ENGINE_SIMT}
DEFAULT_ENGINE = os.environ.get("TDMPC2_B200_ENGINE", "tcgen05")


@dataclass
class Noise:
    """All random numbers of one batched plan() in reference draw order
    (SURVEY.md section 8(a)), ITERATION-major so that every CEM iteration reads one
    contiguous slab (no per-iteration copies):
    prior [E,H,P,A], r [I,E,H,N-P,A], pi [I,E,N,A], qidx [I,E,2] int32, expo [E,K],
    final [E,A] or None (eval_mode)."""
    prior: torch.Tensor
    r: torch.Tensor
    pi: torch.Tensor
    qidx: torch.Tensor
    expo: torch.Tensor
    final: Optional[torch.Tensor]
    shift: Optional[torch.Tensor] = None     # [E, 2] (x, y): ShiftAug's randint(0, 7) of pixel models, layers.py:55 (drawn first)

    @classmethod
    def from_env_major(cls, prior, r, pi, qidx, expo, final, device=None, shift=None) -> "Noise":
        """From the oracle's environment-major layout (r [E,I,...], pi [E,I,...], qidx [E,I,2])."""
        mv = lambda t: t if device is None else t.to(device)
        return cls(mv(prior).contiguous(), mv(r).transpose(0, 1).contiguous(), mv(pi).transpose(0, 1).contiguous(),
                   mv(qidx).to(torch.int32).transpose(0, 1).contiguous(), mv(expo).contiguous(),
                   None if final is None else mv(final).contiguous(),
                   None if shift is None else mv(shift).to(torch.float32).contiguous())

    def tensors(self):
        return [t for t in (self.prior, self.r, self.pi, self.qidx, self.expo, self.final, self.shift) if t is not None]


def alloc_noise(cfg: Config, num_envs: int, device, eval_mode: bool = False) -> Noise:
    """Uninitialised noise buffers of one plan() (the normal draws share ONE flat allocation so that a batched
    draw is a single Philox launch)."""
    H, N, P, A, I, K = (cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim,
                        cfg.iterations, cfg.num_elites)
    E = num_envs
    if cfg.get("rng", "torch") == "philox":      # declared non-parity mode: r / pi are generated inside the kernels
        nz = Noise(torch.empty(E, H, P, A, device=device, dtype=torch.float32), None, None,
                   torch.empty(I, E, 2, device=device, dtype=torch.int32), torch.empty(E, K, device=device, dtype=torch.float32),
                   None if eval_mode else torch.empty(E, A, device=device, dtype=torch.float32))
        if cfg.get("obs", "state") == "rgb":
            nz.shift = torch.empty(E, 2, device=device, dtype=torch.float32)
        return nz
    shapes = [(E, H, P, A), (I, E, H, N - P, A), (I, E, N, A)] + ([] if eval_mode else [(E, A)])
    sizes = [int(torch.Size(sh).numel()) for sh in shapes]
    pad = lambda n: (n + 63) // 64 * 64                     # keep every view 256-byte aligned
    flat = torch.empty(sum(pad(n) for n in sizes), device=device, dtype=torch.float32)
    views, off = [], 0
    for sh, n in zip(shapes, sizes):
        views.append(flat[off:off + n].view(sh))
        off += pad(n)
    nz = Noise(views[0], views[1], views[2], torch.empty(I, E, 2, device=device, dtype=torch.int32),
               torch.empty(E, K, device=device, dtype=torch.float32), None if eval_mode else views[3])
    nz._flat = flat
    if cfg.get("obs", "state") == "rgb":
        nz.shift = torch.empty(E, 2, device=device, dtype=torch.float32)
    return nz


def draw_noise(cfg: Config, num_envs: int, device, eval_mode: bool = False,
               generator: Optional[torch.Generator] = None, reference_order: Optional[bool] = None,
               out: Optional[Noise] = None) -> Noise:
    """Draw the planner's noise with torch's generator on `device`.

    reference_order (default: num_envs == 1): issue the draws one by one in the
    order and shapes of the reference's `_plan` (H x randn[P,A]; per iteration
    randn[H,N-P,A], randn[N,A], randperm(num_q); exponential_[K]; randn[A]) so a
    single-env agent consumes the generator exactly like the reference does.
    Otherwise each kind of draw is one batched call over all environments.
    """
    H, N, P, A, I, K = (cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim,
                        cfg.iterations, cfg.num_elites)
    E, g = num_envs, generator
    kw = dict(device=device, dtype=torch.float32, generator=g)
    if reference_order is None:
        reference_order = (E == 1)
    nz = out if out is not None else alloc_noise(cfg, E, device, eval_mode)
    if nz.shift is not None:      # ShiftAug inside encode(): the first draw of a reference _plan on pixels (layers.py:55)
        nz.shift.copy_(torch.randint(0, 7, (E, 2), device=device, dtype=torch.float32, generator=g))
    if nz.r is None:                       # in-kernel noise: only the small host-side draws remain
        nz.prior.normal_(generator=g)
        if nz.final is not None:
            nz.final.normal_(generator=g)
        nz.qidx.copy_(torch.rand(I, E, cfg.num_q, **kw).argsort(dim=-1)[..., :2])
        nz.expo.exponential_(generator=g)
        return nz
    if reference_order and E == 1:
        for t in range(H if P > 0 else 0):
            nz.prior[0, t] = torch.randn(P, A, **kw)
        for it in range(I):
            nz.r[it, 0] = torch.randn(H, N - P, A, **kw)
            nz.pi[it, 0] = torch.randn(N, A, **kw)
            nz.qidx[it, 0] = torch.randperm(cfg.num_q, device=device, generator=g)[:2].to(torch.int32)
        nz.expo.exponential_(generator=g)
        if not eval_mode:
            nz.final[0] = torch.randn(A, **kw)
        return nz
    flat = getattr(nz, "_flat", None)
    if flat is not None:
        flat.normal_(generator=g)                            # prior | r | pi | final: one launch
    else:
        for t in (nz.prior, nz.r, nz.pi) + (() if nz.final is None else (nz.final,)):
            t.normal_(generator=g)
    # randperm(num_q)[:2] per (iteration, env): the two smallest of num_q iid uniforms
    nz.qidx.copy_(torch.rand(I, E, cfg.num_q, **kw).argsort(dim=-1)[..., :2])
    nz.expo.exponential_(generator=g)
    return nz


def draw_shifts(lead, device, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """ShiftAug's random shifts (layers.py:55) for WorldModel.encode of pixel frames with leading shape `lead`: [B] -> one
    randint(0, 7) draw of (B, 2); [T, B] -> T draws of (B, 2) in order of t, because the reference encodes a 5-D batch
    slice by slice (world_model.py:110-111).  (x, y) pairs as fp32, shape [*lead, 2]."""
    kw = dict(device=device, dtype=torch.float32, generator=generator)
    if len(lead) == 1:
        return torch.randint(0, 7, (lead[0], 2), **kw)
    return torch.stack([torch.randint(0, 7, (lead[1], 2), **kw) for _ in range(lead[0])])


def discount_table(cfg: Config, device) -> torch.Tensor:
    """[num_tasks, H+1] fp32: the running `discount` of tdmpc2.py:125-132 after t steps.
    Single-task: a Python float product (double) cast to fp32 when it multiplies
    the fp32 reward tensor; multi-task: an fp32 tensor product."""
    H = cfg.horizon
    if cfg.multitask:
        g = torch.tensor([get_discount(cfg, ep) for ep in cfg.episode_lengths], dtype=torch.float32)
        cols, d = [torch.ones_like(g)], torch.ones_like(g)
        for _ in range(H):
            d = d * g
            cols.append(d)
        return torch.stack(cols, dim=1).contiguous().to(device)
    g, d, vals = get_discount(cfg, cfg.episode_length), 1, [1.0]
    for _ in range(H):
        d = d * g
        vals.append(d)
    return torch.tensor([vals], dtype=torch.float32, device=device)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _linear(struct, get, prefix: str, ln: bool):
    """A tdmpc2_linear / tdmpc2_linear_grad (`struct`) of the state-dict entries `prefix`.weight / .bias and, when the
    layer has a LayerNorm (`ln`), .ln.weight / .ln.bias; `get(key)` returns the tensor of a key."""
    keys = (".weight", ".bias") + ((".ln.weight", ".ln.bias") if ln else ())
    return struct(*[_ptr(get(prefix + k)) for k in keys])


def _conv(struct, get):
    """A tdmpc2_conv_weights / tdmpc2_conv_grads (`struct`) of the Conv2d modules of layers.conv, Sequential indices 2, 4,
    6, 8 (layers.py:136-150); `get(key)` returns the tensor of a state-dict key."""
    c = struct()
    for i, idx in enumerate((2, 4, 6, 8)):
        c.weight[i], c.bias[i] = _ptr(get(f"_encoder.rgb.{idx}.weight")), _ptr(get(f"_encoder.rgb.{idx}.bias"))
    return c


def _fp32_copies(sd: Dict[str, torch.Tensor], device, keep: list):
    """key -> a contiguous fp32 copy of sd[key] on `device`, appended to `keep` (the C call that reads it is asynchronous)."""
    def get(k):
        keep.append(sd[k].detach().to(device, torch.float32).contiguous())
        return keep[-1]
    return get


class Planner:
    """Owns one tdmpc2_planner handle plus its packed weights and workspace."""

    def __init__(self, cfg: Config, num_envs: int, device, engine: Optional[str] = None):
        self.lib = _cabi.load()                         # raises if the .so is missing
        self.cfg, self.E = cfg, int(num_envs)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _cabi.CabiError("the H100 planner needs a CUDA device; there is no CPU fallback")
        self.rgb = cfg.get("obs", "state") == "rgb"
        d = _cabi.Dims(
            num_envs=self.E, num_samples=cfg.num_samples, num_pi_trajs=cfg.num_pi_trajs, num_elites=cfg.num_elites,
            horizon=cfg.horizon, iterations=cfg.iterations, obs_dim=1 if self.rgb else cfg.obs_shape["state"][0],
            action_dim=cfg.action_dim, latent_dim=cfg.latent_dim, mlp_dim=cfg.mlp_dim, enc_dim=cfg.enc_dim,
            num_enc_layers=0 if self.rgb else cfg.num_enc_layers, task_dim=cfg.task_dim if cfg.multitask else 0,
            num_tasks=len(cfg.tasks) if cfg.multitask else 1, num_q=cfg.num_q, num_bins=cfg.num_bins,
            simnorm_dim=cfg.simnorm_dim, episodic=int(bool(cfg.episodic)), temperature=cfg.temperature,
            min_std=cfg.min_std, max_std=cfg.max_std, log_std_min=float(cfg.log_std_min),
            log_std_dif=float(cfg.log_std_max) - float(cfg.log_std_min))
        self._dims = d
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_planner_create(C.byref(d), C.byref(h)))
            self.h = h
            nb = C.c_size_t()
            _cabi.check(self.lib.tdmpc2_planner_packed_bytes(h, C.byref(nb)))
            self.packed = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
            _cabi.check(self.lib.tdmpc2_planner_workspace_bytes(h, C.byref(nb)))
            self.workspace = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
            _cabi.check(self.lib.tdmpc2_planner_bind(h, self.packed.data_ptr(), self.workspace.data_ptr()))
        self.pix = None
        if self.rgb:           # pixel observations: the conv encoder is its own small object (include/tdmpc2_b200.h)
            C_in = cfg.obs_shape["rgb"][0]
            pd = _cabi.PixelDims(in_channels=C_in, num_channels=cfg.num_channels, simnorm_dim=cfg.simnorm_dim)
            ph = C.c_void_p()
            with torch.cuda.device(self.device):
                _cabi.check(self.lib.tdmpc2_pixel_encoder_create(C.byref(pd), C.byref(ph)))
                nb = C.c_size_t()
                _cabi.check(self.lib.tdmpc2_pixel_encoder_workspace_bytes(ph, C.byref(nb)))
            self.pix = ph
            self.pix_ws = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
            self.pix_z = torch.empty(self.E, cfg.latent_dim, dtype=torch.float32, device=self.device)
            # ShiftAug's base grid, computed by torch.linspace exactly as the reference does (layers.py:50-51)
            eps = 1.0 / (64 + 2 * 3)
            self.pix_grid = torch.linspace(-1.0 + eps, 1.0 - eps, 64 + 2 * 3, device=self.device, dtype=torch.float32)[:64].contiguous()
            self._conv = None
        self.set_engine(engine)
        # arithmetic: 3 = fp32-parity (default); 1 = the declared NON-PARITY fast mode (see include/tdmpc2_b200.h)
        self.passes = int(os.environ.get("TDMPC2_B200_PASSES", cfg.get("passes", 3) or 3))
        _cabi.check(self.lib.tdmpc2_planner_set_passes(self.h, self.passes))
        # noise source: "torch" (default; the reference's draws, parity) or "philox" = the declared NON-PARITY throughput mode
        # (the two large noise tensors are generated inside the kernels: include/tdmpc2_b200.h, tdmpc2_plan_iter_rng)
        self.philox = cfg.get("rng", "torch") == "philox"
        self.rng_state = None
        if self.philox:
            seed = int(cfg.get("rng_seed", torch.initial_seed())) & ((1 << 63) - 1)
            self.rng_state = torch.tensor([seed, 0], dtype=torch.int64, device=self.device)   # {seed, plan counter}
        self._keep = []       # tensors referenced by in-flight async calls
        self.weights_version = None
        self._graphs = {}     # eval_mode -> captured launch chain + its static buffers
        self._e1_noise = {}   # eval_mode -> static noise buffers of plan_interleaved
        self._draw_stream = None
        self._graph_launches = 0
        self.target_blob = None      # target Q ensemble (tdmpc2_planner_bind_target_q), allocated by the first target op
        self.target_version = None
        self._tables = None          # discount powers and two-hot bins (pack)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.tdmpc2_planner_destroy(self.h)
                self.h = None
            if getattr(self, "pix", None):
                self.lib.tdmpc2_pixel_encoder_destroy(self.pix)
                self.pix = None
        except Exception:
            pass

    def set_engine(self, engine: Optional[str]) -> None:
        engine = engine or DEFAULT_ENGINE
        if engine not in ENGINES:
            raise ValueError(f"unknown engine {engine!r}: the engines are 'tcgen05' and 'simt'")
        _cabi.check(self.lib.tdmpc2_planner_set_engine(self.h, ENGINES[engine]))
        self.engine = engine
        # captured training steps of the owning agent (TDMPC2._update_graphed, cfg.compile): their launches name the engine
        self.update_graphs = {}

    @property
    def iter_engine(self) -> str:
        """The engine the planning launches run: "tcgen05" or "simt"."""
        return self.engine

    @property
    def launches(self) -> int:
        """Kernels of this library launched so far (graph replays count the launches they contain)."""
        return int(self.lib.tdmpc2_planner_launch_count(self.h)) + self._graph_launches

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------ weights
    def pack(self, sd: Dict[str, torch.Tensor]) -> None:
        """Pack a reference-layout state dict (tensors on any device) for the kernels."""
        cfg = self.cfg
        keep = []
        f = _fp32_copies(sd, self.device, keep)
        lin = lambda prefix: _linear(_cabi.Linear, f, prefix, prefix + ".ln.weight" in sd)
        W = _cabi.Weights()
        n = 0
        if self.rgb:       # the conv encoder reads these copies at every encode: they stay alive until the next pack
            self._conv_keep = []
            self._conv = _conv(_cabi.ConvWeights, _fp32_copies(sd, self.device, self._conv_keep))
        else:
            while f"_encoder.state.{n}.weight" in sd:
                W.enc[n] = lin(f"_encoder.state.{n}")
                n += 1
        W.num_enc = n
        for i in range(3):
            W.dynamics[i] = lin(f"_dynamics.{i}")
            W.reward[i] = lin(f"_reward.{i}")
            W.pi[i] = lin(f"_pi.{i}")
            W.qs[i] = lin(f"_Qs.params.{i}")
            if cfg.episodic:
                W.termination[i] = lin(f"_termination.{i}")      # world_model.py:28
        if cfg.multitask:
            W.task_emb, W.action_masks = _ptr(f("_task_emb.weight")), _ptr(f("_action_masks"))
        if self._tables is None:      # built once: torch.tensor() of host values is a synchronising copy
            self._tables = (discount_table(cfg, self.device),
                            torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, device=self.device, dtype=torch.float32))  # math.py:80
        disc, bins = self._tables
        W.discount_pow, W.bins = _ptr(disc), _ptr(bins)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            _cabi.check(self.lib.tdmpc2_pack_weights(self.h, C.byref(W), stream.cuda_stream))
            for t in keep:            # `keep` tensors may be freed now: their memory is not reused before the pack ran
                t.record_stream(stream)

    # ------------------------------------------------------------------ hot path
    def prologue(self, obs, task, t0, prev_mean, noise_prior, z=None) -> None:
        """obs [E, obs_dim], or obs None and z [E, L] the latent given in place of encode(obs) (pixel models)."""
        self._keep = [obs, z, task, t0, prev_mean, noise_prior]
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_plan_prologue(self.h, _ptr(obs), _ptr(z), _ptr(task), _ptr(t0), _ptr(prev_mean),
                                                      _ptr(noise_prior), self._stream()))

    def _prologue_obs(self, obs, shift, task, t0, prev_mean, noise_prior) -> None:
        """prologue() on the planning chain's observations: pixel models encode the frames (ShiftAug shifts `shift`) into
        the static pix_z that a captured graph reads, and pass that as z."""
        z = self.encode_pixel_rows(obs, shift, out=self.pix_z) if self.rgb else None
        self.prologue(None if self.rgb else obs, task, t0, prev_mean, noise_prior, z=z)

    def encode_pixel_rows(self, frames, shift, out=None) -> torch.Tensor:
        """z = encode(obs) for any number of pixel frames in one launch: frames [R, C, 64, 64] (any dtype, values 0..255),
        shift [R, 2] (x, y) -> z [R, L], written to `out` (a contiguous [R, L] fp32 tensor) or to a fresh tensor."""
        return self._pixel_encode(frames, shift, out, taped=False)[0]

    def encode_pixel_rows_taped(self, frames, shift, out=None):
        """encode_pixel_rows that also keeps the activations the conv backward needs: -> (z [R, L], tape).  z is
        bit-identical to encode_pixel_rows's."""
        return self._pixel_encode(frames, shift, out, taped=True)

    def _pixel_encode(self, frames, shift, out, taped: bool):
        if self.pix is None or self._conv is None:
            raise _cabi.CabiError("pixel encoding needs a cfg.obs == 'rgb' planner with packed weights")
        frames, shift, R = self._pixel_rows(frames, shift)
        z = self._rows_out(R, self.cfg.latent_dim) if out is None else out
        tape = self._scratch(self.lib.tdmpc2_pixel_encode_tape_bytes, self.pix, R) if taped else None
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_pixel_encode(self.pix, self.pix_ws.data_ptr(), C.byref(self._conv), _ptr(frames),
                                                     _ptr(shift), _ptr(self.pix_grid), R, _ptr(z), _ptr(tape), self._stream()))
        return z, tape

    def _pixel_rows(self, frames, shift):
        frames = frames.to(self.device, torch.float32).contiguous()      # ShiftAug's x.float() (layers.py:44)
        shift = shift.to(self.device, torch.float32).contiguous()
        R = frames.shape[0]
        if frames.ndim != 4 or tuple(frames.shape[1:]) != (self.cfg.obs_shape["rgb"][0], 64, 64) or tuple(shift.shape) != (R, 2):
            raise ValueError(f"frames must be [R, {self.cfg.obs_shape['rgb'][0]}, 64, 64] and shift [R, 2]; got "
                             f"{tuple(frames.shape)} and {tuple(shift.shape)}")
        return frames, shift, R

    def pixel_encode_backward(self, tensor, tape, frames, shift, z, dz, grads) -> None:
        """Adds dL/dparameter of the conv encoder to `grads` (the `.grad` tensors of `_encoder.rgb.{2,4,6,8}.{weight,bias}`
        by state-dict key), given dz = dL/dz [R, L] and the taped forward's tape and z on the same frames and shifts.
        `tensor(key)` returns the model's fp32 tensor of a state-dict key."""
        if self.pix is None:
            raise _cabi.CabiError("pixel_encode_backward needs a cfg.obs == 'rgb' planner")
        frames, shift, R = self._pixel_rows(frames, shift)
        W, G = _conv(_cabi.ConvWeights, tensor), _conv(_cabi.ConvGrads, grads.__getitem__)
        z, dz = z.reshape(R, -1).contiguous(), dz.reshape(R, -1).contiguous()
        ws = self._scratch(self.lib.tdmpc2_pixel_backward_workspace_bytes, self.pix, R)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_pixel_encode_backward(self.pix, C.byref(W), _ptr(frames), _ptr(shift), _ptr(self.pix_grid),
                                                              R, _ptr(tape), _ptr(z), _ptr(dz), C.byref(G), _ptr(ws),
                                                              self._stream()))

    def iterate(self, noise_r, noise_pi, qidx, values_out=None, elite_idx_out=None) -> None:
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_plan_iter(self.h, _ptr(noise_r), _ptr(noise_pi), _ptr(qidx),
                                                  _ptr(values_out), _ptr(elite_idx_out), self._stream()))

    def iterate_rng(self, iteration: int, qidx, values_out=None, elite_idx_out=None) -> None:
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_plan_iter_rng(self.h, _ptr(self.rng_state), int(iteration), _ptr(qidx),
                                                      _ptr(values_out), _ptr(elite_idx_out), self._stream()))

    def epilogue(self, expo, noise_final, action_out, prev_mean_out, pick_out=None) -> None:
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_plan_epilogue(self.h, _ptr(expo), _ptr(noise_final), _ptr(action_out),
                                                      _ptr(prev_mean_out), _ptr(pick_out), self._stream()))

    def get_state(self) -> Dict[str, torch.Tensor]:
        cfg, E = self.cfg, self.E
        kw = dict(device=self.device, dtype=torch.float32)
        out = dict(mean=torch.empty(E, cfg.horizon, cfg.action_dim, **kw),
                   std=torch.empty(E, cfg.horizon, cfg.action_dim, **kw),
                   z=torch.empty(E, cfg.latent_dim, **kw),
                   pi_actions=torch.zeros(E, cfg.horizon, cfg.num_pi_trajs, cfg.action_dim, **kw),
                   score=torch.empty(E, cfg.num_elites, **kw))
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_plan_get_state(self.h, _ptr(out["mean"]), _ptr(out["std"]), _ptr(out["z"]),
                                                       _ptr(out["pi_actions"]), _ptr(out["score"]), self._stream()))
        return out

    def _launch_chain(self, obs, task, t0, prev_mean, noise: Noise, action, new_mean, tr=None) -> None:
        """prologue -> I x iter -> epilogue on the current stream (10 launches for I = 6)."""
        cfg, E, dev = self.cfg, self.E, self.device
        self._prologue_obs(obs, noise.shift, task, t0, prev_mean, noise.prior)
        if tr is not None:
            st = self.get_state()
            tr["z"], tr["pi_actions"] = st["z"], st["pi_actions"]
        for it in range(cfg.iterations):
            qi = noise.qidx[it]
            nr, npi = (None, None) if self.philox else (noise.r[it], noise.pi[it])   # contiguous slabs of the [I, E, ...] tensors
            if tr is not None:
                v, ei = torch.empty(E, cfg.num_samples, device=dev), torch.empty(E, cfg.num_elites, device=dev, dtype=torch.int64)
                if self.philox:
                    self.iterate_rng(it, qi, v, ei)
                else:
                    self.iterate(nr, npi, qi, v, ei)
                tr["values"][:, it], tr["elite_idx"][:, it] = v, ei
                st = self.get_state()
                tr["iter_mean"].append(st["mean"]); tr["iter_std"].append(st["std"])
            elif self.philox:
                self.iterate_rng(it, qi)
            else:
                self.iterate(nr, npi, qi)
        if tr is not None:
            tr["score"] = self.get_state()["score"]
            tr["iter_mean"], tr["iter_std"] = torch.stack(tr["iter_mean"], 1), torch.stack(tr["iter_std"], 1)
        self.epilogue(noise.expo, noise.final, action, new_mean, tr["pick"] if tr is not None else None)

    def plan(self, obs, task, t0, prev_mean, noise: Noise, trace: bool = False):
        """One batched plan().  obs [E,obs_dim] f32, task [E] int32 | None, t0 [E] uint8,
        prev_mean [E,H,A] f32 (all on self.device, contiguous).  Returns (action [E,A],
        new prev_mean [E,H,A], trace dict | None)."""
        cfg, E, dev = self.cfg, self.E, self.device
        for t in noise.tensors():
            if not t.is_contiguous():
                raise ValueError("noise tensors must be contiguous (iteration-major: see planner.Noise)")
        if self.philox:
            self.rng_state[1] += 1                          # a fresh noise stream per plan()
        elif noise.r.shape[:2] != (cfg.iterations, E) or noise.pi.shape[:2] != (cfg.iterations, E):
            raise ValueError("noise.r / noise.pi must be [iterations, num_envs, ...] (Noise.from_env_major converts)")
        action = torch.empty(E, cfg.action_dim, device=dev, dtype=torch.float32)
        new_mean = torch.empty(E, cfg.horizon, cfg.action_dim, device=dev, dtype=torch.float32)
        tr = None
        if trace:
            tr = dict(values=torch.empty(E, cfg.iterations, cfg.num_samples, device=dev),
                      elite_idx=torch.empty(E, cfg.iterations, cfg.num_elites, device=dev, dtype=torch.int64),
                      iter_mean=[], iter_std=[], pick=torch.empty(E, device=dev, dtype=torch.int32))
        self._launch_chain(obs, task, t0, prev_mean, noise, action, new_mean, tr)
        return action, new_mean, tr

    # ------------------------------------------------------------------ CUDA-graph replay of the launch chain
    def plan_graphed(self, obs, task, t0, prev_mean, eval_mode: bool = False,
                     generator: Optional[torch.Generator] = None):
        """plan() for the steady state (reference tdmpc2.py:45-55 replays a `reduce-overhead` CUDA graph): the
        prologue -> I x iter -> epilogue chain is captured ONCE per eval_mode over static buffers and replayed; the
        noise is drawn into the static buffers before every replay (batched draws unless E == 1, see draw_noise).
        Returns (action [E,A], new prev_mean [E,H,A]) -- fresh tensors, the static outputs are copied out."""
        cfg, E, dev = self.cfg, self.E, self.device
        key = bool(eval_mode)
        st = self._graphs.get(key)
        if st is None:
            st = self._capture(key)
        st["obs"].copy_(obs, non_blocking=True)
        st["t0"].copy_(t0, non_blocking=True)
        st["prev"].copy_(prev_mean, non_blocking=True)
        if st["task"] is not None:
            st["task"].copy_(task, non_blocking=True)
        draw_noise(cfg, E, dev, eval_mode=eval_mode, generator=generator, out=st["noise"])
        if self.philox:
            self.rng_state[1] += 1                          # device-side counter: the graph's kernels read it
        st["graph"].replay()
        self._graph_launches += st["launches"]
        return st["action"].clone(), st["new_mean"].clone()

    def plan_interleaved(self, obs, task, t0, prev_mean, eval_mode: bool = False,
                         generator: Optional[torch.Generator] = None):
        """plan() of ONE environment in the reference's draw order (draw_noise, reference_order) with the draws off the
        critical path.  A reference-order call makes 2 + H + 3 I small generator launches (0.6 ms of host time for
        I = 8, and as many tiny kernels): ahead of a graph replay they delay the kernels by that much.  Here the host
        issues each iteration's draws on a side stream right before that iteration's launch; the kernels (0.5 ms each
        at E = 1) are far slower than the host, so the side stream runs an iteration ahead and the main stream sees
        back-to-back planner kernels.  Same generator consumption (the Philox offset advances at call time, whatever the
        stream), same kernels, same results as draw_noise() + plan()."""
        cfg, dev = self.cfg, self.device
        if self.E != 1 or self.philox:
            raise ValueError("plan_interleaved is the one-environment, torch-noise path")
        H, N, P, A, I = cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.iterations
        key = bool(eval_mode)
        nz = self._e1_noise.get(key)
        if nz is None:
            nz = self._e1_noise[key] = alloc_noise(cfg, 1, dev, eval_mode)
        if self._draw_stream is None:
            self._draw_stream = torch.cuda.Stream(device=dev)
        main, side = torch.cuda.current_stream(dev), self._draw_stream
        kw = dict(device=dev, dtype=torch.float32, generator=generator)
        action = torch.empty(1, A, device=dev, dtype=torch.float32)
        new_mean = torch.empty(1, H, A, device=dev, dtype=torch.float32)
        side.wait_stream(main)                        # earlier readers of the static noise buffers are done
        with torch.cuda.stream(side):
            if nz.shift is not None:                                                  # layers.py:55
                nz.shift.copy_(torch.randint(0, 7, (1, 2), device=dev, dtype=torch.float32, generator=generator))
            for t in range(H if P > 0 else 0):                                        # tdmpc2.py:153
                nz.prior[0, t] = torch.randn(P, A, **kw)
            main.wait_event(side.record_event())
        self._prologue_obs(obs, nz.shift, task, t0, prev_mean, nz.prior)
        for it in range(I):
            with torch.cuda.stream(side):
                nz.r[it, 0] = torch.randn(H, N - P, A, **kw)                          # tdmpc2.py:175
                nz.pi[it, 0] = torch.randn(N, A, **kw)                                # world_model.py:166 via tdmpc2.py:134
                nz.qidx[it, 0] = torch.randperm(cfg.num_q, device=dev, generator=generator)[:2].to(torch.int32)
                main.wait_event(side.record_event())
            self.iterate(nz.r[it], nz.pi[it], nz.qidx[it])
        with torch.cuda.stream(side):
            nz.expo.exponential_(generator=generator)                                 # math.py:44 gumbel_softmax_sample
            if not eval_mode:
                nz.final[0] = torch.randn(A, **kw)                                    # tdmpc2.py:203
            main.wait_event(side.record_event())
        self.epilogue(nz.expo, nz.final, action, new_mean)
        return action, new_mean

    def _capture(self, eval_mode: bool):
        cfg, E, dev = self.cfg, self.E, self.device
        f32 = dict(device=dev, dtype=torch.float32)
        obs_shape = tuple(cfg.obs_shape["rgb"]) if self.rgb else (cfg.obs_shape["state"][0],)
        st = dict(obs=torch.zeros(E, *obs_shape, **f32), t0=torch.ones(E, device=dev, dtype=torch.uint8),
                  prev=torch.zeros(E, cfg.horizon, cfg.action_dim, **f32),
                  task=torch.zeros(E, device=dev, dtype=torch.int32) if cfg.multitask else None,
                  noise=alloc_noise(cfg, E, dev, eval_mode), action=torch.empty(E, cfg.action_dim, **f32),
                  new_mean=torch.empty(E, cfg.horizon, cfg.action_dim, **f32))
        draw_noise(cfg, E, dev, eval_mode=eval_mode, out=st["noise"], reference_order=False)
        args = (st["obs"], st["task"], st["t0"], st["prev"], st["noise"], st["action"], st["new_mean"])
        self._launch_chain(*args)                      # eager warm-up: lazy function attributes are set outside capture
        torch.cuda.current_stream(dev).synchronize()
        n0 = self.launches
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._launch_chain(*args)
        st["graph"], st["launches"] = g, self.launches - n0
        self._graph_launches -= st["launches"]         # the capture pass itself launched nothing
        self._graphs[eval_mode] = st
        return st

    # ------------------------------------------------------------------ world-model methods on a flat batch of rows
    # Inputs are [rows, .] fp32 and task [rows] int32 | None, contiguous on self.device; outputs are fresh tensors.
    def pack_target_q(self, sd: Dict[str, torch.Tensor]) -> None:
        """Pack `_target_Qs_params.*` of a reference-layout state dict into the target blob (allocated on first use)."""
        with torch.cuda.device(self.device):
            if self.target_blob is None:
                nb = C.c_size_t()
                _cabi.check(self.lib.tdmpc2_planner_target_q_bytes(self.h, C.byref(nb)))
                blob = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
                _cabi.check(self.lib.tdmpc2_planner_bind_target_q(self.h, blob.data_ptr()))
                self.target_blob = blob
            keep, lins = [], (_cabi.Linear * 3)()
            f = _fp32_copies(sd, self.device, keep)
            for i in range(3):
                pfx = f"_target_Qs_params.{i}"
                lins[i] = _linear(_cabi.Linear, f, pfx, pfx + ".ln.weight" in sd)
            stream = torch.cuda.current_stream(self.device)
            _cabi.check(self.lib.tdmpc2_pack_target_q(self.h, lins, stream.cuda_stream))
            for t in keep:            # `keep` tensors may be freed now: their memory is not reused before the pack ran
                t.record_stream(stream)

    def _rows_out(self, *shape) -> torch.Tensor:
        return torch.empty(*shape, device=self.device, dtype=torch.float32)

    def _scratch(self, query, *args) -> torch.Tensor:
        """An fp32 tape or workspace of the size a `*_bytes` query of the C ABI reports for `args`."""
        nb = C.c_size_t()
        _cabi.check(query(*args, C.byref(nb)))
        return torch.empty(nb.value // 4, device=self.device, dtype=torch.float32)

    def wm_encode(self, obs, task) -> torch.Tensor:
        z = self._rows_out(obs.shape[0], self.cfg.latent_dim)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_encode(self.h, _ptr(obs), _ptr(task), obs.shape[0], _ptr(z), self._stream()))
        return z

    def wm_next(self, z, a, task) -> torch.Tensor:
        out = self._rows_out(z.shape[0], self.cfg.latent_dim)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_next(self.h, _ptr(z), _ptr(a), _ptr(task), z.shape[0], _ptr(out), self._stream()))
        return out

    def wm_reward(self, z, a, task) -> torch.Tensor:
        out = self._rows_out(z.shape[0], self.cfg.num_bins)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_reward(self.h, _ptr(z), _ptr(a), _ptr(task), z.shape[0], _ptr(out), self._stream()))
        return out

    def wm_termination(self, z, sigmoid: bool) -> torch.Tensor:
        out = self._rows_out(z.shape[0], 1)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_termination(self.h, _ptr(z), z.shape[0], int(bool(sigmoid)), _ptr(out),
                                                       self._stream()))
        return out

    def wm_pi(self, z, task, eps):
        """-> action, tanh(mean), log_std [rows, A] and [rows, 2] = (gaussian log-prob, sum of the squash terms)."""
        R, A = z.shape[0], self.cfg.action_dim
        act, mean, ls, lp = self._rows_out(R, A), self._rows_out(R, A), self._rows_out(R, A), self._rows_out(R, 2)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_pi(self.h, _ptr(z), _ptr(task), _ptr(eps), R, _ptr(act), _ptr(mean), _ptr(ls),
                                              _ptr(lp), self._stream()))
        return act, mean, ls, lp

    def wm_q(self, z, a, task, target: bool, return_type: str, qidx=None) -> torch.Tensor:
        """return_type 'all' -> logits [num_q, rows, B]; 'min' / 'avg' of heads qidx [2] int32 -> [rows, 1]."""
        R = z.shape[0]
        rt = {"all": _cabi.Q_ALL, "min": _cabi.Q_MIN, "avg": _cabi.Q_AVG}[return_type]
        out = self._rows_out(self.cfg.num_q, R, self.cfg.num_bins) if rt == _cabi.Q_ALL else self._rows_out(R, 1)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_q(self.h, _ptr(z), _ptr(a), _ptr(task), R, int(bool(target)), rt, _ptr(qidx),
                                             _ptr(out), self._stream()))
        return out

    def td_target(self, next_z, reward, terminated, task, eps, qidx) -> torch.Tensor:
        R = next_z.shape[0]
        out = self._rows_out(R, 1)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_td_target(self.h, _ptr(next_z), _ptr(reward), _ptr(terminated), _ptr(task),
                                                  _ptr(eps), _ptr(qidx), R, _ptr(out), self._stream()))
        return out

    def pi_loss_forward(self, z, task, eps, qidx, drop):
        """update_pi's forward on z [rows, L]: -> tape, action [rows, A], q [rows, 1], [rows, 2] = (gaussian log-prob,
        sum of the squash terms).  drop: Q layer 0's dropout scale [num_q, rows, M] or None."""
        R = z.shape[0]
        tape = self._scratch(self.lib.tdmpc2_pi_loss_tape_bytes, self.h, R)
        act, q, lp = self._rows_out(R, self.cfg.action_dim), self._rows_out(R, 1), self._rows_out(R, 2)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_pi_loss_forward(self.h, _ptr(z), _ptr(task), _ptr(eps), _ptr(qidx), _ptr(drop), R,
                                                        _ptr(tape), _ptr(act), _ptr(q), _ptr(lp), self._stream()))
        return tape, act, q, lp

    def pi_loss_backward(self, tensor, tape, z, task, eps, qidx, drop, T, B, scale, entropy_coef, rho, grads, emb_grad):
        """Adds dL/dparameter of update_pi's loss to `grads` (the 10 `_pi.*` .grad tensors by state-dict key) and, for
        multi-task models, to `emb_grad`.  `tensor(key)` returns the model's fp32 tensor of a state-dict key."""
        W = _cabi.Weights()
        for i in range(3):
            W.pi[i] = _linear(_cabi.Linear, tensor, f"_pi.{i}", i < 2)
            W.qs[i] = _linear(_cabi.Linear, tensor, f"_Qs.params.{i}", i < 2)
        G = _cabi.PiGrads()
        for i in range(3):
            G.weight[i], G.bias[i] = _ptr(grads[f"_pi.{i}.weight"]), _ptr(grads[f"_pi.{i}.bias"])
            if i < 2:
                G.ln_weight[i], G.ln_bias[i] = _ptr(grads[f"_pi.{i}.ln.weight"]), _ptr(grads[f"_pi.{i}.ln.bias"])
        G.task_emb = _ptr(emb_grad)
        ws = self._scratch(self.lib.tdmpc2_pi_loss_workspace_bytes, self.h, max(1, T * B))
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_pi_loss_backward(self.h, C.byref(W), _ptr(tape), _ptr(z), _ptr(task), _ptr(eps),
                                                         _ptr(qidx), _ptr(drop), T, B, _ptr(scale), float(entropy_coef),
                                                         float(rho), C.byref(G), _ptr(ws), self._stream()))

    def wm_loss_forward(self, obs0, action, task, drop, H, B, zs=None):
        """agent._update's taped forward: obs0 [B, obs_dim], action [H B, A], task [H B] | None, drop [num_q, H B, M] | None
        -> tape, zs [H + 1, B, L], Q logits [num_q, H B, num_bins], reward logits [H B, num_bins], termination logits
        [H B, 1] (episodic models) or None.  obs0 None: z_0 is the caller's, in zs[0] of the given zs ([H + 1, B, L] fp32
        contiguous, filled in place; pixel models: encode_pixel_rows_taped(..., out=zs[0]))."""
        if obs0 is None and zs is None:
            raise ValueError("wm_loss_forward without obs0 needs zs, with z_0 in zs[0]")
        cfg, R = self.cfg, H * B
        tape = self._scratch(self.lib.tdmpc2_wm_loss_tape_bytes, self.h, H, B)
        if zs is None:
            zs = self._rows_out(H + 1, B, cfg.latent_dim)
        ql, rl = self._rows_out(cfg.num_q, R, cfg.num_bins), self._rows_out(R, cfg.num_bins)
        tl = self._rows_out(R, 1) if cfg.episodic else None
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_loss_forward(self.h, _ptr(obs0), _ptr(action), _ptr(task), _ptr(drop), H, B, _ptr(zs),
                                                        _ptr(ql), _ptr(rl), _ptr(tl), _ptr(tape), self._stream()))
        return tape, zs, ql, rl, tl

    def _wm_loss_structs(self, tensor, grads):
        """(weights, grads, coefficients) structs of the world-model loss's backward."""
        cfg = self.cfg
        both = lambda k, ln: (_linear(_cabi.Linear, tensor, k, ln), _linear(_cabi.LinearGrad, grads.__getitem__, k, ln))
        W, G = _cabi.Weights(), _cabi.WmGrads()
        n = 0
        while f"_encoder.state.{n}.weight" in grads:
            W.enc[n], G.enc[n] = both(f"_encoder.state.{n}", True)
            n += 1
        W.num_enc = G.num_enc = n
        for i in range(3):
            W.dynamics[i], G.dynamics[i] = both(f"_dynamics.{i}", True)
            W.reward[i], G.reward[i] = both(f"_reward.{i}", i < 2)
            W.qs[i], G.qs[i] = both(f"_Qs.params.{i}", i < 2)
            if cfg.episodic:
                W.termination[i], G.termination[i] = both(f"_termination.{i}", i < 2)
        G.task_emb = _ptr(grads.get("_task_emb.weight"))
        cf = _cabi.WmLossCoefs(cfg.consistency_coef, cfg.reward_coef, cfg.value_coef, cfg.termination_coef, cfg.rho,
                               cfg.vmin, cfg.vmax, cfg.bin_size)
        return W, G, cf

    def wm_loss_backward(self, tensor, tape, obs0, action, task, drop, H, B, zs, ql, rl, tl, next_z, reward, td_target,
                         terminated, grads) -> Optional[torch.Tensor]:
        """Adds dL/dparameter of _update's world-model loss to `grads` (.grad tensors by state-dict key: `_encoder.state.*`,
        `_dynamics.*`, `_reward.*`, `_termination.*`, `_Qs.params.*`, `_task_emb.weight`).  `tensor(key)` returns the
        model's fp32 tensor of a state-dict key.  obs0 None (z_0 was the caller's): the state encoder is skipped
        (`_encoder.*` of `grads` is not touched) and dL/dz_0 [B, L] is returned, for pixel_encode_backward; else None."""
        W, G, cf = self._wm_loss_structs(tensor, grads)
        ws = self._scratch(self.lib.tdmpc2_wm_loss_workspace_bytes, self.h, H, B)
        dz0 = self._rows_out(B, self.cfg.latent_dim) if obs0 is None else None
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_wm_loss_backward(
                self.h, C.byref(W), _ptr(tape), _ptr(obs0), _ptr(action), _ptr(task), _ptr(drop), H, B, _ptr(zs), _ptr(ql),
                _ptr(rl), _ptr(tl), _ptr(next_z), _ptr(reward), _ptr(td_target), _ptr(terminated), C.byref(cf), C.byref(G),
                _ptr(dz0), _ptr(ws), self._stream()))
        return dz0

    def estimate_value(self, z, actions, task, noise_pi, qidx):
        """z [E,N,L], actions [E,H,N,A], noise_pi [E,N,A], qidx [E,2] int32 -> [E,N]."""
        out = torch.empty(self.E, self.cfg.num_samples, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_estimate_value(self.h, _ptr(z), _ptr(actions), _ptr(task), _ptr(noise_pi),
                                                       _ptr(qidx), _ptr(out), self._stream()))
        return out

    def debug_layer(self, layer: int, mode: int, x: torch.Tensor, out_features: int) -> torch.Tensor:
        y = torch.empty(x.shape[0], out_features, device=self.device, dtype=torch.float32)
        x = x.contiguous()
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.tdmpc2_debug_layer(self.h, layer, mode, _ptr(x), x.shape[0], _ptr(y), self._stream()))
        return y
