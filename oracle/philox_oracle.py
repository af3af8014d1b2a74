"""Host reference for the in-kernel noise of the philox planning mode -- TEST INFRASTRUCTURE ONLY.

`tdmpc2_plan_iter_rng` (csrc/rng.cuh) and `tdmpc2_plan_draws` (csrc/draw_kernels.cuh) generate every random number of a
philox plan on the device.  This module restates, in numpy with uint64 arithmetic (no torch in the generator), what they
compute, so that a philox plan can be held to the float64 plan oracle like a torch-noise plan:

  philox4x32_10        <- rng.cuh philox4x32_10 (Salmon et al., SC'11: round multipliers 0xD2511F53 / 0xCD9E8D57,
                          Weyl key increments 0x9E3779B9 / 0xBB67AE85, ten rounds)
  bits4                <- rng_bits4: counter (group lo, group hi, stream, plan lo), key (seed lo, seed hi ^ plan hi)
  normal4              <- rng_normal4: Box-Muller on the kernel's own 24-bit uniforms, evaluated in float64
  uniform4             <- rng_uniform4
  plan_draws           <- plan_draws_kernel: the five small draws of one plan (DESIGN.md section 4.9)
  noise_r / noise_pi   <- noise_r_at / noise_pi_at (plan_kernels.cuh): the iteration noise layout
  plan_noise           -> an oracle.plan_oracle.PlanNoise from given iteration noise and small draws
"""
from __future__ import annotations

import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
PHILOX_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))
TWO_M24 = 2.0 ** -24
RHO_MAX = float(np.sqrt(48.0 * np.log(2.0)))    # sqrt(-2 ln 2^-24): the largest |normal| the generator can produce

# the draw streams of tdmpc2_plan_draws (draw_kernels.cuh)
STREAM_PRIOR, STREAM_QIDX, STREAM_EXPO, STREAM_FINAL, STREAM_SHIFT = (0x80000000 + k for k in range(5))


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters ctr [..., 4] under keys key [..., 2] (uint32 values; leading dimensions broadcast)
    -> uint32 [..., 4]."""
    ctr, key = _u64(ctr), _u64(key)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for _ in range(10):
        p0, p1 = PHILOX_M[0] * c0, PHILOX_M[1] * c2        # exact: both factors are below 2^32
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + PHILOX_W[0]) & M32, (k1 + PHILOX_W[1]) & M32
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), axis=-1).astype(np.uint32)


def bits4(seed, plan, stream, group):
    """rng_bits4: the four raw words of group `group` of stream `stream` under state {seed, plan counter}; every argument
    broadcasts (seed and plan are 64-bit, stream 32-bit, group 64-bit) -> uint32 [..., 4]."""
    seed, plan, stream, group = _u64(seed), _u64(plan), _u64(stream), _u64(group)
    s32 = np.uint64(32)
    c = np.stack(np.broadcast_arrays(group & M32, group >> s32, stream & M32, plan & M32), axis=-1)
    k = np.stack(np.broadcast_arrays(seed & M32, (seed >> s32) ^ (plan >> s32)), axis=-1)
    return philox4x32_10(c, k)


def box_muller_uniforms(w):
    """The kernel's exact Box-Muller uniforms of words w [..., 4]: u1 = ((x >> 8) + 1) 2^-24 in (0, 1] and
    u2 = (y >> 8) 2^-24 in [0, 1) of the pairs (x, y) = (w0, w1) and (w2, w3) -> (u1 [..., 2], u2 [..., 2]), float64."""
    top = (w >> np.uint32(8)).astype(np.float64)
    return (top[..., 0::2] + 1.0) * TWO_M24, top[..., 1::2] * TWO_M24


def normal4(seed, plan, stream, group):
    """rng_normal4 in float64 -> (normals [..., 4], rho [..., 4]): (rho_a cos, rho_a sin, rho_b cos, rho_b sin) with
    rho = sqrt(-2 ln u1) and the angle 2 pi u2; rho is repeated per component for error bounds."""
    u1, u2 = box_muller_uniforms(bits4(seed, plan, stream, group))
    rho = np.sqrt(-2.0 * np.log(u1))
    ang = 2.0 * np.pi * u2
    out = np.stack([rho[..., 0] * np.cos(ang[..., 0]), rho[..., 0] * np.sin(ang[..., 0]),
                    rho[..., 1] * np.cos(ang[..., 1]), rho[..., 1] * np.sin(ang[..., 1])], axis=-1)
    return out, np.repeat(rho, 2, axis=-1)


def uniform4(seed, plan, stream, group):
    """rng_uniform4: (w >> 8) 2^-24 in [0, 1), exact in fp32 and float64 -> [..., 4] float64."""
    return (bits4(seed, plan, stream, group) >> np.uint32(8)).astype(np.float64) * TWO_M24


# ------------------------------------------------------------------------------------------------- the small draws
def _elements(law, seed, plan, stream, n):
    """Element i of a draw: component i % 4 of group i / 4 of its stream."""
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    out = law(seed, plan, stream, g)
    if isinstance(out, tuple):
        return tuple(o.reshape(-1)[:n] for o in out)
    return out.reshape(-1)[:n]


def normals(seed, plan, stream, n):
    """n normals of a draw stream -> (values [n], rho [n])."""
    return _elements(normal4, seed, plan, stream, n)


def expo(seed, plan, n):
    """n exponentials: -ln(1 - u) (1 - u is exact) -> [n] float64."""
    return -np.log(1.0 - _elements(uniform4, seed, plan, STREAM_EXPO, n))


def shift(seed, plan, n):
    """n ShiftAug shifts: floor(7 u) in {0 .. 6} -> [n] float64."""
    return np.floor(7.0 * _elements(uniform4, seed, plan, STREAM_SHIFT, n))


def two_smallest(words):
    """Indices of the two smallest entries of each row of words [rows, num_q], smallest first, of equal words the lower
    index first -> int64 [rows, 2]."""
    return np.argsort(np.asarray(words, dtype=np.uint64), axis=-1, kind="stable")[..., :2].astype(np.int64)


def qidx_words(seed, plan, rows, num_q):
    """The num_q words of each qidx row: row r reads groups r ceil(num_q / 4) .. of the qidx stream -> [rows, num_q]."""
    G = (num_q + 3) // 4
    g = np.arange(rows * G, dtype=np.uint64)
    return bits4(seed, plan, STREAM_QIDX, g).reshape(rows, 4 * G)[:, :num_q]


def qidx(seed, plan, I, E, num_q):
    """The Q-head pairs of one plan: row r = it E + e -> int64 [I, E, 2]."""
    return two_smallest(qidx_words(seed, plan, I * E, num_q)).reshape(I, E, 2)


def plan_draws(seed, plan, E, H, P, A, I, K, num_q, eval_mode=False, pixel=False):
    """Every small draw of one plan at state {seed, plan}, as tdmpc2_plan_draws writes them.  Returns a dict of float64
    arrays (qidx int64): prior [E, H, P, A] (None when P == 0), prior_rho, qidx [I, E, 2], expo [E, K], final [E, A]
    (None in eval mode), final_rho, shift [E, 2] (None unless pixel)."""
    out = dict(prior=None, prior_rho=None, final=None, final_rho=None, shift=None)
    if P > 0:
        v, r = normals(seed, plan, STREAM_PRIOR, E * H * P * A)
        out["prior"], out["prior_rho"] = v.reshape(E, H, P, A), r.reshape(E, H, P, A)
    out["qidx"] = qidx(seed, plan, I, E, num_q)
    out["expo"] = expo(seed, plan, E * K).reshape(E, K)
    if not eval_mode:
        v, r = normals(seed, plan, STREAM_FINAL, E * A)
        out["final"], out["final_rho"] = v.reshape(E, A), r.reshape(E, A)
    if pixel:
        out["shift"] = shift(seed, plan, E * 2).reshape(E, 2)
    return out


# ------------------------------------------------------------------------------------------------- the iteration noise
def r_groups(E, H, N, A):
    """Number of groups of stream 2 it that noise_r spans: ((e H + t) N + n) A4 + a / 4 over every e, t, n < N (the P
    prior rows included) and a, A4 = ceil(A / 4)."""
    return E * H * N * ((A + 3) // 4)


def pi_groups(E, N, A):
    """Number of groups of stream 2 it + 1 that noise_pi spans: (e N + n) A4 + a / 4."""
    return E * N * ((A + 3) // 4)


def layout_r(groups, E, H, N, P, A):
    """noise_r [E, H, N - P, A] from the normals of groups 0 .. r_groups() - 1 of stream 2 it ([groups, 4] or flat)."""
    A4 = (A + 3) // 4
    return groups.reshape(E, H, N, 4 * A4)[:, :, P:, :A]


def layout_pi(groups, E, N, A):
    """noise_pi [E, N, A] from the normals of groups 0 .. pi_groups() - 1 of stream 2 it + 1."""
    A4 = (A + 3) // 4
    return groups.reshape(E, N, 4 * A4)[:, :, :A]


def noise_r(seed, plan, it, E, H, N, P, A):
    """Iteration it's sample noise in float64 -> (values [E, H, N - P, A], rho)."""
    v, r = normal4(seed, plan, 2 * it, np.arange(r_groups(E, H, N, A), dtype=np.uint64))
    return layout_r(v, E, H, N, P, A), layout_r(r, E, H, N, P, A)


def noise_pi(seed, plan, it, E, N, A):
    """Iteration it's terminal policy noise in float64 -> (values [E, N, A], rho)."""
    v, r = normal4(seed, plan, 2 * it + 1, np.arange(pi_groups(E, N, A), dtype=np.uint64))
    return layout_pi(v, E, N, A), layout_pi(r, E, N, A)


def plan_noise(r, pi, prior, qidx, expo, final, shift=None, H=None, A=None):
    """oracle.plan_oracle.PlanNoise from iteration noise r [I, E, H, N - P, A] and pi [I, E, N, A] (iteration-major, as
    generated) and the small draws: prior [E, H, P, A] or None (P == 0: give H and A), qidx [I, E, 2], expo [E, K],
    final [E, A] or None (eval mode: zeros), shift [E, 2] or None.  numpy arrays or torch tensors; values are kept in their
    dtype (the oracle casts to its own)."""
    import torch
    from oracle.plan_oracle import PlanNoise
    t = lambda x: torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x).cpu()
    r, pi, qidx, expo = t(r), t(pi), t(qidx), t(expo)
    E = expo.shape[0]
    if prior is None:
        prior = torch.zeros(E, H, 0, A, dtype=expo.dtype)
    prior = t(prior)
    final = torch.zeros(E, r.shape[-1], dtype=expo.dtype) if final is None else t(final)
    return PlanNoise(prior=prior, r=r.transpose(0, 1).contiguous(), pi=pi.transpose(0, 1).contiguous(),
                     qidx=qidx.to(torch.int64).transpose(0, 1).contiguous(), expo=expo, final=final,
                     shift=None if shift is None else t(shift))
