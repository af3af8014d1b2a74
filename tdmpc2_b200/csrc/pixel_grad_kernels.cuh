// Backward of the pixel encoder (layers.conv, layers.py:136-150) for agent._update on pixel observations: from dL/dz of
// the encoded frames to the gradients of the four Conv2d layers, given the taped forward (pixel_encoder.cuh, P.tape).
//
//   SimNorm back:  dp4 = z * (dz - sum_group dz * z)                                       pixg_simnorm_back
//   conv4 (3x3 s1): dW4, db4 against a3; dA3 = conv4^T(dp4), masked by a3 > 0 -> dp3     pixg_dw<3, 1>, pixg_dx<3, 1>
//   conv3 (3x3 s2): dW3, db3 against a2; dp2 = conv3^T(dp3) masked by a2 > 0              pixg_dw<3, 2>, pixg_dx<3, 2>
//   conv2 (5x5 s2): dW2, db2 against a1; dp1 = conv2^T(dp2) masked by a1 > 0              pixg_dw<5, 2>, pixg_dx<5, 2>
//   conv1 (7x7 s2): dW1, db1 against the ShiftAug + PixelPreprocess image, recomputed     pixg_stage, pixg_dw<7, 2>
//                   from the frames and shifts by pix_stage_value, the forward's own staging function; no dX.
//
// Plain fp32 FFMA (no tensor cores).  Deterministic: every sum runs in a fixed order.  The data gradients are one fmaf
// chain per element (oc, ky, kx ascending).  The weight gradients split the frames into `nsplit` contiguous chunks (a
// function of the shape only); a CTA owns 256 (8 output channels x 1 input column) tiles of one chunk and sums frames and
// positions in ascending order into a partial, and pixg_reduce adds the partials to the gradient in chunk order.  No
// atomics, no allocation, no host synchronisation.
#pragma once
#include "pixel_encoder.cuh"

namespace tdmpc2 {

constexpr int kPgThreads = 256;
constexpr int kPgTargetCtas = 264;     // weight-gradient CTAs per layer the frame split aims for (two per SM on an H100)
constexpr int kPgStageFloats = 4096;   // shared memory of pixg_dw: a [positions][OC] chunk of the output gradient

// Frame chunks of a layer's weight-gradient reduction: enough CTAs to cover the GPU, at most one chunk per frame.
__host__ __device__ __forceinline__ int pixg_cols(int IC, int KK) { return IC * KK + 1; }     // + the bias column
__host__ __device__ __forceinline__ int pixg_ctas_x(int IC, int OC, int KK) {
  return (OC / kPixTO * pixg_cols(IC, KK) + kPgThreads - 1) / kPgThreads;
}
__host__ __device__ __forceinline__ int pixg_nsplit(int IC, int OC, int KK, int64_t rows) {
  const int want = kPgTargetCtas / pixg_ctas_x(IC, OC, KK);
  return static_cast<int>(want < 1 ? 1 : (want > rows ? rows : want));
}

// dp4 [rows][L] = SimNorm's backward per group of V: z (dz - <dz, z>), the group sum in ascending order.
__global__ void __launch_bounds__(kPgThreads) pixg_simnorm_back(const float* __restrict__ z, const float* __restrict__ dz,
                                                                int64_t rows, int L, int V, float* __restrict__ dp) {
  const int64_t ng = rows * (L / V);
  for (int64_t g = blockIdx.x * static_cast<int64_t>(kPgThreads) + threadIdx.x; g < ng; g += static_cast<int64_t>(gridDim.x) * kPgThreads) {
    const int64_t o = g * V;
    float s = 0.f;
    for (int i = 0; i < V; ++i) s = fmaf(dz[o + i], z[o + i], s);
    for (int i = 0; i < V; ++i) dp[o + i] = z[o + i] * (dz[o + i] - s);
  }
}

// dx [rows][IC][IH][IW] = (act > 0) ? sum_{oc, ky, kx} dy[oc][oy][ox] w[oc][ic][ky][kx] : 0, over the (oy, ox) with
// oy S + ky = iy, ox S + kx = ix: the transposed convolution of the output gradient dy [rows][OC][OH][OW], masked by the
// layer input's ReLU (act: the taped post-ReLU map, frame pitch apitch).  One thread per input element; a warp's threads
// share (oc, ky, kx), so the weight loads are broadcasts.
template <int K, int S>
__global__ void __launch_bounds__(kPgThreads) pixg_dx(const float* __restrict__ dy, int OC, int OH, int OW,
                                                      const float* __restrict__ w, const float* __restrict__ act, int64_t apitch,
                                                      int IC, int IH, int IW, int64_t rows, float* __restrict__ dx) {
  const int64_t n = rows * IC * IH * IW;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(kPgThreads) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * kPgThreads) {
    const int ix = static_cast<int>(i % IW);
    int64_t r = i / IW;
    const int iy = static_cast<int>(r % IH);
    r /= IH;
    const int ic = static_cast<int>(r % IC);
    const int64_t e = r / IC;
    float acc = 0.f;
    if (act[e * apitch + (static_cast<int64_t>(ic) * IH + iy) * IW + ix] > 0.f) {
      const float* dye = dy + e * OC * OH * OW;
      for (int oc = 0; oc < OC; ++oc) {
        const float* wp = w + (static_cast<size_t>(oc) * IC + ic) * K * K;
        const float* dp = dye + static_cast<size_t>(oc) * OH * OW;
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          const int ty = iy - ky;
          if (ty < 0 || ty % S != 0 || ty / S >= OH) continue;
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
            const int tx = ix - kx;
            if (tx < 0 || tx % S != 0 || tx / S >= OW) continue;
            acc = fmaf(dp[(ty / S) * OW + tx / S], __ldg(wp + ky * K + kx), acc);
          }
        }
      }
    }
    dx[i] = acc;
  }
}

// img [rows][C][64][64]: conv1's input, recomputed from the frames and shifts exactly as the forward stages it.
__global__ void __launch_bounds__(kPgThreads) pixg_stage(const float* __restrict__ frames, const float* __restrict__ shift,
                                                         const float* __restrict__ grid, int64_t rows, int C, float* __restrict__ img) {
  const int per = C * kPixHW * kPixHW;
  const int64_t n = rows * per;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(kPgThreads) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * kPgThreads) {
    const int64_t e = i / per;
    img[i] = pix_stage_value(frames + e * per, grid, pix_shift_scaled(shift, e, 0), pix_shift_scaled(shift, e, 1),
                             static_cast<int>(i % per));
  }
}

// Partial weight gradient of one Conv2d layer over the frames of chunk blockIdx.y (of nsplit):
//   part[y][oc][col] = sum_{e in chunk} sum_{p} dy[e][oc][p] * in[e][ic][oy S + ky][ox S + kx],  col = (ic, ky, kx),
// and the bias column col = IC K K (input 1).  A thread owns 8 output channels of one column; each chunk of output
// positions of dy is staged in shared memory as [p][OC], so a thread's 8 channels are two float4 loads.
template <int K, int S>
__global__ void __launch_bounds__(kPgThreads) pixg_dw(const float* __restrict__ dy, int OC, int OH, int OW,
                                                      const float* __restrict__ in, int64_t ipitch, int IC, int IH, int IW,
                                                      int64_t rows, int nsplit, float* __restrict__ part) {
  __shared__ __align__(16) float dys[kPgStageFloats];
  constexpr int KK = K * K;
  const int cols = pixg_cols(IC, KK), npos = OH * OW;
  const int PC = max(1, kPgStageFloats / OC);
  const int item = blockIdx.x * kPgThreads + threadIdx.x;
  const bool live = item < OC / kPixTO * cols;
  const int og = live ? item / cols : 0, col = live ? item % cols : 0;
  const bool bias = col == cols - 1;
  const int ic = bias ? 0 : col / KK, ky = bias ? 0 : (col / K) % K, kx = bias ? 0 : col % K;
  const int64_t f0 = rows * blockIdx.y / nsplit, f1 = rows * (blockIdx.y + 1) / nsplit;
  float acc[kPixTO];
#pragma unroll
  for (int o = 0; o < kPixTO; ++o) acc[o] = 0.f;
  for (int64_t e = f0; e < f1; ++e) {
    const float* dye = dy + e * OC * npos;
    const float* ine = in + e * ipitch + (static_cast<int64_t>(ic) * IH + ky) * IW + kx;
    for (int p0 = 0; p0 < npos; p0 += PC) {
      const int np = min(PC, npos - p0);
      __syncthreads();                             // the previous chunk's readers are done
      for (int i = threadIdx.x; i < np * OC; i += kPgThreads) {
        const int oc = i / np, p = i % np;
        dys[p * OC + oc] = dye[static_cast<size_t>(oc) * npos + p0 + p];
      }
      __syncthreads();
      if (live) {
#pragma unroll 1
        for (int p = 0; p < np; ++p) {
          const int pp = p0 + p;
          const float v = bias ? 1.f : __ldg(ine + (pp / OW) * S * IW + (pp % OW) * S);
          const float4 d0 = *reinterpret_cast<const float4*>(dys + p * OC + og * kPixTO);
          const float4 d1 = *reinterpret_cast<const float4*>(dys + p * OC + og * kPixTO + 4);
          acc[0] = fmaf(d0.x, v, acc[0]); acc[1] = fmaf(d0.y, v, acc[1]); acc[2] = fmaf(d0.z, v, acc[2]);
          acc[3] = fmaf(d0.w, v, acc[3]); acc[4] = fmaf(d1.x, v, acc[4]); acc[5] = fmaf(d1.y, v, acc[5]);
          acc[6] = fmaf(d1.z, v, acc[6]); acc[7] = fmaf(d1.w, v, acc[7]);
        }
      }
    }
  }
  if (live) {
    float* pp = part + static_cast<size_t>(blockIdx.y) * OC * cols;
#pragma unroll
    for (int o = 0; o < kPixTO; ++o) pp[static_cast<size_t>(og * kPixTO + o) * cols + col] = acc[o];
  }
}

// dW [OC][cols - 1] += sum_k part[k][oc][col < cols - 1], db [OC] += sum_k part[k][oc][cols - 1], k ascending.
__global__ void __launch_bounds__(kPgThreads) pixg_reduce(const float* __restrict__ part, int nsplit, int OC, int cols,
                                                          float* __restrict__ dw, float* __restrict__ db) {
  const int n = OC * cols;
  for (int i = blockIdx.x * kPgThreads + threadIdx.x; i < n; i += gridDim.x * kPgThreads) {
    float s = 0.f;
    for (int k = 0; k < nsplit; ++k) s += part[static_cast<size_t>(k) * n + i];
    const int oc = i / cols, col = i % cols;
    if (col < cols - 1) dw[static_cast<size_t>(oc) * (cols - 1) + col] += s;
    else db[oc] += s;
  }
}

}  // namespace tdmpc2
