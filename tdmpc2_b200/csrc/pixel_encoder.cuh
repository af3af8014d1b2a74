// Pixel-observation encoder of TD-MPC2 (cfg.obs == 'rgb'), forward only, for the planner's prologue.
//
// Reference: layers.conv (common/layers.py:136-150): ShiftAug (:36-59, applied at inference too -- it sits inside the
// nn.Sequential), PixelPreprocess (:62-71: x / 255 - 0.5), Conv2d(C, nc, 7, stride 2) + ReLU, Conv2d(nc, nc, 5, stride 2)
// + ReLU, Conv2d(nc, nc, 3, stride 2) + ReLU, Conv2d(nc, nc, 3, stride 1), Flatten, SimNorm (:74-88).  64 x 64 inputs
// (asserted at :141) give 29 -> 13 -> 6 -> 4 feature maps, so latent_dim == 16 * nc.
//
// Persistent grid: min(rows, SMs) CTAs, each looping over frames blockIdx.x, blockIdx.x + gridDim.x, ...  Per frame the
// augmented, normalised frame stack is staged in shared memory (C x 64 x 64 fp32), conv1 goes to the CTA's own global
// scratch slot (it does not fit next to its input; SMs x slot stays in L2 whatever the frame count), conv2-4 and SimNorm
// stay in shared memory.  Each conv layer's weights and bias are staged in shared memory once per frame, laid out
// [ic][ky][kx][oc] so that a thread's 8 output channels are two float4 loads; when they do not fit next to the layer's
// activations they are staged in output-channel chunks (and, for the widest frame stacks, input-channel chunks whose
// partial sums wait in the output map).  Each thread computes a register tile of 8 output channels x TP positions.
// Plain fp32 FFMA, the products exact: every output is one fmaf chain, bias first, then ic, ky, kx in ascending order, so
// z does not depend on how frames or tiles are assigned to CTAs and threads.  The summation order differs from ATen's
// (1e-6 relative).
//
// ShiftAug restated: pad 3 with edge replication, sample the padded 70 x 70 image bilinearly (zeros outside, align_corners
// = False) at base + shift * 2/70, where base is linspace(-1 + 1/70, 1 - 1/70, 70)[:64] (computed by the host with
// torch.linspace so that the coordinates are bit-identical to the reference's) and shift is an integer pair in [0, 6]
// drawn by the host (torch.randint, the first random draw of a reference _plan call on pixel observations).  The sample
// points are pixel centres up to fp32 rounding, so the result is the shifted crop plus O(1e-5) of its neighbours -- kept,
// because the reference has it.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

namespace tdmpc2 {

constexpr int kPixHW = 64, kPixPad = 3, kPixPadded = kPixHW + 2 * kPixPad;
constexpr int kPixO1 = 29, kPixO2 = 13, kPixO3 = 6, kPixO4 = 4;
constexpr int kPixThreads = 512;
constexpr int kPixTO = 8;                          // output channels per thread tile (num_channels is a multiple of 8)
constexpr int kPixMaxSmem = 227 * 1024;            // dynamic shared memory an sm_90 CTA can opt in to

struct PixelParams {
  const float* frames;   // [rows, C, 64, 64], 0 .. 255
  const float* shift;    // [rows, 2]: (x, y), integral values in [0, 6]  (layers.py:55)
  const float* grid;     // [64]: linspace(-1 + eps, 1 - eps, 70)[:64]  (layers.py:51)
  const float* w[4];     // Conv2d weights [out, in, k, k] as nn.Conv2d stores them
  const float* b[4];
  float* scratch;        // [gridDim.x][nc * 29 * 29]: one conv1 slot per CTA
  float* z;              // [rows, 16 * nc]
  float* tape;           // optional [rows][pix_tape_floats(nc)]: the post-ReLU maps a1 | a2 | a3 of every frame (backward)
  int64_t rows;
  int C, nc, simnorm;
  int smem_floats;       // dynamic shared memory of the launch, in floats
};

// Shared-memory plan, in floats: the staged frame [C][64][64] during conv1, the maps s2 | s3 | s4 during conv2-4; each
// layer's weight chunk follows its activations.
__host__ __device__ __forceinline__ int pix_stage_floats(int C) { return C * kPixHW * kPixHW; }
__host__ __device__ __forceinline__ int pix_maps_floats(int nc) { return nc * (kPixO2 * kPixO2 + kPixO3 * kPixO3 + kPixO4 * kPixO4); }
// The taped forward's per-frame slot, in floats: a1 [nc][29][29] | a2 [nc][13][13] | a3 [nc][6][6], each segment starting
// on a 64-float boundary.  conv4's output is not taped: SimNorm's backward reads z alone.
__host__ __device__ __forceinline__ int pix_al64(int n) { return (n + 63) / 64 * 64; }
__host__ __device__ __forceinline__ int pix_tape_a2(int nc) { return pix_al64(nc * kPixO1 * kPixO1); }
__host__ __device__ __forceinline__ int pix_tape_a3(int nc) { return pix_tape_a2(nc) + pix_al64(nc * kPixO2 * kPixO2); }
__host__ __device__ __forceinline__ int pix_tape_floats(int nc) { return pix_tape_a3(nc) + pix_al64(nc * kPixO3 * kPixO3); }
// Weight chunk of one layer in `cap` floats: occ output channels x icc input channels ([icc][K][K][occ] + occ biases).
// All output channels with all input channels when they fit, else the widest multiple of 8 output channels, else 8
// output channels and as many input channels as fit (icc < 1: the layer does not fit at all).
__host__ __device__ __forceinline__ void pix_chunk(int IC, int OC, int KK, int cap, int* occ, int* icc) {
  const int o = min(OC, cap / (IC * KK + 1) / kPixTO * kPixTO);
  if (o >= kPixTO) { *occ = o; *icc = IC; return; }
  *occ = kPixTO;
  *icc = min(IC, (cap - kPixTO) / (kPixTO * KK));
}

// ATen's CPU grid sampler (GridSamplerKernel.cpp, align_corners = false): (x + 1) * (size / 2) - 0.5, separate roundings.
__device__ __forceinline__ float pix_unnormalize(float g) {
  return __fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), 0.5f * kPixPadded), 0.5f);
}
__device__ __forceinline__ float pix_padded(const float* img, int py, int px) {   // replicate-padded image, zeros outside
  if (py < 0 || py >= kPixPadded || px < 0 || px >= kPixPadded) return 0.f;
  const int y = min(max(py - kPixPad, 0), kPixHW - 1), x = min(max(px - kPixPad, 0), kPixHW - 1);
  return img[y * kPixHW + x];
}

// Element i = (c * 64 + y) * 64 + x of ShiftAug + PixelPreprocess applied to one frame `img` [C][64][64] (values 0..255),
// shift (sx, sy) already scaled by 2/70.  The forward's staging loop and the backward's recomputation of conv1's input both
// call this, so the two cannot drift apart.
__device__ __forceinline__ float pix_stage_value(const float* __restrict__ img, const float* __restrict__ grid, float sx, float sy,
                                                 int i) {
  const int c = i / (kPixHW * kPixHW), y = (i / kPixHW) % kPixHW, x = i % kPixHW;
  const float fx = pix_unnormalize(__fadd_rn(grid[x], sx)), fy = pix_unnormalize(__fadd_rn(grid[y], sy));
  const float wx = floorf(fx), ny = floorf(fy);
  const float ex = wx + 1.f, sy1 = ny + 1.f;
  const int ix = static_cast<int>(wx), iy = static_cast<int>(ny);
  const float* ch = img + static_cast<size_t>(c) * kPixHW * kPixHW;
  float v = pix_padded(ch, iy, ix) * ((ex - fx) * (sy1 - fy));
  v += pix_padded(ch, iy, ix + 1) * ((fx - wx) * (sy1 - fy));
  v += pix_padded(ch, iy + 1, ix) * ((ex - fx) * (fy - ny));
  v += pix_padded(ch, iy + 1, ix + 1) * ((fx - wx) * (fy - ny));
  return __fsub_rn(__fdiv_rn(v, 255.f), 0.5f);
}
__device__ __forceinline__ float pix_shift_scaled(const float* shift, int64_t e, int k) {
  return __fmul_rn(shift[e * 2 + k], 2.0f / kPixPadded);
}

// out[oc][oy][ox] = act(b[oc] + sum_{ic,ky,kx} in[ic][oy*S+ky][ox*S+kx] * w[oc][ic][ky][kx]), one fmaf chain per output in
// that order.  wsm: `cap` floats of shared memory for the weight chunks.  A thread's tile is 8 output channels x TP
// positions p, p + ntp, ..., so that neighbouring threads read neighbouring positions.  When the input channels come in
// several chunks, the running sums wait in `out` between them (an exact fp32 round trip).  Starts with a barrier (the
// previous layer's output is complete, the previous readers of wsm are done); the caller syncs before reading `out`.
template <int K, int S, int TP, bool RELU>
__device__ __forceinline__ void pix_conv(const float* in, int IC, int IH, int IW, const float* __restrict__ w,
                                         const float* __restrict__ b, int OC, float* out, int OH, int OW, float* wsm,
                                         int cap) {
  constexpr int KK = K * K;
  const int npos = OH * OW, ntp = (npos + TP - 1) / TP;
  int occ, icc;
  pix_chunk(IC, OC, KK, cap, &occ, &icc);
  for (int oc0 = 0; oc0 < OC; oc0 += occ) {
    const int noc = min(occ, OC - oc0);
    for (int ic0 = 0; ic0 < IC; ic0 += icc) {
      const int nic = min(icc, IC - ic0), nw = nic * KK * noc;
      float* bsm = wsm + nw;
      __syncthreads();
      for (int i = threadIdx.x; i < nw; i += kPixThreads) {     // [icl][ky][kx][ocl] <- w[oc0 + ocl][ic0 + icl][ky][kx]
        const int o = i % noc, r = i / noc;
        wsm[i] = __ldg(w + (static_cast<size_t>(oc0 + o) * IC + ic0) * KK + r);
      }
      for (int i = threadIdx.x; i < noc; i += kPixThreads) bsm[i] = __ldg(b + oc0 + i);
      __syncthreads();
      const bool first = ic0 == 0, last = ic0 + nic == IC;
      for (int item = threadIdx.x; item < noc / kPixTO * ntp; item += kPixThreads) {
        const int og = item / ntp, tp = item % ntp;
        int off[TP];
        bool ok[TP];
#pragma unroll
        for (int j = 0; j < TP; ++j) {
          const int p = tp + j * ntp;
          ok[j] = p < npos;
          const int pp = ok[j] ? p : 0;
          off[j] = (pp / OW) * S * IW + (pp % OW) * S;
        }
        float* o_base = out + static_cast<size_t>(oc0 + og * kPixTO) * npos + tp;
        float acc[kPixTO][TP];
#pragma unroll
        for (int o = 0; o < kPixTO; ++o)
#pragma unroll
          for (int j = 0; j < TP; ++j) acc[o][j] = first ? bsm[og * kPixTO + o] : (ok[j] ? o_base[o * npos + j * ntp] : 0.f);
        for (int icl = 0; icl < nic; ++icl) {
          const float* ip = in + static_cast<size_t>(ic0 + icl) * IH * IW;
          const float* wp = wsm + icl * KK * noc + og * kPixTO;
#pragma unroll
          for (int ky = 0; ky < K; ++ky)
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
              const float4 w0 = *reinterpret_cast<const float4*>(wp + (ky * K + kx) * noc);
              const float4 w1 = *reinterpret_cast<const float4*>(wp + (ky * K + kx) * noc + 4);
              const float wv[kPixTO] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
              for (int j = 0; j < TP; ++j) {
                const float v = ip[off[j] + ky * IW + kx];
#pragma unroll
                for (int o = 0; o < kPixTO; ++o) acc[o][j] = fmaf(v, wv[o], acc[o][j]);
              }
            }
        }
#pragma unroll
        for (int o = 0; o < kPixTO; ++o)
#pragma unroll
          for (int j = 0; j < TP; ++j)
            if (ok[j]) o_base[o * npos + j * ntp] = (RELU && last) ? fmaxf(acc[o][j], 0.f) : acc[o][j];
      }
    }
  }
}

__global__ void __launch_bounds__(kPixThreads, 1) pixel_encode_kernel(const PixelParams P) {
  extern __shared__ __align__(16) float pix_smem[];
  const int stage = pix_stage_floats(P.C), maps = pix_maps_floats(P.nc);
  float* s2 = pix_smem;                          // conv2-4 maps: the staged input is dead by then
  float* s3 = s2 + P.nc * kPixO2 * kPixO2;
  float* s4 = s3 + P.nc * kPixO3 * kPixO3;
  const int L = P.nc * kPixO4 * kPixO4;
  for (int64_t e = blockIdx.x; e < P.rows; e += gridDim.x) {
    const float* img = P.frames + e * P.C * kPixHW * kPixHW;
    // conv1's output: this CTA's scratch slot, or the frame's tape slot (a1) when taping
    float* tslot = P.tape ? P.tape + e * pix_tape_floats(P.nc) : nullptr;
    float* s1 = tslot ? tslot : P.scratch + static_cast<size_t>(blockIdx.x) * P.nc * kPixO1 * kPixO1;
    __syncthreads();                             // the previous frame's SimNorm has read s4, which the stage overwrites
    // ---- ShiftAug + PixelPreprocess -> smem [C][64][64]
    const float sx = pix_shift_scaled(P.shift, e, 0), sy = pix_shift_scaled(P.shift, e, 1);
    for (int i = threadIdx.x; i < P.C * kPixHW * kPixHW; i += kPixThreads) pix_smem[i] = pix_stage_value(img, P.grid, sx, sy, i);
    // each pix_conv starts with a barrier: its input is complete (conv1's global slot included -- written and read by
    // this CTA only) and the previous layer no longer reads the smem it stages its weights into
    pix_conv<7, 2, 4, true>(pix_smem, P.C, kPixHW, kPixHW, P.w[0], P.b[0], P.nc, s1, kPixO1, kPixO1, pix_smem + stage,
                            P.smem_floats - stage);
    pix_conv<5, 2, 2, true>(s1, P.nc, kPixO1, kPixO1, P.w[1], P.b[1], P.nc, s2, kPixO2, kPixO2, pix_smem + maps,
                            P.smem_floats - maps);
    pix_conv<3, 2, 1, true>(s2, P.nc, kPixO2, kPixO2, P.w[2], P.b[2], P.nc, s3, kPixO3, kPixO3, pix_smem + maps,
                            P.smem_floats - maps);
    pix_conv<3, 1, 1, false>(s3, P.nc, kPixO3, kPixO3, P.w[3], P.b[3], P.nc, s4, kPixO4, kPixO4, pix_smem + maps,
                             P.smem_floats - maps);
    __syncthreads();
    if (tslot) {                                 // a2, a3: still intact in smem (conv4 staged its weights after s4)
      for (int i = threadIdx.x; i < P.nc * kPixO2 * kPixO2; i += kPixThreads) tslot[pix_tape_a2(P.nc) + i] = s2[i];
      for (int i = threadIdx.x; i < P.nc * kPixO3 * kPixO3; i += kPixThreads) tslot[pix_tape_a3(P.nc) + i] = s3[i];
    }
    // ---- Flatten ([nc][4][4] is already the flattened order) + SimNorm: softmax over groups of `simnorm` consecutive values
    float* zrow = P.z + e * L;
    for (int g0 = threadIdx.x * P.simnorm; g0 < L; g0 += kPixThreads * P.simnorm) {
      float m = -CUDART_INF_F;
      for (int i = 0; i < P.simnorm; ++i) m = fmaxf(m, s4[g0 + i]);
      float t = 0.f;
      for (int i = 0; i < P.simnorm; ++i) t += expf(s4[g0 + i] - m);
      for (int i = 0; i < P.simnorm; ++i) zrow[g0 + i] = __fdiv_rn(expf(s4[g0 + i] - m), t);
    }
  }
}

}  // namespace tdmpc2
