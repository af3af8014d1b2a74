// The small random draws of one plan() on the device (tdmpc2_plan_draws, tdmpc2_act): the policy-prior noise, each CEM
// iteration's Q-head pair, the Gumbel pick's exponentials, the exploration noise and ShiftAug's shifts.  The same
// Philox4x32-10 counter scheme as the iteration kernels' in-kernel noise (rng.cuh) under the same {seed, plan counter}
// state, each kind of draw on a Philox stream of its own, far above the 2 * iteration (+1) streams of
// tdmpc2_plan_iter_rng.  Element i of a draw is component i % 4 of group i / 4 of its stream, so every element can be
// regenerated alone.  Declared non-parity like tdmpc2_plan_iter_rng: these are not torch's streams.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rng.cuh"

namespace tdmpc2 {

constexpr uint32_t kDrawStreamPrior = 0x80000000u;   // noise_prior [E, H, P, A]: standard normals
constexpr uint32_t kDrawStreamQidx = 0x80000001u;    // qidx [I, E, 2]: the two smallest of num_q uniforms, in order
constexpr uint32_t kDrawStreamExpo = 0x80000002u;    // expo [E, K]: -log(u), u in (0, 1]
constexpr uint32_t kDrawStreamFinal = 0x80000003u;   // noise_final [E, A]: standard normals
constexpr uint32_t kDrawStreamShift = 0x80000004u;   // shift [E, 2]: floor(7 u), u in [0, 1)
constexpr int kDrawKinds = 5;

struct DrawParams {
  const unsigned long long* state;
  float* prior;  long long n_prior;      // NULL / 0: not drawn
  int32_t* qidx; long long q_rows; int num_q;
  float* expo;   long long n_expo;
  float* final_; long long n_final;
  float* shift;  long long n_shift;
};

// One launch for every kind: blockIdx.y selects the kind, a grid-stride loop over its groups (rows for qidx).
__global__ void plan_draws_kernel(DrawParams P) {
  const int kind = blockIdx.y;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (kind == 1) {
    if (!P.qidx) return;
    const int groups = (P.num_q + 3) / 4;
    for (long long r = i0; r < P.q_rows; r += stride) {
      uint32_t b0 = 0xffffffffu, b1 = 0xffffffffu;
      int j0 = -1, j1 = -1;
      for (int g = 0; g < groups; ++g) {
        const uint4 u = rng_bits4(P.state, kDrawStreamQidx, static_cast<unsigned long long>(r) * groups + g);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = 4 * g + c;
          if (j >= P.num_q) break;
          // strict comparisons: of equal words the lower index ranks first
          if (j0 < 0 || w[c] < b0) { b1 = b0; j1 = j0; b0 = w[c]; j0 = j; }
          else if (j1 < 0 || w[c] < b1) { b1 = w[c]; j1 = j; }
        }
      }
      P.qidx[2 * r] = j0;
      P.qidx[2 * r + 1] = j1;
    }
    return;
  }
  float* out;
  long long n;
  uint32_t stream;
  switch (kind) {
    case 0: out = P.prior; n = P.n_prior; stream = kDrawStreamPrior; break;
    case 2: out = P.expo; n = P.n_expo; stream = kDrawStreamExpo; break;
    case 3: out = P.final_; n = P.n_final; stream = kDrawStreamFinal; break;
    default: out = P.shift; n = P.n_shift; stream = kDrawStreamShift; break;
  }
  if (!out) return;
  for (long long g = i0; 4 * g < n; g += stride) {
    float v[4];
    if (kind == 0 || kind == 3) {
      const float4 x = rng_normal4(P.state, stream, g);
      v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
    } else {
      const float4 u = rng_uniform4(P.state, stream, g);
      const float uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int c = 0; c < 4; ++c)   // 1 - u is exact (u is a multiple of 2^-24) and lies in (0, 1]
        v[c] = kind == 2 ? -logf(1.0f - uu[c]) : floorf(7.0f * uu[c]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (4 * g + c < n) out[4 * g + c] = v[c];
  }
}

// state[1] += 1: a fresh stream for the next plan, advanced on the device so that a captured launch chain advances too
__global__ void rng_advance_kernel(unsigned long long* state) { state[1] += 1ull; }

}  // namespace tdmpc2
