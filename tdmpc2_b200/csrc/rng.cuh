// In-kernel noise for the DECLARED NON-PARITY throughput mode (tdmpc2_plan_iter_rng): the two large noise tensors of a CEM
// iteration -- randn[H, N-P, A] of the sampled action sequences (reference tdmpc2.py:176) and randn_like[N, A] of the
// terminal policy sample (world_model.py:156) -- are generated where they are consumed instead of being drawn by torch into
// HBM (461 MB per c2 plan) and read back.  Counter-based: Philox4x32-10 (Salmon et al., SC'11; the generator torch itself
// uses, but NOT torch's stream -- ATen's offsets depend on its launch geometry) followed by Box-Muller.  One call yields four
// standard normals for the counter (group index, stream, plan counter) under the 64-bit seed, so any thread can regenerate
// any element: the MPPI refit re-derives the elites' actions that way.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tdmpc2 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}

// The raw Philox output of counter (group, stream, plan counter) under the seed.  state[0] = seed, state[1] = plan counter
// (device memory: the launch chain is replayed as a CUDA graph, so the per-plan value must not be a kernel argument)
__device__ __forceinline__ uint4 rng_bits4(const unsigned long long* __restrict__ state, uint32_t stream, unsigned long long group) {
  const unsigned long long seed = state[0], plan = state[1];
  return philox4x32_10(make_uint4(static_cast<uint32_t>(group), static_cast<uint32_t>(group >> 32), stream, static_cast<uint32_t>(plan)),
                       make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32) ^ static_cast<uint32_t>(plan >> 32)));
}
__device__ __forceinline__ float4 rng_normal4(const unsigned long long* __restrict__ state, uint32_t stream, unsigned long long group) {
  const uint4 u = rng_bits4(state, stream, group);
  // Box-Muller: u1 in (0, 1], u2 in [0, 1)
  const float u1a = (static_cast<float>(u.x >> 8) + 1.0f) * (1.0f / 16777216.0f), u2a = static_cast<float>(u.y >> 8) * (1.0f / 16777216.0f);
  const float u1b = (static_cast<float>(u.z >> 8) + 1.0f) * (1.0f / 16777216.0f), u2b = static_cast<float>(u.w >> 8) * (1.0f / 16777216.0f);
  const float ra = sqrtf(-2.0f * logf(u1a)), rb = sqrtf(-2.0f * logf(u1b));
  float sa, ca, sb, cb;
  sincospif(2.0f * u2a, &sa, &ca);
  sincospif(2.0f * u2b, &sb, &cb);
  return make_float4(ra * ca, ra * sa, rb * cb, rb * sb);
}
__device__ __forceinline__ float rng_pick(const float4& g, int i) { return i == 0 ? g.x : i == 1 ? g.y : i == 2 ? g.z : g.w; }

// Four uniforms in [0, 1): the top 24 bits of each word, so every value is an exact fp32 multiple of 2^-24.
__device__ __forceinline__ float4 rng_uniform4(const unsigned long long* __restrict__ state, uint32_t stream, unsigned long long group) {
  const uint4 u = rng_bits4(state, stream, group);
  const float s = 1.0f / 16777216.0f;
  return make_float4(static_cast<float>(u.x >> 8) * s, static_cast<float>(u.y >> 8) * s, static_cast<float>(u.z >> 8) * s,
                     static_cast<float>(u.w >> 8) * s);
}

// diagnostics / tests: out[4 g .. 4 g + 3] = the four normals of group g
__global__ void rng_debug_kernel(const unsigned long long* state, uint32_t stream, unsigned long long group0, int ngroups, float* out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ngroups) return;
  const float4 v = rng_normal4(state, stream, group0 + g);
  out[4 * g] = v.x; out[4 * g + 1] = v.y; out[4 * g + 2] = v.z; out[4 * g + 3] = v.w;
}

}  // namespace tdmpc2
