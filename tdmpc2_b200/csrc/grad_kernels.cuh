// Backward of agent.update_pi's loss (reference tdmpc2.py:208-239) from the tape of plan_kernel's ROP_PI_LOSS row op.
//
// The loss of a [T, B] batch of latents (row r = t B + b) is
//     mean_t rho^t mean_b -(entropy_coef * scaled_entropy_r + q_r / scale),
// with q_r = (Q_{qidx[0]} + Q_{qidx[1]}) / 2 on (z_r, pi(z_r)) through detached online Q heads.  Its gradient reaches
// the pi MLP's parameters (and, in multi-task models, the task embedding) through two paths: the action the Q heads
// read, and the entropy term.  The kernels below run it as a short launch chain:
//
//   pl_q_head_back   per row and head: dL/dq -> two-hot inverse (symexp of softmax . bins) -> dL/dlogits
//   gemm_f32         dL/dX of Q layers 2 -> 1 -> 0 (only the [emb | action] columns of layer 0's input)
//   pl_ln_back       per row: Mish and LayerNorm (and the dropout scale of Q layer 0) recomputed from the tape
//   pl_pi_head_back  per row: the tanh-Gaussian head -- masks, log_std transform, squash, the entropy quotient
//   gemm_f32 / pl_reduce / pl_colsum / pl_emb_grad   dW, db, dgamma, dbeta of pi layers 2 -> 0 and the embedding
//
// Arithmetic is fp32 FFMA; weights are the fp32 state-dict tensors.  Every reduction over rows runs in a fixed order
// (split-K partials summed split by split, GEMM K tiles and column sums in fixed blocks): two calls on the same inputs
// give the same bits.  Long sums are blocked so that an output's rounding chain stays short: a plain running sum over
// R rows carries ~R roundings, far more than the blocked sums of a float64-checked reference at R in the thousands.
// Nothing allocates or synchronises with the host, so the chain can be captured in a CUDA graph.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tdmpc2 {

// ------------------------------------------------------------------------------------ generic fp32 GEMM
// C[i, j] = sum_k A(i, k) B(k, j) over the batch blockIdx.z / nsplit and the K range of split blockIdx.z % nsplit;
// A(i, k) = A[i * a_i + k * a_k], B(k, j) = B[k * b_k + j * b_j].  Batch z offsets A, C by z * a_z, z * c_z and B by
// (bsel ? bsel[z] : z) * b_z; split s writes its partial sum at C + s * c_s.  Each output is one thread's k loop, summed
// per K tile, then the tile sums in order.
struct GemmArgs {
  const float* A; long long a_i, a_k, a_z;
  const float* B; long long b_k, b_j, b_z; const int* bsel;
  float* C; long long ldc, c_z, c_s;
  int m, n, k, nsplit;
};
constexpr int kGBM = 64, kGBN = 64, kGBK = 16;

__global__ void __launch_bounds__(256) gemm_f32(const GemmArgs g) {
  __shared__ float sA[kGBK][kGBM + 4];
  __shared__ float sB[kGBK][kGBN + 4];
  const int z = blockIdx.z / g.nsplit, s = blockIdx.z % g.nsplit;
  const float* A = g.A + z * g.a_z;
  const float* B = g.B + (g.bsel ? g.bsel[z] : z) * g.b_z;
  float* C = g.C + z * g.c_z + s * g.c_s;
  const int kc = (g.k + g.nsplit - 1) / g.nsplit;
  const int k0 = s * kc, k1 = min(g.k, k0 + kc);
  const int i0 = blockIdx.y * kGBM, j0 = blockIdx.x * kGBN;
  const int tid = threadIdx.x, ti = (tid / 16) * 4, tj = (tid % 16) * 4;
  float acc[4][4] = {};
  for (int kb = k0; kb < k1; kb += kGBK) {
    // tile loads: consecutive threads walk the operand's unit-stride dimension
    for (int e = tid; e < kGBK * kGBM; e += 256) {
      int kk, ii;
      if (g.a_i == 1) { ii = e % kGBM; kk = e / kGBM; } else { kk = e % kGBK; ii = e / kGBK; }
      const int gi = i0 + ii, gk = kb + kk;
      sA[kk][ii] = (gi < g.m && gk < k1) ? A[gi * g.a_i + gk * g.a_k] : 0.f;
    }
    for (int e = tid; e < kGBK * kGBN; e += 256) {
      int kk, jj;
      if (g.b_j == 1) { jj = e % kGBN; kk = e / kGBN; } else { kk = e % kGBK; jj = e / kGBK; }
      const int gj = j0 + jj, gk = kb + kk;
      sB[kk][jj] = (gj < g.n && gk < k1) ? B[gk * g.b_k + gj * g.b_j] : 0.f;
    }
    __syncthreads();
    float t[4][4] = {};
#pragma unroll
    for (int kk = 0; kk < kGBK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&sA[kk][ti]);
      const float4 b = *reinterpret_cast<const float4*>(&sB[kk][tj]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) t[u][v] = fmaf(av[u], bv[v], t[u][v]);
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[u][v] += t[u][v];
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v)
      if (i0 + ti + u < g.m && j0 + tj + v < g.n) C[(i0 + ti + u) * g.ldc + j0 + tj + v] = acc[u][v];
}

// dst[i] += sum_s part[s * stride + i] (s in order), i < n
__global__ void pl_reduce(const float* __restrict__ part, int nsplit, long long stride, long long n, float* __restrict__ dst) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  float v = 0.f;
  for (int s = 0; s < nsplit; ++s) v += part[s * stride + i];
  dst[i] += v;
}

// sum over r < rows of f(r) in a fixed tree: runs of 8 rows, runs of 8 of those, of 8 of those, then in order.  About
// 24 + rows / 512 roundings per sum instead of rows.  f is read 16 rows at a time, so 16 loads are in flight.
template <class F>
__device__ __forceinline__ float pl_tree_sum(int rows, F f) {
  float v = 0.f;
  for (int r3 = 0; r3 < rows; r3 += 512) {
    float s2 = 0.f;
    for (int r2 = r3; r2 < min(rows, r3 + 512); r2 += 64) {
      float s1 = 0.f;
      for (int r1 = r2; r1 < min(rows, r2 + 64); r1 += 16) {
        float x[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) x[u] = r1 + u < rows ? f(r1 + u) : 0.f;
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) { a += x[u]; b += x[8 + u]; }
        s1 += a;
        s1 += b;
      }
      s2 += s1;
    }
    v += s2;
  }
  return v;
}

// dst[j] += sum_r src[r * ld + j] (pl_tree_sum), j < n
__global__ void pl_colsum(const float* __restrict__ src, int rows, int n, long long ld, float* __restrict__ dst) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  dst[j] += pl_tree_sum(rows, [&](int r) { return src[r * ld + j]; });
}

// ------------------------------------------------------------------------------------ per-row phases (warp per row)
__device__ __forceinline__ float pl_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float pl_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// dL/dq of row r: the loss weights q_r / scale by rho^t / (T B) with a minus sign (t = r / B)
__device__ __forceinline__ float pl_row_weight(int r, int Bsz, int Tsz, float rho) {
  return powf(rho, static_cast<float>(r / Bsz)) / (static_cast<float>(Tsz) * static_cast<float>(Bsz));
}

// Per row r and head slot u = blockIdx.y: q_u = symexp(sum_i softmax(l)_i bins_i), q = (q_0 + q_1) / 2.
//   dl[u][r][i] = dq_u exp(|s|) p_i (bins_i - s), s = sum_i p_i bins_i, dq_u = -w_r / (2 scale)
__global__ void __launch_bounds__(256) pl_q_head_back(const float* __restrict__ tape, int pitch, int off0, int off1, int rows,
                                                      int nb, const float* __restrict__ bins, const float* __restrict__ scale,
                                                      int Bsz, int Tsz, float rho, float* __restrict__ dl) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, u = blockIdx.y;
  if (r >= rows) return;
  const float* l = tape + static_cast<size_t>(r) * pitch + (u == 0 ? off0 : off1);
  float m = -INFINITY;
  for (int i = lane; i < nb; i += 32) m = fmaxf(m, l[i]);
  m = pl_warp_max(m);
  float den = 0.f, num = 0.f;
  for (int i = lane; i < nb; i += 32) { const float e = expf(l[i] - m); den += e; num = fmaf(e, bins[i], num); }
  den = pl_warp_sum(den);
  const float sbar = pl_warp_sum(num) / den;
  const float ds = -0.5f * pl_row_weight(r, Bsz, Tsz, rho) / scale[0] * expf(fabsf(sbar));
  float* o = dl + (static_cast<size_t>(u) * rows + r) * nb;
  for (int i = lane; i < nb; i += 32) o[i] = ds * (expf(l[i] - m) / den) * (bins[i] - sbar);
}

// LayerNorm + Mish backward of one hidden layer, per row r and batch u = blockIdx.y (head slot: gamma / beta / dropout
// rows of head hsel[u]).  pre = the tape's pre-LayerNorm row, g = dL/dh of h = mish(gamma n + beta).
//   dy = g mish'(y); dn = dy gamma; dpre = rstd (dn - mean(dn) - n mean(dn n)) [* dropout scale] -> out (may alias g)
// Optional per-row outputs: dyn = dy n and dy (the dgamma / dbeta terms), h (the activation, for dW of the next layer).
struct LnBackArgs {
  const float* tape; int pitch; int off; long long off_z;   // pre row of batch u: tape + r pitch + off + u off_z
  const float* g; float* out; long long ld, g_z;            // [rows, ld] per batch, batch stride g_z
  const float* gamma; const float* beta; const int* hsel;   // [heads, N]
  const float* drop;                                        // dropout scale [heads, rows, N] or nullptr
  float* dyn; float* dy; float* h;                          // [rows, ld] or nullptr
  int rows, N;
  long long o_z;                                            // batch stride of dyn / dy / h (0: shared by every batch)
};
__global__ void __launch_bounds__(256) pl_ln_back(const LnBackArgs a) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, u = blockIdx.y;
  if (r >= a.rows) return;
  const int hd = a.hsel ? a.hsel[u] : 0;
  const float* pre = a.tape + static_cast<size_t>(r) * a.pitch + a.off + u * a.off_z;
  const float* gm = a.gamma + static_cast<size_t>(hd) * a.N;
  const float* bt = a.beta + static_cast<size_t>(hd) * a.N;
  const float* g = a.g + u * a.g_z + static_cast<size_t>(r) * a.ld;
  float* out = a.out + u * a.g_z + static_cast<size_t>(r) * a.ld;
  const float invN = 1.f / static_cast<float>(a.N);
  float s = 0.f;
  for (int j = lane; j < a.N; j += 32) s += pre[j];
  const float mean = pl_warp_sum(s) * invN;
  float sq = 0.f;
  for (int j = lane; j < a.N; j += 32) { const float d = pre[j] - mean; sq = fmaf(d, d, sq); }
  const float rstd = 1.f / sqrtf(pl_warp_sum(sq) * invN + 1e-5f);
  float s1 = 0.f, s2 = 0.f;
  for (int j = lane; j < a.N; j += 32) {
    const float n = (pre[j] - mean) * rstd, y = fmaf(n, gm[j], bt[j]);
    const float e = expf(y), q = e * (e + 2.f), t = y > 20.f ? 1.f : q / (q + 2.f);   // tanh(softplus(y))
    const float sg = 1.f / (1.f + expf(-y));
    const float dy = g[j] * (t + y * sg * (1.f - t * t));
    const float dn = dy * gm[j];
    s1 += dn; s2 = fmaf(dn, n, s2);
    const size_t o = u * a.o_z + static_cast<size_t>(r) * a.ld + j;
    if (a.dyn) { a.dyn[o] = dy * n; a.dy[o] = dy; }
    if (a.h) a.h[o] = y > 20.f ? y : y * t;
    out[j] = dn;                 // dn parked in out until the row's two sums are known (out may alias g: g[j] is read)
  }
  s1 = pl_warp_sum(s1) * invN;
  s2 = pl_warp_sum(s2) * invN;
  const float* dr = a.drop ? a.drop + (static_cast<size_t>(hd) * a.rows + r) * a.N : nullptr;
  __syncwarp();
  for (int j = lane; j < a.N; j += 32) {
    const float n = (pre[j] - mean) * rstd;
    float d = rstd * (out[j] - s1 - n * s2);
    if (dr) d *= dr[j];
    out[j] = d;
  }
}

// The tanh-Gaussian head (world_model.py:144-184, math.py:12-29) backward, per row.  Recomputes from the head's taped
// logits and eps what rows_pi computed: ls = lo + dif/2 (tanh(x) + 1); masked mu, ls, eps; lp = sum(-eps^2/2 - ls - c);
// a = tanh(mu + eps exp(ls)); sq = sum log(relu(1 - a^2) + 1e-6); log_pi = lp - sq;
// scaled_entropy = -log_pi (lp size / (log_pi + 1e-8)).  dL/da arrives from the Q heads (da_q, columns a_off.. of both
// head slots); dL/dscaled_entropy = -entropy_coef w_r.  Writes dL/dlogits [rows, 2A] in the state dict's row order.
struct PiHeadArgs {
  const float* tape; int pitch, off_h, Apad;
  const float* eps; const int* task; const float* masks;    // masks [tasks, A] or nullptr
  const float* da_q; long long da_ld, da_z; int a_off;
  float log_std_min, log_std_dif, entropy_coef, rho;
  const float* scale;
  int rows, A, Bsz, Tsz;
  float* dlog;
};
__global__ void __launch_bounds__(256) pl_pi_head_back(const PiHeadArgs p) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= p.rows) return;
  const float* lg = p.tape + static_cast<size_t>(r) * p.pitch + p.off_h;
  const int task = p.task ? p.task[r] : 0;
  const float* mk = p.masks ? p.masks + static_cast<size_t>(task) * p.A : nullptr;
  float lp = 0.f, sq = 0.f, size = 0.f;
  for (int a = lane; a < p.A; a += 32) {
    const float m = mk ? mk[a] : 1.f;
    const float ls = (p.log_std_min + 0.5f * p.log_std_dif * (tanhf(lg[p.Apad + a]) + 1.f)) * m;
    const float e = p.eps[static_cast<size_t>(r) * p.A + a] * m;
    lp += -0.5f * e * e - ls - 0.9189385175704956f;
    const float act = tanhf(lg[a] * m + e * expf(ls));
    sq += logf(fmaxf(1.f - act * act, 0.f) + 1e-6f);
    size += m;
  }
  lp = pl_warp_sum(lp); sq = pl_warp_sum(sq); size = pl_warp_sum(size);
  const float log_pi = lp - sq, D = log_pi + 1e-8f, slp = lp * size;
  const float dse = -p.entropy_coef * pl_row_weight(r, p.Bsz, p.Tsz, p.rho);
  const float dlog_pi = dse * (-(slp / D) + log_pi * slp / (D * D));
  const float dlp = dlog_pi + dse * (-log_pi / D) * size;
  const float dsq = -dlog_pi;
  float* o = p.dlog + static_cast<size_t>(r) * 2 * p.A;
  for (int a = lane; a < p.A; a += 32) {
    const float m = mk ? mk[a] : 1.f;
    const float th = tanhf(lg[p.Apad + a]);
    const float ls = (p.log_std_min + 0.5f * p.log_std_dif * (th + 1.f)) * m;
    const float e = p.eps[static_cast<size_t>(r) * p.A + a] * m;
    const float sd = expf(ls);
    const float act = tanhf(lg[a] * m + e * sd);
    const float om = 1.f - act * act;
    const size_t qa = static_cast<size_t>(r) * p.da_ld + p.a_off + a;
    float dact = p.da_q[qa] + p.da_q[p.da_z + qa];
    if (om > 0.f) dact += dsq * (-2.f * act) / (om + 1e-6f);
    const float du = dact * om;
    const float dls = du * e * sd - dlp;
    o[a] = du * m;
    o[p.A + a] = dls * m * 0.5f * p.log_std_dif * (1.f - th * th);
  }
}

// x[r] = [z_r | emb_{task[r]}]: the input of pi layer 0 (emb = the max_norm-renormalised rows the forward read)
__global__ void pl_gather_x(const float* __restrict__ z, const float* __restrict__ emb, const int* __restrict__ task, int rows,
                            int L, int T, float* __restrict__ x) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(rows) * (L + T)) return;
  const int r = static_cast<int>(i / (L + T)), c = static_cast<int>(i % (L + T));
  x[i] = c < L ? z[static_cast<size_t>(r) * L + c] : emb[static_cast<size_t>(task[r]) * T + c - L];
}

// dst[t][c] += sum over rows r with task[r] == t (pl_tree_sum) of sum_i src_i[r][c], i over the three [rows, ld] sources
__global__ void pl_emb_grad(const float* __restrict__ s0, const float* __restrict__ s1, const float* __restrict__ s2,
                            long long ld, const int* __restrict__ task, int rows, int tasks, int T, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tasks * T) return;
  const int t = i / T, cc = i % T;
  dst[i] += pl_tree_sum(rows, [&](int r) {
    return task[r] == t ? (s0[r * ld + cc] + s1[r * ld + cc]) + s2[r * ld + cc] : 0.f;
  });
}

// ------------------------------------------------------------------------------------ agent._update (world-model loss)
// The backward of the reference's _update loss (tdmpc2.py:259-313) from the tapes of the row ops ENCODE / NEXT / REWARD /
// Q_ALL / TERM (api.cu, tdmpc2_wm_loss_backward): the heads' row gradients below, then the generic GEMM / LayerNorm
// kernels above through the heads, back through time over the dynamics, and through the encoder.

// Soft cross-entropy backward (math.py:33-37, 58-71) per row r and batch u = blockIdx.y (Q head, or the reward head):
//   tw = two_hot(target_r); dl = w_r (softmax(l) sum(tw) - tw), w_r = coef rho^(r / Bsz)
// two_hot as the reference computes it in fp32: symlog, clamp to [vmin, vmax], divide by bin_size, floor, and the lower
// bin's neighbour at (idx + 1) % nb.
__global__ void __launch_bounds__(256) pl_soft_ce_back(const float* __restrict__ logits, long long l_z, int rows, int nb,
                                                       const float* __restrict__ target, float vmin, float vmax, float bin_size,
                                                       float coef, float rho, int Bsz, float* __restrict__ dl) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, u = blockIdx.y;
  if (r >= rows) return;
  const float* l = logits + u * l_z + static_cast<size_t>(r) * nb;
  const float y = target[r];
  const float sl = copysignf(logf(1.f + fabsf(y)), y);                                // sign(x) log(1 + |x|)
  const float x = fminf(fmaxf(sl, vmin), vmax);
  const float pos = (x - vmin) / bin_size;
  const float fidx = floorf(pos);
  const float off = pos - fidx;
  const int i0 = static_cast<int>(fidx), i1 = (i0 + 1) % nb;
  const float sum_tw = (1.f - off) + off;
  float m = -INFINITY;
  for (int i = lane; i < nb; i += 32) m = fmaxf(m, l[i]);
  m = pl_warp_max(m);
  float den = 0.f;
  for (int i = lane; i < nb; i += 32) den += expf(l[i] - m);
  den = pl_warp_sum(den);
  const float w = coef * powf(rho, static_cast<float>(r / Bsz));
  float* o = dl + u * l_z + static_cast<size_t>(r) * nb;
  for (int i = lane; i < nb; i += 32) {
    const float tw = i == i0 ? 1.f - off : i == i1 ? off : 0.f;
    o[i] = w * (expf(l[i] - m) / den * sum_tw - tw);
  }
}

// BCE-with-logits backward (mean over rows): dl = coef (sigmoid(l) - y)
__global__ void pl_bce_back(const float* __restrict__ l, const float* __restrict__ y, int rows, float coef, float* __restrict__ dl) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  dl[r] = coef * (1.f / (1.f + expf(-l[r])) - y[r]);
}

// LayerNorm + SimNorm backward of the encoder's / the dynamics' last layer, per row r (a.hsel, a.drop unused).  From the
// tape's pre row: n = LayerNorm(pre), y = gamma n + beta, s = softmax of y over groups of V columns.  g = dL/ds:
//   dy = s (g - sum_grp s g); dn = dy gamma; dpre = rstd (dn - mean(dn) - n mean(dn n)) -> out (may alias g)
// Each lane owns whole groups (lane + 32 k), so the group sums stay in the lane.
__global__ void __launch_bounds__(256) pl_ln_simnorm_back(const LnBackArgs a, int V) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= a.rows) return;
  const float* pre = a.tape + static_cast<size_t>(r) * a.pitch + a.off;
  const float* g = a.g + static_cast<size_t>(r) * a.ld;
  float* out = a.out + static_cast<size_t>(r) * a.ld;
  const float invN = 1.f / static_cast<float>(a.N);
  float s = 0.f;
  for (int j = lane; j < a.N; j += 32) s += pre[j];
  const float mean = pl_warp_sum(s) * invN;
  float sq = 0.f;
  for (int j = lane; j < a.N; j += 32) { const float d = pre[j] - mean; sq = fmaf(d, d, sq); }
  const float rstd = 1.f / sqrtf(pl_warp_sum(sq) * invN + 1e-5f);
  float s1 = 0.f, s2 = 0.f;
  for (int c0 = lane * V; c0 < a.N; c0 += 32 * V) {
    float mx = -INFINITY;
    for (int j = c0; j < c0 + V; ++j) mx = fmaxf(mx, fmaf((pre[j] - mean) * rstd, a.gamma[j], a.beta[j]));
    float den = 0.f, sg = 0.f;
    for (int j = c0; j < c0 + V; ++j) {
      const float e = expf(fmaf((pre[j] - mean) * rstd, a.gamma[j], a.beta[j]) - mx);
      den += e; sg = fmaf(e, g[j], sg);
    }
    sg /= den;
    for (int j = c0; j < c0 + V; ++j) {
      const float n = (pre[j] - mean) * rstd;
      const float sm = expf(fmaf(n, a.gamma[j], a.beta[j]) - mx) / den;
      const float dy = sm * (g[j] - sg);
      const float dn = dy * a.gamma[j];
      s1 += dn; s2 = fmaf(dn, n, s2);
      const size_t o = static_cast<size_t>(r) * a.ld + j;
      if (a.dyn) { a.dyn[o] = dy * n; a.dy[o] = dy; }
      out[j] = dn;
    }
  }
  s1 = pl_warp_sum(s1) * invN;
  s2 = pl_warp_sum(s2) * invN;
  __syncwarp();
  for (int c0 = lane * V; c0 < a.N; c0 += 32 * V)
    for (int j = c0; j < c0 + V; ++j) out[j] = rstd * (out[j] - s1 - (pre[j] - mean) * rstd * s2);
}

// dL/dz_t [Bsz, L] of rollout step t (row r = t Bsz + b of the [H, Bsz] head batches):
//   consistency (t >= 1): cons rho^(t-1) (z_t - next_z_{t-1})      (cons = coef 2 / (H Bsz L))
//   + the Q heads' dX (t < H, heads in order) + the reward head's (t < H) + the termination head's (t >= 1, rows of
//   z_1..z_H) + dynamics step t's (t < H); dX of the heads and dynamics carry ld columns, z first.
struct DzArgs {
  const float* zs; const float* next_z;
  const float* dxq; long long q_z; int nq; const float* dxr; const float* dxd; long long ld;
  const float* dxt; long long ldt;
  float cons, rho;
  int t, H, Bsz, L;
  float* dz;
};
__global__ void pl_dz_step(const DzArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.Bsz * a.L) return;
  const int b = i / a.L, c = i % a.L;
  float v = 0.f;
  if (a.t >= 1) {
    const size_t zi = (static_cast<size_t>(a.t) * a.Bsz + b) * a.L + c, ni = (static_cast<size_t>(a.t - 1) * a.Bsz + b) * a.L + c;
    v = a.cons * powf(a.rho, static_cast<float>(a.t - 1)) * (a.zs[zi] - a.next_z[ni]);
  }
  if (a.t < a.H) {
    const size_t row = static_cast<size_t>(a.t) * a.Bsz + b;
    for (int q = 0; q < a.nq; ++q) v += a.dxq[q * a.q_z + row * a.ld + c];
    v += a.dxr[row * a.ld + c];
    v += a.dxd[row * a.ld + c];
  }
  if (a.t >= 1 && a.dxt) v += a.dxt[(static_cast<size_t>(a.t - 1) * a.Bsz + b) * a.ldt + c];
  a.dz[i] = v;
}

// x[r] = [z_r | emb_{task[r]} | a_r]: the input of dynamics / reward / Q layer 0 (T == 0: no embedding columns)
__global__ void pl_gather_xa(const float* __restrict__ z, const float* __restrict__ emb, const int* __restrict__ task,
                             const float* __restrict__ act, int rows, int L, int T, int A, float* __restrict__ x) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int D = L + T + A;
  if (i >= static_cast<long long>(rows) * D) return;
  const int r = static_cast<int>(i / D), c = static_cast<int>(i % D);
  x[i] = c < L ? z[static_cast<size_t>(r) * L + c]
       : c < L + T ? emb[static_cast<size_t>(task[r]) * T + c - L] : act[static_cast<size_t>(r) * A + c - L - T];
}

__global__ void pl_iota(int* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = i;
}

}  // namespace tdmpc2
