// Fused planning kernels for sm_90a (H100).
//
// One persistent kernel template, `plan_kernel<ENGINE, EPISODIC>`, runs the MLP chains of the TD-MPC2 planner on
// 128-row tiles (EPISODIC = termination head in the rollout; compile-time so that an unused feature costs no code).
// All modes share the device code:
//
//   MODE_ENCODE : rows = environments.      z = encode(obs, task)        (reference world_model.py:103-112)
//   MODE_PRIOR  : rows = (env, pi-traj).    the P policy-prior rollouts  (reference tdmpc2.py:154-160)
//   MODE_ITER   : rows = (env, sample).     ONE CEM iteration:           (reference tdmpc2.py:173-197)
//                   sample actions -> H x (reward, dynamics) -> terminal pi -> 2 Q heads
//                   -> value -> [last tile of an env] top-k, MPPI weights, mean/std refit.
//   MODE_VALUE  : MODE_ITER's rollout on caller-given z / actions, no refit (reference tdmpc2.py:122-136)
//   MODE_LAYER  : one layer, for diagnostics.
//   MODE_ROWS   : rows = the caller's flat batch (row r: tile r / 128, tile row r % 128).  ONE world-model method per
//                 launch (RowOp: encode / next / reward / termination / pi / Q / TD target, reference
//                 world_model.py:103-216, tdmpc2.py:242-257).  Its own instantiation plan_kernel<ENGINE, false, true>:
//                 the planning instantiations do not carry its code.  It touches no planner state, only the per-slot
//                 X / H / raw scratch, which is dead between launches.
//
// Every dense layer is `acc = A[128, Kpad] * W[Npad, Kpad]^T` with both operands stored as two fp16 planes (hi, lo;
// x ~= hi + lo to ~22 bits).  A CTA is 384 threads (12 warps).  The tensor-core engine (ENGINE_TC) streams 64-element
// K-chunks of both operands with TMA (128-byte swizzle) through a 3-stage mbarrier ring (warp 8 = producer, warps 9-11
// idle during the GEMM) into two consumer warpgroups (warps 0-7), each of which owns 64 rows x all 128 columns of every
// 128 x 128 output block and runs wgmma (m64n128k16) A_lo*W_hi + A_hi*W_lo + A_hi*W_hi per K-chunk into fresh fp32
// registers; the K-chunk partials are added with round-to-nearest and the block goes to an fp32 scratch row buffer in
// global memory.  The SIMT engine computes the same sums with FFMA on CUDA cores.  Both engines then run the same row
// phases (all 12 warps, warp per row): bias + LayerNorm + Mish / SimNorm, two-hot-inverse, tanh-Gaussian sampling, and
// emit the next layer's fp16 planes.
//
// Activations live in a per-CTA scratch slot (global memory: X planes +
// one in-place hidden buffer, 0.56 MB per slot for the 5M model).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "ptx.cuh"
#include "rng.cuh"

namespace tdmpc2 {

constexpr int kTileM = 128;       // rows per tile
constexpr int kKch = 64;          // K elements per pipeline stage (128 B of fp16: one swizzle row)
constexpr int kStages = 2;
constexpr int kAPlane = kTileM * 128;           // 16 KiB: one 128-row plane of a K-chunk
constexpr int kStageBytes = 6 * kAPlane;        // 96 KiB (the operand smem is kStages * kStageBytes = 192 KiB)
// Tensor-core engine: 3 ring stages of (A hi | A lo | W hi | W lo), 16 KiB each, inside the same 192 KiB.
constexpr int kGStages = 3;
constexpr int kGStageBytes = 4 * kAPlane;
constexpr int kGNb = 128;                        // output columns per block (W rows per stage)
constexpr int kGWarpGroups = 2;                  // consumer warps 0..7: warpgroup g owns rows 64 g.., all 128 columns
constexpr int kGProducerWarp = 4 * kGWarpGroups; // warp 8 issues the TMA loads; warps 9..11 idle during the GEMM
static_assert(kGStages * kGStageBytes <= kStages * kStageBytes, "operand smem layout");
constexpr int kThreads = 384;                   // 12 warps: __launch_bounds__(384, 1) leaves ptxas 168 registers per thread
constexpr int kWarps = kThreads / 32;
constexpr int kMaxWMaps = 8;
constexpr int kMaxHeadCols = 256;  // widest head output (2A or num_bins)
constexpr int kSmemCtrl = 2048;    // barriers, flags (256 B) + G[128] + q1[128] + term[128]
constexpr int kSmemRowBuf = kWarps * kMaxHeadCols * 4;  // one head-output row per warp
constexpr int kSmemRowEnv = kTileM * 4;                 // env index of each tile row
constexpr int kSmemBytes = kStages * kStageBytes + kSmemCtrl + kSmemRowBuf + kSmemRowEnv;

enum Mode { MODE_ENCODE = 0, MODE_PRIOR = 1, MODE_ITER = 2, MODE_VALUE = 3, MODE_LAYER = 4, MODE_ROWS = 5 };
// MODE_ROWS: which world-model method a launch runs (PlanParams::rop)
// ROP_PI_LOSS: agent.update_pi's forward (pi, then the online Q pair's average on pi's action) writing a tape
enum RowOp { ROP_ENCODE = 0, ROP_NEXT = 1, ROP_REWARD = 2, ROP_TERM = 3, ROP_PI = 4, ROP_Q_ALL = 5, ROP_Q_PAIR = 6, ROP_TD = 7,
             ROP_PI_LOSS = 8 };
enum Engine { ENGINE_TC = 0, ENGINE_SIMT = 1 };
// X = [z | emb | a] input planes; H = hidden planes.  ONE hidden buffer is enough: a layer's epilogue only runs after
// every MMA of its GEMM has consumed the A operand, so layer 1 overwrites its own input in place.
enum Buf { BUF_X = 0, BUF_H1 = 1 };
enum Epi { EPI_LN_MISH = 0, EPI_LN_SIMNORM = 1, EPI_TWOHOT = 2, EPI_PI = 3, EPI_RAW = 4, EPI_TERM = 5 };
enum HeadKind { HEAD_REWARD = 0, HEAD_Q1 = 1, HEAD_Q2 = 2 };

struct LayerDev {
  int K, Kpad, N, Npad;
  int wmap;          // which weight tensor map (Kpad class)
  int wrow;          // row of the hi plane inside that class tensor; lo plane at wrow + Npad
  int has_ln;
  float inv_scale;   // 2^-k; the packed planes hold W * 2^k (written by the pack kernel)
  const float* bias; // [Npad] zero padded
  const float* ln_g; // [Npad]
  const float* ln_b; // [Npad]
  const __half* w_hi;  // direct pointers (SIMT engine): [Npad][Kpad]
  const __half* w_lo;
};

struct PlanParams {
  CUtensorMap tmX;                 // [slots*2*128, KpadX] fp16, box 64 x 128
  CUtensorMap tmH;                 // [slots*2*128, KpadH]
  CUtensorMap tmW[kMaxWMaps];      // weights, one map per Kpad class, box 64 x 128
  const LayerDev* layers;
  int E, N, P, Ppad, K, H, obs_dim, A, Apad, L, M, T, B, num_q, simnorm, num_enc;   // Apad = pad32(A): the pi head's
                                                                                  // log_std logits start at column Apad
  int tiles_per_env, ntiles, KpadX, KpadH, NpadMax;
  int li_enc, li_dyn, li_rew, li_pi, li_q;
  float temperature, min_std, max_std, log_std_min, log_std_dif;
  __half* X; __half* Hb; float* raw;       // scratch, indexed by slot = blockIdx.x
  const float* emb; const float* masks; const float* disc_pow; const float* bins;
  int mode;
  // per-call inputs
  const float* obs; const int* task; const float* noise_prior; const float* noise_r; const float* noise_pi;
  const int* qidx; const float* z_rows; const float* actions_explicit;
  // planner state
  float* z; float* pi_actions; float* mean; float* std; float* values; unsigned* env_counter;
  float* score; float* elite_act0; int* elite_idx32;
  long long* elite_idx_out; float* values_out;
  // MODE_LAYER
  int dbg_layer, dbg_mode, dbg_rows; const float* dbg_x; float* dbg_y;
  long long* prof;   // optional [prof_slots][4][12] cycle counters + [32][16] trace stamps of CTA 0 (diagnostics), or nullptr
  int prof_slots;    // = number of scratch slots (SM count)
  int li_term;       // first of the 3 termination-head layers (cfg.episodic, world_model.py:28), or -1
  // Shared-latent fold (MODE_ITER, rollout step t = 0): every sample row of an environment carries the SAME [z | emb]
  // (z.repeat(N), tdmpc2.py:163), so the [z | emb] part of reward.0 / dynamics.0 is a per-environment vector.  The
  // prologue computes zbias[mlp][e][n] = bias[n] + sum_{k < 64 zb_kc0} [z | emb]_e[k] W[n][k] once per plan()
  // (zbias_kernel) and the t = 0 GEMMs of those two layers start at K-chunk zb_kc0 (the action columns) with that
  // vector as their bias.  zb_kc0 == 0: fold off.
  const float* zbias;   // [2 (0 reward, 1 dynamics)][E][zb_pitch]
  int zb_kc0, zb_pitch;
  // 3 = fp32-parity arithmetic (A_lo W_hi + A_hi W_lo + A_hi W_hi); 1 = the DECLARED NON-PARITY fast mode: hi planes only
  // (one fp16 MMA per product, fp32 accumulate), half the operand bytes.  tdmpc2_planner_set_passes.
  int passes;
  // Declared non-parity throughput mode (rng.cuh): non-null = the CEM iteration generates noise_r / noise_pi itself
  // (noise_r / noise_pi are null then); rng_iter = index of this iteration within the plan (selects the Philox stream)
  const unsigned long long* rng_state;
  int rng_iter;
  // MODE_ROWS (world-model methods on the caller's flat batch of `rows` rows; fp32 inputs / outputs, caller-owned)
  int rows, rop;
  int rows_flag;                   // ROP_TERM: 1 = sigmoid; ROP_Q_PAIR / ROP_TD: 0 = min of the two heads, 1 = average
  const float* rows_in;            // obs [rows, obs_dim] (ROP_ENCODE) or z [rows, L]
  const float* rows_act;           // a [rows, A]
  const float* rows_eps;           // pi noise [rows, A]
  const float* rows_reward;        // ROP_TD: reward [rows], terminated [rows]
  const float* rows_term;
  const LayerDev* rows_q;          // the 3 num_q layers of the Q ensemble this launch reads (online or target weights)
  float* rows_out;                 // z' / logits [rows, .]; Q all [num_q, rows, B]; pi action [rows, A]; Q pair / TD [rows]
  float* rows_out2;                // ROP_PI: tanh(mean) [rows, A]
  float* rows_out3;                // ROP_PI: log_std [rows, A]
  float* rows_out4;                // ROP_PI / ROP_PI_LOSS: [rows, 2] = (gaussian log-prob, sum of the squash terms)
  // ROP_PI_LOSS (rows_out = q [rows], rows_flag = 1)
  float* rows_tape;                // [rows, tape.pitch]: see PiTape
  float* rows_act_out;             // action [rows, A]
  const float* rows_drop;          // Q layer 0 dropout scale (mask / (1 - p)) [num_q, rows, M], or nullptr (eval mode)
  // Row pitch (floats) of rows_tape.  ROP_PI_LOSS: PiTape::pitch.  ROP_ENCODE / NEXT / REWARD / TERM / Q_ALL with a
  // non-null rows_tape (agent._update's forward): the pre-LayerNorm rows of every LayerNorm layer of the launch, see
  // WmTape in api.cu; Q_ALL also applies rows_drop to each head's layer 0 then.
  int tape_pitch;
};

// The tape of ROP_PI_LOSS, per row (fp32 offsets): the pre-LayerNorm rows of pi.0 and pi.1 [M], the pi head's logits
// [Apad + A] (log_std logits at column Apad, as in the kernel's head row), then for each selected Q head u the
// pre-LayerNorm rows of its layers 0 (after dropout) and 1 [M] and its logits [B]; the action [A] and q [1] last.
// The backward (grad_kernels.cuh) recomputes every LayerNorm / Mish value from it.
struct PiTape {
  int pi0, pi1, pih, q[2], act, qv, pitch;
};
__host__ __device__ inline PiTape pi_tape(int M, int A, int Apad, int B) {
  PiTape t;
  t.pi0 = 0; t.pi1 = M; t.pih = 2 * M;
  t.q[0] = t.pih + Apad + A; t.q[1] = t.q[0] + 2 * M + B;
  t.act = t.q[1] + 2 * M + B; t.qv = t.act + A;
  t.pitch = (t.qv + 1 + 3) & ~3;
  return t;
}

// The layer table lives in global memory; role loops are full of asm volatile(... "memory") (TMA issue, mbarrier waits,
// fences), each of which would force the compiler to re-read any field it needs afterwards -- a dependent global load
// in the single-thread producer / MMA loops and in the epilogue's inner loops.  Roles therefore work on a by-value copy.
struct LayerRec {
  int K, Kpad, N, Npad, wmap, wrow;
  float inv_scale;
  const float* bias; const float* ln_g; const float* ln_b;
  const __half* w_hi; const __half* w_lo;
};
__device__ __forceinline__ LayerRec layer_rec(const LayerDev& l) {
  LayerRec r;
  r.K = l.K; r.Kpad = l.Kpad; r.N = l.N; r.Npad = l.Npad; r.wmap = l.wmap; r.wrow = l.wrow; r.inv_scale = l.inv_scale;
  r.bias = l.bias; r.ln_g = l.ln_g; r.ln_b = l.ln_b; r.w_hi = l.w_hi; r.w_lo = l.w_lo;
  return r;
}

// What a layer's epilogue has to do besides the activation itself.
struct EpiArgs {
  int kind;                 // Epi
  int dstbuf;               // LN kinds: plane destination buffer (or -1)
  int dst_col0;
  float* out_f32;           // LN kinds / RAW: optional fp32 row output
  int out_pitch;
  const int* rowmap;        // smem [128]: output row of each tile row (or -1), for out_f32
  int head;                 // TWOHOT: HeadKind
  float disc;               // TWOHOT: discount factor applied to this head's value
  int tile;                 // TWOHOT / PI: tile index (row -> env mapping)
  const float* eps_base;    // PI: noise tensor, element (e*eps_rows + idx)*A + a
  int eps_rows;
  float* act_out;           // PI: optional pi_actions output
  int t_out;
  float* tape;              // MODE_ROWS ROP_PI_LOSS: this layer's tape segment of output row 0 (row pitch P.tape pitch)
  const float* drop;        // MODE_ROWS ROP_PI_LOSS, Q layer 0: dropout scale of output row 0 (row pitch N), or nullptr
};

// ------------------------------------------------------------------------------------ small math
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float symexp_f(float x) {   // math.py:50-55
  const float m = expf(fabsf(x)) - 1.f;
  return x > 0.f ? m : (x < 0.f ? -m : 0.f);
}
__device__ __forceinline__ void split_f(float x, __half& h, __half& l) {
  // finite values are clamped into fp16 range; NaN / +-inf stay non-finite so that they poison the row exactly
  // as they do in the reference (whose planner then zeroes the value: nan_to_num, tdmpc2.py:184)
  const bool finite = fabsf(x) <= 3.0e38f;
  x = fminf(fmaxf(x, -65000.f), 65000.f);
  h = finite ? __float2half_rn(x) : __ushort_as_half(static_cast<unsigned short>(0x7fff));
  l = __float2half_rn(finite ? x - __half2float(h) : 0.f);
}
__device__ __forceinline__ void split_store(__half* hi, __half* lo, float x) {
  __half h, l;
  split_f(x, h, l);
  *hi = h;
  *lo = l;
}
__device__ __forceinline__ float nan_to_num0(float v) {   // torch.nan_to_num(0): nan->0, +-inf -> +-FLT_MAX
  if (isnan(v)) return 0.f;
  if (isinf(v)) return v > 0.f ? 3.4028234663852886e38f : -3.4028234663852886e38f;
  return v;
}
__device__ __forceinline__ float4 lds128(const float* p) {   // p must point into shared memory, 16-byte aligned
  float4 r;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(ptx::smem_u32(p)));
  return r;
}
// Diagnostics (cycle counters per role, clock stamps per layer of CTA 0) exist only in builds with -DTDMPC2_PROF
// (tdmpc2_b200.build.build_variant("prof", ["TDMPC2_PROF=1"]), loaded through TDMPC2_B200_LIB): in the product build
// they compile to nothing -- the 8 per-thread 64-bit counters alone cost 16 registers of a 168-register budget.
#ifdef TDMPC2_PROF
constexpr bool kProf = true;
#else
constexpr bool kProf = false;
#endif
__device__ __forceinline__ long long prof_clock() { return kProf ? clock64() : 0ll; }
// Raw clock stamps of CTA 0 (events x layers) appended after the per-CTA counters.
#define TDMPC2_TRACE(P_, c_, ev_)                                                                         \
  do {                                                                                                    \
    if (kProf && (P_).prof && blockIdx.x == 0 && (c_).trace_step < 32)                                              \
      (P_).prof[static_cast<size_t>((P_).prof_slots) * 4 * 12 + (c_).trace_step * 16 + (ev_)] = prof_clock();                                  \
  } while (0)

// ------------------------------------------------------------------------------------ CTA context
struct Ctx {
  uint8_t* stage_base;      // kStages * kStageBytes, 1024-aligned
  uint64_t* g_full;         // [kGStages]  tensor-core engine: operand stage landed (TMA transaction bytes)
  uint64_t* g_empty;        // [kGStages]  tensor-core engine: operand stage consumed (one arrival per consumer warp)
  float* rowbuf;            // [kWarps][kMaxHeadCols]
  float* G;                 // [128] discounted reward sum
  float* q1;                // [128] first Q head
  float* term;              // [128] sticky termination flag of the row (episodic models, tdmpc2.py:126-134)
  int* flags;               // small ints
  int* rowenv;              // [128]
  int slot, warp, lane;
  // pipeline counters (each role keeps its own; persist across layers / tiles)
  uint32_t pa_it, ma_it;
  long long pf0, pf1, pf2, pf3, pf4, pf5, pf6, pf7;   // per-thread cycle accumulators (diagnostics)
  int trace_step;
};

__device__ __forceinline__ __half* plane_ptr(const PlanParams& P, int slot, int buf, int plane) {
  if (buf == BUF_X) return P.X + (static_cast<size_t>(slot) * 2 + plane) * kTileM * P.KpadX;
  return P.Hb + (static_cast<size_t>(slot) * 2 + plane) * kTileM * P.KpadH;
}
__device__ __forceinline__ int plane_pitch(const PlanParams& P, int buf) { return buf == BUF_X ? P.KpadX : P.KpadH; }
__device__ __forceinline__ int plane_row0(const PlanParams& P, int slot, int buf, int plane) {  // TMA row coord
  if (buf == BUF_X) return (slot * 2 + plane) * kTileM;
  return (slot * 2 + plane) * kTileM;
}
__device__ __forceinline__ float* raw_ptr(const PlanParams& P, int slot) {
  return P.raw + static_cast<size_t>(slot) * kTileM * P.NpadMax;
}

// ------------------------------------------------------------------------------------ row -> (env, sample) mapping
struct RowMap {
  int env;     // -1 if the row is padding
  int idx;     // sample index n (ITER/VALUE), pi-trajectory p (PRIOR), unused (ENCODE)
};
__device__ __forceinline__ RowMap map_row(const PlanParams& P, int tile, int r) {
  RowMap m;
  if (P.mode == MODE_ENCODE) {
    m.env = tile * kTileM + r; m.idx = 0;
    if (m.env >= P.E) m.env = -1;
  } else if (P.mode == MODE_PRIOR) {
    const int per = kTileM / P.Ppad;
    m.env = tile * per + r / P.Ppad; m.idx = r % P.Ppad;
    if (m.env >= P.E || m.idx >= P.P) m.env = -1;
  } else {
    m.env = tile / P.tiles_per_env; m.idx = (tile % P.tiles_per_env) * kTileM + r;
    if (m.idx >= P.N) m.env = -1;
  }
  return m;
}

// In-kernel noise (rng.cuh): group indices.  noise_r element (e, t, n, a), n >= P: group ((e H + t) N + n) A4 + a / 4 of
// stream 2 iter; noise_pi element (e, n, a): group (e N + n) A4 + a / 4 of stream 2 iter + 1; A4 = ceil(A / 4).
__device__ __forceinline__ unsigned long long rng_group_r(const PlanParams& P, int e, int t, int n, int a4) {
  return ((static_cast<unsigned long long>(e) * P.H + t) * P.N + n) * static_cast<unsigned>((P.A + 3) >> 2) + a4;
}
__device__ __forceinline__ unsigned long long rng_group_pi(const PlanParams& P, int e, int n, int a4) {
  return (static_cast<unsigned long long>(e) * P.N + n) * static_cast<unsigned>((P.A + 3) >> 2) + a4;
}
__device__ __forceinline__ float noise_r_at(const PlanParams& P, int e, int t, int n, int a) {
  if (P.rng_state) return rng_pick(rng_normal4(P.rng_state, 2u * P.rng_iter, rng_group_r(P, e, t, n, a >> 2)), a & 3);
  return __ldcs(&P.noise_r[((static_cast<size_t>(e) * P.H + t) * (P.N - P.P) + (n - P.P)) * P.A + a]);
}
__device__ __forceinline__ float noise_pi_at(const PlanParams& P, int e, int n, int a) {      // MODE_ITER / VALUE terminal policy sample
  if (P.rng_state) return rng_pick(rng_normal4(P.rng_state, 2u * P.rng_iter + 1u, rng_group_pi(P, e, n, a >> 2)), a & 3);
  return __ldcs(&P.noise_pi[(static_cast<size_t>(e) * P.N + n) * P.A + a]);
}

// action a_t of sample n of env e at CEM time (tdmpc2.py:168-181)
__device__ __forceinline__ float sample_action(const PlanParams& P, int e, int t, int n, int a, int task) {
  float v;
  if (P.actions_explicit) {
    return P.actions_explicit[((static_cast<size_t>(e) * P.H + t) * P.N + n) * P.A + a];
  } else if (n < P.P) {
    v = P.pi_actions[((static_cast<size_t>(e) * P.H + t) * P.P + n) * P.A + a];
  } else {
    const size_t sa = (static_cast<size_t>(e) * P.H + t) * P.A + a;
    const float r = noise_r_at(P, e, t, n, a);
    v = __fadd_rn(P.mean[sa], __fmul_rn(P.std[sa], r));       // mean + std * r, two roundings like eager torch
    v = fminf(fmaxf(v, -1.f), 1.f);
  }
  if (P.masks) v *= P.masks[static_cast<size_t>(task) * P.A + a];
  return v;
}

// ------------------------------------------------------------------------------------ shared per-row commits
// Value bookkeeping of _estimate_value (tdmpc2.py:128-136) for one row; called by exactly one thread per row.
template <bool EPISODIC>
__device__ __forceinline__ void head_commit(const PlanParams& P, Ctx& c, const EpiArgs& ea, int r, float val) {
  // discount * (1 - termination), tdmpc2.py:130,136 (termination is identically 0 unless cfg.episodic)
  const float disc = EPISODIC ? __fmul_rn(ea.disc, __fsub_rn(1.f, c.term[r])) : ea.disc;
  if (ea.head == HEAD_REWARD) {
    c.G[r] = __fadd_rn(c.G[r], __fmul_rn(disc, val));                 // G + discount * reward
  } else if (ea.head == HEAD_Q1) {
    c.q1[r] = val;
  } else {
    const float qavg = __fmul_rn(__fadd_rn(c.q1[r], val), 0.5f);      // Q.sum(0) / 2
    float v = __fadd_rn(c.G[r], __fmul_rn(disc, qavg));               // G + discount * Q
    if (P.mode == MODE_ITER) v = nan_to_num0(v);                        // tdmpc2.py:184
    const RowMap rm = map_row(P, ea.tile, r);
    if (rm.env >= 0) {
      float* dst = (P.mode == MODE_ITER) ? P.values : P.values_out;
      dst[static_cast<size_t>(rm.env) * P.N + rm.idx] = v;
    }
  }
}
// termination = clip(termination + (sigmoid(logit) > 0.5), max=1)  (tdmpc2.py:133-134, world_model.py:132-141).
// torch's fp32 sigmoid returns exactly 0.5 for |x| < ~3e-8, so "> 0.5" is evaluated on the same expression.
__device__ __forceinline__ void term_commit(Ctx& c, int r, float logit) {
  const float sg = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-logit)));
  c.term[r] = fminf(__fadd_rn(c.term[r], sg > 0.5f ? 1.f : 0.f), 1.f);
}
// a = tanh(mean + eps * exp(log_std)) for one (row, action dim)  (world_model.py:151-174)
__device__ __forceinline__ float pi_action(const PlanParams& P, float mu, float ls, float eps, int task, int a) {
  // log_std = low + 0.5 * dif * (tanh(x) + 1)   (math.py:12-13)
  ls = __fadd_rn(P.log_std_min, __fmul_rn(__fmul_rn(0.5f, P.log_std_dif), __fadd_rn(tanhf(ls), 1.f)));
  if (P.masks) { const float mk = P.masks[static_cast<size_t>(task) * P.A + a]; mu *= mk; ls *= mk; eps *= mk; }
  return tanhf(__fadd_rn(mu, __fmul_rn(eps, expf(ls))));
}

// ------------------------------------------------------------------------------------ tensor-core engine: GEMM -> raw scratch
// raw[128, Npad] = A[128, Kpad] * W[Npad, Kpad]^T over K-chunks [kc0, Kpad / 64), through TMA and wgmma (see the top of
// this file).  Each K-chunk (12 wgmma: A_lo*W_hi + A_hi*W_lo + A_hi*W_hi, small terms first, 4 K-steps of 16) is
// accumulated into zeroed registers and then added to the running sum with round-to-nearest, so that a long reduction
// does not inherit the tensor core's internal accumulation rounding.  passes == 1: A_hi*W_hi only, hi planes only.
__device__ __forceinline__ void gemm_tc(const PlanParams& P, Ctx& c, const LayerRec& ly, int srcbuf, int kc0 = 0) {
  const int kc1 = ly.Kpad / kKch;
  const int nnb = ly.Npad / kGNb;
  const bool lo = P.passes != 1;
  if (c.warp == kGProducerWarp) {
    const CUtensorMap* tmA = (srcbuf == BUF_X) ? &P.tmX : &P.tmH;
    const CUtensorMap* tmW = &P.tmW[ly.wmap];
    const int arow_hi = plane_row0(P, c.slot, srcbuf, 0), arow_lo = plane_row0(P, c.slot, srcbuf, 1);
    for (int nb = 0; nb < nnb; ++nb) {
      const int wr = ly.wrow + nb * kGNb;
      for (int kc = kc0; kc < kc1; ++kc) {
        const uint32_t s = c.pa_it % kGStages, ph = (c.pa_it / kGStages) & 1;
        const long long tw = prof_clock();
        ptx::mbar_wait(&c.g_empty[s], ph ^ 1);
        c.pf0 += prof_clock() - tw;
        if (ptx::elect_one()) {
          uint8_t* st = c.stage_base + s * kGStageBytes;
          ptx::mbar_expect_tx(&c.g_full[s], (lo ? 4 : 2) * kAPlane);
          ptx::tma_load_2d(tmA, &c.g_full[s], st, kc * kKch, arow_hi);
          ptx::tma_load_2d(tmW, &c.g_full[s], st + 2 * kAPlane, kc * kKch, wr);
          if (lo) {
            ptx::tma_load_2d(tmA, &c.g_full[s], st + kAPlane, kc * kKch, arow_lo);
            ptx::tma_load_2d(tmW, &c.g_full[s], st + 3 * kAPlane, kc * kKch, wr + ly.Npad);
          }
        }
        __syncwarp();
        ++c.pa_it;
      }
    }
  } else if (c.warp < kGProducerWarp) {
    const int t = threadIdx.x & 127;
    const int r0 = (c.warp >> 2) * 64;
    const int row = r0 + (t >> 5) * 16 + ((t & 31) >> 2), col = 2 * (t & 3);
    float* rawbase = raw_ptr(P, c.slot);
    const uint32_t sbase = ptx::smem_u32(c.stage_base);
    for (int nb = 0; nb < nnb; ++nb) {
      float sum[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) sum[i] = 0.f;
      for (int kc = kc0; kc < kc1; ++kc) {
        const uint32_t s = c.ma_it % kGStages, ph = (c.ma_it / kGStages) & 1;
        const long long tw = prof_clock();
        ptx::mbar_wait(&c.g_full[s], ph);
        c.pf2 += prof_clock() - tw;
        const uint32_t sa = sbase + s * kGStageBytes + r0 * 128, sw = sbase + s * kGStageBytes + 2 * kAPlane;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        ptx::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kKch / 16; ++ks) {
          const uint64_t a_hi = ptx::make_sw128_kmajor_desc(sa + ks * 32), w_hi = ptx::make_sw128_kmajor_desc(sw + ks * 32);
          if (lo) {
            ptx::wgmma_m64n128k16(acc, ptx::make_sw128_kmajor_desc(sa + kAPlane + ks * 32), w_hi);
            ptx::wgmma_m64n128k16(acc, a_hi, ptx::make_sw128_kmajor_desc(sw + kAPlane + ks * 32));
          }
          ptx::wgmma_m64n128k16(acc, a_hi, w_hi);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (c.lane == 0) ptx::mbar_arrive(&c.g_empty[s]);     // this warp's reads of the stage are complete
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
        ++c.ma_it;
      }
      float* o = rawbase + static_cast<size_t>(row) * P.NpadMax + nb * kGNb + col;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        __stcg(reinterpret_cast<float2*>(o + 8 * j), make_float2(sum[4 * j], sum[4 * j + 1]));
        __stcg(reinterpret_cast<float2*>(o + 8 * static_cast<size_t>(P.NpadMax) + 8 * j), make_float2(sum[4 * j + 2], sum[4 * j + 3]));
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------ SIMT engine: GEMM -> raw scratch
// Same operands, plain fp32 FFMA on CUDA cores (exact products of the split operands).
__device__ __forceinline__ void gemm_simt(const PlanParams& P, Ctx& c, const LayerRec& ly, int srcbuf, int kc0 = 0) {
  constexpr int BN = 64, BK = 32;
  float* sA = reinterpret_cast<float*>(c.stage_base);          // [BK][128+4]
  float* sW = sA + BK * (kTileM + 4);                          // [BK][BN+4]
  const __half* a_hi = plane_ptr(P, c.slot, srcbuf, 0);
  const __half* a_lo = plane_ptr(P, c.slot, srcbuf, 1);
  const int pitch = plane_pitch(P, srcbuf);
  const int tid = threadIdx.x;
  const int tr = ((tid & 255) / 16) * 8, tc = (tid % 16) * 4;   // 8 rows x 4 cols per thread (threads 0..255)
  float* rawbase = raw_ptr(P, c.slot);
  for (int n0 = 0; n0 < ly.Npad; n0 += BN) {
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = kc0 * kKch; k0 < ly.Kpad; k0 += BK) {
      for (int i = tid; i < kTileM * BK; i += kThreads) {
        const int r = i / BK, k = i % BK;
        const size_t o = static_cast<size_t>(r) * pitch + k0 + k;
        sA[k * (kTileM + 4) + r] = __half2float(__ldcg(a_hi + o)) + __half2float(__ldcg(a_lo + o));
      }
      for (int i = tid; i < BN * BK; i += kThreads) {
        const int n = i / BK, k = i % BK;
        const size_t o = static_cast<size_t>(n0 + n) * ly.Kpad + k0 + k;
        sW[k * (BN + 4) + n] = __half2float(ly.w_hi[o]) + __half2float(ly.w_lo[o]);
      }
      __syncthreads();
      if (tid < 256) {
#pragma unroll 4
        for (int k = 0; k < BK; ++k) {
          float a[8], w[4];
#pragma unroll
          for (int i = 0; i < 8; ++i) a[i] = sA[k * (kTileM + 4) + tr + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) w[j] = sW[k * (BN + 4) + tc + j];
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
      }
      __syncthreads();
    }
    if (tid < 256) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          __stcg(rawbase + static_cast<size_t>(tr + i) * P.NpadMax + n0 + tc + j, acc[i][j]);
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------ row phases (warp per row)
// SimNorm (layers.py:74-88) of one lane's column: softmax over groups of 8 consecutive columns = 8 adjacent lanes.
__device__ __forceinline__ float simnorm_lane(float y, bool valid) {
  float m = valid ? y : -CUDART_INF_F;
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
  const float e = valid ? expf(y - m) : 0.f;
  float t = e;
  t += __shfl_xor_sync(0xffffffffu, t, 1);
  t += __shfl_xor_sync(0xffffffffu, t, 2);
  t += __shfl_xor_sync(0xffffffffu, t, 4);
  return valid ? __fdiv_rn(e, t) : 0.f;
}

constexpr int kLnRegCols = 16;   // columns per lane of a 512-wide row
constexpr int kLnBatch = 8;      // columns per lane that the output pass carries through activation and stores at once

// Row staging.  A row phase is latency-bound: a warp that loads a row when it starts on it waits for an L2 round trip
// per row.  The operand ring is idle from the end of a GEMM (its __syncthreads: every TMA load has landed and been
// consumed) to the next layer's first TMA load (after publish_planes' proxy fence and barrier), so each warp owns two
// kStageCols-float buffers there.  While the warp works on row r from one, cp.async (L2 only, no registers held) copies
// row r + kWarps of raw into the other.
constexpr int kStageCols = 512;
static_assert(kWarps * 2 * kStageCols * 4 <= kStages * kStageBytes, "row staging buffers");
__device__ __forceinline__ float* row_stage(const Ctx& c, int i) {
  return reinterpret_cast<float*>(c.stage_base) + (c.warp * 2 + (i & 1)) * kStageCols;
}
// copy columns [0, ncols) of raw row r to dst (ncols <= kStageCols, a multiple of 4; raw rows are 16-byte aligned and
// written by the GEMM up to Npad) as one commit group
__device__ __forceinline__ void stage_row(const PlanParams& P, const Ctx& c, int r, int ncols, float* dst) {
  const float* src = raw_ptr(P, c.slot) + static_cast<size_t>(r) * P.NpadMax;
  for (int q = 4 * c.lane; q < ncols; q += 4 * 32) ptx::cp_async_16(dst + q, src + q);
  ptx::cp_async_commit();
}
// Iteration i of a warp's row loop (row r; row r was staged into buffer i by the previous iteration or before the loop):
// stage row r + kWarps into buffer i + 1, wait for row r and make it visible to the whole warp.  The loop body must end
// with __syncwarp() so that no lane still reads buffer i when iteration i + 1 refills it.
__device__ __forceinline__ const float* stage_advance(const PlanParams& P, const Ctx& c, int r, int i, int ncols) {
  if (r + kWarps < kTileM) stage_row(P, c, r + kWarps, ncols, row_stage(c, i + 1));
  else ptx::cp_async_commit();   // an empty group: "all but the newest group" is then always row r
  ptx::cp_async_wait<1>();
  __syncwarp();
  return row_stage(c, i);
}

// Mish(x) = x * tanh(softplus(x)) (layers.py:103; softplus threshold 20) of a lane's batch of columns.
// tanh(log(1+e^x)) = n / (n + 2) with n = e^x (e^x + 2): one exp, one divide, no cancellation.  Three passes over the
// batch, so that its independent exp / divide chains overlap: a divide is a branch (its slow-path call), and a
// column-at-a-time loop runs the chains one after another.  x > 20 returns x; what the other passes computed for it
// (possibly inf / NaN) is discarded.
__device__ __forceinline__ void mish_batch(float (&y)[kLnBatch]) {
  float q[kLnBatch];
#pragma unroll
  for (int u = 0; u < kLnBatch; ++u) {
    const float e = expf(y[u]);
    q[u] = e * (e + 2.f);
  }
#pragma unroll
  for (int u = 0; u < kLnBatch; ++u) q[u] = __fdiv_rn(q[u], q[u] + 2.f);
#pragma unroll
  for (int u = 0; u < kLnBatch; ++u) y[u] = y[u] > 20.f ? y[u] : y[u] * q[u];
}

// LayerNorm (+ Mish | SimNorm) over raw rows; one warp per row, lane-strided columns (lane + 32 j).  raw is written by
// this kernel's GEMM and read with ld.global.cg; bias / gamma / beta are read-only for the kernel's lifetime and go
// through the read-only path (__ldg).  The output pass works on batches of kLnBatch columns per lane: every load of a
// batch is issued before its first store (the stores go through pointers that may alias raw as far as the compiler
// knows), and the batch's activations are independent chains that overlap.
//   - 512-wide rows (every hidden layer of the 5M model): raw is read once, through the staging buffers, so that the next
//     row's copy overlaps this row's work; the 16 values per lane stay in registers from the statistics through the
//     output pass.  (Holding the next row in registers instead spills it: the row phase shares the kernel's 168.)
//   - other widths: raw is read once per statistic and once in the output pass.  (Statistics loads in guarded batches
//     of kLnBatch were measured slower on c3's 1792-wide rows than these loops, which ptxas unrolls with unguarded loads.)
// Every column's value is the same expression in the same order in both paths: same bits.
// ROWS (ROP_PI_LOSS): the pre-LayerNorm value is multiplied by the dropout scale ea.drop (Q layer 0, train mode) and
// stored to the tape ea.tape; compiled out of the planning instantiations.
template <bool ROWS>
__device__ __forceinline__ void rows_ln_act(const PlanParams& P, Ctx& c, const LayerRec& ly, const EpiArgs& ea) {
  const float* rawbase = raw_ptr(P, c.slot);
  const int N = ly.N;
  const float invN = 1.f / static_cast<float>(N);
  __half* dhi = ea.dstbuf >= 0 ? plane_ptr(P, c.slot, ea.dstbuf, 0) : nullptr;
  __half* dlo = ea.dstbuf >= 0 ? plane_ptr(P, c.slot, ea.dstbuf, 1) : nullptr;
  const int pitch = ea.dstbuf >= 0 ? plane_pitch(P, ea.dstbuf) : 0;
  const float inv_scale = ly.inv_scale;
  const float* bias = ly.bias; const float* lg = ly.ln_g; const float* lb = ly.ln_b;
  const int ncolj = (N + 31) / 32;
  // activation and stores of row r's batch y = columns lane + 32 (j0 + u); warp-uniform (SimNorm shuffles across lanes)
  auto act_store = [&](float (&y)[kLnBatch], int j0, int r) {
    if (ea.kind == EPI_LN_MISH) {
      mish_batch(y);
    } else {
#pragma unroll
      for (int u = 0; u < kLnBatch; ++u)
        if (j0 + u < ncolj) y[u] = simnorm_lane(y[u], c.lane + 32 * (j0 + u) < N);
    }
    if (dhi) {
      __half* hi = dhi + static_cast<size_t>(r) * pitch + ea.dst_col0;
      __half* lo = dlo + static_cast<size_t>(r) * pitch + ea.dst_col0;
#pragma unroll
      for (int u = 0; u < kLnBatch; ++u) {
        const int col = c.lane + 32 * (j0 + u);
        if (col < N) split_store(hi + col, lo + col, y[u]);
      }
    }
    const int orow = ea.rowmap ? ea.rowmap[r] : r;
    if (ea.out_f32 && orow >= 0) {
      float* o = ea.out_f32 + static_cast<size_t>(orow) * ea.out_pitch;
#pragma unroll
      for (int u = 0; u < kLnBatch; ++u) {
        const int col = c.lane + 32 * (j0 + u);
        if (col < N) o[col] = y[u];
      }
    }
  };
  if (N == 32 * kLnRegCols) {
    // Rows arrive through the warp's staging buffers (see stage_row): row r + kWarps is copied while row r is computed.
    stage_row(P, c, c.warp, N, row_stage(c, 0));
    for (int r = c.warp, i = 0; r < kTileM; r += kWarps, ++i) {
      const float* row = stage_advance(P, c, r, i, N);
      float x[kLnRegCols];
#pragma unroll
      for (int j = 0; j < kLnRegCols; ++j) x[j] = row[c.lane + 32 * j];
      const bool live = ROWS && ea.rowmap[r] >= 0;
      const float* drow = live && ea.drop ? ea.drop + static_cast<size_t>(ea.rowmap[r]) * N : nullptr;
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < kLnRegCols; ++j) {
        x[j] = fmaf(x[j], inv_scale, __ldg(bias + c.lane + 32 * j));
        if (ROWS && drow) x[j] *= drow[c.lane + 32 * j];
        s += x[j];
      }
      if (ROWS && live && ea.tape) {
        float* trow = ea.tape + static_cast<size_t>(ea.rowmap[r]) * P.tape_pitch;
#pragma unroll
        for (int j = 0; j < kLnRegCols; ++j) trow[c.lane + 32 * j] = x[j];
      }
      const float mean = warp_sum(s) * invN;
      float sq = 0.f;
#pragma unroll
      for (int j = 0; j < kLnRegCols; ++j) {
        const float d = x[j] - mean;
        sq = fmaf(d, d, sq);
      }
      const float var = warp_sum(sq) * invN;
      const float rstd = 1.f / sqrtf(var + 1e-5f);   // nn.LayerNorm eps (layers.py:101)
#pragma unroll
      for (int j0 = 0; j0 < kLnRegCols; j0 += kLnBatch) {
        float y[kLnBatch];
#pragma unroll
        for (int u = 0; u < kLnBatch; ++u) {
          const int col = c.lane + 32 * (j0 + u);
          y[u] = (x[j0 + u] - mean) * rstd * __ldg(lg + col) + __ldg(lb + col);
        }
        act_store(y, j0, r);
      }
      __syncwarp();   // every lane has read buffer i before the next iteration refills it
    }
  } else if (ROWS && (ea.drop || ea.tape)) {
    // other widths with a dropout scale or a tape (ROP_PI_LOSS; kept apart so that the planning path's code is untouched):
    // the statistics pass tapes the pre-LayerNorm row, the later passes recompute it.  Padding rows have neither.
    for (int r = c.warp; r < kTileM; r += kWarps) {
      const float* rr = rawbase + static_cast<size_t>(r) * P.NpadMax;
      const int orow = ea.rowmap[r];
      const float* drow = ea.drop && orow >= 0 ? ea.drop + static_cast<size_t>(orow) * N : nullptr;
      float* trow = ea.tape && orow >= 0 ? ea.tape + static_cast<size_t>(orow) * P.tape_pitch : nullptr;
      float s = 0.f;
      for (int col = c.lane; col < N; col += 32) {
        float v = fmaf(__ldcg(rr + col), inv_scale, __ldg(bias + col));
        if (drow) v *= drow[col];
        if (trow) trow[col] = v;
        s += v;
      }
      const float mean = warp_sum(s) * invN;
      auto pre = [&](int col) {
        const float v = fmaf(__ldcg(rr + col), inv_scale, __ldg(bias + col));
        return drow ? v * drow[col] : v;
      };
      float sq = 0.f;
      for (int col = c.lane; col < N; col += 32) {
        const float d = pre(col) - mean;
        sq = fmaf(d, d, sq);
      }
      const float var = warp_sum(sq) * invN;
      const float rstd = 1.f / sqrtf(var + 1e-5f);
      for (int j0 = 0; j0 < ncolj; j0 += kLnBatch) {
        float y[kLnBatch];
#pragma unroll
        for (int u = 0; u < kLnBatch; ++u) {
          const int col = c.lane + 32 * (j0 + u);
          y[u] = col < N ? (pre(col) - mean) * rstd * __ldg(lg + col) + __ldg(lb + col) : 0.f;
        }
        act_store(y, j0, r);
      }
    }
  } else {
    for (int r = c.warp; r < kTileM; r += kWarps) {
      const float* rr = rawbase + static_cast<size_t>(r) * P.NpadMax;
      float s = 0.f;
      for (int col = c.lane; col < N; col += 32) s += fmaf(__ldcg(rr + col), inv_scale, __ldg(bias + col));
      const float mean = warp_sum(s) * invN;
      float sq = 0.f;
      for (int col = c.lane; col < N; col += 32) {
        const float d = fmaf(__ldcg(rr + col), inv_scale, __ldg(bias + col)) - mean;
        sq = fmaf(d, d, sq);
      }
      const float var = warp_sum(sq) * invN;
      const float rstd = 1.f / sqrtf(var + 1e-5f);
      for (int j0 = 0; j0 < ncolj; j0 += kLnBatch) {
        float y[kLnBatch];
#pragma unroll
        for (int u = 0; u < kLnBatch; ++u) {
          const int col = c.lane + 32 * (j0 + u);
          y[u] = col < N ? (fmaf(__ldcg(rr + col), inv_scale, __ldg(bias + col)) - mean) * rstd * __ldg(lg + col) + __ldg(lb + col)
                         : 0.f;
        }
        act_store(y, j0, r);
      }
    }
  }
}

// A head row is at most kMaxHeadCols wide: kHeadRegCols columns per lane (lane + 32 j) fit in registers.
constexpr int kHeadRegCols = kMaxHeadCols / 32;
static_assert(kMaxHeadCols <= kStageCols, "a head row fits a staging buffer");

// two_hot_inv (math.py:74-83): softmax over the bins, expectation under linspace(vmin,vmax,B), symexp.  y = the lane's
// logits (columns lane + 32 j < B); per bin and per lane the same expressions in the same order as a strided loop.
__device__ __forceinline__ float two_hot_inv_row(const PlanParams& P, Ctx& c, const float (&y)[kHeadRegCols]) {
  float bin[kHeadRegCols];
#pragma unroll
  for (int j = 0; j < kHeadRegCols; ++j) bin[j] = c.lane + 32 * j < P.B ? __ldg(P.bins + c.lane + 32 * j) : 0.f;
  float m = -CUDART_INF_F;
#pragma unroll
  for (int j = 0; j < kHeadRegCols; ++j)
    if (c.lane + 32 * j < P.B) m = fmaxf(m, y[j]);
  m = warp_max(m);
  float e[kHeadRegCols];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kHeadRegCols; ++j) {
    e[j] = expf(y[j] - m);
    if (c.lane + 32 * j < P.B) s += e[j];
  }
  s = warp_sum(s);
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < kHeadRegCols; ++j)
    if (c.lane + 32 * j < P.B) acc = fmaf(__fdiv_rn(e[j], s), bin[j], acc);
  acc = warp_sum(acc);
  return symexp_f(acc);
}

// ------------------------------------------------------------------------------------ MODE_ROWS epilogues
// torch.min(0) of two values: NaN if either is NaN (fminf would return the other one)
__device__ __forceinline__ float nan_min(float a, float b) { return (isnan(a) || isnan(b)) ? CUDART_NAN_F : fminf(a, b); }

// Q pair (world_model.py:211-216) and TD target (tdmpc2.py:255-257) of tile row r; one thread per row.
__device__ __forceinline__ void rows_commit(const PlanParams& P, Ctx& c, const EpiArgs& ea, int r, float val) {
  if (ea.head == HEAD_Q1) { c.q1[r] = val; return; }
  const float q = P.rows_flag ? __fmul_rn(__fadd_rn(c.q1[r], val), 0.5f) : nan_min(c.q1[r], val);   // Q.sum(0) / 2 | Q.min(0)
  const int row = c.rowenv[r];
  if (row < 0) return;
  if (P.rop == ROP_TD) {
    // reward + discount * (1 - terminated) * Q, evaluated left to right like the reference's fp32 expression
    const int task = P.task ? P.task[row] : 0;
    const float disc = P.disc_pow[static_cast<size_t>(task) * (P.H + 1) + 1];
    P.rows_out[row] = __fadd_rn(P.rows_reward[row], __fmul_rn(__fmul_rn(disc, __fsub_rn(1.f, P.rows_term[row])), q));
  } else {
    P.rows_out[row] = q;
    if (P.rows_tape) {
      const PiTape tp = pi_tape(P.M, P.A, P.Apad, P.B);
      P.rows_tape[static_cast<size_t>(row) * P.tape_pitch + tp.qv] = q;
    }
  }
}

// WorldModel.pi (world_model.py:144-184, math.py:12-29) for tile row r: the action goes to the X action columns (the
// TD target's Q heads read it there) and, for ROP_PI, to the outputs with tanh(mean), log_std and the two row sums the
// host turns into entropy / scaled_entropy.
__device__ __forceinline__ void rows_pi(const PlanParams& P, Ctx& c, const float* myrow, int r, __half* xhi, __half* xlo) {
  const int row = c.rowenv[r];
  const int e = row < 0 ? 0 : row;
  const int task = P.task ? P.task[e] : 0;
  float lp = 0.f, sq = 0.f;
  for (int a = c.lane; a < P.A; a += 32) {
    float mu = myrow[a];
    float ls = __fadd_rn(P.log_std_min, __fmul_rn(__fmul_rn(0.5f, P.log_std_dif), __fadd_rn(tanhf(myrow[P.Apad + a]), 1.f)));
    float eps = P.rows_eps[static_cast<size_t>(e) * P.A + a];
    if (P.masks) { const float mk = P.masks[static_cast<size_t>(task) * P.A + a]; mu *= mk; ls *= mk; eps *= mk; }
    lp += __fsub_rn(__fsub_rn(__fmul_rn(-0.5f, __fmul_rn(eps, eps)), ls), 0.9189385175704956f);   // gaussian_logprob
    const float act = tanhf(__fadd_rn(mu, __fmul_rn(eps, expf(ls))));
    sq += logf(__fadd_rn(fmaxf(__fsub_rn(1.f, __fmul_rn(act, act)), 0.f), 1e-6f));                // squash
    const size_t o = static_cast<size_t>(r) * P.KpadX + P.L + P.T + a;
    split_store(xhi + o, xlo + o, act);
    if (P.rows_out2 && row >= 0) {
      const size_t ro = static_cast<size_t>(row) * P.A + a;
      P.rows_out[ro] = act;
      P.rows_out2[ro] = tanhf(mu);
      P.rows_out3[ro] = ls;
    }
    if (P.rows_tape && row >= 0) {
      P.rows_act_out[static_cast<size_t>(row) * P.A + a] = act;
      P.rows_tape[static_cast<size_t>(row) * P.tape_pitch + pi_tape(P.M, P.A, P.Apad, P.B).act + a] = act;
    }
  }
  lp = warp_sum(lp);
  sq = warp_sum(sq);
  if (P.rows_out4 && row >= 0 && c.lane == 0) { P.rows_out4[2 * static_cast<size_t>(row)] = lp; P.rows_out4[2 * static_cast<size_t>(row) + 1] = sq; }
}

// Planning pi head (PRIOR / ITER / VALUE) for tile row r: the sampled action goes to the X action columns and, for the
// policy prior, to pi_actions.
__device__ __forceinline__ void pi_row(const PlanParams& P, Ctx& c, const EpiArgs& ea, const float* myrow, int r, __half* xhi, __half* xlo) {
  const RowMap rm = map_row(P, ea.tile, r);
  const int e = rm.env < 0 ? 0 : rm.env, idx = rm.env < 0 ? 0 : rm.idx;
  const int task = P.task ? P.task[e] : 0;
  for (int a = c.lane; a < P.A; a += 32) {
    const float eps = ea.eps_base ? __ldcs(&ea.eps_base[(static_cast<size_t>(e) * ea.eps_rows + idx) * P.A + a])
                                  : noise_pi_at(P, e, idx, a);        // eps_base == nullptr: in-kernel noise (ITER)
    const float act = pi_action(P, myrow[a], myrow[P.Apad + a], eps, task, a);
    const size_t o = static_cast<size_t>(r) * P.KpadX + P.L + P.T + a;
    split_store(xhi + o, xlo + o, act);
    if (ea.act_out && rm.env >= 0)
      ea.act_out[((static_cast<size_t>(e) * P.H + ea.t_out) * P.P + idx) * P.A + a] = act;
  }
}

template <bool EPISODIC, bool ROWS>
__device__ __forceinline__ void rows_head(const PlanParams& P, Ctx& c, const LayerRec& ly, const EpiArgs& ea) {
  float* myrow = c.rowbuf + c.warp * kMaxHeadCols;
  __half* xhi = plane_ptr(P, c.slot, BUF_X, 0);
  __half* xlo = plane_ptr(P, c.slot, BUF_X, 1);
  const int N = ly.N;
  // Rows arrive through the warp's staging buffers like rows_ln_act's 512-wide rows.  Heads are at most kMaxHeadCols
  // wide; only a diagnostic MODE_LAYER EPI_RAW row can be wider than a buffer, and it reads raw directly.
  const bool staged = N <= kStageCols;
  const int n4 = (N + 3) & ~3;
  if (staged) stage_row(P, c, c.warp, n4, row_stage(c, 0));
  for (int r = c.warp, i = 0; r < kTileM; r += kWarps, ++i) {
    const float* row = staged ? stage_advance(P, c, r, i, n4) : raw_ptr(P, c.slot) + static_cast<size_t>(r) * P.NpadMax;
    if (ea.kind == EPI_RAW) {
      const int orow = ea.rowmap ? ea.rowmap[r] : r;
      if (orow >= 0)
        for (int col = c.lane; col < N; col += 32) {
          float v = fmaf(row[col], ly.inv_scale, __ldg(ly.bias + col));
          if (ROWS && ea.head) v = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v)));      // termination: sigmoid
          ea.out_f32[static_cast<size_t>(orow) * ea.out_pitch + col] = v;
        }
    } else {
      // out[col] = raw * inv_scale + bias (plain Linear, no LN), the lane's columns lane + 32 j in registers
      float y[kHeadRegCols];
#pragma unroll
      for (int j = 0; j < kHeadRegCols; ++j) {
        const int col = c.lane + 32 * j;
        y[j] = col < N ? fmaf(row[col], ly.inv_scale, __ldg(ly.bias + col)) : 0.f;
      }
      if (ROWS && ea.tape && c.rowenv[r] >= 0) {      // ROP_PI_LOSS: the head's logits go to the tape
        float* t = ea.tape + static_cast<size_t>(c.rowenv[r]) * P.tape_pitch;
#pragma unroll
        for (int j = 0; j < kHeadRegCols; ++j)
          if (c.lane + 32 * j < N) t[c.lane + 32 * j] = y[j];
      }
      if (EPISODIC && ea.kind == EPI_TERM) {
        if (c.lane == 0) term_commit(c, r, y[0]);
      } else if (ea.kind == EPI_TWOHOT) {
        const float v = two_hot_inv_row(P, c, y);
        if (c.lane == 0) {
          if (ROWS) rows_commit(P, c, ea, r, v);
          else head_commit<EPISODIC>(P, c, ea, r, v);
        }
      } else if (ea.kind == EPI_PI) {
        // the pi head reads its mean and log_std columns (a, Apad + a) through the warp's smem row buffer
#pragma unroll
        for (int j = 0; j < kHeadRegCols; ++j)
          if (c.lane + 32 * j < N) myrow[c.lane + 32 * j] = y[j];
        __syncwarp();
        if (ROWS) rows_pi(P, c, myrow, r, xhi, xlo);
        else pi_row(P, c, ea, myrow, r, xhi, xlo);
      }
    }
    __syncwarp();
  }
}

// Make generic-proxy global writes (activation planes) visible to the TMA unit
// (async proxy) before the next layer's loads, and sync the CTA.
__device__ __forceinline__ void publish_planes() {
  __threadfence();
  ptx::fence_proxy_async_all();
  __syncthreads();
}

// ------------------------------------------------------------------------------------ one layer
// GEMM + epilogue; on return the epilogue's outputs are published (CTA-synchronised, TMA-visible).
template <int ENGINE, bool EPISODIC, bool ROWS>
__device__ __forceinline__ void run_layer(const PlanParams& P, Ctx& c, const LayerDev& ly_global, int srcbuf, const EpiArgs& ea,
                                          int kc0 = 0, const float* bias_override = nullptr) {
  LayerRec ly = layer_rec(ly_global);                // registers: see LayerRec
  if (bias_override) ly.bias = bias_override;        // shared-latent fold: see PlanParams::zbias
  const bool is_ln = (ea.kind == EPI_LN_MISH || ea.kind == EPI_LN_SIMNORM);
  const long long tl = prof_clock();
  if (threadIdx.x == 0) TDMPC2_TRACE(P, c, 0);
  if (ENGINE == ENGINE_TC) gemm_tc(P, c, ly, srcbuf, kc0);
  else gemm_simt(P, c, ly, srcbuf, kc0);
  if (threadIdx.x == 0) TDMPC2_TRACE(P, c, 3);
  if (is_ln) rows_ln_act<ROWS>(P, c, ly, ea);
  else rows_head<EPISODIC, ROWS>(P, c, ly, ea);
  c.pf1 += prof_clock() - tl;
  const long long tp = prof_clock();
  publish_planes();
  c.pf3 += prof_clock() - tp;
}

// ------------------------------------------------------------------------------------ top-k + MPPI refit
// Runs in the LAST CTA to finish a tile of environment e (tdmpc2.py:184-197).
// The thread group that runs the CTA-wide glue phases: the whole CTA (bar 0).
struct GroupAll { static constexpr int N = kThreads; __device__ static int tid() { return threadIdx.x; } __device__ static void sync() { __syncthreads(); } };

template <class G>
__device__ __forceinline__ void refit_env(const PlanParams& P, uint8_t* scratch, size_t scratch_bytes, int e, int task) {
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(scratch);
  int nsort = 1;
  while (nsort < P.N) nsort <<= 1;
  const float* vals = P.values + static_cast<size_t>(e) * P.N;
  for (int i = G::tid(); i < nsort; i += G::N) {
    unsigned long long k = 0ull;   // sentinel: sorts last
    if (i < P.N) {
      const float v = __ldcg(vals + i);
      unsigned u = __float_as_uint(v);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      k = (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<unsigned>(i));
      if (P.values_out) P.values_out[static_cast<size_t>(e) * P.N + i] = v;
    }
    keys[i] = k;
  }
  G::sync();
  // bitonic sort, descending (value desc, index asc on ties)
  for (int k2 = 2; k2 <= nsort; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = G::tid(); i < nsort; i += G::N) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          const bool desc = ((i & k2) == 0);
          if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
        }
      }
      G::sync();
    }
  }
  float* escore = reinterpret_cast<float*>(keys + nsort);     // [K]
  int* eidx = reinterpret_cast<int*>(escore + P.K);           // [K]
  float* red = reinterpret_cast<float*>(eidx + P.K);          // [2]
  const float vmax = __ldcg(vals + (0xFFFFFFFFu - static_cast<unsigned>(keys[0] & 0xFFFFFFFFull)));
  for (int k = G::tid(); k < P.K; k += G::N) {
    const int idx = static_cast<int>(0xFFFFFFFFu - static_cast<unsigned>(keys[k] & 0xFFFFFFFFull));
    eidx[k] = idx;
    escore[k] = expf(__fmul_rn(P.temperature, __ldcg(vals + idx) - vmax));   // exp(T * (v - max))
    P.elite_idx32[static_cast<size_t>(e) * P.K + k] = idx;
    if (P.elite_idx_out) P.elite_idx_out[static_cast<size_t>(e) * P.K + k] = idx;
  }
  G::sync();
  if (G::tid() == 0) {
    float s = 0.f;
    for (int k = 0; k < P.K; ++k) s += escore[k];
    red[0] = s;
  }
  G::sync();
  for (int k = G::tid(); k < P.K; k += G::N) escore[k] = __fdiv_rn(escore[k], red[0]);   // score /= score.sum(0)
  G::sync();
  if (G::tid() == 0) {
    float s = 0.f;
    for (int k = 0; k < P.K; ++k) s += escore[k];
    red[1] = s + 1e-9f;                                        // score.sum(0) + 1e-9
  }
  G::sync();
  const float denom = red[1];
  for (int k = G::tid(); k < P.K; k += G::N) P.score[static_cast<size_t>(e) * P.K + k] = escore[k];
  // Gather the elites' actions once, all loads independent (the weighted sums below then run out of smem).
  const int HA = P.H * P.A;
  float* eact = reinterpret_cast<float*>(scratch + 65536);          // [K][H*A]; keys/score/idx stay below 64 KiB
  const bool staged = static_cast<size_t>(P.K) * HA * 4 <= (scratch_bytes - 65536) &&
                      static_cast<size_t>(nsort) * 8 + static_cast<size_t>(P.K) * 8 + 16 <= 65536;
  if (staged) {
    for (int i = G::tid(); i < P.K * HA; i += G::N) {
      const int k = i / HA, ta = i % HA;
      eact[i] = sample_action(P, e, ta / P.A, eidx[k], ta % P.A, task);
    }
    G::sync();
  }
  for (int i = G::tid(); i < HA; i += G::N) {
    const int t = i / P.A, a = i % P.A;
    float m = 0.f;
    for (int k = 0; k < P.K; ++k) m = fmaf(escore[k], staged ? eact[k * HA + i] : sample_action(P, e, t, eidx[k], a, task), m);
    m = __fdiv_rn(m, denom);
    float var = 0.f;
    for (int k = 0; k < P.K; ++k) {
      const float act = staged ? eact[k * HA + i] : sample_action(P, e, t, eidx[k], a, task);
      const float d = act - m;
      var = fmaf(escore[k], d * d, var);
      if (t == 0) P.elite_act0[(static_cast<size_t>(e) * P.K + k) * P.A + a] = act;
    }
    float sd = sqrtf(__fdiv_rn(var, denom));
    sd = fminf(fmaxf(sd, P.min_std), P.max_std);
    if (P.masks) { const float mk = P.masks[static_cast<size_t>(task) * P.A + a]; m *= mk; sd *= mk; }
    // every read of the OLD mean/std of this environment happened above (eact gather, or this thread's own
    // (t, a) in the unstaged path): safe to overwrite now.
    const size_t sa = (static_cast<size_t>(e) * P.H + t) * P.A + a;
    P.mean[sa] = m;
    P.std[sa] = sd;
  }
  G::sync();
}

// ------------------------------------------------------------------------------------ the kernel
// EPISODIC (cfg.episodic, single-task models): every rollout step gains the 3-layer termination head on z_{t+1}
// and the value bookkeeping its sticky (1 - termination) factor (tdmpc2.py:126-136); compiled out otherwise.
// ROWS: MODE_ROWS only (world-model methods on a flat batch); compiled out of the planning instantiations.
template <int ENGINE, bool EPISODIC = false, bool ROWS = false>
__global__ void __launch_bounds__(kThreads, 1) plan_kernel(const __grid_constant__ PlanParams P) {
  constexpr int SPT = EPISODIC ? 9 : 6;      // layer steps per rollout time step (ITER / VALUE)
  extern __shared__ uint8_t smem_raw[];
  Ctx c;
  {
    // The operand tiles need 1024-byte alignment (128-byte swizzle atoms).  The kernel has no static shared memory, so
    // the dynamic window starts right after the 1 KiB the system reserves per CTA: it IS 1024-aligned, which is checked
    // here instead of being fixed up -- every smem pointer below is then the array symbol plus a compile-time constant.
    if ((ptx::smem_u32(smem_raw) & 1023u) != 0u) __trap();   // (no printf: see ptx::mbar_wait)
    c.stage_base = smem_raw;
    uint8_t* ctrl = c.stage_base + kStages * kStageBytes;
    c.g_full = reinterpret_cast<uint64_t*>(ctrl);
    c.g_empty = c.g_full + kGStages;
    c.flags = reinterpret_cast<int*>(c.g_empty + kGStages);     // [8]  (ends at ctrl + 80)
    c.G = reinterpret_cast<float*>(ctrl + 256);                 // [128]
    c.q1 = c.G + kTileM;                                        // [128]  (ends at ctrl + 1280)
    c.term = c.q1 + kTileM;                                     // [128]  (ends at ctrl + 1792 <= kSmemCtrl)
    c.rowbuf = reinterpret_cast<float*>(ctrl + kSmemCtrl);
    c.rowenv = reinterpret_cast<int*>(ctrl + kSmemCtrl + kSmemRowBuf);
  }
  c.slot = blockIdx.x;
  c.warp = threadIdx.x >> 5;
  c.lane = threadIdx.x & 31;
  c.pa_it = c.ma_it = 0;
  c.pf0 = c.pf1 = c.pf2 = c.pf3 = c.pf4 = c.pf5 = c.pf6 = c.pf7 = 0;
  c.trace_step = 1 << 30;
  const long long t_kernel0 = prof_clock();
  int* rowenv = c.rowenv;

  if (ENGINE == ENGINE_TC) {
    if (threadIdx.x == 0) {
      for (int s = 0; s < kGStages; ++s) { ptx::mbar_init(&c.g_full[s], 1); ptx::mbar_init(&c.g_empty[s], 4 * kGWarpGroups); }
      ptx::fence_barrier_init();
      ptx::prefetch_tensormap(&P.tmX);
      ptx::prefetch_tensormap(&P.tmH);
    }
    __syncthreads();
  }

  const LayerDev* LY = P.layers;

  for (int tile = static_cast<int>(blockIdx.x); tile < P.ntiles; tile += gridDim.x) {
    // ---------------- tile set-up: fill the input planes of X ----------------
    const long long t_setup = prof_clock();
    for (int r = threadIdx.x; r < kTileM; r += kThreads) {
      rowenv[r] = ROWS ? (tile * kTileM + r < P.rows ? tile * kTileM + r : -1) : map_row(P, tile, r).env;
      c.G[r] = 0.f; c.q1[r] = 0.f;
      if (EPISODIC) c.term[r] = 0.f;
    }
    __syncthreads();
    __half* xhi = plane_ptr(P, c.slot, BUF_X, 0);
    __half* xlo = plane_ptr(P, c.slot, BUF_X, 1);
    const int env_tile = (P.mode == MODE_ITER || P.mode == MODE_VALUE) ? tile / P.tiles_per_env : 0;
    const int task_tile = (P.task && (P.mode == MODE_ITER || P.mode == MODE_VALUE)) ? P.task[env_tile] : 0;

    if (ROWS) {
      // the call's input columns, zeros in every other column of X (stale action columns of an earlier launch
      // must not reach a GEMM) and in the padding rows:
      //   encode [obs | emb]; next / reward / Q [z | emb | a]; termination [z]; pi / TD target [z | emb]
      const int in_w = P.rop == ROP_ENCODE ? P.obs_dim : P.L;
      const int W = in_w + (P.rop == ROP_TERM ? 0 : P.T);
      const bool has_a = P.rop == ROP_NEXT || P.rop == ROP_REWARD || P.rop == ROP_Q_ALL || P.rop == ROP_Q_PAIR;
      for (int i = threadIdx.x; i < kTileM * P.KpadX; i += kThreads) {
        const int r = i / P.KpadX, col = i % P.KpadX;
        const int e = rowenv[r];
        float x = 0.f;
        if (e >= 0) {
          if (col < in_w) x = P.rows_in[static_cast<size_t>(e) * in_w + col];
          else if (col < W) x = P.emb[static_cast<size_t>(P.task ? P.task[e] : 0) * P.T + (col - in_w)];
          else if (has_a && col < W + P.A) x = P.rows_act[static_cast<size_t>(e) * P.A + (col - W)];
        }
        split_store(xhi + static_cast<size_t>(r) * P.KpadX + col, xlo + static_cast<size_t>(r) * P.KpadX + col, x);
      }
    } else if (P.mode == MODE_LAYER) {
      const LayerDev& ly = LY[P.dbg_layer];
      for (int i = threadIdx.x; i < kTileM * ly.Kpad; i += kThreads) {
        const int r = i / ly.Kpad, col = i % ly.Kpad;
        const float x = (r < P.dbg_rows && col < ly.K) ? P.dbg_x[static_cast<size_t>(r) * ly.K + col] : 0.f;
        split_store(xhi + static_cast<size_t>(r) * P.KpadX + col, xlo + static_cast<size_t>(r) * P.KpadX + col, x);
      }
      for (int r = threadIdx.x; r < kTileM; r += kThreads) rowenv[r] = r < P.dbg_rows ? r : -1;
    } else if (P.mode == MODE_ENCODE) {
      // [obs | task_emb]  (world_model.py:108-109)
      const int W = P.obs_dim + P.T;
      for (int i = threadIdx.x; i < kTileM * W; i += kThreads) {
        const int r = i / W, col = i % W;
        const RowMap rm = map_row(P, tile, r);
        const int e = rm.env < 0 ? 0 : rm.env;
        const float x = col < P.obs_dim ? P.obs[static_cast<size_t>(e) * P.obs_dim + col]
                                        : P.emb[static_cast<size_t>(P.task ? P.task[e] : 0) * P.T + (col - P.obs_dim)];
        split_store(xhi + static_cast<size_t>(r) * P.KpadX + col, xlo + static_cast<size_t>(r) * P.KpadX + col, x);
      }
    } else if (P.mode == MODE_ITER && !P.z_rows && ((P.L & 7) == 0) && ((P.T & 7) == 0) && (P.L + P.T) / 8 <= kThreads) {
      // [z | task_emb | .]: every row of an ITER tile carries the SAME latent (z.repeat(N), tdmpc2.py:163):
      // split 8 columns once, then broadcast them down the rows with 16-byte stores.
      const int nch = (P.L + P.T) / 8;
      const int ngrp = kThreads / nch;
      const int ch = threadIdx.x % nch, rg = threadIdx.x / nch;
      if (rg < ngrp) {
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float x[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int col = ch * 8 + 2 * j + u;
            x[u] = col < P.L ? P.z[static_cast<size_t>(env_tile) * P.L + col]
                             : P.emb[static_cast<size_t>(task_tile) * P.T + (col - P.L)];
            x[u] = (fabsf(x[u]) <= 3.0e38f) ? fminf(fmaxf(x[u], -65000.f), 65000.f) : CUDART_NAN_F;   // keep NaN/inf poisonous
          }
          const __half2 h2 = __floats2half2_rn(x[0], x[1]);
          const float2 hf = __half22float2(h2);
          const __half2 l2 = __floats2half2_rn(x[0] - hf.x, x[1] - hf.y);
          hw[j] = *reinterpret_cast<const uint32_t*>(&h2);
          lw[j] = *reinterpret_cast<const uint32_t*>(&l2);
        }
        for (int r = rg; r < kTileM; r += ngrp) {
          __stcg(reinterpret_cast<uint4*>(xhi + static_cast<size_t>(r) * P.KpadX + ch * 8), make_uint4(hw[0], hw[1], hw[2], hw[3]));
          __stcg(reinterpret_cast<uint4*>(xlo + static_cast<size_t>(r) * P.KpadX + ch * 8), make_uint4(lw[0], lw[1], lw[2], lw[3]));
        }
      }
    } else {
      // [z | task_emb | a]  (world_model.py:119-120); the action columns are written per step
      const int W = P.L + P.T;
      for (int i = threadIdx.x; i < kTileM * W; i += kThreads) {
        const int r = i / W, col = i % W;
        const RowMap rm = map_row(P, tile, r);
        const int e = rm.env < 0 ? 0 : rm.env;
        float x;
        if (col < P.L) {
          x = P.z_rows ? P.z_rows[(static_cast<size_t>(e) * P.N + (rm.env < 0 ? 0 : rm.idx)) * P.L + col]
                       : P.z[static_cast<size_t>(e) * P.L + col];
        } else {
          x = P.emb[static_cast<size_t>(P.task ? P.task[e] : 0) * P.T + (col - P.L)];
        }
        split_store(xhi + static_cast<size_t>(r) * P.KpadX + col, xlo + static_cast<size_t>(r) * P.KpadX + col, x);
      }
    }
    if (P.mode == MODE_ITER && !P.actions_explicit && !P.rng_state && threadIdx.x <= P.H) {
      // This tile's slabs of the (HBM-resident, read-once) noise tensors are contiguous: ask for them now, so that the
      // per-step action pass and the terminal policy sample find them in L2 instead of paying DRAM latency.
      const int n0 = (tile % P.tiles_per_env) * kTileM, n1 = min(n0 + kTileM, P.N);
      const int t = threadIdx.x;
      if (t < P.H) {
        const int r0 = max(n0, P.P) - P.P, r1 = n1 - P.P;
        if (r1 > r0)
          ptx::bulk_prefetch_l2(P.noise_r + ((static_cast<size_t>(env_tile) * P.H + t) * (P.N - P.P) + r0) * P.A,
                                static_cast<size_t>(r1 - r0) * P.A * sizeof(float));
      } else {
        ptx::bulk_prefetch_l2(P.noise_pi + (static_cast<size_t>(env_tile) * P.N + n0) * P.A, static_cast<size_t>(n1 - n0) * P.A * sizeof(float));
      }
    }
    publish_planes();
    c.pf4 += prof_clock() - t_setup;

    // ---------------- the tile's layer program: ONE run_layer call site ----------------
    //   ENCODE : enc.0 .. enc.(n-1)
    //   PRIOR  : per t: pi.0-2 [, dyn.0-2 if t < H-1]
    //   ITER   : per t: [a_t -> X] rew.0-2, dyn.0-2 [, term.0-2 if EPISODIC] ; then pi.0-2, q_a.0-2, q_b.0-2
    int nsteps;
    if (ROWS) nsteps = P.rop == ROP_ENCODE ? P.num_enc : P.rop == ROP_Q_ALL ? 3 * P.num_q : P.rop == ROP_Q_PAIR ? 6
                     : (P.rop == ROP_TD || P.rop == ROP_PI_LOSS) ? 9 : 3;
    else if (P.mode == MODE_LAYER) nsteps = 1;
    else if (P.mode == MODE_ENCODE) nsteps = P.num_enc;
    else if (P.mode == MODE_PRIOR) nsteps = 6 * (P.H - 1) + 3;
    else nsteps = SPT * P.H + 9;
    const float* dpow = P.disc_pow + static_cast<size_t>(task_tile) * (P.H + 1);
    const int* qi = (P.mode == MODE_ITER || P.mode == MODE_VALUE) ? P.qidx + static_cast<size_t>(env_tile) * 2 : nullptr;

    for (int sidx = 0; sidx < nsteps; ++sidx) {
      EpiArgs ea;
      ea.kind = EPI_LN_MISH; ea.dstbuf = -1; ea.dst_col0 = 0; ea.out_f32 = nullptr; ea.out_pitch = 0; ea.rowmap = nullptr;
      ea.head = 0; ea.disc = 0.f; ea.tile = tile; ea.eps_base = nullptr; ea.eps_rows = 0; ea.act_out = nullptr; ea.t_out = 0;
      ea.tape = nullptr; ea.drop = nullptr;
      int li, src;
      int kc0 = 0;                       // first K-chunk of the GEMM and bias vector: the shared-latent fold (PlanParams::zbias)
      const float* bias_ov = nullptr;
      const LayerDev* lyt = LY;          // layer table of this step (MODE_ROWS Q heads: P.rows_q)
      if (ROWS) {
        // ROWS program:  encode enc.0..n-1 | next dyn.0-2 | reward rew.0-2 | termination term.0-2 | pi pi.0-2
        //                | Q all: head h = 0..num_q-1, layers 0-2 | Q pair: heads qidx[0], qidx[1] | TD: pi.0-2, then Q pair
        const int l = P.rop == ROP_ENCODE ? sidx : sidx % 3;
        src = l == 0 ? BUF_X : BUF_H1;
        ea.rowmap = rowenv;
        const bool last = P.rop == ROP_ENCODE ? sidx == P.num_enc - 1 : l == 2;
        if (!last) { ea.kind = EPI_LN_MISH; ea.dstbuf = BUF_H1; }
        // agent._update's forward (rows_tape non-null): every LayerNorm layer tapes its pre-LayerNorm row at the layer's
        // column offset (encoder: hidden layers enc_dim wide, the SimNorm layer last; MLPs: layers 0 and 1 M wide)
        if (P.rop == ROP_ENCODE) {
          li = P.li_enc + sidx;
          if (last) { ea.kind = EPI_LN_SIMNORM; ea.out_f32 = P.rows_out; ea.out_pitch = P.L; }
          if (P.rows_tape) ea.tape = P.rows_tape + sidx * LY[P.li_enc].N;
        } else if (P.rop == ROP_NEXT) {
          li = P.li_dyn + l;
          if (last) { ea.kind = EPI_LN_SIMNORM; ea.out_f32 = P.rows_out; ea.out_pitch = P.L; }
          if (P.rows_tape) ea.tape = P.rows_tape + l * P.M;
        } else if (P.rop == ROP_REWARD) {
          li = P.li_rew + l;
          if (last) { ea.kind = EPI_RAW; ea.out_f32 = P.rows_out; ea.out_pitch = P.B; }
          else if (P.rows_tape) ea.tape = P.rows_tape + l * P.M;
        } else if (P.rop == ROP_TERM) {
          li = P.li_term + l;
          if (last) { ea.kind = EPI_RAW; ea.out_f32 = P.rows_out; ea.out_pitch = 1; ea.head = P.rows_flag; }
          else if (P.rows_tape) ea.tape = P.rows_tape + l * P.M;
        } else if (P.rop == ROP_PI || ((P.rop == ROP_TD || P.rop == ROP_PI_LOSS) && sidx < 3)) {
          li = P.li_pi + l;
          if (last) ea.kind = EPI_PI;
          if (P.rop == ROP_PI_LOSS) {
            const PiTape tp = pi_tape(P.M, P.A, P.Apad, P.B);
            ea.tape = P.rows_tape + (l == 0 ? tp.pi0 : l == 1 ? tp.pi1 : tp.pih);
          }
        } else {
          const int u = (P.rop == ROP_TD || P.rop == ROP_PI_LOSS) ? sidx / 3 - 1 : sidx / 3;     // head slot
          const int h = P.rop == ROP_Q_ALL ? u : P.qidx[u];
          lyt = P.rows_q;
          li = 3 * h + l;
          if (P.rop == ROP_PI_LOSS) {
            ea.tape = P.rows_tape + pi_tape(P.M, P.A, P.Apad, P.B).q[u] + l * P.M;
            if (l == 0 && P.rows_drop) ea.drop = P.rows_drop + static_cast<size_t>(h) * P.rows * P.M;
          }
          if (P.rop == ROP_Q_ALL && P.rows_tape && !last) {
            ea.tape = P.rows_tape + (2 * h + l) * P.M;
            if (l == 0 && P.rows_drop) ea.drop = P.rows_drop + static_cast<size_t>(h) * P.rows * P.M;
          }
          if (last && P.rop == ROP_Q_ALL) {
            ea.kind = EPI_RAW; ea.out_f32 = P.rows_out + static_cast<size_t>(h) * P.rows * P.B; ea.out_pitch = P.B;
          } else if (last) {
            ea.kind = EPI_TWOHOT; ea.head = u == 0 ? HEAD_Q1 : HEAD_Q2;
          }
        }
      } else if (P.mode == MODE_LAYER) {
        li = P.dbg_layer; src = BUF_X;
        ea.kind = P.dbg_mode == 0 ? EPI_RAW : (P.dbg_mode == 1 ? EPI_LN_MISH : EPI_LN_SIMNORM);
        ea.out_f32 = P.dbg_y; ea.out_pitch = LY[li].N; ea.rowmap = rowenv;
      } else if (P.mode == MODE_ENCODE) {
        li = P.li_enc + sidx;
        src = sidx == 0 ? BUF_X : BUF_H1;
        if (sidx == P.num_enc - 1) { ea.kind = EPI_LN_SIMNORM; ea.out_f32 = P.z; ea.out_pitch = P.L; ea.rowmap = rowenv; }
        else { ea.kind = EPI_LN_MISH; ea.dstbuf = BUF_H1; }
      } else {
        // which MLP, which of its 3 layers
        int mlp, l, t = 0;       // mlp: 0 reward, 1 dynamics, 2 pi, 3 q_a, 4 q_b, 5 termination
        if (P.mode == MODE_PRIOR) {
          t = sidx / 6; l = sidx % 6;
          mlp = l < 3 ? 2 : 1; l %= 3;
        } else if (sidx < SPT * P.H) {
          t = sidx / SPT; l = sidx % SPT;
          mlp = l < 3 ? 0 : ((EPISODIC && l >= 6) ? 5 : 1); l %= 3;
          if (mlp == 0 && l == 0) {
            // X action columns <- a_t  (tdmpc2.py:176-181)
            const long long t_act = prof_clock();
            if (P.actions_explicit) {
              for (int i = threadIdx.x; i < kTileM * P.A; i += kThreads) {
                const int r = i / P.A, a = i % P.A;
                const RowMap rm = map_row(P, tile, r);
                const float v = sample_action(P, env_tile, t, rm.env < 0 ? 0 : rm.idx, a, task_tile);
                const size_t o = static_cast<size_t>(r) * P.KpadX + P.L + P.T + a;
                split_store(xhi + o, xlo + o, v);
              }
            } else {
              // mean/std/mask of step t staged in smem, then one pass of independent, coalesced noise loads
              float* sm_mean = c.rowbuf; float* sm_std = c.rowbuf + kMaxHeadCols; float* sm_mask = c.rowbuf + 2 * kMaxHeadCols;
              for (int a = threadIdx.x; a < P.A; a += kThreads) {
                const size_t sa = (static_cast<size_t>(env_tile) * P.H + t) * P.A + a;
                sm_mean[a] = P.mean[sa]; sm_std[a] = P.std[sa];
                sm_mask[a] = P.masks ? P.masks[static_cast<size_t>(task_tile) * P.A + a] : 1.f;
              }
              __syncthreads();
              const int n0 = (tile % P.tiles_per_env) * kTileM;
              const float* nz = P.noise_r + (static_cast<size_t>(env_tile) * P.H + t) * (P.N - P.P) * P.A;
              const float* pa = P.pi_actions + (static_cast<size_t>(env_tile) * P.H + t) * P.P * P.A;
              const int ng = (P.A + 7) >> 3;
              if ((((P.L + P.T) & 7) == 0) && (P.L + P.T + 8 * ng <= P.KpadX)) {
                // one (row, 8 action columns) item per thread: every load of the pass is in flight at once, two 16-byte
                // stores per item (columns past A are zero-weight padding of X: zeros there are harmless)
                for (int i = threadIdx.x; i < kTileM * ng; i += kThreads) {
                  const int r = i / ng, g8 = (i % ng) * 8;
                  const int n = min(n0 + r, P.N - 1);
                  const float* src = (n < P.P) ? pa + static_cast<size_t>(n) * P.A : nz + static_cast<size_t>(n - P.P) * P.A;
                  float x[8];
                  if (n >= P.P && P.rng_state) {                               // in-kernel noise: two groups of four
                    const float4 g0 = rng_normal4(P.rng_state, 2u * P.rng_iter, rng_group_r(P, env_tile, t, n, g8 >> 2));
                    const float4 g1 = rng_normal4(P.rng_state, 2u * P.rng_iter, rng_group_r(P, env_tile, t, n, (g8 >> 2) + 1));
                    x[0] = g0.x; x[1] = g0.y; x[2] = g0.z; x[3] = g0.w; x[4] = g1.x; x[5] = g1.y; x[6] = g1.z; x[7] = g1.w;
                  } else {
#pragma unroll
                    for (int u = 0; u < 8; ++u)                                // noise is one-shot: evict-first
                      x[u] = (g8 + u < P.A) ? (n < P.P ? src[g8 + u] : __ldcs(src + g8 + u)) : 0.f;
                  }
                  uint32_t hw[4], lw[4];
#pragma unroll
                  for (int u = 0; u < 8; u += 2) {
                    __half h[2], l[2];
#pragma unroll
                    for (int w = 0; w < 2; ++w) {
                      const int a = min(g8 + u + w, P.A - 1);
                      float v = x[u + w];
                      if (n >= P.P) v = fminf(fmaxf(__fadd_rn(sm_mean[a], __fmul_rn(sm_std[a], v)), -1.f), 1.f);
                      v = (g8 + u + w < P.A) ? v * sm_mask[a] : 0.f;
                      split_f(v, h[w], l[w]);
                    }
                    hw[u >> 1] = static_cast<uint32_t>(__half_as_ushort(h[0])) | (static_cast<uint32_t>(__half_as_ushort(h[1])) << 16);
                    lw[u >> 1] = static_cast<uint32_t>(__half_as_ushort(l[0])) | (static_cast<uint32_t>(__half_as_ushort(l[1])) << 16);
                  }
                  const size_t o = static_cast<size_t>(r) * P.KpadX + P.L + P.T + g8;
                  __stcg(reinterpret_cast<uint4*>(xhi + o), make_uint4(hw[0], hw[1], hw[2], hw[3]));
                  __stcg(reinterpret_cast<uint4*>(xlo + o), make_uint4(lw[0], lw[1], lw[2], lw[3]));
                }
              } else {
#pragma unroll 4
                for (int i = threadIdx.x; i < kTileM * P.A; i += kThreads) {
                  const int r = i / P.A, a = i % P.A;
                  const int n = min(n0 + r, P.N - 1);
                  float v;
                  if (n < P.P) v = pa[static_cast<size_t>(n) * P.A + a];
                  else {
                    v = __fadd_rn(sm_mean[a], __fmul_rn(sm_std[a], noise_r_at(P, env_tile, t, n, a)));   // one-shot: evict-first
                    v = fminf(fmaxf(v, -1.f), 1.f);
                  }
                  v *= sm_mask[a];
                  const size_t o = static_cast<size_t>(r) * P.KpadX + P.L + P.T + a;
                  split_store(xhi + o, xlo + o, v);
                }
              }
            }
            publish_planes();
            c.pf5 += prof_clock() - t_act;
          }
        } else {
          const int u = sidx - SPT * P.H;
          mlp = 2 + u / 3; l = u % 3;
        }
        src = l == 0 ? BUF_X : BUF_H1;
        const int base = (EPISODIC && mlp == 5) ? P.li_term
                         : mlp == 0 ? P.li_rew : mlp == 1 ? P.li_dyn : mlp == 2 ? P.li_pi : P.li_q + 3 * qi[mlp - 3];
        li = base + l;
        if (P.mode == MODE_ITER && P.zb_kc0 > 0 && sidx < SPT * P.H && t == 0 && l == 0 && mlp <= 1) {
          // t = 0: the rows of the tile share [z | emb]; its product with reward.0 / dynamics.0 was folded into a
          // per-environment bias by the prologue, the GEMM only covers the action columns
          kc0 = P.zb_kc0;
          bias_ov = P.zbias + (static_cast<size_t>(mlp) * P.E + env_tile) * P.zb_pitch;
        }
        if (l < 2) {
          ea.kind = EPI_LN_MISH; ea.dstbuf = BUF_H1;
        } else if (mlp == 0) {                 // reward (world_model.py:123-130) + two_hot_inv
          ea.kind = EPI_TWOHOT; ea.head = HEAD_REWARD; ea.disc = dpow[t];
        } else if (mlp == 1) {                 // z <- next(z, a)  (world_model.py:114-121)
          ea.kind = EPI_LN_SIMNORM; ea.dstbuf = BUF_X; ea.dst_col0 = 0;
        } else if (mlp == 2) {                 // a = pi(z)  (world_model.py:144-174) -> X action columns
          ea.kind = EPI_PI;
          if (P.mode == MODE_PRIOR) {          // eps = noise_prior[e, t, p, :]
            ea.eps_base = P.noise_prior + static_cast<size_t>(t) * P.P * P.A; ea.eps_rows = P.H * P.P;
            ea.act_out = P.pi_actions; ea.t_out = t;
          } else {                             // eps = noise_pi[e, n, :]
            ea.eps_base = P.rng_state ? nullptr : P.noise_pi; ea.eps_rows = P.N;
          }
        } else if (EPISODIC && mlp == 5) {     // termination(z_{t+1})  (world_model.py:132-141), input [z | emb]
          ea.kind = EPI_TERM;
        } else {                               // Q heads (world_model.py:186-216)
          ea.kind = EPI_TWOHOT; ea.head = (mlp == 3) ? HEAD_Q1 : HEAD_Q2; ea.disc = dpow[P.H];
        }
      }
      c.trace_step = (tile == static_cast<int>(blockIdx.x)) ? sidx : (1 << 30);
      run_layer<ENGINE, EPISODIC, ROWS>(P, c, lyt[li], src, ea, kc0, bias_ov);
    }

    const long long t_refit = prof_clock();
    if (P.mode == MODE_ITER) {
      // last CTA to finish a tile of this environment refits its mean/std
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned old = atomicAdd(&P.env_counter[env_tile], 1u);
        c.flags[0] = (old == static_cast<unsigned>(P.tiles_per_env - 1));
        if (c.flags[0]) P.env_counter[env_tile] = 0;
      }
      __syncthreads();
      if (c.flags[0]) {
        __threadfence();
        refit_env<GroupAll>(P, c.stage_base, static_cast<size_t>(kStages) * kStageBytes, env_tile, task_tile);
      }
      publish_planes();     // refit_env wrote the stage smem through the generic proxy; TMA reuses it next tile
    }
    c.pf6 += prof_clock() - t_refit;
  }

  if (kProf && P.prof) {
    // rows: 0 TMA producer (warp 8 lane 0), 1 consumer warpgroup 0 (thread 0), 2 consumer warpgroup 1 (thread 128),
    //       3 idle warp 9 during the GEMM
    // cols: 0 stage-empty wait cycles, 1 cycles inside layers, 2 stage-full wait, 3 publish, 4 tile set-up, 5 whole kernel,
    //       6 action pass, 7 refit
    const int who = (threadIdx.x == kGProducerWarp * 32) ? 0 : (threadIdx.x == 0) ? 1 : (threadIdx.x == 128) ? 2
                    : (threadIdx.x == (kGProducerWarp + 1) * 32) ? 3 : -1;
    if (who >= 0) {
      long long* o = P.prof + (static_cast<size_t>(blockIdx.x) * 4 + who) * 12;
      o[0] = c.pf0; o[1] = c.pf1; o[2] = c.pf2; o[3] = c.pf3; o[4] = c.pf4; o[5] = prof_clock() - t_kernel0;
      o[6] = c.pf5; o[7] = c.pf6; o[8] = c.pf7;
    }
  }
}

// ------------------------------------------------------------------------------------ small kernels
// mean/std initialisation (tdmpc2.py:164-167)
__global__ void init_state_kernel(float* mean, float* std, unsigned* env_counter, const float* prev_mean,
                                  const uint8_t* t0, int E, int H, int A, float max_std) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < E) env_counter[i] = 0;
  if (i >= E * H * A) return;
  const int a = i % A, t = (i / A) % H, e = i / (A * H);
  float m = 0.f;
  if (!t0[e] && t < H - 1) m = prev_mean[(static_cast<size_t>(e) * H + t + 1) * A + a];
  mean[i] = m;
  std[i] = max_std;
}

// Shared-latent fold (PlanParams::zbias): zbias[mlp][e][n] = bias[n] + 2^-k * sum_{k < Kz} x_e[k] * (W_hi + W_lo)[n][k], x_e = [z_e | emb_task(e)],
// for mlp 0 = reward.0, 1 = dynamics.0 (world_model.py:114-130: both take [z | emb | a]).  fp32 FFMA over the packed
// planes (whose sum is W * 2^k to ~22 bits, the operand the tensor-core path multiplies with).  Block = 4 environments
// x 64 output columns; a warp owns 8 columns, its lanes stride over k (coalesced half2 loads of the K-major rows).
constexpr int kZbEnvs = 4, kZbCols = 64, kZbKc = 1024;
__global__ void __launch_bounds__(256) zbias_kernel(const LayerDev* __restrict__ layers, int li_rew, int li_dyn, const float* __restrict__ z,
                                                    const float* __restrict__ emb, const int* __restrict__ task, int E, int L, int T,
                                                    int Kz, float* __restrict__ out, int pitch) {
  __shared__ float xs[kZbEnvs][kZbKc];
  const int mlp = blockIdx.z;
  const LayerDev& ly = layers[mlp == 0 ? li_rew : li_dyn];
  const int e0 = blockIdx.y * kZbEnvs, n0 = blockIdx.x * kZbCols;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[8][kZbEnvs];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int i = 0; i < kZbEnvs; ++i) acc[j][i] = 0.f;
  for (int kb = 0; kb < Kz; kb += kZbKc) {
    const int kn = min(kZbKc, Kz - kb);
    __syncthreads();
    for (int i = threadIdx.x; i < kZbEnvs * kn; i += blockDim.x) {
      const int ei = i / kn, k = kb + i % kn, e = min(e0 + ei, E - 1);
      xs[ei][i % kn] = k < L ? z[static_cast<size_t>(e) * L + k] : emb[static_cast<size_t>(task ? task[e] : 0) * T + (k - L)];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + warp * 8 + j;
      if (n >= ly.Npad) continue;
      const __half2* wh = reinterpret_cast<const __half2*>(ly.w_hi + static_cast<size_t>(n) * ly.Kpad + kb);
      const __half2* wl = reinterpret_cast<const __half2*>(ly.w_lo + static_cast<size_t>(n) * ly.Kpad + kb);
      for (int k2 = lane; k2 < kn / 2; k2 += 32) {          // Kz and kZbKc are multiples of 64
        const float2 h = __half22float2(wh[k2]), l = __half22float2(wl[k2]);
        const float w0 = h.x + l.x, w1 = h.y + l.y;
#pragma unroll
        for (int i = 0; i < kZbEnvs; ++i) acc[j][i] = fmaf(xs[i][2 * k2 + 1], w1, fmaf(xs[i][2 * k2], w0, acc[j][i]));
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int n = n0 + warp * 8 + j;
#pragma unroll
    for (int i = 0; i < kZbEnvs; ++i) {
      const float v = warp_sum(acc[j][i]);
      if (lane == 0 && n < ly.Npad && e0 + i < E)
        out[(static_cast<size_t>(mlp) * E + e0 + i) * pitch + n] = fmaf(v, ly.inv_scale, ly.bias[n]);
    }
  }
}

// final action (tdmpc2.py:199-206, math.py:86-94); one warp per environment
__global__ void pick_kernel(const float* score, const float* elite_act0, const float* mean, const float* std,
                            const float* expo, const float* noise_final, float* action, float* prev_mean_out,
                            int* pick_out, int E, int K, int H, int A) {
  const int e = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (e >= E) return;
  // argmax_k softmax(log(score_k) - log(expo_k)) == argmax of the logits (first max on ties)
  // NaN logits (score == 0 together with expo == 0, or a NaN temperature) never win a comparison: the pick then stays
  // at elite 0 (in range), where torch.argmax would return the first NaN position -- degenerate input either way.
  float best = -CUDART_INF_F;
  int bi = 0x7fffffff;
  for (int k = lane; k < K; k += 32) {
    const float g = __fadd_rn(logf(score[static_cast<size_t>(e) * K + k]), -logf(expo[static_cast<size_t>(e) * K + k]));
    if (g > best || (g == best && k < bi)) { best = g; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (bi < 0 || bi >= K) bi = 0;
  if (lane == 0 && pick_out) pick_out[e] = bi;
  for (int a = lane; a < A; a += 32) {
    float v = elite_act0[(static_cast<size_t>(e) * K + bi) * A + a];
    if (noise_final) v = __fadd_rn(v, __fmul_rn(std[(static_cast<size_t>(e) * H) * A + a], noise_final[static_cast<size_t>(e) * A + a]));
    action[static_cast<size_t>(e) * A + a] = fminf(fmaxf(v, -1.f), 1.f);
  }
  for (int i = lane; i < H * A; i += 32) prev_mean_out[static_cast<size_t>(e) * H * A + i] = mean[static_cast<size_t>(e) * H * A + i];
}

}  // namespace tdmpc2
