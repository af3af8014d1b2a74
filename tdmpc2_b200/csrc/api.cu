// Host side of the C ABI declared in include/tdmpc2_b200.h: planner object,
// memory layout of the packed weights and the workspace, TMA descriptor set-up,
// weight packing kernels and the launch sequence of the fused planning kernels.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tdmpc2_b200.h"
#include "plan_kernels.cuh"
#include "grad_kernels.cuh"
#include "pixel_encoder.cuh"
#include "pixel_grad_kernels.cuh"

using namespace tdmpc2;

// ------------------------------------------------------------------------------------ errors
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return fail(TDMPC2_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

static unsigned env_uint(const char* name, unsigned dflt) {
  const char* v = getenv(name);
  return (v && *v) ? static_cast<unsigned>(strtoul(v, nullptr, 10)) : dflt;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
// a workspace / tape segment of n floats at `off`, the next one starting on a 64-float boundary
static size_t take64(size_t& off, size_t n) { const size_t o = off; off += (n + 63) / 64 * 64; return o; }
static inline int pad_to(int x, int a) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------ pack kernels
__global__ void absmax_kernel(const float* __restrict__ w, size_t n, unsigned* slot) {
  float m = 0.f;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(slot, __float_as_uint(m));   // non-negative floats order like uints
}

// W[N, K] fp32 row-major -> two fp16 planes [Npad, Kpad] of W * 2^k, zero padded.
// 2^k puts max|W| in [128, 256): fp16 hi keeps 11 bits, lo the next 11, both in the normal range.
// Output row n takes source row n (n < split_at) or split_at + (n - split_to) (n >= split_to): the pi head's
// log_std rows are moved to a 32-aligned column (column Apad of the head's output row).
__device__ __forceinline__ int src_index(int n, int src_n, int split_at, int split_to) {
  if (n < split_at) return n;
  if (n >= split_to && n - split_to + split_at < src_n) return n - split_to + split_at;
  return -1;
}
__global__ void split_weight_kernel(const float* __restrict__ w, int N, int K, int Npad, int Kpad, __half* hi,
                                    __half* lo, const unsigned* absmax_slot, LayerDev* entry, int src_n, int split_at,
                                    int split_to) {
  const float amax = __uint_as_float(*absmax_slot);
  int ex = 0;
  float scale = 1.f;
  if (amax > 0.f && isfinite(amax)) {
    frexpf(amax, &ex);                 // amax = m * 2^ex, m in [0.5, 1)
    scale = ldexpf(1.f, 8 - ex);       // amax * scale in [128, 256)
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) entry->inv_scale = 1.f / scale;
  const size_t total = static_cast<size_t>(Npad) * Kpad;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(i / Kpad), k = static_cast<int>(i % Kpad);
    float x = 0.f;
    const int sn = src_index(n, src_n, split_at, split_to);
    if (n < N && k < K && sn >= 0) x = w[static_cast<size_t>(sn) * K + k] * scale;
    const __half h = __float2half_rn(x);
    hi[i] = h;
    lo[i] = __float2half_rn(x - __half2float(h));
  }
}

__global__ void pad_vector_kernel(const float* __restrict__ src, int n, int npad, float* dst, float fill, int src_n,
                                  int split_at, int split_to) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npad) return;
  const int si = src_index(i, src_n, split_at, split_to);
  dst[i] = (i < n && src && si >= 0) ? src[si] : fill;
}

// nn.Embedding(max_norm=1) (world_model.py:21): rows with ||w|| > 1 are scaled by 1/(||w|| + 1e-7) at lookup.
__global__ void emb_renorm_kernel(const float* __restrict__ emb, int T, float* out) {
  const int row = blockIdx.x;
  float s = 0.f;
  for (int i = threadIdx.x; i < T; i += 32) { const float v = emb[static_cast<size_t>(row) * T + i]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  const float nrm = sqrtf(s);
  const float sc = nrm > 1.f ? 1.f / (nrm + 1e-7f) : 1.f;
  for (int i = threadIdx.x; i < T; i += 32) out[static_cast<size_t>(row) * T + i] = emb[static_cast<size_t>(row) * T + i] * sc;
}

// ------------------------------------------------------------------------------------ planner
struct LayerHost {
  int K, Kpad, N, Npad, wmap, wrow, has_ln;
  int src_n, split_at, split_to;                   // source rows and the optional row remap (pi head)
  size_t off_hi, off_lo, off_bias, off_g, off_b;   // byte offsets into the packed blob
};

// Byte layout of a packed weight blob: layer table | absmax slots | per-layer vectors | `extra` bytes of the caller |
// one 1024-aligned weight map per Kpad class, map m read through the TMA map tmW[base_map + m].
struct BlobLayout {
  int base_map = 0, nmaps = 0;
  int map_kpad[kMaxWMaps], map_rows[kMaxWMaps];
  size_t map_off[kMaxWMaps];
  size_t off_table = 0, off_absmax = 0, off_extra = 0, bytes = 0;
};

// Assigns the weight maps of `layers` (a new class per new Kpad, numbered from base_map), their rows in those maps and
// every byte offset.  false: the classes do not fit the kMaxWMaps TMA maps (`b` is then empty).
static bool layout_blob(std::vector<LayerHost>& layers, int base_map, size_t extra, BlobLayout& b) {
  b = BlobLayout{};
  b.base_map = base_map;
  for (auto& l : layers) {
    int m = 0;
    while (m < b.nmaps && b.map_kpad[m] != l.Kpad) ++m;
    if (m == b.nmaps) {
      if (base_map + b.nmaps == kMaxWMaps) { b = BlobLayout{}; return false; }
      b.map_kpad[m] = l.Kpad;
      b.map_rows[m] = 0;
      ++b.nmaps;
    }
    l.wmap = base_map + m;
    l.wrow = b.map_rows[m];
    b.map_rows[m] += 2 * l.Npad;
  }
  size_t off = 0;
  b.off_table = off; off = align_up(off + layers.size() * sizeof(LayerDev), 256);
  b.off_absmax = off; off = align_up(off + layers.size() * sizeof(unsigned), 256);
  for (auto& l : layers) {
    l.off_bias = off; off = align_up(off + l.Npad * 4, 256);
    l.off_g = off; off = align_up(off + l.Npad * 4, 256);
    l.off_b = off; off = align_up(off + l.Npad * 4, 256);
  }
  b.off_extra = off; off += extra;
  for (int m = 0; m < b.nmaps; ++m) {
    off = align_up(off, 1024);
    b.map_off[m] = off;
    off += static_cast<size_t>(b.map_rows[m]) * b.map_kpad[m] * 2;
  }
  b.bytes = align_up(off, 1024);
  for (auto& l : layers) {
    l.off_hi = b.map_off[l.wmap - base_map] + static_cast<size_t>(l.wrow) * l.Kpad * 2;
    l.off_lo = l.off_hi + static_cast<size_t>(l.Npad) * l.Kpad * 2;
  }
  return true;
}

// Target Q ensemble (_target_Qs_params.*, world_model.py:41): its own caller-owned blob, so that a planner that never
// runs a target op keeps its packed_bytes.  Same layer shapes as the online heads; its maps follow the online ones.
struct TargetQ {
  std::vector<LayerHost> layers;   // 3 * num_q, head h layer l at 3 h + l
  BlobLayout lay;                  // lay.bytes == 0: the model's maps leave no room (target ops unsupported)
  uint8_t* blob = nullptr;
  bool packed = false;
};

struct tdmpc2_planner {
  tdmpc2_dims d;
  int num_sms = 0, nslots = 0;
  std::vector<LayerHost> layers;
  int li_enc = 0, li_dyn = 0, li_rew = 0, li_pi = 0, li_q = 0, li_term = -1, num_enc = 0;
  int KpadX = 0, KpadH = 0, NpadMax = 0, Ppad = 1, tiles_per_env = 0;
  // packed blob: the layers' layout, then the extra vectors in its `extra` bytes
  BlobLayout lay;
  size_t off_emb = 0, off_masks = 0, off_disc = 0, off_bins = 0;
  // workspace offsets
  size_t off_X = 0, off_H = 0, off_raw = 0, off_z = 0, off_pia = 0, off_mean = 0, off_std = 0, off_values = 0,
         off_counter = 0, off_score = 0, off_eact = 0, off_eidx = 0, off_zbias = 0, ws_bytes = 0;
  uint8_t* packed = nullptr;
  uint8_t* ws = nullptr;
  PlanParams base;
  int engine = TDMPC2_ENGINE_TCGEN05;
  bool bound = false, weights_ok = false;
  bool attr_done[6] = {};           // dynamic-smem opt-in done, per plan_kernel instantiation
  TargetQ tq;
  int64_t launches = 0;
  size_t l2_window_bytes = 0;       // > 0: launches carry a persisting-L2 access-policy window over the activation scratch
  float l2_hit_ratio = 1.f;
  int passes = 3;                   // 3 = fp32-parity arithmetic, 1 = declared non-parity fast mode (PlanParams::passes)
  int zb_kc0 = 0, zb_pitch = 0;     // shared-latent fold (PlanParams::zbias): K-chunks of [z | emb] folded into a per-env bias
  const int32_t* cur_task = nullptr;
  long long* prof = nullptr;
};

extern "C" int tdmpc2_abi_version(void) { return TDMPC2_B200_ABI_VERSION; }
extern "C" const char* tdmpc2_last_error(void) { return g_err.c_str(); }

static int check_device(int* num_sms) {
  int dev = 0, ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(TDMPC2_ERR_NO_DEVICE, "no CUDA device: the planner has no CPU fallback");
  }
  CUDA_TRY(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0)
    return fail(TDMPC2_ERR_NO_DEVICE, "device %d (%s) is sm_%d%d; this library is built for sm_90a only", dev, prop.name,
                prop.major, prop.minor);
  *num_sms = prop.multiProcessorCount;
  return 0;
}

extern "C" int tdmpc2_planner_create(const tdmpc2_dims* dims, tdmpc2_planner** out) {
  if (!dims || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  const tdmpc2_dims& d = *dims;
  if (d.episodic != 0 && d.episodic != 1) return fail(TDMPC2_ERR_INVALID, "episodic must be 0 or 1");
  if (d.episodic && d.task_dim > 0)   // WorldModel.termination asserts task is None (world_model.py:136)
    return fail(TDMPC2_ERR_UNSUPPORTED, "episodic (termination head) models are single-task in the reference");
  if (d.num_envs < 1 || d.num_samples < 1 || d.horizon < 1 || d.iterations < 1 || d.obs_dim < 1 || d.action_dim < 1 ||
      d.latent_dim < 1 || d.mlp_dim < 1 || d.enc_dim < 1 || d.num_enc_layers < 0 || d.num_q < 2 || d.num_bins < 0 ||
      d.task_dim < 0 || d.num_tasks < 1)
    return fail(TDMPC2_ERR_INVALID, "non-positive dimension");
  if (d.num_bins < 2)   // math.two_hot_inv's num_bins == 0 (raw) / == 1 (symexp only) regression heads (math.py:76-79)
    return fail(TDMPC2_ERR_UNSUPPORTED, "num_bins=%d: only the discrete-regression heads (num_bins >= 2) are built; the "
                "reference's num_bins 0 / 1 scalar heads are not supported by the fused planner", d.num_bins);
  if (d.num_elites < 1 || d.num_elites > d.num_samples) return fail(TDMPC2_ERR_INVALID, "num_elites must be in [1, num_samples]");
  if (d.num_pi_trajs < 0 || d.num_pi_trajs > 128 || d.num_pi_trajs > d.num_samples)
    return fail(TDMPC2_ERR_INVALID, "num_pi_trajs must be in [0, min(128, num_samples)]");
  if (d.num_samples > 4096) return fail(TDMPC2_ERR_INVALID, "num_samples > 4096 unsupported");
  if (d.num_elites > 1024) return fail(TDMPC2_ERR_INVALID, "num_elites > 1024 unsupported");
  if (pad_to(d.action_dim, 32) + d.action_dim > kMaxHeadCols || d.num_bins > kMaxHeadCols)
    return fail(TDMPC2_ERR_INVALID, "pad32(action_dim)+action_dim and num_bins must be <= %d", kMaxHeadCols);
  if (d.simnorm_dim != 8 || d.latent_dim % 8 != 0)
    return fail(TDMPC2_ERR_INVALID, "simnorm_dim must be 8 and divide latent_dim");
  const int n_hidden = d.num_enc_layers - 1 > 1 ? d.num_enc_layers - 1 : 1;   // layers.py:157
  if (n_hidden + 1 > TDMPC2_MAX_ENC_LAYERS) return fail(TDMPC2_ERR_INVALID, "too many encoder layers");
  int num_sms = 0;
  int rc = check_device(&num_sms);
  if (rc) return rc;

  tdmpc2_planner* p = new tdmpc2_planner();
  p->d = d;
  p->num_sms = num_sms;
  p->nslots = num_sms;
  const int L = d.latent_dim, M = d.mlp_dim, A = d.action_dim, T = d.task_dim, B = d.num_bins;
  const int D = L + T + A;
  auto add = [&](int K, int N, bool ln) {
    LayerHost l{};
    l.K = K; l.Kpad = pad_to(K, kKch); l.N = N; l.Npad = pad_to(N, 128); l.has_ln = ln ? 1 : 0;
    l.src_n = N; l.split_at = N; l.split_to = N;
    p->layers.push_back(l);
    return static_cast<int>(p->layers.size()) - 1;
  };
  // encoder: mlp(obs+T, n_hidden*[enc_dim], L, act=SimNorm)  (layers.py:157-159); num_enc_layers == 0: the model has no
  // state encoder (pixel observations: tdmpc2_pixel_encode + tdmpc2_plan_prologue_latent supply the latent)
  p->num_enc = d.num_enc_layers == 0 ? 0 : n_hidden + 1;
  p->li_enc = static_cast<int>(p->layers.size());
  if (p->num_enc > 0) { int k = d.obs_dim + T; for (int i = 0; i < n_hidden; ++i) { add(k, d.enc_dim, true); k = d.enc_dim; } add(k, L, true); }
  p->li_dyn = static_cast<int>(p->layers.size()); add(D, M, true); add(M, M, true); add(M, L, true);
  p->li_rew = static_cast<int>(p->layers.size()); add(D, M, true); add(M, M, true); add(M, B, false);
  p->li_pi = static_cast<int>(p->layers.size()); add(L + T, M, true); add(M, M, true);
  {
    // pi head: rows [0, A) = mean logits, rows [A, 2A) = log_std logits, the latter moved to column pad32(A)
    const int Apad = pad_to(A, 32);
    const int i = add(M, Apad + A, false);
    p->layers[i].src_n = 2 * A; p->layers[i].split_at = A; p->layers[i].split_to = Apad;
  }
  p->li_q = static_cast<int>(p->layers.size());
  for (int h = 0; h < d.num_q; ++h) { add(D, M, true); add(M, M, true); add(M, B, false); }
  // termination head: mlp(L+T, 2*[M], 1) on z_{t+1}  (world_model.py:28); appended so the other layer indices stay put
  p->li_term = -1;
  if (d.episodic) { p->li_term = static_cast<int>(p->layers.size()); add(L + T, M, true); add(M, M, true); add(M, 1, false); }

  // ---- packed blob layout; the extra vectors sit between the per-layer vectors and the weight maps
  const size_t emb_bytes = align_up(static_cast<size_t>(d.num_tasks) * std::max(T, 1) * 4, 256);
  const size_t mask_bytes = align_up(static_cast<size_t>(d.num_tasks) * A * 4, 256);
  const size_t disc_bytes = align_up(static_cast<size_t>(d.num_tasks) * (d.horizon + 1) * 4, 256);
  const size_t bins_bytes = align_up(static_cast<size_t>(B) * 4, 256);
  if (!layout_blob(p->layers, 0, emb_bytes + mask_bytes + disc_bytes + bins_bytes, p->lay)) {
    delete p;
    return fail(TDMPC2_ERR_INVALID, "more than %d distinct padded input widths", kMaxWMaps);
  }
  p->off_emb = p->lay.off_extra;
  p->off_masks = p->off_emb + emb_bytes;
  p->off_disc = p->off_masks + mask_bytes;
  p->off_bins = p->off_disc + disc_bytes;

  p->KpadX = std::max(pad_to(D, kKch), pad_to(d.obs_dim + T, kKch));
  p->KpadH = std::max(pad_to(M, kKch), pad_to(d.enc_dim, kKch));
  p->NpadMax = 0;
  for (auto& l : p->layers) p->NpadMax = std::max(p->NpadMax, l.Npad);
  p->Ppad = 1;
  while (p->Ppad < d.num_pi_trajs) p->Ppad <<= 1;
  p->tiles_per_env = (d.num_samples + kTileM - 1) / kTileM;

  // ---- workspace layout
  const size_t E = d.num_envs, H = d.horizon, N = d.num_samples, K = d.num_elites, P = d.num_pi_trajs;
  size_t off = 0;
  p->off_X = off; off = align_up(off + static_cast<size_t>(p->nslots) * 2 * kTileM * p->KpadX * 2, 1024);
  p->off_H = off; off = align_up(off + static_cast<size_t>(p->nslots) * 2 * kTileM * p->KpadH * 2, 1024);
  p->off_raw = off; off = align_up(off + static_cast<size_t>(p->nslots) * kTileM * p->NpadMax * 4, 1024);
  p->off_z = off; off = align_up(off + E * L * 4, 256);
  p->off_pia = off; off = align_up(off + E * H * std::max<size_t>(P, 1) * A * 4, 256);
  p->off_mean = off; off = align_up(off + E * H * A * 4, 256);
  p->off_std = off; off = align_up(off + E * H * A * 4, 256);
  p->off_values = off; off = align_up(off + E * N * 4, 256);
  p->off_counter = off; off = align_up(off + E * 4, 256);
  p->off_score = off; off = align_up(off + E * K * 4, 256);
  p->off_eact = off; off = align_up(off + E * K * A * 4, 256);
  p->off_eidx = off; off = align_up(off + E * K * 4, 256);
  // shared-latent fold: whole 64-column chunks of [z | emb] (TDMPC2_B200_ZFOLD=0 turns it off: A/B knob)
  p->zb_pitch = p->layers[p->li_rew].Npad;
  p->zb_kc0 = env_uint("TDMPC2_B200_ZFOLD", 1) ? (L + T) / kKch : 0;
  p->off_zbias = off; off = align_up(off + 2 * E * static_cast<size_t>(p->zb_pitch) * 4, 256);
  p->ws_bytes = align_up(off, 1024);

  // ---- target Q blob: copies of the online heads' layers, with weight maps of their own after the online ones
  TargetQ& tq = p->tq;
  tq.layers.assign(p->layers.begin() + p->li_q, p->layers.begin() + p->li_q + 3 * d.num_q);
  if (!layout_blob(tq.layers, p->lay.nmaps, 0, tq.lay)) tq.layers.clear();
  *out = p;
  return 0;
}

extern "C" void tdmpc2_planner_destroy(tdmpc2_planner* p) { delete p; }
extern "C" int tdmpc2_planner_packed_bytes(const tdmpc2_planner* p, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  *out = p->lay.bytes;
  return 0;
}
extern "C" int tdmpc2_planner_workspace_bytes(const tdmpc2_planner* p, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  *out = p->ws_bytes;
  return 0;
}
extern "C" int tdmpc2_planner_layer_count(const tdmpc2_planner* p) { return p ? static_cast<int>(p->layers.size()) : -1; }
extern "C" int64_t tdmpc2_planner_launch_count(const tdmpc2_planner* p) { return p ? p->launches : -1; }
extern "C" int tdmpc2_planner_set_profile(tdmpc2_planner* p, long long* device_buf) {
  if (!p) return fail(TDMPC2_ERR_INVALID, "null planner");
  p->prof = device_buf;
  return 0;
}
extern "C" int tdmpc2_planner_set_engine(tdmpc2_planner* p, int engine) {
  if (!p || (engine != TDMPC2_ENGINE_TCGEN05 && engine != TDMPC2_ENGINE_SIMT && engine != TDMPC2_ENGINE_TCGEN05_2SM &&
             engine != TDMPC2_ENGINE_TCGEN05_PP && engine != TDMPC2_ENGINE_TCGEN05_2SM_PF))
    return fail(TDMPC2_ERR_INVALID, "bad engine");
  p->engine = engine;
  return 0;
}

// The tensor-core engine adds every 64-element K-chunk's partial sum with round-to-nearest, which is finer than any
// segment length these calls can ask for: they validate their argument and change nothing on this build.
extern "C" int tdmpc2_planner_set_kseg(tdmpc2_planner* p, int k_elems) {
  if (!p || k_elems < 0) return fail(TDMPC2_ERR_INVALID, "bad kseg");
  return 0;
}
extern "C" int tdmpc2_planner_set_head_kseg(tdmpc2_planner* p, int k_elems) {
  if (!p || k_elems < 0) return fail(TDMPC2_ERR_INVALID, "bad head kseg");
  return 0;
}

extern "C" int tdmpc2_planner_set_passes(tdmpc2_planner* p, int passes) {
  if (!p || (passes != 1 && passes != 3)) return fail(TDMPC2_ERR_INVALID, "passes must be 3 (fp32 parity) or 1 (non-parity fast mode)");
  p->passes = passes;
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_map(EncodeTiledFn enc, CUtensorMap* m, void* base, uint64_t kpad, uint64_t rows) {
  cuuint64_t dims[2] = {kpad, rows};
  cuuint64_t strides[1] = {kpad * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kKch), static_cast<cuuint32_t>(kTileM)};
  cuuint32_t estr[2] = {1, 1};
  // 64-column boxes (operand loads): 128-byte rows, 128B swizzle (the wgmma operand layout)
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(TDMPC2_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) kpad=%llu rows=%llu", (int)r,
                                     (unsigned long long)kpad, (unsigned long long)rows);
  return 0;
}

// Binds `blob`, laid out by `lay`, to its TMA weight maps and writes its layer table (host part; inv_scale is filled by
// the pack kernel).
static int bind_blob(EncodeTiledFn enc, CUtensorMap* tmW, const std::vector<LayerHost>& layers, const BlobLayout& lay,
                     uint8_t* blob) {
  int rc;
  for (int m = 0; m < lay.nmaps; ++m)
    if ((rc = make_map(enc, &tmW[lay.base_map + m], blob + lay.map_off[m], lay.map_kpad[m], lay.map_rows[m]))) return rc;
  std::vector<LayerDev> tab(layers.size());
  for (size_t i = 0; i < tab.size(); ++i) {
    const LayerHost& l = layers[i];
    LayerDev& t = tab[i];
    t.K = l.K; t.Kpad = l.Kpad; t.N = l.N; t.Npad = l.Npad; t.wmap = l.wmap; t.wrow = l.wrow; t.has_ln = l.has_ln;
    t.inv_scale = 1.f;
    t.bias = reinterpret_cast<const float*>(blob + l.off_bias);
    t.ln_g = reinterpret_cast<const float*>(blob + l.off_g);
    t.ln_b = reinterpret_cast<const float*>(blob + l.off_b);
    t.w_hi = reinterpret_cast<const __half*>(blob + l.off_hi);
    t.w_lo = reinterpret_cast<const __half*>(blob + l.off_lo);
  }
  CUDA_TRY(cudaMemcpy(blob + lay.off_table, tab.data(), tab.size() * sizeof(LayerDev), cudaMemcpyHostToDevice));
  return 0;
}

static EncodeTiledFn encode_tiled_fn() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return reinterpret_cast<EncodeTiledFn>(fn);
}

extern "C" int tdmpc2_planner_bind(tdmpc2_planner* p, void* packed, void* workspace) {
  if (!p || !packed || !workspace) return fail(TDMPC2_ERR_INVALID, "null argument");
  if ((reinterpret_cast<uintptr_t>(packed) & 255) || (reinterpret_cast<uintptr_t>(workspace) & 255))
    return fail(TDMPC2_ERR_INVALID, "buffers must be 256-byte aligned");
  p->packed = static_cast<uint8_t*>(packed);
  p->ws = static_cast<uint8_t*>(workspace);
  CUDA_TRY(cudaMemset(p->ws, 0, p->ws_bytes));
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return fail(TDMPC2_ERR_CUDA, "cuTensorMapEncodeTiled not available");

  const tdmpc2_dims& d = p->d;
  PlanParams& B = p->base;
  memset(&B, 0, sizeof(B));
  int rc;
  if ((rc = make_map(enc, &B.tmX, p->ws + p->off_X, p->KpadX, static_cast<uint64_t>(p->nslots) * 2 * kTileM))) return rc;
  if ((rc = make_map(enc, &B.tmH, p->ws + p->off_H, p->KpadH, static_cast<uint64_t>(p->nslots) * 2 * kTileM))) return rc;
  if ((rc = bind_blob(enc, B.tmW, p->layers, p->lay, p->packed))) return rc;

  B.layers = reinterpret_cast<const LayerDev*>(p->packed + p->lay.off_table);
  B.E = d.num_envs; B.N = d.num_samples; B.P = d.num_pi_trajs; B.Ppad = p->Ppad; B.K = d.num_elites; B.H = d.horizon;
  B.obs_dim = d.obs_dim; B.A = d.action_dim; B.Apad = pad_to(d.action_dim, 32); B.L = d.latent_dim; B.M = d.mlp_dim; B.T = d.task_dim; B.B = d.num_bins;
  B.num_q = d.num_q; B.simnorm = d.simnorm_dim; B.num_enc = p->num_enc;
  B.tiles_per_env = p->tiles_per_env; B.KpadX = p->KpadX; B.KpadH = p->KpadH; B.NpadMax = p->NpadMax;
  B.li_enc = p->li_enc; B.li_dyn = p->li_dyn; B.li_rew = p->li_rew; B.li_pi = p->li_pi; B.li_q = p->li_q; B.li_term = p->li_term;
  B.temperature = d.temperature; B.min_std = d.min_std; B.max_std = d.max_std;
  B.log_std_min = d.log_std_min; B.log_std_dif = d.log_std_dif;
  B.X = reinterpret_cast<__half*>(p->ws + p->off_X);
  B.Hb = reinterpret_cast<__half*>(p->ws + p->off_H);
  B.raw = reinterpret_cast<float*>(p->ws + p->off_raw);
  B.emb = d.task_dim > 0 ? reinterpret_cast<const float*>(p->packed + p->off_emb) : nullptr;
  B.masks = nullptr;   // set by pack_weights when the model is multi-task
  B.disc_pow = reinterpret_cast<const float*>(p->packed + p->off_disc);
  B.bins = reinterpret_cast<const float*>(p->packed + p->off_bins);
  B.z = reinterpret_cast<float*>(p->ws + p->off_z);
  B.pi_actions = reinterpret_cast<float*>(p->ws + p->off_pia);
  B.mean = reinterpret_cast<float*>(p->ws + p->off_mean);
  B.std = reinterpret_cast<float*>(p->ws + p->off_std);
  B.values = reinterpret_cast<float*>(p->ws + p->off_values);
  B.env_counter = reinterpret_cast<unsigned*>(p->ws + p->off_counter);
  B.score = reinterpret_cast<float*>(p->ws + p->off_score);
  B.elite_act0 = reinterpret_cast<float*>(p->ws + p->off_eact);
  B.elite_idx32 = reinterpret_cast<int*>(p->ws + p->off_eidx);
  B.zbias = reinterpret_cast<const float*>(p->ws + p->off_zbias);
  B.zb_kc0 = 0; B.zb_pitch = p->zb_pitch;       // zb_kc0 is set on the CEM-iteration launches only
  p->bound = true;
  p->weights_ok = false;
  p->tq.blob = nullptr;       // re-encoded maps / table: the target blob must be bound again
  p->tq.packed = false;
  return 0;
}

// Pack Linear `lin` (head `head` of a stacked ensemble tensor) into layer li of `layers`, laid out in `blob` by `lay`.
static int pack_layer(tdmpc2_planner* p, const std::vector<LayerHost>& layers, const BlobLayout& lay, uint8_t* blob,
                      int li, const tdmpc2_linear& lin, size_t head, cudaStream_t st) {
  const LayerHost& l = layers[li];
  LayerDev* table = reinterpret_cast<LayerDev*>(blob + lay.off_table);
  unsigned* absmax = reinterpret_cast<unsigned*>(blob + lay.off_absmax);
  if (!lin.weight || !lin.bias) return fail(TDMPC2_ERR_INVALID, "layer %d: null weight/bias", li);
  if (l.has_ln && (!lin.ln_weight || !lin.ln_bias)) return fail(TDMPC2_ERR_INVALID, "layer %d: missing LayerNorm tensors", li);
  const float* W = lin.weight + head * static_cast<size_t>(l.src_n) * l.K;
  const size_t n = static_cast<size_t>(l.src_n) * l.K;
  const int blocks = static_cast<int>(std::min<size_t>((n + 255) / 256, 1024));
  absmax_kernel<<<blocks, 256, 0, st>>>(W, n, absmax + li);
  const size_t tot = static_cast<size_t>(l.Npad) * l.Kpad;
  split_weight_kernel<<<static_cast<int>(std::min<size_t>((tot + 255) / 256, 2048)), 256, 0, st>>>(
      W, l.N, l.K, l.Npad, l.Kpad, reinterpret_cast<__half*>(blob + l.off_hi),
      reinterpret_cast<__half*>(blob + l.off_lo), absmax + li, table + li, l.src_n, l.split_at, l.split_to);
  const int vb = (l.Npad + 255) / 256;
  pad_vector_kernel<<<vb, 256, 0, st>>>(lin.bias + head * l.src_n, l.N, l.Npad, reinterpret_cast<float*>(blob + l.off_bias),
                                        0.f, l.src_n, l.split_at, l.split_to);
  pad_vector_kernel<<<vb, 256, 0, st>>>(l.has_ln ? lin.ln_weight + head * l.src_n : nullptr, l.N, l.Npad,
                                        reinterpret_cast<float*>(blob + l.off_g), 1.f, l.src_n, l.split_at, l.split_to);
  pad_vector_kernel<<<vb, 256, 0, st>>>(l.has_ln ? lin.ln_bias + head * l.src_n : nullptr, l.N, l.Npad,
                                        reinterpret_cast<float*>(blob + l.off_b), 0.f, l.src_n, l.split_at, l.split_to);
  p->launches += 5;
  return 0;
}

extern "C" int tdmpc2_pack_weights(tdmpc2_planner* p, const tdmpc2_weights* w, void* stream_) {
  if (!p || !w) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (!p->bound) return fail(TDMPC2_ERR_STATE, "tdmpc2_planner_bind must be called first");
  if (w->num_enc != p->num_enc) return fail(TDMPC2_ERR_INVALID, "expected %d encoder layers, got %d", p->num_enc, w->num_enc);
  const tdmpc2_dims& d = p->d;
  if (d.task_dim > 0 && (!w->task_emb || !w->action_masks)) return fail(TDMPC2_ERR_INVALID, "multi-task model needs task_emb and action_masks");
  if (!w->discount_pow || !w->bins) return fail(TDMPC2_ERR_INVALID, "discount_pow and bins are required");
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(p->packed + p->lay.off_absmax, 0, p->layers.size() * sizeof(unsigned), st));
  auto pack_one = [&](int li, const tdmpc2_linear& lin, size_t head) -> int {
    return pack_layer(p, p->layers, p->lay, p->packed, li, lin, head, st);
  };
  int rc;
  for (int i = 0; i < p->num_enc; ++i) if ((rc = pack_one(p->li_enc + i, w->enc[i], 0))) return rc;
  for (int i = 0; i < 3; ++i) {
    if ((rc = pack_one(p->li_dyn + i, w->dynamics[i], 0))) return rc;
    if ((rc = pack_one(p->li_rew + i, w->reward[i], 0))) return rc;
    if ((rc = pack_one(p->li_pi + i, w->pi[i], 0))) return rc;
    for (int h = 0; h < d.num_q; ++h) if ((rc = pack_one(p->li_q + 3 * h + i, w->qs[i], h))) return rc;
    if (d.episodic && (rc = pack_one(p->li_term + i, w->termination[i], 0))) return rc;
  }
  if (d.task_dim > 0) {
    emb_renorm_kernel<<<d.num_tasks, 32, 0, st>>>(w->task_emb, d.task_dim, reinterpret_cast<float*>(p->packed + p->off_emb));
    CUDA_TRY(cudaMemcpyAsync(p->packed + p->off_masks, w->action_masks, static_cast<size_t>(d.num_tasks) * d.action_dim * 4,
                             cudaMemcpyDeviceToDevice, st));
    p->base.masks = reinterpret_cast<const float*>(p->packed + p->off_masks);
    p->launches += 1;
  } else {
    p->base.masks = nullptr;
  }
  CUDA_TRY(cudaMemcpyAsync(p->packed + p->off_disc, w->discount_pow, static_cast<size_t>(d.num_tasks) * (d.horizon + 1) * 4,
                           cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(p->packed + p->off_bins, w->bins, static_cast<size_t>(d.num_bins) * 4, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaGetLastError());
  p->weights_ok = true;
  return 0;
}

// ------------------------------------------------------------------------------------ launches
// The engine the CEM-iteration launches of this planner actually run.  The CTA-pair and ping-pong engines (2, 3, 4) are
// built on Blackwell's cta_group::2 MMAs; on sm_90a they run as the single-CTA tensor-core engine 0.
extern "C" int tdmpc2_planner_iter_engine(const tdmpc2_planner* p) {
  if (!p) return -1;
  return p->engine == TDMPC2_ENGINE_SIMT ? TDMPC2_ENGINE_SIMT : TDMPC2_ENGINE_TCGEN05;
}

// Launch attributes shared by every plan_kernel launch: when enabled (tdmpc2_planner_set_l2_persist), an access-policy
// window that keeps the per-CTA activation scratch (X + H planes, contiguous in the workspace) resident in the
// persisting part of L2, so that its dirty lines are not written back to HBM while noise and weights stream through.
struct LaunchCfg {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  LaunchCfg(tdmpc2_planner* p, int grid, size_t smem, cudaStream_t st);
};

// Every plan_kernel launch.  The instantiation follows the engine and the kind of launch: planning, the rollout modes of
// an episodic model (MODE_ITER / MODE_VALUE with the termination head), or row mode.  Row launches are not profiled.
static int launch(tdmpc2_planner* p, const PlanParams& prm, void* stream_) {
  using Kernel = void (*)(PlanParams);
  static const Kernel kernels[2][3] = {
      {plan_kernel<ENGINE_TC>, plan_kernel<ENGINE_TC, true>, plan_kernel<ENGINE_TC, false, true>},
      {plan_kernel<ENGINE_SIMT>, plan_kernel<ENGINE_SIMT, true>, plan_kernel<ENGINE_SIMT, false, true>}};
  const bool rows = prm.mode == MODE_ROWS;
  const int kind = rows ? 2 : (p->d.episodic && (prm.mode == MODE_ITER || prm.mode == MODE_VALUE)) ? 1 : 0;
  const int engine = p->engine == TDMPC2_ENGINE_SIMT ? 1 : 0;
  const Kernel kernel = kernels[engine][kind];
  bool& attr_done = p->attr_done[3 * engine + kind];
  if (!attr_done) {     // > 48 KiB of dynamic shared memory needs the opt-in, once per kernel instantiation
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_done = true;
  }
  PlanParams prm2 = prm;
  prm2.prof = rows ? nullptr : p->prof;
  prm2.prof_slots = p->nslots;
  prm2.passes = p->passes;
  LaunchCfg lc(p, std::min(prm.ntiles, p->nslots), kSmemBytes, static_cast<cudaStream_t>(stream_));
  CUDA_TRY(cudaLaunchKernelEx(&lc.cfg, kernel, prm2));
  CUDA_TRY(cudaGetLastError());
  p->launches += 1;
  return 0;
}

LaunchCfg::LaunchCfg(tdmpc2_planner* p, int grid, size_t smem, cudaStream_t st) {
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  int n = 0;
  if (p->l2_window_bytes > 0) {
    attr[n].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[n].val.accessPolicyWindow.base_ptr = p->ws + p->off_X;
    attr[n].val.accessPolicyWindow.num_bytes = p->l2_window_bytes;
    attr[n].val.accessPolicyWindow.hitRatio = p->l2_hit_ratio;
    attr[n].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr[n].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
}

// Keep the activation scratch in the persisting part of L2 (0 = off).  Sets the device's persisting-L2 carve-out to
// what the scratch needs (capped by the device maximum) -- a device-wide setting, hence opt-in.
extern "C" int tdmpc2_planner_set_l2_persist(tdmpc2_planner* p, int enable) {
  if (!p) return fail(TDMPC2_ERR_INVALID, "null planner");
  if (!p->bound) return fail(TDMPC2_ERR_STATE, "tdmpc2_planner_bind must be called first");
  if (!enable) { p->l2_window_bytes = 0; return 0; }
  int dev = 0, max_persist = 0, max_window = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
  const size_t scratch = p->off_raw - p->off_X;              // X planes + H planes of all slots
  if (max_persist <= 0 || max_window <= 0) return fail(TDMPC2_ERR_UNSUPPORTED, "device has no persisting L2");
  const size_t carve = std::min<size_t>(scratch, static_cast<size_t>(max_persist));
  CUDA_TRY(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve));
  p->l2_window_bytes = std::min<size_t>(scratch, static_cast<size_t>(max_window));
  p->l2_hit_ratio = std::min(1.0f, static_cast<float>(carve) / static_cast<float>(p->l2_window_bytes));
  return 0;
}

static int ready(tdmpc2_planner* p) {
  if (!p) return fail(TDMPC2_ERR_INVALID, "null planner");
  if (!p->bound || !p->weights_ok) return fail(TDMPC2_ERR_STATE, "planner needs bind() and pack_weights() first");
  return 0;
}

// obs != nullptr: z = encode(obs, task) through the state encoder; z_in != nullptr: the latent is given (pixel models)
static int prologue_impl(tdmpc2_planner* p, const float* obs, const float* z_in, const int32_t* task, const uint8_t* t0,
                         const float* prev_mean, const float* noise_prior, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  if ((!obs && !z_in) || !t0 || !prev_mean) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (obs && p->num_enc == 0) return fail(TDMPC2_ERR_STATE, "this planner was created without a state encoder (num_enc_layers = 0): use tdmpc2_plan_prologue_latent");
  if (d.task_dim > 0 && !task) return fail(TDMPC2_ERR_INVALID, "multi-task model needs task indices");
  if (d.num_pi_trajs > 0 && !noise_prior) return fail(TDMPC2_ERR_INVALID, "noise_prior is required when num_pi_trajs > 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  p->cur_task = d.task_dim > 0 ? task : nullptr;
  const int n = d.num_envs * d.horizon * d.action_dim;
  init_state_kernel<<<(std::max(n, d.num_envs) + 255) / 256, 256, 0, st>>>(p->base.mean, p->base.std, p->base.env_counter,
                                                                          prev_mean, t0, d.num_envs, d.horizon, d.action_dim,
                                                                          d.max_std);
  p->launches += 1;
  PlanParams prm = p->base;
  prm.task = p->cur_task;
  if (obs) {
    prm.obs = obs;
    prm.mode = MODE_ENCODE;
    prm.ntiles = (d.num_envs + kTileM - 1) / kTileM;
    if ((rc = launch(p, prm, st))) return rc;
  } else {
    CUDA_TRY(cudaMemcpyAsync(p->base.z, z_in, static_cast<size_t>(d.num_envs) * d.latent_dim * 4, cudaMemcpyDeviceToDevice, st));
  }
  if (p->zb_kc0 > 0) {
    // shared-latent fold: [z | emb] . W of reward.0 / dynamics.0, once per plan() (z is the same in every CEM iteration)
    const dim3 grid((p->zb_pitch + kZbCols - 1) / kZbCols, (d.num_envs + kZbEnvs - 1) / kZbEnvs, 2);
    zbias_kernel<<<grid, 256, 0, st>>>(p->base.layers, p->li_rew, p->li_dyn, p->base.z, p->base.emb, p->cur_task, d.num_envs,
                                       d.latent_dim, d.task_dim, p->zb_kc0 * kKch, reinterpret_cast<float*>(p->ws + p->off_zbias),
                                       p->zb_pitch);
    CUDA_TRY(cudaGetLastError());
    p->launches += 1;
  }
  if (d.num_pi_trajs > 0) {
    prm.mode = MODE_PRIOR;
    prm.noise_prior = noise_prior;
    const int per = kTileM / p->Ppad;
    prm.ntiles = (d.num_envs + per - 1) / per;
    if ((rc = launch(p, prm, st))) return rc;
  }
  return 0;
}

extern "C" int tdmpc2_plan_prologue(tdmpc2_planner* p, const float* obs, const int32_t* task, const uint8_t* t0,
                                    const float* prev_mean, const float* noise_prior, void* stream_) {
  if (!obs) return fail(TDMPC2_ERR_INVALID, "null argument");
  return prologue_impl(p, obs, nullptr, task, t0, prev_mean, noise_prior, stream_);
}
extern "C" int tdmpc2_plan_prologue_latent(tdmpc2_planner* p, const float* z, const int32_t* task, const uint8_t* t0,
                                           const float* prev_mean, const float* noise_prior, void* stream_) {
  if (!z) return fail(TDMPC2_ERR_INVALID, "null argument");
  return prologue_impl(p, nullptr, z, task, t0, prev_mean, noise_prior, stream_);
}

// ------------------------------------------------------------------------------------ pixel encoder (cfg.obs == 'rgb')
struct tdmpc2_pixel_encoder {
  tdmpc2_pixel_dims d;
  int num_sms = 0;                 // the persistent grid's width: one conv1 scratch slot per SM
  size_t ws_bytes = 0, smem = 0;
  bool attr_done = false;
};

extern "C" int tdmpc2_pixel_encoder_create(const tdmpc2_pixel_dims* dims, tdmpc2_pixel_encoder** out) {
  if (!dims || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  const tdmpc2_pixel_dims& d = *dims;
  if (d.num_envs < 1 || d.in_channels < 1 || d.num_channels < 8 || d.num_channels % 8 != 0 || d.simnorm_dim < 1 ||
      (16 * d.num_channels) % d.simnorm_dim != 0)
    return fail(TDMPC2_ERR_INVALID, "pixel encoder: num_channels must be a positive multiple of 8 and simnorm_dim must divide 16 * num_channels");
  int num_sms = 0;
  int rc = check_device(&num_sms);
  if (rc) return rc;
  // shared memory: the activations of the larger phase (staged frame / conv2-4 maps), plus every layer's weights and bias
  // next to its activations when they fit the opt-in maximum; otherwise the kernel stages them in chunks
  const size_t stage = pix_stage_floats(d.in_channels), maps = pix_maps_floats(d.num_channels), nc = d.num_channels;
  const size_t want = std::max({stage + nc * (d.in_channels * 49 + 1), maps + nc * (nc * 25 + 1), std::max(stage, maps)});
  const size_t smem = std::min(want * 4, static_cast<size_t>(kPixMaxSmem));
  const int cap1 = static_cast<int>(smem / 4) - static_cast<int>(stage), cap2 = static_cast<int>(smem / 4) - static_cast<int>(maps);
  int occ = 0, icc1 = 0, icc2 = 0, icc3 = 0;
  if (cap1 > 0) pix_chunk(d.in_channels, d.num_channels, 49, cap1, &occ, &icc1);
  if (cap2 > 0) { pix_chunk(d.num_channels, d.num_channels, 25, cap2, &occ, &icc2); pix_chunk(d.num_channels, d.num_channels, 9, cap2, &occ, &icc3); }
  if (std::max(stage, maps) * 4 > static_cast<size_t>(kPixMaxSmem) || icc1 < 1 || icc2 < 1 || icc3 < 1)
    return fail(TDMPC2_ERR_INVALID, "pixel encoder: %d input channels do not fit shared memory", d.in_channels);
  tdmpc2_pixel_encoder* e = new tdmpc2_pixel_encoder();
  e->d = d;
  e->num_sms = num_sms;
  e->ws_bytes = align_up(static_cast<size_t>(num_sms) * d.num_channels * kPixO1 * kPixO1 * 4, 256);
  e->smem = smem;
  *out = e;
  return 0;
}
extern "C" void tdmpc2_pixel_encoder_destroy(tdmpc2_pixel_encoder* e) { delete e; }
extern "C" int tdmpc2_pixel_encoder_workspace_bytes(const tdmpc2_pixel_encoder* e, size_t* out) {
  if (!e || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  *out = e->ws_bytes;
  return 0;
}

// One launch over `rows` frames: min(rows, SMs) CTAs, each looping over its frames with its own conv1 scratch slot.
// tape != nullptr: the frames' post-ReLU maps are written to it as well (conv1 straight into the frame's slot).
static int pixel_launch(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                        const float* shift, const float* grid_base, int64_t rows, float* z_out, float* tape, void* stream_) {
  if (!workspace || !w || !frames || !shift || !grid_base || !z_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  for (int i = 0; i < 4; ++i) if (!w->weight[i] || !w->bias[i]) return fail(TDMPC2_ERR_INVALID, "pixel encoder: null conv weight");
  PixelParams P{};
  P.frames = frames; P.shift = shift; P.grid = grid_base; P.scratch = static_cast<float*>(workspace); P.z = z_out; P.tape = tape;
  for (int i = 0; i < 4; ++i) { P.w[i] = w->weight[i]; P.b[i] = w->bias[i]; }
  P.rows = rows; P.C = e->d.in_channels; P.nc = e->d.num_channels; P.simnorm = e->d.simnorm_dim;
  P.smem_floats = static_cast<int>(e->smem / 4);
  if (!e->attr_done) {
    CUDA_TRY(cudaFuncSetAttribute(pixel_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(e->smem)));
    e->attr_done = true;
  }
  const int grid = static_cast<int>(std::min<int64_t>(rows, e->num_sms));
  pixel_encode_kernel<<<grid, kPixThreads, e->smem, static_cast<cudaStream_t>(stream_)>>>(P);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int tdmpc2_pixel_encode(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                                   const float* shift, const float* grid_base, float* z_out, void* stream_) {
  if (!e) return fail(TDMPC2_ERR_INVALID, "null argument");
  return pixel_launch(e, workspace, w, frames, shift, grid_base, e->d.num_envs, z_out, nullptr, stream_);
}

extern "C" int tdmpc2_pixel_encode_rows(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w,
                                        const float* frames, const float* shift, const float* grid_base, int64_t rows,
                                        float* z_out, void* stream_) {
  if (!e) {                        // an encoder exists only where a device does: report the missing device first
    int n = 0;
    const int rc = check_device(&n);
    return rc ? rc : fail(TDMPC2_ERR_INVALID, "null pixel encoder");
  }
  return pixel_launch(e, workspace, w, frames, shift, grid_base, rows, z_out, nullptr, stream_);
}

// ---- the conv encoder's backward (pixel_grad_kernels.cuh): taped forward, then the chain from dL/dz to the conv grads
extern "C" int tdmpc2_pixel_encode_tape_bytes(const tdmpc2_pixel_encoder* e, int64_t rows, size_t* out) {
  if (!e || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  *out = static_cast<size_t>(rows) * pix_tape_floats(e->d.num_channels) * 4;
  return 0;
}

extern "C" int tdmpc2_pixel_encode_taped(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w,
                                         const float* frames, const float* shift, const float* grid_base, int64_t rows,
                                         float* z_out, float* tape, void* stream_) {
  if (!e || !tape) return fail(TDMPC2_ERR_INVALID, "null argument");
  return pixel_launch(e, workspace, w, frames, shift, grid_base, rows, z_out, tape, stream_);
}

// Workspace of the backward (floats): the data gradients dp4 [rows][16 nc], dp3 [rows][nc 36], dp2 [rows][nc 169],
// dp1 [rows][nc 841], conv1's recomputed input [rows][C 4096], and the weight-gradient partials of the largest layer.
struct PixGradWs {
  size_t dp4, dp3, dp2, dp1, img, part, floats;
};
static PixGradWs pix_grad_ws(const tdmpc2_pixel_dims& d, int64_t rows) {
  const size_t R = static_cast<size_t>(rows), nc = d.num_channels, C = d.in_channels;
  PixGradWs w;
  size_t off = 0;
  w.dp4 = take64(off, R * nc * kPixO4 * kPixO4);
  w.dp3 = take64(off, R * nc * kPixO3 * kPixO3);
  w.dp2 = take64(off, R * nc * kPixO2 * kPixO2);
  w.dp1 = take64(off, R * nc * kPixO1 * kPixO1);
  w.img = take64(off, R * pix_stage_floats(d.in_channels));
  const int IC[4] = {static_cast<int>(C), static_cast<int>(nc), static_cast<int>(nc), static_cast<int>(nc)};
  const int KK[4] = {49, 25, 9, 9};
  size_t part = 0;
  for (int l = 0; l < 4; ++l)
    part = std::max(part, static_cast<size_t>(pixg_nsplit(IC[l], d.num_channels, KK[l], rows)) * nc * pixg_cols(IC[l], KK[l]));
  w.part = take64(off, part);
  w.floats = off;
  return w;
}

extern "C" int tdmpc2_pixel_backward_workspace_bytes(const tdmpc2_pixel_encoder* e, int64_t rows, size_t* out) {
  if (!e || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  *out = pix_grad_ws(e->d, rows).floats * 4;
  return 0;
}

extern "C" int tdmpc2_pixel_encode_backward(tdmpc2_pixel_encoder* e, const tdmpc2_conv_weights* w, const float* frames,
                                            const float* shift, const float* grid_base, int64_t rows, const float* tape,
                                            const float* z, const float* dz, const tdmpc2_conv_grads* grads, void* workspace,
                                            void* stream_) {
  if (!e || !w || !frames || !shift || !grid_base || !tape || !z || !dz || !grads || !workspace)
    return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  for (int i = 0; i < 4; ++i)
    if (!w->weight[i] || !w->bias[i] || !grads->weight[i] || !grads->bias[i])
      return fail(TDMPC2_ERR_INVALID, "pixel encoder: null conv weight or gradient");
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int C = e->d.in_channels, nc = e->d.num_channels, L = nc * kPixO4 * kPixO4;
  const int64_t tp = pix_tape_floats(nc);
  const PixGradWs W = pix_grad_ws(e->d, rows);
  float* ws = static_cast<float*>(workspace);
  float *dp4 = ws + W.dp4, *dp3 = ws + W.dp3, *dp2 = ws + W.dp2, *dp1 = ws + W.dp1, *img = ws + W.img, *part = ws + W.part;
  auto blocks = [](int64_t n) { return static_cast<int>(std::min<int64_t>((n + kPgThreads - 1) / kPgThreads, 1 << 20)); };
  // the weight and bias gradients of layer l from its output gradient dy and its input x (frame pitch xp)
  auto dw = [&](int l, auto kern, int KK, const float* dy, int OH, const float* x, int64_t xp, int IC, int IH) -> int {
    const int ns = pixg_nsplit(IC, nc, KK, rows), cols = pixg_cols(IC, KK);
    kern<<<dim3(pixg_ctas_x(IC, nc, KK), ns), kPgThreads, 0, st>>>(dy, nc, OH, OH, x, xp, IC, IH, IH, rows, ns, part);
    CUDA_TRY(cudaGetLastError());
    pixg_reduce<<<blocks(static_cast<int64_t>(nc) * cols), kPgThreads, 0, st>>>(part, ns, nc, cols, grads->weight[l], grads->bias[l]);
    CUDA_TRY(cudaGetLastError());
    return 0;
  };
  int rc;
  pixg_simnorm_back<<<blocks(rows * (L / e->d.simnorm_dim)), kPgThreads, 0, st>>>(z, dz, rows, L, e->d.simnorm_dim, dp4);
  CUDA_TRY(cudaGetLastError());
  if ((rc = dw(3, pixg_dw<3, 1>, 9, dp4, kPixO4, tape + pix_tape_a3(nc), tp, nc, kPixO3))) return rc;
  pixg_dx<3, 1><<<blocks(rows * nc * kPixO3 * kPixO3), kPgThreads, 0, st>>>(dp4, nc, kPixO4, kPixO4, w->weight[3], tape + pix_tape_a3(nc),
                                                                            tp, nc, kPixO3, kPixO3, rows, dp3);
  CUDA_TRY(cudaGetLastError());
  if ((rc = dw(2, pixg_dw<3, 2>, 9, dp3, kPixO3, tape + pix_tape_a2(nc), tp, nc, kPixO2))) return rc;
  pixg_dx<3, 2><<<blocks(rows * nc * kPixO2 * kPixO2), kPgThreads, 0, st>>>(dp3, nc, kPixO3, kPixO3, w->weight[2], tape + pix_tape_a2(nc),
                                                                            tp, nc, kPixO2, kPixO2, rows, dp2);
  CUDA_TRY(cudaGetLastError());
  if ((rc = dw(1, pixg_dw<5, 2>, 25, dp2, kPixO2, tape, tp, nc, kPixO1))) return rc;
  pixg_dx<5, 2><<<blocks(rows * nc * kPixO1 * kPixO1), kPgThreads, 0, st>>>(dp2, nc, kPixO2, kPixO2, w->weight[1], tape, tp, nc, kPixO1,
                                                                            kPixO1, rows, dp1);
  CUDA_TRY(cudaGetLastError());
  pixg_stage<<<blocks(rows * pix_stage_floats(C)), kPgThreads, 0, st>>>(frames, shift, grid_base, rows, C, img);
  CUDA_TRY(cudaGetLastError());
  return dw(0, pixg_dw<7, 2>, 49, dp1, kPixO1, img, pix_stage_floats(C), C, kPixHW);
}

extern "C" int tdmpc2_plan_iter(tdmpc2_planner* p, const float* noise_r, const float* noise_pi, const int32_t* qidx,
                                float* values_out, int64_t* elite_idx_out, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  if (!noise_pi || !qidx || (d.num_samples > d.num_pi_trajs && !noise_r)) return fail(TDMPC2_ERR_INVALID, "null argument");
  PlanParams prm = p->base;
  prm.task = p->cur_task;
  prm.mode = MODE_ITER;
  prm.noise_r = noise_r; prm.noise_pi = noise_pi; prm.qidx = qidx;
  prm.values_out = values_out;
  prm.elite_idx_out = reinterpret_cast<long long*>(elite_idx_out);
  prm.ntiles = d.num_envs * p->tiles_per_env;
  prm.zb_kc0 = p->zb_kc0;
  return launch(p, prm, stream_);
}

// Declared non-parity throughput mode: the iteration generates its two large noise tensors itself (rng.cuh).
extern "C" int tdmpc2_plan_iter_rng(tdmpc2_planner* p, const uint64_t* rng_state, int iteration, const int32_t* qidx,
                                    float* values_out, int64_t* elite_idx_out, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  if (!rng_state || !qidx || iteration < 0) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (p->engine == TDMPC2_ENGINE_SIMT) return fail(TDMPC2_ERR_UNSUPPORTED, "in-kernel noise needs a tensor-core engine");
  PlanParams prm = p->base;
  prm.task = p->cur_task;
  prm.mode = MODE_ITER;
  prm.noise_r = nullptr; prm.noise_pi = nullptr; prm.qidx = qidx;
  prm.rng_state = reinterpret_cast<const unsigned long long*>(rng_state);
  prm.rng_iter = iteration;
  prm.values_out = values_out;
  prm.elite_idx_out = reinterpret_cast<long long*>(elite_idx_out);
  prm.ntiles = d.num_envs * p->tiles_per_env;
  prm.zb_kc0 = p->zb_kc0;
  return launch(p, prm, stream_);
}
// Diagnostics / tests: the normals of `ngroups` consecutive groups of one stream (4 per group).
extern "C" int tdmpc2_debug_rng(const uint64_t* rng_state, uint32_t stream, uint64_t group0, int ngroups, float* out, void* stream_) {
  if (!rng_state || !out || ngroups < 1) return fail(TDMPC2_ERR_INVALID, "bad debug_rng arguments");
  rng_debug_kernel<<<(ngroups + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const unsigned long long*>(rng_state), stream, group0, ngroups, out);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int tdmpc2_plan_epilogue(tdmpc2_planner* p, const float* expo, const float* noise_final, float* action_out,
                                    float* prev_mean_out, int32_t* pick_out, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  if (!expo || !action_out || !prev_mean_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  const tdmpc2_dims& d = p->d;
  const int warps_per_block = 4;
  pick_kernel<<<(d.num_envs + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, static_cast<cudaStream_t>(stream_)>>>(
      p->base.score, p->base.elite_act0, p->base.mean, p->base.std, expo, noise_final, action_out, prev_mean_out, pick_out,
      d.num_envs, d.num_elites, d.horizon, d.action_dim);
  CUDA_TRY(cudaGetLastError());
  p->launches += 1;
  return 0;
}

extern "C" int tdmpc2_plan_get_state(tdmpc2_planner* p, float* mean, float* std, float* z, float* pi_actions, float* score,
                                     void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const size_t E = d.num_envs, H = d.horizon, A = d.action_dim;
  if (mean) CUDA_TRY(cudaMemcpyAsync(mean, p->base.mean, E * H * A * 4, cudaMemcpyDeviceToDevice, st));
  if (std) CUDA_TRY(cudaMemcpyAsync(std, p->base.std, E * H * A * 4, cudaMemcpyDeviceToDevice, st));
  if (z) CUDA_TRY(cudaMemcpyAsync(z, p->base.z, E * d.latent_dim * 4, cudaMemcpyDeviceToDevice, st));
  if (pi_actions && d.num_pi_trajs > 0)
    CUDA_TRY(cudaMemcpyAsync(pi_actions, p->base.pi_actions, E * H * d.num_pi_trajs * A * 4, cudaMemcpyDeviceToDevice, st));
  if (score) CUDA_TRY(cudaMemcpyAsync(score, p->base.score, E * d.num_elites * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int tdmpc2_estimate_value(tdmpc2_planner* p, const float* z, const float* actions, const int32_t* task,
                                     const float* noise_pi, const int32_t* qidx, float* value_out, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  if (!z || !actions || !noise_pi || !qidx || !value_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (d.task_dim > 0 && !task) return fail(TDMPC2_ERR_INVALID, "multi-task model needs task indices");
  PlanParams prm = p->base;
  prm.task = d.task_dim > 0 ? task : nullptr;
  prm.mode = MODE_VALUE;
  prm.z_rows = z; prm.actions_explicit = actions; prm.noise_pi = noise_pi; prm.qidx = qidx;
  prm.values_out = value_out;
  prm.ntiles = d.num_envs * p->tiles_per_env;
  return launch(p, prm, stream_);
}

extern "C" int tdmpc2_debug_layer(tdmpc2_planner* p, int layer, int mode, const float* x, int rows, float* y, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  if (layer < 0 || layer >= static_cast<int>(p->layers.size()) || rows < 1 || rows > kTileM || !x || !y || mode < 0 || mode > 2)
    return fail(TDMPC2_ERR_INVALID, "bad debug_layer arguments");
  if (mode != 0 && !p->layers[layer].has_ln) return fail(TDMPC2_ERR_INVALID, "layer %d has no LayerNorm", layer);
  if (p->layers[layer].Kpad > p->KpadX) return fail(TDMPC2_ERR_INVALID, "layer %d input wider than the X scratch", layer);
  PlanParams prm = p->base;
  prm.mode = MODE_LAYER;
  prm.dbg_layer = layer; prm.dbg_mode = mode; prm.dbg_rows = rows; prm.dbg_x = x; prm.dbg_y = y;
  prm.ntiles = 1;
  return launch(p, prm, stream_);
}

// ------------------------------------------------------------------------------------ target Q ensemble
extern "C" int tdmpc2_planner_target_q_bytes(const tdmpc2_planner* p, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (p->tq.lay.bytes == 0) return fail(TDMPC2_ERR_UNSUPPORTED, "the model's weight maps leave no room for the target Q maps (%d)", kMaxWMaps);
  *out = p->tq.lay.bytes;
  return 0;
}

extern "C" int tdmpc2_planner_bind_target_q(tdmpc2_planner* p, void* blob) {
  if (!p || !blob) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (!p->bound) return fail(TDMPC2_ERR_STATE, "tdmpc2_planner_bind must be called first");
  if (p->tq.lay.bytes == 0) return fail(TDMPC2_ERR_UNSUPPORTED, "the model's weight maps leave no room for the target Q maps");
  if (reinterpret_cast<uintptr_t>(blob) & 255) return fail(TDMPC2_ERR_INVALID, "buffers must be 256-byte aligned");
  TargetQ& tq = p->tq;
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return fail(TDMPC2_ERR_CUDA, "cuTensorMapEncodeTiled not available");
  int rc;
  if ((rc = bind_blob(enc, p->base.tmW, tq.layers, tq.lay, static_cast<uint8_t*>(blob)))) return rc;
  tq.blob = static_cast<uint8_t*>(blob);
  tq.packed = false;
  return 0;
}

extern "C" int tdmpc2_pack_target_q(tdmpc2_planner* p, const tdmpc2_linear* target_qs, void* stream_) {
  if (!p || !target_qs) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (!p->bound || !p->tq.blob) return fail(TDMPC2_ERR_STATE, "tdmpc2_planner_bind_target_q must be called first");
  TargetQ& tq = p->tq;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(tq.blob + tq.lay.off_absmax, 0, tq.layers.size() * sizeof(unsigned), st));
  int rc;
  for (int h = 0; h < p->d.num_q; ++h)
    for (int l = 0; l < 3; ++l)
      if ((rc = pack_layer(p, tq.layers, tq.lay, tq.blob, 3 * h + l, target_qs[l], h, st))) return rc;
  CUDA_TRY(cudaGetLastError());
  tq.packed = true;
  return 0;
}

// ------------------------------------------------------------------------------------ world-model methods (MODE_ROWS)
static int rows_ready(tdmpc2_planner* p, int rows) {
  if (!p) {
    int n = 0;
    const int rc = check_device(&n);
    return rc ? rc : fail(TDMPC2_ERR_INVALID, "null planner");
  }
  int rc = ready(p);
  if (rc) return rc;
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  return 0;
}

static PlanParams rows_params(tdmpc2_planner* p, int rop, int rows, const int32_t* task) {
  PlanParams prm = p->base;
  prm.mode = MODE_ROWS;
  prm.rop = rop;
  prm.rows = rows;
  prm.task = p->d.task_dim > 0 ? task : nullptr;
  prm.rows_q = reinterpret_cast<const LayerDev*>(p->packed + p->lay.off_table) + p->li_q;
  prm.ntiles = (rows + kTileM - 1) / kTileM;
  return prm;
}

static int need_task(tdmpc2_planner* p, const int32_t* task) {
  if (p->d.task_dim > 0 && !task) return fail(TDMPC2_ERR_INVALID, "multi-task model needs task indices");
  return 0;
}

extern "C" int tdmpc2_wm_encode(tdmpc2_planner* p, const float* obs, const int32_t* task, int rows, float* z_out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!obs || !z_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (p->num_enc == 0) return fail(TDMPC2_ERR_STATE, "this planner was created without a state encoder (num_enc_layers = 0)");
  PlanParams prm = rows_params(p, ROP_ENCODE, rows, task);
  prm.rows_in = obs; prm.rows_out = z_out;
  return launch(p, prm, stream_);
}

static int rows_za(tdmpc2_planner* p, int rop, const float* z, const float* a, const int32_t* task, int rows, float* out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!z || !a || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  PlanParams prm = rows_params(p, rop, rows, task);
  prm.rows_in = z; prm.rows_act = a; prm.rows_out = out;
  return launch(p, prm, stream_);
}
extern "C" int tdmpc2_wm_next(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, float* z_out, void* stream_) {
  return rows_za(p, ROP_NEXT, z, a, task, rows, z_out, stream_);
}
extern "C" int tdmpc2_wm_reward(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, float* logits_out,
                                void* stream_) {
  return rows_za(p, ROP_REWARD, z, a, task, rows, logits_out, stream_);
}

extern "C" int tdmpc2_wm_termination(tdmpc2_planner* p, const float* z, int rows, int sigmoid, float* out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc) return rc;
  if (!z || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (p->d.task_dim > 0 || !p->d.episodic)   // world_model.py:28,136: an episodic single-task model has the head
    return fail(TDMPC2_ERR_UNSUPPORTED, "termination needs an episodic single-task model");
  PlanParams prm = rows_params(p, ROP_TERM, rows, nullptr);
  prm.rows_in = z; prm.rows_out = out; prm.rows_flag = sigmoid ? 1 : 0;
  return launch(p, prm, stream_);
}

extern "C" int tdmpc2_wm_pi(tdmpc2_planner* p, const float* z, const int32_t* task, const float* eps, int rows, float* action_out,
                            float* mean_out, float* log_std_out, float* log_prob_out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!z || !eps || !action_out || !mean_out || !log_std_out || !log_prob_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  PlanParams prm = rows_params(p, ROP_PI, rows, task);
  prm.rows_in = z; prm.rows_eps = eps;
  prm.rows_out = action_out; prm.rows_out2 = mean_out; prm.rows_out3 = log_std_out; prm.rows_out4 = log_prob_out;
  return launch(p, prm, stream_);
}

static int select_q(tdmpc2_planner* p, int target, PlanParams& prm) {
  if (!target) return 0;
  if (!p->tq.blob || !p->tq.packed)
    return fail(TDMPC2_ERR_STATE, "target Q op before tdmpc2_planner_bind_target_q + tdmpc2_pack_target_q");
  prm.rows_q = reinterpret_cast<const LayerDev*>(p->tq.blob + p->tq.lay.off_table);
  return 0;
}

extern "C" int tdmpc2_wm_q(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, int target,
                           int return_type, const int32_t* qidx, float* out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!z || !a || !out || (return_type != TDMPC2_Q_ALL && !qidx)) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (return_type != TDMPC2_Q_ALL && return_type != TDMPC2_Q_MIN && return_type != TDMPC2_Q_AVG)
    return fail(TDMPC2_ERR_INVALID, "bad return_type %d", return_type);
  PlanParams prm = rows_params(p, return_type == TDMPC2_Q_ALL ? ROP_Q_ALL : ROP_Q_PAIR, rows, task);
  if ((rc = select_q(p, target, prm))) return rc;
  prm.rows_in = z; prm.rows_act = a; prm.rows_out = out; prm.qidx = qidx;
  prm.rows_flag = return_type == TDMPC2_Q_AVG ? 1 : 0;
  return launch(p, prm, stream_);
}

extern "C" int tdmpc2_td_target(tdmpc2_planner* p, const float* next_z, const float* reward, const float* terminated,
                                const int32_t* task, const float* eps, const int32_t* qidx, int rows, float* out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!next_z || !reward || !terminated || !eps || !qidx || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  PlanParams prm = rows_params(p, ROP_TD, rows, task);
  if ((rc = select_q(p, 1, prm))) return rc;
  prm.rows_in = next_z; prm.rows_eps = eps; prm.qidx = qidx;
  prm.rows_reward = reward; prm.rows_term = terminated; prm.rows_out = out;
  return launch(p, prm, stream_);
}

// ------------------------------------------------------------------------------------ agent.update_pi (ROP_PI_LOSS + grad_kernels.cuh)
static PiTape planner_tape(const tdmpc2_planner* p) {
  return pi_tape(p->d.mlp_dim, p->d.action_dim, pad_to(p->d.action_dim, 32), p->d.num_bins);
}

// Workspace of the backward, in floats: the per-row gradients of every layer it walks through, and the split-K
// partials of the dW reductions (nsplit row blocks, summed in order by pl_reduce).
struct PiWs {
  size_t dl, gq, gq2, dxq, dlog, gp, gp2, dyn, dy, hb, xb, dxe, part, floats;
  int nsplit;
};
static PiWs pi_ws(const tdmpc2_planner* p, int rows) {
  const tdmpc2_dims& d = p->d;
  const size_t R = rows, M = d.mlp_dim, nb = d.num_bins, TA = d.task_dim + d.action_dim, LT = d.latent_dim + d.task_dim;
  PiWs w;
  w.nsplit = std::max(1, std::min(8, rows / 256));
  size_t off = 0;
  auto take = [&](size_t n) { const size_t o = off; off += (n + 63) / 64 * 64; return o; };
  w.dl = take(2 * R * nb); w.gq = take(2 * R * M); w.gq2 = take(2 * R * M); w.dxq = take(2 * R * TA);
  w.dlog = take(R * 2 * d.action_dim); w.gp = take(R * M); w.gp2 = take(R * M); w.dyn = take(R * M); w.dy = take(R * M);
  w.hb = take(R * M); w.xb = take(R * LT); w.dxe = take(R * TA);
  w.part = take(static_cast<size_t>(w.nsplit) * M * std::max({M, LT, static_cast<size_t>(2 * d.action_dim)}));
  w.floats = off;
  return w;
}

extern "C" int tdmpc2_pi_loss_tape_bytes(const tdmpc2_planner* p, int rows, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  *out = static_cast<size_t>(rows) * planner_tape(p).pitch * 4;
  return 0;
}

extern "C" int tdmpc2_pi_loss_workspace_bytes(const tdmpc2_planner* p, int rows, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  *out = pi_ws(p, rows).floats * 4;
  return 0;
}

extern "C" int tdmpc2_pi_loss_forward(tdmpc2_planner* p, const float* z, const int32_t* task, const float* eps,
                                      const int32_t* qidx, const float* dropout_mask, int rows, float* tape, float* action_out,
                                      float* q_out, float* log_prob_out, void* stream_) {
  int rc = rows_ready(p, rows);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!z || !eps || !qidx || !tape || !action_out || !q_out || !log_prob_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  PlanParams prm = rows_params(p, ROP_PI_LOSS, rows, task);
  prm.rows_in = z; prm.rows_eps = eps; prm.qidx = qidx; prm.rows_flag = 1;       // 'avg' of the online pair
  prm.rows_tape = tape; prm.rows_act_out = action_out; prm.rows_out = q_out; prm.rows_out4 = log_prob_out;
  prm.rows_drop = dropout_mask; prm.tape_pitch = planner_tape(p).pitch;
  return launch(p, prm, stream_);
}

static int gemm(const GemmArgs& g, int batch, cudaStream_t st) {
  const dim3 grid((g.n + kGBN - 1) / kGBN, (g.m + kGBM - 1) / kGBM, batch * g.nsplit);
  gemm_f32<<<grid, 256, 0, st>>>(g);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int tdmpc2_pi_loss_backward(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* z,
                                       const int32_t* task, const float* eps, const int32_t* qidx, const float* dropout_mask,
                                       int T, int B, const float* scale, float entropy_coef, float rho,
                                       const tdmpc2_pi_grads* gr, void* workspace, void* stream_) {
  if (T < 1 || B < 1) {
    int n = 0;
    const int rc = check_device(&n);
    return rc ? rc : fail(TDMPC2_ERR_INVALID, "T and B must be >= 1");
  }
  if (static_cast<long long>(T) * B > 0x7fffffff) return fail(TDMPC2_ERR_INVALID, "T * B too large");
  const int R = T * B;
  int rc = rows_ready(p, R);
  if (rc || (rc = need_task(p, task))) return rc;
  if (!w || !tape || !z || !eps || !qidx || !scale || !gr || !workspace) return fail(TDMPC2_ERR_INVALID, "null argument");
  for (int i = 0; i < 3; ++i) {
    if (!w->pi[i].weight || !w->qs[i].weight || !gr->weight[i] || !gr->bias[i]) return fail(TDMPC2_ERR_INVALID, "null weight or gradient");
    if (i < 2 && (!w->pi[i].ln_weight || !w->qs[i].ln_weight || !w->qs[i].ln_bias || !w->pi[i].ln_bias || !gr->ln_weight[i] ||
                  !gr->ln_bias[i]))
      return fail(TDMPC2_ERR_INVALID, "null LayerNorm tensor or gradient");
  }
  const tdmpc2_dims& d = p->d;
  if (d.task_dim > 0 && !gr->task_emb) return fail(TDMPC2_ERR_INVALID, "multi-task model needs the task-embedding gradient");
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const PiTape tp = planner_tape(p);
  const PiWs L = pi_ws(p, R);
  float* ws = static_cast<float*>(workspace);
  const long long M = d.mlp_dim, nb = d.num_bins, A = d.action_dim, Tq = d.task_dim, TA = Tq + A, Lz = d.latent_dim;
  const long long LT = Lz + Tq, D = Lz + Tq + A;
  float *dl = ws + L.dl, *gq = ws + L.gq, *gq2 = ws + L.gq2, *dxq = ws + L.dxq, *dlog = ws + L.dlog, *gp = ws + L.gp,
        *gp2 = ws + L.gp2, *dyn = ws + L.dyn, *dy = ws + L.dy, *hb = ws + L.hb, *xb = ws + L.xb, *dxe = ws + L.dxe,
        *part = ws + L.part;
  const dim3 rows8((R + 7) / 8), rows8x2((R + 7) / 8, 2);
  const int* task_rows = d.task_dim > 0 ? task : nullptr;
  auto colsum = [&](const float* src, long long n, long long ld, float* dst) -> int {
    pl_colsum<<<static_cast<int>((n + 127) / 128), 128, 0, st>>>(src, R, static_cast<int>(n), ld, dst);
    CUDA_TRY(cudaGetLastError());
    return 0;
  };
  // dst += src^T x [rows, n] over the rows, in nsplit row blocks summed in order
  auto dweight = [&](const float* src, long long m, const float* x, long long n, long long ldx, float* dst) -> int {
    GemmArgs g{src, 1, m, 0, x, ldx, 1, 0, nullptr, part, n, 0, m * n, static_cast<int>(m), static_cast<int>(n), R, L.nsplit};
    int rc2 = gemm(g, 1, st);
    if (rc2) return rc2;
    pl_reduce<<<static_cast<int>((m * n + 255) / 256), 256, 0, st>>>(part, L.nsplit, m * n, m * n, dst);
    CUDA_TRY(cudaGetLastError());
    return 0;
  };
  LnBackArgs lb{};
  lb.tape = tape; lb.pitch = tp.pitch; lb.rows = R; lb.N = static_cast<int>(M); lb.ld = M;

  // ---- the two Q heads: two-hot inverse -> layer 2 -> LN/Mish 1 -> layer 1 -> LN/Mish/dropout 0 -> [emb | a] columns
  pl_q_head_back<<<rows8x2, 256, 0, st>>>(tape, tp.pitch, tp.q[0] + 2 * static_cast<int>(M), tp.q[1] + 2 * static_cast<int>(M), R,
                                          static_cast<int>(nb), p->base.bins, scale, B, T, rho, dl);
  CUDA_TRY(cudaGetLastError());
  if ((rc = gemm(GemmArgs{dl, nb, 1, R * nb, w->qs[2].weight, M, 1, nb * M, qidx, gq, M, R * M, 0,
                          R, static_cast<int>(M), static_cast<int>(nb), 1}, 2, st))) return rc;
  lb.off = tp.q[0] + static_cast<int>(M); lb.off_z = tp.q[1] - tp.q[0]; lb.g = gq; lb.out = gq; lb.g_z = R * M;
  lb.gamma = w->qs[1].ln_weight; lb.beta = w->qs[1].ln_bias; lb.hsel = qidx;
  pl_ln_back<<<rows8x2, 256, 0, st>>>(lb);
  CUDA_TRY(cudaGetLastError());
  if ((rc = gemm(GemmArgs{gq, M, 1, R * M, w->qs[1].weight, M, 1, M * M, qidx, gq2, M, R * M, 0,
                          R, static_cast<int>(M), static_cast<int>(M), 1}, 2, st))) return rc;
  lb.off = tp.q[0]; lb.g = gq2; lb.out = gq2; lb.gamma = w->qs[0].ln_weight; lb.beta = w->qs[0].ln_bias; lb.drop = dropout_mask;
  pl_ln_back<<<rows8x2, 256, 0, st>>>(lb);
  CUDA_TRY(cudaGetLastError());
  if ((rc = gemm(GemmArgs{gq2, M, 1, R * M, w->qs[0].weight + Lz, D, 1, M * D, qidx, dxq, TA, R * TA, 0,
                          R, static_cast<int>(TA), static_cast<int>(M), 1}, 2, st))) return rc;

  // ---- the tanh-Gaussian head, then pi layers 2 -> 0 with their parameter gradients
  PiHeadArgs ph{};
  ph.tape = tape; ph.pitch = tp.pitch; ph.off_h = tp.pih; ph.Apad = pad_to(d.action_dim, 32);
  ph.eps = eps; ph.task = task_rows; ph.masks = p->base.masks;
  ph.da_q = dxq; ph.da_ld = TA; ph.da_z = R * TA; ph.a_off = static_cast<int>(Tq);
  ph.log_std_min = d.log_std_min; ph.log_std_dif = d.log_std_dif; ph.entropy_coef = entropy_coef; ph.rho = rho; ph.scale = scale;
  ph.rows = R; ph.A = d.action_dim; ph.Bsz = B; ph.Tsz = T; ph.dlog = dlog;
  pl_pi_head_back<<<rows8, 256, 0, st>>>(ph);
  CUDA_TRY(cudaGetLastError());
  if ((rc = gemm(GemmArgs{dlog, 2 * A, 1, 0, w->pi[2].weight, M, 1, 0, nullptr, gp, M, 0, 0,
                          R, static_cast<int>(M), static_cast<int>(2 * A), 1}, 1, st))) return rc;
  lb.off = tp.pi1; lb.off_z = 0; lb.g = gp; lb.out = gp; lb.g_z = 0; lb.gamma = w->pi[1].ln_weight; lb.beta = w->pi[1].ln_bias;
  lb.hsel = nullptr; lb.drop = nullptr; lb.dyn = dyn; lb.dy = dy; lb.h = hb;
  pl_ln_back<<<rows8, 256, 0, st>>>(lb);                       // gp <- dL/dpre of pi.1; hb <- pi.1's activation
  CUDA_TRY(cudaGetLastError());
  if ((rc = colsum(dyn, M, M, gr->ln_weight[1])) || (rc = colsum(dy, M, M, gr->ln_bias[1]))) return rc;
  if ((rc = dweight(dlog, 2 * A, hb, M, M, gr->weight[2])) || (rc = colsum(dlog, 2 * A, 2 * A, gr->bias[2]))) return rc;
  if ((rc = gemm(GemmArgs{gp, M, 1, 0, w->pi[1].weight, M, 1, 0, nullptr, gp2, M, 0, 0,
                          R, static_cast<int>(M), static_cast<int>(M), 1}, 1, st))) return rc;
  lb.off = tp.pi0; lb.g = gp2; lb.out = gp2; lb.gamma = w->pi[0].ln_weight; lb.beta = w->pi[0].ln_bias;
  pl_ln_back<<<rows8, 256, 0, st>>>(lb);                       // gp2 <- dL/dpre of pi.0; hb <- pi.0's activation
  CUDA_TRY(cudaGetLastError());
  if ((rc = colsum(dyn, M, M, gr->ln_weight[0])) || (rc = colsum(dy, M, M, gr->ln_bias[0]))) return rc;
  if ((rc = dweight(gp, M, hb, M, M, gr->weight[1])) || (rc = colsum(gp, M, M, gr->bias[1]))) return rc;
  const float* x = z;
  if (Tq > 0) {
    pl_gather_x<<<static_cast<int>((R * LT + 255) / 256), 256, 0, st>>>(z, p->base.emb, task, R, static_cast<int>(Lz),
                                                                       static_cast<int>(Tq), xb);
    CUDA_TRY(cudaGetLastError());
    x = xb;
  }
  if ((rc = dweight(gp2, M, x, LT, LT, gr->weight[0])) || (rc = colsum(gp2, M, M, gr->bias[0]))) return rc;
  if (Tq > 0) {
    // the embedding enters pi.0's and both Q heads' layer-0 inputs: dL/demb of each row, scattered by task in row order
    if ((rc = gemm(GemmArgs{gp2, M, 1, 0, w->pi[0].weight + Lz, LT, 1, 0, nullptr, dxe, TA, 0, 0,
                            R, static_cast<int>(Tq), static_cast<int>(M), 1}, 1, st))) return rc;
    pl_emb_grad<<<static_cast<int>((d.num_tasks * Tq + 127) / 128), 128, 0, st>>>(dxe, dxq, dxq + R * TA, TA, task, R, d.num_tasks,
                                                                                static_cast<int>(Tq), gr->task_emb);
    CUDA_TRY(cudaGetLastError());
  }
  return 0;
}

// ------------------------------------------------------------------------------------ agent._update (row-op tapes + grad_kernels.cuh)
// The forward's tape (floats): one segment per row op, each [rows, pitch] of the pre-LayerNorm rows of its LayerNorm
// layers in layer order -- encoder [B, (n_enc - 1) enc_dim + L] (empty without a state encoder); dynamics [H B, 2 M + L] (step t's rows at t B);
// reward [H B, 2 M]; Q 'all' [H B, 2 M num_q] (head h's layers 0, 1 at (2 h + l) M, layer 0 after dropout);
// termination [H B, 2 M] (episodic).
struct WmTape {
  int p_enc, p_dyn, p_rew, p_q, p_term;
  size_t enc, dyn, rew, q, term, floats;
};
static WmTape wm_tape(const tdmpc2_planner* p, int H, int B) {
  const tdmpc2_dims& d = p->d;
  const size_t R = static_cast<size_t>(H) * B;
  WmTape t;
  t.p_enc = p->num_enc > 0 ? (p->num_enc - 1) * d.enc_dim + d.latent_dim : 0;
  t.p_dyn = 2 * d.mlp_dim + d.latent_dim; t.p_rew = 2 * d.mlp_dim; t.p_q = 2 * d.mlp_dim * d.num_q; t.p_term = 2 * d.mlp_dim;
  size_t off = 0;
  t.enc = take64(off, static_cast<size_t>(B) * t.p_enc);
  t.dyn = take64(off, R * t.p_dyn);
  t.rew = take64(off, R * t.p_rew);
  t.q = take64(off, R * t.p_q);
  t.term = d.episodic ? take64(off, R * t.p_term) : 0;
  t.floats = off;
  return t;
}

// Workspace of the backward (floats; ints for the head index array).
struct WmWs {
  size_t dlr, dlq, dlt, gA, gB, dyn, dy, hb, dxr, dxq, dxt, dxd, xa, dz, dp2, dyn2, dy2, dp1, dyn1, dy1, h1, dp0, dyn0, dy0,
      h0, ea, eb, edyn, edy, eh, ex, exe, zero, part, iota, floats;
  int nsplit;
};
static WmWs wm_ws(const tdmpc2_planner* p, int H, int B) {
  const tdmpc2_dims& d = p->d;
  const size_t R = static_cast<size_t>(H) * B, M = d.mlp_dim, L = d.latent_dim, T = d.task_dim, nb = d.num_bins, nq = d.num_q;
  const size_t LT = L + T, D = L + T + d.action_dim;
  // the encoder's segments are empty without a state encoder (pixel models: the conv encoder has its own workspace)
  const bool enc = p->num_enc > 0;
  const size_t E = enc ? d.enc_dim : 0, EL = enc ? std::max(E, L) : 0, OT = enc ? d.obs_dim + T : 0, BE = enc ? B : 0;
  WmWs w;
  w.nsplit = std::max(1, std::min(8, static_cast<int>(R / 256)));
  size_t off = 0;
  w.dlr = take64(off, R * nb); w.dlq = take64(off, nq * R * nb); w.dlt = take64(off, R);
  w.gA = take64(off, nq * R * M); w.gB = take64(off, nq * R * M); w.dyn = take64(off, nq * R * M); w.dy = take64(off, nq * R * M);
  w.hb = take64(off, nq * R * M);
  w.dxr = take64(off, R * LT); w.dxq = take64(off, nq * R * LT); w.dxt = take64(off, R * L); w.dxd = take64(off, R * LT);
  w.xa = take64(off, R * D); w.dz = take64(off, B * L);
  w.dp2 = take64(off, R * L); w.dyn2 = take64(off, R * L); w.dy2 = take64(off, R * L);
  w.dp1 = take64(off, R * M); w.dyn1 = take64(off, R * M); w.dy1 = take64(off, R * M); w.h1 = take64(off, R * M);
  w.dp0 = take64(off, R * M); w.dyn0 = take64(off, R * M); w.dy0 = take64(off, R * M); w.h0 = take64(off, R * M);
  w.ea = take64(off, B * EL); w.eb = take64(off, B * EL); w.edyn = take64(off, B * EL); w.edy = take64(off, B * EL);
  w.eh = take64(off, B * EL); w.ex = take64(off, B * OT); w.exe = take64(off, BE * LT);
  w.zero = take64(off, R * LT);
  w.part = take64(off, static_cast<size_t>(w.nsplit) * std::max({M, L, E, nb}) * std::max({M, D, E, OT}));
  w.iota = take64(off, nq);
  w.floats = off;
  return w;
}

static int wm_dims_ok(const tdmpc2_planner* p, int H, int B) {
  if (H < 1 || B < 1) return fail(TDMPC2_ERR_INVALID, "H and B must be >= 1");
  if (static_cast<long long>(H + 1) * B > 0x7fffffff) return fail(TDMPC2_ERR_INVALID, "H * B too large");
  return 0;
}
static int wm_needs_encoder(const tdmpc2_planner* p) {
  if (p->num_enc == 0)
    return fail(TDMPC2_ERR_UNSUPPORTED, "this planner has no state encoder (pixel model): use tdmpc2_wm_loss_forward_latent / "
                                        "tdmpc2_wm_loss_backward_latent with tdmpc2_pixel_encode_taped / tdmpc2_pixel_encode_backward");
  return 0;
}

extern "C" int tdmpc2_wm_loss_tape_bytes(const tdmpc2_planner* p, int H, int B, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  int rc = wm_dims_ok(p, H, B);
  if (rc) return rc;
  *out = wm_tape(p, H, B).floats * 4;
  return 0;
}

extern "C" int tdmpc2_wm_loss_workspace_bytes(const tdmpc2_planner* p, int H, int B, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  int rc = wm_dims_ok(p, H, B);
  if (rc) return rc;
  *out = wm_ws(p, H, B).floats * 4;
  return 0;
}

// latent: zs[0] is the caller's (the pixel encoder wrote it), and the ENCODE launch is skipped
static int wm_forward_impl(tdmpc2_planner* p, bool latent, const float* obs0, const float* action, const int32_t* task,
                           const float* dropout_mask, int H, int B, float* zs, float* q_logits, float* reward_logits,
                           float* term_logits, float* tape, void* stream_) {
  int rc = rows_ready(p, B);
  if (rc || (rc = wm_dims_ok(p, H, B)) || (!latent && (rc = wm_needs_encoder(p))) || (rc = need_task(p, task))) return rc;
  if ((!latent && !obs0) || !action || !zs || !q_logits || !reward_logits || !tape) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (p->d.episodic && !term_logits) return fail(TDMPC2_ERR_INVALID, "episodic model needs term_logits");
  const tdmpc2_dims& d = p->d;
  const int R = H * B;
  const size_t L = d.latent_dim, A = d.action_dim;
  const WmTape tp = wm_tape(p, H, B);
  PlanParams prm;
  if (!latent) {
    prm = rows_params(p, ROP_ENCODE, B, task);
    prm.rows_in = obs0; prm.rows_out = zs; prm.rows_tape = tape + tp.enc; prm.tape_pitch = tp.p_enc;
    if ((rc = launch(p, prm, stream_))) return rc;
  }
  for (int t = 0; t < H; ++t) {
    const size_t r0 = static_cast<size_t>(t) * B;
    prm = rows_params(p, ROP_NEXT, B, task ? task + r0 : nullptr);
    prm.rows_in = zs + r0 * L; prm.rows_act = action + r0 * A; prm.rows_out = zs + (r0 + B) * L;
    prm.rows_tape = tape + tp.dyn + r0 * tp.p_dyn; prm.tape_pitch = tp.p_dyn;
    if ((rc = launch(p, prm, stream_))) return rc;
  }
  prm = rows_params(p, ROP_Q_ALL, R, task);
  prm.rows_in = zs; prm.rows_act = action; prm.rows_out = q_logits;
  prm.rows_tape = tape + tp.q; prm.tape_pitch = tp.p_q; prm.rows_drop = dropout_mask;
  if ((rc = launch(p, prm, stream_))) return rc;
  prm = rows_params(p, ROP_REWARD, R, task);
  prm.rows_in = zs; prm.rows_act = action; prm.rows_out = reward_logits; prm.rows_tape = tape + tp.rew; prm.tape_pitch = tp.p_rew;
  if ((rc = launch(p, prm, stream_))) return rc;
  if (d.episodic) {
    prm = rows_params(p, ROP_TERM, R, nullptr);
    prm.rows_in = zs + static_cast<size_t>(B) * L; prm.rows_out = term_logits; prm.rows_flag = 0;
    prm.rows_tape = tape + tp.term; prm.tape_pitch = tp.p_term;
    if ((rc = launch(p, prm, stream_))) return rc;
  }
  return 0;
}

extern "C" int tdmpc2_wm_loss_forward(tdmpc2_planner* p, const float* obs0, const float* action, const int32_t* task,
                                      const float* dropout_mask, int H, int B, float* zs, float* q_logits, float* reward_logits,
                                      float* term_logits, float* tape, void* stream_) {
  return wm_forward_impl(p, false, obs0, action, task, dropout_mask, H, B, zs, q_logits, reward_logits, term_logits, tape, stream_);
}

extern "C" int tdmpc2_wm_loss_forward_latent(tdmpc2_planner* p, const float* action, const int32_t* task,
                                             const float* dropout_mask, int H, int B, float* zs, float* q_logits,
                                             float* reward_logits, float* term_logits, float* tape, void* stream_) {
  return wm_forward_impl(p, true, nullptr, action, task, dropout_mask, H, B, zs, q_logits, reward_logits, term_logits, tape, stream_);
}

static bool lin_ok(const tdmpc2_linear& l, bool ln) { return l.weight && l.bias && (!ln || (l.ln_weight && l.ln_bias)); }
static bool grad_ok(const tdmpc2_linear_grad& g, bool ln) { return g.weight && g.bias && (!ln || (g.ln_weight && g.ln_bias)); }

// dz0 != nullptr (latent): step 4 (the state encoder) is skipped and dL/dz_0 [B, L] is copied to dz0 instead
static int wm_backward_impl(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* obs0,
                            const float* action, const int32_t* task, const float* dropout_mask, int H, int B,
                            const float* zs, const float* q_logits, const float* reward_logits, const float* term_logits,
                            const float* next_z, const float* reward, const float* td_target, const float* terminated,
                            const tdmpc2_wm_loss_coefs* cf, const tdmpc2_wm_grads* gr, float* dz0, void* workspace, void* stream_) {
  const bool latent = dz0 != nullptr;
  int rc = rows_ready(p, B);
  if (rc || (rc = wm_dims_ok(p, H, B)) || (!latent && (rc = wm_needs_encoder(p))) || (rc = need_task(p, task))) return rc;
  const tdmpc2_dims& d = p->d;
  if (!w || !tape || (!latent && !obs0) || !action || !zs || !q_logits || !reward_logits || !next_z || !reward || !td_target || !cf || !gr ||
      !workspace)
    return fail(TDMPC2_ERR_INVALID, "null argument");
  if (d.episodic && (!term_logits || !terminated)) return fail(TDMPC2_ERR_INVALID, "episodic model needs term_logits and terminated");
  if (!latent && (w->num_enc != p->num_enc || gr->num_enc != p->num_enc))
    return fail(TDMPC2_ERR_INVALID, "num_enc differs from the planner's");
  for (int i = 0; !latent && i < p->num_enc; ++i)
    if (!lin_ok(w->enc[i], true) || !grad_ok(gr->enc[i], true)) return fail(TDMPC2_ERR_INVALID, "null encoder tensor or gradient");
  for (int i = 0; i < 3; ++i) {
    if (!lin_ok(w->dynamics[i], true) || !lin_ok(w->reward[i], i < 2) || !lin_ok(w->qs[i], i < 2) || !grad_ok(gr->dynamics[i], true) ||
        !grad_ok(gr->reward[i], i < 2) || !grad_ok(gr->qs[i], i < 2))
      return fail(TDMPC2_ERR_INVALID, "null weight or gradient");
    if (d.episodic && (!lin_ok(w->termination[i], i < 2) || !grad_ok(gr->termination[i], i < 2)))
      return fail(TDMPC2_ERR_INVALID, "null termination weight or gradient");
  }
  if (d.task_dim > 0 && !gr->task_emb) return fail(TDMPC2_ERR_INVALID, "multi-task model needs the task-embedding gradient");
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const WmTape tp = wm_tape(p, H, B);
  const WmWs W = wm_ws(p, H, B);
  float* ws = static_cast<float*>(workspace);
  const int R = H * B, nq = d.num_q;
  const long long M = d.mlp_dim, nb = d.num_bins, A = d.action_dim, Tq = d.task_dim, Lz = d.latent_dim, E = d.enc_dim;
  const long long LT = Lz + Tq, D = Lz + Tq + A, OT = d.obs_dim + Tq;
  const float fH = static_cast<float>(H), fB = static_cast<float>(B);
  float* X = ws + W.xa;
  int* iota = reinterpret_cast<int*>(ws + W.iota);
  auto ok = [&]() -> int { CUDA_TRY(cudaGetLastError()); return 0; };
  auto colsum = [&](const float* src, int rows, long long n, long long ld, float* dst) -> int {
    pl_colsum<<<static_cast<int>((n + 127) / 128), 128, 0, st>>>(src, rows, static_cast<int>(n), ld, dst);
    return ok();
  };
  // dst [m, n] += src^T x over `rows` rows (src [rows, m], x [rows, n] with row pitch ldx), split-K partials summed in order
  auto dweight = [&](const float* src, long long m, const float* x, long long n, long long ldx, int rows, float* dst) -> int {
    GemmArgs g{src, 1, m, 0, x, ldx, 1, 0, nullptr, ws + W.part, n, 0, m * n, static_cast<int>(m), static_cast<int>(n), rows, W.nsplit};
    int rc2 = gemm(g, 1, st);
    if (rc2) return rc2;
    pl_reduce<<<static_cast<int>((m * n + 255) / 256), 256, 0, st>>>(ws + W.part, W.nsplit, m * n, m * n, dst);
    return ok();
  };
  // out [rows, n] = g [rows, k] W[:, :n] (W [k, ldw]), batched over `batch` heads (g, out strides; W by bsel)
  auto dinput = [&](const float* g, long long k, const float* Wt, long long ldw, long long w_z, const int* bsel, int batch,
                    long long n, float* out, long long ldo, long long o_z, int rows) -> int {
    return gemm(GemmArgs{g, k, 1, static_cast<long long>(rows) * k, Wt, ldw, 1, w_z, bsel, out, ldo, o_z, 0, rows,
                         static_cast<int>(n), static_cast<int>(k), 1}, batch, st);
  };
  // the three layers of a head MLP (NormedLinear 0, 1 and a plain Linear 2) from dL/dlogits dl [batch, R, nout]: parameter
  // gradients of every layer (layer 0's input x0 [R, K0], row pitch ld0) and dX [batch, R, nx] of layer 0's first nx
  // input columns (ld ldx)
  auto head_back = [&](const float* dl, long long nout, const tdmpc2_linear* lw, const tdmpc2_linear_grad* lg, int batch,
                       const float* tape_seg, int pitch, long long off_z, const float* drop, const float* x0, long long K0,
                       long long ld0, long long nx, float* dx, long long ldx) -> int {
    int rc2;
    float *gA = ws + W.gA, *gB = ws + W.gB, *dyn = ws + W.dyn, *dy = ws + W.dy, *hb = ws + W.hb;
    const long long RM = static_cast<long long>(R) * M;
    const int* hs = batch > 1 ? iota : nullptr;
    if ((rc2 = dinput(dl, nout, lw[2].weight, M, nout * M, hs, batch, M, gA, M, RM, R))) return rc2;
    LnBackArgs lb{};
    lb.tape = tape_seg; lb.pitch = pitch; lb.rows = R; lb.N = static_cast<int>(M); lb.ld = M; lb.off_z = off_z; lb.g_z = RM;
    lb.o_z = RM; lb.hsel = hs; lb.dyn = dyn; lb.dy = dy; lb.h = hb;
    lb.off = static_cast<int>(M); lb.g = gA; lb.out = gA; lb.gamma = lw[1].ln_weight; lb.beta = lw[1].ln_bias;
    pl_ln_back<<<dim3((R + 7) / 8, batch), 256, 0, st>>>(lb);
    if ((rc2 = ok())) return rc2;
    for (int h = 0; h < batch; ++h) {
      const long long o = h * RM;
      if ((rc2 = colsum(dyn + o, R, M, M, lg[1].ln_weight + h * M)) || (rc2 = colsum(dy + o, R, M, M, lg[1].ln_bias + h * M)) ||
          (rc2 = dweight(dl + h * R * nout, nout, hb + o, M, M, R, lg[2].weight + h * nout * M)) ||
          (rc2 = colsum(dl + h * R * nout, R, nout, nout, lg[2].bias + h * nout)))
        return rc2;
    }
    if ((rc2 = dinput(gA, M, lw[1].weight, M, M * M, hs, batch, M, gB, M, RM, R))) return rc2;
    lb.off = 0; lb.g = gB; lb.out = gB; lb.gamma = lw[0].ln_weight; lb.beta = lw[0].ln_bias; lb.drop = drop;
    pl_ln_back<<<dim3((R + 7) / 8, batch), 256, 0, st>>>(lb);
    if ((rc2 = ok())) return rc2;
    for (int h = 0; h < batch; ++h) {
      const long long o = h * RM;
      if ((rc2 = colsum(dyn + o, R, M, M, lg[0].ln_weight + h * M)) || (rc2 = colsum(dy + o, R, M, M, lg[0].ln_bias + h * M)) ||
          (rc2 = dweight(gA + o, M, hb + o, M, M, R, lg[1].weight + h * M * M)) || (rc2 = colsum(gA + o, R, M, M, lg[1].bias + h * M)) ||
          (rc2 = dweight(gB + o, M, x0, K0, ld0, R, lg[0].weight + h * M * K0)) || (rc2 = colsum(gB + o, R, M, M, lg[0].bias + h * M)))
        return rc2;
    }
    return dinput(gB, M, lw[0].weight, K0, M * K0, hs, batch, nx, dx, ldx, static_cast<long long>(R) * ldx, R);
  };

  pl_iota<<<1, 32 * ((nq + 31) / 32), 0, st>>>(iota, nq);
  if ((rc = ok())) return rc;
  // X = [zs[:H] | emb | action]: the layer-0 input of the dynamics, reward and Q heads (z columns first)
  pl_gather_xa<<<static_cast<int>((R * D + 255) / 256), 256, 0, st>>>(zs, p->base.emb, task, action, R, static_cast<int>(Lz),
                                                                     static_cast<int>(Tq), static_cast<int>(A), X);
  if ((rc = ok())) return rc;

  // ---- 1. the heads, all H B rows at once: Q (batched over heads), reward, termination
  pl_soft_ce_back<<<dim3((R + 7) / 8, nq), 256, 0, st>>>(q_logits, static_cast<long long>(R) * nb, R, static_cast<int>(nb), td_target,
                                                         cf->vmin, cf->vmax, cf->bin_size, cf->value / (fH * nq * fB), cf->rho, B,
                                                         ws + W.dlq);
  if ((rc = ok())) return rc;
  if ((rc = head_back(ws + W.dlq, nb, w->qs, gr->qs, nq, tape + tp.q, tp.p_q, 2 * M, dropout_mask, X, D, D, LT, ws + W.dxq, LT)))
    return rc;
  pl_soft_ce_back<<<dim3((R + 7) / 8, 1), 256, 0, st>>>(reward_logits, 0, R, static_cast<int>(nb), reward, cf->vmin, cf->vmax,
                                                        cf->bin_size, cf->reward / (fH * fB), cf->rho, B, ws + W.dlr);
  if ((rc = ok())) return rc;
  if ((rc = head_back(ws + W.dlr, nb, w->reward, gr->reward, 1, tape + tp.rew, tp.p_rew, 0, nullptr, X, D, D, LT, ws + W.dxr, LT)))
    return rc;
  if (d.episodic) {
    pl_bce_back<<<(R + 255) / 256, 256, 0, st>>>(term_logits, terminated, R, cf->termination / (fH * fB), ws + W.dlt);
    if ((rc = ok())) return rc;
    // termination reads [z_{t+1}] alone: its layer-0 input is zs[1:], a contiguous [R, L] block
    if ((rc = head_back(ws + W.dlt, 1, w->termination, gr->termination, 1, tape + tp.term, tp.p_term, 0, nullptr,
                        zs + static_cast<size_t>(B) * Lz, Lz, Lz, Lz, ws + W.dxt, Lz)))
      return rc;
  }

  // ---- 2. back through time: dz_t, then dynamics step t - 1 (layers 2 -> 0) to its [z | emb] input columns
  DzArgs za{};
  za.zs = zs; za.next_z = next_z; za.dxq = ws + W.dxq; za.q_z = static_cast<long long>(R) * LT; za.nq = nq; za.dxr = ws + W.dxr;
  za.dxd = ws + W.dxd; za.ld = LT; za.dxt = d.episodic ? ws + W.dxt : nullptr; za.ldt = Lz;
  za.cons = cf->consistency * 2.f / (fH * fB * static_cast<float>(Lz)); za.rho = cf->rho; za.H = H; za.Bsz = B;
  za.L = static_cast<int>(Lz); za.dz = ws + W.dz;
  const int dz_blocks = static_cast<int>((B * Lz + 255) / 256), b8 = (B + 7) / 8;
  for (int t = H; t >= 1; --t) {
    za.t = t;
    pl_dz_step<<<dz_blocks, 256, 0, st>>>(za);
    if ((rc = ok())) return rc;
    const size_t r0 = static_cast<size_t>(t - 1) * B;
    const float* tseg = tape + tp.dyn + r0 * tp.p_dyn;
    LnBackArgs lb{};
    lb.tape = tseg; lb.pitch = tp.p_dyn; lb.rows = B; lb.off = static_cast<int>(2 * M); lb.N = static_cast<int>(Lz); lb.ld = Lz;
    lb.g = ws + W.dz; lb.out = ws + W.dp2 + r0 * Lz; lb.gamma = w->dynamics[2].ln_weight; lb.beta = w->dynamics[2].ln_bias;
    lb.dyn = ws + W.dyn2 + r0 * Lz; lb.dy = ws + W.dy2 + r0 * Lz;
    pl_ln_simnorm_back<<<b8, 256, 0, st>>>(lb, d.simnorm_dim);
    if ((rc = ok())) return rc;
    if ((rc = dinput(ws + W.dp2 + r0 * Lz, Lz, w->dynamics[2].weight, M, 0, nullptr, 1, M, ws + W.dp1 + r0 * M, M, 0, B))) return rc;
    lb.off = static_cast<int>(M); lb.N = static_cast<int>(M); lb.ld = M; lb.g = lb.out = ws + W.dp1 + r0 * M;
    lb.gamma = w->dynamics[1].ln_weight; lb.beta = w->dynamics[1].ln_bias;
    lb.dyn = ws + W.dyn1 + r0 * M; lb.dy = ws + W.dy1 + r0 * M; lb.h = ws + W.h1 + r0 * M;
    pl_ln_back<<<b8, 256, 0, st>>>(lb);
    if ((rc = ok())) return rc;
    if ((rc = dinput(ws + W.dp1 + r0 * M, M, w->dynamics[1].weight, M, 0, nullptr, 1, M, ws + W.dp0 + r0 * M, M, 0, B))) return rc;
    lb.off = 0; lb.g = lb.out = ws + W.dp0 + r0 * M; lb.gamma = w->dynamics[0].ln_weight; lb.beta = w->dynamics[0].ln_bias;
    lb.dyn = ws + W.dyn0 + r0 * M; lb.dy = ws + W.dy0 + r0 * M; lb.h = ws + W.h0 + r0 * M;
    pl_ln_back<<<b8, 256, 0, st>>>(lb);
    if ((rc = ok())) return rc;
    if ((rc = dinput(ws + W.dp0 + r0 * M, M, w->dynamics[0].weight, D, 0, nullptr, 1, LT, ws + W.dxd + r0 * LT, LT, 0, B))) return rc;
  }
  za.t = 0;
  pl_dz_step<<<dz_blocks, 256, 0, st>>>(za);
  if ((rc = ok())) return rc;

  // ---- 3. the dynamics' parameter gradients: one reduction over all H B taped rows per layer
  const tdmpc2_linear_grad* gd = gr->dynamics;
  if ((rc = dweight(ws + W.dp2, Lz, ws + W.h1, M, M, R, gd[2].weight)) || (rc = colsum(ws + W.dp2, R, Lz, Lz, gd[2].bias)) ||
      (rc = colsum(ws + W.dyn2, R, Lz, Lz, gd[2].ln_weight)) || (rc = colsum(ws + W.dy2, R, Lz, Lz, gd[2].ln_bias)) ||
      (rc = dweight(ws + W.dp1, M, ws + W.h0, M, M, R, gd[1].weight)) || (rc = colsum(ws + W.dp1, R, M, M, gd[1].bias)) ||
      (rc = colsum(ws + W.dyn1, R, M, M, gd[1].ln_weight)) || (rc = colsum(ws + W.dy1, R, M, M, gd[1].ln_bias)) ||
      (rc = dweight(ws + W.dp0, M, X, D, D, R, gd[0].weight)) || (rc = colsum(ws + W.dp0, R, M, M, gd[0].bias)) ||
      (rc = colsum(ws + W.dyn0, R, M, M, gd[0].ln_weight)) || (rc = colsum(ws + W.dy0, R, M, M, gd[0].ln_bias)))
    return rc;

  if (latent) CUDA_TRY(cudaMemcpyAsync(dz0, ws + W.dz, static_cast<size_t>(B) * Lz * 4, cudaMemcpyDeviceToDevice, st));
  // ---- 4. dz_0 through the encoder: the SimNorm layer, then the Mish layers down to layer 0 (input [obs | emb])
  if (!latent) {
    const int ne = p->num_enc;
    float *cur = ws + W.ea, *nxt = ws + W.eb;
    LnBackArgs lb{};
    lb.tape = tape + tp.enc; lb.pitch = tp.p_enc; lb.rows = B; lb.off = static_cast<int>((ne - 1) * E); lb.N = static_cast<int>(Lz);
    lb.ld = Lz; lb.g = ws + W.dz; lb.out = cur; lb.gamma = w->enc[ne - 1].ln_weight; lb.beta = w->enc[ne - 1].ln_bias;
    lb.dyn = ws + W.edyn; lb.dy = ws + W.edy;
    pl_ln_simnorm_back<<<b8, 256, 0, st>>>(lb, d.simnorm_dim);
    if ((rc = ok())) return rc;
    if ((rc = colsum(ws + W.edyn, B, Lz, Lz, gr->enc[ne - 1].ln_weight)) || (rc = colsum(ws + W.edy, B, Lz, Lz, gr->enc[ne - 1].ln_bias)) ||
        (rc = colsum(cur, B, Lz, Lz, gr->enc[ne - 1].bias)))
      return rc;
    long long n_cur = Lz;
    for (int i = ne - 2; i >= 0; --i) {
      if ((rc = dinput(cur, n_cur, w->enc[i + 1].weight, E, 0, nullptr, 1, E, nxt, E, 0, B))) return rc;
      LnBackArgs le{};
      le.tape = tape + tp.enc; le.pitch = tp.p_enc; le.rows = B; le.off = static_cast<int>(i * E); le.N = static_cast<int>(E); le.ld = E;
      le.g = le.out = nxt; le.gamma = w->enc[i].ln_weight; le.beta = w->enc[i].ln_bias;
      le.dyn = ws + W.edyn; le.dy = ws + W.edy; le.h = ws + W.eh;
      pl_ln_back<<<b8, 256, 0, st>>>(le);
      if ((rc = ok())) return rc;
      if ((rc = dweight(cur, n_cur, ws + W.eh, E, E, B, gr->enc[i + 1].weight)) ||
          (rc = colsum(ws + W.edyn, B, E, E, gr->enc[i].ln_weight)) || (rc = colsum(ws + W.edy, B, E, E, gr->enc[i].ln_bias)) ||
          (rc = colsum(nxt, B, E, E, gr->enc[i].bias)))
        return rc;
      std::swap(cur, nxt);
      n_cur = E;
    }
    const float* xe = obs0;
    if (Tq > 0) {
      pl_gather_x<<<static_cast<int>((B * OT + 255) / 256), 256, 0, st>>>(obs0, p->base.emb, task, B, d.obs_dim, static_cast<int>(Tq),
                                                                         ws + W.ex);
      if ((rc = ok())) return rc;
      xe = ws + W.ex;
    }
    if ((rc = dweight(cur, n_cur, xe, OT, OT, B, gr->enc[0].weight))) return rc;
    if (Tq > 0 && (rc = dinput(cur, n_cur, w->enc[0].weight + d.obs_dim, OT, 0, nullptr, 1, Tq, ws + W.exe + Lz, LT, 0, B)))
      return rc;
  }
  {
    if (Tq > 0) {
      // ---- 5. the task embedding: encoder layer 0 (without the latent variant), dynamics layer 0, reward layer 0, each Q
      // head's layer 0, in order
      CUDA_TRY(cudaMemsetAsync(ws + W.zero, 0, static_cast<size_t>(R) * LT * 4, st));
      const float* z0 = ws + W.zero;
      const dim3 eg(static_cast<int>((d.num_tasks * Tq + 127) / 128));
      if (!latent) pl_emb_grad<<<eg, 128, 0, st>>>(ws + W.exe + Lz, z0, z0, LT, task, B, d.num_tasks, static_cast<int>(Tq), gr->task_emb);
      pl_emb_grad<<<eg, 128, 0, st>>>(ws + W.dxd + Lz, z0, z0, LT, task, R, d.num_tasks, static_cast<int>(Tq), gr->task_emb);
      pl_emb_grad<<<eg, 128, 0, st>>>(ws + W.dxr + Lz, z0, z0, LT, task, R, d.num_tasks, static_cast<int>(Tq), gr->task_emb);
      for (int h = 0; h < nq; ++h)
        pl_emb_grad<<<eg, 128, 0, st>>>(ws + W.dxq + h * static_cast<long long>(R) * LT + Lz, z0, z0, LT, task, R, d.num_tasks,
                                        static_cast<int>(Tq), gr->task_emb);
      if ((rc = ok())) return rc;
    }
  }
  return 0;
}

extern "C" int tdmpc2_wm_loss_backward(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* obs0,
                                       const float* action, const int32_t* task, const float* dropout_mask, int H, int B,
                                       const float* zs, const float* q_logits, const float* reward_logits, const float* term_logits,
                                       const float* next_z, const float* reward, const float* td_target, const float* terminated,
                                       const tdmpc2_wm_loss_coefs* cf, const tdmpc2_wm_grads* gr, void* workspace, void* stream_) {
  return wm_backward_impl(p, w, tape, obs0, action, task, dropout_mask, H, B, zs, q_logits, reward_logits, term_logits, next_z,
                          reward, td_target, terminated, cf, gr, nullptr, workspace, stream_);
}

extern "C" int tdmpc2_wm_loss_backward_latent(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* action,
                                              const int32_t* task, const float* dropout_mask, int H, int B, const float* zs,
                                              const float* q_logits, const float* reward_logits, const float* term_logits,
                                              const float* next_z, const float* reward, const float* td_target,
                                              const float* terminated, const tdmpc2_wm_loss_coefs* cf, const tdmpc2_wm_grads* gr,
                                              float* dz0, void* workspace, void* stream_) {
  if (!dz0) return fail(TDMPC2_ERR_INVALID, "null argument");
  return wm_backward_impl(p, w, tape, nullptr, action, task, dropout_mask, H, B, zs, q_logits, reward_logits, term_logits, next_z,
                          reward, td_target, terminated, cf, gr, dz0, workspace, stream_);
}
