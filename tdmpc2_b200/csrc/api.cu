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
#include "buffer_kernels.cuh"
#include "draw_kernels.cuh"

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
// the check after each launch of a backward chain: its error, or an earlier kernel's, as TDMPC2_ERR_CUDA
static int launch_ok() { CUDA_TRY(cudaGetLastError()); return 0; }

static unsigned env_uint(const char* name, unsigned dflt) {
  const char* v = getenv(name);
  return (v && *v) ? static_cast<unsigned>(strtoul(v, nullptr, 10)) : dflt;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
// a workspace / tape segment of n floats at `off`, the next one starting on a 64-float boundary
static size_t take64(size_t& off, size_t n) { const size_t o = off; off += (n + 63) / 64 * 64; return o; }
static inline int pad_to(int x, int a) { return (x + a - 1) / a * a; }

#include "model_file.cuh"

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
  // state encoder (pixel observations: tdmpc2_pixel_encode supplies the latent, tdmpc2_plan_prologue's z)
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
  if (!p || (engine != TDMPC2_ENGINE_TCGEN05 && engine != TDMPC2_ENGINE_SIMT))
    return fail(TDMPC2_ERR_INVALID, "bad engine: 0 (tensor cores) or 1 (SIMT)");
  p->engine = engine;
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
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(std::min(prm.ntiles, p->nslots)); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = kSmemBytes;
  cfg.stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, prm2));
  CUDA_TRY(cudaGetLastError());
  p->launches += 1;
  return 0;
}

static int ready(tdmpc2_planner* p) {
  if (!p) return fail(TDMPC2_ERR_INVALID, "null planner");
  if (!p->bound || !p->weights_ok) return fail(TDMPC2_ERR_STATE, "planner needs bind() and pack_weights() first");
  return 0;
}

// obs != nullptr: z = encode(obs, task) through the state encoder; z_in != nullptr: the latent is given (pixel models)
extern "C" int tdmpc2_plan_prologue(tdmpc2_planner* p, const float* obs, const float* z_in, const int32_t* task, const uint8_t* t0,
                                    const float* prev_mean, const float* noise_prior, void* stream_) {
  if (!obs == !z_in) return fail(TDMPC2_ERR_INVALID, "exactly one of obs and z must be non-NULL");
  int rc = ready(p);
  if (rc) return rc;
  const tdmpc2_dims& d = p->d;
  if (!t0 || !prev_mean) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (obs && p->num_enc == 0) return fail(TDMPC2_ERR_STATE, "this planner was created without a state encoder (num_enc_layers = 0): pass z, not obs");
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
  if (d.in_channels < 1 || d.num_channels < 8 || d.num_channels % 8 != 0 || d.simnorm_dim < 1 ||
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
extern "C" int tdmpc2_pixel_encode(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                                   const float* shift, const float* grid_base, int64_t rows, float* z_out, float* tape,
                                   void* stream_) {
  if (!e) {                        // an encoder exists only where a device does: report the missing device first
    int n = 0;
    const int rc = check_device(&n);
    return rc ? rc : fail(TDMPC2_ERR_INVALID, "null pixel encoder");
  }
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

// ---- the conv encoder's backward (pixel_grad_kernels.cuh): taped forward, then the chain from dL/dz to the conv grads
extern "C" int tdmpc2_pixel_encode_tape_bytes(const tdmpc2_pixel_encoder* e, int64_t rows, size_t* out) {
  if (!e || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (rows < 1) return fail(TDMPC2_ERR_INVALID, "rows must be >= 1");
  *out = static_cast<size_t>(rows) * pix_tape_floats(e->d.num_channels) * 4;
  return 0;
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
    if (const int rc = launch_ok()) return rc;
    pixg_reduce<<<blocks(static_cast<int64_t>(nc) * cols), kPgThreads, 0, st>>>(part, ns, nc, cols, grads->weight[l], grads->bias[l]);
    return launch_ok();
  };
  int rc;
  pixg_simnorm_back<<<blocks(rows * (L / e->d.simnorm_dim)), kPgThreads, 0, st>>>(z, dz, rows, L, e->d.simnorm_dim, dp4);
  if ((rc = launch_ok())) return rc;
  if ((rc = dw(3, pixg_dw<3, 1>, 9, dp4, kPixO4, tape + pix_tape_a3(nc), tp, nc, kPixO3))) return rc;
  pixg_dx<3, 1><<<blocks(rows * nc * kPixO3 * kPixO3), kPgThreads, 0, st>>>(dp4, nc, kPixO4, kPixO4, w->weight[3], tape + pix_tape_a3(nc),
                                                                            tp, nc, kPixO3, kPixO3, rows, dp3);
  if ((rc = launch_ok())) return rc;
  if ((rc = dw(2, pixg_dw<3, 2>, 9, dp3, kPixO3, tape + pix_tape_a2(nc), tp, nc, kPixO2))) return rc;
  pixg_dx<3, 2><<<blocks(rows * nc * kPixO2 * kPixO2), kPgThreads, 0, st>>>(dp3, nc, kPixO3, kPixO3, w->weight[2], tape + pix_tape_a2(nc),
                                                                            tp, nc, kPixO2, kPixO2, rows, dp2);
  if ((rc = launch_ok())) return rc;
  if ((rc = dw(1, pixg_dw<5, 2>, 25, dp2, kPixO2, tape, tp, nc, kPixO1))) return rc;
  pixg_dx<5, 2><<<blocks(rows * nc * kPixO1 * kPixO1), kPgThreads, 0, st>>>(dp2, nc, kPixO2, kPixO2, w->weight[1], tape, tp, nc, kPixO1,
                                                                            kPixO1, rows, dp1);
  if ((rc = launch_ok())) return rc;
  pixg_stage<<<blocks(rows * pix_stage_floats(C)), kPgThreads, 0, st>>>(frames, shift, grid_base, rows, C, img);
  if ((rc = launch_ok())) return rc;
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

// The small draws of one plan (draw_kernels.cuh), every kind in one launch.
extern "C" int tdmpc2_plan_draws(tdmpc2_planner* p, const uint64_t* rng_state, int eval_mode, float* noise_prior, int32_t* qidx,
                                 float* expo, float* noise_final, float* shift, void* stream_) {
  if (!p) return fail(TDMPC2_ERR_INVALID, "null planner");
  const tdmpc2_dims& d = p->d;
  if (!rng_state || !qidx || !expo || (d.num_pi_trajs > 0 && !noise_prior) || (!eval_mode && !noise_final))
    return fail(TDMPC2_ERR_INVALID, "null argument");
  const long long E = d.num_envs, H = d.horizon, A = d.action_dim;
  DrawParams P{};
  P.state = reinterpret_cast<const unsigned long long*>(rng_state);
  P.prior = d.num_pi_trajs > 0 ? noise_prior : nullptr;
  P.n_prior = E * H * d.num_pi_trajs * A;
  P.qidx = qidx;
  P.q_rows = static_cast<long long>(d.iterations) * E;
  P.num_q = d.num_q;
  P.expo = expo;
  P.n_expo = E * d.num_elites;
  P.final_ = eval_mode ? nullptr : noise_final;
  P.n_final = E * A;
  P.shift = shift;
  P.n_shift = E * 2;
  const long long work = std::max({(P.n_prior + 3) / 4, P.q_rows, (P.n_expo + 3) / 4, (P.n_final + 3) / 4, (P.n_shift + 3) / 4});
  const unsigned blocks = static_cast<unsigned>(std::max<long long>(1, std::min<long long>((work + 255) / 256, 1024)));
  plan_draws_kernel<<<dim3(blocks, kDrawKinds), 256, 0, static_cast<cudaStream_t>(stream_)>>>(P);
  CUDA_TRY(cudaGetLastError());
  p->launches += 1;
  return 0;
}

// tdmpc2_act's scratch: the draws and, for pixel models, the encoded latent
struct ActScratch {
  size_t prior, qidx, expo, final_, shift, z, bytes;
};
static ActScratch act_scratch(const tdmpc2_dims& d, bool pixel) {
  const size_t E = d.num_envs, H = d.horizon, A = d.action_dim;
  ActScratch s{};
  size_t off = 0;
  auto take = [&](size_t n) { const size_t o = off; off = align_up(off + n, 256); return o; };
  s.prior = take(E * H * std::max(d.num_pi_trajs, 1) * A * 4);
  s.qidx = take(static_cast<size_t>(d.iterations) * E * 2 * 4);
  s.expo = take(E * d.num_elites * 4);
  s.final_ = take(E * A * 4);
  s.shift = take(E * 2 * 4);
  s.z = pixel ? take(E * d.latent_dim * 4) : 0;
  s.bytes = off;
  return s;
}

extern "C" int tdmpc2_act_scratch_bytes(const tdmpc2_planner* p, const tdmpc2_pixel_encoder* e, size_t* out) {
  if (!p || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  *out = act_scratch(p->d, e != nullptr).bytes;
  return 0;
}

extern "C" int tdmpc2_act(tdmpc2_planner* p, tdmpc2_pixel_encoder* e, void* enc_workspace, const tdmpc2_conv_weights* conv,
                          const tdmpc2_act_args* a, void* scratch, void* stream_) {
  int rc = ready(p);
  if (rc) return rc;
  if (!a || !scratch || !a->t0 || !a->rng_state || !a->prev_mean || !a->action_out) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(TDMPC2_ERR_INVALID, "scratch must be 256-byte aligned");
  if (p->engine == TDMPC2_ENGINE_SIMT) return fail(TDMPC2_ERR_UNSUPPORTED, "in-kernel noise needs a tensor-core engine");
  const tdmpc2_dims& d = p->d;
  const bool pixel = p->num_enc == 0;
  if (pixel) {
    if (!e || !enc_workspace || !conv || !a->frames || !a->grid_base)
      return fail(TDMPC2_ERR_INVALID, "a planner without a state encoder acts on frames: e, enc_workspace, conv, frames and grid_base are needed");
    if (16 * e->d.num_channels != d.latent_dim) return fail(TDMPC2_ERR_INVALID, "the pixel encoder's latent is not the planner's latent_dim");
  } else if (e || !a->obs) {
    return fail(TDMPC2_ERR_INVALID, "a state model acts on obs, with no pixel encoder");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  unsigned long long* state = reinterpret_cast<unsigned long long*>(a->rng_state);
  rng_advance_kernel<<<1, 1, 0, st>>>(state);
  CUDA_TRY(cudaGetLastError());
  p->launches += 1;
  const ActScratch s = act_scratch(d, pixel);
  unsigned char* base = static_cast<unsigned char*>(scratch);
  float* prior = d.num_pi_trajs > 0 ? reinterpret_cast<float*>(base + s.prior) : nullptr;
  int32_t* qidx = reinterpret_cast<int32_t*>(base + s.qidx);
  float* expo = reinterpret_cast<float*>(base + s.expo);
  float* fin = a->eval_mode ? nullptr : reinterpret_cast<float*>(base + s.final_);
  float* shift = pixel ? reinterpret_cast<float*>(base + s.shift) : nullptr;
  if ((rc = tdmpc2_plan_draws(p, a->rng_state, a->eval_mode, prior, qidx, expo, fin, shift, stream_))) return rc;
  float* z = nullptr;
  if (pixel) {
    z = reinterpret_cast<float*>(base + s.z);
    if ((rc = tdmpc2_pixel_encode(e, enc_workspace, conv, a->frames, shift, a->grid_base, d.num_envs, z, nullptr, stream_))) return rc;
    p->launches += 1;
  }
  if ((rc = tdmpc2_plan_prologue(p, pixel ? nullptr : a->obs, z, a->task, a->t0, a->prev_mean, prior, stream_))) return rc;
  for (int it = 0; it < d.iterations; ++it)
    if ((rc = tdmpc2_plan_iter_rng(p, a->rng_state, it, qidx + static_cast<size_t>(it) * d.num_envs * 2, nullptr, nullptr, stream_)))
      return rc;
  return tdmpc2_plan_epilogue(p, expo, fin, a->action_out, a->prev_mean, nullptr, stream_);
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

// ------------------------------------------------------------------------------------ backward chains (grad_kernels.cuh)
// The number of row blocks a dW reduction over `rows` rows is split into: at most 8, of at least 256 rows each.
static int dw_nsplit(size_t rows) { return std::max(1, std::min(8, static_cast<int>(rows / 256))); }

// The launch context of a backward chain: its stream, and the split-K partials [nsplit, m n] of dweight.  Each member
// issues its kernels in order, each followed by the launch check.
struct Bwd {
  cudaStream_t st;
  float* part;
  int nsplit;

  int gemm(const GemmArgs& g, int batch) const {
    gemm_f32<<<dim3((g.n + kGBN - 1) / kGBN, (g.m + kGBM - 1) / kGBM, batch * g.nsplit), 256, 0, st>>>(g);
    return launch_ok();
  }
  // out [rows, n] = g [rows, k] W[:, :n] (W [k, ldw]), batched over `batch` heads (g, out strides; W by bsel)
  int dinput(const float* g, long long k, const float* Wt, long long ldw, long long w_z, const int* bsel, int batch, long long n,
             float* out, long long ldo, long long o_z, int rows) const {
    return gemm(GemmArgs{g, k, 1, static_cast<long long>(rows) * k, Wt, ldw, 1, w_z, bsel, out, ldo, o_z, 0, rows,
                         static_cast<int>(n), static_cast<int>(k), 1}, batch);
  }
  // dst [m, n] += src^T x over `rows` rows (src [rows, m], x [rows, n] with row pitch ldx), split-K partials summed in order
  int dweight(const float* src, long long m, const float* x, long long n, long long ldx, int rows, float* dst) const {
    const int rc = gemm(GemmArgs{src, 1, m, 0, x, ldx, 1, 0, nullptr, part, n, 0, m * n, static_cast<int>(m), static_cast<int>(n),
                                 rows, nsplit}, 1);
    if (rc) return rc;
    pl_reduce<<<static_cast<int>((m * n + 255) / 256), 256, 0, st>>>(part, nsplit, m * n, m * n, dst);
    return launch_ok();
  }
  // dst [n] += the column sums of src [rows, n] (row pitch ld)
  int colsum(const float* src, int rows, long long n, long long ld, float* dst) const {
    pl_colsum<<<static_cast<int>((n + 127) / 128), 128, 0, st>>>(src, rows, static_cast<int>(n), ld, dst);
    return launch_ok();
  }
  // LayerNorm + Mish backward of a layer of width N, in place on g [batch, rows, N]: batch u reads row r's pre-LayerNorm
  // values at tape + r pitch + off + u off_z, and the LayerNorm parameters and dropout scale of head hsel[u] (head 0
  // without hsel).  dyn, dy and h (laid out like g) may be null.
  int ln_back(const float* tape, int pitch, long long off, int rows, long long N, const tdmpc2_linear& lw, float* g, float* dyn,
              float* dy, float* h, const float* drop = nullptr, int batch = 1, const int* hsel = nullptr, long long off_z = 0) const {
    LnBackArgs a{};
    a.tape = tape; a.pitch = pitch; a.off = static_cast<int>(off); a.off_z = off_z; a.g = g; a.out = g; a.ld = N; a.g_z = rows * N;
    a.o_z = a.g_z; a.gamma = lw.ln_weight; a.beta = lw.ln_bias; a.hsel = hsel; a.drop = drop; a.dyn = dyn; a.dy = dy; a.h = h;
    a.rows = rows; a.N = static_cast<int>(N);
    pl_ln_back<<<dim3((rows + 7) / 8, batch), 256, 0, st>>>(a);
    return launch_ok();
  }
  // LayerNorm + SimNorm (groups of V) backward of a layer of width N from dL/ds g [rows, N] to out; dyn and dy may be null
  int ln_simnorm_back(const float* tape, int pitch, long long off, int rows, long long N, const tdmpc2_linear& lw, const float* g,
                      float* out, float* dyn, float* dy, int V) const {
    LnBackArgs a{};
    a.tape = tape; a.pitch = pitch; a.off = static_cast<int>(off); a.g = g; a.out = out; a.ld = N; a.gamma = lw.ln_weight;
    a.beta = lw.ln_bias; a.dyn = dyn; a.dy = dy; a.rows = rows; a.N = static_cast<int>(N);
    pl_ln_simnorm_back<<<(rows + 7) / 8, 256, 0, st>>>(a, V);
    return launch_ok();
  }
};

// head_back's scratch, each [batch, rows, M]: dL/dpre of layers 1 and 0, and the dgamma / dbeta row terms and the
// activation of the layer below (written only with parameter gradients)
struct HeadWs {
  float *g1, *g0, *dyn, *dy, *h;
};

// The backward of `batch` head MLPs (NormedLinear 0 and 1, then a plain Linear 2) over `rows` rows, from dL/dlogits
// dl [batch, rows, nout].  Batch u is head hsel[u] (u without hsel) of the stacked weights lw; layer l's pre-LayerNorm
// values of its row r are at tape + r pitch + off0 + l M + u off_z; drop is layer 0's dropout scale, or null.  With lg,
// ADDS every layer's parameter gradients, reading layer 0's input x0 [rows, K0].  With dx, writes dL/dX [batch, rows, ldx]
// of layer 0's input columns col .. col + nx.
static int head_back(const Bwd& b, int rows, long long M, int batch, const int* hsel, const float* dl, long long nout,
                     const tdmpc2_linear* lw, const tdmpc2_linear_grad* lg, const float* tape, int pitch, int off0, long long off_z,
                     const float* drop, const float* x0, long long K0, long long col, long long nx, float* dx, long long ldx,
                     const HeadWs& s) {
  const long long RM = rows * M;
  float *dyn = lg ? s.dyn : nullptr, *dy = lg ? s.dy : nullptr, *h = lg ? s.h : nullptr;
  int rc;
  if ((rc = b.dinput(dl, nout, lw[2].weight, M, nout * M, hsel, batch, M, s.g1, M, RM, rows)) ||
      (rc = b.ln_back(tape, pitch, off0 + M, rows, M, lw[1], s.g1, dyn, dy, h, nullptr, batch, hsel, off_z)))
    return rc;
  for (int u = 0; lg && u < batch; ++u) {
    const long long o = u * RM;
    if ((rc = b.colsum(dyn + o, rows, M, M, lg[1].ln_weight + u * M)) || (rc = b.colsum(dy + o, rows, M, M, lg[1].ln_bias + u * M)) ||
        (rc = b.dweight(dl + u * rows * nout, nout, h + o, M, M, rows, lg[2].weight + u * nout * M)) ||
        (rc = b.colsum(dl + u * rows * nout, rows, nout, nout, lg[2].bias + u * nout)))
      return rc;
  }
  if ((rc = b.dinput(s.g1, M, lw[1].weight, M, M * M, hsel, batch, M, s.g0, M, RM, rows)) ||
      (rc = b.ln_back(tape, pitch, off0, rows, M, lw[0], s.g0, dyn, dy, h, drop, batch, hsel, off_z)))
    return rc;
  for (int u = 0; lg && u < batch; ++u) {
    const long long o = u * RM;
    if ((rc = b.colsum(dyn + o, rows, M, M, lg[0].ln_weight + u * M)) || (rc = b.colsum(dy + o, rows, M, M, lg[0].ln_bias + u * M)) ||
        (rc = b.dweight(s.g1 + o, M, h + o, M, M, rows, lg[1].weight + u * M * M)) ||
        (rc = b.colsum(s.g1 + o, rows, M, M, lg[1].bias + u * M)) ||
        (rc = b.dweight(s.g0 + o, M, x0, K0, K0, rows, lg[0].weight + u * M * K0)) ||
        (rc = b.colsum(s.g0 + o, rows, M, M, lg[0].bias + u * M)))
      return rc;
  }
  return dx ? b.dinput(s.g0, M, lw[0].weight + col, K0, M * K0, hsel, batch, nx, dx, ldx, rows * ldx, rows) : 0;
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
  w.nsplit = dw_nsplit(R);
  size_t off = 0;
  w.dl = take64(off, 2 * R * nb); w.gq = take64(off, 2 * R * M); w.gq2 = take64(off, 2 * R * M); w.dxq = take64(off, 2 * R * TA);
  w.dlog = take64(off, R * 2 * d.action_dim); w.gp = take64(off, R * M); w.gp2 = take64(off, R * M); w.dyn = take64(off, R * M);
  w.dy = take64(off, R * M); w.hb = take64(off, R * M); w.xb = take64(off, R * LT); w.dxe = take64(off, R * TA);
  w.part = take64(off, static_cast<size_t>(w.nsplit) * M * std::max({M, LT, static_cast<size_t>(2 * d.action_dim)}));
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
  const Bwd bw{st, ws + L.part, L.nsplit};
  const long long M = d.mlp_dim, nb = d.num_bins, A = d.action_dim, Tq = d.task_dim, TA = Tq + A, Lz = d.latent_dim;
  const long long LT = Lz + Tq, D = Lz + Tq + A;
  float *dl = ws + L.dl, *dxq = ws + L.dxq, *dlog = ws + L.dlog, *xb = ws + L.xb, *dxe = ws + L.dxe;

  // ---- the two Q heads: two-hot inverse, then dX of their [emb | a] input columns (no parameter gradients: detached)
  pl_q_head_back<<<dim3((R + 7) / 8, 2), 256, 0, st>>>(tape, tp.pitch, tp.q[0] + 2 * static_cast<int>(M), tp.q[1] + 2 * static_cast<int>(M),
                                                       R, static_cast<int>(nb), p->base.bins, scale, B, T, rho, dl);
  if ((rc = launch_ok()) ||
      (rc = head_back(bw, R, M, 2, qidx, dl, nb, w->qs, nullptr, tape, tp.pitch, tp.q[0], tp.q[1] - tp.q[0], dropout_mask, nullptr,
                      D, Lz, TA, dxq, TA, HeadWs{ws + L.gq, ws + L.gq2, nullptr, nullptr, nullptr})))
    return rc;

  // ---- the tanh-Gaussian head, then pi layers 2 -> 0 with their parameter gradients and, for multi-task models, dX of
  // pi.0's embedding columns
  PiHeadArgs ph{};
  ph.tape = tape; ph.pitch = tp.pitch; ph.off_h = tp.pih; ph.Apad = pad_to(d.action_dim, 32);
  ph.eps = eps; ph.task = d.task_dim > 0 ? task : nullptr; ph.masks = p->base.masks;
  ph.da_q = dxq; ph.da_ld = TA; ph.da_z = R * TA; ph.a_off = static_cast<int>(Tq);
  ph.log_std_min = d.log_std_min; ph.log_std_dif = d.log_std_dif; ph.entropy_coef = entropy_coef; ph.rho = rho; ph.scale = scale;
  ph.rows = R; ph.A = d.action_dim; ph.Bsz = B; ph.Tsz = T; ph.dlog = dlog;
  pl_pi_head_back<<<(R + 7) / 8, 256, 0, st>>>(ph);
  if ((rc = launch_ok())) return rc;
  const float* x = z;     // pi.0's input [z | emb]
  if (Tq > 0) {
    pl_gather_x<<<static_cast<int>((R * LT + 255) / 256), 256, 0, st>>>(z, p->base.emb, task, R, static_cast<int>(Lz),
                                                                       static_cast<int>(Tq), xb);
    if ((rc = launch_ok())) return rc;
    x = xb;
  }
  const tdmpc2_linear_grad pg[3] = {{gr->weight[0], gr->bias[0], gr->ln_weight[0], gr->ln_bias[0]},
                                    {gr->weight[1], gr->bias[1], gr->ln_weight[1], gr->ln_bias[1]},
                                    {gr->weight[2], gr->bias[2], nullptr, nullptr}};
  if ((rc = head_back(bw, R, M, 1, nullptr, dlog, 2 * A, w->pi, pg, tape, tp.pitch, tp.pi0, 0, nullptr, x, LT, Lz, Tq,
                      Tq > 0 ? dxe : nullptr, TA, HeadWs{ws + L.gp, ws + L.gp2, ws + L.dyn, ws + L.dy, ws + L.hb})))
    return rc;
  if (Tq > 0) {
    // the embedding enters pi.0's and both Q heads' layer-0 inputs: dL/demb of each row, scattered by task in row order
    pl_emb_grad<<<static_cast<int>((d.num_tasks * Tq + 127) / 128), 128, 0, st>>>(dxe, dxq, dxq + R * TA, TA, task, R, d.num_tasks,
                                                                                static_cast<int>(Tq), gr->task_emb);
    if ((rc = launch_ok())) return rc;
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
  w.nsplit = dw_nsplit(R);
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
    return fail(TDMPC2_ERR_UNSUPPORTED, "this planner has no state encoder (pixel model): pass obs0 = NULL, with zs[0] from a taped "
                                        "tdmpc2_pixel_encode and dz0 for tdmpc2_pixel_encode_backward");
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

// obs0 == nullptr (latent): zs[0] is the caller's (the pixel encoder wrote it), and the ENCODE launch is skipped
extern "C" int tdmpc2_wm_loss_forward(tdmpc2_planner* p, const float* obs0, const float* action, const int32_t* task,
                                      const float* dropout_mask, int H, int B, float* zs, float* q_logits, float* reward_logits,
                                      float* term_logits, float* tape, void* stream_) {
  const bool latent = obs0 == nullptr;
  int rc = rows_ready(p, B);
  if (rc || (rc = wm_dims_ok(p, H, B)) || (!latent && (rc = wm_needs_encoder(p))) || (rc = need_task(p, task))) return rc;
  if (!action || !zs || !q_logits || !reward_logits || !tape) return fail(TDMPC2_ERR_INVALID, "null argument");
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

static bool lin_ok(const tdmpc2_linear& l, bool ln) { return l.weight && l.bias && (!ln || (l.ln_weight && l.ln_bias)); }
static bool grad_ok(const tdmpc2_linear_grad& g, bool ln) { return g.weight && g.bias && (!ln || (g.ln_weight && g.ln_bias)); }

// obs0 == nullptr (latent): step 4 (the state encoder) is skipped and dL/dz_0 [B, L] is copied to dz0 instead
extern "C" int tdmpc2_wm_loss_backward(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* obs0,
                                       const float* action, const int32_t* task, const float* dropout_mask, int H, int B,
                                       const float* zs, const float* q_logits, const float* reward_logits, const float* term_logits,
                                       const float* next_z, const float* reward, const float* td_target, const float* terminated,
                                       const tdmpc2_wm_loss_coefs* cf, const tdmpc2_wm_grads* gr, float* dz0, void* workspace,
                                       void* stream_) {
  const bool latent = obs0 == nullptr;
  int rc = rows_ready(p, B);
  if (rc || (rc = wm_dims_ok(p, H, B)) || (!latent && (rc = wm_needs_encoder(p))) || (rc = need_task(p, task))) return rc;
  if (latent != (dz0 != nullptr)) return fail(TDMPC2_ERR_INVALID, "dz0 must be non-NULL exactly when obs0 is NULL");
  const tdmpc2_dims& d = p->d;
  if (!w || !tape || !action || !zs || !q_logits || !reward_logits || !next_z || !reward || !td_target || !cf || !gr ||
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
  const Bwd bw{st, ws + W.part, W.nsplit};
  const int R = H * B, nq = d.num_q;
  const long long M = d.mlp_dim, nb = d.num_bins, A = d.action_dim, Tq = d.task_dim, Lz = d.latent_dim, E = d.enc_dim;
  const long long LT = Lz + Tq, D = Lz + Tq + A, OT = d.obs_dim + Tq;
  const float fH = static_cast<float>(H), fB = static_cast<float>(B);
  float* X = ws + W.xa;
  int* iota = reinterpret_cast<int*>(ws + W.iota);
  const HeadWs hw{ws + W.gA, ws + W.gB, ws + W.dyn, ws + W.dy, ws + W.hb};

  pl_iota<<<1, 32 * ((nq + 31) / 32), 0, st>>>(iota, nq);
  if ((rc = launch_ok())) return rc;
  // X = [zs[:H] | emb | action]: the layer-0 input of the dynamics, reward and Q heads (z columns first)
  pl_gather_xa<<<static_cast<int>((R * D + 255) / 256), 256, 0, st>>>(zs, p->base.emb, task, action, R, static_cast<int>(Lz),
                                                                     static_cast<int>(Tq), static_cast<int>(A), X);
  if ((rc = launch_ok())) return rc;

  // ---- 1. the heads, all H B rows at once: Q (batched over heads), reward, termination
  pl_soft_ce_back<<<dim3((R + 7) / 8, nq), 256, 0, st>>>(q_logits, static_cast<long long>(R) * nb, R, static_cast<int>(nb), td_target,
                                                         cf->vmin, cf->vmax, cf->bin_size, cf->value / (fH * nq * fB), cf->rho, B,
                                                         ws + W.dlq);
  if ((rc = launch_ok()) ||
      (rc = head_back(bw, R, M, nq, iota, ws + W.dlq, nb, w->qs, gr->qs, tape + tp.q, tp.p_q, 0, 2 * M, dropout_mask, X, D, 0, LT,
                      ws + W.dxq, LT, hw)))
    return rc;
  pl_soft_ce_back<<<dim3((R + 7) / 8, 1), 256, 0, st>>>(reward_logits, 0, R, static_cast<int>(nb), reward, cf->vmin, cf->vmax,
                                                        cf->bin_size, cf->reward / (fH * fB), cf->rho, B, ws + W.dlr);
  if ((rc = launch_ok()) ||
      (rc = head_back(bw, R, M, 1, nullptr, ws + W.dlr, nb, w->reward, gr->reward, tape + tp.rew, tp.p_rew, 0, 0, nullptr, X, D, 0,
                      LT, ws + W.dxr, LT, hw)))
    return rc;
  if (d.episodic) {
    pl_bce_back<<<(R + 255) / 256, 256, 0, st>>>(term_logits, terminated, R, cf->termination / (fH * fB), ws + W.dlt);
    // termination reads [z_{t+1}] alone: its layer-0 input is zs[1:], a contiguous [R, L] block
    if ((rc = launch_ok()) ||
        (rc = head_back(bw, R, M, 1, nullptr, ws + W.dlt, 1, w->termination, gr->termination, tape + tp.term, tp.p_term, 0, 0,
                        nullptr, zs + static_cast<size_t>(B) * Lz, Lz, 0, Lz, ws + W.dxt, Lz, hw)))
      return rc;
  }

  // ---- 2. back through time: dz_t, then dynamics step t - 1 (layers 2 -> 0) to its [z | emb] input columns
  DzArgs za{};
  za.zs = zs; za.next_z = next_z; za.dxq = ws + W.dxq; za.q_z = static_cast<long long>(R) * LT; za.nq = nq; za.dxr = ws + W.dxr;
  za.dxd = ws + W.dxd; za.ld = LT; za.dxt = d.episodic ? ws + W.dxt : nullptr; za.ldt = Lz;
  za.cons = cf->consistency * 2.f / (fH * fB * static_cast<float>(Lz)); za.rho = cf->rho; za.H = H; za.Bsz = B;
  za.L = static_cast<int>(Lz); za.dz = ws + W.dz;
  const int dz_blocks = static_cast<int>((B * Lz + 255) / 256);
  for (int t = H; t >= 1; --t) {
    za.t = t;
    pl_dz_step<<<dz_blocks, 256, 0, st>>>(za);
    if ((rc = launch_ok())) return rc;
    const size_t r0 = static_cast<size_t>(t - 1) * B;
    const float* tseg = tape + tp.dyn + r0 * tp.p_dyn;
    float *dp2 = ws + W.dp2 + r0 * Lz, *dp1 = ws + W.dp1 + r0 * M, *dp0 = ws + W.dp0 + r0 * M;
    if ((rc = bw.ln_simnorm_back(tseg, tp.p_dyn, 2 * M, B, Lz, w->dynamics[2], ws + W.dz, dp2, ws + W.dyn2 + r0 * Lz,
                                 ws + W.dy2 + r0 * Lz, d.simnorm_dim)) ||
        (rc = bw.dinput(dp2, Lz, w->dynamics[2].weight, M, 0, nullptr, 1, M, dp1, M, 0, B)) ||
        (rc = bw.ln_back(tseg, tp.p_dyn, M, B, M, w->dynamics[1], dp1, ws + W.dyn1 + r0 * M, ws + W.dy1 + r0 * M, ws + W.h1 + r0 * M)) ||
        (rc = bw.dinput(dp1, M, w->dynamics[1].weight, M, 0, nullptr, 1, M, dp0, M, 0, B)) ||
        (rc = bw.ln_back(tseg, tp.p_dyn, 0, B, M, w->dynamics[0], dp0, ws + W.dyn0 + r0 * M, ws + W.dy0 + r0 * M, ws + W.h0 + r0 * M)) ||
        (rc = bw.dinput(dp0, M, w->dynamics[0].weight, D, 0, nullptr, 1, LT, ws + W.dxd + r0 * LT, LT, 0, B)))
      return rc;
  }
  za.t = 0;
  pl_dz_step<<<dz_blocks, 256, 0, st>>>(za);
  if ((rc = launch_ok())) return rc;

  // ---- 3. the dynamics' parameter gradients: one reduction over all H B taped rows per layer
  const tdmpc2_linear_grad* gd = gr->dynamics;
  if ((rc = bw.dweight(ws + W.dp2, Lz, ws + W.h1, M, M, R, gd[2].weight)) || (rc = bw.colsum(ws + W.dp2, R, Lz, Lz, gd[2].bias)) ||
      (rc = bw.colsum(ws + W.dyn2, R, Lz, Lz, gd[2].ln_weight)) || (rc = bw.colsum(ws + W.dy2, R, Lz, Lz, gd[2].ln_bias)) ||
      (rc = bw.dweight(ws + W.dp1, M, ws + W.h0, M, M, R, gd[1].weight)) || (rc = bw.colsum(ws + W.dp1, R, M, M, gd[1].bias)) ||
      (rc = bw.colsum(ws + W.dyn1, R, M, M, gd[1].ln_weight)) || (rc = bw.colsum(ws + W.dy1, R, M, M, gd[1].ln_bias)) ||
      (rc = bw.dweight(ws + W.dp0, M, X, D, D, R, gd[0].weight)) || (rc = bw.colsum(ws + W.dp0, R, M, M, gd[0].bias)) ||
      (rc = bw.colsum(ws + W.dyn0, R, M, M, gd[0].ln_weight)) || (rc = bw.colsum(ws + W.dy0, R, M, M, gd[0].ln_bias)))
    return rc;

  if (latent) CUDA_TRY(cudaMemcpyAsync(dz0, ws + W.dz, static_cast<size_t>(B) * Lz * 4, cudaMemcpyDeviceToDevice, st));
  // ---- 4. dz_0 through the encoder: the SimNorm layer, then the Mish layers down to layer 0 (input [obs | emb])
  if (!latent) {
    const int ne = p->num_enc;
    const float* te = tape + tp.enc;
    float *cur = ws + W.ea, *nxt = ws + W.eb;
    if ((rc = bw.ln_simnorm_back(te, tp.p_enc, (ne - 1) * E, B, Lz, w->enc[ne - 1], ws + W.dz, cur, ws + W.edyn, ws + W.edy,
                                 d.simnorm_dim)) ||
        (rc = bw.colsum(ws + W.edyn, B, Lz, Lz, gr->enc[ne - 1].ln_weight)) ||
        (rc = bw.colsum(ws + W.edy, B, Lz, Lz, gr->enc[ne - 1].ln_bias)) || (rc = bw.colsum(cur, B, Lz, Lz, gr->enc[ne - 1].bias)))
      return rc;
    long long n_cur = Lz;
    for (int i = ne - 2; i >= 0; --i) {
      if ((rc = bw.dinput(cur, n_cur, w->enc[i + 1].weight, E, 0, nullptr, 1, E, nxt, E, 0, B)) ||
          (rc = bw.ln_back(te, tp.p_enc, i * E, B, E, w->enc[i], nxt, ws + W.edyn, ws + W.edy, ws + W.eh)) ||
          (rc = bw.dweight(cur, n_cur, ws + W.eh, E, E, B, gr->enc[i + 1].weight)) ||
          (rc = bw.colsum(ws + W.edyn, B, E, E, gr->enc[i].ln_weight)) || (rc = bw.colsum(ws + W.edy, B, E, E, gr->enc[i].ln_bias)) ||
          (rc = bw.colsum(nxt, B, E, E, gr->enc[i].bias)))
        return rc;
      std::swap(cur, nxt);
      n_cur = E;
    }
    const float* xe = obs0;
    if (Tq > 0) {
      pl_gather_x<<<static_cast<int>((B * OT + 255) / 256), 256, 0, st>>>(obs0, p->base.emb, task, B, d.obs_dim, static_cast<int>(Tq),
                                                                         ws + W.ex);
      if ((rc = launch_ok())) return rc;
      xe = ws + W.ex;
    }
    if ((rc = bw.dweight(cur, n_cur, xe, OT, OT, B, gr->enc[0].weight)) ||
        (Tq > 0 && (rc = bw.dinput(cur, n_cur, w->enc[0].weight + d.obs_dim, OT, 0, nullptr, 1, Tq, ws + W.exe + Lz, LT, 0, B))))
      return rc;
  }
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
    if ((rc = launch_ok())) return rc;
  }
  return 0;
}

// ------------------------------------------------------------------------------------ replay buffer: Buffer.sample
static int buffer_vec_bytes(int64_t row_bytes, const void* a, const void* b) {
  const uintptr_t m = static_cast<uintptr_t>(row_bytes) | reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b);
  for (int v = 16; v > 1; v /= 2)
    if ((m & (v - 1)) == 0) return v;
  return 1;
}

extern "C" int tdmpc2_buffer_sample(const tdmpc2_buffer_field* fields, int num_fields, int64_t capacity,
                                    const int64_t* traj_start, const int64_t* traj_len, int64_t num_traj,
                                    const int64_t* traj_idx, const float* u, int B, int H, void* stream_) {
  if (!fields || !traj_start || !traj_len || !traj_idx || !u) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (num_fields < 1 || num_fields > kBufMaxFields)
    return fail(TDMPC2_ERR_INVALID, "num_fields = %d outside [1, %d]", num_fields, kBufMaxFields);
  if (capacity < 1 || num_traj < 1 || B < 1 || H < 1)
    return fail(TDMPC2_ERR_INVALID, "capacity = %lld, num_traj = %lld, B = %d, H = %d must all be >= 1",
                static_cast<long long>(capacity), static_cast<long long>(num_traj), B, H);
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    return fail(TDMPC2_ERR_NO_DEVICE, "no CUDA device: the buffer's sampler has no CPU fallback");
  }
  CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0)
    return fail(TDMPC2_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, major, minor);
  BufParams prm{};
  prm.nf = num_fields;
  prm.B = B;
  prm.H = H;
  prm.capacity = capacity;
  prm.num_traj = num_traj;
  prm.traj_start = traj_start;
  prm.traj_len = traj_len;
  prm.traj_idx = traj_idx;
  prm.u = u;
  int64_t units = 0;
  for (int i = 0; i < num_fields; ++i) {
    const tdmpc2_buffer_field& in = fields[i];
    if (!in.out || in.row_bytes < 1 || in.first_step < 0 || in.steps < 1 || in.first_step + in.steps > H + 1)
      return fail(TDMPC2_ERR_INVALID, "field %d: out = %p, row_bytes = %lld, first_step = %d, steps = %d (H = %d)", i, in.out,
                  static_cast<long long>(in.row_bytes), in.first_step, in.steps, H);
    const void* src = in.storage;
    if (src && in.host) {
      void* d = nullptr;
      CUDA_TRY(cudaHostGetDevicePointer(&d, const_cast<void*>(src), 0));
      src = d;
    }
    BufField& f = prm.f[i];
    f.src = static_cast<const unsigned char*>(src);
    f.dst = static_cast<unsigned char*>(in.out);
    f.vec = buffer_vec_bytes(in.row_bytes, src, in.out);
    const int64_t vpr = in.row_bytes / f.vec;
    if (vpr > (int64_t(1) << 30)) return fail(TDMPC2_ERR_INVALID, "field %d: row_bytes = %lld is too large", i,
                                               static_cast<long long>(in.row_bytes));
    f.vpr = static_cast<int32_t>(vpr);
    f.segs = vpr >= kBufUnitVecs ? static_cast<int32_t>((vpr + kBufUnitVecs - 1) / kBufUnitVecs) : 1;
    f.rpu = vpr >= kBufUnitVecs ? 1 : static_cast<int32_t>(std::min<int64_t>(32, kBufUnitVecs / vpr));
    f.first_step = in.first_step;
    f.steps = in.steps;
    f.unit_begin = units;
    const int64_t rows = static_cast<int64_t>(in.steps) * B;
    if (rows * f.segs >= (int64_t(1) << 31)) return fail(TDMPC2_ERR_INVALID, "field %d: %lld rows of %lld bytes is too large", i,
                                                          static_cast<long long>(rows), static_cast<long long>(in.row_bytes));
    units += f.rpu == 1 ? rows * f.segs : (rows + f.rpu - 1) / f.rpu;
  }
  prm.units = units;
  const int64_t ctas = (units + kBufThreads / 32 - 1) / (kBufThreads / 32);
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(ctas, 1 << 30));
  buffer_sample_kernel<<<grid, kBufThreads, 0, static_cast<cudaStream_t>(stream_)>>>(prm);
  CUDA_TRY(cudaGetLastError());
  return 0;
}
