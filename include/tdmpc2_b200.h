/*
 * tdmpc2_b200.h -- C ABI of the H100-native TD-MPC2 planning hot path.
 *
 * The reference (nicklashansen/tdmpc2) has no FFI / plugin API: its planner is
 * the Python method TDMPC2._plan (tdmpc2/tdmpc2.py:138-206) calling
 * WorldModel.{encode,next,reward,pi,Q} (tdmpc2/common/world_model.py:103-216).
 * This header is the boundary a binding would target instead: plain pointers
 * and sizes, no torch types.  Each entry point names the reference code it
 * replaces.  INTEGRATION.md shows the ctypes stub (tdmpc2_b200/_cabi.py is it).
 *
 * Conventions
 *   - every function returns 0 on success or a negative tdmpc2_status; the
 *     message is available from tdmpc2_last_error() (thread-local);
 *   - all device memory is CALLER-OWNED (torch tensors in the Python host):
 *     contiguous, 256-byte aligned; the library never allocates device memory;
 *   - all work is enqueued on the caller's `stream` (a cudaStream_t passed as
 *     void*); no host synchronisation, except in create/bind/pack which are
 *     set-up calls;
 *   - fp32 tensors, int32 task / q-head indices, uint8 flags, int64 elite
 *     indices (torch.topk's dtype);
 *   - there is NO CPU fallback: every call fails with TDMPC2_ERR_NO_DEVICE
 *     unless the current device is sm_90 (H100).
 *
 * Batched semantics (new in this build): a leading environment axis E.  Each
 * environment is one independent reference _plan call (own obs, task, t0,
 * _prev_mean, noise); E == 1 is exactly the reference.
 */
#ifndef TDMPC2_B200_H_
#define TDMPC2_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TDMPC2_B200_ABI_VERSION 7   /* 2: tdmpc2_weights.termination, dims.episodic = 1 accepted; 3: tdmpc2_planner_set_l2_persist;
                                       4: tdmpc2_planner_set_passes (declared non-parity fast mode), set_kseg, iter_engine;
                                       5: pixel encoder (tdmpc2_pixel_*), tdmpc2_plan_prologue_latent, dims.num_enc_layers = 0;
                                       6: tdmpc2_plan_iter_rng (declared non-parity in-kernel noise), tdmpc2_debug_rng;
                                       7: world-model methods on a flat batch (tdmpc2_wm_*, tdmpc2_td_target), target Q blob;
                                          later, additive: tdmpc2_pixel_encode_rows (old callers and bindings unaffected);
                                          later, additive: agent.update_pi (tdmpc2_pi_loss_*, tdmpc2_pi_grads),
                                          agent._update (tdmpc2_wm_loss_*, tdmpc2_wm_grads);
                                          later, additive: agent._update of pixel models (tdmpc2_pixel_encode_taped,
                                          tdmpc2_pixel_encode_backward, tdmpc2_conv_grads, tdmpc2_wm_loss_*_latent) */
#define TDMPC2_MAX_ENC_LAYERS 8

typedef enum tdmpc2_status {
  TDMPC2_OK = 0,
  TDMPC2_ERR_INVALID = -1,     /* bad dims / null pointer / unsupported config */
  TDMPC2_ERR_NO_DEVICE = -2,   /* no CUDA device, or device is not sm_90      */
  TDMPC2_ERR_CUDA = -3,        /* a CUDA runtime / driver call failed          */
  TDMPC2_ERR_STATE = -4,       /* call order violated (e.g. plan before bind)  */
  TDMPC2_ERR_UNSUPPORTED = -5  /* config outside what the reference's planner itself accepts (multi-task episodic) */
} tdmpc2_status;

/* GEMM engine used by the fused MLP kernels. */
typedef enum tdmpc2_engine {
  TDMPC2_ENGINE_TCGEN05 = 0,   /* TMA + wgmma (3x fp16-split, fp32 register accumulate): the product path */
  TDMPC2_ENGINE_SIMT = 1,      /* CUDA-core fp32 FFMA over the same packed operands: bring-up / diagnostics  */
  /* Engines 2 - 4 (CTA pairs, ping-pong halves, weight prefetch) were designed around cta_group::2 MMAs, which sm_90a
     does not have.  They are accepted and run as engine 0 (tdmpc2_planner_iter_engine reports 0). */
  TDMPC2_ENGINE_TCGEN05_2SM = 2,
  TDMPC2_ENGINE_TCGEN05_PP = 3,
  TDMPC2_ENGINE_TCGEN05_2SM_PF = 4
} tdmpc2_engine;

/* Planner + model dimensions.  Mirrors the keys the reference reads from cfg:
 * planning block config.yaml:33-42, architecture config.yaml:54-64, MODEL_SIZE
 * common/__init__.py:1-24, env dims envs/__init__.py:76-82. */
typedef struct tdmpc2_dims {
  int32_t num_envs;        /* E  (this rank's shard)                                   */
  int32_t num_samples;     /* N  cfg.num_samples                                        */
  int32_t num_pi_trajs;    /* P  cfg.num_pi_trajs                                       */
  int32_t num_elites;      /* K  cfg.num_elites                                         */
  int32_t horizon;         /* H  cfg.horizon                                            */
  int32_t iterations;      /* I  effective loop count (after tdmpc2.py:34's += 2)       */
  int32_t obs_dim;         /* cfg.obs_shape['state'][0]                                 */
  int32_t action_dim;      /* A                                                          */
  int32_t latent_dim;      /* L                                                          */
  int32_t mlp_dim;         /* M                                                          */
  int32_t enc_dim;
  int32_t num_enc_layers;  /* cfg.num_enc_layers: encoder has max(n-1,1)+1 Linear layers */
  int32_t task_dim;        /* T, 0 for single-task                                       */
  int32_t num_tasks;       /* len(cfg.tasks); 1 for single-task                          */
  int32_t num_q;
  int32_t num_bins;        /* B (two-hot regression bins; must be > 1)                   */
  int32_t simnorm_dim;     /* 8                                                          */
  int32_t episodic;        /* cfg.episodic: 1 adds the termination head (single-task)    */
  float temperature;       /* cfg.temperature                                            */
  float min_std, max_std;
  float log_std_min, log_std_dif;   /* WorldModel buffers, world_model.py:34-35          */
} tdmpc2_dims;

/* One Linear (+ optional LayerNorm) of the reference state dict
 * (layers.NormedLinear, layers.py:94-111).  Device pointers, fp32, row-major
 * `weight[out, in]` exactly as nn.Linear stores it; ln_* NULL for plain Linear. */
typedef struct tdmpc2_linear {
  const float* weight;
  const float* bias;
  const float* ln_weight;
  const float* ln_bias;
} tdmpc2_linear;

/* Device pointers into WorldModel.state_dict() tensors (SURVEY.md section 8(b)). */
typedef struct tdmpc2_weights {
  int32_t num_enc;                              /* number of encoder Linear layers          */
  tdmpc2_linear enc[TDMPC2_MAX_ENC_LAYERS];     /* _encoder.state.{i}.*                     */
  tdmpc2_linear dynamics[3];                    /* _dynamics.{0,1,2}.*                      */
  tdmpc2_linear reward[3];                      /* _reward.{0,1,2}.*   (layer 2: no LN)     */
  tdmpc2_linear pi[3];                          /* _pi.{0,1,2}.*       (layer 2: no LN)     */
  tdmpc2_linear qs[3];                          /* _Qs.params.{0,1,2}.* leading [num_q] dim */
  const float* task_emb;                        /* _task_emb.weight [num_tasks, T] or NULL  */
  const float* action_masks;                    /* _action_masks [num_tasks, A] or NULL     */
  const float* discount_pow;                    /* [num_tasks, H+1]: gamma_task^t, computed by
                                                   the host the way tdmpc2.py:125-132 does  */
  const float* bins;                            /* torch.linspace(vmin, vmax, B), math.py:80 */
  tdmpc2_linear termination[3];                 /* _termination.{0,1,2}.* (layer 2: no LN, 1 output), read only
                                                   when dims.episodic; world_model.py:28,132-141            */
} tdmpc2_weights;

typedef struct tdmpc2_planner tdmpc2_planner;    /* opaque host-side context */

/* ---- set-up ------------------------------------------------------------- */
int tdmpc2_abi_version(void);
const char* tdmpc2_last_error(void);

/* Validates dims, lays out the packed-weight blob and the workspace.  Needs a
 * current sm_90 device (queries SM count).  No device memory is allocated. */
int tdmpc2_planner_create(const tdmpc2_dims* dims, tdmpc2_planner** out);
void tdmpc2_planner_destroy(tdmpc2_planner* p);
int tdmpc2_planner_packed_bytes(const tdmpc2_planner* p, size_t* out);
int tdmpc2_planner_workspace_bytes(const tdmpc2_planner* p, size_t* out);
/* Attach caller-owned device buffers (sizes from the two calls above), zero the
 * workspace and encode the TMA descriptors.  Synchronous. */
int tdmpc2_planner_bind(tdmpc2_planner* p, void* packed, void* workspace);
int tdmpc2_planner_set_engine(tdmpc2_planner* p, int engine);
/* The engine the CEM-iteration launches actually run: the requested one falls back (3 -> 2 -> 0) when the model or the
 * batch shape does not fit it.  -1 on a null planner. */
int tdmpc2_planner_iter_engine(const tdmpc2_planner* p);
/* enable != 0: every planning launch carries an access-policy window that keeps the per-CTA activation scratch in the
 * persisting part of L2 (sets the DEVICE-wide cudaLimitPersistingL2CacheSize, hence opt-in); 0 switches it off.
 * No reference counterpart (the reference's activations are ordinary torch tensors). */
int tdmpc2_planner_set_l2_persist(tdmpc2_planner* p, int enable);
/* Reduction-segment knobs (k_elems >= 0) of the wide layers and of the head layers.  The wgmma engine already adds the
 * partial sum of every 64-element K-chunk with round-to-nearest, so on this build they validate their argument and
 * change nothing.  No reference counterpart. */
int tdmpc2_planner_set_kseg(tdmpc2_planner* p, int k_elems);
int tdmpc2_planner_set_head_kseg(tdmpc2_planner* p, int k_elems);
/* Arithmetic of the tensor-core engine 0.  passes = 3 (default): every product is three fp16 MMAs over the hi / lo
 * operand planes -- the mode whose results match the reference's fp32 plan() (tdmpc2.py:138-206) within 1e-4.
 * passes = 1: DECLARED NON-PARITY fast mode -- hi planes only (one fp16 MMA per product, fp32 accumulate; ~1e-3
 * value error, elite sets differ from the reference's): for throughput studies, never the headline number.
 * Engine 1 (SIMT) ignores it. */
int tdmpc2_planner_set_passes(tdmpc2_planner* p, int passes);
/* Replaces: agent.load()/WorldModel.to(device) weight placement (tdmpc2.py:81-95).
 * Packs the state-dict tensors into the kernel layout: per Linear two fp16
 * planes (hi, lo) of weight * 2^k, K-major, zero-padded; applies the
 * nn.Embedding(max_norm=1) renormalisation (world_model.py:21). */
int tdmpc2_pack_weights(tdmpc2_planner* p, const tdmpc2_weights* w, void* stream);

/* ---- the hot path -------------------------------------------------------- */
/* Replaces tdmpc2.py:153-170: z = encode(obs, task); the P policy-prior
 * trajectories; mean/std initialisation incl. the warm start from _prev_mean.
 *   obs [E, obs_dim]; task [E] int32 or NULL (single-task); t0 [E] uint8;
 *   prev_mean [E, H, A]; noise_prior [E, H, P, A] (draw 1 of SURVEY 8(a)). */
int tdmpc2_plan_prologue(tdmpc2_planner* p, const float* obs, const int32_t* task,
                         const uint8_t* t0, const float* prev_mean,
                         const float* noise_prior, void* stream);
/* The same with the latent given: z [E, L] replaces encode(obs, task).  For models without a state encoder
 * (dims.num_enc_layers = 0; cfg.obs == 'rgb': z comes from tdmpc2_pixel_encode). */
int tdmpc2_plan_prologue_latent(tdmpc2_planner* p, const float* z, const int32_t* task,
                                const uint8_t* t0, const float* prev_mean,
                                const float* noise_prior, void* stream);

/* DECLARED NON-PARITY throughput mode of tdmpc2_plan_iter: the two large noise tensors (tdmpc2.py:176, world_model.py:156) are
 * generated inside the kernel -- Philox4x32-10 + Box-Muller under rng_state = {seed, plan counter} (device memory, uint64[2];
 * the caller bumps the counter once per plan()), stream 2 * iteration (+1 for the policy sample) -- instead of being drawn by
 * torch into HBM.  Not torch's stream: actions differ from the reference's for the same torch seed; never the headline number. */
int tdmpc2_plan_iter_rng(tdmpc2_planner* p, const uint64_t* rng_state, int iteration, const int32_t* qidx,
                         float* values_out, int64_t* elite_idx_out, void* stream);
/* Diagnostics: out[4 g + i] = normal i of group group0 + g of `stream` (what the kernels consume). */
int tdmpc2_debug_rng(const uint64_t* rng_state, uint32_t stream, uint64_t group0, int ngroups, float* out, void* stream_);

/* ---- pixel observations (cfg.obs == 'rgb') ------------------------------- */
/* Replaces WorldModel.encode for obs type 'rgb' (world_model.py:103-112 -> layers.conv, layers.py:136-150): ShiftAug
 * (layers.py:36-59; part of the nn.Sequential, hence applied at inference too), PixelPreprocess (:62-71), four
 * Conv2d (7/2, 5/2, 3/2, 3/1) with ReLU between them, Flatten, SimNorm.  64 x 64 frames; latent_dim = 16 * num_channels. */
typedef struct tdmpc2_pixel_dims {
  int32_t num_envs;        /* E                                                          */
  int32_t in_channels;     /* cfg.obs_shape['rgb'][0] (3 x frame stack)                  */
  int32_t num_channels;    /* cfg.num_channels (config.yaml:58), a multiple of 8         */
  int32_t simnorm_dim;     /* cfg.simnorm_dim                                            */
} tdmpc2_pixel_dims;
typedef struct tdmpc2_conv_weights {   /* device pointers into the state dict: _encoder.rgb.{2,4,6,8}.{weight,bias} */
  const float* weight[4];              /* [out, in, k, k] as nn.Conv2d stores them       */
  const float* bias[4];
} tdmpc2_conv_weights;
typedef struct tdmpc2_pixel_encoder tdmpc2_pixel_encoder;
int tdmpc2_pixel_encoder_create(const tdmpc2_pixel_dims* dims, tdmpc2_pixel_encoder** out);
void tdmpc2_pixel_encoder_destroy(tdmpc2_pixel_encoder* e);
int tdmpc2_pixel_encoder_workspace_bytes(const tdmpc2_pixel_encoder* e, size_t* out);
/*   frames [E, C, 64, 64] fp32 in 0..255; shift [E, 2] = the (x, y) values torch.randint(0, 7) draws in ShiftAug
 *   (layers.py:55), as floats; grid_base [64] = torch.linspace(-1 + 1/70, 1 - 1/70, 70)[:64] (layers.py:51);
 *   z_out [E, 16 * num_channels]; workspace: caller-owned, tdmpc2_pixel_encoder_workspace_bytes. */
int tdmpc2_pixel_encode(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                        const float* shift, const float* grid_base, float* z_out, void* stream);
/* The same encoder over any number of frames, e.g. WorldModel.encode(obs[1:]) of _update (tdmpc2.py:262) on a
 * [T, B, C, 64, 64] batch flattened by the caller: frames [rows, C, 64, 64], shift [rows, 2], z_out [rows, 16 * num_channels].
 * One launch, the same workspace as tdmpc2_pixel_encode (its size does not depend on rows), no allocation and no host
 * synchronisation (capturable in a CUDA graph).  z of a frame is bit-identical to tdmpc2_pixel_encode's for the same
 * frame and shift.  rows < 1 or a null pointer: TDMPC2_ERR_INVALID. */
int tdmpc2_pixel_encode_rows(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                             const float* shift, const float* grid_base, int64_t rows, float* z_out, void* stream);
/* Training (agent._update of pixel models, tdmpc2.py:266-309).  tdmpc2_pixel_encode_taped is tdmpc2_pixel_encode_rows that
 * also writes each frame's post-ReLU maps to `tape` ([rows] slots of tape_bytes / rows; z is bit-identical to the untaped
 * launch).  tdmpc2_pixel_encode_backward ADDS dL/dparameter of the four Conv2d layers to `grads`, like autograd
 * accumulates .grad, given dz = dL/dz [rows, 16 * num_channels], the forward's z and tape and its frames and shifts
 * (conv1's input is recomputed).  fp32 FFMA; reductions over frames in a fixed order (repeated calls give identical bits);
 * no allocation, no host synchronisation.  workspace: tdmpc2_pixel_backward_workspace_bytes(rows). */
typedef struct tdmpc2_conv_grads {   /* .grad of _encoder.rgb.{2,4,6,8}.{weight,bias} */
  float* weight[4];
  float* bias[4];
} tdmpc2_conv_grads;
int tdmpc2_pixel_encode_tape_bytes(const tdmpc2_pixel_encoder* e, int64_t rows, size_t* out);
int tdmpc2_pixel_encode_taped(tdmpc2_pixel_encoder* e, void* workspace, const tdmpc2_conv_weights* w, const float* frames,
                              const float* shift, const float* grid_base, int64_t rows, float* z_out, float* tape, void* stream);
int tdmpc2_pixel_backward_workspace_bytes(const tdmpc2_pixel_encoder* e, int64_t rows, size_t* out);
int tdmpc2_pixel_encode_backward(tdmpc2_pixel_encoder* e, const tdmpc2_conv_weights* w, const float* frames,
                                 const float* shift, const float* grid_base, int64_t rows, const float* tape, const float* z,
                                 const float* dz, const tdmpc2_conv_grads* grads, void* workspace, void* stream);

/* Replaces ONE pass of the loop tdmpc2.py:173-197 (sample, _estimate_value
 * :122-136, topk, MPPI weights, refit) for all E environments.
 *   noise_r  [E, H, N-P, A]  (tdmpc2.py:176)
 *   noise_pi [E, N, A]       (terminal pi(), world_model.py:156)
 *   qidx     [E, 2] int32    (randperm(num_q)[:2], world_model.py:212)
 * Optional outputs (NULL to skip): values [E, N] (after nan_to_num),
 * elite_idx [E, K] int64 sorted by value desc (ties: lower index first). */
int tdmpc2_plan_iter(tdmpc2_planner* p, const float* noise_r, const float* noise_pi,
                     const int32_t* qidx, float* values_out, int64_t* elite_idx_out,
                     void* stream);

/* Replaces tdmpc2.py:199-206: gumbel pick (math.py:86-94, `expo` [E, K] are the
 * exponential_() draws), optional exploration noise (`noise_final` [E, A], NULL
 * == eval_mode), clamp, and the _prev_mean update.
 *   action_out [E, A]; prev_mean_out [E, H, A]; pick_out [E] int32 or NULL. */
int tdmpc2_plan_epilogue(tdmpc2_planner* p, const float* expo, const float* noise_final,
                         float* action_out, float* prev_mean_out, int32_t* pick_out,
                         void* stream);

/* Current CEM state (after prologue / any iteration): mean, std [E, H, A];
 * z [E, L]; pi_actions [E, H, P, A]; score [E, K].  NULL to skip an output. */
int tdmpc2_plan_get_state(tdmpc2_planner* p, float* mean, float* std, float* z,
                          float* pi_actions, float* score, void* stream);

/* Replaces TDMPC2._estimate_value (tdmpc2.py:122-136) as a stand-alone call:
 *   z [E, N, L], actions [E, H, N, A], noise_pi [E, N, A], qidx [E, 2] -> value [E, N]
 * (no nan_to_num; E == 1 is the reference's signature). */
int tdmpc2_estimate_value(tdmpc2_planner* p, const float* z, const float* actions,
                          const int32_t* task, const float* noise_pi, const int32_t* qidx,
                          float* value_out, void* stream);

/* ---- world-model methods on a flat batch of rows ------------------------------
 * The training-side and analysis calls of the reference's WorldModel (world_model.py:103-216) and TDMPC2._td_target
 * (tdmpc2.py:242-257), each one launch of the fused kernel over `rows` independent rows (any count >= 1; a leading
 * [H, B] of the reference is flattened by the caller).  They share the planner's packed weights and scratch, and leave
 * its planning state untouched.  Every random number is an input (the reference draws them inside pi() and Q()).
 *   task: int32 [rows] or NULL (single-task); all fp32 row tensors are contiguous [rows, .]. */

/* The target Q ensemble (_target_Qs_params.*, world_model.py:41) lives in its own caller-owned blob, so that a planner
 * that never runs a target op keeps its memory.  bytes: size of that blob (TDMPC2_ERR_UNSUPPORTED when the model's
 * weight-map classes leave no room for the target's).  bind: attach it (256-byte aligned; again after
 * tdmpc2_planner_bind).  pack: target_qs[l] = _target_Qs_params.{l}.* with the leading [num_q] dim; call again after
 * every target update (soft_update_target_Q, world_model.py:76-80).  Ops with target weights fail with
 * TDMPC2_ERR_STATE until both ran. */
int tdmpc2_planner_target_q_bytes(const tdmpc2_planner* p, size_t* out);
int tdmpc2_planner_bind_target_q(tdmpc2_planner* p, void* blob);
int tdmpc2_pack_target_q(tdmpc2_planner* p, const tdmpc2_linear target_qs[3], void* stream);

/* Replaces WorldModel.encode (world_model.py:103-112), state observations: obs [rows, obs_dim] -> z_out [rows, L]. */
int tdmpc2_wm_encode(tdmpc2_planner* p, const float* obs, const int32_t* task, int rows, float* z_out, void* stream);
/* Replaces WorldModel.next (world_model.py:114-121): z [rows, L], a [rows, A] -> z_out [rows, L]. */
int tdmpc2_wm_next(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, float* z_out, void* stream);
/* Replaces WorldModel.reward (world_model.py:123-130): -> logits_out [rows, num_bins]. */
int tdmpc2_wm_reward(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, float* logits_out,
                     void* stream);
/* Replaces WorldModel.termination (world_model.py:132-141; episodic single-task models, else TDMPC2_ERR_UNSUPPORTED):
 * out [rows, 1] = sigmoid(logit) (sigmoid != 0) or the logit (unnormalized=True). */
int tdmpc2_wm_termination(tdmpc2_planner* p, const float* z, int rows, int sigmoid, float* out, void* stream);
/* Replaces WorldModel.pi (world_model.py:144-184) with eps [rows, A] = its randn_like draw: action_out, mean_out
 * (= tanh(mean), info["mean"]), log_std_out [rows, A]; log_prob_out [rows, 2] = (gaussian_logprob(eps, log_std),
 * sum of the squash terms log(relu(1 - action^2) + 1e-6)) (math.py:16-29): entropy = -(lp - sq); scaled_entropy =
 * entropy * lp * size / (lp - sq + 1e-8), size = A or the task's action-mask sum. */
int tdmpc2_wm_pi(tdmpc2_planner* p, const float* z, const int32_t* task, const float* eps, int rows, float* action_out,
                 float* mean_out, float* log_std_out, float* log_prob_out, void* stream);
/* Replaces WorldModel.Q (world_model.py:186-216).  target != 0: the target ensemble (else the online one; `detach`
 * reads the same weights).  TDMPC2_Q_ALL: out [num_q, rows, num_bins] logits, qidx unused; TDMPC2_Q_MIN / _AVG:
 * qidx [2] int32 (= randperm(num_q)[:2]), out [rows, 1] = min (NaN-propagating, like torch.min) or average of the
 * two heads' two_hot_inv values. */
typedef enum tdmpc2_q_return { TDMPC2_Q_ALL = 0, TDMPC2_Q_MIN = 1, TDMPC2_Q_AVG = 2 } tdmpc2_q_return;
int tdmpc2_wm_q(tdmpc2_planner* p, const float* z, const float* a, const int32_t* task, int rows, int target,
                int return_type, const int32_t* qidx, float* out, void* stream);
/* Replaces TDMPC2._td_target (tdmpc2.py:242-257) in one launch: action = pi(next_z) with eps [rows, A], then
 * out [rows, 1] = reward + discount[task] * (1 - terminated) * min(Q_target[qidx[0]], Q_target[qidx[1]]);
 * reward, terminated [rows, 1]. */
int tdmpc2_td_target(tdmpc2_planner* p, const float* next_z, const float* reward, const float* terminated,
                     const int32_t* task, const float* eps, const int32_t* qidx, int rows, float* out, void* stream);

/* ---- agent.update_pi (tdmpc2.py:208-239) ------------------------------------------------------------------------
 * The policy loss of a [T, B] batch of latents zs (rows = T B, row r = t B + b):
 *   action = pi(zs) with eps [rows, A]; q = Q(zs, action, 'avg') of the ONLINE heads qidx[0], qidx[1] (detached: the Q
 *   weights get no gradient, the action does); loss = mean_t rho^t mean_b -(entropy_coef scaled_entropy + q / scale).
 * forward: one launch of the fused row kernel.  It writes action_out [rows, A], q_out [rows, 1], log_prob_out [rows, 2]
 * (as tdmpc2_wm_pi's) and the caller-owned tape [tape_bytes] the backward reads.  dropout_mask: NULL (eval mode) or
 * [num_q, rows, mlp_dim] = the train-mode Dropout(cfg.dropout) scale mask / (1 - p) of Q layer 0 (layers.py:104-108),
 * head h's rows at h rows mlp_dim; applied to the pre-LayerNorm output.
 * backward: from the tape, the same eps / qidx / dropout_mask and task, the fp32 state-dict tensors w->pi, w->qs, and
 * scale [1] (device memory: RunningScale.value), ADDS dL/dparameter to grads (like autograd accumulates .grad):
 * _pi.{0,1,2}.weight / .bias, _pi.{0,1}.ln.weight / .ln.bias, and for multi-task models _task_emb.weight.grad (pi's and
 * both Q heads' layer-0 inputs).  Reductions over rows run in a fixed order: repeated calls give identical bits.
 * workspace: caller-owned, workspace_bytes(rows).  No allocation, no host synchronisation (capturable). */
typedef struct tdmpc2_pi_grads {
  float* weight[3];
  float* bias[3];
  float* ln_weight[2];
  float* ln_bias[2];
  float* task_emb;         /* [num_tasks, T]; NULL for single-task models */
} tdmpc2_pi_grads;
int tdmpc2_pi_loss_tape_bytes(const tdmpc2_planner* p, int rows, size_t* out);
int tdmpc2_pi_loss_workspace_bytes(const tdmpc2_planner* p, int rows, size_t* out);
int tdmpc2_pi_loss_forward(tdmpc2_planner* p, const float* z, const int32_t* task, const float* eps, const int32_t* qidx,
                           const float* dropout_mask, int rows, float* tape, float* action_out, float* q_out,
                           float* log_prob_out, void* stream);
int tdmpc2_pi_loss_backward(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* z, const int32_t* task,
                            const float* eps, const int32_t* qidx, const float* dropout_mask, int T, int B, const float* scale,
                            float entropy_coef, float rho, const tdmpc2_pi_grads* grads, void* workspace, void* stream);

/* ---- agent._update: the world model's loss (tdmpc2.py:259-313), state observations ------------------------------
 * forward: the latent rollout of a [H + 1, B] batch (row r of a [H, B] batch is t B + b), as row launches that also
 * write the caller-owned tape [tape_bytes] (the pre-LayerNorm row of every LayerNorm layer, DESIGN section 4.4):
 *   encode(obs0 [B, obs_dim]) -> zs[0]; next(zs[t], action[t]) -> zs[t + 1] for t < H, written in place into
 *   zs [H + 1, B, L]; Q 'all' on (zs[:H], action) with dropout_mask (NULL: eval mode; else [num_q, H B, mlp_dim] of
 *   mask / (1 - p) on each head's layer 0) -> q_logits [num_q, H B, num_bins]; reward(zs[:H], action) -> reward_logits
 *   [H B, num_bins]; episodic models: termination(zs[1:]) -> term_logits [H B] (else NULL).
 *   task: NULL (single-task) or [H B] per-row task indices.  Pixel models (no state encoder): TDMPC2_ERR_UNSUPPORTED.
 * backward: from the tape, the forward's inputs and outputs, next_z [H, B, L] (encode(obs[1:])), reward / td_target /
 *   terminated [H B] and the loss coefficients, ADDS dL/dparameter of
 *     consistency * sum_t rho^t mse(zs[t+1], next_z[t]) / H + reward * sum_t rho^t soft_ce(reward logits, r_t).mean() / H
 *     + value * sum_{t,q} rho^t soft_ce(Q_q logits, td_t).mean() / (H num_q) + termination * bce(term logits, terminated)
 *   to grads (encoder, dynamics, reward, termination, the stacked Q heads, and the task embedding through every layer-0
 *   input), like autograd accumulates .grad.  fp32 FFMA on the fp32 tensors w; reductions over rows in a fixed order
 *   (repeated calls give identical bits); no allocation, no host synchronisation.  workspace: workspace_bytes(H, B). */
typedef struct tdmpc2_linear_grad {
  float* weight;
  float* bias;
  float* ln_weight;        /* NULL for a plain Linear (an MLP's layer 2) */
  float* ln_bias;
} tdmpc2_linear_grad;
typedef struct tdmpc2_wm_grads {
  int32_t num_enc;
  tdmpc2_linear_grad enc[TDMPC2_MAX_ENC_LAYERS];
  tdmpc2_linear_grad dynamics[3];
  tdmpc2_linear_grad reward[3];
  tdmpc2_linear_grad termination[3];   /* episodic models */
  tdmpc2_linear_grad qs[3];            /* [num_q] leading dim, like _Qs.params.* */
  float* task_emb;                     /* [num_tasks, T]; NULL for single-task models */
} tdmpc2_wm_grads;
typedef struct tdmpc2_wm_loss_coefs {
  float consistency, reward, value, termination, rho;
  float vmin, vmax, bin_size;          /* two_hot's range and bin width (math.py:58-71) */
} tdmpc2_wm_loss_coefs;
int tdmpc2_wm_loss_tape_bytes(const tdmpc2_planner* p, int H, int B, size_t* out);
int tdmpc2_wm_loss_workspace_bytes(const tdmpc2_planner* p, int H, int B, size_t* out);
int tdmpc2_wm_loss_forward(tdmpc2_planner* p, const float* obs0, const float* action, const int32_t* task,
                           const float* dropout_mask, int H, int B, float* zs, float* q_logits, float* reward_logits,
                           float* term_logits, float* tape, void* stream);
int tdmpc2_wm_loss_backward(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* obs0,
                            const float* action, const int32_t* task, const float* dropout_mask, int H, int B,
                            const float* zs, const float* q_logits, const float* reward_logits, const float* term_logits,
                            const float* next_z, const float* reward, const float* td_target, const float* terminated,
                            const tdmpc2_wm_loss_coefs* coefs, const tdmpc2_wm_grads* grads, void* workspace, void* stream);
/* Planners without a state encoder (pixel models, num_enc_layers = 0) get TDMPC2_ERR_UNSUPPORTED from the two calls above;
 * they use these.  _latent forward: zs[0] ([B, L]) is the caller's, written by tdmpc2_pixel_encode_taped; the rest as
 * tdmpc2_wm_loss_forward.  _latent backward: as tdmpc2_wm_loss_backward without the state encoder (grads->enc and
 * w->enc are not read), and dL/dz_0 [B, L] is written to dz0, for tdmpc2_pixel_encode_backward.  tape_bytes and
 * workspace_bytes answer for both variants. */
int tdmpc2_wm_loss_forward_latent(tdmpc2_planner* p, const float* action, const int32_t* task, const float* dropout_mask,
                                  int H, int B, float* zs, float* q_logits, float* reward_logits, float* term_logits,
                                  float* tape, void* stream);
int tdmpc2_wm_loss_backward_latent(tdmpc2_planner* p, const tdmpc2_weights* w, const float* tape, const float* action,
                                   const int32_t* task, const float* dropout_mask, int H, int B, const float* zs,
                                   const float* q_logits, const float* reward_logits, const float* term_logits,
                                   const float* next_z, const float* reward, const float* td_target, const float* terminated,
                                   const tdmpc2_wm_loss_coefs* coefs, const tdmpc2_wm_grads* grads, float* dz0,
                                   void* workspace, void* stream);

/* Diagnostics: y[rows, out] = act(LN(x W^T + b)) for ONE packed layer, through
 * the same fused kernels (rows <= 128).  layer index: 0.. = enc, then dynamics
 * 0-2, reward 0-2, pi 0-2, then q-head h layer l = base + 3*h + l.
 * mode: 0 = raw linear output, 1 = LN+Mish, 2 = LN+SimNorm. */
int tdmpc2_debug_layer(tdmpc2_planner* p, int layer, int mode, const float* x, int rows,
                       float* y, void* stream);
int tdmpc2_planner_layer_count(const tdmpc2_planner* p);
/* Diagnostics: per-CTA cycle counters.  device_buf: int64 [num_SMs][4 roles][12 counters] or NULL to disable.
 * roles: TMA producer, MMA issuer, epilogue thread, idle warp; counters: barrier-wait cycles,
 * cycles inside fused layers, accumulator-ready wait, publish (fence + CTA sync), -, whole kernel. */
int tdmpc2_planner_set_profile(tdmpc2_planner* p, long long* device_buf);
/* Number of kernel launches this planner has enqueued so far. */
int64_t tdmpc2_planner_launch_count(const tdmpc2_planner* p);

#ifdef __cplusplus
}
#endif
#endif /* TDMPC2_B200_H_ */
