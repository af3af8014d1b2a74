/* Plan from a plain C host: load a model file, act on observations read from a raw file, write the actions.
 * No Python, no torch: the header, libtdmpc2_b200 and the CUDA runtime.
 *
 *   gcc -std=c11 -Iinclude -I/usr/local/cuda/include examples/c_act.c -Ltdmpc2_b200 -ltdmpc2_b200 \
 *       -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,$PWD/tdmpc2_b200 -o c_act
 *   ./c_act MODEL OBS ACTIONS [--envs E] [--steps S] [--seed N] [--task K] [--eval] [--graph N]
 *
 * MODEL is what agent.export(fp) wrote.  OBS holds S x E observations, raw fp32: [E, obs_dim] per step for state models,
 * [E, C, 64, 64] frames (0..255) for pixel models.  ACTIONS receives S x [E, A] raw fp32.  Step 0 starts an episode in
 * every environment (t0 = 1).  Every random draw is made on the device (tdmpc2_act) under {seed, plan counter}, the
 * counter starting at 0.  --task K plans every environment for task K of a multi-task model (default 0).
 * --graph N: afterwards, capture one tdmpc2_act (t0 = 0, the last step's observations) in a CUDA graph, replay it N times
 * and print the time per replay from CUDA events. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "tdmpc2_b200.h"

#define TRY(call)                                                                    \
  do {                                                                               \
    int rc_ = (call);                                                                \
    if (rc_ != 0) {                                                                  \
      fprintf(stderr, "%s failed (%d): %s\n", #call, rc_, tdmpc2_last_error());     \
      return 1;                                                                      \
    }                                                                                \
  } while (0)
#define CUDA(call)                                                                   \
  do {                                                                               \
    cudaError_t e_ = (call);                                                         \
    if (e_ != cudaSuccess) {                                                         \
      fprintf(stderr, "%s failed: %s\n", #call, cudaGetErrorString(e_));            \
      return 1;                                                                      \
    }                                                                                \
  } while (0)

static void* dalloc(size_t n) {
  void* p = NULL;
  return cudaMalloc(&p, n ? n : 1) == cudaSuccess ? p : NULL;
}

int main(int argc, char** argv) {
  if (argc < 4) {
    fprintf(stderr, "usage: %s MODEL OBS ACTIONS [--envs E] [--steps S] [--seed N] [--task K] [--eval] [--graph N]\n", argv[0]);
    return 2;
  }
  int envs = 0, steps = 1, task_id = 0, eval_mode = 0, graph = 0;
  unsigned long long seed = 1;
  for (int i = 4; i < argc; ++i) {
    const char* a = argv[i];
    const char* v = i + 1 < argc ? argv[i + 1] : NULL;
    if (!strcmp(a, "--eval")) { eval_mode = 1; continue; }
    if (!v) { fprintf(stderr, "%s needs a value\n", a); return 2; }
    if (!strcmp(a, "--envs")) envs = atoi(v);
    else if (!strcmp(a, "--steps")) steps = atoi(v);
    else if (!strcmp(a, "--seed")) seed = strtoull(v, NULL, 10);
    else if (!strcmp(a, "--task")) task_id = atoi(v);
    else if (!strcmp(a, "--graph")) graph = atoi(v);
    else { fprintf(stderr, "unknown option %s\n", a); return 2; }
    ++i;
  }
  if (steps < 1) { fprintf(stderr, "--steps must be >= 1\n"); return 2; }

  /* 1. the model file and its dims */
  tdmpc2_model_file* mf = NULL;
  TRY(tdmpc2_model_file_open(argv[1], &mf));
  tdmpc2_dims d;
  tdmpc2_pixel_dims pd;
  int32_t is_pixel = 0;
  TRY(tdmpc2_model_file_dims(mf, &d, &pd, &is_pixel));
  if (envs > 0) d.num_envs = envs;
  const int E = d.num_envs, A = d.action_dim, H = d.horizon;
  const size_t obs_elems = is_pixel ? (size_t)pd.in_channels * 64 * 64 : (size_t)d.obs_dim;

  /* 2. planner, pixel encoder, weights */
  cudaStream_t stream;
  CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  tdmpc2_planner* p = NULL;
  TRY(tdmpc2_planner_create(&d, &p));
  size_t packed_bytes = 0, ws_bytes = 0, model_bytes = 0, scratch_bytes = 0, enc_ws_bytes = 0;
  TRY(tdmpc2_planner_packed_bytes(p, &packed_bytes));
  TRY(tdmpc2_planner_workspace_bytes(p, &ws_bytes));
  TRY(tdmpc2_model_file_device_bytes(mf, &d, &model_bytes));
  void *packed = dalloc(packed_bytes), *ws = dalloc(ws_bytes), *model = dalloc(model_bytes);
  if (!packed || !ws || !model) { fprintf(stderr, "cudaMalloc failed\n"); return 1; }
  TRY(tdmpc2_planner_bind(p, packed, ws));
  tdmpc2_weights w;
  tdmpc2_conv_weights conv;
  const float* grid_base = NULL;
  TRY(tdmpc2_model_file_upload(mf, &d, model, &w, &conv, &grid_base, stream));
  TRY(tdmpc2_pack_weights(p, &w, stream));
  tdmpc2_pixel_encoder* enc = NULL;
  void* enc_ws = NULL;
  if (is_pixel) {
    TRY(tdmpc2_pixel_encoder_create(&pd, &enc));
    TRY(tdmpc2_pixel_encoder_workspace_bytes(enc, &enc_ws_bytes));
    if (!(enc_ws = dalloc(enc_ws_bytes))) { fprintf(stderr, "cudaMalloc failed\n"); return 1; }
  }
  TRY(tdmpc2_act_scratch_bytes(p, enc, &scratch_bytes));

  /* 3. per-call buffers */
  float *obs = dalloc(E * obs_elems * 4), *prev_mean = dalloc((size_t)E * H * A * 4), *action = dalloc((size_t)E * A * 4);
  uint8_t* t0 = dalloc(E);
  int32_t* task = d.task_dim > 0 ? dalloc((size_t)E * 4) : NULL;
  uint64_t* rng_state = dalloc(16);
  void* scratch = dalloc(scratch_bytes);
  if (!obs || !prev_mean || !action || !t0 || !rng_state || !scratch || (d.task_dim > 0 && !task)) {
    fprintf(stderr, "cudaMalloc failed\n");
    return 1;
  }
  const uint64_t state0[2] = {seed, 0};
  CUDA(cudaMemcpy(rng_state, state0, sizeof state0, cudaMemcpyHostToDevice));
  CUDA(cudaMemset(prev_mean, 0, (size_t)E * H * A * 4));
  if (task) {
    int32_t* th = malloc((size_t)E * 4);
    for (int e = 0; e < E; ++e) th[e] = task_id;
    CUDA(cudaMemcpy(task, th, (size_t)E * 4, cudaMemcpyHostToDevice));
    free(th);
  }

  /* 4. observations in, actions out */
  FILE* fo = fopen(argv[2], "rb");
  FILE* fa = fopen(argv[3], "wb");
  if (!fo || !fa) { fprintf(stderr, "cannot open %s or %s\n", argv[2], argv[3]); return 1; }
  float* obs_h = malloc(E * obs_elems * 4);
  float* act_h = malloc((size_t)E * A * 4);
  tdmpc2_act_args args;
  memset(&args, 0, sizeof args);
  args.obs = is_pixel ? NULL : obs;
  args.frames = is_pixel ? obs : NULL;
  args.task = task;
  args.t0 = t0;
  args.eval_mode = eval_mode;
  args.rng_state = rng_state;
  args.prev_mean = prev_mean;
  args.action_out = action;
  args.grid_base = grid_base;
  for (int s = 0; s < steps; ++s) {
    if (fread(obs_h, 4, E * obs_elems, fo) != E * obs_elems) { fprintf(stderr, "%s: short read at step %d\n", argv[2], s); return 1; }
    CUDA(cudaMemcpyAsync(obs, obs_h, E * obs_elems * 4, cudaMemcpyHostToDevice, stream));
    CUDA(cudaMemsetAsync(t0, s == 0 ? 1 : 0, E, stream));
    TRY(tdmpc2_act(p, enc, enc_ws, is_pixel ? &conv : NULL, &args, scratch, stream));
    CUDA(cudaMemcpyAsync(act_h, action, (size_t)E * A * 4, cudaMemcpyDeviceToHost, stream));
    CUDA(cudaStreamSynchronize(stream));
    if (fwrite(act_h, 4, (size_t)E * A, fa) != (size_t)E * A) { fprintf(stderr, "%s: write failed\n", argv[3]); return 1; }
  }
  fclose(fo);
  fclose(fa);
  printf("acted %d steps x %d environments (%s model, %s mode)\n", steps, E, is_pixel ? "pixel" : "state",
         eval_mode ? "eval" : "explore");

  /* 5. one call as a CUDA graph, replayed with fresh noise each time (the counter is in device memory) */
  if (graph > 0) {
    cudaGraph_t g;
    cudaGraphExec_t ge;
    CUDA(cudaMemsetAsync(t0, 0, E, stream));
    CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    TRY(tdmpc2_act(p, enc, enc_ws, is_pixel ? &conv : NULL, &args, scratch, stream));
    CUDA(cudaStreamEndCapture(stream, &g));
    CUDA(cudaGraphInstantiate(&ge, g, 0));
    for (int i = 0; i < 10; ++i) CUDA(cudaGraphLaunch(ge, stream));
    cudaEvent_t a, b;
    CUDA(cudaEventCreate(&a));
    CUDA(cudaEventCreate(&b));
    CUDA(cudaEventRecord(a, stream));
    for (int i = 0; i < graph; ++i) CUDA(cudaGraphLaunch(ge, stream));
    CUDA(cudaEventRecord(b, stream));
    CUDA(cudaEventSynchronize(b));
    float ms = 0.f;
    CUDA(cudaEventElapsedTime(&ms, a, b));
    printf("graph: %d replays, %.4f ms per act (E = %d)\n", graph, ms / graph, E);
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    cudaGraphExecDestroy(ge);
    cudaGraphDestroy(g);
  }

  free(obs_h);
  free(act_h);
  cudaFree(obs); cudaFree(prev_mean); cudaFree(action); cudaFree(t0); cudaFree(task); cudaFree(rng_state); cudaFree(scratch);
  cudaFree(packed); cudaFree(ws); cudaFree(model); cudaFree(enc_ws);
  if (enc) tdmpc2_pixel_encoder_destroy(enc);
  tdmpc2_planner_destroy(p);
  tdmpc2_model_file_close(mf);
  cudaStreamDestroy(stream);
  return 0;
}
