/* Minimal C host of the C ABI (include/tdmpc2_b200.h): no Python, no torch.
 *
 *   gcc -std=c11 -Iinclude examples/c_host.c -Ltdmpc2_b200 -ltdmpc2_b200 -Wl,-rpath,$PWD/tdmpc2_b200 -o c_host
 *
 * Creates a planner for a small single-task model and prints the sizes of the two caller-owned device buffers
 * (packed weights, workspace).  A real host then allocates them (cudaMalloc), calls tdmpc2_planner_bind(),
 * fills a tdmpc2_weights with device pointers to the checkpoint tensors, tdmpc2_pack_weights(), and per environment
 * step runs tdmpc2_plan_prologue() -> iterations x tdmpc2_plan_iter() -> tdmpc2_plan_epilogue() on its stream
 * (INTEGRATION.md section 2).  Without an sm_90 device tdmpc2_planner_create() fails with TDMPC2_ERR_NO_DEVICE:
 * there is no CPU fallback. */
#include <stdio.h>
#include <string.h>

#include "tdmpc2_b200.h"

int main(void) {
  printf("tdmpc2_b200 ABI version %d (header %d)\n", tdmpc2_abi_version(), TDMPC2_B200_ABI_VERSION);
  if (tdmpc2_abi_version() != TDMPC2_B200_ABI_VERSION) return 2;

  tdmpc2_dims d;
  memset(&d, 0, sizeof d);
  d.num_envs = 4; d.num_samples = 512; d.num_pi_trajs = 24; d.num_elites = 64; d.horizon = 3; d.iterations = 6;
  d.obs_dim = 24; d.action_dim = 6; d.latent_dim = 512; d.mlp_dim = 512; d.enc_dim = 256; d.num_enc_layers = 2;
  d.task_dim = 0; d.num_tasks = 1; d.num_q = 5; d.num_bins = 101; d.simnorm_dim = 8; d.episodic = 0;
  d.temperature = 0.5f; d.min_std = 0.05f; d.max_std = 2.0f; d.log_std_min = -10.0f; d.log_std_dif = 12.0f;

  tdmpc2_planner* p = NULL;
  int rc = tdmpc2_planner_create(&d, &p);
  if (rc != TDMPC2_OK) {
    printf("tdmpc2_planner_create: %d (%s)\n", rc, tdmpc2_last_error());
    return rc == TDMPC2_ERR_NO_DEVICE ? 0 : 1;   /* expected on a machine without a H100 */
  }
  size_t packed = 0, ws = 0;
  tdmpc2_planner_packed_bytes(p, &packed);
  tdmpc2_planner_workspace_bytes(p, &ws);
  printf("planner: %d packed layers, %zu bytes of packed weights, %zu bytes of workspace\n",
         tdmpc2_planner_layer_count(p), packed, ws);
  tdmpc2_planner_destroy(p);
  return 0;
}
