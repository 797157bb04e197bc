// HalfCheetah (mujoco/gym) family: host-side handle over the two-lane physics kernel.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace epb {

struct MjcPool;

MjcPool* mjc_pool_create(int num_envs, int precision, int frame_skip, double ctrl_cost_weight,
                         double forward_reward_weight, double reset_noise_scale);
void mjc_pool_destroy(MjcPool* m);
int64_t mjc_model_blob(void* dst, int64_t cap);  // sizeof(hcm::HcModel); fills dst if it fits
int mjc_state_reals(const MjcPool* m);  // persistent reals per env (qpos, qvel, warmstart, ...)
// constraint rows per lane the two-lane kernel keeps in shared memory for a launch of n rows
int mjc_pair_rows(const MjcPool* m, int n);
cudaError_t mjc_launch_step(MjcPool* m, const StateView& sv, const OutView& ov,
                            const double* d_action, const int32_t* d_env_ids, int n,
                            int force_reset, cudaStream_t stream);
cudaError_t mjc_launch_rollout(MjcPool* m, const StateView& sv, const OutView& ov,
                               const double* d_actions, int T, cudaStream_t stream);

}  // namespace epb
