// pose_kernels.cuh -- device job descriptor + launcher of the motion-only BA kernel, shared by pose_opt.cu
// (C ABI) and pipeline.cu (device-resident tracking front-end).
#pragma once
#include "common.cuh"
#include "pose_jobs.h"

namespace plp {

plp_status launch_pose_opt(plp_ctx *ctx, const PoseJob *d_jobs, int batch, const plp_camera &cam,
                           const plp_pose_opt_cfg &cfg);

}  // namespace plp
