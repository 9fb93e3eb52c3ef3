// camera_kernels.cuh -- device code of keypoint undistortion (camera.cu and pipeline.cu launch it).  Free of host-side CUDA
// runtime dependencies so that tests/cta_emu can compile the same text for the host (see plane_kernels.cuh).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "camera_jobs.h"
#include "cammath.h"

namespace plp {

namespace {

constexpr int kUndistThreads = 256;

// undistort_keypoints + convert_keypoints_to_bearings, one thread per keypoint slot (FP64; at most 20 perspective or
// 10 fisheye iterations).  Slots past a frame's keypoint count are left untouched.
__global__ void __launch_bounds__(kUndistThreads) undistort_keypoints_kernel(UndistJob J) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)J.batch * J.cap) return;
    const int b = (int)(i / J.cap), j = (int)(i % J.cap);
    if (j >= (J.n_kp ? J.n_kp[b] : J.cap)) return;
    const plp_keypoint in = J.kp[i];
    plp_keypoint o;
    cam_undistort(J.model, J.K, J.k, in.x, in.y, &o.x, &o.y);
    // perspective.cc:155-161: pt, angle, size and octave; the rest keeps cv::KeyPoint's defaults
    o.size = in.size;
    o.angle = in.angle;
    o.response = 0.0f;
    o.octave = in.octave;
    o.class_id = -1;
    J.out[i] = o;
    if (J.bearings) cam_bearing(J.K_cfg, o.x, o.y, J.bearings + 3 * i);
}

}  // namespace

}  // namespace plp
