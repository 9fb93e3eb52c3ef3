// camera_emu.cc -- csrc/camera_kernels.cuh executed on the host (see cta_emu.h): the undistortion kernel's indexing over
// batch x capacity slots and per-frame keypoint counts, against the oracle.
#include "cta_emu.h"

#include "camera_kernels.cuh"

using namespace plp;

extern "C" void emu_undistort_batch(int model, const double *K_cfg, const double *k_cfg, int batch, int cap,
                                    const plp_keypoint *kp, const int32_t *n_kp, plp_keypoint *out, double *bearings) {
    UndistJob J;
    J.model = model;
    cam_round_params(K_cfg, k_cfg, J.K, J.k);
    for (int i = 0; i < 4; ++i) J.K_cfg[i] = K_cfg[i];
    J.batch = batch;
    J.cap = cap;
    J.kp = kp;
    J.n_kp = n_kp;
    J.out = out;
    J.bearings = bearings;
    const unsigned n = (unsigned)(batch * cap);
    emu_launch(undistort_keypoints_kernel, (n + kUndistThreads - 1) / kUndistThreads, (unsigned)kUndistThreads, J);
}
