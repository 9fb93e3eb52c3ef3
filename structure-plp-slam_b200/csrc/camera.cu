// camera.cu -- camera::perspective / camera::fisheye undistort_keypoints + convert_keypoints_to_bearings
// (camera/perspective.cc:130-175, camera/fisheye.cc:172-215) and compute_image_bounds (perspective.cc:100-127,
// fisheye.cc:101-169) (sm_90a).
//
// One thread per keypoint runs OpenCV's iteration in FP64 with cammath.h -- the text the oracle compiles, with -fmad=false,
// hence bit-identical.  The image bounds are a host computation (four corners, once per camera).
#include "common.cuh"
#include "pack.cuh"
#include "camera_kernels.cuh"

using namespace plp;

namespace plp {

plp_status make_undist_job(const plp_camera *cam, const plp_distortion *dist, UndistJob *J) {
    PLP_REQUIRE(cam && dist, "null pointer");
    PLP_REQUIRE(dist->model == 0 || dist->model == 1, "distortion model must be 0 (perspective) or 1 (fisheye)");
    memset(J, 0, sizeof(*J));
    J->model = dist->model;
    const double K_cfg[4] = {cam->fx, cam->fy, cam->cx, cam->cy};
    double k_cfg[5];
    for (int i = 0; i < 5; ++i) k_cfg[i] = (dist->model == 1 && i == 4) ? 0.0 : dist->k[i];
    cam_round_params(K_cfg, k_cfg, J->K, J->k);
    for (int i = 0; i < 4; ++i) J->K_cfg[i] = K_cfg[i];
    return PLP_OK;
}

bool distortion_is_identity(const plp_distortion *dist) {
    if (!dist || dist->model != 0) return dist == nullptr;  // fisheye with k = 0 is still the equidistant model
    for (int i = 0; i < 5; ++i)
        if ((float)dist->k[i] != 0.0f) return false;
    return true;
}

plp_status launch_undistort(plp_ctx *ctx, const UndistJob &J) {
    const size_t n = (size_t)J.batch * J.cap;
    if (n == 0) return PLP_OK;
    PLP_LAUNCH(ctx, undistort_keypoints_kernel, (unsigned)div_up((int)n, kUndistThreads), kUndistThreads, 0, J);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

}  // namespace plp

extern "C" {

plp_status plp_camera_image_bounds(const plp_camera *cam, const plp_distortion *dist, int cols, int rows,
                                   float bounds_out[4]) {
    PLP_REQUIRE(cam && dist && bounds_out, "null pointer");
    PLP_REQUIRE(cols >= 1 && rows >= 1, "sizes");
    PLP_REQUIRE(dist->model == 0 || dist->model == 1, "distortion model must be 0 (perspective) or 1 (fisheye)");
    const double K_cfg[4] = {cam->fx, cam->fy, cam->cx, cam->cy};
    cam_image_bounds(dist->model, K_cfg, dist->k, (unsigned)cols, (unsigned)rows, bounds_out);
    return PLP_OK;
}

plp_status plp_undistort_keypoints(plp_ctx *ctx, const plp_camera *cam, const plp_distortion *dist, const plp_keypoint *kp,
                                   int n, plp_keypoint *undist_out, double *bearings_out) {
    PLP_REQUIRE(ctx && cam && dist, "null pointer");
    PLP_REQUIRE(n >= 0, "sizes");
    if (n == 0) return PLP_OK;  // perspective.cc:132-137: empty input, empty output
    PLP_REQUIRE(kp && undist_out, "null pointer");
    UndistJob J;
    PLP_TRY(make_undist_job(cam, dist, &J));
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    Packer pk;
    const size_t o_in = pk.add(kp, (size_t)n * sizeof(plp_keypoint));
    const size_t o_out = pk.reserve((size_t)n * sizeof(plp_keypoint));
    const size_t o_b = pk.reserve(bearings_out ? (size_t)n * 24 : 0);
    uint8_t *d;
    PLP_TRY(pk.upload(ctx, 0, &d));
    J.batch = 1;
    J.cap = n;
    J.kp = Packer::at<plp_keypoint>(d, o_in);
    J.n_kp = nullptr;
    J.out = Packer::at<plp_keypoint>(d, o_out);
    J.bearings = bearings_out ? Packer::at<double>(d, o_b) : nullptr;
    PLP_TRY(launch_undistort(ctx, J));
    PLP_CUDA_TRY(cudaMemcpyAsync(undist_out, J.out, (size_t)n * sizeof(plp_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
    if (bearings_out)
        PLP_CUDA_TRY(cudaMemcpyAsync(bearings_out, J.bearings, (size_t)n * 24, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_undistort_keypoints_batch_dev(plp_ctx *ctx, const plp_camera *cam, const plp_distortion *dist, int batch,
                                             int cap, const plp_keypoint *d_kp, const int32_t *d_n_kp,
                                             plp_keypoint *d_undist_out, double *d_bearings_out) {
    PLP_REQUIRE(ctx && cam && dist && d_kp && d_n_kp && d_undist_out, "null pointer");
    PLP_REQUIRE(batch >= 0 && cap >= 1, "sizes");
    UndistJob J;
    PLP_TRY(make_undist_job(cam, dist, &J));
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    J.batch = batch;
    J.cap = cap;
    J.kp = d_kp;
    J.n_kp = d_n_kp;
    J.out = d_undist_out;
    J.bearings = d_bearings_out;
    return launch_undistort(ctx, J);
}

}  // extern "C"
