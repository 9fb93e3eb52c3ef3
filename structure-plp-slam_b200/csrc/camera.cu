// camera.cu -- camera::perspective / camera::fisheye undistort_keypoints + convert_keypoints_to_bearings
// (camera/perspective.cc:130-175, camera/fisheye.cc:172-215) and compute_image_bounds (perspective.cc:100-127,
// fisheye.cc:101-169) (sm_90a).
//
// One thread per keypoint runs OpenCV's iteration in FP64 with cammath.h -- the text the oracle compiles, with -fmad=false,
// hence bit-identical.  The image bounds are a host computation (four corners, once per camera).
//
// util::stereo_rectifier (util/stereo_rectifier.cc:39-92): the float maps are built on the host once per rectifier
// (rectmath.h), converted to cv::remap's fixed point and kept on the device; rectify_kernel (rectify_kernels.cuh) remaps a
// batch of one side per launch.
#include "common.cuh"
#include "camera_kernels.cuh"
#include "rectify_kernels.cuh"
#include "rectmath.h"

using namespace plp;

struct plp_stereo_rectifier {
    int device = 0;
    int rows = 0, cols = 0, map_pitch = 0;
    short2 *d_xy[2] = {nullptr, nullptr};
    uint16_t *d_frac[2] = {nullptr, nullptr};
    std::vector<float> map_x[2], map_y[2];  // the float maps, rows x cols (plp_stereo_rectifier_maps)
};

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
    DevLayout L;
    J.batch = 1;
    J.cap = n;
    L.in(J.kp, kp, n);
    J.n_kp = nullptr;
    L.out(J.out, n);
    J.bearings = nullptr;
    if (bearings_out) L.out(J.bearings, (size_t)n * 3);
    PLP_TRY(stage(ctx, 0, L));
    PLP_TRY(launch_undistort(ctx, J));
    PLP_CUDA_TRY(to_host(ctx, undist_out, J.out, n));
    if (bearings_out) PLP_CUDA_TRY(to_host(ctx, bearings_out, J.bearings, (size_t)n * 3));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

}  // extern "C"

namespace {

plp_status launch_rectify(plp_ctx *ctx, const plp_stereo_rectifier *r, int side, const uint8_t *d_in, int batch,
                          size_t in_step, uint8_t *d_out, size_t out_step) {
    if (batch == 0) return PLP_OK;
    PLP_REQUIRE((((uintptr_t)d_out | out_step) & 3) == 0, "rectified rows are stored as 32-bit words");
    RectJob J;
    J.xy = r->d_xy[side];
    J.frac = r->d_frac[side];
    J.rows = r->rows;
    J.cols = r->cols;
    J.map_pitch = r->map_pitch;
    J.batch = batch;
    unsigned gx, gy;
    rect_grid(r->rows, r->cols, batch, &gx, &gy, &J.frames_per_cta);
    J.in = d_in;
    J.in_step = in_step;
    J.out = d_out;
    J.out_step = out_step;
    PLP_LAUNCH(ctx, rectify_kernel, dim3(gx, gy), kRectThreads, 0, J);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

}  // namespace

extern "C" {

plp_status plp_stereo_rectifier_create(plp_ctx *ctx, const plp_stereo_rectifier_params *params, int rows, int cols,
                                       plp_stereo_rectifier **out) {
    PLP_REQUIRE(ctx && params && out, "null pointer");
    *out = nullptr;
    PLP_REQUIRE(rows >= 1 && cols >= 1 && rows <= 65535 * kRectTileH, "sizes");
    PLP_REQUIRE(params->model == 0 || params->model == 1, "rectifier model must be 0 (perspective) or 1 (fisheye)");
    plp_stereo_rectifier *r = new plp_stereo_rectifier;
    r->device = ctx->device;
    r->rows = rows;
    r->cols = cols;
    r->map_pitch = rect_map_pitch(cols);
    const double Kr[4] = {params->fx, params->fy, params->cx, params->cy};
    const double *K[2] = {params->K_left, params->K_right}, *D[2] = {params->D_left, params->D_right},
                 *R[2] = {params->R_left, params->R_right};
    const size_t n = (size_t)rows * cols, nm = (size_t)rows * r->map_pitch;
    std::vector<short2> xy(nm);
    std::vector<uint16_t> frac(nm);
    for (int s = 0; s < 2; ++s) {
        r->map_x[s].resize(n);
        r->map_y[s].resize(n);
        if (rect_build_maps(params->model, K[s], D[s], R[s], Kr, rows, cols, r->map_x[s].data(), r->map_y[s].data())) {
            plp_stereo_rectifier_destroy(r);
            set_error("invalid argument: K_rect * R_%s is singular", s ? "right" : "left");
            return PLP_ERR_INVALID;
        }
        rect_fixed_map(r->map_x[s].data(), r->map_y[s].data(), rows, cols, xy.data(), frac.data());
        cudaError_t e = cudaSetDevice(ctx->device);
        if (e == cudaSuccess) e = cudaMalloc(&r->d_xy[s], nm * sizeof(short2));
        if (e == cudaSuccess) e = cudaMalloc(&r->d_frac[s], nm * sizeof(uint16_t));
        if (e == cudaSuccess) e = cudaMemcpy(r->d_xy[s], xy.data(), nm * sizeof(short2), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(r->d_frac[s], frac.data(), nm * sizeof(uint16_t), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            set_error("stereo rectifier: %s", cudaGetErrorString(e));
            plp_stereo_rectifier_destroy(r);
            return PLP_ERR_CUDA;
        }
    }
    *out = r;
    return PLP_OK;
}

void plp_stereo_rectifier_destroy(plp_stereo_rectifier *r) {
    if (!r) return;
    cudaSetDevice(r->device);
    for (int s = 0; s < 2; ++s) {
        cudaFree(r->d_xy[s]);
        cudaFree(r->d_frac[s]);
    }
    delete r;
}

plp_status plp_stereo_rectifier_maps(const plp_stereo_rectifier *r, int side, float *map_x, float *map_y) {
    PLP_REQUIRE(r && map_x && map_y, "null pointer");
    PLP_REQUIRE(side == 0 || side == 1, "side must be 0 (left) or 1 (right)");
    memcpy(map_x, r->map_x[side].data(), r->map_x[side].size() * sizeof(float));
    memcpy(map_y, r->map_y[side].data(), r->map_y[side].size() * sizeof(float));
    return PLP_OK;
}

plp_status plp_stereo_rectify(plp_ctx *ctx, const plp_stereo_rectifier *r, const uint8_t *left, const uint8_t *right,
                              size_t step, uint8_t *left_out, uint8_t *right_out, size_t out_step) {
    PLP_REQUIRE(ctx && r && left && right && left_out && right_out, "null pointer");
    PLP_REQUIRE(ctx->device == r->device, "the context and the rectifier are on different devices");
    PLP_REQUIRE(step >= (size_t)r->cols && out_step >= (size_t)r->cols, "steps");
    const size_t cols = (size_t)r->cols, rows = (size_t)r->rows, pitch = (size_t)div_up(r->cols, 16) * 16;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    uint8_t *d;
    PLP_TRY(ctx_scratch(ctx, 0, 2 * rows * (cols + pitch), (void **)&d));
    const uint8_t *src[2] = {left, right};
    uint8_t *dst[2] = {left_out, right_out};
    for (int s = 0; s < 2; ++s) {
        // the outputs first: the kernel stores words, so their base and pitch are multiples of 16
        uint8_t *d_out = d + s * rows * pitch, *d_in = d + 2 * rows * pitch + s * rows * cols;
        PLP_CUDA_TRY(cudaMemcpy2DAsync(d_in, cols, src[s], step, cols, rows, cudaMemcpyHostToDevice, ctx->stream));
        PLP_TRY(launch_rectify(ctx, r, s, d_in, 1, cols, d_out, pitch));
        PLP_CUDA_TRY(cudaMemcpy2DAsync(dst[s], out_step, d_out, pitch, cols, rows, cudaMemcpyDeviceToHost, ctx->stream));
    }
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_stereo_rectify_batch_dev(plp_ctx *ctx, const plp_stereo_rectifier *r, int side, const uint8_t *d_in,
                                        int batch, size_t in_step, uint8_t *d_out, size_t out_step) {
    PLP_REQUIRE(ctx && r && d_in && d_out, "null pointer");
    PLP_REQUIRE(side == 0 || side == 1, "side must be 0 (left) or 1 (right)");
    PLP_REQUIRE(batch >= 0, "batch");
    PLP_REQUIRE(ctx->device == r->device, "the context and the rectifier are on different devices");
    PLP_REQUIRE(in_step >= (size_t)r->cols && out_step >= (size_t)r->cols, "steps");
    // the output is a level 0 the ORB extractor reads through TMA: base and step multiples of 16
    PLP_REQUIRE((((uintptr_t)d_out | out_step) & 15) == 0, "d_out and out_step must be multiples of 16");
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    return launch_rectify(ctx, r, side, d_in, batch, in_step, d_out, out_step);
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
