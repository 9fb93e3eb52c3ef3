// oracle/camera.cc -- camera::perspective / camera::fisheye keypoint undistortion, bearings and image bounds (TEST
// INFRASTRUCTURE ONLY).  Follows the reference's camera/perspective.cc and camera/fisheye.cc; OpenCV's
// undistortPoints / fisheye::undistortPoints are restated in cammath.h (see its header).
#include "camera.h"
#include "cammath.h"

extern "C" {

void orc_undistort_keypoints(int model, const double *K, const double *D, const float *xy, int n, float *undist_xy) {
    // perspective.cc:47-48 / fisheye.cc:47-48: cv::Mat_<float> camera matrix and coefficients
    double Kf[4], kf[5];
    cam_round_params(K, D, Kf, kf);
    for (int i = 0; i < n; ++i)  // perspective.cc:145-162 / fisheye.cc:187-203, one point at a time like OpenCV
        cam_undistort(model, Kf, kf, xy[2 * i], xy[2 * i + 1], &undist_xy[2 * i], &undist_xy[2 * i + 1]);
}

void orc_bearings(const double *K, const float *undist_xy, int n, double *bearings) {
    for (int i = 0; i < n; ++i) cam_bearing(K, undist_xy[2 * i], undist_xy[2 * i + 1], bearings + 3 * i);
}

void orc_image_bounds(int model, const double *K, const double *D, int cols, int rows, float *bounds) {
    cam_image_bounds(model, K, D, (unsigned)cols, (unsigned)rows, bounds);
}

}  // extern "C"
