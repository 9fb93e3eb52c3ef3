/* cammath.h -- keypoint undistortion, bearings and image bounds of camera::perspective and camera::fisheye
 * (camera/perspective.cc:100-175, camera/fisheye.cc:101-216) in plain IEEE-754 double / float arithmetic (+, -, *, /,
 * sqrt, tan; no FMA), so that a host build (-ffp-contract=off) and a device build (-fmad=false) round alike.
 *
 * The reference undistorts through OpenCV with the camera matrix and coefficients stored as cv::Mat_<float>
 * (perspective.cc:47-48, fisheye.cc:47-48); OpenCV widens them to double.  So the undistortion below takes the
 * FLOAT-ROUNDED fx, fy, cx, cy and k (cam_round_params), while the bearings use the config's double fx_, cx_.
 *   - perspective: cv::undistortPoints(R = none, P = K, TermCriteria(EPS | MAX_ITER, 20, 1e-6)), OpenCV's
 *     cvUndistortPointsInternal loop for the 5-coefficient model.  The tilt matrices are the identity and the
 *     coefficients k[5..13] are zero; the terms they contribute add exactly +0 and are left out.
 *   - fisheye: cv::fisheye::undistortPoints(R = none, P = K) with its default TermCriteria(MAX_ITER + EPS, 10, 1e-8):
 *     Newton iteration on theta, (-1e6, -1e6) for points that do not converge or whose theta changes sign.
 * The products with the identity / K matrices are written out term by term in OpenCV's order (Matx: s = 0, s += a*b), so
 * even the sign of a zero matches.  tests/test_camera_oracle.py pins the oracle's copy to cv2 bit for bit.
 *
 * This file exists twice with identical text (oracle/cammath.h and structure-plp-slam_b200/csrc/cammath.h); the oracle
 * never includes product code and vice versa.  tests/test_camera_oracle.py checks that the copies stay identical.
 */
#ifndef PLP_CAMMATH_H
#define PLP_CAMMATH_H

#include <math.h>

#if defined(__CUDACC__)
#define CAM_HD __host__ __device__ __forceinline__
#define CAM_H static inline __host__
#else
#define CAM_HD static inline
#define CAM_H static inline
#endif

#define CAM_PERSPECTIVE 0
#define CAM_FISHEYE 1

/* fx, fy, cx, cy and k as cv::Mat_<float> holds them, widened back to double */
CAM_HD void cam_round_params(const double K_cfg[4], const double k_cfg[5], double K[4], double k[5]) {
    for (int i = 0; i < 4; ++i) K[i] = (double)(float)K_cfg[i];
    for (int i = 0; i < 5; ++i) k[i] = (double)(float)k_cfg[i];
}

/* cv::undistortPoints of one float point; K = (fx, fy, cx, cy), k = (k1, k2, p1, p2, k3), both float-rounded */
CAM_HD void cam_undistort_perspective(const double K[4], const double k[5], float pu, float pv, float *xo, float *yo) {
    const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
    const double ifx = 1. / fx, ify = 1. / fy;
    const double u = pu, v = pv;
    double x = (u - cx) * ifx;
    double y = (v - cy) * ify;
    /* invMatTilt * (x, y, 1), invProj = 1 */
    const double ux = ((0.0 + 1.0 * x) + 0.0 * y) + 0.0 * 1.0;
    const double uy = ((0.0 + 0.0 * x) + 1.0 * y) + 0.0 * 1.0;
    const double x0 = 1.0 * ux, y0 = 1.0 * uy;
    x = x0;
    y = y0;
    double error = 1.7976931348623157e308; /* DBL_MAX */
    for (int j = 0;; ++j) {
        if (j >= 20) break;          /* COUNT */
        if (error < 1e-6) break;     /* EPS */
        double r2 = x * x + y * y;
        const double icdist = 1.0 / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) { /* OpenCV regression_14583: give up on the point */
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        const double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x);
        const double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
        /* reprojection error of the current estimate */
        r2 = x * x + y * y;
        const double r4 = r2 * r2, r6 = r4 * r2;
        const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
        const double cdist = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6;
        const double icdist2 = 1. / 1.0;
        const double xd0 = x * cdist * icdist2 + k[2] * a1 + k[3] * a2;
        const double yd0 = y * cdist * icdist2 + k[2] * a3 + k[3] * a1;
        const double tx = ((0.0 + 1.0 * xd0) + 0.0 * yd0) + 0.0 * 1.0;
        const double ty = ((0.0 + 0.0 * xd0) + 1.0 * yd0) + 0.0 * 1.0;
        const double xd = 1.0 * tx, yd = 1.0 * ty;
        const double x_proj = xd * fx + cx;
        const double y_proj = yd * fy + cy;
        const double ex = x_proj - u, ey = y_proj - v;
        error = sqrt(ex * ex + ey * ey);
    }
    /* RR = P * I = K */
    const double xx = ((0.0 + fx * x) + 0.0 * y) + cx;
    const double yy = ((0.0 + 0.0 * x) + fy * y) + cy;
    const double ww = 1. / (((0.0 + 0.0 * x) + 0.0 * y) + 1.0);
    *xo = (float)(xx * ww);
    *yo = (float)(yy * ww);
}

/* cv::fisheye::undistortPoints of one float point; K = (fx, fy, cx, cy), k = (k1, k2, k3, k4), both float-rounded */
CAM_HD void cam_undistort_fisheye(const double K[4], const double k[4], float pu, float pv, float *xo, float *yo) {
    const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
    const double eps = 1e-8;
    const double pw0 = ((double)pu - cx) / fx, pw1 = ((double)pv - cy) / fy;
    double theta_d = sqrt(pw0 * pw0 + pw1 * pw1);
    /* the model is valid up to 180 degrees of FOV: clip */
    const double half_pi = 3.14159265358979323846 / 2.;
    theta_d = theta_d < -half_pi ? -half_pi : theta_d;
    theta_d = theta_d > half_pi ? half_pi : theta_d;
    int converged = 0;
    double theta = theta_d;
    double scale = 0.0;
    if (fabs(theta_d) > eps) {
        for (int j = 0; j < 10; ++j) {
            const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
            const double k0_theta2 = k[0] * theta2, k1_theta4 = k[1] * theta4, k2_theta6 = k[2] * theta6,
                         k3_theta8 = k[3] * theta8;
            const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                     (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
            theta = theta - theta_fix;
            if (fabs(theta_fix) < eps) {
                converged = 1;
                break;
            }
        }
        scale = tan(theta) / theta_d;
    } else {
        converged = 1;
    }
    const int theta_flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
    if (converged && !theta_flipped) {
        const double pu0 = pw0 * scale, pu1 = pw1 * scale;
        const double pr0 = ((0.0 + fx * pu0) + 0.0 * pu1) + cx * 1.0;
        const double pr1 = ((0.0 + 0.0 * pu0) + fy * pu1) + cy * 1.0;
        const double pr2 = ((0.0 + 0.0 * pu0) + 0.0 * pu1) + 1.0 * 1.0;
        *xo = (float)(pr0 / pr2);
        *yo = (float)(pr1 / pr2);
    } else {
        *xo = -1000000.0f;
        *yo = -1000000.0f;
    }
}

/* undistort_keypoints of one point for either model (float-rounded K and k) */
CAM_HD void cam_undistort(int model, const double K[4], const double k[5], float pu, float pv, float *xo, float *yo) {
    if (model == CAM_FISHEYE)
        cam_undistort_fisheye(K, k, pu, pv, xo, yo);
    else
        cam_undistort_perspective(K, k, pu, pv, xo, yo);
}

/* convert_keypoints_to_bearings (perspective.cc:165-175, fisheye.cc:205-215; identical text): the config's DOUBLE
 * fx_, fy_, cx_, cy_ and the float undistorted point */
CAM_HD void cam_bearing(const double K_cfg[4], float x, float y, double b[3]) {
    const double x_normalized = ((double)x - K_cfg[2]) / K_cfg[0];
    const double y_normalized = ((double)y - K_cfg[3]) / K_cfg[1];
    const double l2_norm = sqrt(x_normalized * x_normalized + y_normalized * y_normalized + 1.0);
    b[0] = x_normalized / l2_norm;
    b[1] = y_normalized / l2_norm;
    b[2] = 1.0 / l2_norm;
}

/* compute_image_bounds (perspective.cc:100-127, fisheye.cc:101-169): out = (min_x, max_x, min_y, max_y).  K_cfg, k_cfg:
 * the config's doubles (the zero-distortion test and the wide-FOV test read those; the undistortion rounds them). */
CAM_H void cam_image_bounds(int model, const double K_cfg[4], const double k_cfg[5], unsigned cols, unsigned rows,
                            float out[4]) {
    const int nk = model == CAM_FISHEYE ? 4 : 5;
    int zero = 1;
    for (int i = 0; i < nk; ++i) zero = zero && k_cfg[i] == 0;
    if (zero) {
        out[0] = 0.0f;
        out[1] = (float)cols;
        out[2] = 0.0f;
        out[3] = (float)rows;
        return;
    }
    double K[4], k[5];
    cam_round_params(K_cfg, k_cfg, K, k);
    const double fx_ = K_cfg[0], fy_ = K_cfg[1], cx_ = K_cfg[2], cy_ = K_cfg[3];
    if (model == CAM_FISHEYE) {
        const double pwx = (0.0 - cx_) / fx_;
        const double pwy = (0.0 - cy_) / fy_;
        const double theta_d = sqrt(pwx * pwx + pwy * pwy);
        if (theta_d > 1.57079632679489661923) { /* M_PI_2: the four corners are out of view (fisheye.cc:113-148) */
            /* top (cx, 0), right (cols, cy), left (0, cy), bottom (cx, rows); cv::KeyPoint stores float */
            float ux[4], uy[4];
            const float px[4] = {(float)cx_, (float)cols, 0.0f, (float)cx_};
            const float py[4] = {0.0f, (float)cy_, (float)cy_, (float)rows};
            for (int i = 0; i < 4; ++i) cam_undistort_fisheye(K, k, px[i], py[i], &ux[i], &uy[i]);
            const float deg_thr = 5.0f;
            const float dist_thr_x = (float)(fx_ / tan(deg_thr * 3.14159265358979323846 / 180.0));
            const float dist_thr_y = (float)(fy_ / tan(deg_thr * 3.14159265358979323846 / 180.0));
            const float min_x_thr = (float)(-dist_thr_x + cx_);
            const float max_x_thr = (float)(dist_thr_x + cx_);
            const float min_y_thr = (float)(-dist_thr_y + cy_);
            const float max_y_thr = (float)(dist_thr_y + cy_);
            const float undist_min_x = ux[2], undist_max_x = ux[1], undist_min_y = uy[0], undist_max_y = uy[3];
            out[0] = (undist_min_x < min_x_thr || undist_min_x > cx_) ? min_x_thr : undist_min_x;
            out[1] = (undist_max_x > max_x_thr || undist_max_x < cx_) ? max_x_thr : undist_max_x;
            out[2] = (undist_min_y < min_y_thr || undist_min_y > cy_) ? min_y_thr : undist_min_y;
            out[3] = (undist_max_y > max_y_thr || undist_max_y < cy_) ? max_y_thr : undist_max_y;
            return;
        }
    }
    /* left top, right top, left bottom, right bottom */
    const float px[4] = {0.0f, (float)cols, 0.0f, (float)cols};
    const float py[4] = {0.0f, 0.0f, (float)rows, (float)rows};
    float ux[4], uy[4];
    for (int i = 0; i < 4; ++i) cam_undistort(model, K, k, px[i], py[i], &ux[i], &uy[i]);
    out[0] = ux[2] < ux[0] ? ux[2] : ux[0];   /* std::min(a, b) = (b < a) ? b : a */
    out[1] = ux[1] < ux[3] ? ux[3] : ux[1];   /* std::max(a, b) = (a < b) ? b : a */
    out[2] = uy[1] < uy[0] ? uy[1] : uy[0];
    out[3] = uy[2] < uy[3] ? uy[3] : uy[2];
}

#endif
