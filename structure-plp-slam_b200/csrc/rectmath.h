/* rectmath.h -- the undistort-rectify maps of util::stereo_rectifier (util/stereo_rectifier.cc:39-80) in plain IEEE-754
 * double arithmetic (+, -, *, /, sqrt, atan; no FMA), so that every build of this text (-ffp-contract=off on the host,
 * -fmad=false under nvcc) produces the same float maps.
 *
 *   - model 0: cv::initUndistortRectifyMap(K, D, R, K_rect, size, CV_32F), radial-tangential (k1, k2, p1, p2, k3).
 *   - model 1: cv::fisheye::initUndistortRectifyMap(K, D, R, K_rect, size, CV_32F), equidistant (k1, k2, k3, k4).
 * K, D and R are the config's doubles (parse_vector_as_mat, CV_64F).  K_rect is camera::perspective::cv_cam_matrix_, a
 * cv::Mat_<float>: its fx, fy, cx, cy are rounded to float before OpenCV widens them back to double.
 *
 * iR = inv(K_rect * R) is the closed-form 3x3 inverse (determinant and cofactors in OpenCV's order).  That is what
 * cv::initUndistortRectifyMap computes (DECOMP_LU).  cv::fisheye::initUndistortRectifyMap inverts with DECOMP_SVD, which is
 * not restated: for the fisheye model the closed form is an empirical match -- bit for bit on the TUM-VI and synthetic
 * fisheye maps the tests pin -- and a new fisheye configuration can differ from cv2 in the last bit of a map entry where
 * the two inverses differ.  Pixel (j, i) of the
 * output maps to the ray (j, i, 1) * iR^T; the perspective model forms it as (i * iR01 + iR02) + j * iR00, the fisheye
 * model accumulates iR00 along the row as cv::fisheye::initUndistortRectifyMap does.  tests/test_rectify_oracle.py pins
 * both to cv2 bit for bit.  The maps are built once per rectifier on the host; they are not on the per-frame path.
 */
#ifndef PLP_RECTMATH_H
#define PLP_RECTMATH_H

#include <math.h>

#include "cammath.h"

/* the closed-form inverse of a row-major 3x3 (cv::invert, DECOMP_LU, n == 3; see above for the fisheye model); returns 0
 * when the determinant is 0 */
CAM_H int rect_inv3(const double m[9], double t[9]) {
#define M_(r, c) m[3 * (r) + (c)]
    double d = M_(0, 0) * (M_(1, 1) * M_(2, 2) - M_(1, 2) * M_(2, 1)) - M_(0, 1) * (M_(1, 0) * M_(2, 2) - M_(1, 2) * M_(2, 0)) +
               M_(0, 2) * (M_(1, 0) * M_(2, 1) - M_(1, 1) * M_(2, 0));
    if (d == 0.0) return 0;
    d = 1. / d;
    t[0] = (M_(1, 1) * M_(2, 2) - M_(1, 2) * M_(2, 1)) * d;
    t[1] = (M_(0, 2) * M_(2, 1) - M_(0, 1) * M_(2, 2)) * d;
    t[2] = (M_(0, 1) * M_(1, 2) - M_(0, 2) * M_(1, 1)) * d;
    t[3] = (M_(1, 2) * M_(2, 0) - M_(1, 0) * M_(2, 2)) * d;
    t[4] = (M_(0, 0) * M_(2, 2) - M_(0, 2) * M_(2, 0)) * d;
    t[5] = (M_(0, 2) * M_(1, 0) - M_(0, 0) * M_(1, 2)) * d;
    t[6] = (M_(1, 0) * M_(2, 1) - M_(1, 1) * M_(2, 0)) * d;
    t[7] = (M_(0, 1) * M_(2, 0) - M_(0, 0) * M_(2, 1)) * d;
    t[8] = (M_(0, 0) * M_(1, 1) - M_(0, 1) * M_(1, 0)) * d;
#undef M_
    return 1;
}

/* The float maps of one side: map_x, map_y are rows x cols, row-major.  K, R: row-major 3x3 doubles; D: 5 doubles (the
 * fisheye model reads D[0..3]); Kr = (fx, fy, cx, cy) of the rectified camera as the config gives them.  Returns 0, or -1
 * for a model other than 0 / 1, a size <= 0 or a singular K_rect * R (nothing is written then). */
CAM_H int rect_build_maps(int model, const double K[9], const double D[5], const double R[9], const double Kr[4], int rows,
                          int cols, float *map_x, float *map_y) {
    if ((model != CAM_PERSPECTIVE && model != CAM_FISHEYE) || rows <= 0 || cols <= 0) return -1;
    /* K_rect as cv::Mat_<float>, widened */
    const double A[9] = {(double)(float)Kr[0], 0.0, (double)(float)Kr[2], 0.0, (double)(float)Kr[1], (double)(float)Kr[3],
                         0.0, 0.0, 1.0};
    double AR[9], ir[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += A[3 * r + k] * R[3 * k + c];
            AR[3 * r + c] = s;
        }
    if (!rect_inv3(AR, ir)) return -1;
    const double fx = K[0], fy = K[4], u0 = K[2], v0 = K[5];
    if (model == CAM_PERSPECTIVE) {
        const double k1 = D[0], k2 = D[1], p1 = D[2], p2 = D[3], k3 = D[4];
        for (int i = 0; i < rows; ++i) {
            const double bx = i * ir[1] + ir[2], by = i * ir[4] + ir[5], bw = i * ir[7] + ir[8];
            for (int j = 0; j < cols; ++j) {
                const double _x = bx + j * ir[0], _y = by + j * ir[3], _w = bw + j * ir[6];
                const double w = 1. / _w, x = _x * w, y = _y * w;
                const double x2 = x * x, y2 = y * y;
                const double r2 = x2 + y2, _2xy = 2 * x * y;
                const double kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2;
                const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2);
                const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy;
                map_x[(long)i * cols + j] = (float)(fx * xd + u0);
                map_y[(long)i * cols + j] = (float)(fy * yd + v0);
            }
        }
    } else {
        const double k1 = D[0], k2 = D[1], k3 = D[2], k4 = D[3];
        for (int i = 0; i < rows; ++i) {
            double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
            for (int j = 0; j < cols; ++j) {
                double u, v;
                if (_w <= 0) {
                    u = (_x > 0) ? -HUGE_VAL : HUGE_VAL;
                    v = (_y > 0) ? -HUGE_VAL : HUGE_VAL;
                } else {
                    const double x = _x / _w, y = _y / _w;
                    const double r = sqrt(x * x + y * y);
                    const double theta = atan(r);
                    const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2,
                                 theta8 = theta4 * theta4;
                    const double theta_d = theta * (1 + k1 * theta2 + k2 * theta4 + k3 * theta6 + k4 * theta8);
                    const double scale = (r == 0) ? 1.0 : theta_d / r;
                    u = fx * x * scale + u0;
                    v = fy * y * scale + v0;
                }
                map_x[(long)i * cols + j] = (float)u;
                map_y[(long)i * cols + j] = (float)v;
                _x += ir[0];
                _y += ir[3];
                _w += ir[6];
            }
        }
    }
    return 0;
}

#endif
