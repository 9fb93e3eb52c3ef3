/* oracle/camera.h -- camera::perspective / camera::fisheye undistortion, bearings and image bounds (TEST INFRASTRUCTURE
 * ONLY); see oracle.h.  The arithmetic is cammath.h. */
#ifndef PLP_ORACLE_CAMERA_H
#define PLP_ORACLE_CAMERA_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* K = config (fx, fy, cx, cy), D = config (k1, k2, p1, p2, k3) for model 0 (perspective) or (k1, k2, k3, k4, unused) for
 * model 1 (fisheye), both as the YAML doubles. */

/* perspective.cc:130-163 / fisheye.cc:172-204 undistort_keypoints on the points xy (n x 2 float) -> undist_xy (n x 2) */
void orc_undistort_keypoints(int model, const double *K, const double *D, const float *xy, int n, float *undist_xy);
/* perspective.cc:165-175 / fisheye.cc:205-215 convert_keypoints_to_bearings of the undistorted points -> n x 3 */
void orc_bearings(const double *K, const float *undist_xy, int n, double *bearings);
/* perspective.cc:100-127 / fisheye.cc:101-169 compute_image_bounds -> (min_x, max_x, min_y, max_y) */
void orc_image_bounds(int model, const double *K, const double *D, int cols, int rows, float *bounds);
#ifdef __cplusplus
}
#endif
#endif
