// local_map_oracle.cc -- CPU restatement of frame::can_observe (data/frame.cc:797-824) as search_local_landmarks
// (tracking_module.cc:928-962) applies it, TEST INFRASTRUCTURE ONLY.  tests/local_map_data.py chains it with the oracle
// library's match_frame_and_landmarks and pose_optimize.  Compiled with -ffp-contract=off like the oracle library.
#include <stdint.h>

#include <cmath>

extern "C" {

struct lmo_camera {  // the layout of plp_camera
    double fx, fy, cx, cy, focal_x_baseline, true_baseline;
    float min_x, max_x, min_y, max_y;
    int32_t setup_type;
};

// data/landmark.cc:341-362 (float log of a float ratio, like the reference's std::log on floats)
static unsigned predict_scale_level(float max_valid_dist, float cam_to_lm_dist, float log_scale_factor, unsigned num_levels) {
    const float ratio = max_valid_dist / cam_to_lm_dist;
    const int pred = static_cast<int>(std::ceil(std::log(ratio) / log_scale_factor));
    if (pred < 0) return 0;
    if (num_levels <= static_cast<unsigned>(pred)) return num_levels - 1;
    return static_cast<unsigned>(pred);
}

// For each of the m landmarks at the pose T_cw (4 x 4 row-major): skip[i] (excluded or erased) -> 0, else
// can_observe(lm, 0.5): observable[i], the reprojection rounded to float and the predicted scale level (-1 if not
// observable).  gate_out (optional): 0 observable, 1 skipped, 2 reprojection, 3 distance, 4 viewing angle.
int lmo_can_observe(const lmo_camera *cam, const double *T, int m, const double *pos_w, const double *normal,
                    const float *min_d, const float *max_d, const float *max_raw, const uint8_t *skip,
                    float log_scale_factor, int num_levels, uint8_t *observable, float *reproj_x, float *reproj_y,
                    int32_t *level, int32_t *gate_out) {
    // frame.cc:750: cam_center_ = -R^T t
    double c[3];
    for (int r = 0; r < 3; ++r) c[r] = -(T[0 * 4 + r] * T[3] + T[1 * 4 + r] * T[7] + T[2 * 4 + r] * T[11]);
    int num = 0;
    for (int i = 0; i < m; ++i) {
        observable[i] = 0;
        reproj_x[i] = reproj_y[i] = 0.0f;
        level[i] = -1;
        int gate = 1;
        if (!skip || !skip[i]) {
            const double *X = pos_w + 3 * i;
            // camera::reproject_to_image (perspective.cc:190-209; fisheye.cc:231-250 is the same formula)
            const double pc0 = T[0] * X[0] + T[1] * X[1] + T[2] * X[2] + T[3];
            const double pc1 = T[4] * X[0] + T[5] * X[1] + T[6] * X[2] + T[7];
            const double pc2 = T[8] * X[0] + T[9] * X[1] + T[10] * X[2] + T[11];
            gate = 2;
            if (pc2 > 0.0) {
                const double z_inv = 1.0 / pc2;
                const double u = cam->fx * pc0 * z_inv + cam->cx;
                const double v = cam->fy * pc1 * z_inv + cam->cy;
                if (cam->min_x < u && u < cam->max_x && cam->min_y < v && v < cam->max_y) {
                    const double d0 = X[0] - c[0], d1 = X[1] - c[1], d2 = X[2] - c[2];
                    const double dist = std::sqrt(d0 * d0 + d1 * d1 + d2 * d2);
                    const float fdist = (float)dist;  // landmark::is_inside_in_orb_scale(const float)
                    gate = 3;
                    if (min_d[i] <= fdist && fdist <= max_d[i]) {
                        const double *n = normal + 3 * i;
                        const double ray_cos = (d0 * n[0] + d1 * n[1] + d2 * n[2]) / dist;
                        gate = 4;
                        if (!(ray_cos < 0.5)) {
                            gate = 0;
                            observable[i] = 1;
                            reproj_x[i] = (float)u;
                            reproj_y[i] = (float)v;
                            level[i] = (int32_t)predict_scale_level(max_raw[i], fdist, log_scale_factor, (unsigned)num_levels);
                            ++num;
                        }
                    }
                }
            }
        }
        if (gate_out) gate_out[i] = gate;
    }
    return num;
}

}  // extern "C"
