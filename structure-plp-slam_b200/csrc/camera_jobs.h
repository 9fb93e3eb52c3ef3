// camera_jobs.h -- job descriptor of the keypoint undistortion kernel (plain struct; shared by camera.cu, the tracker
// state of tracker.h and the device-code header that tests/cta_emu also compiles for the host).
#pragma once
#include <stdint.h>

#include "../../include/plpslam_b200.h"

namespace plp {

struct UndistJob {
    int model;
    double K[4];      // float-rounded fx, fy, cx, cy (cv::Mat_<float>) -- the undistortion
    double k[5];      // float-rounded coefficients
    double K_cfg[4];  // the config's doubles -- the bearings
    int batch, cap;   // frame b owns kp[b * cap, b * cap + n_kp[b])
    const plp_keypoint *kp;
    const int32_t *n_kp;  // NULL: every frame holds `cap` keypoints
    plp_keypoint *out;
    double *bearings;     // x 3; may be NULL
};

}  // namespace plp
