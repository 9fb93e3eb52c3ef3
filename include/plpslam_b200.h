/*
 * plpslam_b200.h -- C ABI of libplpslam_b200.so
 *
 * H100-native (sm_90a) replacement for the per-frame hot path of
 * Structure-PLP-SLAM.  The reference has no FFI: its "operator API" is the
 * public methods of a handful of C++ classes (SURVEY.md section 8(b)).  Each
 * entry point below names the reference method it replaces (file:line under
 * /root/reference/src/PLPSLAM).  The reference-side adapters that marshal
 * data::frame / data::keyframe into these PODs are shown in INTEGRATION.md and
 * shipped as headers under structure-plp-slam_b200/host/.
 *
 * Conventions
 *   - plain C types only, no exceptions cross this boundary; every function
 *     returns a plp_status and plp_last_error() gives the message;
 *   - "host" entry points take host pointers and perform the H2D/D2H copies
 *     themselves; "_dev" entry points take device pointers (already resident in
 *     HBM) and enqueue work on the context stream without synchronising;
 *   - there is NO CPU fallback: if no CUDA device is usable every compute entry
 *     point returns PLP_ERR_NO_DEVICE.
 *   - all batched entry points have the batch (frames / problems) as the
 *     leading dimension of every array.
 */
#ifndef PLPSLAM_B200_H
#define PLPSLAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLP_API __attribute__((visibility("default")))

typedef enum plp_status {
    PLP_OK = 0,
    PLP_ERR_INVALID = 1,   /* bad argument (null pointer, negative size, ...)      */
    PLP_ERR_NO_DEVICE = 2, /* no usable CUDA device -- never falls back to the CPU */
    PLP_ERR_CUDA = 3,      /* a CUDA runtime call failed, see plp_last_error()     */
    PLP_ERR_CAPACITY = 4,  /* an input exceeds the capacity the handle was made for */
    PLP_ERR_NCCL = 5
} plp_status;

/* ------------------------------------------------------------------------ */
/* context                                                                  */
/* ------------------------------------------------------------------------ */
typedef struct plp_ctx plp_ctx; /* one per (thread, device): stream + scratch */

PLP_API const char *plp_last_error(void);
PLP_API int plp_version(void);
PLP_API int plp_device_count(void);
PLP_API plp_status plp_ctx_create(int device, plp_ctx **out);
/* high_priority != 0: the context's stream gets the device's highest stream priority, so that its (small, latency-bound)
 * kernels are placed on the SMs ahead of the pending CTAs of normal-priority streams -- used to run the one-CTA-per-frame
 * matcher / pose optimiser of one sub-batch underneath the extraction kernels of the next. */
PLP_API plp_status plp_ctx_create_ex(int device, int high_priority, plp_ctx **out);
PLP_API void plp_ctx_destroy(plp_ctx *ctx);
PLP_API plp_status plp_ctx_sync(plp_ctx *ctx);
/* cudaStream_t of the context as an opaque pointer (for event timing by the harness) */
PLP_API void *plp_ctx_stream(plp_ctx *ctx);
/* device-memory helpers so that non-CUDA hosts (ctypes, cgo, ...) can keep data resident */
PLP_API plp_status plp_dev_alloc(plp_ctx *ctx, size_t bytes, void **out);
PLP_API plp_status plp_dev_free(plp_ctx *ctx, void *ptr);
PLP_API plp_status plp_dev_upload(plp_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
PLP_API plp_status plp_dev_download(plp_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
/* asynchronous variants (no synchronisation; the host buffer should be pinned) and a cross-context dependency: the
 * waiter's stream waits for everything enqueued so far on the other context's stream.  Two contexts on one device give
 * two streams: the copies and the low-occupancy kernels of one sub-batch overlap the compute of the other. */
PLP_API plp_status plp_dev_upload_async(plp_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
PLP_API plp_status plp_dev_download_async(plp_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
PLP_API plp_status plp_ctx_wait_ctx(plp_ctx *waiter, plp_ctx *other);
PLP_API plp_status plp_host_alloc_pinned(size_t bytes, void **out);
PLP_API plp_status plp_host_free_pinned(void *ptr);
/* number of kernels this library has launched since the context was created */
PLP_API uint64_t plp_ctx_launch_count(plp_ctx *ctx);
/* per-kernel device timing (CUDA events on the context stream around every launch); the report is a JSON object
 * {kernel_name: {count, total_ms}} of the launches since timing was enabled.  For measurement only. */
PLP_API plp_status plp_ctx_kernel_timing(plp_ctx *ctx, int enable);
PLP_API plp_status plp_ctx_kernel_timing_report(plp_ctx *ctx, char *buf, size_t buf_bytes);

/* ------------------------------------------------------------------------ */
/* 256-bit Hamming  (match/base.h:43-93)                                    */
/* ------------------------------------------------------------------------ */
#define PLP_HAMMING_DIST_THR_LOW 50   /* match/base.h:38 */
#define PLP_HAMMING_DIST_THR_HIGH 100 /* match/base.h:39 */
#define PLP_MAX_HAMMING_DIST 256      /* match/base.h:40 */

/* dist[i*nb + j] = popcount(a[i] xor b[j]) over 32-byte rows; replaces
 * compute_descriptor_distance_32/_64 (match/base.h:43-93) evaluated over a block. */
PLP_API plp_status plp_hamming_matrix(plp_ctx *ctx, const uint8_t *desc_a, int na,
                                      const uint8_t *desc_b, int nb, uint16_t *dist_out);

/* Exact 1-NN over 32-byte rows; replaces BinaryDescriptorMatcher::match(query, train, matches)
 * (feature/line_descriptor/binary_descriptor_matcher.cpp:197-254).  Ties resolve to the
 * lowest train index.  nn_idx[i] = -1 when nt == 0. */
PLP_API plp_status plp_hamming_nn(plp_ctx *ctx, const uint8_t *query, int nq, const uint8_t *train,
                                  int nt, int32_t *nn_idx, uint16_t *nn_dist);

/* ------------------------------------------------------------------------ */
/* frame features as the matchers see them                                   */
/* ------------------------------------------------------------------------ */
typedef struct plp_grid {
    /* camera::base grid (camera/base.h:91,147-160; camera/perspective.cc:53-56) */
    float min_x, min_y; /* img_bounds_.min_x_/min_y_ */
    double inv_cell_width, inv_cell_height;
    int32_t num_cols, num_rows; /* 64 x 48 */
} plp_grid;

typedef struct plp_frame_points {
    int32_t n;              /* frame::num_keypts_                                      */
    const float *x;         /* undist_keypts_[i].pt.x                                  */
    const float *y;         /* undist_keypts_[i].pt.y                                  */
    const int32_t *octave;  /* undist_keypts_[i].octave                                */
    const float *angle;     /* undist_keypts_[i].angle (deg); may be NULL if unused    */
    const float *x_right;   /* stereo_x_right_[i] (<0: monocular); NULL == all -1      */
    const uint8_t *desc;    /* descriptors_.row(i), n x 32                             */
    const uint8_t *claimed; /* landmarks_[i] && landmarks_[i]->has_observation(); NULL == none */
} plp_frame_points;

typedef struct plp_frame_lines {
    int32_t n;             /* frame::_num_keylines                                     */
    const float *sx, *sy;  /* _keylsd[i].getStartPoint()                               */
    const float *ex, *ey;  /* _keylsd[i].getEndPoint()                                 */
    const int32_t *octave; /* _keylsd[i].octave                                        */
    /* level the reference compares in the ratio test: it reads undist_keypts_[i].octave
     * (match/projection.cc:170,175 -- a point octave at a line index); the adapter passes
     * exactly that array so the behaviour is unchanged. */
    const int32_t *ratio_level;
    const float *x_right_sp, *x_right_ep; /* _stereo_x_right_cooresponding_to_keylines; NULL == none */
    const uint8_t *desc;                  /* _lbd_descr.row(i), n x 32                */
    const uint8_t *claimed;               /* _landmarks_line[i] && has_observation()   */
} plp_frame_lines;

typedef struct plp_camera {
    /* camera::perspective (camera/perspective.cc:40-56,190-209) */
    double fx, fy, cx, cy;
    double focal_x_baseline; /* bf; <= 0 for monocular */
    double true_baseline;
    float min_x, max_x, min_y, max_y; /* img_bounds_ */
    int32_t setup_type;               /* 0 Monocular, 1 Stereo, 2 RGBD (camera/base.h setup_type_t) */
} plp_camera;

typedef struct plp_distortion {
    /* Camera.model and its coefficients as the config gives them (the library rounds them to float, as the reference's
     * cv::Mat_<float> does): model 0 perspective, k = (k1, k2, p1, p2, k3); model 1 fisheye, k = (k1, k2, k3, k4, -). */
    int32_t model;
    double k[5];
} plp_distortion;


/* ------------------------------------------------------------------------ */
/* projection matchers (match/projection.cc)                                 */
/* ------------------------------------------------------------------------ */

/* projection::match_frame_and_landmarks (match/projection.cc:37-121).
 * One query per local landmark that passed frame::can_observe, in the order of
 * `local_landmarks`.  best_idx_out[q] = keypoint index written to frm.landmarks_ or -1.
 * Sequential "skip already claimed keypoints" semantics are reproduced exactly. */
typedef struct plp_landmark_queries {
    int32_t m;
    const float *reproj_x, *reproj_y; /* reproj_in_tracking_                    */
    const float *x_right;             /* x_right_in_tracking_                   */
    const int32_t *scale_level;       /* scale_level_in_tracking_               */
    const uint8_t *desc;              /* landmark::get_descriptor(), m x 32     */
    const uint8_t *valid;             /* is_observable_in_tracking_ && !will_be_erased(); NULL == all */
} plp_landmark_queries;

PLP_API plp_status plp_match_frame_and_landmarks(plp_ctx *ctx, const plp_frame_points *frm,
                                                 const plp_grid *grid, const float *scale_factors,
                                                 int num_levels, const plp_landmark_queries *q,
                                                 float margin, float lowe_ratio,
                                                 int32_t *best_idx_out, uint32_t *num_matches_out);

/* projection::match_current_and_last_frames (match/projection.cc:214-358).
 * Inputs are the last frame's keypoints that own a landmark: world position, octave, angle,
 * descriptor of the landmark; `valid` = lm != nullptr && !outlier_flags_.
 * matched_last_idx_out[n_curr]: index into the last-frame arrays assigned to each current
 * keypoint (curr_frm.landmarks_) after the orientation check, or -1. */
typedef struct plp_last_frame_points {
    int32_t n;
    const double *pos_w;   /* n x 3, lm->get_pos_in_world()               */
    const int32_t *octave; /* last_frm.keypts_[i].octave                  */
    const float *angle;    /* last_frm.undist_keypts_[i].angle            */
    const uint8_t *desc;   /* lm->get_descriptor(), n x 32                */
    const uint8_t *valid;  /* lm && !last_frm.outlier_flags_[i]           */
} plp_last_frame_points;

PLP_API plp_status plp_match_current_and_last_frames(
    plp_ctx *ctx, const plp_frame_points *curr, const plp_grid *grid, const float *scale_factors,
    int num_levels, const plp_camera *cam, const double *pose_cw_curr /*4x4 row-major*/,
    const double *pose_cw_last /*4x4 row-major*/, const plp_last_frame_points *last, float margin,
    int check_orientation, int32_t *matched_last_idx_out, uint32_t *num_matches_out);

/* projection::match_frame_and_landmarks_line (match/projection.cc:124-212) */
typedef struct plp_line_queries {
    int32_t m;
    const float *sp_x, *sp_y, *ep_x, *ep_y; /* _reproj_in_tracking_sp / _ep      */
    const int32_t *scale_level;             /* _scale_level_in_tracking          */
    const uint8_t *desc;
    const uint8_t *valid;
} plp_line_queries;

PLP_API plp_status plp_match_frame_and_landmarks_line(plp_ctx *ctx, const plp_frame_lines *frm,
                                                      const float *scale_factors_lsd,
                                                      int num_levels_lsd, const plp_line_queries *q,
                                                      float margin, float lowe_ratio,
                                                      int32_t *best_idx_out,
                                                      uint32_t *num_matches_out);

/* projection::match_current_and_last_frames_line (match/projection.cc:361-527) */
typedef struct plp_last_frame_lines {
    int32_t n;
    const double *pos_w;   /* n x 6, Line::get_pos_in_world(): (sp, ep)    */
    const int32_t *octave; /* last_frm._keylsd[i].octave                   */
    const uint8_t *desc;
    const uint8_t *valid; /* lm_line && !last_frm._outlier_flags_line[i]   */
} plp_last_frame_lines;

PLP_API plp_status plp_match_current_and_last_frames_line(
    plp_ctx *ctx, const plp_frame_lines *curr, const float *scale_factors_lsd, int num_levels_lsd,
    const plp_camera *cam, const double *pose_cw_curr, const double *pose_cw_last,
    const plp_last_frame_lines *last, float margin, int32_t *matched_last_idx_out,
    uint32_t *num_matches_out);

/* projection::match_frame_and_keyframe (match/projection.cc:529-645), the relocalisation matcher.  The adapter walks
 * keyfrm->get_landmarks() exactly like the reference and flattens one query per keyframe keypoint index: `valid` =
 * lm && !lm->will_be_erased() && !already_matched_lms.count(lm) && reprojected inside the image && inside
 * [0.7 min_valid_dist, 1.3 max_valid_dist] (:543-582); reproj = camera_->reproject_to_image; scale_level =
 * lm->predict_scale_level(cam_to_lm_dist, &curr_frm) (host libm logf, data/landmark.cc:319-340); q_angle =
 * keyfrm->undist_keypts_[idx].angle.  frm->claimed[i] = (curr_frm.landmarks_[i] != nullptr) (:604).  The window is
 * margin * scale_factors[level] over levels [level - 1, level + 1]; best Hamming <= hamm_dist_thr; keypoints are
 * claimed in query order; then the orientation histogram.  matched_kf_idx_out[n]: query index assigned to each
 * keypoint of the frame (curr_frm.landmarks_[i] = landmarks[idx]) or -1. */
PLP_API plp_status plp_match_frame_and_keyframe(plp_ctx *ctx, const plp_frame_points *frm, const plp_grid *grid,
                                                const float *scale_factors, int num_levels,
                                                const plp_landmark_queries *q, const float *q_angle, float margin,
                                                unsigned hamm_dist_thr, int check_orientation,
                                                int32_t *matched_kf_idx_out, uint32_t *num_matches_out);

/* projection::match_frame_and_keyframe_line (match/projection.cc:648-779): as above for line landmarks; `valid`
 * additionally encodes the partial-occlusion rule (:699-718: at least one end point, or the mid point, inside the
 * image); no orientation check. */
PLP_API plp_status plp_match_frame_and_keyframe_line(plp_ctx *ctx, const plp_frame_lines *frm,
                                                     const float *scale_factors_lsd, int num_levels_lsd,
                                                     const plp_line_queries *q, float margin, unsigned hamm_dist_thr,
                                                     int32_t *matched_kf_idx_out, uint32_t *num_matches_out);

/* robust::brute_force_match (match/robust.cc:257-385).
 * frame = "1", keyframe = "2".  kf_valid[j] = lm_2 && !lm_2->will_be_erased().
 * matched_kf_idx_in_frm_out[n_frm] = matched_indices_2_in_1 after the orientation check. */
PLP_API plp_status plp_match_brute_force(plp_ctx *ctx, const uint8_t *frm_desc,
                                         const float *frm_angle, int n_frm,
                                         const uint8_t *kf_desc, const float *kf_angle,
                                         const uint8_t *kf_valid, int n_kf, float lowe_ratio,
                                         int check_orientation, int32_t *matched_kf_idx_in_frm_out,
                                         uint32_t *num_matches_out);

/* ------------------------------------------------------------------------ */
/* ORB extraction  (feature/orb_extractor.{h,cc})                            */
/* ------------------------------------------------------------------------ */
typedef struct plp_orb_params { /* feature/orb_params.h:39-70 */
    uint32_t max_num_keypts;
    float scale_factor;
    uint32_t num_levels;
    uint32_t ini_fast_thr;
    uint32_t min_fast_thr;
} plp_orb_params;

typedef struct plp_keypoint { /* binary layout of cv::KeyPoint (28 bytes) */
    float x, y;               /* pt */
    float size, angle, response;
    int32_t octave, class_id;
} plp_keypoint;

/* camera::{perspective,fisheye}::compute_image_bounds (perspective.cc:100-127, fisheye.cc:101-169) of cam's fx, fy, cx, cy
 * (host computation): bounds_out = (min_x, max_x, min_y, max_y), the img_bounds_ of plp_camera and of the grid. */
PLP_API plp_status plp_camera_image_bounds(const plp_camera *cam, const plp_distortion *dist, int cols, int rows,
                                           float bounds_out[4]);
/* undistort_keypoints + convert_keypoints_to_bearings (perspective.cc:130-175, fisheye.cc:172-215).  Host pointers.
 * undist_out[i] = kp[i] with pt undistorted (cv::undistortPoints / cv::fisheye::undistortPoints); angle, size and octave
 * copied, response 0, class_id -1.  bearings_out (n x 3) may be NULL.  n == 0 -> PLP_OK. */
PLP_API plp_status plp_undistort_keypoints(plp_ctx *ctx, const plp_camera *cam, const plp_distortion *dist,
                                           const plp_keypoint *kp, int n, plp_keypoint *undist_out, double *bearings_out);
/* Device-resident batched form for the layout plp_orb_extract_batch_dev writes: frame b owns d_kp[b * cap ..] with
 * d_n_kp[b] keypoints.  Writes d_undist_out (batch x cap) and, when not NULL, d_bearings_out (batch x cap x 3); slots past
 * a frame's count are left untouched.  No synchronisation. */
PLP_API plp_status plp_undistort_keypoints_batch_dev(plp_ctx *ctx, const plp_camera *cam, const plp_distortion *dist,
                                                     int batch, int cap, const plp_keypoint *d_kp, const int32_t *d_n_kp,
                                                     plp_keypoint *d_undist_out, double *d_bearings_out);

/* util::stereo_rectifier (util/stereo_rectifier.cc:39-92): the StereoRectifier.* config keys and the rectified camera. */
typedef struct plp_stereo_rectifier_params {
    int32_t model;  /* StereoRectifier.model: 0 perspective, D = (k1, k2, p1, p2, k3); 1 fisheye, D = (k1, k2, k3, k4, -) */
    double K_left[9], D_left[5], R_left[9];    /* row-major, as the config lists them */
    double K_right[9], D_right[5], R_right[9];
    double fx, fy, cx, cy; /* Camera.fx ... of the rectified camera (rounded to float, like cv_cam_matrix_) */
} plp_stereo_rectifier_params;
typedef struct plp_stereo_rectifier plp_stereo_rectifier;

/* The constructor: both sides' maps (cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap, CV_32F) for a
 * rows x cols camera, kept on ctx's device.  PLP_ERR_INVALID for a model other than 0 / 1, a size <= 0 or a singular
 * K_rect * R.  The rectifier may be used with any context on the same device. */
PLP_API plp_status plp_stereo_rectifier_create(plp_ctx *ctx, const plp_stereo_rectifier_params *params, int rows, int cols,
                                               plp_stereo_rectifier **out);
PLP_API void plp_stereo_rectifier_destroy(plp_stereo_rectifier *r);
/* stereo_rectifier::rectify: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of both host images (rows x cols, row stride
 * step) into left_out / right_out (row stride out_step).  Synchronous. */
PLP_API plp_status plp_stereo_rectify(plp_ctx *ctx, const plp_stereo_rectifier *r, const uint8_t *left, const uint8_t *right,
                                      size_t step, uint8_t *left_out, uint8_t *right_out, size_t out_step);
/* Device-resident batch of one side (0 left, 1 right): frame b is read from d_in + b * rows * in_step and written to
 * d_out + b * rows * out_step, only the first cols bytes of each row.  d_out and out_step must be multiples of 16, so d_out
 * is a level 0 plp_orb_extract_batch_dev reads as it is.  Enqueued on ctx's stream, no synchronisation. */
PLP_API plp_status plp_stereo_rectify_batch_dev(plp_ctx *ctx, const plp_stereo_rectifier *r, int side, const uint8_t *d_in,
                                                int batch, size_t in_step, uint8_t *d_out, size_t out_step);
/* The float maps of one side (host copies, rows x cols each). */
PLP_API plp_status plp_stereo_rectifier_maps(const plp_stereo_rectifier *r, int side, float *map_x, float *map_y);

typedef struct plp_image_view { /* one pyramid level, device memory */
    const uint8_t *data;
    int32_t rows, cols;
    size_t step;
} plp_image_view;

typedef struct plp_orb plp_orb; /* one per orb_extractor instance (never re-entered, frame.cc:456-457) */

/* orb_extractor::orb_extractor(const orb_params&) (orb_extractor.cc:66-71, initialize() :235-287).
 * The handle is specialised for one image size and a maximum batch of frames. */
PLP_API plp_status plp_orb_create(plp_ctx *ctx, const plp_orb_params *params, int rows, int cols,
                                  int max_batch, plp_orb **out);
PLP_API void plp_orb_destroy(plp_orb *orb);
/* keypoint capacity per frame of the output arrays (the quadtree may exceed max_num_keypts, see DESIGN.md) */
PLP_API int plp_orb_capacity(const plp_orb *orb);
/* orb_extractor::get_scale_factors / get_inv_scale_factors / get_level_sigma_sq / get_inv_level_sigma_sq
 * (orb_extractor.cc:215-233); each array has num_levels entries. */
PLP_API plp_status plp_orb_get_tables(const plp_orb *orb, float *scale_factors, float *inv_scale_factors,
                                      float *level_sigma_sq, float *inv_level_sigma_sq,
                                      uint32_t *num_keypts_per_level);

/* orb_extractor::extract(in_image, in_image_mask, keypts, out_descriptors) (orb_extractor.cc:73-160).
 * Host pointers.  mask may be NULL (image mask or the rectangle mask of orb_extractor.cc:297-313, which the
 * adapter rasterises exactly like the reference).  Empty image (rows*cols == 0 or img == NULL) -> *n_out = 0,
 * PLP_OK, like the silent return at orb_extractor.cc:76-79.  kp_out/desc_out must hold plp_orb_capacity()
 * entries. */
PLP_API plp_status plp_orb_extract(plp_orb *orb, const uint8_t *img, int rows, int cols, size_t step,
                                   const uint8_t *mask, size_t mask_step, plp_keypoint *kp_out,
                                   uint8_t *desc_out, int *n_out);
/* Same for a batch of `batch` equally sized frames stored back to back (frame stride rows*step). */
PLP_API plp_status plp_orb_extract_batch(plp_orb *orb, const uint8_t *imgs, int batch, size_t step,
                                         plp_keypoint *kp_out, uint8_t *desc_out, int32_t *n_out);
/* Device-resident variant: d_imgs (batch x rows x step) stays in HBM; results are written to device arrays
 * of batch x capacity entries; no synchronisation.  d_status[b] != 0 flags a capacity overflow in frame b. */
PLP_API plp_status plp_orb_extract_batch_dev(plp_orb *orb, const uint8_t *d_imgs, int batch, size_t step,
                                             plp_keypoint *d_kp_out, uint8_t *d_desc_out,
                                             int32_t *d_n_out, int32_t *d_status);
/* orb_extractor::image_pyramid_ (orb_extractor.h:101) of frame b of the most recent extraction. */
PLP_API plp_status plp_orb_get_pyramid(const plp_orb *orb, int b, int level, plp_image_view *out);
/* debug/parity taps of the most recent extraction (host copies): FAST candidates of one level in the
 * reference's cell order, coordinates relative to the 19-px border (orb_extractor.cc:424-434). */
PLP_API plp_status plp_orb_debug_candidates(plp_orb *orb, int b, int level, plp_keypoint *out, int cap,
                                            int *n_out);
/* The blurred level (cv::GaussianBlur 7x7, sigma 2, BORDER_REFLECT_101) the descriptors of frame b of the most recent
 * extraction sample, copied densely into out (rows x cols of that level, as plp_orb_get_pyramid reports them). */
PLP_API plp_status plp_orb_debug_blurred(plp_orb *orb, int b, int level, uint8_t *out);

/* robust::match_for_triangulation (match/robust.cc:43-216): for every landmark-free keypoint of keyframe 1 (visited in
 * the order of its BoW feature vector: ascending node id, then the node's index list) the landmark-free, not yet taken
 * keypoint of keyframe 2 in the SAME BoW node with the smallest Hamming distance <= 50 (ties: the later one in the
 * node's list) that is not within 3 deg of the epipole (monocular pairs only, :150-161) and satisfies the epipolar
 * constraint of E_12 within 0.2 deg x scale_factors_1[octave_1] (robust.cc:387-406); then the orientation histogram.
 * The feature vectors are DBoW2::FeatureVector / fbow::BoWFeatVector flattened in iteration order (node ids ascending).
 * epipole_bearing_in_2 = camera_->reproject_to_bearing(rot_2w, trans_2w, cam_center_1) (:54-57).
 * matched_idx2_in_1_out[n1] = matched_indices_2_in_keyfrm_1 after the orientation check (-1: none); the adapter turns
 * it into matched_idx_pairs in ascending idx_1 order (:201-213). */
typedef struct plp_keyframe_points {
    int32_t n;                   /* keyframe::num_keypts_                                            */
    const uint8_t *desc;         /* descriptors_, n x 32                                             */
    const float *angle;          /* undist_keypts_[i].angle (may be NULL without orientation check)  */
    const int32_t *octave;       /* undist_keypts_[i].octave (used for keyframe 1 only)              */
    const double *bearings;      /* bearings_, n x 3                                                 */
    const uint8_t *has_landmark; /* get_landmarks()[i] != nullptr                                    */
    const float *x_right;        /* stereo_x_right_ (NULL == monocular)                              */
} plp_keyframe_points;

typedef struct plp_bow_feature_vector {
    int32_t num_nodes;
    const uint32_t *node_ids; /* ascending                            */
    const int32_t *offsets;   /* num_nodes + 1, into indices          */
    const uint32_t *indices;  /* keypoint indices of each node        */
} plp_bow_feature_vector;

PLP_API plp_status plp_match_for_triangulation(plp_ctx *ctx, const plp_keyframe_points *kf1,
                                               const plp_keyframe_points *kf2, const plp_bow_feature_vector *fv1,
                                               const plp_bow_feature_vector *fv2, const double *E_12 /*3x3 row-major*/,
                                               const double *epipole_bearing_in_2 /*3*/, const float *scale_factors_1,
                                               int num_levels, int check_orientation,
                                               int32_t *matched_idx2_in_1_out, uint32_t *num_matches_out);

/* landmark::compute_descriptor / Line::compute_descriptor (data/landmark.cc:181-247, data/landmark_line.cc:215-283) for
 * a batch of landmarks (the mapping thread calls it for every landmark touched by a new keyframe or a fuse,
 * mapping_module.cc:704,756): descs holds the observation descriptors of landmark l at rows offsets[l] .. offsets[l+1];
 * best_idx_out[l] = local index of the observation whose median Hamming distance to all observations
 * (element floor(0.5 (k - 1)) of the sorted row) is smallest, first one on ties; -1 for a landmark without observations
 * (the reference returns without touching descriptor_). */
PLP_API plp_status plp_landmark_compute_descriptor_batch(plp_ctx *ctx, const uint8_t *descs, const int32_t *offsets,
                                                         int num_landmarks, int32_t *best_idx_out);

/* ------------------------------------------------------------------------ */
/* fuse matchers  (match/fuse.{h,cc})                                        */
/* ------------------------------------------------------------------------ */
/* match::fuse::replace_duplication / detect_duplication / replace_duplication_line (match/fuse.cc:40-151, 153-300,
 * 304-503), the step after triangulation in mapping_module::fuse_landmark_duplication[_line] (mapping_module.cc:701-812)
 * and in the loop corrector (global_optimization_module.cc:632, detect_duplication with the corrected Sim3).
 *
 * In the reference every landmark's search -- reprojection into the target keyframe, visibility / distance / viewing-
 * angle gates, predict_scale_level, the window query, the level and chi-square gates and the best Hamming distance
 * <= HAMMING_DIST_THR_LOW (ties: first in get_keypoints_in_cell order) -- reads only the landmark and the keyframe's
 * features, never the state written by earlier landmarks (there is no "claimed" skip in fuse.cc).  Only the EFFECT
 * (add_observation / replace, :265-296) is sequential.  The entry points therefore return best_idx for every
 * (target keyframe, landmark) pair of a batch -- mapping_module.cc:711-714 is `num_targets` keyframes x one landmark
 * list, :749 is one keyframe x the united landmark list -- and the adapter applies the effects in the reference's order,
 * re-checking will_be_erased() / is_observed_in_keyframe() at apply time and re-issuing the search for landmarks whose
 * descriptor was recomputed by landmark::replace (data/landmark.cc:429) before the remaining targets (INTEGRATION.md).
 *
 * predict_scale_level (data/landmark.cc:341-362) = clamp(ceil(logf(max_valid_dist_ / dist) / log_scale_factor)) is
 * evaluated on the device as a comparison of the float ratio against num_levels - 1 thresholds that the library derives
 * on the host from the caller's libm logf (smallest float r with logf(r) / log_scale_factor > k), so the level is the
 * host's, bit for bit, for every ratio. */
typedef struct plp_fuse_landmarks { /* landmarks_to_check in the caller's iteration order */
    int32_t m;
    const double *pos_w;             /* get_pos_in_world(): m x 3 (points) or m x 6 (lines: sp, ep)             */
    const double *obs_mean_normal;   /* get_obs_mean_normal(), m x 3 (points only; NULL for lines)               */
    const float *min_valid_dist;     /* get_min_valid_distance() (0.7 / 0.8 x min_valid_dist_)                   */
    const float *max_valid_dist;     /* get_max_valid_distance() (1.3 / 1.2 x max_valid_dist_)                   */
    const float *max_valid_dist_raw; /* max_valid_dist_, the numerator of predict_scale_level                    */
    const uint8_t *desc;             /* get_descriptor(), m x 32                                                  */
    const uint8_t *valid;            /* lm && !lm->will_be_erased(); NULL == all                                  */
} plp_fuse_landmarks;

typedef struct plp_fuse_target_points {
    plp_frame_points pts; /* keyfrm->undist_keypts_ (x, y, octave), stereo_x_right_, descriptors_; angle/claimed unused */
    double rot_cw[9];     /* keyfrm->get_rotation() (or the Sim3 rotation / s, fuse.cc:46-49), row-major            */
    double trans_cw[3];   /* keyfrm->get_translation() (or Sim3 translation / s)                                    */
    double cam_center[3]; /* keyfrm->get_cam_center() (or -rot_cw^T trans_cw)                                        */
    const uint8_t *skip;  /* m entries: lm->is_observed_in_keyframe(keyfrm) / valid_lms_in_keyfrm.count(lm); NULL == none */
} plp_fuse_target_points;

typedef struct plp_fuse_target_lines {
    plp_frame_lines lines; /* keyfrm->_keylsd (sx, sy, ex, ey, octave), _lbd_descr; the other members unused */
    double rot_cw[9], trans_cw[3], cam_center[3];
    const uint8_t *skip;
} plp_fuse_target_lines;

#define PLP_FUSE_DETECT 0  /* detect_duplication: signed level gate [pred - 1, pred], no chi-square gate (fuse.cc:113-121) */
#define PLP_FUSE_REPLACE 1 /* replace_duplication: unsigned level gate (pred == 0 rejects every candidate, :228-236),
                              chi-square gate 5.99146 / 7.81473 on the reprojection error (:238-266)                 */

/* best_idx_out[t * lms->m + i] = keypoint index of target t matched to landmark i, or -1 (any `continue` of the
 * reference loop body).  best_dist_out (optional, same shape) = its Hamming distance, 0xFFFF when unmatched. */
PLP_API plp_status plp_fuse_search_points(plp_ctx *ctx, const plp_fuse_target_points *targets, int num_targets,
                                          const plp_grid *grid, const plp_camera *cam, const float *scale_factors,
                                          const float *inv_level_sigma_sq, int num_levels, float log_scale_factor,
                                          const plp_fuse_landmarks *lms, float margin, int mode, int32_t *best_idx_out,
                                          uint16_t *best_dist_out);
/* replace_duplication_line (fuse.cc:304-503): candidates = get_keylines_in_cell over all keylines (both end points
 * within margin x _scale_factors_lsd[pred] of the reprojected line), chi-square gate 5.99146 on the two point-to-line
 * errors, best LBD Hamming distance <= 50 (ties: smallest keyline index). */
PLP_API plp_status plp_fuse_search_lines(plp_ctx *ctx, const plp_fuse_target_lines *targets, int num_targets,
                                         const plp_camera *cam, const float *scale_factors_lsd,
                                         const float *inv_level_sigma_sq_lsd, int num_levels_lsd,
                                         float log_scale_factor_lsd, const plp_fuse_landmarks *lms, float margin,
                                         int32_t *best_idx_out, uint16_t *best_dist_out);

/* Parity tap (host only, no device work): thr_out[k], 1 <= k < num_levels, is the smallest float ratio whose
 * predict_scale_level is >= k under the calling process's libm logf; thr_out[0] is unused (set to 0).  The kernels
 * evaluate predict_scale_level as count(ratio >= thr[k]). */
PLP_API plp_status plp_fuse_level_thresholds(float log_scale_factor, int num_levels, float *thr_out);

/* ------------------------------------------------------------------------ */
/* BoW: vocabulary tree transform and match::bow_tree  (data/frame.cc:785-795, */
/* match/bow_tree.{h,cc})                                                     */
/* ------------------------------------------------------------------------ */
/* The DBoW2 vocabulary (data/bow_vocabulary.h:40) on the device.  plp_bow_vocab_load reads the binary file the reference
 * loads with bow_vocab_->loadFromBinaryFile (system.cc:82; orb_vocab/orb_vocab.dbow2: header {u32 n_nodes, u32 node_size
 * = 41, i32 k, i32 L, i32 scoring, i32 weighting}, then n_nodes - 1 records {i32 parent, u8 descriptor[32], f32 weight,
 * u8 is_leaf}; node 0 is the root, children are ordered by node id, words are numbered in file order).
 * plp_bow_vocab_create takes the same records as arrays (entry i describes node i + 1). */
typedef struct plp_bow_vocab plp_bow_vocab;
PLP_API plp_status plp_bow_vocab_create(plp_ctx *ctx, int k, int L, int num_nodes, const int32_t *parent,
                                        const uint8_t *desc, const float *weight, const uint8_t *is_leaf,
                                        plp_bow_vocab **out);
PLP_API plp_status plp_bow_vocab_load(plp_ctx *ctx, const char *path, plp_bow_vocab **out);
PLP_API void plp_bow_vocab_destroy(plp_bow_vocab *v);
PLP_API plp_status plp_bow_vocab_info(const plp_bow_vocab *v, int32_t *k, int32_t *L, int32_t *num_nodes,
                                      int32_t *num_words);
/* frame::compute_bow / keyframe::compute_bow (data/frame.cc:785-795): TemplatedVocabulary::transform(features, bow_vec,
 * bow_feat_vec, levelsup = 4).  Per descriptor row: the word reached by descending the tree along the child with the
 * smallest Hamming distance (first child on ties), its weight, and the id of the node passed at level L - levelsup.
 * The adapter folds the rows into the two std::maps exactly like DBoW2: rows with weight > 0 only,
 * bow_vec[word_id] += weight in row order then L1-normalised over ascending word ids, bow_feat_vec[node_id].push_back(row). */
PLP_API plp_status plp_bow_transform(plp_bow_vocab *v, const uint8_t *desc, int n, int levelsup, int32_t *word_id_out,
                                     int32_t *node_id_out, float *weight_out);
/* Device-resident variant for the batched front end (rows = batch x plp_orb_capacity(), rows past a frame's keypoint
 * count are computed and ignored by the caller); runs on the vocabulary context's stream, no synchronisation. */
PLP_API plp_status plp_bow_transform_dev(plp_bow_vocab *v, const uint8_t *d_desc, int n, int levelsup,
                                         int32_t *d_word_id_out, int32_t *d_node_id_out, float *d_weight_out);

/* match::bow_tree::match_frame_and_keyframe (match/bow_tree.cc:41-165): side 1 = the keyframe (valid = lm &&
 * !lm->will_be_erased()), side 2 = the frame (valid = NULL); match::bow_tree::match_keyframes (:167-305): side 1 =
 * keyfrm_1, side 2 = keyfrm_2, both with valid flags.  For every node id present in both feature vectors, every valid
 * side-1 keypoint of the node (in list order) takes the not-yet-taken valid side-2 keypoint OF THE SAME NODE with the
 * smallest Hamming distance (first on ties) if it is <= 50 and passes lowe_ratio against the second smallest; then the
 * orientation histogram.  A keypoint index may appear in at most one node of a feature vector (true for DBoW2's
 * transform), which makes the nodes independent: one warp per node, sequential inside the node.  A call takes a batch
 * of pairs (module/relocalizer.cc:79: one frame x every relocalisation candidate; module/loop_detector.cc:356: the current
 * keyframe x every loop candidate; module/frame_tracker.cc:130-139: one pair). */
typedef struct plp_bow_side {
    int32_t n;            /* num_keypts_                                       */
    const uint8_t *desc;  /* descriptors_, n x 32                              */
    const float *angle;   /* keypts_[i].angle; NULL without orientation check  */
    const uint8_t *valid; /* see above; NULL == all                            */
    plp_bow_feature_vector fv; /* bow_feat_vec_ flattened in iteration order   */
} plp_bow_side;

typedef struct plp_bow_pair {
    const plp_bow_side *side1, *side2;
    int32_t *matched_2_of_1_out; /* side1->n entries or NULL: index on side 2 matched to each side-1 keypoint, -1 none */
    int32_t *matched_1_of_2_out; /* side2->n entries or NULL (matched_lms_in_frm[i] = keyfrm_lms[matched_1_of_2[i]])   */
    uint32_t num_matches;        /* out */
} plp_bow_pair;

PLP_API plp_status plp_match_bow_tree(plp_ctx *ctx, plp_bow_pair *pairs, int num_pairs, float lowe_ratio,
                                      int check_orientation);

/* ------------------------------------------------------------------------ */
/* essential-matrix RANSAC  (solve/essential_solver.{h,cc})                  */
/* ------------------------------------------------------------------------ */
/* solve::essential_solver::find_via_ransac(max_num_iter, recompute) (solve/essential_solver.cc:37-121), the inlier filter
 * of robust::match_frame_and_keyframe (match/robust.cc:218-255: brute_force_match, then find_via_ransac(50, false)).
 * matches_12[i] = {index into bearings_1, index into bearings_2}.  `samples` holds the num_iter x 8 match indices the
 * reference draws with util::create_random_array(8, 0, num_matches - 1) per iteration (the reference seeds a fresh
 * mt19937 from std::random_device each time, util/random_array.cc:37-44, so its result is not reproducible; with the
 * samples as an input the result is a deterministic function of them).  All num_iter hypotheses are evaluated
 * concurrently (one CTA each: eight-point solve, inlier test over all matches, score summed in match order); the first
 * hypothesis with the largest score wins exactly like the reference's sequential `best_score_ < score_in_sac` scan.
 * Outputs: is_inlier_out[num_matches], best_E_21_out[9] (row-major), *best_score_out, *solution_is_valid_out
 * (best_score > 0 and >= 8 inliers; with fewer than 8 matches: 0 and nothing else is touched, :45-49).
 * The two Eigen::JacobiSVD calls of compute_E_21 are restated with cyclic Jacobi rotations (csrc/essmath.h). */
PLP_API plp_status plp_essential_ransac(plp_ctx *ctx, const double *bearings_1, int n1, const double *bearings_2, int n2,
                                        const int32_t *matches_12, int num_matches, const int32_t *samples,
                                        int num_iter, int recompute, uint8_t *is_inlier_out, double *best_E_21_out,
                                        double *best_score_out, int32_t *solution_is_valid_out);

/* ------------------------------------------------------------------------ */
/* plane RANSAC  (planar_mapping_module.{h,cc})                              */
/* ------------------------------------------------------------------------ */
/* Planar_Mapping_module::estimate_plane_sequential_RANSAC (planar_mapping_module.cc:412-591, mode 0) and
 * update_plane_via_RANSAC (:593-733, mode 1) with estimate_plane_SVD (:735-771): the landmarks linked to one plane
 * instance, `num_iter` hypotheses.  The random index draws are an input (num_iter x sample_size indices, drawn by the
 * adapter exactly like :447-457 / :620-632; the reference seeds its mt19937 from std::random_device).  Every hypothesis
 * (sample fit, inlier test of all landmarks, refit on the inliers) is evaluated by its own CTA; the reference's
 * sequential bookkeeping -- best_error also drops to a SAMPLE residual (:461-464), the Plane object takes the sample fit
 * of every iteration (:465-467), early exit of mode 0 (:526-534) -- is replayed over the results in iteration order, and
 * step [4] filters the best inlier list with the equation the Plane holds at the end.
 * valid[j] = !lms[j]->will_be_erased() (NULL == all).  eq_inout / plane_error_inout: the Plane's equation and
 * best_error_ before and after the call (they are mutated every iteration, also when the call fails).
 * inlier_out[j] = 1 for the landmarks the plane keeps.  *status_out: 1 = true, 0 = false, 2 = false + set_invalid().
 * Eigen::JacobiSVD is restated with cyclic Jacobi rotations on the 3 x 3 scatter matrix (csrc/planemath.h); the sign of
 * the plane normal is arbitrary in both. */
typedef struct plp_plane_ransac_cfg {
    int32_t mode;              /* 0 estimate_plane_sequential_RANSAC, 1 update_plane_via_RANSAC */
    int32_t points_per_ransac; /* POINTS_PER_RANSAC */
    double planar_distance_thresh, final_error_thresh, inliers_ratio_thr;
    double initial_best_error; /* mode 1: plane->get_best_error() (:609) */
} plp_plane_ransac_cfg;
PLP_API plp_status plp_plane_ransac(plp_ctx *ctx, const double *pos_w, const uint8_t *valid, int n,
                                    const int32_t *samples, int num_iter, int sample_size,
                                    const plp_plane_ransac_cfg *cfg, double *eq_inout /*4*/, double *plane_error_inout,
                                    uint8_t *inlier_out, int32_t *status_out);

/* ------------------------------------------------------------------------ */
/* stereo matching  (match/stereo.{h,cc})                                    */
/* ------------------------------------------------------------------------ */
/* match::stereo::compute(stereo_x_right, depths) (match/stereo.cc:45-150): per left keypoint the Hamming-closest right
 * keypoint in the row band (+-2 * scale), octave +-1 and disparity range [0, focal_x_baseline / true_baseline), best
 * distance < (100 + 50) / 2; 11 x 11 L1 patch slide over +-5 px at the keypoint's octave with parabola refinement;
 * matches whose patch correlation exceeds twice the median are dropped.  The image pyramids are the ones the two
 * extractors hold from their most recent extraction (orb_extractor::image_pyramid_, passed by frame.cc:475).
 * Outputs have one entry per left keypoint (-1 = no stereo match), like the vectors the reference resizes at :51-52.
 * best_right_out (optional parity tap): index of the Hamming-closest right keypoint before the sub-pixel stage. */
PLP_API plp_status plp_stereo_compute(plp_ctx *ctx, const plp_orb *left, const plp_orb *right,
                                      const plp_keypoint *kp_left, const uint8_t *desc_left, int n_left,
                                      const plp_keypoint *kp_right, const uint8_t *desc_right, int n_right,
                                      float focal_x_baseline, float true_baseline, float *stereo_x_right_out,
                                      float *depths_out, int32_t *best_right_out);
/* Device-resident batched variant: the arrays are the outputs of plp_orb_extract_batch_dev of the two handles
 * (batch x plp_orb_capacity() entries); no synchronisation. */
PLP_API plp_status plp_stereo_compute_batch_dev(plp_ctx *ctx, const plp_orb *left, const plp_orb *right, int batch,
                                                const plp_keypoint *d_kp_left, const uint8_t *d_desc_left,
                                                const int32_t *d_n_left, const plp_keypoint *d_kp_right,
                                                const uint8_t *d_desc_right, const int32_t *d_n_right,
                                                float focal_x_baseline, float true_baseline,
                                                float *d_stereo_x_right_out, float *d_depths_out,
                                                int32_t *d_best_right_out);

/* ------------------------------------------------------------------------ */
/* LSD + LBD line extraction  (feature/line_extractor.{h,cc},                */
/* feature/line_descriptor/{LSDDetector_custom,binary_descriptor_custom}.cpp) */
/* ------------------------------------------------------------------------ */
typedef struct plp_keyline { /* binary layout of cv::line_descriptor::KeyLine (descriptor_custom.hpp:105-199, 68 bytes) */
    float angle;             /* atan2(endPointY - startPointY, endPointX - startPointX)        */
    int32_t class_id;        /* running index over the segments longer than min_length          */
    int32_t octave;          /* always 0: the reference detects on one octave (line_extractor.cc:54) */
    float pt_x, pt_y;        /* midpoint                                                        */
    float response;          /* lineLength / max(cols, rows)                                    */
    float size;
    float start_x, start_y, end_x, end_y;
    float s_oct_x, s_oct_y, e_oct_x, e_oct_y;
    float line_length;
    int32_t num_pixels;      /* cv::LineIterator count                                          */
} plp_keyline;

typedef struct plp_line plp_line; /* one per LineFeatureTracker instance; fixed image size and maximum batch */

/* LineFeatureTracker::LineFeatureTracker(camera::base*) (line_extractor.cc:50-58); LSD options are the ones
 * extract_LSD_LBD hard-codes (line_extractor.cc:113-122): refine 1, scale 0.5, sigma_scale 0.6, quant 2, ang_th 22.5,
 * log_eps 1, density_th 0.6, n_bins 1024, min_length 0.125 * min(cols, rows). */
PLP_API plp_status plp_line_create(plp_ctx *ctx, int rows, int cols, int max_batch, plp_line **out);
PLP_API void plp_line_destroy(plp_line *h);
/* keyline capacity per frame of the output arrays */
PLP_API int plp_line_capacity(const plp_line *h);
/* LineFeatureTracker::extract_LSD_LBD(img, frame_keylsd, frame_lbd_descr, keyline_functions) (line_extractor.cc:88-160).
 * Host pointers.  kl_out / lbd_out (x 32 bytes) / fn_out (x 3 doubles: the 2-D line function sp x ep / |(l0, l1)|,
 * line_extractor.cc:147-159) must hold plp_line_capacity() entries.  The identity remap the reference rebuilds every
 * frame (line_extractor.cc:60-86, 103) returns the input bit for bit and is skipped.  An image without a segment
 * longer than min_length yields *n_out = 0. */
PLP_API plp_status plp_line_extract(plp_line *h, const uint8_t *img, int rows, int cols, size_t step,
                                    plp_keyline *kl_out, uint8_t *lbd_out, double *fn_out, int *n_out);
/* Same for `batch` equally sized frames stored back to back (frame stride rows*step). */
PLP_API plp_status plp_line_extract_batch(plp_line *h, const uint8_t *imgs, int batch, size_t step,
                                          plp_keyline *kl_out, uint8_t *lbd_out, double *fn_out, int32_t *n_out);
/* Device-resident variant: no synchronisation; d_status[b] != 0 flags a capacity overflow in frame b. */
PLP_API plp_status plp_line_extract_batch_dev(plp_line *h, const uint8_t *d_imgs, int batch, size_t step,
                                              plp_keyline *d_kl_out, uint8_t *d_lbd_out, double *d_fn_out,
                                              int32_t *d_n_out, int32_t *d_status);
/* parity taps of the most recent extraction (host copies): the raw cv::LineSegmentDetector segments of frame b
 * (x1, y1, x2, y2 in detection order), the half-resolution image LSD works on, and the 72-float LBD vectors. */
PLP_API plp_status plp_line_debug_segments(plp_line *h, int b, float *segs_out, int cap, int *n_out);
/* the region-growing kernel keeps the half-resolution image in shared memory for batches that fit the resident frames
 * (2 per SM at VGA) and reads it through L2 for larger batches (6 frames per SM); this forces the second variant so that
 * the parity tests cover both */
PLP_API plp_status plp_line_debug_force_global_image(plp_line *h, int on);
/* region growing variant: 0 automatic (multi-warp rounds for at most half a wave of frames, out of order for a live frame through
 * the host entry point), 1 one warp
 * per frame, 2 speculative multi-warp rounds with in-order commit, 3 out of order with a reorder buffer and in-order commit;
 * all of them produce the sequential result bit for bit.
 * grow_stats (8 values): {rounds, seeds run, seeds redone after a conflict, then SM cycles warp 0 spent scanning for seeds,
 * on its own seed, waiting for the slowest warp of the round, committing} of frame b in the last multi-warp run. */
PLP_API plp_status plp_line_debug_grow_variant(plp_line *h, int variant);
PLP_API plp_status plp_line_debug_grow_stats(plp_line *h, int b, unsigned long long *out8);
/* host-pointer calls of at most two frames (a live frame / stereo pair) take the out-of-order kernel in automatic mode; this
 * counts the calls that were re-run with the round protocol because that kernel gave up (expected: 0) */
PLP_API int plp_line_debug_ooo_fallbacks(const plp_line *h);
PLP_API plp_status plp_line_debug_scaled(plp_line *h, int b, uint8_t *out /* (rows/2) x (cols/2) */);
PLP_API plp_status plp_line_debug_lbd_float(plp_line *h, int b, float *out /* n x 72 */, int cap);

/* ------------------------------------------------------------------------ */
/* motion-only BA  (optimize/pose_optimizer.cc, pose_optimizer_extended_line.cc) */
/* ------------------------------------------------------------------------ */
typedef struct plp_pt_obs { /* one matched keypoint (pose_optimizer.cc:126-151) */
    double pos_w[3];        /* lm->get_pos_in_world()                                  */
    float obs_x, obs_y;     /* undist_keypts_[idx].pt                                  */
    float x_right;          /* stereo_x_right_[idx]; < 0 => monocular 2-D edge         */
    float inv_sigma_sq;     /* inv_level_sigma_sq_[undist_keypt.octave]                */
} plp_pt_obs;

typedef struct plp_line_obs { /* one matched keyline (pose_optimizer_extended_line.cc:160-188) */
    double plucker[6];        /* Line::get_PlueckerCoord(): (n, d), data/landmark_line.cc:60-77 */
    float sp_x, sp_y, ep_x, ep_y; /* _keylsd[idx].getStartPoint()/getEndPoint()          */
    float inv_sigma_sq;       /* _inv_level_sigma_sq_lsd[keyline.octave]                 */
    float pad;
} plp_line_obs;

typedef struct plp_pose_opt_cfg {
    int32_t num_trials;    /* 4  (optimize/pose_optimizer.h:46) */
    int32_t num_each_iter; /* 10 */
} plp_pose_opt_cfg;

/* optimize::pose_optimizer::optimize(data::frame&) (pose_optimizer.cc:53-229) when n_lines == 0 and
 * pose_optimizer_extended_line::optimize (pose_optimizer_extended_line.cc:62-305) otherwise.
 * pts/lines hold only the keypoints/keylines that own a landmark (the adapter keeps the index map).
 * Returns through n_inliers_out the reference's return value (num_init_obs - num_bad_obs); when fewer than
 * 5 point observations are given the pose is left untouched and 0 is returned (pose_optimizer.cc:153-156). */
PLP_API plp_status plp_pose_optimize(plp_ctx *ctx, const plp_camera *cam, const double *T_cw_in /*4x4*/,
                                     const plp_pt_obs *pts, int n_pts, const plp_line_obs *lines, int n_lines,
                                     const plp_pose_opt_cfg *cfg, double *T_cw_out /*4x4*/, uint8_t *pt_outlier,
                                     uint8_t *line_outlier, int32_t *n_inliers_out);

/* Batched: frame b owns pts[pt_offsets[b] .. pt_offsets[b+1]) and lines[line_offsets[b] .. line_offsets[b+1]).
 * Host pointers; one launch for the whole batch (one CTA per frame). */
PLP_API plp_status plp_pose_optimize_batch(plp_ctx *ctx, const plp_camera *cam, int batch, const double *T_cw_in,
                                           const plp_pt_obs *pts, const int32_t *pt_offsets,
                                           const plp_line_obs *lines, const int32_t *line_offsets,
                                           const plp_pose_opt_cfg *cfg, double *T_cw_out, uint8_t *pt_outlier,
                                           uint8_t *line_outlier, int32_t *n_inliers_out);
/* Device-resident variant of the batched call (all pointers in HBM, no synchronisation).
 * d_lm_iters_out (optional, batch entries) receives the number of LM iterations executed per frame. */
PLP_API plp_status plp_pose_optimize_batch_dev(plp_ctx *ctx, const plp_camera *cam, int batch,
                                               const double *d_T_cw_in, const plp_pt_obs *d_pts,
                                               const int32_t *d_pt_offsets, const plp_line_obs *d_lines,
                                               const int32_t *d_line_offsets, int max_edges_per_frame,
                                               const plp_pose_opt_cfg *cfg, double *d_T_cw_out,
                                               uint8_t *d_pt_outlier, uint8_t *d_line_outlier,
                                               int32_t *d_n_inliers_out, int32_t *d_lm_iters_out);

/* ------------------------------------------------------------------------ */
/* frame-batched tracking front-end (module/frame_tracker.cc:52-124)         */
/* ------------------------------------------------------------------------ */
/* frame_tracker::motion_based_track for a batch of independent (current frame, last-frame landmarks, predicted
 * pose) triples, chained on the device after plp_orb_extract_batch_dev: match_current_and_last_frames (margin,
 * retried with 2*margin below 20 matches) -> pose_optimizer::optimize -> discard_outliers.  Monocular. */
typedef struct plp_tracker plp_tracker;

typedef struct plp_track_last { /* device pointers; frame b owns [offsets[b], offsets[b+1]) */
    const double *pos_w;        /* x 3: lm->get_pos_in_world() of the last frame's landmarks        */
    const int32_t *octave;      /* last_frm.keypts_[i].octave                                        */
    const float *angle;         /* last_frm.undist_keypts_[i].angle                                  */
    const uint8_t *desc;        /* x 32                                                              */
    const uint8_t *valid;       /* lm && !outlier_flags_ ; may be NULL                               */
    const int32_t *offsets;     /* batch + 1                                                         */
    const double *pose_pred;    /* batch x 16: velocity * last_frm.cam_pose_cw_ (frame_tracker.cc:58) */
    const double *pose_last;    /* batch x 16: last_frm.cam_pose_cw_                                 */
} plp_track_last;

PLP_API plp_status plp_tracker_create(plp_ctx *ctx, const plp_camera *cam, const plp_grid *grid,
                                      const float *scale_factors, const float *inv_level_sigma_sq,
                                      int num_levels, int max_batch, int kp_capacity, int max_last_points,
                                      plp_tracker **out);
/* A tracker for a distorted camera (frame.cc:68-86): motion_track_batch_dev first undistorts the current frames'
 * keypoints (plp_undistort_keypoints_batch_dev into tracker-owned arrays), and the grid, the window queries and the pose
 * optimiser's observations use the undistorted coordinates.  cam's min/max and grid must be built from
 * plp_camera_image_bounds.  dist == NULL or a perspective model with all coefficients 0 is plp_tracker_create: no extra
 * launch, the same outputs. */
PLP_API plp_status plp_tracker_create_ex(plp_ctx *ctx, const plp_camera *cam, const plp_grid *grid,
                                         const float *scale_factors, const float *inv_level_sigma_sq,
                                         int num_levels, int max_batch, int kp_capacity, int max_last_points,
                                         const plp_distortion *dist, plp_tracker **out);
/* The undistorted keypoints (max_batch x kp_capacity) and bearings (x 3) of the most recent motion_track_batch_dev of a
 * distorted tracker: device pointers owned by the tracker, valid once its stream has reached that call.  A tracker
 * without distortion has none (PLP_ERR_INVALID): its undistorted keypoints are the ORB keypoints. */
PLP_API plp_status plp_tracker_undistorted(const plp_tracker *t, const plp_keypoint **d_undist_kp,
                                           const double **d_bearings);
PLP_API void plp_tracker_destroy(plp_tracker *t);
/* d_kp/d_desc/d_n_kp: the arrays written by plp_orb_extract_batch_dev (batch x kp_capacity entries).
 * Outputs (device): matched_out[batch x kp_capacity] = last-frame landmark index kept on each keypoint after
 * discard_outliers (-1: none); pose_out[batch x 16]; num_valid_out[batch] (tracking succeeded iff >= 20);
 * n_inliers_out[batch] = pose_optimizer return value; lm_iters_out[batch] = LM iterations executed. */
PLP_API plp_status plp_tracker_motion_track_batch_dev(plp_tracker *t, int batch, const plp_keypoint *d_kp,
                                                      const uint8_t *d_desc, const int32_t *d_n_kp,
                                                      const plp_track_last *last, float margin,
                                                      int32_t *d_matched_out, double *d_pose_out,
                                                      int32_t *d_num_valid_out, int32_t *d_n_inliers_out,
                                                      int32_t *d_lm_iters_out);

/* tracking_module::optimize_current_frame_with_local_map (tracking_module.cc:732-835), monocular points, for the frames
 * of the tracker's most recent motion_track_batch_dev whose motion track succeeded (num_valid >= 20):
 * search_local_landmarks (the landmarks the motion track matched are excluded, inliers and outliers of its pose
 * optimisation alike; frame::can_observe at the motion-tracked pose; match_frame_and_landmarks with `margin` and Lowe
 * ratio 0.8) -> pose_optimizer::optimize from the motion pose -> the outliers lose their landmark. */
typedef struct plp_track_local { /* device pointers; frame b's local landmarks are rows [offsets[b], offsets[b+1]) in local_landmarks_ order */
    const double *pos_w, *obs_mean_normal;                             /* x 3 */
    const float *min_valid_dist, *max_valid_dist, *max_valid_dist_raw; /* get_min/max_valid_distance(), max_valid_dist_ */
    const uint8_t *desc;                                               /* x 32 */
    const uint8_t *valid;                                              /* !will_be_erased(); may be NULL */
    const int32_t *offsets;                                            /* batch + 1 */
    const int32_t *last_local_idx; /* one per plp_track_last row: that landmark's index in the same frame's local list, or -1 */
} plp_track_local;

/* Allocates the local-map scratch for max_batch frames of up to max_local_points local landmarks each and builds the
 * predict_scale_level table for log_scale_factor (frame::log_scale_factor_, a float); call it once, outside the hot path. */
PLP_API plp_status plp_tracker_reserve_local_map(plp_tracker *t, float log_scale_factor, int max_local_points);
/* Follows motion_track_batch_dev for the same frames on the same stream (batch <= that call's batch), and reads its
 * inputs and outputs: they must be intact.  No host synchronisation.  Outputs (device):
 *   matched_out / local_out [batch x kp_capacity]: the last-frame row (as motion_track's matched_out) or the index in the
 *     frame's local list that each keypoint holds after the outlier drop; the other entry is -1;
 *   observable_out [rows of local]: can_observe passed (the caller's increase_num_observable);
 *   pose_out [batch x 16]; num_tracked_out = inliers of the second pose optimisation (the caller applies 20, or 40
 *     after relocalisation); n_inliers_out = the optimiser's return value; lm_iters_out;
 *   status_out: 0, 1 = the frame's local list exceeds max_local_points, 2 = a last_local_idx entry is out of range.
 * After a plp_tracker_keyframe_track_batch_dev of the same batch (batch <= its batch), a frame with stage 1 is taken from
 * that call instead: active iff its keyframe track succeeded, starting from its pose, with the keyframe landmarks its pose
 * optimisation observed excluded through plp_track_keyframe.local_idx, and matched_out holding keyframe rows; status 2
 * if its local_idx block is missing or out of range.
 * A frame whose motion track failed, or with status != 0, keeps the motion pose with every per-keypoint output -1, every
 * observable flag 0, 0 iterations and num_tracked 0.  Without a reservation, or with batch > max_batch or no preceding
 * motion track: PLP_ERR_INVALID and nothing is launched. */
PLP_API plp_status plp_tracker_local_map_track_batch_dev(plp_tracker *t, int batch, const plp_track_local *local,
                                                         float margin, int32_t *d_matched_out, int32_t *d_local_out,
                                                         uint8_t *d_observable_out, double *d_pose_out,
                                                         int32_t *d_num_tracked_out, int32_t *d_n_inliers_out,
                                                         int32_t *d_lm_iters_out, int32_t *d_status_out);

/* frame_tracker::bow_match_based_track (module/frame_tracker.cc:126-189) against each frame's reference keyframe
 * (curr_frm.ref_keyfrm_), for the frames of the tracker's most recent motion_track_batch_dev that the reference hands to
 * it: the motion model is not usable, or the motion track failed.  frame::compute_bow (transform, levelsup 4) ->
 * bow_tree::match_frame_and_keyframe (Lowe 0.7, orientation check) -> below 20 matches the frame fails; else
 * pose_optimizer::optimize from last_frm.cam_pose_cw_ (the motion call's pose_last) -> discard_outliers.  Monocular. */
typedef struct plp_track_keyframe { /* device pointers except num_keyframes; keyframe k owns rows [row_offsets[k], row_offsets[k+1]) */
    int32_t num_keyframes;           /* K (host value), at most the reserved max_keyframes                              */
    const int32_t *kf_of_frame;      /* batch: index of frame b's reference keyframe                                    */
    const int32_t *row_offsets;      /* K + 1                                                                            */
    const uint8_t *desc;             /* x 32: descriptors_                                                               */
    const float *angle;              /* keypts_[i].angle                                                                 */
    const uint8_t *valid;            /* lm && !lm->will_be_erased(); NULL == all                                         */
    const double *pos_w;             /* x 3: lm->get_pos_in_world() (read for valid rows only)                           */
    const int32_t *fv_offsets;       /* K + 1: keyframe k's bow_feat_vec_ nodes are [fv_offsets[k], fv_offsets[k+1])     */
    const uint32_t *node_ids;        /* ascending within a keyframe                                                      */
    const int32_t *node_begin;       /* nodes + 1: node a's rows are indices[node_begin[a] .. node_begin[a+1])           */
    const uint32_t *indices;         /* keyframe-local row numbers                                                       */
    const int32_t *local_idx;        /* optional: per frame, one entry per row of its keyframe: that landmark's index in
                                        the frame's local list (plp_track_local), or -1; read by the local-map stage     */
    const int32_t *local_idx_offsets; /* batch + 1 (with local_idx)                                                      */
} plp_track_keyframe;

/* Allocates the keyframe-track scratch for max_batch frames whose keyframes hold up to max_keyframe_points rows each, in
 * tables of up to max_keyframes keyframes; call it once, outside the hot path.  A kp_capacity whose feature-vector kernel
 * needs more shared memory (12 bytes per keypoint) than the device offers: PLP_ERR_CAPACITY, nothing allocated. */
PLP_API plp_status plp_tracker_reserve_keyframe_track(plp_tracker *t, int max_keyframes, int max_keyframe_points);
/* Follows motion_track_batch_dev on the same stream (batch <= that call's batch) and reads its inputs, outputs and
 * scratch; writes none of them.  Frame b runs the stage iff d_motion_valid[b] == 0 (NULL: all 1; the reference's
 * velocity_is_valid_ && last_reloc_frm_id_ + 2 < curr_frm_.id_) or its motion num_valid < 20.  No host synchronisation.
 * vocab must live on the tracker's device; its kernels run on the tracker's stream.  Outputs (device):
 *   stage_out[batch]: 0 = the motion result stands, 1 = the keyframe stage ran (tracking succeeded iff num_valid >= 20);
 *   kf_matched_out[batch x kp_capacity]: the keyframe row each keypoint keeps after discard_outliers, or -1;
 *   num_bow_matches_out[batch]: match_frame_and_keyframe's count (0 where the stage did not run);
 *   pose_out[batch x 16]: the optimiser result, or pose_last where it did not run;
 *   num_valid_out, n_inliers_out, lm_iters_out [batch] (0 where the optimiser did not run);
 *   status_out[batch]: 0, 1 = the keyframe has more than max_keyframe_points rows, 2 = kf_of_frame out of [0, K); such a
 *     frame (stage 1) fails like a track with no match.
 * Without a reservation, with K > max_keyframes, with no preceding motion track or with batch above its batch:
 * PLP_ERR_INVALID and nothing is launched.  A following local_map_track_batch_dev of the same batch starts each stage-1
 * frame from this call's result (see INTEGRATION.md). */
PLP_API plp_status plp_tracker_keyframe_track_batch_dev(plp_tracker *t, plp_bow_vocab *vocab, int batch,
                                                        const plp_track_keyframe *kf, const uint8_t *d_motion_valid,
                                                        int32_t *d_stage_out, int32_t *d_kf_matched_out,
                                                        int32_t *d_num_bow_matches_out, double *d_pose_out,
                                                        int32_t *d_num_valid_out, int32_t *d_n_inliers_out,
                                                        int32_t *d_lm_iters_out, int32_t *d_status_out);
/* The BoW rows (transform with levelsup 4: word id, node id, weight; max_batch x kp_capacity) of the most recent
 * keyframe_track_batch_dev, for the frames it ran the stage on (stage 1, status 0): device pointers owned by the
 * tracker, valid once its stream has reached that call.  A keyframe made from such a frame takes its bow_vec_ /
 * bow_feat_vec_ from these rows (plp_bow_transform's layout) instead of transforming again. */
PLP_API plp_status plp_tracker_keyframe_bow(const plp_tracker *t, const int32_t **d_word_id, const int32_t **d_node_id,
                                            const float **d_weight);

/* frame_tracker::robust_match_based_track (module/frame_tracker.cc:192-245) against each frame's reference keyframe, for
 * the frames whose keyframe track (the preceding plp_tracker_keyframe_track_batch_dev of the same batch) ran and failed:
 * robust::brute_force_match (Lowe 0.8, no orientation check; frame = side 1) -> the match list in frame keypoint order
 * -> essential_solver(frm.bearings_, keyfrm->bearings_, matches).find_via_ransac(50, false) -> the inlier matches;
 * below 20 the frame fails, else pose_optimizer::optimize from last_frm.cam_pose_cw_ -> discard_outliers.  Monocular.
 * Allocates the scratch for max_batch frames; call it once, outside the hot path (a second call replaces the first).
 * Refuses a tracker whose kp_capacity exceeds the brute-force matcher's 4096 (PLP_ERR_INVALID) or the hypothesis
 * kernel's shared memory (PLP_ERR_CAPACITY), before allocating anything. */
PLP_API plp_status plp_tracker_reserve_robust_track(plp_tracker *t);
/* Follows keyframe_track_batch_dev on the same stream (batch <= that call's batch) and reads the keyframe table it was
 * given (rows, desc, valid, pos_w, kf_of_frame, local_idx: keep it alive) and the motion and keyframe calls' outputs and
 * scratch; writes none of them.  d_kf_bearings: keyfrm->bearings_, one row of 3 doubles per keyframe-table row.  The
 * frame bearings are the undistortion's (distorted tracker) or convert_keypoints_to_bearings of the keypoints.  The
 * RANSAC sample sets are drawn on the device from `seed` (see plp_tracker_robust_samples).  No host synchronisation.
 * Outputs (device):
 *   stage_out[batch]: 1 = the stage ran (keyframe stage 1 and keyframe num_valid < 20; tracking succeeded iff
 *     num_valid >= 20), else 0;
 *   kf_matched_out[batch x kp_capacity]: the keyframe row each keypoint keeps after discard_outliers, or -1;
 *   num_bf_matches_out[batch]: the brute-force match count, num_robust_matches_out[batch]: the RANSAC inliers among
 *     them (0 if the solution is not valid) (both 0 where the stage did not run);
 *   pose_out[batch x 16]: the optimiser result, or pose_last where it did not run or found fewer than 20 robust matches;
 *   num_valid_out, n_inliers_out, lm_iters_out [batch] (0 where the optimiser did not run);
 *   status_out[batch]: the keyframe call's status; a frame with status != 0 fails like a track with no match.
 * Without a reservation, with no preceding keyframe track since the last motion track, or with batch above its batch:
 * PLP_ERR_INVALID and nothing is launched.  A following local_map_track_batch_dev of the same batch starts each frame
 * that ran this stage from its result (see INTEGRATION.md). */
PLP_API plp_status plp_tracker_robust_track_batch_dev(plp_tracker *t, int batch, const double *d_kf_bearings,
                                                      uint64_t seed, int32_t *d_stage_out, int32_t *d_kf_matched_out,
                                                      int32_t *d_num_bf_matches_out, int32_t *d_num_robust_matches_out,
                                                      double *d_pose_out, int32_t *d_num_valid_out,
                                                      int32_t *d_n_inliers_out, int32_t *d_lm_iters_out,
                                                      int32_t *d_status_out);
/* The RANSAC sample sets of the most recent robust_track_batch_dev (max_batch x 50 x 8 indices into the frame's
 * brute-force match list, -1 where none were drawn): a device pointer owned by the tracker, valid once its stream has
 * reached that call.  They are util::create_random_array(8, 0, n - 1) over a counter-based generator keyed by
 * (seed, frame, hypothesis); see csrc/ransac_sample.h. */
PLP_API plp_status plp_tracker_robust_samples(const plp_tracker *t, const int32_t **d_samples);

/* ------------------------------------------------------------------------ */
/* local bundle adjustment (optimize/local_bundle_adjuster*.cc)               */
/* ------------------------------------------------------------------------ */
/* The graph the reference gathers at local_bundle_adjuster.cc:72-272 (pointer-graph walk, stays in the adapter):
 * keyframes = local + fixed, local point / line landmarks, one edge per observation, optional point-to-plane
 * edges (local_bundle_adjuster_extended_plane.cc:309-345).  Edges must be grouped by ascending landmark index
 * (that is the order in which the reference creates them). */
typedef struct plp_ba_problem {
    double fx, fy, cx, cy, focal_x_baseline;
    int32_t setup_type; /* 0 Monocular: point-edge Huber delta sqrt(5.991), else sqrt(7.815) */
    int32_t n_kf;
    const double *kf_pose_cw; /* n_kf x 16 row-major */
    const uint8_t *kf_fixed;  /* keyframe id == 0 or "fixed keyframe" (local_bundle_adjuster.cc:197-213) */
    int32_t n_pts;
    const double *pt_pos_w; /* n_pts x 3 */
    int32_t n_pt_edges;
    const int32_t *pt_edge_kf, *pt_edge_lm;
    const float *pt_edge_obs;          /* x 3: undist_keypt.pt.x, .y, stereo_x_right (< 0: monocular edge) */
    const float *pt_edge_inv_sigma_sq; /* inv_level_sigma_sq_[octave] */
    int32_t n_lines;
    const double *line_plucker; /* n_lines x 6, Line::get_PlueckerCoord() */
    int32_t n_line_edges;
    const int32_t *line_edge_kf, *line_edge_lm;
    const float *line_edge_obs; /* x 4: keyline start / end point */
    const float *line_edge_inv_sigma_sq;
    int32_t n_plane_edges; /* at most one per point landmark */
    const int32_t *plane_edge_lm;
    const double *plane_edge_fn; /* x 4: plane (n, d) */
} plp_ba_problem;

typedef struct plp_ba_cfg {
    int32_t num_first_iter;  /* 5  (optimize/local_bundle_adjuster.h:47-49) */
    int32_t num_second_iter; /* 10 */
    int32_t num_ctas;        /* landmark shards per GPU; 0 = automatic */
} plp_ba_cfg;

typedef struct plp_ba_result {
    double *kf_pose_cw;         /* n_kf x 16 (fixed keyframes are returned unchanged) */
    double *pt_pos_w;           /* n_pts x 3 */
    double *line_plucker;       /* n_lines x 6 */
    uint8_t *pt_edge_outlier;   /* outlier_observations (local_bundle_adjuster.cc:342-372) */
    uint8_t *line_edge_outlier; /* outlier_observations_line */
    int32_t iters_first, iters_second, lm_tries;
    double final_chi2;
} plp_ba_result;

typedef struct plp_ba plp_ba;           /* a problem resident on one GPU */
typedef struct plp_ba_comm plp_ba_comm; /* NCCL communicator for landmark-sharded multi-GPU BA */

/* local_bundle_adjuster[_extended_line|_extended_plane]::optimize(curr_keyfrm, force_stop_flag) after the gather.
 * force_stop may be NULL; it is polled between chunks of LM iterations (mapping_module.cc:159-164). */
PLP_API plp_status plp_local_ba(plp_ctx *ctx, const plp_ba_problem *p, const plp_ba_cfg *cfg,
                                volatile const uint8_t *force_stop, plp_ba_result *r);
/* optimize::global_bundle_adjuster::optimize (optimize/global_bundle_adjuster.cc:64-253) on the same problem layout:
 * every keyframe / point / line landmark of the map, kf_fixed = (keyframe id == 0) only, ONE optimize(num_iter) with or
 * without the Huber kernel (use_huber_kernel_), no outlier rounds (the outlier arrays of `r` come back zero).  Up to 32
 * non-fixed keyframes (the map-initialisation call, module/initializer.cc:306-307: 2 keyframes, 20 iterations) share the
 * in-shared-memory reduced-camera solve of the local adjuster; larger maps (after a loop closure,
 * module/loop_bundle_adjuster.cc:81-82) keep the reduced system dense in HBM: FP64 atomics per landmark, right-looking
 * blocked Cholesky with FP64 tensor-core (DMMA) trailing updates.  plp_local_ba / plp_ba_create take the same path for a
 * local window of more than 32 non-fixed keyframes (fixed keyframes are never bounded). */
PLP_API plp_status plp_global_ba(plp_ctx *ctx, const plp_ba_problem *p, int num_iter, int use_huber_kernel,
                                 volatile const uint8_t *force_stop, plp_ba_result *r);
/* split form: upload once, solve (repeatable), destroy.  With `comm`, `p` holds THIS RANK's block of landmarks
 * (all keyframes, its points/lines and their edges); every rank calls the same functions. */
PLP_API plp_status plp_ba_create(plp_ctx *ctx, const plp_ba_problem *p, const plp_ba_cfg *cfg, plp_ba_comm *comm,
                                 plp_ba **out);
PLP_API plp_status plp_ba_solve(plp_ba *ba, volatile const uint8_t *force_stop, plp_ba_result *r);
PLP_API void plp_ba_destroy(plp_ba *ba);
/* benchmark hook: run `tries` LM tries (linearise + Schur + solve + update + accept/reject) from the initial state */
PLP_API plp_status plp_ba_bench_tries(plp_ba *ba, int tries, int32_t *iters_done, int32_t *tries_done);
/* test read-back of ONE try's linear algebra: from the initial state (Huber kernel on) the lambda-initialisation try and the
 * first real try run exactly as in plp_ba_bench_tries(ba, 1, ...); then the reduced camera system that try solved comes back:
 *   packed  n_pairs * 36 + 12 * n_free + 1 doubles, n_pairs = n_free (n_free + 1) / 2:
 *           [S: the upper 6 x 6 blocks (i, j), i <= j, row-wise over the free keyframes, lambda NOT yet on the diagonal |
 *            g: 6 n_free | bp = -Jp^T w e: 6 n_free | robust chi2 of the linearisation point]
 *   dp      6 * n_free: the pose step, solution of (S + lambda I) dp = g (zero if the system was not positive definite)
 *   lambda  the damping of that try (already inside the Schur term: S = Hpp - sum_l W (Hll + lambda I)^-1 W^T)
 * Both representations (shared-memory and dense-in-HBM) fill the same layout.  Any of the three outputs may be NULL. */
PLP_API plp_status plp_ba_debug_try(plp_ba *ba, double *packed, double *dp, double *lambda);

/* multi-GPU: rank 0 creates a 128-byte id, the launcher broadcasts it, every rank joins */
PLP_API plp_status plp_ba_comm_unique_id(uint8_t id_out[128]);
PLP_API plp_status plp_ba_comm_init(plp_ctx *ctx, const uint8_t id[128], int world, int rank, plp_ba_comm **out);
PLP_API void plp_ba_comm_destroy(plp_ba_comm *comm);
/* number of ncclAllReduce calls issued through the communicator so far (measurement: all-reduces per LM try) */
PLP_API uint64_t plp_ba_comm_allreduce_count(const plp_ba_comm *comm);
/* 1 if the communicator's small all-reduces run as the one-shot kernel over NVLink peer memory (ranks on one node, CUDA IPC
 * available; PLP_BA_PEER=0 forces NCCL), and how many all-reduces took that path */
PLP_API int plp_ba_comm_peer_active(const plp_ba_comm *comm);
PLP_API uint64_t plp_ba_comm_peer_count(const plp_ba_comm *comm);

#ifdef __cplusplus
}
#endif
#endif /* PLPSLAM_B200_H */
