/*
 * plslam_b200.h — C ABI of the CUDA (H100, sm_90a) stereo point+line front-end.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference (rubengooj/pl-slam) consumes the
 * per-frame hot path through the C++ class API of stvo-pl (StVO::StereoFrame / StereoFrameHandler,
 * free functions match()/matchGrid()) and of the vendored 3rdparty/line_descriptor; none of it is a
 * C ABI.  Every entry point below names the reference interface it replaces (file:line relative to
 * the reference tree).  The C++ shim in pl-slam_b200/cpp/ re-creates the class API on top of these
 * functions; INTEGRATION.md shows the binding a pl-slam maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types cross the boundary;
 *   - every function returns plf_status (0 = ok, <0 = error); plf_last_error() gives the text;
 *   - "host" entry points take HOST pointers and copy H2D/D2H internally (the reference-facing
 *     calls); the *_dev / plf_batch_* entry points work on buffers already resident in HBM;
 *   - no CPU fallback exists: without a CUDA device plf_create fails with PLF_ERR_NO_DEVICE.
 */
#ifndef PLSLAM_B200_H
#define PLSLAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLF_ABI_VERSION 1
#define PLF_DESC_BYTES 32 /* ORB rBRIEF-256 and LBD-256: 32 bytes per descriptor */

typedef int plf_status;
enum {
  PLF_OK = 0,
  PLF_ERR_INVALID = -1,   /* bad argument */
  PLF_ERR_NO_DEVICE = -2, /* no CUDA device / CUDA runtime failure at create */
  PLF_ERR_CUDA = -3,      /* CUDA runtime error during a call */
  PLF_ERR_CAPACITY = -4,  /* a fixed-capacity device buffer overflowed (see plf_limits) */
  PLF_ERR_STATE = -5      /* call sequence error */
};

typedef struct plf_ctx plf_ctx; /* opaque; one per (device, stream); not thread-safe per ctx */

/* Front-end parameters: the stvo-pl Config keys that pl-slam inherits
 * (config/config/config_euroc.yaml:9-77, SlamConfig : Config at include/slamConfig.h:28). */
typedef struct plf_params {
  /* switches (config_euroc.yaml:9-18).  has_points / has_lines = 0 disables that kind in the batched front-end as stvo-pl
   * does in extraction and f2fTracking: its n_kp_* / n_lines_* are reported as 0 and it contributes no stereo rows, no
   * matches and no pose rows.  Both 0 is rejected by plf_create (PLF_ERR_INVALID).  The standalone operators (plf_orb,
   * plf_lsd, plf_detect_lines) ignore the switches. */
  int has_points, has_lines, best_lr_matches;
  /* point tracking (config_euroc.yaml:22-25) */
  float max_dist_epip, min_disp, min_ratio_12_p;
  /* line tracking (config_euroc.yaml:27-34).  line_sim_th: direction gate of the windowed matcher (matching_strategy != 0
   * and plf_match_grid_lines).  f2f_overlap_th: carried for API parity, IGNORED (stvo-pl's matchF2FLines does not gate on
   * overlap in the version pl-slam builds against). */
  float line_sim_th, stereo_overlap_th, f2f_overlap_th, min_line_length, line_horiz_th,
      min_ratio_12_l, ls_min_disp_ratio;
  /* optimiser (config_euroc.yaml:43-51) */
  double homog_th;
  int min_features, max_iters, max_iters_ref;
  double min_error, min_error_change, inlier_k; /* inlier_k: IGNORED - the outlier gate is the in-tree twin's chi2 threshold
                                                   sqrt(7.815) (src/mapHandler.cpp:3460,3479), not stvo-pl's MAD-scaled inlier_k */
  /* ORB (config_euroc.yaml:59-67).  Supported: 1..8 levels, orb_wta_k 2, orb_score 1 (FAST), orb_patch_size 31, and
   * orb_edge_th >= 19 (the reference configs' value: the oriented 31-pixel patch reaches 18 pixels from a keypoint, which
   * OpenCV covers with a border-reflected padding the device path does not build); every pyramid level must measure at
   * least 2 orb_edge_th + 8 pixels.  Other values fail with PLF_ERR_INVALID. */
  int orb_nfeatures;
  float orb_scale_factor;
  int orb_nlevels, orb_edge_th, orb_wta_k, orb_score, orb_patch_size, orb_fast_th;
  /* LSD (config_euroc.yaml:68-77).  Only lsd_refine = 0 is supported; as in OpenCV, lsd_log_eps and lsd_density_th then
   * have no effect.  lsd_n_bins must be in [1, 1024] and the Gaussian kernel 1 + 2 ceil(3.717 sigma) at most 15 taps
   * (sigma = lsd_sigma_scale, divided by lsd_scale below 1); other values fail with PLF_ERR_INVALID. */
  int lsd_nfeatures, lsd_refine;
  double lsd_scale, lsd_sigma_scale, lsd_quant, lsd_ang_th, lsd_log_eps, lsd_density_th; /* LSDOptions: double */
  int lsd_n_bins;
  /* matching strategy (config_euroc.yaml:55-57 `matching_strategy`, `matching_s_ws`, `matching_f2f_ws`).
   * 0 (default here): descriptor-only association - stereo and frame-to-frame matches come from match() (brute-force
   * NNR + mutual).  != 0 (the reference configs select 3): windowed - stereo association runs matchGrid() over the
   * 48 x 64 GridStructure of the right image with the window (matching_s_ws, 0) x (0, 0); frame-to-frame tracking
   * follows the in-tree analogue's control flow (src/mapHandler.cpp:247-278, :379-425): matchGrid() in a
   * +-matching_f2f_ws window around the projected feature, match() when fewer than min_pt_matches / min_ls_matches
   * (src/slamConfig.cpp:85-86) survive. */
  int matching_strategy, matching_s_ws, matching_f2f_ws, min_pt_matches, min_ls_matches;
} plf_params;

/* Rectified pinhole stereo rig (stvo-pl PinholeStereoCamera; schema
 * config/dataset_params/kitti00-02.yaml:1-21). */
typedef struct plf_camera {
  int width, height;
  double fx, fy, cx, cy, b;
} plf_camera;

/* Fixed device capacities chosen at create time. */
typedef struct plf_limits {
  int max_batch;     /* stereo pairs per plf_batch_* call */
  int max_keypoints; /* ORB keypoints per image (all levels, ties included) */
  int max_segments;  /* raw LSD segments per image */
  int max_lines;     /* KeyLines kept per image after the top-K */
} plf_limits;

/* Fills *p with the reference defaults (config/config/config_euroc.yaml). */
void plf_default_params(plf_params* p);
void plf_default_limits(plf_limits* l);

int plf_abi_version(void);
/* Human-readable text of the last error on this ctx (or of the last failed plf_create if ctx==NULL). */
const char* plf_last_error(const plf_ctx* ctx);

/* Replaces: `new StereoFrameHandler(cam)` app/plslam_dataset.cpp:109 (+ Config singleton load,
 * src/slamConfig.cpp:106-164). Allocates all device buffers for `limits` on `device`. */
plf_status plf_create(const plf_params* params, const plf_camera* cam, const plf_limits* limits,
                      int device, plf_ctx** out);
void plf_destroy(plf_ctx* ctx);
/* Number of kernels this ctx has launched since creation (bench.py "gpu_launches"). */
long long plf_launch_count(const plf_ctx* ctx);
/* The CUDA stream (cudaStream_t) all work of this ctx is enqueued on, for event timing. */
void* plf_stream(const plf_ctx* ctx);
plf_status plf_sync(plf_ctx* ctx);

/* Per-kernel device timing of plf_batch_run (CUDA events on plf_stream; replaces the reference's only
 * instrumentation, the ms Timer around insertStereoPair+optimizePose, app/plslam_dataset.cpp:126-132).
 * plf_profile_read: after a run with profiling on, ms[i] = device time of stage i, names_buf = ';'-separated
 * stage names; *n = number of stages. */
plf_status plf_profile_enable(plf_ctx* ctx, int on);
plf_status plf_profile_read(plf_ctx* ctx, char* names_buf, int buf_len, float* ms, int cap, int* n);

/* ------------------------------------------------------------------------------------------------
 * Descriptor matching (SURVEY §8 a4/a5)
 * ---------------------------------------------------------------------------------------------- */

/* Hamming 2-nearest-neighbour search.  Replaces cv::BFMatcher(NORM_HAMMING).knnMatch(k=2) as
 * called by stvo-pl matchNNR (call sites src/mapHandler.cpp:277,424,597,712,3223,3249) and the
 * popcount primitive 3rdparty/line_descriptor/src/bitops_custom.hpp:83-96.
 * d1: n1 x 32 bytes (queries), d2: n2 x 32 bytes (train), row-major, host pointers.
 * Outputs (host, length n1): index and distance of the nearest and second nearest train row under
 * the (distance, index) lexicographic order (OpenCV's tie rule); idx = -1, dist = -1 when absent. */
plf_status plf_hamming_knn2(plf_ctx* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                            int32_t* idx1, int32_t* dist1, int32_t* idx2, int32_t* dist2);

/* NNR + mutual-consistency matcher.  Replaces stvo-pl `int match(const Mat&, const Mat&, float nnr,
 * vector<int>& matches_12)` (src/mapHandler.cpp:277,424,597,712,3223,3249).
 * matches_12[i] = j if row i of d1 matches row j of d2 (best.distance < nnr * second.distance in
 * f32, and — when best_lr != 0 — i is also the ratio-accepted best of j in the reverse direction),
 * else -1.  *n_matches receives the count (the reference's return value). */
plf_status plf_match(plf_ctx* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2, float nnr,
                     int best_lr, int32_t* matches_12, int* n_matches);

/* Windowed greedy matcher.  Replaces stvo-pl `int matchGrid(const vector<point_2d>&, const Mat& d1, const GridStructure&,
 * const Mat& d2, const GridWindow&, vector<int>& matches_12)` and its lines overload `matchGrid(const vector<line_2d>&,
 * d1, grid, d2, const vector<pair<double,double>>& directions2, w, matches_12)`, called at src/mapHandler.cpp:271,591
 * (points) and :418,706 (lines); grids built at :260-264, :398-411; window :266-269.  stvo-pl is not vendored: semantics
 * restated from SURVEY Appendix A.3 (oracle/matchgrid.py, "parity unpinned"); candidates are visited in ascending index
 * order where stvo-pl iterates an unordered_set.
 * All coordinates are integer GRID cells (x in [0, grid_cols), y in [0, grid_rows)), i.e. what the reference obtains by
 * scaling pixels with inv_width = GRID_COLS / width, inv_height = GRID_ROWS / height and truncating to int.
 *   The GridStructure is passed as it is held - per cell, the list of train indices pushed into it with
 *   grid.at(x, y).push_back(idx): cell (x, y) owns cell_items[cell_start[x * grid_rows + y] .. cell_start[.. + 1]);
 *   a train line appears in every cell of its getLineCoords() walk; indices outside [0, n2) are ignored.
 *   points: q_cell [n1][2] = cells of the projected query points (pj_points);
 *   lines:  q_line [n1][4] = (x1, y1, x2, y2) end-point cells of the projected query lines (looked up along their
 *           Bresenham walk), t_dir [n2][2] = directions2.
 * Query order matters: with best_lr a candidate counts for query i only if it beats every earlier query's distance to
 * it.  matches_12[i] = j or -1; *n_matches = the reference's return value.  n1, n2 <= 8192. */
typedef struct plf_grid_window {
  int width_lo, width_hi;    /* GridWindow::width  (first, second) */
  int height_lo, height_hi;  /* GridWindow::height (first, second) */
} plf_grid_window;
plf_status plf_match_grid_points(plf_ctx* ctx, const int* q_cell, const uint8_t* d1, int n1, const int* cell_start,
                                 const int* cell_items, const uint8_t* d2, int n2, int grid_cols, int grid_rows,
                                 plf_grid_window w, float nnr, int best_lr, int32_t* matches_12, int* n_matches);
plf_status plf_match_grid_lines(plf_ctx* ctx, const int* q_line, const uint8_t* d1, int n1, const int* cell_start,
                                const int* cell_items, const double* t_dir, const uint8_t* d2, int n2, int grid_cols,
                                int grid_rows, plf_grid_window w, float nnr, double line_sim_th, int best_lr,
                                int32_t* matches_12, int* n_matches);

/* Landmark descriptor maintenance, batched (SURVEY §8(f) f3).  Replaces the body of MapPoint::updateAverageDescDir and
 * MapLine::updateAverageDescDir (src/mapFeatures.cpp:51-93, 121-163), called on every observation add (:48, :118).
 * desc: the observed descriptors of all landmarks, concatenated, [offsets[n_landmarks]][32] (host); landmark l owns
 * rows offsets[l] .. offsets[l+1]-1 (2 .. 64 of them); dirs: the matching observation directions [.][3] f64, or NULL.
 * med_idx[l] = index WITHIN landmark l of the descriptor the reference would copy into med_desc (smallest element at
 * position int(1 + 0.5 (n-1)) of its sorted distance row, first on ties); med_dir[l] = mean direction (sum in
 * observation order / n; the reference's accumulator is uninitialised, :88-90 - zero here, deliberately). */
plf_status plf_median_descriptors(plf_ctx* ctx, const uint8_t* desc, const int* offsets, const double* dirs,
                                  int n_landmarks, int* med_idx, double* med_dir);

/* ------------------------------------------------------------------------------------------------
 * Point features (SURVEY §8 a1)
 * ---------------------------------------------------------------------------------------------- */

/* Field-for-field mirror of cv::KeyPoint (pt.x, pt.y, size, angle, response, octave, class_id); 28 bytes. */
typedef struct plf_keypoint {
  float x, y;
  float size, angle, response;
  int octave, class_id;
} plf_keypoint;

/* ORB detect + describe on one image.  Replaces stvo-pl StereoFrame::detectPointFeatures ->
 * cv::ORB::create(orb_nfeatures, orb_scale_factor, orb_nlevels, orb_edge_th, 0, orb_wta_k, orb_score,
 * orb_patch_size, orb_fast_th)->detectAndCompute(img, Mat(), kps, desc, false)
 * (parameters config/config/config_euroc.yaml:59-67; descriptor rows used at src/mapHandler.cpp:86-88,302).
 * Output order is canonical (octave, y, x): OpenCV's own order inside a level is the implementation-defined
 * result of std::nth_element (KeyPointsFilter::retainBest); the SET of keypoints, every field and every
 * descriptor are identical to OpenCV's.  kps/desc: host buffers with room for `cap` entries; *n receives
 * the count (PLF_ERR_CAPACITY if it exceeds cap or the ctx limit max_keypoints).  Work is enqueued on plf_stream in a
 * working state of its own (one image, rebuilt when the image size changes) and never touches the batched pipeline's
 * buffers, so a call between batches in flight is safe. */
plf_status plf_orb(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, plf_keypoint* kps,
                   uint8_t* desc, int cap, int* n);

/* ------------------------------------------------------------------------------------------------
 * Line features (SURVEY §8 a2/a3)
 * ---------------------------------------------------------------------------------------------- */

/* Field-for-field mirror of cv::line_descriptor::KeyLine
 * (3rdparty/line_descriptor/include/line_descriptor/descriptor_custom.hpp:105-176); 68 bytes. */
typedef struct plf_keyline {
  float angle;
  int class_id;
  int octave;
  float ptx, pty;
  float response;
  float size;
  float startPointX, startPointY, endPointX, endPointY;
  float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
  float lineLength;
  int numOfPixels;
} plf_keyline;

/* Raw LSD segments.  Replaces cv::createLineSegmentDetector(lsd_refine (0), lsd_scale, lsd_sigma_scale, lsd_quant,
 * lsd_ang_th, lsd_log_eps, lsd_density_th, lsd_n_bins)->detect(img, lines) as called at
 * 3rdparty/line_descriptor/src/LSDDetector_custom.cpp:246-264.  segs: cap x 4 floats (x1,y1,x2,y2), OpenCV's
 * output order (seed order).  *n receives the count.  Work is enqueued on plf_stream in a working state of its own (one
 * image, rebuilt when the image size changes, shared with plf_detect_lines) and never touches the batched pipeline's
 * buffers, so a call between batches in flight is safe. */
plf_status plf_lsd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, float* segs, int cap, int* n);

/* Line features of one image.  Replaces stvo-pl StereoFrame::detectLineFeatures (LSD branch):
 * LSDDetectorC::detect(img, lines, scale, 1, opts) (LSDDetector_custom.cpp:218-324, opts.min_length =
 * min_line_length * min(w,h)), then — when more than lsd_nfeatures lines are found and lsd_nfeatures != 0 — sort by
 * response (descending; ties keep detection order), keep lsd_nfeatures and set class_id = rank, then
 * BinaryDescriptor::compute (binary_descriptor_custom.cpp:524).  keylines/desc: host buffers of `cap` entries.
 * Enqueued on plf_stream in plf_lsd's working state; never touches the batched pipeline's buffers, so a call between
 * batches in flight is safe. */
plf_status plf_detect_lines(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                            plf_keyline* keylines, uint8_t* desc, int cap, int* n);

/* Test hook: evaluates the device port of glibc sinf/cosf used by the LSD region-angle update. */
plf_status plf_debug_sincosf(plf_ctx* ctx, const float* in, float* s, float* c, int n);

/* LBD prelude: GaussianBlur 5x5 sigma 1 then Sobel k=3 to CV_16S.  Replaces
 * BinaryDescriptor::computeSobel (binary_descriptor_custom.cpp:373-398 -> :350-370).
 * img: h rows of `stride` bytes (host). dxdy: h*w interleaved int16 pairs (dx,dy) (host). */
plf_status plf_lbd_gradients(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, int16_t* dxdy);

/* LBD descriptors.  Replaces BinaryDescriptor::compute(image, keylines, descriptors, returnFloat)
 * (binary_descriptor_custom.cpp:524-528 -> computeImpl :539-687 -> computeLBD :1026-1372).
 * Uses from each KeyLine: sPointInOctave*, ePointInOctave*, numOfPixels, angle (octave 0 only, as the
 * front-end calls it).  desc: n x 32 bytes (host).  desc_float (optional): n x 72 floats.
 * n == 0 returns PLF_OK without touching desc (the reference prints a message and returns). */
plf_status plf_lbd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                   const plf_keyline* keylines, int n, uint8_t* desc, float* desc_float);

/* ------------------------------------------------------------------------------------------------
 * Pose refinement (SURVEY §8 a8/a9)
 * ---------------------------------------------------------------------------------------------- */

typedef struct plf_gn_opts {
  double homog_th;   /* Config::homogTh (config_euroc.yaml:45; src/mapHandler.cpp:3344,3355) */
  int max_iters;     /* stage 1 iterations (config_euroc.yaml:47) */
  int max_iters_ref; /* stage 2 iterations (config_euroc.yaml:48) */
  double eps_err;    /* stop if e < eps_err (twin: DBL_EPSILON :3434; stvo-pl: min_error) */
  double eps_change; /* stop if |e - e_prev| < eps_change (twin: DBL_EPSILON; stvo-pl: min_error_change) */
  double eps_step;   /* stop if |dx| < eps_step (twin: DBL_EPSILON :3441) */
} plf_gn_opts;

typedef struct plf_pose_result {
  double T[16];   /* row-major 4x4 pose increment (T_inc / stvo-pl DT) */
  double cov[36]; /* H^-1 of the last accumulation (DT_cov, src/mapHandler.cpp:3491) */
  double x[6];    /* logmap_se3(T) = [t; w] */
  double err;     /* normalised weighted error of the last accumulation */
  int iters1, iters2, n_inliers_pt, n_inliers_ls;
} plf_pose_result;

/* Two-stage robust (Cauchy) Gauss-Newton on point + line reprojection residuals.  Replaces
 * StereoFrameHandler::optimizePose (app/plslam_dataset.cpp:128; src/mapHandler.cpp:780); arithmetic of
 * its in-tree twin MapHandler::computeRelativePoseRobustGN (src/mapHandler.cpp:3566-3957).
 * P: np x 3 (3-D points, previous camera frame), pl_obs: np x 2 (observed pixels, current frame),
 * sP,eP: nl x 3 (3-D endpoints), le_obs: nl x 3 (observed normalised line), all f64 host arrays;
 * inlier_pt / inlier_ls: u8 flags, in (rows to use) and out (after the chi2 gate).  T_init: row-major
 * 4x4 or NULL (identity).  opts NULL => thresholds from the ctx params (stvo-pl min_error/min_error_change). */
plf_status plf_gn_pose(plf_ctx* ctx, const plf_gn_opts* opts, const double* P, const double* pl_obs,
                       uint8_t* inlier_pt, int np, const double* sP, const double* eP,
                       const double* le_obs, uint8_t* inlier_ls, int nl, const double* T_init,
                       plf_pose_result* out);

/* Local bundle adjustment (SURVEY 8(f) f4).  Replaces MapHandler::levMarquardtOptimizationLBA (src/mapHandler.cpp:1332-1989),
 * the numerical core of MapHandler::localBundleAdjustment (:1220-1330): Levenberg-Marquardt over the local keyframes'
 * poses, the local 3-D points and the local 3-D segments with Cauchy-weighted residuals, solved on the device through the
 * Schur complement on the landmarks.  The caller (MapHandler) assembles the lists exactly as :1224-1319 does:
 *   kf_pose  [n_kf][6]  x_kf_w of the local keyframes (se(3) vectors [t; w]), in / out
 *   pt       [n_pt][3]  point3D of the local map points, in / out;   ls [n_ls][6]  line3D (start | end), in / out
 *   fixed_T  [n_fixed][16]  T_kf_w (row-major) of the keyframes that observe local landmarks but are not optimised
 *   observations, grouped per landmark in ascending local landmark index (obs_aux(1), :1257,:1298):
 *     *_obs_lm   local landmark index          *_obs_kf  local keyframe index (obs_aux(4)), or -1 - k for fixed_T[k]
 *     pt_obs_xy [.][2] observed pixel          ls_obs_le [.][3] observed (normalised) line equation
 *   pt_moved / ls_moved (may be NULL): 1 where the landmark moved by more than 0.01 - the reference then clears its
 *     inlier flag (:1826-1851).
 * opts: lambda / lambda_k / max_iters = SlamConfig::lambdaLbaLM / lambdaLbaK / maxItersLba (src/slamConfig.cpp:64-66);
 * ref_quirks = 1 reproduces four oddities of the reference as written (oracle/lba.c lists them with their lines),
 * 0 follows its evident intent.  Returns PLF_ERR_INVALID for an empty problem (the reference returns -1, :1324-1328), NULL
 * arrays, ungrouped observations or out-of-range indices, and PLF_ERR_CAPACITY beyond 64 local keyframes.  A landmark
 * without observations, or whose first-pass block (the sum of w Jx Jx^T over its rows) has an exactly zero diagonal
 * entry - e.g. one seen once, at its exact projection - is refused with PLF_ERR_INVALID naming it, before any step and
 * with the inputs unchanged: the reference would factor a zero pivot (its SimplicialLDLT's failure is not checked),
 * and the landmark, then every keyframe that observes it, would turn NaN.  The context stays usable after any error. */
typedef struct plf_lba_opts {
  double lambda, lambda_k;
  int max_iters;
  double homog_th, min_error, min_error_change;
  int ref_quirks;
} plf_lba_opts;
typedef struct plf_lba_problem {
  int n_kf, n_pt, n_ls, n_fixed;
  double* kf_pose;
  double* pt;
  double* ls;
  const double* fixed_T;
  int n_pt_obs;
  const int* pt_obs_lm;
  const int* pt_obs_kf;
  const double* pt_obs_xy;
  int n_ls_obs;
  const int* ls_obs_lm;
  const int* ls_obs_kf;
  const double* ls_obs_le;
  uint8_t* pt_moved;
  uint8_t* ls_moved;
} plf_lba_problem;
typedef struct plf_lba_result {
  int iters;     /* value of the reference's loop counter at exit */
  double err;    /* last normalised weighted error */
  double lambda; /* final damping */
} plf_lba_result;
plf_status plf_local_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* problem, plf_lba_result* out);

/* Global bundle adjustment.  Replaces MapHandler::levMarquardtOptimizationGBA (src/mapHandler.cpp:2101-2699), the
 * numerical core of MapHandler::globalBundleAdjustment (:1995-2099): the same Levenberg-Marquardt as plf_local_ba over
 * every live keyframe except keyframe 0 and every landmark of the map.  The problem has plf_local_ba's layout, assembled
 * as :1995-2090 does:
 *   kf_pose  x_kf_w of every live keyframe except keyframe 0, in kf_idx order (:2001-2014), in / out
 *   pt / ls  every point / line landmark, in map order, in / out
 *   fixed_T  T_kf_w of keyframe 0 (and of any other keyframe the caller holds fixed)
 *   observations grouped per landmark in ascending landmark order (:2017-2090).  Observations made by erased keyframes
 *   are skipped by the reference (:2131, :2239), so the caller leaves them out, and leaves out a landmark whose
 *   observations all came from erased keyframes: a landmark without observations is refused.
 *   pt_moved / ls_moved may be NULL (the reference has no such write-back; they are filled as plf_local_ba fills them).
 * opts: lambda / lambda_k / max_iters = SlamConfig::lambdaLbaLM / lambdaLbaK / maxItersLba, which GBA reuses (:2116, :2391);
 * min_error = min_error_change = DBL_EPSILON, the literals of :2637, :2667.  ref_quirks = 1 reproduces six oddities of
 * the reference as written (oracle/gba.py lists them as g1-g6 with their lines), 0 follows its evident intent.
 * Limits: n_kf <= 4096 (else PLF_ERR_CAPACITY).  PLF_ERR_INVALID for an empty problem, a landmark without observations
 * or with a zero diagonal entry in its first-pass block (as plf_local_ba), ungrouped observations, out-of-range indices
 * or NULL arrays; the context stays usable after any error.
 * Work is enqueued on plf_stream and uses scratch slot 10 (shared with plf_local_ba), which stays allocated until
 * plf_destroy: about 288 n_kf^2 bytes for the dense reduced system (1.2 GB at 2048 keyframes, 4.8 GB at 4096) plus
 * 144 bytes per observation and about 650 bytes per landmark.  Up to n_kf = 64 the reduced system is factored by one CTA as in
 * plf_local_ba; beyond, by a tiled LDL^T across the GPU that skips exactly-zero tiles. */
plf_status plf_global_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* problem, plf_lba_result* out);

/* Loop-closure pose-graph optimisation.  Replaces the g2o call of MapHandler::loopClosureOptimizationCovGraphG2O
 * (src/mapHandler.cpp:4185-4410): computeInitialGuess() then optimize(max_iters) of g2o's Levenberg-Marquardt over
 * VertexSE3 / EdgeSE3 with identity information and g2o's 10 trials per iteration.  The caller builds the graph as
 * :4198-4290 do and writes the poses back as :4298-4398 do (INTEGRATION.md §4 f7):
 *   T     [n_v][16]  row-major isometries (T_kf_w of the live keyframes 0 .. kf_curr_idx, in id order), in / out
 *   fixed [n_v]      1 for a vertex held fixed (keyframe 0)
 *   from / to / Z [n_e]  edge k measures Z[k] (row-major) between vertex from[k] (g2o's vertex 0) and to[k]: the error
 *                    is the MQT vector (t; q_x, q_y, q_z), w >= 0, of Z^-1 T_from^-1 T_to.  Edges in creation order:
 *                    the kf2kf edges (i asc, j asc), then the loop edges, measuring expmap_se3(lc_pose).
 * Initial guess: a breadth-first search from the fixed vertices (ascending id), visiting each vertex's edges in the
 * order given, sets every reached free vertex to parent * Z (parent = from) or parent * Z^-1.  A vertex without edges is
 * never touched; an edge between two fixed vertices adds to chi2 only.  Each trial solves (H + lambda I) x = b with the
 * tiled LDL^T of plf_global_ba; H and b are summed in a fixed order, so two calls give bit-identical results.
 * opts: max_iters = SlamConfig::maxItersPGO (100; 0 returns the initial guess), lambda_init = setUserLambdaInit (1e-10).
 * out: iterations run, the stop reason (PLF_PGO_STOP_*), trials over the call, chi2 after the initial guess, final
 *   chi2 and lambda; trace (may be NULL) receives the first trace_cap trials, n_trace of them (g2o's verbose output).
 * Limits: at most 4096 free vertices with edges (PLF_ERR_CAPACITY, before any allocation).  PLF_ERR_INVALID for NULL
 * arrays, out-of-range or self edges, non-finite T or Z, a lambda_init that is not positive and finite (g2o would derive
 * one from H instead), and a connected component with edges but no fixed vertex.  The context stays usable after any
 * error.  Work is enqueued on plf_stream and uses scratch slot 10 (shared with the bundle adjustments): 288 n_free^2
 * bytes for the dense system (4.8 GB at 4096 free vertices) plus about 790 bytes per edge, 260 per vertex and 200 per
 * free vertex; out->scratch_bytes reports what the call carved. */
enum { PLF_PGO_STOP_MAX_ITERS = 0, PLF_PGO_STOP_TRIALS = 1, PLF_PGO_STOP_RHO_ZERO = 2, PLF_PGO_STOP_LAMBDA = 3 };
typedef struct plf_pgo_opts {
  int max_iters;
  double lambda_init;
} plf_pgo_opts;
typedef struct plf_pgo_problem {
  int n_v, n_e;
  double* T;
  const uint8_t* fixed;
  const int* from;
  const int* to;
  const double* Z;
} plf_pgo_problem;
typedef struct plf_pgo_trial {
  int iter, accepted;
  double lambda;   /* the damping the trial solved with */
  double chi, chi_t, rho;
} plf_pgo_trial;
typedef struct plf_pgo_result {
  int iters, stop, trials;
  double chi2_init, chi2, lambda;
  plf_pgo_trial* trace;  /* in: caller's array (may be NULL) */
  int trace_cap;         /* in */
  int n_trace;           /* out: min(trials, trace_cap) */
  size_t scratch_bytes;  /* out: device scratch the call carved */
} plf_pgo_result;
plf_status plf_pose_graph(plf_ctx* ctx, const plf_pgo_opts* opts, const plf_pgo_problem* problem, plf_pgo_result* out);

/* Relative pose between two keyframes (SURVEY 8(f) f2).  Replaces MapHandler::isLoopClosure (src/mapHandler.cpp:3192-3300:
 * match() on the points :3223 and on the lines :3249 of kf0 / kf1, the inlier-ratio pre-condition :3277-3299) followed by
 * MapHandler::computeRelativePoseRobustGN (:3566-3957: two-stage robust GN from identity with the chi2 gate in between,
 * both stages stopping on DBL_EPSILON; acceptance tests residual / covariance eigenvalue / translation / rotation
 * :3875-3906; pose_inc = logmap_se3(inverse_se3(expmap_se3(x_inc))) :3951).  max_iters / max_iters_ref, min_ratio_12_*,
 * has_points / has_lines, best_lr_matches and homog_th come from the ctx params (SlamConfig inherits them). */
typedef struct plf_lc_params {
  double lc_res;          /* SlamConfig::lcRes()  src/slamConfig.cpp:73  (config_euroc.yaml:116: 1.5) */
  double lc_unc;          /* lcUnc  :74   maximum largest eigenvalue of H^-1 */
  double lc_inl;          /* lcInl  :75   (evaluated but overridden by the reference, mapHandler.cpp:3900) */
  double lc_trs;          /* lcTrs  :76 */
  double lc_rot;          /* lcRot  :77   degrees */
  double lc_inlier_ratio; /* lcInlierRatio :83, percent */
} plf_lc_params;
typedef struct plf_lc_keyframe {  /* the stereo-valid features of a KeyFrame's frame (host arrays) */
  int n_pt, n_ls;
  const uint8_t* pdesc; /* n_pt x 32  stereo_frame->pdesc_l */
  const double* P;      /* n_pt x 3   stereo_pt[i]->P   (read for kf0) */
  const double* pl;     /* n_pt x 2   stereo_pt[i]->pl  (read for kf1) */
  const uint8_t* ldesc; /* n_ls x 32 */
  const double* sP;     /* n_ls x 3   (kf0) */
  const double* eP;     /* n_ls x 3   (kf0) */
  const double* le;     /* n_ls x 3   stereo_ls[i]->le (kf1) */
} plf_lc_keyframe;
typedef struct plf_lc_result {
  int accepted;        /* the reference's return value */
  int estimated;       /* 0: stopped at the inlier-ratio pre-condition */
  int common_pt, common_ls;
  int n_pt, n_ls;      /* inlier correspondences written to pt_pairs / ls_pairs (accepted only) */
  double inl_ratio_pt, inl_ratio_ls;
  double err, max_cov_eig, ratio_inliers, t, r;
  double x_inc[6];     /* logmap_se3(T_inc) */
  double pose_inc[6];  /* accepted only */
} plf_lc_result;
/* pt_pairs / ls_pairs: (i1 in kf0, i2 in kf1) per surviving correspondence, capacity cap_* pairs (may be NULL). */
plf_status plf_loop_closure_pose(plf_ctx* ctx, const plf_lc_params* lc, const plf_lc_keyframe* kf0,
                                 const plf_lc_keyframe* kf1, plf_lc_result* out, int32_t* pt_pairs, int cap_pt,
                                 int32_t* ls_pairs, int cap_ls);

/* se(3) helpers of stvo-pl auxiliar.h used throughout src/mapHandler.cpp (e.g. :137-142,:3439,:3558):
 * op 0 = expmap_se3 (in: 6 = [t; w], out: 16 row-major), op 1 = logmap_se3 (in: 16, out: 6). */
plf_status plf_se3(plf_ctx* ctx, int op, const double* in, double* out);

/* ------------------------------------------------------------------------------------------------
 * Batched per-frame front-end (SURVEY §8 a6, a7, a10; call pattern app/plslam_dataset.cpp:111-163)
 * ---------------------------------------------------------------------------------------------- */

/* What StereoFrameHandler exposes after insertStereoPair + optimizePose for one frame. */
typedef struct plf_frame_result {
  double DT[16];     /* curr_frame->DT = inverse_se3(optimised increment), row-major; identity if status != 0 */
  double DT_cov[36]; /* curr_frame->DT_cov */
  double err;        /* curr_frame->err_norm (-1 when no optimisation ran) */
  int status;        /* 0 = tracked, 1 = fewer than min_features correspondences, 2 = first frame (initialize) */
  int n_kp_l, n_kp_r, n_lines_l, n_lines_r; /* detected features per image */
  int n_stereo_pt, n_stereo_ls;             /* stereo_pt.size(), stereo_ls.size() */
  int n_matched_pt, n_matched_ls;           /* matched_pt.size(), matched_ls.size() */
  int n_inliers_pt, n_inliers_ls;           /* n_inliers_pt, n_inliers_ls */
  int iters1, iters2;
} plf_frame_result;

/* Host destination for the stereo-valid features of one frame (the StereoFrame fields KeyFrame copies,
 * src/keyFrame.cpp:39-53; row i of pdesc/ldesc <-> stereo_pt[i]/stereo_ls[i]).  Any array may be NULL. */
typedef struct plf_frame_view {
  int cap_pt, cap_ls;  /* in: capacity of the arrays; out: n_pt / n_ls filled */
  int n_pt, n_ls;
  double* pt_pl;       /* n_pt x 2   PointFeature::pl */
  double* pt_disp;     /* n_pt       PointFeature::disp */
  double* pt_P;        /* n_pt x 3   PointFeature::P */
  int32_t* pt_octave;  /* n_pt */
  uint8_t* pdesc;      /* n_pt x 32  StereoFrame::pdesc_l */
  double* ls_spl;      /* n_ls x 2   LineFeature::spl */
  double* ls_epl;      /* n_ls x 2 */
  double* ls_sdisp;    /* n_ls */
  double* ls_edisp;    /* n_ls */
  double* ls_sP;       /* n_ls x 3 */
  double* ls_eP;       /* n_ls x 3 */
  double* ls_le;       /* n_ls x 3   LineFeature::le (normalised line equation) */
  float* ls_angle;     /* n_ls */
  uint8_t* ldesc;      /* n_ls x 32  StereoFrame::ldesc_l */
} plf_frame_view;

/* Forget the previous frame (next batch starts with initialize(), app/plslam_dataset.cpp:115). */
plf_status plf_reset_sequence(plf_ctx* ctx);

/* Replaces B consecutive iterations of the VO part of the hot loop:
 *   StVO->insertStereoPair(img_l, img_r, k); StVO->optimizePose();   (app/plslam_dataset.cpp:127-128)
 * left/right: B images each, h rows of `stride` bytes, image k at offset k*stride*h (host).  out: B results.
 * The caller chains Tfw = prev.Tfw * DT (as optimizePose does) and applies its keyframe policy. */
plf_status plf_process_batch(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride,
                             plf_frame_result* out);

/* The three phases of plf_process_batch, for streaming callers and callers that keep images resident in HBM:
 * upload (asynchronous H2D into the image slot the GPU is not reading) -> run (all kernels, asynchronous; consumes the
 * most recent upload) -> download (waits for the OLDEST batch in flight and returns its B results).
 * Batches are software-pipelined on the device: up to THREE may be in flight (run, run, run, download, run, ...);
 * a fourth plf_batch_run returns PLF_ERR_STATE.  Results are identical to run/download pairs.  plf_get_frame /
 * plf_get_matches refer to the batch most recently RUN, so call them with a single batch in flight. */
plf_status plf_batch_upload(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride);
plf_status plf_batch_run(plf_ctx* ctx, int B);
plf_status plf_batch_download(plf_ctx* ctx, int B, plf_frame_result* out);
/* Poses of the OLDEST batch in flight, device to device: dst_device[B][16] f64 (DT, row-major) is filled on `stream`
 * (a cudaStream_t of the caller; NULL = an internal stream, synchronised before returning) behind that batch's match
 * phase - the buffer a multi-GPU caller passes to its NCCL pose all-gather on the same stream (SURVEY 8e; the reference
 * has no counterpart: app/plslam_dataset.cpp:148-154 reads curr_frame->Tfw on the host).  The batch stays in flight
 * until plf_batch_download. */
plf_status plf_batch_device_poses(plf_ctx* ctx, int B, double* dst_device, void* stream);
/* Device buffer [2*max_batch][h][pitch] read by plf_batch_run (image 2k = left k, 2k+1 = right k), pitch = width rounded up
 * to a multiple of 16 bytes (every halo tile of every image is then a legal TMA box). */
void* plf_batch_device_images(plf_ctx* ctx);

/* Stereo-valid features of frame k of the last batch (what `new KeyFrame(StVO->curr_frame)` deep-copies,
 * app/plslam_dataset.cpp:143, src/keyFrame.cpp:39-53). */
plf_status plf_get_frame(plf_ctx* ctx, int k, plf_frame_view* view);

/* Host destination for StereoFrameHandler::matched_pt / matched_ls of pair k (src/mapHandler.cpp:770-778 reads
 * them; fields as written by the in-tree analogue :326-328,:482-487).  Any array may be NULL. */
typedef struct plf_match_view {
  int cap_pt, cap_ls;
  int n_pt, n_ls;
  double* P;          /* n_pt x 3  PointFeature::P (previous frame) */
  double* pl_obs;     /* n_pt x 2  PointFeature::pl_obs (current frame) */
  uint8_t* inlier_pt; /* n_pt      PointFeature::inlier after optimizePose */
  double* sP;         /* n_ls x 3 */
  double* eP;         /* n_ls x 3 */
  double* le_obs;     /* n_ls x 3  LineFeature::le_obs */
  uint8_t* inlier_ls; /* n_ls */
} plf_match_view;
plf_status plf_get_matches(plf_ctx* ctx, int k, plf_match_view* view);

/* Keyframe matching (SURVEY 8(f) f1): the matching parts of MapHandler::matchKF2KFPoints / matchKF2KFLines and
 * matchMap2KFPoints / matchMap2KFLines, called by lookForCommonMatches (src/mapHandler.cpp:754-821), on the device from one
 * upload to one download: projection, visibility, compaction, GridStructure cells, matchGrid() in a +-matching_f2f_ws
 * window, the match() fallback and the epipolar gate.  The landmark bookkeeping that follows each (new MapPoint / MapLine,
 * observations, full_graph) stays with the caller.  has_points / has_lines, best_lr_matches, matching_f2f_ws,
 * min_pt_matches / min_ls_matches, min_ratio_12_p / min_ratio_12_l, line_sim_th and the camera come from the ctx (SlamConfig
 * inherits them).  Work is enqueued on plf_stream, so a call between batches in flight is safe.  A kind returns 0 (every
 * entry -1) when it is disabled or the keyframe has no stereo features of it.  Semantics reproduced as written, quirks
 * included (DESIGN.md 8): see oracle/kfmatching.py. */
typedef struct plf_kf_match_opts {
  int fast_matching;    /* SlamConfig::fastMatching  src/slamConfig.cpp:43: 0 = brute-force match() only, and only when
                           the fallback condition holds (else no pairs) */
  double max_kf_epip_p; /* SlamConfig::maxKFEpipP  :51 */
  double max_kf_epip_l; /* SlamConfig::maxKFEpipL  :52 */
} plf_kf_match_opts;

/* matchKF2KFPoints + matchKF2KFLines (src/mapHandler.cpp:234-278, :365-426), matching part.
 * prev / curr: the stereo-valid features of the two keyframes in the layout plf_get_frame fills; read: n_pt, n_ls, pt_P,
 * pdesc, ls_sP, ls_eP, ldesc (prev) and n_pt, n_ls, pt_pl, pdesc, ls_spl, ls_epl, ldesc (curr).  DT: row-major 4x4
 * (MapHandler::DT).  m_pt[prev->n_pt], m_ls[prev->n_ls]: matches_12 (curr index or -1).  *n_pt, *n_ls: the reference's
 * return values (may be NULL).  The projected query lines stay in pixels as the reference leaves them (:392-393).
 * n_pt, n_ls <= 8192 per keyframe; device scratch 2 x prev->n_* x curr->n_* bytes per kind, kept until plf_destroy. */
plf_status plf_match_kf2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_frame_view* prev,
                           const plf_frame_view* curr, const double DT[16], int32_t* m_pt, int32_t* m_ls, int* n_pt,
                           int* n_ls);

/* The landmarks of MapHandler::map_points / map_lines, in index order (host arrays). */
typedef struct plf_local_map {
  int n_pt;
  const double* pt_X;      /* [n_pt][3] MapPoint::point3D */
  const uint8_t* pt_desc;  /* [n_pt][32] MapPoint::med_desc */
  const uint8_t* pt_use;   /* [n_pt] 1 = non-null && local && kf_obs_list.back() != kf_idx (:547); NULL = all */
  int n_ls;
  const double* ls_X;      /* [n_ls][6] MapLine::line3D (start | end) */
  const uint8_t* ls_desc;  /* [n_ls][32] */
  const uint8_t* ls_use;   /* [n_ls] (:648); NULL = all */
} plf_local_map;

/* matchMap2KFPoints + matchMap2KFLines (src/mapHandler.cpp:532-632, :634-752): visibility, matching and the epipolar gate.
 * Twf: row-major 4x4 (MapHandler::Twf).  kf: read n_pt, n_ls, pt_pl, pdesc, ls_spl, ls_epl, ls_le, ldesc.
 * kf_pt_lm / kf_ls_lm: the keyframe features' landmark index, -1 = unmatched (:565, :670); NULL = all unmatched.
 * lm_pt[map->n_pt], lm_ls[map->n_ls]: per landmark (original index) the keyframe feature (original index) it was matched
 * to and that passed the gate, else -1.  *n_pt / *n_ls: the reference's return values (matches minus gate rejects).
 * At most 65535 landmarks and 8192 keyframe features per kind.  Device scratch: the windowed matcher's distance matrix is
 * sized from the uncompacted counts, 2 x (map->n_*) x (kf->n_*) bytes per kind (about 1 GB at both limits), and stays
 * allocated in the ctx (scratch grows, never shrinks) until plf_destroy. */
plf_status plf_match_map2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_local_map* map, const double Twf[16],
                            const plf_frame_view* kf, const int32_t* kf_pt_lm, const int32_t* kf_ls_lm, int32_t* lm_pt,
                            int32_t* lm_ls, int* n_pt, int* n_ls);

/* ------------------------------------------------------------------------------------------------
 * Place recognition: DBoW2 bag-of-words vectors and L1 scores (SURVEY 8(f) f5)
 * ---------------------------------------------------------------------------------------------- */

/* A DBoW2 TemplatedVocabulary<FORB> as its YAML file lists it (3rdparty/DBoW2/include/DBoW2/TemplatedVocabulary.h:1437-1486):
 * the nodes in FILE order (the root, id 0, is not listed; a parent's children keep file order, which decides ties in the
 * descent), then the words.  Node ids must be 1..n_nodes.  Only scoring 0 (L1_NORM) and weighting 0 (TF_IDF), the types of
 * pl-slam's vocabularies, are supported. */
typedef struct plf_vocab {
  int k, L, scoring, weighting;
  int n_nodes;
  int32_t* node_id;   /* [n_nodes] */
  int32_t* parent_id; /* [n_nodes] */
  double* weight;     /* [n_nodes] idf weight; a word of weight <= 0 drops the features that reach it (:1073) */
  uint8_t* desc;      /* [n_nodes][32] */
  int n_words;
  int32_t* word_id;   /* [n_words] */
  int32_t* word_node; /* [n_words] */
} plf_vocab;

/* Reads a vocabulary YAML file in the form TemplatedVocabulary::save writes and load reads (:1317-1486), e.g. the files of
 * the reference's vocabulary/voc.tar.gz.  Host only (no device, no ctx); errors: plf_last_error(NULL).  PLF_ERR_INVALID for
 * a malformed file: scoring other than L1 or weighting other than TF-IDF, k outside 1..32, duplicate or out-of-range node
 * ids, a missing parent or a cycle, more than k children, a leaf without a word or a word on an inner node, duplicate or
 * out-of-range word ids, a descriptor that is not 32 integers in 0..255.  On success the arrays are malloc'ed; release
 * them with plf_vocab_free.  A plf_vocab may also be filled by the caller from its own arrays. */
plf_status plf_vocab_read_yml(const char* path, plf_vocab* out);   /* numbers are read in the C locale */
void plf_vocab_free(plf_vocab* v);

/* Uploads the vocabulary of kind 0 (points, ORB) or 1 (lines, LBD), validated by the rules of plf_vocab_read_yml, and
 * empties that kind's database.  The tree is stored re-laid out by parent (each node's children contiguous, in file order):
 * 48 bytes per node. */
plf_status plf_bow_set_vocabulary(plf_ctx* ctx, int kind, const plf_vocab* voc);

/* Replaces the transform and scoring part of MapHandler::insertKFBowVectorP / L / PL (src/mapHandler.cpp:3007-3128) and the
 * transform of MapHandler::initialize (:82-98): the BoW vectors of the keyframe's stereo descriptors, kf->pdesc [n_pt][32]
 * and kf->ldesc [n_ls][32] (the rows of pdesc_l / ldesc_l), are computed with TemplatedVocabulary::transform (:1046-1101,
 * :1198-1239), stored under kf_idx, and scored with L1Scoring::score (ScoringObject.cpp:23-68) against every keyframe
 * stored before: score_p / score_l [kf_idx + 1] (either may be NULL), entry i = score(v_kf_idx, v_i), entry kf_idx the
 * self-score, NaN for an index never inserted or erased.  Bit-exact to DBoW2 (sums in its order).  A kind disabled by
 * has_points / has_lines is not touched (its row is left as it is) and needs no vocabulary; an enabled kind without one
 * returns PLF_ERR_STATE.  kf_idx must exceed every index inserted into the kind before (gaps are absent keyframes) and be
 * below 2^24; n_pt, n_ls <= 8192.  Other values return PLF_ERR_INVALID and change nothing.  One upload, kernels on
 * plf_stream, one download.  Database, per kind: 12 bytes per stored (word, value) entry plus 8 bytes per keyframe index;
 * it grows by reallocation (doubling) and never shrinks until the vocabulary is set again or plf_destroy.  At most 2^31 - 1
 * entries per kind (PLF_ERR_CAPACITY beyond, nothing changed). */
plf_status plf_bow_insert(plf_ctx* ctx, int kf_idx, const plf_frame_view* kf, double* score_p, double* score_l);

/* The counterpart of removeRedundantKFs deleting a keyframe (src/mapHandler.cpp:2931-2932): later rows report NaN for it.
 * Erasing an absent index is a no-op; kf_idx < 0 returns PLF_ERR_INVALID. */
plf_status plf_bow_erase(plf_ctx* ctx, int kf_idx);

/* The stored BowVector (KeyFrame::descDBoW_P / descDBoW_L) of keyframe kf_idx, kind 0 / 1, in ascending word order: *n
 * entries.  words / values may be NULL to query *n; PLF_ERR_CAPACITY if *n > cap.  An absent keyframe or a kind never
 * inserted returns PLF_ERR_INVALID. */
plf_status plf_bow_get(plf_ctx* ctx, int kf_idx, int kind, int cap, uint32_t* words, double* values, int* n);

/* Debug: device-clock timeline (ms) of the two most recent batches of the software pipeline: for each, the start/end of
 * the E (extract), G (region growing) and M (match/track/pose) phases relative to the older batch's E start.
 * No reference counterpart (the reference times whole calls with its Timer, app/plslam_dataset.cpp:126-132). */
plf_status plf_debug_timeline(plf_ctx* ctx, float out[12]);

#ifdef __cplusplus
}
#endif
#endif /* PLSLAM_B200_H */
