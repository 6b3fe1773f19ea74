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
  PLF_ERR_CAPACITY = -4,  /* a fixed-capacity device buffer overflowed: a plf_limits field or one of the internal
                           * capacities listed below plf_limits; plf_last_error names the one that was hit */
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
/* Internal capacities of the extraction kernels, not fields of plf_limits (DESIGN.md section 8).  Rendered and natural
 * images stay far below them; an image built for it can reach each, the call then returns PLF_ERR_CAPACITY, never a
 * truncated result, and plf_last_error names it - raising plf_limits does not move them:
 *   ORB_SORT_CAP = 4096   keypoints kept on ONE pyramid level (csrc/orb.cu, k_select_sort).  retainBest keeps every
 *                         corner that ties the level's threshold score, so a binary image of several thousand equal
 *                         corners reaches it whatever orb_nfeatures is; so does an orb_nfeatures that gives one level a
 *                         share above 4096 (about 12 700 at 4 levels) on an image with that many corners.  At the default
 *                         max_keypoints (4096) the declared limit is always met first.
 *   candidate capacity    FAST corners (after the 3 x 3 suppression) of ONE pyramid level: min(w h / 9 + 64, 32768) of
 *                         the level's size (csrc/orb.cu, k_fast_nms).  Isolated bright pixels every 4 columns and rows
 *                         give w h / 16 corners: above 32768 from about 760 x 760 or 1280 x 720 upwards.
 *   KL_SORT_CAP = 4096    KeyLines of one image that can be ranked for the top lsd_nfeatures (csrc/lsd.cu, k_keylines);
 *                         lsd_nfeatures = 0 ranks nothing and is bounded by max_segments / max_lines only. */

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

/* Test hook: the batched windowed matcher (that of matching_strategy 3 and of plf_match_kf2kf / plf_match_map2kf's
 * fast_matching), unchanged, on n_prob problems laid out at uniform capacities K (queries) and Kt (train features):
 *   q_geo [n_prob][K][2|4]  points: query cells (x, y); lines: integer end points (x1, y1, x2, y2), in grid cells;
 *   t_geo [n_prob][Kt][2|4] the train cells / end points (a train line is in each cell of its Bresenham walk);
 *   t_dir [n_prob][Kt][2]   lines: directions2 (may be NULL for points);
 *   d1 [n_prob][K][32], d2 [n_prob][Kt][32], n1 [n_prob], n2 [n_prob]: the counts, each clamped to K / Kt;
 *   q_slot [n_prob] or NULL: problem p reads the query descriptors and count of slot q_slot[p] (d1 and n1), and its own
 *   query geometry q_geo[p].
 * The grid is grid_cols x grid_rows cells with window w; clip (lines) walks only the steps of a query line whose window
 * can reach the grid, for queries far outside it.  Out: matches_12 [n_prob][K] (-1 past the problem's count) and
 * n_matches [n_prob].  PLF_ERR_INVALID before any work for n_prob outside [0, 65535], K outside [0, 65535], Kt outside
 * [0, 8192], a grid of no cell or of more than 4096 cells, a q_slot entry outside [0, n_prob), a negative count or a
 * NULL array. */
plf_status plf_debug_match_grid_batch(plf_ctx* ctx, int n_prob, int K, int Kt, const int* q_geo, const int* t_geo,
                                      const double* t_dir, const uint8_t* d1, const uint8_t* d2, const int* n1,
                                      const int* n2, const int* q_slot, int grid_cols, int grid_rows, plf_grid_window w,
                                      int is_lines, int clip, float nnr, double line_sim_th, int best_lr,
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
 * the count (PLF_ERR_CAPACITY if it exceeds cap, the ctx limit max_keypoints or an internal capacity listed below
 * plf_limits; nothing is written to kps / desc then, and the next call starts clean).  Work is enqueued on plf_stream in a
 * working state of its own (one image, rebuilt when the image size changes) and never touches the batched pipeline's
 * buffers, so a call between batches in flight is safe. */
/* img is 8-bit single-channel (grey); colour input is the batched pipeline's only (plf_batch_upload_color). */
plf_status plf_orb(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, plf_keypoint* kps,
                   uint8_t* desc, int cap, int* n);

/* plf_orb restricted to a mask: cv::ORB::detectAndCompute(img, mask, ...).  mask: w x h uint8 host array, mask_stride bytes
 * per row (>= w), any non-zero value allowing a corner.  Pyramid level l >= 1 uses resize(mask of level l-1,
 * INTER_LINEAR_EXACT) thresholded to 255 (THRESH_TOZERO at 254), as OpenCV builds it, so a pixel near a mask edge is
 * masked on the coarser levels.  FAST and its non-maximum suppression run on the whole image; masked corners are dropped
 * after them, before the per-level retainBest, so the level quotas fill from allowed corners (a masked corner still
 * suppresses a weaker allowed neighbour).  An all-zero mask gives no keypoints.  Same buffers, errors and working state as
 * plf_orb; PLF_ERR_INVALID for a NULL mask or mask_stride < w. */
plf_status plf_orb_masked(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, const uint8_t* mask, int mask_stride,
                          plf_keypoint* kps, uint8_t* desc, int cap, int* n);

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
 * output order (seed order).  *n receives the count (PLF_ERR_CAPACITY beyond cap or max_segments: nothing is written to
 * segs, and the next call starts clean).  Work is enqueued on plf_stream in a working state of its own (one
 * image, rebuilt when the image size changes, shared with plf_detect_lines) and never touches the batched pipeline's
 * buffers, so a call between batches in flight is safe. */
/* img is 8-bit single-channel (grey), as for plf_orb.  The segments are raw: no mask applies to them (the masks of
 * plf_detect_lines_masked and plf_set_sequence_mask act on KeyLines). */
plf_status plf_lsd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, float* segs, int cap, int* n);

/* Line features of one image.  Replaces stvo-pl StereoFrame::detectLineFeatures (LSD branch):
 * LSDDetectorC::detect(img, lines, scale, 1, opts) (LSDDetector_custom.cpp:218-324, opts.min_length =
 * min_line_length * min(w,h)), then — when more than lsd_nfeatures lines are found and lsd_nfeatures != 0 — sort by
 * response (descending; ties keep detection order), keep lsd_nfeatures and set class_id = rank, then
 * BinaryDescriptor::compute (binary_descriptor_custom.cpp:524).  keylines/desc: host buffers of `cap` entries
 * (PLF_ERR_CAPACITY beyond cap, max_segments, max_lines or - when lines are ranked - KL_SORT_CAP).
 * Enqueued on plf_stream in plf_lsd's working state; never touches the batched pipeline's buffers, so a call between
 * batches in flight is safe. */
/* img is 8-bit single-channel (grey), as for plf_orb. */
plf_status plf_detect_lines(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                            plf_keyline* keylines, uint8_t* desc, int cap, int* n);

/* plf_detect_lines restricted to a mask: LSDDetectorC::detect(img, lines, scale, 1, opts, mask).  mask: w x h uint8 host
 * array, mask_stride bytes per row (>= w).  After the end point clamp and the min_length filter, a KeyLine is deleted when
 * the mask is 0 at both (int)-truncated end points (LSDDetector_custom.cpp:310-322); one allowed end point keeps it.  The
 * survivors keep the class_id the length filter gave them; the lsd_nfeatures top-K then ranks the survivors only.  Same
 * buffers, errors and working state as plf_detect_lines; PLF_ERR_INVALID for a NULL mask or mask_stride < w. */
plf_status plf_detect_lines_masked(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, const uint8_t* mask,
                                   int mask_stride, plf_keyline* keylines, uint8_t* desc, int cap, int* n);

/* Test hook: evaluates the device port of glibc sinf/cosf used by the LSD region-angle update. */
plf_status plf_debug_sincosf(plf_ctx* ctx, const float* in, float* s, float* c, int n);

/* Test hook: the gradient stage of LSD (pre-blur, resample and gradient in one kernel) on n w x h uint8 images (row pitch
 * `pitch`, image stride img_stride bytes, both multiples of 16).  sizes[6] receives {ws, hs, nxb, KS, TH, P}: the scaled
 * size, the 512-column segments per row, and the kernel's launch (pre-blur taps, scaled rows per CTA, column pieces per
 * segment); with any output NULL nothing runs.  Outputs: pix [n][hs*ws] records as 2 uint32 {angle bits, table index}
 * (untouched pixels read {-1024.f, 0}), seedlist [n][hs*ws] (entries past a segment's count read 0), segcnt [n][hs][nxb],
 * maxmag2 [n]. */
plf_status plf_debug_lsd_pre(plf_ctx* ctx, const uint8_t* imgs, int n, int w, int h, int pitch, size_t img_stride,
                             int* sizes, uint32_t* pix, uint32_t* seedlist, int* segcnt, int* maxmag2);

/* Test hook: factors the symmetric n x n matrix S (n = 6 n6, row-major, only its lower triangle is read) as L D L^T
 * without pivoting and solves S x = g, with the factorisation of plf_global_ba / plf_pose_graph beyond 64 keyframes
 * (path 0: the tiled one, 1 <= n6 <= 4096, as one system on its own) or that of plf_local_ba (path 1: one CTA,
 * 1 <= n6 <= 64).  On return the lower triangle of S holds
 * L strictly below the diagonal and D on it (entries above the diagonal are unspecified), x the solution, and nz
 * (path 0 only, may be NULL; n_t x n_t bytes, n_t = ceil(n / 64)) the zero flag of each L tile (i > k) as the panel
 * kernel set it, 0 elsewhere.  A bad path, an n6 out of range or a NULL S, g or x returns PLF_ERR_INVALID. */
plf_status plf_debug_ldlt(plf_ctx* ctx, int path, int n6, double* S, const double* g, double* x, uint8_t* nz);

/* Test hook: plf_debug_ldlt's path 0 on n matrices of mixed sizes in one launch chain, the batched tiled LDL^T of
 * plf_global_ba_batch: matrix i is n6[i] (1 <= n6[i] <= 4096) with S[i], g[i], x[i] and nz[i] (nz or nz[i] may be NULL)
 * as plf_debug_ldlt takes them, and comes out as plf_debug_ldlt(ctx, 0, ...) leaves it.  n < 0, n > 65535, an n6 out of
 * range or a NULL S, g or x returns PLF_ERR_INVALID; n = 0 returns PLF_OK. */
plf_status plf_debug_ldlt_batch(plf_ctx* ctx, int n, const int* n6, double* const* S, const double* const* g,
                                double* const* x, uint8_t* const* nz);

/* LBD prelude: GaussianBlur 5x5 sigma 1 then Sobel k=3 to CV_16S.  Replaces
 * BinaryDescriptor::computeSobel (binary_descriptor_custom.cpp:373-398 -> :350-370).
 * img: h rows of `stride` bytes (host). dxdy: h*w interleaved int16 pairs (dx,dy) (host). */
plf_status plf_lbd_gradients(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, int16_t* dxdy);

/* LBD descriptors.  Replaces BinaryDescriptor::compute(image, keylines, descriptors, returnFloat)
 * (binary_descriptor_custom.cpp:524-528 -> computeImpl :539-687 -> computeLBD :1026-1372).
 * Uses from each KeyLine: sPointInOctave*, ePointInOctave*, numOfPixels, angle (octave 0 only, as the
 * front-end calls it).  desc: n x 32 bytes (host).  desc_float (optional): n x 72 floats.
 * n == 0 returns PLF_OK without touching desc (the reference prints a message and returns). */
/* img is 8-bit single-channel (grey), as for plf_orb. */
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
 * 4x4 or NULL (identity).  opts NULL => thresholds from the ctx params (stvo-pl min_error/min_error_change).
 * Projects with the context's camera (plf_create); plf_gn_pose_batch takes a sequence's. */
plf_status plf_gn_pose(plf_ctx* ctx, const plf_gn_opts* opts, const double* P, const double* pl_obs,
                       uint8_t* inlier_pt, int np, const double* sP, const double* eP,
                       const double* le_obs, uint8_t* inlier_ls, int nl, const double* T_init,
                       plf_pose_result* out);

/* Many pose refinements in one call: the lookForCommonMatches refinements (src/mapHandler.cpp:768-808) of several
 * sequences' new keyframes, each with its sequence's camera, in one upload, one launch and one download with one host
 * synchronisation.
 *   problems [n_problems]  plf_gn_pose's arguments per problem (inlier flags in / out, out: its result)
 *   seq      [n_problems]  or NULL: the camera of problem p.  seq[p] = -1 (or seq NULL) uses the context's camera;
 *                          0 <= seq[p] < n (plf_set_max_sequences) uses what plf_get_sequence_camera(ctx, seq[p]) returns
 *                          at the time of the call.  Only fx, fy, cx and cy enter.
 * One opts serves every problem (NULL = the ctx params, as plf_gn_pose).  Problem p's out and inlier flags are
 * bit-identical to what plf_gn_pose returns for it on a context created with its camera: the solver sums in a fixed order,
 * so the same rows in the same order give the same bits.  plf_gn_pose is this call with one problem.
 * Refusals before any work, naming the problem and the rule, with nothing written: PLF_ERR_INVALID when n_problems < 0, a
 * seq entry is out of range, or a count is negative or an array NULL while its count is > 0.  n_problems = 0 returns
 * PLF_OK and launches nothing.  Launches: 1.  Work is enqueued on plf_stream; device scratch (plf_gn_pose's slot, kept
 * until plf_destroy): 41 bytes per point row, 73 per line row and about 0.8 KB per problem, each part rounded up to 256
 * bytes; the context's pinned staging buffer holds the inputs and outputs. */
typedef struct plf_gn_problem {
  const double* P; const double* pl_obs; uint8_t* inlier_pt; int np;   /* as plf_gn_pose; inlier flags in / out */
  const double* sP; const double* eP; const double* le_obs; uint8_t* inlier_ls; int nl;
  const double* T_init;          /* NULL = identity */
  plf_pose_result out;           /* out */
} plf_gn_problem;
plf_status plf_gn_pose_batch(plf_ctx* ctx, const plf_gn_opts* opts, int n_problems, plf_gn_problem* problems,
                             const int32_t* seq);

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
/* Projects with the context's camera (plf_create), not a sequence's (plf_set_sequence_camera); plf_local_ba_batch
 * takes a sequence's.  The call is plf_local_ba_batch's launch chain with one problem: all opts.max_iters rounds are
 * enqueued at once and a round after the problem has stopped still costs its eight launches (each returning at once),
 * so the call's time grows with max_iters, not with the iterations run; one host synchronisation, after the download.
 * Work is enqueued on plf_stream and uses the scratch slot plf_global_ba and plf_pose_graph use (not
 * plf_local_ba_batch's), which stays allocated until plf_destroy: the sizes plf_local_ba_batch lists for one problem. */
plf_status plf_local_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* problem, plf_lba_result* out);

/* Many local bundle adjustments in one call: the local maps of several sequences' new keyframes, each with its
 * sequence's camera, solved in one launch chain with one host synchronisation (after the download).
 *   problems [n_problems]  plf_local_ba's layout and rules, each in / out as in plf_local_ba
 *   seq      [n_problems]  or NULL: the camera of problem p.  seq[p] = -1 (or seq NULL) uses the context's camera;
 *                          0 <= seq[p] < n (plf_set_max_sequences) uses what plf_get_sequence_camera(ctx, seq[p]) returns
 *                          at the time of the call.  Only fx, fy, cx and cy enter the LBA.
 *   out      [n_problems]  or NULL;  status [n_problems], required.
 * Problem p gets the result plf_local_ba(ctx, opts, &problems[p], &out[p]) gives with problem p's camera: the same
 * iteration count and exit, moved flags, lambda and err to rounding, every block to rounding of the step (the sums are
 * float atomics, as in plf_local_ba: no bit-reproducibility promise).  One opts applies to every problem.
 * Refusals before any work: PLF_ERR_INVALID or PLF_ERR_CAPACITY, and nothing is written (no problem's arrays, out or
 * status), when n_problems < 0, a seq entry is out of range, or any problem breaks one of plf_local_ba's host-side rules
 * (empty problem, NULL arrays, ungrouped observations, out-of-range indices, a landmark without observations, more than
 * 64 local keyframes); the message names the problem index and the rule.  n_problems = 0 returns PLF_OK.
 * Refusal on the device: a landmark whose first-pass block has an exactly zero diagonal entry refuses its problem only:
 * status[p] = PLF_ERR_INVALID, and its arrays and out[p] are left unchanged.  Every other problem is solved and written
 * back with status PLF_OK.  The call then returns PLF_ERR_INVALID, and plf_last_error names the first refused problem and
 * its landmark; else PLF_OK.  The context stays usable after any error.
 * All opts.max_iters rounds are enqueued at once, and a round in which every problem has stopped still costs its eight
 * launches (each returning at once), so the call's time grows with max_iters, not with the iterations run.
 * Work is enqueued on plf_stream and uses its own scratch slot (not plf_local_ba's), which stays allocated until
 * plf_destroy: 144 bytes per observation, 629 per landmark plus 24 per landmark coordinate (X, X0 and the step), 704 per
 * local keyframe, 288 per local keyframe^2 of each problem, 256 per fixed keyframe and about 240 per problem, each part
 * rounded up to 256 bytes; the context's pinned staging buffer holds the inputs and outputs.  The rules for batches in
 * flight are plf_local_ba's. */
plf_status plf_local_ba_batch(plf_ctx* ctx, const plf_lba_opts* opts, int n_problems, const plf_lba_problem* problems,
                              const int32_t* seq, plf_lba_result* out, plf_status* status);

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
 * The call is plf_global_ba_batch's launch chain with one problem: all opts.max_iters rounds are enqueued at once, and
 * a round after the problem has stopped still costs its launches (8, plus 5 n_t + 1 beyond 64 keyframes, each returning
 * at once), so the call's time grows with max_iters, not with the iterations run; one host synchronisation, after the
 * download.
 * Work is enqueued on plf_stream and uses the scratch slot plf_local_ba and plf_pose_graph use (not
 * plf_global_ba_batch's), which stays allocated until plf_destroy: about 288 n_kf^2 bytes for the dense reduced system
 * (1.2 GB at 2048 keyframes, 4.8 GB at 4096) plus 144 bytes per observation and about 650 bytes per landmark.  Up to
 * n_kf = 64 the reduced system is factored by one CTA as in plf_local_ba; beyond, by a tiled LDL^T across the GPU that
 * skips exactly-zero tiles (n_t = ceil(6 n_kf / 64) tile columns).  Projects with the context's camera, as
 * plf_local_ba; plf_global_ba_batch takes a sequence's. */
plf_status plf_global_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* problem, plf_lba_result* out);

/* Many global bundle adjustments in one call: the maps of several sequences that end together, each with its sequence's
 * camera, solved in one launch chain with one host synchronisation (after the download).  The contract is
 * plf_local_ba_batch's, with plf_global_ba's rules per problem:
 *   problems [n_problems]  plf_global_ba's layout and rules, each in / out as in plf_global_ba
 *   seq      [n_problems]  or NULL: the camera of problem p, as in plf_local_ba_batch (-1: the context's camera;
 *                          0 <= seq[p] < n: plf_get_sequence_camera(ctx, seq[p]) at the time of the call; fx, fy, cx, cy)
 *   out      [n_problems]  or NULL;  status [n_problems], required.
 * Problem p gets what plf_global_ba gives it on a context created with p's camera: the same iteration count, the same
 * moved flags, lambda and err to rounding, every block to rounding of the step (both sum with float atomics).  One opts
 * applies to every problem; ref_quirks selects plf_global_ba's quirk set (g1-g6).
 * Refusals before any work, with nothing written (no problem's arrays, out or status) and a message naming the problem
 * and the rule: PLF_ERR_INVALID when n_problems < 0, a seq entry is out of range, or a problem breaks one of
 * plf_global_ba's host-side rules (empty problem, NULL arrays, ungrouped observations, out-of-range indices, a landmark
 * without observations); PLF_ERR_CAPACITY beyond 4096 keyframes in a problem or 65535 problems.  n_problems = 0 returns
 * PLF_OK.  Refusal on the device: as plf_local_ba_batch, a landmark whose first-pass block has an exactly zero diagonal
 * entry refuses its own problem only (status[p] = PLF_ERR_INVALID, its arrays and out[p] unchanged), the others are
 * solved and written back, and the call returns PLF_ERR_INVALID naming the first refused problem and its landmark.
 * Problems up to 64 keyframes are factored by one CTA each, as in plf_local_ba_batch; larger ones by the tiled LDL^T of
 * plf_global_ba, one launch per stage and tile column over all of them, at the largest problem's tile count n_t =
 * ceil(6 n_kf / 64).  All opts.max_iters rounds are enqueued at once: 2 launches per call, 8 per round (9 in round 0,
 * 10 under ref_quirks) and, when a problem has more than 64 keyframes, 5 n_t + 1 more per round, whatever the number of
 * problems and the iterations they run.
 * Work is enqueued on plf_stream and uses plf_local_ba_batch's scratch slot, which stays allocated until plf_destroy:
 * its parts as listed there (288 bytes per keyframe^2 of each problem is the dense reduced system, 1.2 GB at 2048
 * keyframes), plus 32768 n_t + n_t^2 bytes of tile work and 48 bytes of table per problem over 64 keyframes.  When the
 * summed systems do not fit on the device the call fails with PLF_ERR_CUDA, as plf_global_ba does when its scratch cannot
 * be allocated, and the context stays usable.  The rules for batches in flight are plf_global_ba's. */
plf_status plf_global_ba_batch(plf_ctx* ctx, const plf_lba_opts* opts, int n_problems, const plf_lba_problem* problems,
                               const int32_t* seq, plf_lba_result* out, plf_status* status);

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
 * error.  Work is enqueued on plf_stream and uses the scratch slot of plf_local_ba and plf_global_ba: 288 n_free^2
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

/* Many loop-closure pose graphs in one call: the sequences whose loop closures became ready together
 * (INTEGRATION.md §4a), optimised in lockstep rounds with one launch chain and one host synchronisation per round.
 *   problems [n_problems]  plf_pose_graph's layout and rules, T updated in place
 *   out      [n_problems]  plf_pose_graph's result of each problem, with its own trace / trace_cap (trace may be NULL)
 * One opts serves every problem.  Problem p's T, iters, stop, trials, chi2_init, chi2, lambda and trace rows are
 * bit-identical to what plf_pose_graph returns for it alone, whatever the other problems are and in whatever order they
 * come.  plf_pose_graph is this call with one problem.
 * Refusals before any work, with nothing written (no T, no out field): PLF_ERR_INVALID when n_problems < 0, opts is NULL,
 * problems or out is NULL with problems, or a problem breaks one of plf_pose_graph's rules (the message starts
 * "plf_pose_graph_batch: problem k: " and goes on as plf_pose_graph's); PLF_ERR_CAPACITY beyond 65535 problems or 4096
 * free vertices with edges in a problem.  n_problems = 0 returns PLF_OK and launches nothing.  When the problems' dense
 * systems do not fit on the device together the call fails with PLF_ERR_CUDA naming the scratch, and nothing is written.
 * The context stays usable after any error.
 * Rounds: round 0 evaluates every problem's initial chi2; each later round is one trial (one solve of (H + lambda I) x = b)
 * of every problem still running.  g2o's decisions (rho, acceptance, the lambda schedule, the 10-trial loop and the stop
 * tests) stay on the host, in double, per problem.  The call synchronises 2 + max_p trials_p times.
 * Launches: round 0: 2 (1 when no problem has an edge); a later round: 5 n_t + 4, plus 1 (the linearisation) when a
 * running problem starts an iteration in it, with n_t = ceil(6 n_free / 64) of the largest problem still running.  They
 * do not depend on n_problems: plf_pose_graph launches the same for its one problem.
 * Work is enqueued on plf_stream and uses plf_pose_graph's scratch slot: the sum of what each problem takes there (288
 * n_free^2 bytes of dense system, about 790 bytes per edge, 260 per vertex and 200 per free vertex, 32768 n_t + n_t^2
 * bytes of tile work) plus about 300 bytes per problem; out[p].scratch_bytes reports the call's total.  The context's
 * pinned staging buffer holds the inputs, the poses and the per-round control. */
plf_status plf_pose_graph_batch(plf_ctx* ctx, const plf_pgo_opts* opts, int n_problems, const plf_pgo_problem* problems,
                                plf_pgo_result* out);

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
/* pt_pairs / ls_pairs: (i1 in kf0, i2 in kf1) per surviving correspondence, capacity cap_* pairs (may be NULL).
 * At most 65535 features of a kind per keyframe (the matcher's 16-bit indices).  Uses the context's camera (plf_create);
 * plf_loop_closure_pose_batch takes a sequence's.  This call is plf_loop_closure_pose_batch with one problem. */
plf_status plf_loop_closure_pose(plf_ctx* ctx, const plf_lc_params* lc, const plf_lc_keyframe* kf0,
                                 const plf_lc_keyframe* kf1, plf_lc_result* out, int32_t* pt_pairs, int cap_pt,
                                 int32_t* ls_pairs, int cap_ls);

/* Many loop-closure checks in one call: the candidates of several sequences' new keyframes (the loop-closure thread,
 * src/mapHandler.cpp:1130-1214), each with its sequence's camera, in one upload, one launch chain and one download with
 * one host synchronisation.
 *   problems [n_problems]  kf0 = the candidate (map_keyframes[lc_kf_idx]), kf1 = the new keyframe, both read as
 *                          plf_loop_closure_pose reads them; pt_pairs / cap_pt, ls_pairs / cap_ls as there (may be NULL);
 *                          out: its result; status: PLF_OK, or PLF_ERR_CAPACITY when its pairs exceed its capacity
 *   seq      [n_problems]  or NULL: the camera of problem p, as in plf_gn_pose_batch (only fx, fy, cx, cy enter)
 * One lc and the context's parameters serve every problem.  Problem p's out, pairs and status are bit-identical to what
 * plf_loop_closure_pose returns for it on a context created with its camera.
 * Capacity: a problem whose surviving pairs exceed its capacity gets status PLF_ERR_CAPACITY and what the single call
 * writes then (the first cap_* pairs, n_pt / n_ls, accepted = 0, no pose_inc); every other problem is solved and written.
 * The call then returns PLF_ERR_CAPACITY, and plf_last_error names the first such problem.
 * Refusals before any work, naming the problem and the rule, with nothing written (no out, pairs or status):
 * PLF_ERR_INVALID when n_problems < 0, lc or problems is NULL, a seq entry is out of range, a keyframe is NULL or has a
 * negative count, a matched kind's arrays are NULL (the single call's "arrays missing" rules) or it has more than 65535
 * features in a keyframe; PLF_ERR_CAPACITY when n_problems > 65535 (the matcher's grid.y; no chunking).  n_problems = 0
 * returns PLF_OK and launches nothing.  The context stays usable after any error.
 * Launches: per kind that some problem matches (enabled, features of it in both keyframes), the forward 2-NN, the reverse
 * one (best_lr_matches) and the ratio / mutual check over all its problems: 3 (2 without best_lr_matches); then 3 more:
 * the inlier-ratio pre-condition with the compaction of the matches into solver rows, the pose solver and the acceptance
 * tests.  9 at the defaults; they do not depend on n_problems.  Work is enqueued on plf_stream; device scratch (its own slot, kept until plf_destroy): about
 * 125 bytes per kf0 point, 181 per kf0 line, 56 per kf1 point, 64 per kf1 line and 1.3 KB per problem, each part rounded
 * up to 256 bytes; the context's pinned staging buffer holds the inputs and outputs. */
typedef struct plf_lc_problem {
  const plf_lc_keyframe* kf0;    /* the candidate, map_keyframes[lc_kf_idx] (read as plf_loop_closure_pose reads it) */
  const plf_lc_keyframe* kf1;    /* the new keyframe */
  int32_t* pt_pairs; int cap_pt; /* out, may be NULL: as plf_loop_closure_pose */
  int32_t* ls_pairs; int cap_ls;
  plf_lc_result out;             /* out */
  int status;                    /* out: PLF_OK, or PLF_ERR_CAPACITY when this problem's pairs exceed its capacity */
} plf_lc_problem;
plf_status plf_loop_closure_pose_batch(plf_ctx* ctx, const plf_lc_params* lc, int n_problems, plf_lc_problem* problems,
                                       const int32_t* seq);

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

/* Forget the previous frame of every sequence (next batch starts with initialize(), app/plslam_dataset.cpp:115).  No batch
 * may be in flight (PLF_ERR_STATE). */
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
 * plf_get_matches refer to the batch most recently RUN, so call them with a single batch in flight.
 * plf_batch_download returns PLF_ERR_CAPACITY when an image of THAT batch overflowed a capacity (the batches in flight
 * before and after it are not affected, and the message names the kind and the limit).  out[] is written all the same:
 * the rows of pairs whose own images and whose sequence's previous frame stayed within the capacities are exact; the row
 * of the overflowing pair is computed from its truncated feature lists (counts never exceed the limits) and is not the
 * reference's result.  That pair's truncated frame is also what its sequence carries, so restart the sequence
 * (plf_batch_run_sequences, restart[k] = 1) with its next pair; INTEGRATION.md section 4a. */
plf_status plf_batch_upload(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride);
plf_status plf_batch_run(plf_ctx* ctx, int B);
plf_status plf_batch_download(plf_ctx* ctx, int B, plf_frame_result* out);

/* The colour form of plf_batch_upload: left/right hold B images each of h rows of `stride` bytes, image k at offset
 * k*stride*h (host), every row w pixels of `channels` interleaved bytes as in a cv::Mat: 3 = BGR (CV_8UC3), 4 = BGRA
 * (CV_8UC4).  stride >= channels * w; dense and strided rows are both accepted.  Its place in the upload -> run ->
 * download protocol is plf_batch_upload's (up to three batches in flight; grey and colour uploads may alternate freely).
 *   - The run that consumes the upload converts it to grey on the device, byte for byte cv::cvtColor(COLOR_BGR2GRAY) /
 *     (COLOR_BGRA2GRAY) of OpenCV 4 (alpha is ignored; DESIGN.md section 8), before extraction reads it.  Pairs of a
 *     rectified sequence (plf_set_sequence_rectification) are remapped first, every channel with its maps, and converted
 *     after, as stvo-pl's reader remaps the colour image it read and the detectors convert it; the two orders differ.
 *   - Once the run is issued, plf_batch_device_images holds the grey (and where rectified, remapped) images.  Run each
 *     upload once, as for grey uploads.  Everything after the conversion is the grey pipeline's.
 *   - The standalone operators (plf_orb, plf_lsd, plf_detect_lines, plf_lbd) take grey images only.
 * Device memory: the first colour upload allocates a landing buffer of 2 max_batch h w channels bytes (plus the batch's
 * pair table), grown once if 4 channels follow 3, kept until plf_destroy: about 2.9 GB at 1242 x 375, max_batch 1024 and
 * 3 channels (3.8 GB with 4).  A context that never uploads colour allocates nothing for it.
 * PLF_ERR_INVALID, naming the argument, for channels other than 3 or 4, B outside [1, max_batch], a NULL image or
 * stride < channels * w, with nothing changed; PLF_ERR_CUDA when the landing buffer cannot be allocated, with the
 * earlier uploads left as they were. */
plf_status plf_batch_upload_color(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride, int channels);

/* The image sizes the batched pipeline accepts besides the context's own (plf_create's camera), which it always accepts:
 * wh holds n (width, height) pairs, 0 <= n <= 8; n = 0 restores the single-size context.  A batch is of one size, the
 * size of the upload it runs; consecutive batches, and the batches in flight together, may be of different sizes.  A
 * sequence takes its size from its camera (plf_set_sequence_camera).  Each pair's results are bit for bit those of that
 * sequence alone on a context created at its size with its camera (DESIGN.md section 8).
 *   - Valid only before the first plf_batch_* call (PLF_ERR_STATE after), like plf_set_max_sequences.
 *   - Each size is checked as the pipeline checks the context's: every ORB level at least 2 orb_edge_th + 8 pixels wide
 *     and high, below 4096 pixels, and an LSD scaled size inside the kernels' limits.  PLF_ERR_INVALID, naming the size
 *     and what it fails, for a size that does not pass, for n out of range, or when a sequence has a camera of a size
 *     the new list lacks; nothing changes on a refusal.  A size equal to the context's or repeated is accepted once.
 *   - Device memory: every buffer of the pipeline is sized for the largest requirement over the sizes, so a context of
 *     sizes within a few per cent in area takes about what a context of the largest one takes. */
plf_status plf_set_image_sizes(plf_ctx* ctx, int n, const int32_t* wh);
/* plf_batch_upload (channels 1) or plf_batch_upload_color (3 = BGR, 4 = BGRA) of B pairs of w x h images, a size the
 * context accepts (plf_create's or one of plf_set_image_sizes').  The protocol, the landing buffer and the refusals are
 * theirs; an undeclared size is refused (PLF_ERR_INVALID, listing the accepted sizes) with nothing changed.  The run
 * that consumes the upload refuses a pair whose sequence is of another size.  plf_batch_upload and
 * plf_batch_upload_color upload the context's size. */
plf_status plf_batch_upload_sized(plf_ctx* ctx, int B, int w, int h, const uint8_t* left, const uint8_t* right, int stride,
                                  int channels);

/* Restricts ORB and line detection on the pairs of the most recent upload to masks that come with it, one per image, as
 * the detectors' mask arguments do (cv::ORB::detectAndCompute(img, mask), LSDDetectorC::detect(..., mask)): for masks that
 * change every frame, such as a segmentation network's dynamic objects.
 *   - Layout: mask_l / mask_r hold B masks each, h rows of `stride` bytes, mask k at offset k*stride*h, like
 *     plf_batch_upload's images.  One channel, any non-zero value allowed, of the most recent upload's size
 *     (plf_batch_device_layout) and in the geometry the detectors see: after rectification and after the grey conversion.
 *   - They belong to the most recent upload (grey, colour, sized, or images written through plf_batch_device_images), and
 *     the run that consumes it uses them.  The next upload, and any later run, starts without them.  Calling again before
 *     the run replaces them.
 *   - A NULL side has no pair masks; its images keep their sequence's mask (plf_set_sequence_mask), if any.
 *   - An image with a pair mask and a sequence mask is restricted to their pixelwise AND (non-zero where both are).  ORB's
 *     mask pyramid is built from that AND, as one mask given to detectAndCompute.
 *   - Memory: host memory, pageable or pinned, or device memory of the context's device (a torch CUDA tensor's
 *     data_ptr(), say).  Finish writing the masks before the call (for a PyTorch producer, synchronise its stream), and
 *     keep them unchanged until that batch's plf_batch_download returns.
 *   - The copy is asynchronous, on the upload stream, and waits for the earlier runs of the same image slot to have read
 *     that slot's masks.  The rest of each mask's pyramid is built on the device by the run.
 * Device memory: the first call allocates two blocks, one per upload slot, each of 2 max_batch ORB mask pyramids of the
 * largest image size (about 2.5 w h bytes each at 4 levels of scale 1.2), kept until plf_destroy: about 4.8 GB at
 * 1242 x 375, 4 levels and max_batch 1024.  A context that never calls it allocates, copies and launches nothing for it.
 * Refusals happen before anything is enqueued, name the argument and change nothing: PLF_ERR_STATE before the first upload;
 * PLF_ERR_INVALID for B outside [1, max_batch], both masks NULL, stride < w, or device memory of another device;
 * PLF_ERR_CUDA when the blocks cannot be allocated.  plf_batch_run_sequences refuses a B other than the masks' B
 * (PLF_ERR_INVALID, before anything is enqueued). */
plf_status plf_batch_upload_masks(plf_ctx* ctx, int B, const uint8_t* mask_l, const uint8_t* mask_r, int stride);

/* Number of sequences a context can track at once (default 1), 1 <= n <= 2^20.  Call it before the first plf_batch_* call:
 * PLF_ERR_STATE once the pipeline exists, PLF_ERR_INVALID for n out of range.  Each sequence keeps one carried frame slot
 * on the device (84 * max_keypoints + 156 * max_lines + 8 bytes). */
plf_status plf_set_max_sequences(plf_ctx* ctx, int n);
/* plf_batch_run for pairs of several sequences.  seq[k] in [0, n) is the sequence of pair k (NULL = all 0).
 * Pairs of one sequence appear in temporal order within the batch, and may be interleaved with other sequences in
 * any way.  Pair k is tracked against the previous pair of seq[k] in this batch.  If there is none, it is tracked
 * against that sequence's last pair in the most recent earlier run that contained it.
 * restart (NULL = none): restart[k] != 0 makes pair k a first frame (status 2), like plf_reset_sequence.  So does
 * the first pair a sequence ever has.  Restart flags are per pair, so they are valid with batches in flight; the
 * sequence state is resolved when a batch is run.
 * Invalid arguments return PLF_ERR_INVALID before anything is enqueued, and no sequence state changes.
 * plf_batch_run(ctx, B) is plf_batch_run_sequences(ctx, B, NULL, NULL); plf_reset_sequence forgets every sequence's
 * previous frame.  Results, plf_get_frame(k) and plf_get_matches(k) stay indexed by pair k of the batch. */
/* A batch is of one image size: a pair whose sequence's camera (plf_set_sequence_camera) is of another size than the upload
 * the run consumes is refused, naming the pair, the sequence and both sizes (PLF_ERR_INVALID, before anything is
 * enqueued). */
plf_status plf_batch_run_sequences(plf_ctx* ctx, int B, const int32_t* seq, const uint8_t* restart);
/* The calibration of sequence s, 0 <= s < n (plf_set_max_sequences).  The sequences of one context may differ in fx, fy,
 * cx, cy and b, and in the image size among the sizes the context accepts (plf_set_image_sizes); they share the
 * parameters and the limits.  cam == NULL returns s to the context's camera (plf_create).  Without declared sizes
 * cam->width and cam->height must equal the context's; with them, (cam->width, cam->height) must be one of the accepted
 * sizes (the refusal lists them).  fx, fy and b must be finite and > 0; cx and cy must be finite.  A change of s's size
 * while s has rectification maps or masks, which were built for its old size, is refused, naming them: clear them first.
 * Anything else returns PLF_ERR_INVALID, naming the field, and changes nothing.  The call may be made at any
 * time: before or after the pipeline exists, and with batches in flight.
 *   - The camera is resolved when a batch is run, like restart flags and sequence state.  Batches already run keep the
 *     calibration they were run with; the next plf_batch_run_sequences that holds s uses the new one, for every pair of
 *     s in that batch.
 *   - A successful call restarts s, even with NULL or unchanged values: the first pair of s in the next run that holds
 *     it is a first frame (status 2), since its carried frame was triangulated with another camera.
 *   - plf_set_max_sequences drops every sequence's camera; plf_reset_sequence keeps them.
 *   - plf_batch_run and plf_process_batch run sequence 0, so they use sequence 0's camera.
 * The keyframe and back-end operators use the context's camera in their single form and take a sequence's per problem in
 * their batch form: plf_match_kf2kf_batch, plf_match_map2kf_batch, plf_local_ba_batch, plf_global_ba_batch,
 * plf_gn_pose_batch and plf_loop_closure_pose_batch.  Place recognition's
 * batch form, plf_bow_insert_batch, takes a sequence's bag-of-words database instead: its vectors do not depend on the
 * camera, so plf_set_sequence_camera leaves that database as it is. */
plf_status plf_set_sequence_camera(plf_ctx* ctx, int s, const plf_camera* cam);
/* The calibration the next batch will use for sequence s: its own, or the context's camera. */
plf_status plf_get_sequence_camera(const plf_ctx* ctx, int s, plf_camera* out);

/* Front-end settings of sequence s of the batched front-end (p == NULL: back to the context's plf_params), so that
 * recordings of different pl-slam configs (config_kitti.yaml, config_euroc.yaml, ...) share one context.  The caller
 * fills a whole plf_params from the sequence's config, as for plf_create.  plf_sequence_param_fields classifies the fields:
 *   - PLF_PARAM_SEQUENCE fields may differ from the context's: orb_nfeatures, orb_fast_th, orb_nlevels, lsd_nfeatures,
 *     min_line_length, best_lr_matches, max_dist_epip, min_disp, min_ratio_12_p, min_ratio_12_l, line_sim_th,
 *     stereo_overlap_th, line_horiz_th, ls_min_disp_ratio, matching_strategy, matching_s_ws, matching_f2f_ws,
 *     min_pt_matches, min_ls_matches, homog_th, min_features, max_iters, max_iters_ref, min_error, min_error_change.
 *     Each int of them must be >= 0 and each float or double finite.  orb_nlevels must also be <= the context's (the
 *     sequence detects on its first orb_nlevels levels with its own nfeaturesPerLevel split, as cv::ORB with that many
 *     levels does).  matching_strategy != 0 is accepted only in a context created with matching_strategy != 0, whose
 *     windowed buffers exist; a strategy-0 sequence in such a context takes the brute-force match() result for every pair.
 *   - PLF_PARAM_CONTEXT fields must equal the context's: has_points, has_lines, orb_scale_factor, orb_edge_th, orb_wta_k,
 *     orb_score, orb_patch_size and every other lsd_* field.  They fix buffer geometry, tables, tensor maps or which launch
 *     chains exist.
 *   - PLF_PARAM_IGNORED fields (inlier_k, f2f_overlap_th) are accepted and have no effect, as for the context.
 * A refusal returns PLF_ERR_INVALID, naming the field, and changes nothing.  plf_create does not apply these range checks.
 * The call may be made at any time: before or after the pipeline exists, and with batches in flight.
 *   - The settings are resolved when a batch is run.  Batches already run keep the settings they were run with.
 *   - A successful call restarts s, even with NULL or unchanged values: its next pair is a first frame (status 2), since
 *     its carried frame was extracted and matched under the old settings.
 *   - plf_set_max_sequences drops every sequence's settings; plf_reset_sequence keeps them.
 *   - plf_batch_run and plf_process_batch run sequence 0 with sequence 0's settings.
 *   - With plf_set_adaptive_fast, a sequence's first frame is detected at its own orb_fast_th.
 * Only the batched front-end reads them.  The keyframe and back-end batch operators (plf_match_kf2kf_batch,
 * plf_match_map2kf_batch, plf_gn_pose_batch, plf_local_ba_batch, plf_global_ba_batch, plf_loop_closure_pose_batch, ...)
 * and every standalone operator keep using the context's plf_params. */
plf_status plf_set_sequence_params(plf_ctx* ctx, int s, const plf_params* p);
/* The settings the next batch will use for sequence s: its own, or the context's plf_params. */
plf_status plf_get_sequence_params(const plf_ctx* ctx, int s, plf_params* out);
enum { PLF_PARAM_SEQUENCE = 1, PLF_PARAM_CONTEXT = 2, PLF_PARAM_IGNORED = 3 };
/* The classification plf_set_sequence_params applies: for each field i of plf_params, i < min(cap, return value), its name
 * to names[i] and its class (PLF_PARAM_*) to classes[i], either array may be NULL.  Returns the number of fields. */
int plf_sequence_param_fields(const char** names, int* classes, int cap);

/* Rectification of sequence s's raw pairs before extraction: stvo-pl's dataset reader
 * cv::remap(img, out, map1, map2, INTER_LINEAR) with the default BORDER_CONSTANT 0, per image.  map1_*: w x h x 2 int16
 * (x, y) and map2_*: w x h uint16, as cv::initUndistortRectifyMap(..., CV_16SC2) or cv::convertMaps give them, for the
 * sequence's w x h (its camera's, plf_set_sequence_camera; host arrays, copied).  All four NULL clears it.  The camera of the rectified images (P1's fx, fy, cx, cy
 * and the baseline) is the caller's to set with plf_set_sequence_camera.
 *   - map2 is read as OpenCV reads it, map2 & 1023; map1 may point anywhere: taps outside the image read 0.  The result is
 *     byte for byte cv::remap's (DESIGN.md section 8).
 *   - The call may be made at any time, like plf_set_sequence_camera: the maps are resolved when a batch is run, so
 *     batches already run keep the maps they were run with.  With batches in flight the call waits until their
 *     rectifications (the first work of each run) have finished.
 *   - A successful call restarts s, even when it clears maps or sets the same ones: its next pair is a first frame
 *     (status 2).
 *   - plf_set_max_sequences drops every sequence's maps; plf_reset_sequence keeps them.
 *   - plf_batch_run_sequences rectifies the pairs of rectified sequences in the image slot it consumes, in place, before
 *     extraction reads it (plf_batch_device_images then holds the rectified images).  Run each upload once: a second run
 *     of the same slot would rectify it again.  A batch without a pair of a rectified sequence does no rectification work.
 *   - The standalone operators (plf_orb, plf_lsd, plf_detect_lines, plf_lbd) do not rectify, nor take colour.
 *   - A colour upload (plf_batch_upload_color) of a rectified sequence is remapped per channel, then converted to grey.
 * Device memory: 12 w h bytes per rectified sequence (4.3 MB at 752 x 480, 5.6 MB at 1242 x 375), allocated when its maps
 * are first set and freed when they are cleared, by plf_set_max_sequences or by plf_destroy.  The first run with a
 * rectified pair also allocates a scratch of 2 max_batch h pitch bytes (plus its pair table) kept until plf_destroy.
 * PLF_ERR_INVALID for s out of range or some but not all of the four pointers NULL, with nothing changed; PLF_ERR_CUDA
 * when the maps cannot be allocated or copied. */
plf_status plf_set_sequence_rectification(plf_ctx* ctx, int s, const int16_t* map1_l, const uint16_t* map2_l,
                                          const int16_t* map1_r, const uint16_t* map2_r);

/* Restricts the batched pipeline's ORB and line detection on sequence s's left / right images to masks, as
 * plf_orb_masked and plf_detect_lines_masked do (the masks the detectors' mask arguments take; stvo-pl passes none).
 * mask_l, mask_r: w x h uint8 (host arrays, copied), stride bytes per row, of the sequence's image size (its camera's,
 * plf_set_sequence_camera), in the geometry the detectors see: after rectification for a rectified sequence, one channel
 * for colour input.  The ORB pyramid of a mask is built in its size's level layout.  Both NULL clears them; one NULL masks only the
 * other image.
 *   - Each mask's ORB pyramid is built on the device once, by this call.  Extraction then reads it: features under the mask
 *     never reach the per-level retainBest, the line top-K, stereo association, tracking or the pose.
 *   - The call may be made at any time, like plf_set_sequence_camera: the masks are resolved when a batch is run, so
 *     batches already run keep the masks they were run with.  When s had a mask and batches are in flight, the call waits
 *     until their extraction and line stages have finished, then frees the old pyramids; the new ones are separate blocks.
 *   - It does not restart s: a mask changes what is detected, not the calibration.  The next pair is tracked against the
 *     previous frame as it was extracted.
 *   - plf_set_max_sequences drops every sequence's masks; plf_reset_sequence keeps them.
 *   - A batch without a masked image reads no mask and runs the unmasked kernels.
 * Device memory: one ORB pyramid's bytes per masked image (about 2.5 w h at 4 levels of scale 1.2: 1.2 MB at 1242 x 375),
 * allocated by the call and freed when cleared, by plf_set_max_sequences or by plf_destroy.
 * PLF_ERR_INVALID for s out of range or, with a mask given, stride < w, with nothing changed; PLF_ERR_CUDA when a pyramid
 * cannot be allocated or built, with nothing changed.  Errors of the ORB configuration are plf_orb's. */
plf_status plf_set_sequence_mask(plf_ctx* ctx, int s, const uint8_t* mask_l, const uint8_t* mask_r, int stride);

/* Whether sequence s has a left / right mask (plf_set_sequence_mask): *left, *right = 1 or 0.  PLF_ERR_INVALID for s out of
 * range or a NULL pointer. */
plf_status plf_get_sequence_mask_set(plf_ctx* ctx, int s, int* left, int* right);

/* stvo-pl's adaptative_fast (config_euroc.yaml:17, :36-41): each sequence's FAST threshold follows its last tracked frame.
 * The fields are the config keys fast_min_th, fast_max_th, fast_inc_th, fast_feat_th and fast_err_th. */
typedef struct plf_adaptive_fast {
  int min_th, max_th, inc_th, feat_th;
  double err_th;
} plf_adaptive_fast;
/* Turns the adaptation on (cfg != NULL) or off (NULL, the default) for the batched pipeline; plf_orb and the other
 * standalone detectors keep plf_params.orb_fast_th.  With it on, pair k of a batch is detected (both images) at its
 * sequence's threshold, and after the pose that threshold moves by the rule of DESIGN.md section 8:
 *   first frame (status 2)                      unchanged
 *   DT == identity exactly, or err > err_th     th = max(min_th, th - 2 inc_th)   (status 1 has DT = identity)
 *   else n_inliers_pt <  feat_th                th = max(min_th, th - 2 inc_th)
 *   else n_inliers_pt <  2 feat_th              th = max(min_th, th - inc_th)
 *   else n_inliers_pt >  3 feat_th              th = min(max_th, th + inc_th)
 * Every first frame of a sequence (its first pair, restart[k], plf_reset_sequence, plf_set_sequence_camera) is detected
 * at orb_fast_th (clamped to [0, 255]).  Frame k of a sequence needs the threshold frame k-1's pose gives, so with the
 * adaptation on a batch may hold at most one pair of each sequence: plf_batch_run_sequences refuses a batch with two pairs
 * of one sequence (PLF_ERR_INVALID, before anything is enqueued, no sequence state changed).  A single sequence therefore
 * runs B = 1; many sequences run round-robin, one pair of each per batch (INTEGRATION.md section 4a).
 * Valid only with no batch in flight (PLF_ERR_STATE).  PLF_ERR_INVALID, naming the field, unless
 * 0 <= min_th <= max_th <= 255, inc_th >= 0, feat_th >= 0 and err_th is finite; nothing changes on a refusal.  A successful
 * call sets every sequence's threshold back to orb_fast_th. */
plf_status plf_set_adaptive_fast(plf_ctx* ctx, const plf_adaptive_fast* cfg);
/* *th = the FAST threshold the next pair of sequence s will be detected with (orb_fast_th with the adaptation off or when
 * that pair is a first frame).  May be called at any time; with batches in flight it waits for their match phases. */
plf_status plf_get_sequence_fast_th(plf_ctx* ctx, int s, int* th);

/* stvo-pl's use_motion_model (config_euroc.yaml:18): each sequence's next pair starts from a constant-motion prediction.
 * Turns it on (on != 0) or off (0, the default) for the batched pipeline.  With it on, after pair k of sequence s the
 * prediction of s's next pair is T = inverse_se3(DT_k) (the optimiser's transform, previous frame into current) when pair
 * k is a good solution (stvo-pl's isGoodSolution, DESIGN.md section 8):
 *   status 0, every entry of DT finite, and none of err < 0, err > 1, min eig(DT_cov) < 0, max eig(DT_cov) > 1
 * (so a NaN err or eigenvalue passes; a DT_cov with a non-finite entry has NaN eigenvalues), else the identity.  The next
 * pair projects the previous frame's points and line end points through T before the windowed frame-to-frame matching
 * (matching_strategy != 0) and seeds the pose solver with it (T_init).  Every first frame (its first pair, restart[k],
 * plf_reset_sequence, plf_set_sequence_camera, plf_set_sequence_rectification) starts from the identity, and a successful
 * call with on != 0 sets every sequence's prediction back to it.  As with plf_set_adaptive_fast a batch may hold at most
 * one pair of each sequence (plf_batch_run_sequences refuses it otherwise, PLF_ERR_INVALID, before anything is enqueued).
 * Valid only with no batch in flight (PLF_ERR_STATE). */
plf_status plf_set_motion_model(plf_ctx* ctx, int on);
/* T (row-major 4x4) = the prediction the next pair of sequence s will start from, *valid = 1 when it came from a good
 * solution (identity and 0 with the model off or when that pair is a first frame).  May be called at any time; with
 * batches in flight it waits for their match phases. */
plf_status plf_get_sequence_motion(plf_ctx* ctx, int s, double T[16], int* valid);
/* The device rule of plf_set_motion_model on n caller results, for tests that put a decision exactly on an edge: DT [n][16],
 * DT_cov [n][36], err [n], status [n] in; T_out [n][16] (the prediction) and valid_out [n] out.  One launch on the
 * context's stream.  PLF_ERR_INVALID for n < 0 or an array NULL (n > 0). */
plf_status plf_debug_motion_prior(plf_ctx* ctx, int n, const double* DT, const double* DT_cov, const double* err,
                                  const int32_t* status, double* T_out, int32_t* valid_out);
/* Poses of the OLDEST batch in flight, device to device: dst_device[B][16] f64 (DT, row-major) is filled on `stream`
 * (a cudaStream_t of the caller; NULL = an internal stream, synchronised before returning) behind that batch's match
 * phase - the buffer a multi-GPU caller passes to its NCCL pose all-gather on the same stream (SURVEY 8e; the reference
 * has no counterpart: app/plslam_dataset.cpp:148-154 reads curr_frame->Tfw on the host).  The batch stays in flight
 * until plf_batch_download. */
plf_status plf_batch_device_poses(plf_ctx* ctx, int B, double* dst_device, void* stream);
/* Device buffer [2*max_batch][h][pitch] read by plf_batch_run (image 2k = left k, 2k+1 = right k), pitch = width rounded up
 * to a multiple of 16 bytes (every halo tile of every image is then a legal TMA box); h, w and pitch are those of the
 * most recent upload's image size (plf_batch_device_layout).  It is the slot of the most recent
 * upload; once that upload has been run, the pairs of rectified sequences (plf_set_sequence_rectification) in it are the
 * rectified images, and a colour upload (plf_batch_upload_color) is its grey conversion. */
void* plf_batch_device_images(plf_ctx* ctx);
/* The layout of plf_batch_device_images' slot: the width, height and row pitch of the most recent upload's images (the
 * context's size before any upload; plf_batch_upload_sized uploads the others).  Image z starts pitch * h bytes after
 * image z - 1.  PLF_ERR_INVALID for a NULL pointer. */
plf_status plf_batch_device_layout(plf_ctx* ctx, int* w, int* h, int* pitch);

/* What the front-end derives from an image size, as the library computes it (host only: needs no device or context):
 * the 16-byte row pitch of the device images, the ORB pyramid's level sizes, the LSD scaled size and the windowed
 * matcher's grid scales (64 / w, 48 / h).  params NULL = plf_default_params.  PLF_ERR_INVALID, with the reason in
 * plf_last_error(NULL), for a size the pipeline would refuse (plf_set_image_sizes). */
typedef struct plf_image_geometry {
  int pitch;
  int orb_nlevels;
  int orb_w[8], orb_h[8];
  int lsd_w, lsd_h;
  double grid_iw, grid_ih;
} plf_image_geometry;
plf_status plf_get_image_geometry(const plf_params* params, int w, int h, plf_image_geometry* out);

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
 * inherits them): the single calls use the context's camera of plf_create, the batch calls (plf_match_kf2kf_batch,
 * plf_match_map2kf_batch) a sequence's per problem (plf_set_sequence_camera).  Work is enqueued on plf_stream, so a call
 * between batches in flight is safe.  A kind returns 0 (every entry -1) when it is disabled or the keyframe has no stereo
 * features of it.  Semantics reproduced as written, quirks included (DESIGN.md 8): see oracle/kfmatching.py. */
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

/* Many keyframe matchings in one call: the new keyframes of several sequences, each against its previous keyframe
 * (plf_match_kf2kf_batch) or its local map (plf_match_map2kf_batch), each with its sequence's camera, in one upload, one
 * launch chain and one download with one host synchronisation.
 *   problems [n_problems]  the single call's inputs and outputs per problem (n_pt / n_ls: its return values)
 *   seq      [n_problems]  or NULL: the camera of problem p, as in plf_local_ba_batch.  seq[p] = -1 (or seq NULL) uses
 *                          the context's camera; 0 <= seq[p] < n (plf_set_max_sequences) uses what
 *                          plf_get_sequence_camera(ctx, seq[p]) returns at the time of the call.  Only fx, fy, cx and cy
 *                          enter; the image size and the grid scales stay the context's.
 * Problem p's outputs are bit-identical to what the single call returns for its inputs on a context created with its
 * camera and the same parameters.  One opts and the context's parameters apply to every problem.
 * Refusals before any work: PLF_ERR_INVALID when n_problems < 0, a seq entry is out of range, or a problem breaks a
 * host-side rule of the single call (NULL arrays with a count > 0, a NaN in DT / Twf, more than 8192 features or 65535
 * landmarks per kind); PLF_ERR_CAPACITY when n_problems > 65535 (the grids' y dimension; no chunking).  The message names
 * the problem index and the rule, and nothing is written: unlike the single call, no output is pre-filled.
 * n_problems = 0 returns PLF_OK.  The context stays usable after any error.
 * Launches: 5 per kind active in some problem, plus the windowed matcher's 3 (points) / 4 (lines) per chunk of problems
 * when fast_matching, plus 2 or 3 (best_lr_matches) per kind when some problem can take the match() fallback; they do
 * not depend on n_problems while the matcher's problems fit one chunk.  Device scratch: the single call's per problem, except
 * that the windowed matcher's arrays are sized at the batch's largest counts K (queries) and Kt (train) per kind, so one
 * large map pads every problem of the batch to its size.  Its distance matrix takes 2 K Kt bytes per problem and kind,
 * in chunks of at most 2 GB (a batch beyond one chunk costs the matcher's launches once per chunk). */
typedef struct plf_kf2kf_problem {
  const plf_frame_view* prev;   /* read as plf_match_kf2kf reads it */
  const plf_frame_view* curr;
  double DT[16];                /* row-major MapHandler::DT */
  int32_t* m_pt;                /* out [prev->n_pt] */
  int32_t* m_ls;                /* out [prev->n_ls] */
  int n_pt, n_ls;               /* out: the reference's return values */
} plf_kf2kf_problem;
plf_status plf_match_kf2kf_batch(plf_ctx* ctx, const plf_kf_match_opts* opts, int n_problems, plf_kf2kf_problem* problems,
                                 const int32_t* seq);

typedef struct plf_map2kf_problem {
  const plf_local_map* map;
  const plf_frame_view* kf;     /* read as plf_match_map2kf reads it */
  double Twf[16];               /* row-major MapHandler::Twf */
  const int32_t* kf_pt_lm;      /* [kf->n_pt] or NULL = all unmatched */
  const int32_t* kf_ls_lm;      /* [kf->n_ls] or NULL */
  int32_t* lm_pt;               /* out [map->n_pt] */
  int32_t* lm_ls;               /* out [map->n_ls] */
  int n_pt, n_ls;               /* out: the reference's return values */
} plf_map2kf_problem;
plf_status plf_match_map2kf_batch(plf_ctx* ctx, const plf_kf_match_opts* opts, int n_problems, plf_map2kf_problem* problems,
                                  const int32_t* seq);

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
 * empties that kind's database: the context's and every sequence's (plf_bow_insert_batch).  The tree is stored re-laid out by parent (each node's children contiguous, in file order):
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

/* Many keyframe inserts in one call: the new keyframes of several sequences, each transformed, stored and scored in its
 * sequence's own database (the reference scores a keyframe against its own map's keyframes only, src/mapHandler.cpp:
 * 3019-3028), in one upload, three launches and one download with one host synchronisation.
 *   problems [n_problems]  kf_idx, kf (read: n_pt, n_ls, pdesc, ldesc), score_p / score_l: as plf_bow_insert's arguments
 *   seq      [n_problems]  or NULL: the DATABASE of problem p.  seq[p] = -1 (or seq NULL) is the context's database, the
 *                          one plf_bow_insert / plf_bow_erase / plf_bow_get use; 0 <= seq[p] < n (plf_set_max_sequences)
 *                          is sequence seq[p]'s.
 * Every database holds, per kind, the stored vectors under their indices and its own `last` index; all of them share the
 * context's two vocabularies.  Each database numbers its keyframes from 0 by itself.
 *   - Equality: problem p's rows, its stored vector (plf_bow_get_seq) and every later row scored against it are
 *     bit-identical to plf_bow_insert on a context whose only database is p's, with the same vocabularies, the same
 *     earlier inserts and erasures of that database, and this batch's problems of that database made one by one in
 *     problem order.
 *   - Several problems may target one database: their kf_idx must rise in problem order, and a later one's row includes
 *     the earlier ones.
 *   - Isolation: a row covers its own database only; an index stored by another sequence is NaN there, as any absent one.
 *   - Kinds: has_points / has_lines apply as in plf_bow_insert: a disabled kind's row is left as it is and needs no
 *     vocabulary.
 *   - Lifecycle: plf_bow_set_vocabulary(kind) empties that kind in every database; plf_bow_clear_sequence(s) empties both
 *     kinds of s and frees their device memory; plf_set_max_sequences drops every sequence's databases;
 *     plf_reset_sequence and plf_set_sequence_camera leave them as they are.
 *   - A sequence never inserted into holds no device memory (one host pointer).  A sequence database's first allocation
 *     is 1024 entries and 64 indices per kind (the context's: 65536 and 1024); each grows by doubling, as plf_bow_insert's.
 * Refusals before any work, naming the problem and the rule, with nothing changed: PLF_ERR_INVALID when n_problems < 0,
 * a seq entry is outside [-1, n), kf is NULL, kf_idx is outside [0, 2^24) or, for an enabled kind, does not exceed its
 * database's last index or an earlier problem's kf_idx on the same database, a count is outside [0, 8192], or
 * descriptors are NULL with a count > 0; PLF_ERR_STATE when an enabled kind has no vocabulary; PLF_ERR_CAPACITY when a
 * database would pass 2^31 - 1 entries or n_problems > 65535 (the assembly's grid.y; no chunking).  n_problems = 0
 * returns PLF_OK.  The context stays usable after any error.
 * Launches: the transform (when any feature is enabled), the assembly and the scoring (when any row is requested); they
 * do not depend on n_problems.  Each problem reserves as many entries as it has features in its database; when two
 * problems share a database, the unused part of the earlier one's reservation stays a hole (not returned by
 * plf_bow_get_seq).  Work is enqueued on plf_stream; device scratch (PLF_SCR_BOW) and the pinned staging buffer hold 32
 * bytes per feature and 124 per problem in, the rows and 8 bytes per problem out, 12 bytes per feature of work. */
typedef struct plf_bow_problem {
  int kf_idx;                  /* index in its database, as plf_bow_insert's kf_idx */
  const plf_frame_view* kf;    /* read: n_pt, n_ls, pdesc, ldesc (as plf_bow_insert reads it) */
  double* score_p;             /* out [kf_idx + 1] or NULL, as plf_bow_insert */
  double* score_l;
} plf_bow_problem;
plf_status plf_bow_insert_batch(plf_ctx* ctx, int n_problems, plf_bow_problem* problems, const int32_t* seq);
/* plf_bow_erase on sequence s's database (s = -1: the context's; exactly plf_bow_erase).  s outside [-1, n) returns
 * PLF_ERR_INVALID; erasing from a sequence never inserted into is a no-op. */
plf_status plf_bow_erase_seq(plf_ctx* ctx, int s, int kf_idx);
/* plf_bow_get on sequence s's database (s = -1: the context's; exactly plf_bow_get).  s outside [-1, n) returns
 * PLF_ERR_INVALID. */
plf_status plf_bow_get_seq(plf_ctx* ctx, int s, int kf_idx, int kind, int cap, uint32_t* words, double* values, int* n);
/* Empties both kinds of sequence s's database and frees its device memory, for a new recording that takes over slot s
 * (INTEGRATION.md section 4a).  0 <= s < n, else PLF_ERR_INVALID; the next insert into s may start again at kf_idx 0. */
plf_status plf_bow_clear_sequence(plf_ctx* ctx, int s);

/* Loop-closure candidate detection (SURVEY 8(f) f5): the score combination of MapHandler::insertKFBowVectorP / L / PL
 * (src/mapHandler.cpp:3007-3128) and lookForLoopCandidates (:3130-3190), fused behind the insert and scoring of
 * plf_bow_insert_batch.  The options are the SlamConfig values lookForLoopCandidates reads. */
typedef struct plf_lc_detect_opts {
  int lc_kf_dist;        /* SlamConfig::lcKFDist     src/slamConfig.cpp:80 (50) */
  int lc_kf_max_dist;    /* lcKFMaxDist              :81 (50) */
  int lc_nkf_closest;    /* lcNKFClosest             :82 (4)  */
  int min_lm_cov_graph;  /* minLMCovGraph            :61 (75) */
  int min_kf_local_map;  /* minKFLocalMap            :62 (3)  */
} plf_lc_detect_opts;

typedef struct plf_lc_detect_result {
  int candidate;     /* kf_prev_idx, or -1 when lookForLoopCandidates returns false */
  int best;          /* idx_max (first of the sorted list), -1 when the list is not sorted */
  int n_listed;      /* max_confmat.size() */
  int n_closest;     /* Nkf_closest (0 when not evaluated) */
  double min_score;  /* lc_min_score; NaN when the list is not sorted (the reference never computes it then) */
} plf_lc_detect_result;

typedef struct plf_lc_detect_problem {
  int kf_idx;                   /* as plf_bow_problem */
  const plf_frame_view* kf;     /* read: n_pt, n_ls, pdesc, ldesc, pt_pl, ls_spl, ls_epl */
  const uint32_t* covis;        /* [kf_idx]: full_graph[kf_idx][i] (symmetric), or NULL = all zero */
  float* conf;                  /* out [kf_idx+1] or NULL: conf_matrix[kf_idx][i]; NaN where absent */
  double* score_p, *score_l;    /* out or NULL, exactly as plf_bow_problem */
  plf_lc_detect_result result;  /* out */
} plf_lc_detect_problem;

/* plf_bow_insert_batch, then per problem the conf_matrix column of its keyframe and lookForLoopCandidates on it, in one
 * upload, five launches whatever the batch size, one download and one host synchronisation.
 *   - Insert and score: exactly plf_bow_insert_batch (its refusals, its database state afterwards, bit-identical rows
 *     and stored vectors).  The rows stay on the device; only those requested (score_p / score_l not NULL) come back.
 *   - conf[i] for every live i <= kf_idx, as insertKFBowVector* writes conf_matrix[kf_idx][i], by has_points /
 *     has_lines: P only (float)score_p; L only (float)score_l; both: score = 0.0; score += (sp n_pt + sl n_ls) / n_pl;
 *     score += (sp std_pt + sl std_ls) / std_pl, in double in that order, rounded to float.  std_pt = stdv(pt_pl x) +
 *     stdv(pt_pl y) over the n_pt points, std_ls the same over the line midpoints (spl + epl) * 0.5; stdv is stvo-pl's
 *     vector_stdv (sequential mean, sqrt(sum (x - mean)^2 / (n - 1)), 0 for no element; DESIGN.md 8).  One point or line
 *     alone, no feature at all or std_pl = 0 make the whole column NaN, and a NaN column yields no candidate.
 *   - Detection: live i < kf_idx - lc_kf_dist are listed; with more than lc_kf_max_dist of them (a size_t comparison:
 *     a negative lc_kf_max_dist never passes) lc_min_score is the minimum over i < kf_idx with covis[i] >=
 *     (unsigned)min_lm_cov_graph or kf_idx - i <= min_kf_local_map + 3 of the scores in (0.001, 1.0) (absent i count as
 *     0); best is the listed maximum, and Nkf_closest counts the other listed i with |i - best| <= lc_kf_max_dist and
 *     score >= lc_min_score * 0.8.  Scores go through float and then double, as the reference reads conf_matrix.
 *   - One deviation: among equal maxima, best is the lowest index.  The reference's std::sort (sort_confmat_by_score)
 *     orders equal scores stably only below 17 listed keyframes under libstdc++; above that their order is
 *     implementation-defined.  NaN scores rank below every number (a column is NaN whole, so this only decides
 *     plf_debug_loop_candidates' inputs).
 * Refusals: those of plf_bow_insert_batch, and opts NULL (PLF_ERR_INVALID), before any work, naming the problem and the
 * rule.  A problem with covis NULL has no covisibility; its pt_pl / ls_spl / ls_epl are read only when both kinds are
 * enabled, and must then be non-NULL where their count is > 0.  A keyframe is live when every enabled kind stores it.  Device scratch (PLF_SCR_BOW) adds 24 bytes per point and 40 per
 * line, 4 per keyframe index (covis) in, and 13 + 8 per enabled kind per keyframe index of the rows and columns. */
plf_status plf_bow_detect(plf_ctx* ctx, const plf_lc_detect_opts* opts, plf_lc_detect_problem* problem);  /* context's database */
plf_status plf_bow_detect_batch(plf_ctx* ctx, const plf_lc_detect_opts* opts, int n_problems,
                                plf_lc_detect_problem* problems, const int32_t* seq);  /* seq as plf_bow_insert_batch */
/* The detection kernel of plf_bow_detect_batch on caller-supplied columns, for tests that put a decision exactly on a
 * threshold: problem p is kf_idx[p] with conf[p] [kf_idx[p] + 1] (conf_matrix[i][kf_idx]), live[p] [kf_idx[p] + 1]
 * (map_keyframes[i] != NULL) and covis[p] [kf_idx[p]] or NULL.  One upload, one launch, one download.  PLF_ERR_INVALID
 * for opts or out NULL, n < 0, a kf_idx outside [0, 2^24) or a conf / live NULL; PLF_ERR_CAPACITY for n > 65535. */
plf_status plf_debug_loop_candidates(plf_ctx* ctx, const plf_lc_detect_opts* opts, int n, const int* kf_idx,
                                     const float* const* conf, const uint8_t* const* live,
                                     const uint32_t* const* covis, plf_lc_detect_result* out);

/* Debug: device-clock timeline (ms) of the two most recent batches of the software pipeline: for each, the start/end of
 * the E (extract), G (region growing) and M (match/track/pose) phases relative to the older batch's E start.
 * No reference counterpart (the reference times whole calls with its Timer, app/plslam_dataset.cpp:126-132). */
plf_status plf_debug_timeline(plf_ctx* ctx, float out[12]);

#ifdef __cplusplus
}
#endif
#endif /* PLSLAM_B200_H */
