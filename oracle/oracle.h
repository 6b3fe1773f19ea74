/* oracle/oracle.h — declarations of the CPU oracle (TEST INFRASTRUCTURE ONLY; see oracle/__init__.py). */
#ifndef PLF_ORACLE_H
#define PLF_ORACLE_H
#include <stdint.h>

/* Mirrors cv::line_descriptor::KeyLine (3rdparty/line_descriptor/include/line_descriptor/descriptor_custom.hpp:105-176)
 * and, field for field, plf_keyline in include/plslam_b200.h. */
typedef struct orc_keyline {
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
} orc_keyline;

void orc_gaussian_kernel_q8(int ksize, double sigma, int* taps);
void orc_blur_taps_u8(const uint8_t* src, int w, int h, int ksize, const int* taps, uint8_t* dst);
void orc_gaussian_blur_u8(const uint8_t* src, int w, int h, int ksize, double sigma, uint8_t* dst);
void orc_sobel3_i16(const uint8_t* src, int w, int h, int16_t* dx, int16_t* dy);
void orc_lbd_weights(double* gaussCoefL, double* gaussCoefG);
void orc_lbd_compute(const uint8_t* img, int w, int h, const orc_keyline* kls, int n, uint8_t* desc_bin,
                     float* desc_float);
int orc_keylines_from_segments(const float* segs, int m, int w, int h, double min_length, orc_keyline* out);

/* ---- ORB (oracle/orb.c) ---- */
typedef struct orc_keypoint {
  float x, y;      /* cv::KeyPoint.pt (level-0 coordinates) */
  float size, angle, response;
  int octave;
  int lx, ly;      /* integer coordinates inside its pyramid level (not a cv::KeyPoint field) */
} orc_keypoint;
void orc_resize_linear_exact(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh, double inv_scale_x,
                             double inv_scale_y);
void orc_fast_score_map(const uint8_t* img, int w, int h, int threshold, uint8_t* score);
float orc_fast_atan2(float y, float x);
void orc_gaussian_kernel_f32(int ksize, double sigma, float* k);
void orc_orb_blur7(const uint8_t* src, int w, int h, uint8_t* dst);
int orc_orb_detect_and_compute(const uint8_t* image, int w, int h, int nfeatures, float scaleFactor, int nlevels,
                               int edgeThreshold, int patchSize, int fastThreshold, orc_keypoint* kps,
                               uint8_t* desc, int cap);

/* ---- LSD (oracle/lsd.c) ---- */
uint8_t* orc_lsd_scaled_image(const uint8_t* img, int w, int h, double scale, double sigma_scale, int* ow, int* oh);
int orc_lsd_detect(const uint8_t* img, int w, int h, double scale, double sigma_scale, double quant, double ang_th,
                   int n_bins, int order_mode, int trig_mode, float* segs, int cap);

/* ---- Gauss-Newton pose refinement (oracle/gn.c) ---- */
typedef struct orc_camera { int width, height; double fx, fy, cx, cy, b; } orc_camera;
typedef struct orc_gn_opts {
  double homog_th;       /* Config::homogTh, config_euroc.yaml:45 */
  int max_iters;         /* stage 1, config_euroc.yaml:47 */
  int max_iters_ref;     /* stage 2, config_euroc.yaml:48 */
  double eps_err;        /* stop if e < eps_err           (twin: DBL_EPSILON; stvo-pl: min_error) */
  double eps_change;     /* stop if |e - e_prev| < eps_change (twin: DBL_EPSILON; stvo-pl: min_error_change) */
  double eps_step;       /* stop if |dx| < eps_step        (twin: DBL_EPSILON) */
} orc_gn_opts;
typedef struct orc_pose_result {
  double T[16];   /* row-major 4x4 increment T_inc */
  double cov[36]; /* H^-1 of the last accumulation */
  double x[6];    /* logmap_se3(T) = [t; w] */
  double err;
  int iters1, iters2, n_inliers_pt, n_inliers_ls;
} orc_pose_result;
void orc_expmap_se3(const double* x, double* T);
void orc_logmap_se3(const double* T, double* x);
void orc_inverse_se3(const double* T, double* Ti);
void orc_colpiv_qr_solve6(const double* H, const double* g, double* x);
int orc_inverse6(const double* A, double* Ainv);
void orc_gn_pose(const orc_camera* cam, const orc_gn_opts* o, const double* P, const double* obs, uint8_t* inl_p,
                 int np, const double* sP, const double* eP, const double* le, uint8_t* inl_l, int nl,
                 const double* T_init, orc_pose_result* out);
/* Stop-decision trace of orc_gn_pose_trace: one record per accumulation of either stage, in order. */
enum { ORC_GN_CONTINUE = 0, ORC_GN_EXIT_ERROR = 1, ORC_GN_EXIT_STEP = 2, ORC_GN_EXIT_MAXIT = 3 };
typedef struct orc_gn_trace_rec {
  int stage;     /* 0 (robust) or 1 (refinement after the gate) */
  int exit;      /* ORC_GN_CONTINUE, or why the stage ended on this iteration */
  double e;      /* normalised error of this iteration's accumulation */
  double e_prev; /* the error the change test compared it with */
  double step;   /* ||dx|| of the step taken; -1 when the error test stopped the stage first */
} orc_gn_trace_rec;
typedef struct orc_gn_trace {
  orc_gn_trace_rec* rec;
  int cap, n;        /* records available / accumulations made (those past cap are counted, not stored) */
  int stage_exit[2]; /* why each stage ended (ORC_GN_EXIT_MAXIT also for a stage of 0 iterations) */
} orc_gn_trace;
void orc_gn_pose_trace(const orc_camera* cam, const orc_gn_opts* o, const double* P, const double* obs, uint8_t* inl_p,
                       int np, const double* sP, const double* eP, const double* le, uint8_t* inl_l, int nl,
                       const double* T_init, orc_pose_result* out, orc_gn_trace* tr);

/* ---- local bundle adjustment (oracle/lba.c; src/mapHandler.cpp:1332-1989) ---- */
typedef struct orc_lba_opts {
  double lambda;           /* SlamConfig::lambdaLbaLM  (src/slamConfig.cpp:64: 0.00001) */
  double lambda_k;         /* SlamConfig::lambdaLbaK   (:65: 10) */
  int max_iters;           /* SlamConfig::maxItersLba  (:66: 15) */
  double homog_th;         /* SlamConfig::homogTh */
  double min_error;        /* Config::minError */
  double min_error_change; /* Config::minErrorChange */
  int ref_quirks;          /* 1: reproduce the reference as written (see lba.c), 0: the evident intent */
} orc_lba_opts;
typedef struct orc_lba_result {
  int iters;
  double err;
  double lambda;
  int zero_lm; /* rc ORC_LBA_ZERO_BLOCK: the landmark (points first, then lines) whose block has a zero diagonal entry */
} orc_lba_result;
/* return codes: 0, -1 (empty problem, as the reference), ORC_LBA_ZERO_BLOCK (a landmark's first-pass block D has an
 * exactly zero diagonal entry, e.g. a landmark without observations or whose every row has a zero Jacobian: refused
 * before any step, X unchanged) */
enum { ORC_LBA_ZERO_BLOCK = -2 };
/* Iteration trace of orc_local_ba_trace: record 0 is the first pass, record i the i-th LM iteration. */
enum { ORC_LBA_CONTINUE = 0, ORC_LBA_STOP_CHANGE = 1, ORC_LBA_STOP_MIN_ERROR = 2, ORC_LBA_STOP_STEP = 3, ORC_LBA_STOP_MAXIT = 4 };
typedef struct orc_lba_trace_rec {
  double err;    /* normalised error of the pass */
  double lambda; /* the damping of its solve (the current lambda when the error tests stopped the run first) */
  double step;   /* |DX| of its solve; -1 when the error tests stopped the run first */
  int applied;   /* 1 when its step was applied; 0 when the error grew (solved, not applied) or no step was solved */
  int stop;      /* ORC_LBA_CONTINUE, or why the run ended after this pass (CHANGE / MIN_ERROR: the error tests, no solve) */
} orc_lba_trace_rec;
typedef struct orc_lba_trace {
  orc_lba_trace_rec* rec;
  int cap, n; /* records available / passes made (those past cap are counted, not stored) */
} orc_lba_trace;
int orc_local_ba(const orc_camera* cam, const orc_lba_opts* o, int nkf, int npt, int nls, double* X, int n_fixed,
                 const double* fixed_T, int npo, const int* po_lm, const int* po_kf, const double* po_xy, int nlo,
                 const int* lo_lm, const int* lo_kf, const double* lo_le, uint8_t* pt_moved, uint8_t* ls_moved,
                 orc_lba_result* out);
int orc_local_ba_trace(const orc_camera* cam, const orc_lba_opts* o, int nkf, int npt, int nls, double* X, int n_fixed,
                       const double* fixed_T, int npo, const int* po_lm, const int* po_kf, const double* po_xy, int nlo,
                       const int* lo_lm, const int* lo_kf, const double* lo_le, uint8_t* pt_moved, uint8_t* ls_moved,
                       orc_lba_result* out, orc_lba_trace* tr);
#endif
