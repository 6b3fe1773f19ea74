// stvo_shim.h — C++ host side of the drop-in boundary: the StVO:: class API that pl-slam consumes
// (SURVEY.md §8b, Appendix A.1), implemented on top of the C ABI in include/plslam_b200.h.
//
// pl-slam includes stvo-pl's stereoFrame.h / stereoFrameHandler.h / stereoFeatures.h / pinholeStereoCamera.h
// (include/keyFrame.h:35-37, include/mapHandler.h:54-55, app/plslam_dataset.cpp:27-28) and links libstvo.so
// (CMakeLists.txt:67).  This header re-creates the members and methods pl-slam touches — same names, argument
// meaning and error behaviour (std::runtime_error for impossible states, identity pose in-band when tracking
// fails) — so that src/keyFrame.cpp and the VO part of app/plslam_dataset.cpp compile against it.
//
// The reference's value types are cv::Mat and Eigen matrices; neither library exists in this image, so the shim is
// written against two tiny stand-ins (plf::Image, plf::MatN) with the accessors pl-slam uses.  A build that has
// OpenCV/Eigen maps them 1:1 (cv::Mat::data/step -> Image, Eigen::Matrix4d(row-major copy) -> Mat4d); see
// INTEGRATION.md.
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <stdexcept>
#include <string>
#include <vector>

#include "plslam_b200.h"

namespace plf {

struct Image {  // view of an 8-bit image of 1 (grey), 3 (BGR) or 4 (BGRA) interleaved channels (cv::Mat CV_8UC1 / 3 / 4:
                // data, cols, rows, step, channels())
  const uint8_t* data = nullptr;
  int cols = 0, rows = 0, step = 0;
  int channels = 1;
};

// Fixed-size f64 matrix / vector with the Eigen accessors pl-slam uses on stvo-pl's types: (r, c), (i), [i], Identity(),
// Zero().  Vectors are R x 1.
template <int R, int C>
struct Mat {
  std::array<double, R * C> v{};
  Mat() = default;
  Mat(double a, double b) { static_assert(R * C == 2, "2-vector"); v[0] = a; v[1] = b; }
  Mat(double a, double b, double c) { static_assert(R * C == 3, "3-vector"); v[0] = a; v[1] = b; v[2] = c; }
  double& operator()(int r, int c) { return v[r * C + c]; }
  double operator()(int r, int c) const { return v[r * C + c]; }
  double& operator()(int i) { return v[i]; }
  double operator()(int i) const { return v[i]; }
  double& operator[](int i) { return v[i]; }
  double operator[](int i) const { return v[i]; }
  double* data() { return v.data(); }
  const double* data() const { return v.data(); }
  static Mat Identity() {
    Mat m;
    for (int i = 0; i < (R < C ? R : C); ++i) m(i, i) = 1.0;
    return m;
  }
  static Mat Zero() { return Mat(); }
  bool operator==(const Mat& o) const { return v == o.v; }
};
using Matrix3d = Mat<3, 3>;
using Matrix4d = Mat<4, 4>;
using Matrix6d = Mat<6, 6>;
using Vector2d = Mat<2, 1>;
using Vector3d = Mat<3, 1>;
using Vector6d = Mat<6, 1>;

inline Matrix4d operator*(const Matrix4d& a, const Matrix4d& b) {
  Matrix4d c;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += a(i, k) * b(k, j);
      c(i, j) = s;
    }
  return c;
}

inline Matrix4d inverse_se3(const Matrix4d& T) {  // stvo-pl auxiliar: [R^T, -R^T t]
  Matrix4d Ti = Matrix4d::Identity();
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Ti(i, j) = T(j, i);
    Ti(i, 3) = -(T(0, i) * T(0, 3) + T(1, i) * T(1, 3) + T(2, i) * T(2, 3));
  }
  return Ti;
}

inline double det6(Matrix6d a) {  // LU with partial pivoting
  double det = 1;
  for (int k = 0; k < 6; ++k) {
    int p = k;
    for (int i = k + 1; i < 6; ++i)
      if (std::fabs(a(i, k)) > std::fabs(a(p, k))) p = i;
    if (a(p, k) == 0) return 0;
    if (p != k) {
      for (int j = 0; j < 6; ++j) std::swap(a(k, j), a(p, j));
      det = -det;
    }
    det *= a(k, k);
    for (int i = k + 1; i < 6; ++i) {
      const double f = a(i, k) / a(k, k);
      for (int j = k; j < 6; ++j) a(i, j) -= f * a(k, j);
    }
  }
  return det;
}

// stvo-pl auxiliar.h se(3) helpers on the host (x = [t; w], SURVEY Appendix A.4); the device versions are plf_se3.
inline Matrix4d expmap_se3(const Vector6d& x) {
  Matrix4d T = Matrix4d::Identity();
  const double wx = x(3), wy = x(4), wz = x(5), th = std::sqrt(wx * wx + wy * wy + wz * wz);
  if (th < 1e-6) {
    for (int i = 0; i < 3; ++i) T(i, 3) = x(i);
    return T;
  }
  const double s[3][3] = {{0, -wz / th, wy / th}, {wz / th, 0, -wx / th}, {-wy / th, wx / th, 0}};
  double s2[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) s2[i][j] = s[i][0] * s[0][j] + s[i][1] * s[1][j] + s[i][2] * s[2][j];
  const double a = std::sin(th), b = 1.0 - std::cos(th), c = (1.0 - std::cos(th)) / th, d = (th - std::sin(th)) / th;
  for (int i = 0; i < 3; ++i) {
    double t = 0;
    for (int j = 0; j < 3; ++j) {
      T(i, j) = (i == j ? 1.0 : 0.0) + s[i][j] * a + s2[i][j] * b;
      t += ((i == j ? 1.0 : 0.0) + s[i][j] * c + s2[i][j] * d) * x(j);
    }
    T(i, 3) = t;
  }
  return T;
}

inline Vector6d logmap_se3(const Matrix4d& T) {
  Vector6d x;
  double c = (T(0, 0) + T(1, 1) + T(2, 2) - 1.0) / 2.0;
  c = c > 1 ? 1 : (c < -1 ? -1 : c);
  const double th = std::acos(c);
  double w[3] = {0, 0, 0};
  if (th >= 1e-6) {
    const double k = th / (2.0 * std::sin(th));
    w[0] = k * (T(2, 1) - T(1, 2)); w[1] = k * (T(0, 2) - T(2, 0)); w[2] = k * (T(1, 0) - T(0, 1));
  }
  const double t[3] = {T(0, 3), T(1, 3), T(2, 3)};
  if (th < 1e-6) {
    for (int i = 0; i < 3; ++i) { x(i) = t[i]; x(3 + i) = w[i]; }
    return x;
  }
  // V^-1 = I - 0.5 [w]x + (1/th^2)(1 - (th sin th) / (2 (1 - cos th))) [w]x^2
  const double W[3][3] = {{0, -w[2], w[1]}, {w[2], 0, -w[0]}, {-w[1], w[0], 0}};
  const double kk = (1.0 - th * std::sin(th) / (2.0 * (1.0 - std::cos(th)))) / (th * th);
  for (int i = 0; i < 3; ++i) {
    double r = 0;
    for (int j = 0; j < 3; ++j) {
      double w2 = W[i][0] * W[0][j] + W[i][1] * W[1][j] + W[i][2] * W[2][j];
      r += ((i == j ? 1.0 : 0.0) - 0.5 * W[i][j] + kk * w2) * t[j];
    }
    x(i) = r;
    x(3 + i) = w[i];
  }
  return x;
}

}  // namespace plf

// stvo-pl gridStructure.h [UPSTREAM-RECALL, SURVEY A.2]: 48 x 64 matching grid
#define STVO_GRID_ROWS 48
#define STVO_GRID_COLS 64

namespace StVO {

using plf::Matrix3d;
using plf::Matrix4d;
using plf::Matrix6d;
using plf::Vector2d;
using plf::Vector3d;
using plf::Vector6d;
using plf::expmap_se3;
using plf::inverse_se3;
using plf::logmap_se3;
// The image type of StereoFrame::img_l / img_r and of initialize / insertStereoPair: cv::Mat in a build that has OpenCV
// (define STVO_SHIM_WITH_OPENCV after including <opencv2/core.hpp>; the shim reads data / cols / rows / step / channels()
// / depth() only), the plf::Image view otherwise.  Grey, BGR and BGRA frames are accepted; colour ones are converted to
// grey on the device, as stvo-pl's detectors convert them, and StereoFrame keeps the caller's colour view.
#ifdef STVO_SHIM_WITH_OPENCV
typedef cv::Mat Image;
inline int image_channels(const cv::Mat& m) { return m.channels(); }
inline bool image_8bit(const cv::Mat& m) { return m.depth() == CV_8U; }
#else
typedef plf::Image Image;
inline int image_channels(const plf::Image& m) { return m.channels; }
inline bool image_8bit(const plf::Image&) { return true; }
#endif

// stvo-pl PinholeStereoCamera (uses: app/plslam_dataset.cpp:84,97; src/mapHandler.cpp:255,551,1384-1385,3344)
class PinholeStereoCamera {
 public:
  PinholeStereoCamera(int width, int height, double fx, double fy, double cx, double cy, double b)
      : c_{width, height, fx, fy, cx, cy, b} {}
  int getWidth() const { return c_.width; }
  int getHeight() const { return c_.height; }
  double getFx() const { return c_.fx; }
  double getFy() const { return c_.fy; }
  double getCx() const { return c_.cx; }
  double getCy() const { return c_.cy; }
  double getB() const { return c_.b; }
  Vector2d projection(const Vector3d& P) const { return {c_.cx + c_.fx * P[0] / P[2], c_.cy + c_.fy * P[1] / P[2]}; }
  Vector3d backProjection(double u, double v, double disp) const {
    const double Z = c_.fx * c_.b / disp;
    return {Z * (u - c_.cx) / c_.fx, Z * (v - c_.cy) / c_.fy, Z};
  }
  const plf_camera& raw() const { return c_; }

 private:
  plf_camera c_;
};

// stvo-pl PointFeature / LineFeature: the members pl-slam reads or writes (SURVEY Appendix A.1)
struct PointFeature {
  Vector2d pl{}, pl_obs{};
  double disp = 0;
  Vector3d P{};
  int idx = -1, level = 0;
  bool inlier = true;
  double sigma2 = 1.0;
  PointFeature() = default;
  PointFeature(const Vector3d& P_, const Vector2d& pl_obs_) : pl_obs(pl_obs_), P(P_) {}  // src/mapHandler.cpp:3232
  PointFeature* safeCopy() const { return new PointFeature(*this); }                      // src/keyFrame.cpp:48
};

struct LineFeature {
  Vector2d spl{}, epl{}, spl_obs{}, epl_obs{};
  double sdisp = 0, edisp = 0, sdisp_obs = 0, edisp_obs = 0;
  Vector3d sP{}, eP{}, le{}, le_obs{};
  double angle = 0;
  int idx = -1, level = 0;
  bool inlier = true;
  double sigma2 = 1.0;
  LineFeature() = default;
  LineFeature(const Vector3d& sP_, const Vector3d& eP_, const Vector3d& le_obs_, const Vector2d& spl_, const Vector2d& epl_)
      : spl(spl_), epl(epl_), sP(sP_), eP(eP_), le_obs(le_obs_) {}  // src/mapHandler.cpp:3259
  LineFeature* safeCopy() const { return new LineFeature(*this); }   // src/keyFrame.cpp:53
};

// N x 32 descriptor block (stands in for the CV_8U cv::Mat pdesc_l / ldesc_l; row(i) <-> stereo_pt[i]/stereo_ls[i])
struct DescMat {
  std::vector<uint8_t> data;
  int rows = 0;
  static constexpr int cols = PLF_DESC_BYTES;
  const uint8_t* row(int i) const { return data.data() + (size_t)i * cols; }
  // cv::Mat::ptr<uchar>(i): the same expression then reads both the shim's block and a continuous CV_8U cv::Mat
  template <typename T> const T* ptr(int i = 0) const { return reinterpret_cast<const T*>(row(i)); }
};

// stvo-pl StereoFrame: the fields KeyFrame deep-copies (src/keyFrame.cpp:39-53)
class StereoFrame {
 public:
  StereoFrame(const Image& img_l_, const Image& img_r_, int idx, PinholeStereoCamera* cam_)
      : frame_idx(idx), img_l(img_l_), img_r(img_r_), cam(cam_) {
    // grid-cell scales, as the reference uses them (src/mapHandler.cpp:256,263,404-408: `pl(0) * curr_frame->inv_width`
    // feeds GridStructure::at / matchGrid): stvo-pl sets GRID_COLS / width and GRID_ROWS / height  [UPSTREAM-RECALL]
    inv_width = STVO_GRID_COLS / static_cast<double>(cam->getWidth());
    inv_height = STVO_GRID_ROWS / static_cast<double>(cam->getHeight());
  }
  ~StereoFrame() {
    for (auto* p : stereo_pt) delete p;
    for (auto* l : stereo_ls) delete l;
  }
  StereoFrame(const StereoFrame&) = delete;
  StereoFrame& operator=(const StereoFrame&) = delete;

  int frame_idx;
  Image img_l, img_r;
  Matrix4d Tfw = Matrix4d::Identity(), DT = Matrix4d::Identity();
  Matrix6d Tfw_cov = Matrix6d::Zero(), DT_cov = Matrix6d::Zero();
  double err_norm = -1;
  std::vector<PointFeature*> stereo_pt;
  std::vector<LineFeature*> stereo_ls;
  DescMat pdesc_l, pdesc_r, ldesc_l, ldesc_r;  // *_r kept for API shape; the hot path only consumes *_l
  PinholeStereoCamera* cam;
  double inv_width, inv_height;
};

// stvo-pl StereoFrameHandler (driven at app/plslam_dataset.cpp:109-159; reused at src/mapHandler.cpp:769-807)
class StereoFrameHandler {
 public:
  // adaptive_fast: stvo-pl's adaptative_fast with its fast_*_th values, or NULL for a fixed orb_fast_th.  One frame per
  // call (B = 1) is what makes the adaptation exact: frame k is detected at the threshold frame k-1's pose gave.
  // use_motion_model: stvo-pl's use_motion_model; frame k starts from the prediction frame k-1's pose gave (B = 1 again).
  explicit StereoFrameHandler(PinholeStereoCamera* cam_, const plf_params* params = nullptr, int device = 0,
                              const plf_adaptive_fast* adaptive_fast = nullptr, bool use_motion_model = false) : cam(cam_) {
    plf_limits lim;
    plf_default_limits(&lim);
    lim.max_batch = 1;  // the class API is one frame per call; batched callers use plf_process_batch directly
    if (params) prm_ = *params; else plf_default_params(&prm_);
    if (plf_create(&prm_, &cam->raw(), &lim, device, &ctx_) != PLF_OK)
      throw std::runtime_error(std::string("[StereoFrameHandler] ") + plf_last_error(nullptr));
    if ((adaptive_fast && plf_set_adaptive_fast(ctx_, adaptive_fast) != PLF_OK) ||
        (use_motion_model && plf_set_motion_model(ctx_, 1) != PLF_OK)) {
      const std::string e = plf_last_error(ctx_);
      plf_destroy(ctx_);
      throw std::runtime_error("[StereoFrameHandler] " + e);
    }
    lim_ = lim;
  }
  ~StereoFrameHandler() {
    for (auto* p : matched_pt) delete p;
    for (auto* l : matched_ls) delete l;
    delete prev_frame;
    delete curr_frame;
    plf_destroy(ctx_);
  }

  // app/plslam_dataset.cpp:115
  void initialize(const Image& img_l, const Image& img_r, int idx) {
    check(plf_reset_sequence(ctx_));
    delete prev_frame;
    prev_frame = run_frame(img_l, img_r, idx);
    if (last_.status != 2) throw std::runtime_error("[StereoFrameHandler] initialize: unexpected tracking state");
    prev_frame->Tfw = Matrix4d::Identity();
    prev_frame->Tfw_cov = Matrix6d::Identity();
    prev_frame->DT = Matrix4d::Identity();
    max_idx_pt = (int)prev_frame->stereo_pt.size();
    max_idx_ls = (int)prev_frame->stereo_ls.size();
    for (int i = 0; i < max_idx_pt; ++i) prev_frame->stereo_pt[i]->idx = i;
    for (int i = 0; i < max_idx_ls; ++i) prev_frame->stereo_ls[i]->idx = i;
    T_prevKF = Matrix4d::Identity();
    cov_prevKF_currF = Matrix6d::Zero();
    prev_f_iskf = true;
    N_prevKF_currF = 0;
  }

  // app/plslam_dataset.cpp:127 — extraction, stereo association and frame-to-frame tracking
  void insertStereoPair(const Image& img_l, const Image& img_r, int idx) {
    if (!prev_frame) throw std::runtime_error("[StereoFrameHandler] insertStereoPair before initialize");
    delete curr_frame;
    curr_frame = run_frame(img_l, img_r, idx);
    fetch_matches();
  }

  // app/plslam_dataset.cpp:128; src/mapHandler.cpp:780.  The pose increment was computed on the device in the same
  // launch sequence as the tracking; this publishes it exactly as stvo-pl's optimizePose does.
  void optimizePose() {
    if (!curr_frame) throw std::runtime_error("[StereoFrameHandler] optimizePose without a current frame");
    if (last_.status == 0) {
      std::memcpy(curr_frame->DT.v.data(), last_.DT, sizeof last_.DT);
      std::memcpy(curr_frame->DT_cov.v.data(), last_.DT_cov, sizeof last_.DT_cov);
      curr_frame->err_norm = last_.err;
      curr_frame->Tfw = prev_frame->Tfw * curr_frame->DT;
      curr_frame->Tfw_cov = prev_frame->Tfw_cov;  // covariance composition (unccomp_se3) stays with the caller
    } else {  // not enough features: identity motion, as stvo-pl falls back
      curr_frame->DT = Matrix4d::Identity();
      curr_frame->DT_cov = Matrix6d::Zero();
      curr_frame->err_norm = -1;
      curr_frame->Tfw = prev_frame->Tfw;
      curr_frame->Tfw_cov = prev_frame->Tfw_cov;
    }
    n_inliers_pt = last_.n_inliers_pt;
    n_inliers_ls = last_.n_inliers_ls;
    n_inliers = n_inliers_pt + n_inliers_ls;
  }

  // app/plslam_dataset.cpp:135 — SURVEY Appendix A.2 (entropy ratio of the pose covariance OR motion since last KF)
  bool needNewKF(double min_entropy_ratio = 0.85, double max_kf_t_dist = 5.0, double max_kf_r_dist = 15.0) {
    const double two_pi_e = 3.0 * (1.0 + std::log(2.0 * std::acos(-1.0)));
    if (prev_f_iskf) {
      const double d = plf::det6(curr_frame->DT_cov);
      entropy_first_prevKF = d != 0.0 ? two_pi_e + 0.5 * std::log(d) : -999999999.99;
      prev_f_iskf = false;
    }
    const Matrix4d DTk = plf::inverse_se3(curr_frame->Tfw) * T_prevKF;
    const double t = std::sqrt(DTk(0, 3) * DTk(0, 3) + DTk(1, 3) * DTk(1, 3) + DTk(2, 3) * DTk(2, 3));
    double c = (DTk(0, 0) + DTk(1, 1) + DTk(2, 2) - 1.0) / 2.0;
    c = c > 1 ? 1 : (c < -1 ? -1 : c);
    const double r = std::acos(c) * 180.0 / std::acos(-1.0);
    for (int i = 0; i < 36; ++i) cov_prevKF_currF.v[i] += curr_frame->DT_cov.v[i];
    const double entropy_curr = two_pi_e + 0.5 * std::log(plf::det6(cov_prevKF_currF));
    const double ratio = entropy_curr / entropy_first_prevKF;
    const bool lost = curr_frame->DT_cov == Matrix6d::Zero() && curr_frame->DT == Matrix4d::Identity();
    if (ratio < min_entropy_ratio || std::isnan(ratio) || std::isinf(ratio) || lost || t > max_kf_t_dist ||
        r > max_kf_r_dist || N_prevKF_currF > 10)
      return true;
    ++N_prevKF_currF;
    return false;
  }

  // app/plslam_dataset.cpp:145
  void currFrameIsKF() {
    prev_f_iskf = true;
    T_prevKF = curr_frame->Tfw;
    cov_prevKF_currF = Matrix6d::Zero();
    N_prevKF_currF = 0;
  }

  // stvo-pl's orb_fast_th member: the FAST threshold the next frame is detected with (initialize() uses orb_fast_th).
  // With adaptive_fast the device moves it after every tracked frame, so updateFrame has nothing left to do for it.
  int orbFastTh() {
    int th = 0;
    check(plf_get_sequence_fast_th(ctx_, 0, &th));
    return th;
  }

  // The motion prediction (row-major 4x4) the next frame starts from: inverse(prev_frame->DT) after a good solution, else
  // the identity (DESIGN.md section 8); returns whether it came from a good solution.
  bool motionPrior(double T[16]) {
    int valid = 0;
    check(plf_get_sequence_motion(ctx_, 0, T, &valid));
    return valid != 0;
  }

  // app/plslam_dataset.cpp:159
  void updateFrame() {
    for (auto* p : matched_pt) delete p;
    for (auto* l : matched_ls) delete l;
    matched_pt.clear();
    matched_ls.clear();
    delete prev_frame;
    prev_frame = curr_frame;
    curr_frame = nullptr;
  }

  StereoFrame* prev_frame = nullptr;
  StereoFrame* curr_frame = nullptr;
  std::list<PointFeature*> matched_pt;
  std::list<LineFeature*> matched_ls;
  int n_inliers = 0, n_inliers_pt = 0, n_inliers_ls = 0;
  int max_idx_pt = 0, max_idx_ls = 0;
  PinholeStereoCamera* cam;
  const plf_frame_result& last_result() const { return last_; }
  plf_ctx* ctx() { return ctx_; }

 private:
  void check(plf_status st) {
    if (st != PLF_OK) throw std::runtime_error(std::string("[StereoFrameHandler] ") + plf_last_error(ctx_));
  }

  StereoFrame* run_frame(const Image& l, const Image& r, int idx) {
    if (l.cols != cam->getWidth() || l.rows != cam->getHeight() || r.cols != l.cols || r.rows != l.rows || (size_t)l.step != (size_t)r.step)
      throw std::runtime_error("[StereoFrameHandler] image size does not match the camera");
    const int ch = image_channels(l);
    if (!image_8bit(l) || !image_8bit(r) || image_channels(r) != ch || (ch != 1 && ch != 3 && ch != 4))
      throw std::runtime_error("[StereoFrameHandler] images must be 8-bit grey, BGR or BGRA, both alike");
    if (ch == 1) {
      check(plf_process_batch(ctx_, 1, l.data, r.data, (int)(size_t)l.step, &last_));
    } else {
      check(plf_batch_upload_color(ctx_, 1, l.data, r.data, (int)(size_t)l.step, ch));
      check(plf_batch_run(ctx_, 1));
      check(plf_batch_download(ctx_, 1, &last_));
    }
    auto* f = new StereoFrame(l, r, idx, cam);
    const int K = lim_.max_keypoints, Ln = lim_.max_lines;
    std::vector<double> pl(2 * (size_t)K), disp(K), P(3 * (size_t)K), spl(2 * (size_t)Ln), epl(2 * (size_t)Ln), sd(Ln), ed(Ln),
        sP(3 * (size_t)Ln), eP(3 * (size_t)Ln), le(3 * (size_t)Ln);
    std::vector<int32_t> oct(K);
    std::vector<float> ang(Ln);
    f->pdesc_l.data.resize((size_t)K * 32);
    f->ldesc_l.data.resize((size_t)Ln * 32);
    plf_frame_view v{};
    v.cap_pt = K; v.cap_ls = Ln;
    v.pt_pl = pl.data(); v.pt_disp = disp.data(); v.pt_P = P.data(); v.pt_octave = oct.data(); v.pdesc = f->pdesc_l.data.data();
    v.ls_spl = spl.data(); v.ls_epl = epl.data(); v.ls_sdisp = sd.data(); v.ls_edisp = ed.data(); v.ls_sP = sP.data();
    v.ls_eP = eP.data(); v.ls_le = le.data(); v.ls_angle = ang.data(); v.ldesc = f->ldesc_l.data.data();
    check(plf_get_frame(ctx_, 0, &v));
    f->pdesc_l.rows = v.n_pt; f->pdesc_l.data.resize((size_t)v.n_pt * 32);
    f->ldesc_l.rows = v.n_ls; f->ldesc_l.data.resize((size_t)v.n_ls * 32);
    for (int i = 0; i < v.n_pt; ++i) {
      auto* p = new PointFeature();
      p->pl = {pl[2 * i], pl[2 * i + 1]};
      p->disp = disp[i];
      p->P = {P[3 * i], P[3 * i + 1], P[3 * i + 2]};
      p->level = oct[i];
      f->stereo_pt.push_back(p);
    }
    for (int i = 0; i < v.n_ls; ++i) {
      auto* q = new LineFeature();
      q->spl = {spl[2 * i], spl[2 * i + 1]}; q->epl = {epl[2 * i], epl[2 * i + 1]};
      q->sdisp = sd[i]; q->edisp = ed[i];
      q->sP = {sP[3 * i], sP[3 * i + 1], sP[3 * i + 2]}; q->eP = {eP[3 * i], eP[3 * i + 1], eP[3 * i + 2]};
      q->le = {le[3 * i], le[3 * i + 1], le[3 * i + 2]};
      q->angle = ang[i];
      f->stereo_ls.push_back(q);
    }
    return f;
  }

  void fetch_matches() {
    for (auto* p : matched_pt) delete p;
    for (auto* l : matched_ls) delete l;
    matched_pt.clear();
    matched_ls.clear();
    const int K = lim_.max_keypoints, Ln = lim_.max_lines;
    std::vector<double> P(3 * (size_t)K), obs(2 * (size_t)K), sP(3 * (size_t)Ln), eP(3 * (size_t)Ln), le(3 * (size_t)Ln);
    std::vector<uint8_t> ip(K), il(Ln);
    plf_match_view m{};
    m.cap_pt = K; m.cap_ls = Ln;
    m.P = P.data(); m.pl_obs = obs.data(); m.inlier_pt = ip.data(); m.sP = sP.data(); m.eP = eP.data(); m.le_obs = le.data();
    m.inlier_ls = il.data();
    check(plf_get_matches(ctx_, 0, &m));
    for (int i = 0; i < m.n_pt; ++i) {
      auto* p = new PointFeature({P[3 * i], P[3 * i + 1], P[3 * i + 2]}, {obs[2 * i], obs[2 * i + 1]});
      p->inlier = ip[i] != 0;
      matched_pt.push_back(p);
    }
    for (int i = 0; i < m.n_ls; ++i) {
      auto* l = new LineFeature({sP[3 * i], sP[3 * i + 1], sP[3 * i + 2]}, {eP[3 * i], eP[3 * i + 1], eP[3 * i + 2]},
                                {le[3 * i], le[3 * i + 1], le[3 * i + 2]}, {}, {});
      l->inlier = il[i] != 0;
      matched_ls.push_back(l);
    }
  }

  plf_ctx* ctx_ = nullptr;
  plf_params prm_;
  plf_limits lim_;
  plf_frame_result last_{};
  Matrix4d T_prevKF = Matrix4d::Identity();
  Matrix6d cov_prevKF_currF = Matrix6d::Zero();
  double entropy_first_prevKF = 0;
  bool prev_f_iskf = true;
  int N_prevKF_currF = 0;
};

// Free matcher of stvo-pl matching.h: int match(const Mat&, const Mat&, float nnr, vector<int>&)
// (src/mapHandler.cpp:277,424,597,712,3223,3249) on a handler's context.
inline int match(plf_ctx* ctx, const DescMat& d1, const DescMat& d2, float nnr, std::vector<int>& matches_12, bool best_lr = true) {
  matches_12.assign(d1.rows, -1);
  int n = 0;
  if (plf_match(ctx, d1.data.data(), d1.rows, d2.data.data(), d2.rows, nnr, best_lr ? 1 : 0, matches_12.data(), &n) != PLF_OK)
    throw std::runtime_error(std::string("[match] ") + plf_last_error(ctx));
  return n;
}

// ---- stvo-pl gridStructure.h / matching.h: the windowed matcher pl-slam uses when SlamConfig::fastMatching() ----------
// (src/mapHandler.cpp:251-271 points, :382-418 lines; also :580-591, :686-706).  Cell coordinates are ints: callers scale
// pixels by inv_width = GRID_COLS / width, inv_height = GRID_ROWS / height and the pair<double,double> -> pair<int,int>
// conversion truncates.  [UPSTREAM-RECALL]: restated from SURVEY Appendix A.3, see oracle/matchgrid.py.
#define GRID_ROWS STVO_GRID_ROWS
#define GRID_COLS STVO_GRID_COLS
typedef std::pair<int, int> point_2d;
typedef std::pair<point_2d, point_2d> line_2d;

struct GridWindow {
  std::pair<int, int> width, height;
};

inline void normalize(std::pair<double, double>& v) {  // unguarded, as upstream
  const double m = std::sqrt(v.first * v.first + v.second * v.second);
  v.first /= m;
  v.second /= m;
}

// cells of the 8-connected line between two cells, end points included
inline void getLineCoords(double x1d, double y1d, double x2d, double y2d, std::list<point_2d>& line_coords) {
  line_coords.clear();
  int x1 = (int)x1d, y1 = (int)y1d, x2 = (int)x2d, y2 = (int)y2d;
  const bool steep = std::abs(y2 - y1) > std::abs(x2 - x1);
  if (steep) { std::swap(x1, y1); std::swap(x2, y2); }
  if (x1 > x2) { std::swap(x1, x2); std::swap(y1, y2); }
  const int dx = x2 - x1, dy = std::abs(y2 - y1), ystep = y1 < y2 ? 1 : -1;
  int err = dx / 2, y = y1;
  for (int x = x1; x <= x2; ++x) {
    line_coords.emplace_back(steep ? y : x, steep ? x : y);
    err -= dy;
    if (err < 0) { y += ystep; err += dx; }
  }
}

class GridStructure {
 public:
  int rows, cols;
  GridStructure(int rows_, int cols_) : rows(rows_), cols(cols_), grid(cols_, std::vector<std::list<int>>(rows_)) {
    if (rows_ <= 0 || cols_ <= 0) throw std::runtime_error("[GridStructure] invalid dimension");
  }
  std::list<int>& at(int x, int y) { return (x >= 0 && x < cols && y >= 0 && y < rows) ? grid[x][y] : out_of_bounds; }
  void clear() { for (auto& c : grid) for (auto& l : c) l.clear(); }
  // the C ABI's form: cell (x, y) owns items[start[x*rows+y] .. start[x*rows+y+1])
  void flatten(std::vector<int>& start, std::vector<int>& items) const {
    start.assign(1, 0); items.clear();
    for (int x = 0; x < cols; ++x)
      for (int y = 0; y < rows; ++y) {
        items.insert(items.end(), grid[x][y].begin(), grid[x][y].end());
        start.push_back((int)items.size());
      }
  }
 private:
  std::vector<std::vector<std::list<int>>> grid;
  std::list<int> out_of_bounds;
};

inline int matchGrid(plf_ctx* ctx, const std::vector<point_2d>& points, const DescMat& d1, const GridStructure& grid,
                     const DescMat& d2, const GridWindow& w, std::vector<int>& matches_12, float nnr, bool best_lr = true) {
  if ((int)points.size() != d1.rows) throw std::runtime_error("[matchGrid] each point needs a corresponding descriptor!");
  std::vector<int> q; q.reserve(2 * points.size());
  for (const auto& p : points) { q.push_back(p.first); q.push_back(p.second); }
  std::vector<int> start, items;
  grid.flatten(start, items);
  matches_12.assign(d1.rows, -1);
  int n = 0;
  const plf_grid_window gw = {w.width.first, w.width.second, w.height.first, w.height.second};
  if (plf_match_grid_points(ctx, q.data(), d1.data.data(), d1.rows, start.data(), items.data(), d2.data.data(), d2.rows,
                            grid.cols, grid.rows, gw, nnr, best_lr ? 1 : 0, matches_12.data(), &n) != PLF_OK)
    throw std::runtime_error(std::string("[matchGrid] ") + plf_last_error(ctx));
  return n;
}

inline int matchGrid(plf_ctx* ctx, const std::vector<line_2d>& lines, const DescMat& d1, const GridStructure& grid,
                     const DescMat& d2, const std::vector<std::pair<double, double>>& directions2, const GridWindow& w,
                     std::vector<int>& matches_12, float nnr, double line_sim_th, bool best_lr = true) {
  if ((int)lines.size() != d1.rows) throw std::runtime_error("[matchGrid] each line needs a corresponding descriptor!");
  if ((int)directions2.size() != d2.rows) throw std::runtime_error("[matchGrid] each train line needs a direction!");
  std::vector<int> q; q.reserve(4 * lines.size());
  for (const auto& l : lines) { q.push_back(l.first.first); q.push_back(l.first.second); q.push_back(l.second.first); q.push_back(l.second.second); }
  std::vector<double> dir; dir.reserve(2 * directions2.size());
  for (const auto& v : directions2) { dir.push_back(v.first); dir.push_back(v.second); }
  std::vector<int> start, items;
  grid.flatten(start, items);
  matches_12.assign(d1.rows, -1);
  int n = 0;
  const plf_grid_window gw = {w.width.first, w.width.second, w.height.first, w.height.second};
  if (plf_match_grid_lines(ctx, q.data(), d1.data.data(), d1.rows, start.data(), items.data(), dir.data(), d2.data.data(),
                           d2.rows, grid.cols, grid.rows, gw, nnr, line_sim_th, best_lr ? 1 : 0, matches_12.data(), &n) != PLF_OK)
    throw std::runtime_error(std::string("[matchGrid] ") + plf_last_error(ctx));
  return n;
}

}  // namespace StVO
