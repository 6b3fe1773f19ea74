// Relative pose between two keyframes for loop closure / keyframe refinement (SURVEY §8(f) f2): the composition
// MapHandler::isLoopClosure (src/mapHandler.cpp:3192-3300) -> computeRelativePoseRobustGN (:3566-3957) performs, on
// the operators of this library: match() twice (points :3223, lines :3249) -> the two-stage robust Gauss-Newton of
// plf_gn_pose (the in-tree twin of optimizePose IS this function, :3566-3872) -> the acceptance tests (:3875-3906) ->
// pose_inc and the surviving correspondences (:3909-3950).
//
// The matching and the pose refinement run on the device (k_hamming_knn2_mma / k_nnr_mutual / k_gn_pose through the host
// entry points); what is left on the host is the decision block: five scalar comparisons, one symmetric 6x6
// eigenvalue (cyclic Jacobi) and the se(3) maps, all f64.
#include <float.h>
#include <math.h>

#include "plf_internal.h"
#include "plf_se3.cuh"

// largest eigenvalue of a symmetric 6x6 matrix (cyclic Jacobi; Eigen's SelfAdjointEigenSolver sorts ascending and the
// reference reads element 5, :3883-3885)
static double sym6_max_eig(const double* A_in) {
  double A[36];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) A[6 * i + j] = 0.5 * (A_in[6 * i + j] + A_in[6 * j + i]);
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0;
    for (int i = 0; i < 6; ++i)
      for (int j = i + 1; j < 6; ++j) off += A[6 * i + j] * A[6 * i + j];
    if (off < 1e-300) break;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) {
        const double apq = A[6 * p + q];
        if (apq == 0.0) continue;
        const double theta = (A[6 * q + q] - A[6 * p + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; ++k) {  // A <- J^T A J
          const double akp = A[6 * k + p], akq = A[6 * k + q];
          A[6 * k + p] = c * akp - s * akq;
          A[6 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 6; ++k) {
          const double apk = A[6 * p + k], aqk = A[6 * q + k];
          A[6 * p + k] = c * apk - s * aqk;
          A[6 * q + k] = s * apk + c * aqk;
        }
      }
  }
  double m = A[0];
  for (int i = 1; i < 6; ++i) m = A[7 * i] > m ? A[7 * i] : m;
  return m;
}

extern "C" plf_status plf_loop_closure_pose(plf_ctx* ctx, const plf_lc_params* lc, const plf_lc_keyframe* kf0,
                                            const plf_lc_keyframe* kf1, plf_lc_result* out, int32_t* pt_pairs,
                                            int cap_pt, int32_t* ls_pairs, int cap_ls) {
  if (!ctx || !lc || !kf0 || !kf1 || !out || kf0->n_pt < 0 || kf1->n_pt < 0 || kf0->n_ls < 0 || kf1->n_ls < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_loop_closure_pose: bad arguments");
  memset(out, 0, sizeof *out);
  const plf_params& P = ctx->params;
  plf_status st;
  // ---- find matches between both KFs (:3217-3273) ----
  std::vector<int32_t> m_pt(std::max(kf0->n_pt, 1), -1), m_ls(std::max(kf0->n_ls, 1), -1);
  int common_pt = 0, common_ls = 0;
  if (P.has_points && kf0->n_pt > 0 && kf1->n_pt > 0) {
    if (!kf0->pdesc || !kf1->pdesc || !kf0->P || !kf1->pl) return plf_fail(ctx, PLF_ERR_INVALID, "plf_loop_closure_pose: point arrays missing");
    if ((st = plf_match(ctx, kf0->pdesc, kf0->n_pt, kf1->pdesc, kf1->n_pt, P.min_ratio_12_p, P.best_lr_matches, m_pt.data(), &common_pt))) return st;
  }
  if (P.has_lines && kf0->n_ls > 0 && kf1->n_ls > 0) {
    if (!kf0->ldesc || !kf1->ldesc || !kf0->sP || !kf0->eP || !kf1->le) return plf_fail(ctx, PLF_ERR_INVALID, "plf_loop_closure_pose: line arrays missing");
    if ((st = plf_match(ctx, kf0->ldesc, kf0->n_ls, kf1->ldesc, kf1->n_ls, P.min_ratio_12_l, P.best_lr_matches, m_ls.data(), &common_ls))) return st;
  }
  std::vector<double> gP, gO, gs, ge, gl;
  std::vector<int32_t> ip, il;  // (i1, i2) per correspondence
  for (int i1 = 0; i1 < kf0->n_pt && common_pt > 0; ++i1) {
    const int i2 = m_pt[i1];
    if (i2 < 0) continue;
    gP.insert(gP.end(), kf0->P + 3 * (size_t)i1, kf0->P + 3 * (size_t)i1 + 3);
    gO.insert(gO.end(), kf1->pl + 2 * (size_t)i2, kf1->pl + 2 * (size_t)i2 + 2);
    ip.push_back(i1); ip.push_back(i2);
  }
  for (int i1 = 0; i1 < kf0->n_ls && common_ls > 0; ++i1) {
    const int i2 = m_ls[i1];
    if (i2 < 0) continue;
    gs.insert(gs.end(), kf0->sP + 3 * (size_t)i1, kf0->sP + 3 * (size_t)i1 + 3);
    ge.insert(ge.end(), kf0->eP + 3 * (size_t)i1, kf0->eP + 3 * (size_t)i1 + 3);
    gl.insert(gl.end(), kf1->le + 3 * (size_t)i2, kf1->le + 3 * (size_t)i2 + 3);
    il.push_back(i1); il.push_back(i2);
  }
  out->common_pt = common_pt;
  out->common_ls = common_ls;
  // ---- inlier-ratio pre-condition (:3277-3299); x / 0 follows IEEE as in the reference (inf / nan compare false) ----
  auto std_max = [](double a, double b) { return a < b ? b : a; };  // std::max's NaN behaviour (0 / 0 when a frame is empty)
  const double rp = std_max(100.0 * common_pt / kf0->n_pt, 100.0 * common_pt / kf1->n_pt);
  const double rl = std_max(100.0 * common_ls / kf0->n_ls, 100.0 * common_ls / kf1->n_ls);
  out->inl_ratio_pt = rp;
  out->inl_ratio_ls = rl;
  bool cond = false;
  if (P.has_points && P.has_lines) cond = rp > lc->lc_inlier_ratio && rl > lc->lc_inlier_ratio;
  else if (P.has_points) cond = rp > lc->lc_inlier_ratio;
  else if (P.has_lines) cond = rl > lc->lc_inlier_ratio;
  if (!cond) return PLF_OK;  // accepted = 0, nothing estimated
  // ---- computeRelativePoseRobustGN (:3566-3872): both stages stop on DBL_EPSILON, iteration counts from the config ----
  const int np = (int)ip.size() / 2, nl = (int)il.size() / 2;
  std::vector<uint8_t> inl_p(std::max(np, 1), 1), inl_l(std::max(nl, 1), 1);
  plf_gn_opts o = {P.homog_th, P.max_iters, P.max_iters_ref, DBL_EPSILON, DBL_EPSILON, DBL_EPSILON};
  plf_pose_result r;
  if ((st = plf_gn_pose(ctx, &o, gP.data(), gO.data(), inl_p.data(), np, gs.data(), ge.data(), gl.data(), inl_l.data(), nl, nullptr, &r))) return st;
  out->estimated = 1;
  out->err = r.err;
  memcpy(out->x_inc, r.x, sizeof r.x);
  // ---- Check whether it is Loop Closure or not (:3875-3906) ----
  out->max_cov_eig = sym6_max_eig(r.cov);
  int n_inl = 0;
  for (int i = 0; i < np; ++i) n_inl += inl_p[i] != 0;
  for (int i = 0; i < nl; ++i) n_inl += inl_l[i] != 0;
  out->ratio_inliers = (double)n_inl / (double)(np + nl);
  out->t = sqrt(r.x[0] * r.x[0] + r.x[1] * r.x[1] + r.x[2] * r.x[2]);
  out->r = sqrt(r.x[3] * r.x[3] + r.x[4] * r.x[4] + r.x[5] * r.x[5]) * 180.f / 3.1415926535897932384626433832795;
  const bool lc_res = r.err < lc->lc_res, lc_unc = out->max_cov_eig < lc->lc_unc;
  const bool lc_inl = true;  // the reference overrides its own inlier-ratio test (`lc_inl = true;`, :3900)
  const bool lc_trs = out->t < lc->lc_trs, lc_rot = out->r < lc->lc_rot;
  if (!(lc_res && lc_unc && lc_inl && lc_trs && lc_rot)) return PLF_OK;
  // ---- accepted: inlier correspondences and pose_inc = logmap(inverse(expmap(x_inc))) (:3909-3951) ----
  int kp = 0, kl = 0;
  for (int i = 0; i < np; ++i)
    if (inl_p[i]) {
      if (kp < cap_pt && pt_pairs) { pt_pairs[2 * kp] = ip[2 * i]; pt_pairs[2 * kp + 1] = ip[2 * i + 1]; }
      ++kp;
    }
  for (int i = 0; i < nl; ++i)
    if (inl_l[i]) {
      if (kl < cap_ls && ls_pairs) { ls_pairs[2 * kl] = il[2 * i]; ls_pairs[2 * kl + 1] = il[2 * i + 1]; }
      ++kl;
    }
  out->n_pt = kp;
  out->n_ls = kl;
  if ((pt_pairs && kp > cap_pt) || (ls_pairs && kl > cap_ls))
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_loop_closure_pose: %d point / %d line correspondences exceed the caller's capacity", kp, kl);
  double T[16], Ti[16];
  if ((st = plf_se3(ctx, 0, r.x, T))) return st;  // expmap_se3(x_inc)
  d_inverse_se3(T, Ti);
  if ((st = plf_se3(ctx, 1, Ti, out->pose_inc))) return st;
  out->accepted = 1;
  return PLF_OK;
}
