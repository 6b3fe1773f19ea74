/*
 * oracle/gn.c — CPU restatement of the robust point+line Gauss-Newton pose refinement.
 * TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * Follows the in-tree twin of stvo-pl's StereoFrameHandler::optimizePose:
 *   MapHandler::computeRelativePoseGN        src/mapHandler.cpp:3302-3564
 *   MapHandler::computeRelativePoseRobustGN  src/mapHandler.cpp:3566-3957 (two stages + chi2 gate)
 * point row :3331-3367, line row :3371-3426, normalise :3432, stop tests :3434,:3441, solve :3437-3438
 * (Eigen ColPivHouseholderQR), update T = T * inverse_se3(expmap_se3(dx)) :3439, outlier gate
 * > sqrt(7.815) :3451-3482, refinement :3753-3872, cov = H^-1 :3491.
 * se(3) helpers follow SURVEY.md Appendix A.4 (stvo-pl auxiliar; ordering [t; w] confirmed at
 * src/mapHandler.cpp:3513-3514); stvo-pl is not vendored => these are "parity unpinned".
 * Pinhole projection: (cx + fx X/Z, cy + fy Y/Z) (cam->projection, src/mapHandler.cpp:255,3336).
 *
 * The twin stops on numeric_limits<double>::epsilon(); stvo-pl stops on Config::minError /
 * minErrorChange.  Both thresholds are parameters here (eps_err, eps_change, eps_step).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "oracle.h"

/* ---- se(3) ------------------------------------------------------------------------------------ */
static void mat3_mul(const double* A, const double* B, double* C) {
  double t[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) t[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  memcpy(C, t, sizeof t);
}
static void skew(const double* w, double* S) {
  S[0] = 0; S[1] = -w[2]; S[2] = w[1];
  S[3] = w[2]; S[4] = 0; S[5] = -w[0];
  S[6] = -w[1]; S[7] = w[0]; S[8] = 0;
}

/* x = [t; w] -> T (row-major 4x4) */
void orc_expmap_se3(const double* x, double* T) {
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {x[0], x[1], x[2]};
  const double* w = x + 3;
  double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (!(theta < 0.000001)) {
    double s[9], s2[9], V[9];
    skew(w, s);
    for (int i = 0; i < 9; i++) s[i] /= theta;
    mat3_mul(s, s, s2);
    double sn = sin(theta), cs = cos(theta);
    for (int i = 0; i < 9; i++) {
      double I = (i % 4 == 0) ? 1.0 : 0.0;
      R[i] = I + s[i] * sn + s2[i] * (1.0 - cs);
      V[i] = I + s[i] * (1.0 - cs) / theta + s2[i] * (theta - sn) / theta;
    }
    double tt[3];
    for (int i = 0; i < 3; i++) tt[i] = V[3 * i] * t[0] + V[3 * i + 1] * t[1] + V[3 * i + 2] * t[2];
    memcpy(t, tt, sizeof tt);
  }
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) T[4 * i + j] = R[3 * i + j];
    T[4 * i + 3] = t[i];
  }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
}

void orc_inverse_se3(const double* T, double* Ti) {
  double R[9], t[3] = {T[3], T[7], T[11]};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[3 * i + j] = T[4 * j + i]; /* transpose */
  double out[16];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) out[4 * i + j] = R[3 * i + j];
    out[4 * i + 3] = -(R[3 * i] * t[0] + R[3 * i + 1] * t[1] + R[3 * i + 2] * t[2]);
  }
  out[12] = out[13] = out[14] = 0;
  out[15] = 1;
  memcpy(Ti, out, sizeof out);
}

static int inv3(const double* A, double* Ai) {
  double det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
  double id = 1.0 / det;
  Ai[0] = (A[4] * A[8] - A[5] * A[7]) * id; Ai[1] = (A[2] * A[7] - A[1] * A[8]) * id; Ai[2] = (A[1] * A[5] - A[2] * A[4]) * id;
  Ai[3] = (A[5] * A[6] - A[3] * A[8]) * id; Ai[4] = (A[0] * A[8] - A[2] * A[6]) * id; Ai[5] = (A[2] * A[3] - A[0] * A[5]) * id;
  Ai[6] = (A[3] * A[7] - A[4] * A[6]) * id; Ai[7] = (A[1] * A[6] - A[0] * A[7]) * id; Ai[8] = (A[0] * A[4] - A[1] * A[3]) * id;
  return det != 0;
}

void orc_logmap_se3(const double* T, double* x) {
  double R[9], Vt[3] = {T[3], T[7], T[11]}, w[3] = {0, 0, 0};
  double V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[3 * i + j] = T[4 * i + j];
  double cosine = (R[0] + R[4] + R[8] - 1.0) / 2.0;
  if (cosine > 1.0) cosine = 1.0; else if (cosine < -1.0) cosine = -1.0;
  double sine = sqrt(1.0 - cosine * cosine);
  if (sine > 1.0) sine = 1.0; else if (sine < -1.0) sine = -1.0;
  double theta = acos(cosine);
  if (theta > 0.000001) {
    /* w_hat = theta (R - R^T) / (2 sine); w = skewcoords(w_hat) */
    double k = theta / (2.0 * sine);
    w[0] = k * (R[7] - R[5]);
    w[1] = k * (R[2] - R[6]);
    w[2] = k * (R[3] - R[1]);
    double s[9], s2[9];
    skew(w, s);
    for (int i = 0; i < 9; i++) s[i] /= theta;
    mat3_mul(s, s, s2);
    for (int i = 0; i < 9; i++) {
      double I = (i % 4 == 0) ? 1.0 : 0.0;
      V[i] = I + s[i] * (1.0 - cosine) / theta + s2[i] * (theta - sine) / theta;
    }
  }
  double Vi[9];
  inv3(V, Vi);
  for (int i = 0; i < 3; i++) x[i] = Vi[3 * i] * Vt[0] + Vi[3 * i + 1] * Vt[1] + Vi[3 * i + 2] * Vt[2];
  x[3] = w[0]; x[4] = w[1]; x[5] = w[2];
}

static void mat4_mul(const double* A, const double* B, double* C) {
  double t[16];
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      double a = 0;
      for (int k = 0; k < 4; k++) a += A[4 * i + k] * B[4 * k + j];
      t[4 * i + j] = a;
    }
  memcpy(C, t, sizeof t);
}

/* ---- 6x6 column-pivoting Householder QR solve (Eigen ColPivHouseholderQR::solve semantics) ------ */
void orc_colpiv_qr_solve6(const double* Hin, const double* gin, double* x) {
  const int n = 6;
  double A[36], b[6], colnorm[6];
  int perm[6];
  memcpy(A, Hin, sizeof A);
  memcpy(b, gin, sizeof b);
  for (int j = 0; j < n; j++) {
    perm[j] = j;
    double s = 0;
    for (int i = 0; i < n; i++) s += A[n * i + j] * A[n * i + j];
    colnorm[j] = s;
  }
  double maxnorm2 = 0;
  for (int j = 0; j < n; j++) if (colnorm[j] > maxnorm2) maxnorm2 = colnorm[j];
  double thresh = DBL_EPSILON * n; /* Eigen: threshold = eps * diagonalSize, relative to max pivot */
  double maxpivot = 0;
  int rank = n;
  double R_diag[6];
  for (int k = 0; k < n; k++) {
    /* pivot: column with the largest remaining squared norm (recomputed, as Eigen effectively does) */
    int piv = k;
    double best = -1;
    for (int j = k; j < n; j++) {
      double s = 0;
      for (int i = k; i < n; i++) s += A[n * i + j] * A[n * i + j];
      colnorm[j] = s;
      if (s > best) { best = s; piv = j; }
    }
    if (piv != k) {
      for (int i = 0; i < n; i++) { double t = A[n * i + k]; A[n * i + k] = A[n * i + piv]; A[n * i + piv] = t; }
      int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
    }
    /* Householder on column k, rows k..n-1 */
    double c0 = A[n * k + k], tail = 0;
    for (int i = k + 1; i < n; i++) tail += A[n * i + k] * A[n * i + k];
    double beta, tau, v[6];
    if (tail == 0) {
      tau = 0; beta = c0;
      for (int i = k + 1; i < n; i++) v[i] = 0;
    } else {
      beta = sqrt(c0 * c0 + tail);
      if (c0 >= 0) beta = -beta;
      for (int i = k + 1; i < n; i++) v[i] = A[n * i + k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    v[k] = 1;
    /* apply H = I - tau v v^T to the remaining columns and to b */
    for (int j = k + 1; j < n; j++) {
      double s = 0;
      for (int i = k; i < n; i++) s += v[i] * A[n * i + j];
      s *= tau;
      for (int i = k; i < n; i++) A[n * i + j] -= s * v[i];
    }
    {
      double s = 0;
      for (int i = k; i < n; i++) s += v[i] * b[i];
      s *= tau;
      for (int i = k; i < n; i++) b[i] -= s * v[i];
    }
    A[n * k + k] = beta;
    for (int i = k + 1; i < n; i++) A[n * i + k] = 0;
    R_diag[k] = beta;
    if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
  }
  rank = 0;
  for (int k = 0; k < n; k++) if (fabs(R_diag[k]) > maxpivot * thresh) rank++;
  double y[6] = {0, 0, 0, 0, 0, 0};
  for (int i = rank - 1; i >= 0; i--) {
    double s = b[i];
    for (int j = i + 1; j < rank; j++) s -= A[n * i + j] * y[j];
    y[i] = s / A[n * i + i];
  }
  for (int j = 0; j < n; j++) x[perm[j]] = (j < rank) ? y[j] : 0.0;
}

/* 6x6 inverse by partial-pivot Gauss-Jordan (Eigen Matrix6d::inverse() is PartialPivLU based). */
int orc_inverse6(const double* Ain, double* Ainv) {
  const int n = 6;
  double A[36], I[36];
  memcpy(A, Ain, sizeof A);
  for (int i = 0; i < 36; i++) I[i] = (i % 7 == 0) ? 1.0 : 0.0;
  int ok = 1;
  for (int k = 0; k < n; k++) {
    int p = k;
    for (int i = k + 1; i < n; i++) if (fabs(A[n * i + k]) > fabs(A[n * p + k])) p = i;
    if (p != k)
      for (int j = 0; j < n; j++) {
        double t = A[n * k + j]; A[n * k + j] = A[n * p + j]; A[n * p + j] = t;
        t = I[n * k + j]; I[n * k + j] = I[n * p + j]; I[n * p + j] = t;
      }
    double d = A[n * k + k];
    if (d == 0) ok = 0;
    double id = 1.0 / d;
    for (int j = 0; j < n; j++) { A[n * k + j] *= id; I[n * k + j] *= id; }
    for (int i = 0; i < n; i++) {
      if (i == k) continue;
      double f = A[n * i + k];
      if (f == 0) continue;
      for (int j = 0; j < n; j++) { A[n * i + j] -= f * A[n * k + j]; I[n * i + j] -= f * I[n * k + j]; }
    }
  }
  memcpy(Ainv, I, sizeof I);
  return ok;
}

/* ---- residuals / Jacobians ---------------------------------------------------------------------- */
static inline double robustWeightCauchy(double r) { return 1.0 / (1.0 + r * r); }

static inline void transform(const double* T, const double* P, double* Q) {
  for (int i = 0; i < 3; i++) Q[i] = T[4 * i] * P[0] + T[4 * i + 1] * P[1] + T[4 * i + 2] * P[2] + T[4 * i + 3];
}
static inline void project(const orc_camera* c, const double* P, double* p) {
  p[0] = c->cx + c->fx * P[0] / P[2];
  p[1] = c->cy + c->fy * P[1] / P[2];
}
static inline double dmax(double a, double b) { return a > b ? a : b; }

static void jac6(double fgz2, double gx, double gy, double gz, double ax, double ay, double* J) {
  J[0] = +fgz2 * ax * gz;
  J[1] = +fgz2 * ay * gz;
  J[2] = -fgz2 * (gx * ax + gy * ay);
  J[3] = -fgz2 * (gx * gy * ax + gy * gy * ay + gz * gz * ay);
  J[4] = +fgz2 * (gx * gx * ax + gz * gz * ax + gx * gy * ay);
  J[5] = +fgz2 * (gx * gz * ay - gy * gz * ax);
}

static double point_residual(const orc_camera* cam, const double* T, const double* P, const double* obs, double* e2,
                             double* Pc) {
  double p[2];
  transform(T, P, Pc);
  project(cam, Pc, p);
  e2[0] = p[0] - obs[0];
  e2[1] = p[1] - obs[1];
  return sqrt(e2[0] * e2[0] + e2[1] * e2[1]);
}
static double line_residual(const orc_camera* cam, const double* T, const double* sP, const double* eP, const double* l,
                            double* e2, double* sPc, double* ePc) {
  double sp[2], ep[2];
  transform(T, sP, sPc);
  project(cam, sPc, sp);
  transform(T, eP, ePc);
  project(cam, ePc, ep);
  e2[0] = l[0] * sp[0] + l[1] * sp[1] + l[2];
  e2[1] = l[0] * ep[0] + l[1] * ep[1] + l[2];
  return sqrt(e2[0] * e2[0] + e2[1] * e2[1]);
}

/* One optimizeFunctions pass (:3326-3432): H (6x6 row-major), g, e (normalised), returns N. */
static int gn_accumulate(const orc_camera* cam, double homog_th, const double* T, const double* P, const double* obs,
                         const uint8_t* inl_p, int np, const double* sP, const double* eP, const double* le,
                         const uint8_t* inl_l, int nl, double* H, double* g, double* e_out) {
  double Hp[36] = {0}, Hl[36] = {0}, gp[6] = {0}, gl[6] = {0}, e_p = 0, e_l = 0;
  int N_p = 0, N_l = 0;
  for (int i = 0; i < np; i++) {
    if (!inl_p[i]) continue;
    double e2[2], Pc[3], J[6];
    double r = point_residual(cam, T, P + 3 * i, obs + 2 * i, e2, Pc);
    double gz2 = Pc[2] * Pc[2];
    double fgz2 = cam->fx / dmax(homog_th, gz2);
    jac6(fgz2, Pc[0], Pc[1], Pc[2], e2[0], e2[1], J);
    double d = dmax(homog_th, r);
    for (int k = 0; k < 6; k++) J[k] = J[k] / d;
    double w = robustWeightCauchy(r);
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < 6; b++) Hp[6 * a + b] += J[a] * J[b] * w;
    for (int a = 0; a < 6; a++) gp[a] += J[a] * r * w;
    e_p += r * r * w;
    N_p++;
  }
  for (int i = 0; i < nl; i++) {
    if (!inl_l[i]) continue;
    double e2[2], sPc[3], ePc[3], Js[6], Je[6], J[6];
    const double* l = le + 3 * i;
    double r = line_residual(cam, T, sP + 3 * i, eP + 3 * i, l, e2, sPc, ePc);
    double fgz2 = cam->fx / dmax(homog_th, sPc[2] * sPc[2]);
    jac6(fgz2, sPc[0], sPc[1], sPc[2], l[0], l[1], Js);
    fgz2 = cam->fx / dmax(homog_th, ePc[2] * ePc[2]);
    jac6(fgz2, ePc[0], ePc[1], ePc[2], l[0], l[1], Je);
    double d = dmax(homog_th, r);
    for (int k = 0; k < 6; k++) J[k] = (Js[k] * e2[0] + Je[k] * e2[1]) / d;
    double w = robustWeightCauchy(r);
    for (int a = 0; a < 6; a++)
      for (int b = 0; b < 6; b++) Hl[6 * a + b] += J[a] * J[b] * w;
    for (int a = 0; a < 6; a++) gl[a] += J[a] * r * w;
    e_l += r * r * w;
    N_l++;
  }
  for (int i = 0; i < 36; i++) H[i] = Hp[i] + Hl[i];
  for (int i = 0; i < 6; i++) g[i] = gp[i] + gl[i];
  *e_out = (e_p + e_l) / (N_l + N_p);
  return N_l + N_p;
}

static void trace_put(orc_gn_trace* tr, const orc_gn_trace_rec* r) {
  if (tr->n < tr->cap) tr->rec[tr->n] = *r;
  tr->n++;
}

/* One stage.  tr (may be NULL) receives one record per accumulation and the stage's exit reason. */
static int gn_stage(const orc_camera* cam, const orc_gn_opts* o, int max_iters, double* T, const double* P,
                    const double* obs, const uint8_t* inl_p, int np, const double* sP, const double* eP,
                    const double* le, const uint8_t* inl_l, int nl, double* H, double* g, double* e, double* err_prev,
                    int stage, orc_gn_trace* tr) {
  int it = 0, why = ORC_GN_EXIT_MAXIT;
  for (; it < max_iters; it++) {
    gn_accumulate(cam, o->homog_th, T, P, obs, inl_p, np, sP, eP, le, inl_l, nl, H, g, e);
    orc_gn_trace_rec rec = {stage, ORC_GN_CONTINUE, *e, *err_prev, -1.0};
    if (fabs(*e - *err_prev) < o->eps_change || *e < o->eps_err) {
      why = rec.exit = ORC_GN_EXIT_ERROR;
      if (tr) trace_put(tr, &rec);
      break;
    }
    double dx[6], E[16], Ei[16];
    orc_colpiv_qr_solve6(H, g, dx);
    orc_expmap_se3(dx, E);
    orc_inverse_se3(E, Ei);
    mat4_mul(T, Ei, T);
    double nrm = 0;
    for (int k = 0; k < 6; k++) nrm += dx[k] * dx[k];
    rec.step = sqrt(nrm);
    if (sqrt(nrm) < o->eps_step) {
      why = rec.exit = ORC_GN_EXIT_STEP;
      if (tr) trace_put(tr, &rec);
      it++;
      break;
    }
    if (it + 1 == max_iters) rec.exit = ORC_GN_EXIT_MAXIT;
    if (tr) trace_put(tr, &rec);
    *err_prev = *e;
  }
  if (tr) tr->stage_exit[stage] = why;
  return it;
}

/* Two-stage robust GN (:3566-3957).  T_init/T_out row-major 4x4.  inl_* are updated in place. */
static void gn_pose(const orc_camera* cam, const orc_gn_opts* o, const double* P, const double* obs, uint8_t* inl_p,
                    int np, const double* sP, const double* eP, const double* le, uint8_t* inl_l, int nl,
                    const double* T_init, orc_pose_result* out, orc_gn_trace* tr) {
  double T[16], H[36] = {0}, g[6] = {0}, e = 0, err_prev = 999999999.9;
  memcpy(T, T_init, sizeof T);
  out->iters1 = gn_stage(cam, o, o->max_iters, T, P, obs, inl_p, np, sP, eP, le, inl_l, nl, H, g, &e, &err_prev, 0, tr);
  const double gate = sqrt(7.815);
  for (int i = 0; i < np; i++) {
    if (!inl_p[i]) continue;
    double e2[2], Pc[3];
    if (point_residual(cam, T, P + 3 * i, obs + 2 * i, e2, Pc) > gate) inl_p[i] = 0;
  }
  for (int i = 0; i < nl; i++) {
    if (!inl_l[i]) continue;
    double e2[2], a[3], b[3];
    if (line_residual(cam, T, sP + 3 * i, eP + 3 * i, le + 3 * i, e2, a, b) > gate) inl_l[i] = 0;
  }
  out->iters2 = gn_stage(cam, o, o->max_iters_ref, T, P, obs, inl_p, np, sP, eP, le, inl_l, nl, H, g, &e, &err_prev, 1, tr);
  memcpy(out->T, T, sizeof T);
  orc_logmap_se3(T, out->x);
  out->err = e;
  orc_inverse6(H, out->cov);
  int a = 0, b = 0;
  for (int i = 0; i < np; i++) a += inl_p[i] != 0;
  for (int i = 0; i < nl; i++) b += inl_l[i] != 0;
  out->n_inliers_pt = a;
  out->n_inliers_ls = b;
}

void orc_gn_pose(const orc_camera* cam, const orc_gn_opts* o, const double* P, const double* obs, uint8_t* inl_p,
                 int np, const double* sP, const double* eP, const double* le, uint8_t* inl_l, int nl,
                 const double* T_init, orc_pose_result* out) {
  gn_pose(cam, o, P, obs, inl_p, np, sP, eP, le, inl_l, nl, T_init, out, NULL);
}

/* orc_gn_pose plus the stop-decision trace: what each stop test saw, so that a caller comparing iteration counts
 * with a solver that sums in another order can tell whether a test sat on its threshold. */
void orc_gn_pose_trace(const orc_camera* cam, const orc_gn_opts* o, const double* P, const double* obs, uint8_t* inl_p,
                       int np, const double* sP, const double* eP, const double* le, uint8_t* inl_l, int nl,
                       const double* T_init, orc_pose_result* out, orc_gn_trace* tr) {
  tr->n = 0;
  gn_pose(cam, o, P, obs, inl_p, np, sP, eP, le, inl_l, nl, T_init, out, tr);
}
