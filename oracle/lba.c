/*
 * oracle/lba.c — CPU restatement of PL-SLAM's local bundle adjustment (SURVEY.md section 8(f) row f4).
 * TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * Follows MapHandler::levMarquardtOptimizationLBA, src/mapHandler.cpp:1332-1989 (called from
 * MapHandler::localBundleAdjustment :1220-1330 with X = [x_kf_w of the local keyframes | point3D of the local points |
 * line3D of the local lines] and one Vector6i per observation):
 *   first pass on the map's values :1352-1541, lambda *= max |H_ii| :1543-1550, H_ii += lambda H_ii and
 *   SimplicialLDLT solve :1552-1556, update T = expmap(X) * inverse(expmap(DX)) / X += DX :1558-1570,
 *   LM iterations :1577-1797 (point rows :1587-1666, line rows :1668-1771, normalise :1773, stop tests :1775,:1805,
 *   lambda schedule :1785-1803), landmark "moved more than 0.01" flags :1826-1851.
 * Point row: Jacobians :1384-1400, weight robustWeightCauchy :1402-1403, accumulation :1406-1425.
 * Line row: :1441-1534.
 *
 * Things the reference does that look unintended, and what happens here (opts.ref_quirks = 1 reproduces them, 0 = the
 * evident intent):
 *   (q1) :1541 `err /= (Npt_obs + Nls_obs)` divides by two counters that are never incremented (0): err_prev becomes
 *        +inf (or NaN for a zero error).  With ref_quirks = 0 the divisor is the number of observations.
 *   (q2) :1678-1679 in the LM iterations both end points of a line landmark are read from the SAME block of X, at stride
 *        3 (`6*Nkf+3*Npt+3*lm_idx_loc`), instead of head / tail of the landmark's own 6 values at stride 6.
 *   (q3) :1681 in the LM iterations the line rows take the observing keyframe's pose from the MAP (the pose before this
 *        optimisation) even when the keyframe is being optimised; the point rows use X (:1600-1603).
 *   (q4) :1716,:1723 etc. the line rows of the LM iterations clamp with the literal 0.0000001 instead of
 *        SlamConfig::homogTh() (identical for the default homog_th).
 * The lambda schedule (:1785-1790: divide by lambda_k when the error grew - without applying the step - multiply
 * otherwise) and the normalisation by the number of landmarks (:1773) are kept as written in both modes.
 * SimplicialLDLT (AMD-ordered sparse LDL^T) is restated as a dense LDL^T without pivoting.
 * A landmark whose first-pass block has an exactly zero diagonal entry (no observation, or every row with a zero
 * Jacobian: a single observation at its exact projection) would make the reference factor a zero pivot, whose failure
 * it does not check; here, as on the device, the problem is refused (ORC_LBA_ZERO_BLOCK) before any step.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

static inline double cauchy(double r) { return 1.0 / (1.0 + r * r); }
static inline double dmax2(double a, double b) { return a > b ? a : b; }

static void jac_pose(double gz2, double fxdx, double fydy, double gx, double gy, double gz, double* J) {
  J[0] = +gz2 * fxdx * gz;
  J[1] = +gz2 * fydy * gz;
  J[2] = -gz2 * (fxdx * gx + fydy * gy);
  J[3] = -gz2 * (fxdx * gx * gy + fydy * gy * gy + fydy * gz * gz);
  J[4] = +gz2 * (fxdx * gx * gx + fxdx * gz * gz + fydy * gx * gy);
  J[5] = +gz2 * (fydy * gx * gz - fxdx * gy * gz);
}

/* row vector (3) times the rotation block of the row-major 4x4 T: out_j = sum_i v_i R_ij */
static void rowvec_times_R(const double* v, const double* T, double* out) {
  for (int j = 0; j < 3; j++) out[j] = v[0] * T[j] + v[1] * T[4 + j] + v[2] * T[8 + j];
}

typedef struct {
  const orc_camera* cam;
  int nkf, npt, nls, N;
  double* H; /* N x N row-major */
  double* g;
  double err;
} acc_t;

static void add_point_row(acc_t* a, double homog, const double* Tiw_inv, const double* Xwj, const double* obs, int kf_loc, int lm_loc) {
  const orc_camera* c = a->cam;
  double Xwi[3];
  for (int i = 0; i < 3; i++) Xwi[i] = Tiw_inv[4 * i] * Xwj[0] + Tiw_inv[4 * i + 1] * Xwj[1] + Tiw_inv[4 * i + 2] * Xwj[2] + Tiw_inv[4 * i + 3];
  const double px = c->cx + c->fx * Xwi[0] / Xwi[2], py = c->cy + c->fy * Xwi[1] / Xwi[2];
  const double dx = obs[0] - px, dy = obs[1] - py;
  const double nrm = sqrt(dx * dx + dy * dy);
  const double gx = Xwi[0], gy = Xwi[1], gz = Xwi[2];
  const double gz2 = 1.0 / dmax2(homog, gz * gz);
  const double fxdx = c->fx * dx, fydy = c->fy * dy;
  double JT[6], J3[3], JX[3];
  jac_pose(gz2, fxdx, fydy, gx, gy, gz, JT);
  const double den = dmax2(homog, nrm);
  for (int i = 0; i < 6; i++) JT[i] = JT[i] / den;
  J3[0] = +gz2 * fxdx * gz; J3[1] = +gz2 * fydy * gz; J3[2] = -gz2 * (fxdx * gx + fydy * gy);
  rowvec_times_R(J3, Tiw_inv, JX);
  for (int i = 0; i < 3; i++) JX[i] = JX[i] / den;
  const double w = cauchy(nrm);
  const int N = a->N, idx = 6 * kf_loc, jdx = 6 * a->nkf + 3 * lm_loc;
  if (kf_loc >= 0) {
    for (int i = 0; i < 6; i++) a->g[idx + i] += JT[i] * nrm * w;
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) a->H[(size_t)(idx + i) * N + idx + j] += JT[i] * JT[j] * w;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 6; j++) {
        const double h = JX[i] * JT[j] * w;
        a->H[(size_t)(jdx + i) * N + idx + j] += h;
        a->H[(size_t)(idx + j) * N + jdx + i] += h;
      }
  }
  for (int i = 0; i < 3; i++) a->g[jdx + i] += JX[i] * nrm * w;
  a->err += nrm * nrm * w;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) a->H[(size_t)(jdx + i) * N + jdx + j] += JX[i] * JX[j] * w;
}

static void add_line_row(acc_t* a, double homog, const double* Tiw_inv, const double* Pwj, const double* Qwj, const double* l, int kf_loc, int lm_loc) {
  const orc_camera* c = a->cam;
  double Pwi[3], Qwi[3];
  for (int i = 0; i < 3; i++) {
    Pwi[i] = Tiw_inv[4 * i] * Pwj[0] + Tiw_inv[4 * i + 1] * Pwj[1] + Tiw_inv[4 * i + 2] * Pwj[2] + Tiw_inv[4 * i + 3];
    Qwi[i] = Tiw_inv[4 * i] * Qwj[0] + Tiw_inv[4 * i + 1] * Qwj[1] + Tiw_inv[4 * i + 2] * Qwj[2] + Tiw_inv[4 * i + 3];
  }
  const double ppx = c->cx + c->fx * Pwi[0] / Pwi[2], ppy = c->cy + c->fy * Pwi[1] / Pwi[2];
  const double qpx = c->cx + c->fx * Qwi[0] / Qwi[2], qpy = c->cy + c->fy * Qwi[1] / Qwi[2];
  const double e0 = l[0] * ppx + l[1] * ppy + l[2], e1 = l[0] * qpx + l[1] * qpy + l[2];
  const double nrm = sqrt(e0 * e0 + e1 * e1);
  /* NOTE (reference, :1470-1471): fxlx = fx * l_err(0), fyly = fy * l_err(1) - the two residuals, not the line's normal */
  const double fxlx = c->fx * e0, fyly = c->fy * e1;
  const double den = dmax2(homog, nrm);
  double JP[6], JQ[6], J3[3], JPw[3], JQw[3], JT[6], JL[6];
  {
    const double gx = Pwi[0], gy = Pwi[1], gz = Pwi[2], gz2 = 1.0 / dmax2(homog, gz * gz);
    jac_pose(gz2, fxlx, fyly, gx, gy, gz, JP);
    J3[0] = +gz2 * fxlx * gz; J3[1] = +gz2 * fyly * gz; J3[2] = -gz2 * (fxlx * gx + fyly * gy);
    rowvec_times_R(J3, Tiw_inv, JPw);
    for (int i = 0; i < 3; i++) JPw[i] = JPw[i] * e0 / den;
  }
  {
    const double gx = Qwi[0], gy = Qwi[1], gz = Qwi[2], gz2 = 1.0 / dmax2(homog, gz * gz);
    jac_pose(gz2, fxlx, fyly, gx, gy, gz, JQ);
    J3[0] = +gz2 * fxlx * gz; J3[1] = +gz2 * fyly * gz; J3[2] = -gz2 * (fxlx * gx + fyly * gy);
    rowvec_times_R(J3, Tiw_inv, JQw);
    for (int i = 0; i < 3; i++) JQw[i] = JQw[i] * e1 / den;
  }
  for (int i = 0; i < 6; i++) JT[i] = (JP[i] * e0 + JQ[i] * e1) / den;
  for (int i = 0; i < 3; i++) { JL[i] = JPw[i]; JL[3 + i] = JQw[i]; }
  const double w = cauchy(nrm);
  const int N = a->N, idx = 6 * kf_loc, jdx = 6 * a->nkf + 3 * a->npt + 6 * lm_loc;
  if (kf_loc >= 0) {
    for (int i = 0; i < 6; i++) a->g[idx + i] += JT[i] * nrm * w;
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) a->H[(size_t)(idx + i) * N + idx + j] += JT[i] * JT[j] * w;
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) {
        const double h = JL[i] * JT[j] * w;
        a->H[(size_t)(jdx + i) * N + idx + j] += h;
        a->H[(size_t)(idx + j) * N + jdx + i] += h;
      }
  }
  for (int i = 0; i < 6; i++) a->g[jdx + i] += JL[i] * nrm * w;
  a->err += nrm * nrm * w;
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) a->H[(size_t)(jdx + i) * N + jdx + j] += JL[i] * JL[j] * w;
}

/* dense LDL^T without pivoting, in place on the lower triangle; solves H x = g */
static void ldlt_solve(double* H, const double* g, double* x, int N) {
  for (int j = 0; j < N; j++) {
    double d = H[(size_t)j * N + j];
    for (int k = 0; k < j; k++) d -= H[(size_t)j * N + k] * H[(size_t)j * N + k] * H[(size_t)k * N + k];
    H[(size_t)j * N + j] = d;
    for (int i = j + 1; i < N; i++) {
      double v = H[(size_t)i * N + j];
      for (int k = 0; k < j; k++) v -= H[(size_t)i * N + k] * H[(size_t)j * N + k] * H[(size_t)k * N + k];
      H[(size_t)i * N + j] = v / d;
    }
  }
  for (int i = 0; i < N; i++) {
    double v = g[i];
    for (int k = 0; k < i; k++) v -= H[(size_t)i * N + k] * x[k];
    x[i] = v;
  }
  for (int i = 0; i < N; i++) x[i] /= H[(size_t)i * N + i];
  for (int i = N - 1; i >= 0; i--) {
    double v = x[i];
    for (int k = i + 1; k < N; k++) v -= H[(size_t)k * N + i] * x[k];
    x[i] = v;
  }
}

static void apply_step(double* X, const double* DX, int nkf, int N) {
  for (int i = 0; i < nkf; i++) {
    double Tp[16], E[16], Ei[16], Tc[16];
    orc_expmap_se3(X + 6 * i, Tp);
    orc_expmap_se3(DX + 6 * i, E);
    orc_inverse_se3(E, Ei);
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) {
        double a = 0;
        for (int k = 0; k < 4; k++) a += Tp[4 * r + k] * Ei[4 * k + c];
        Tc[4 * r + c] = a;
      }
    orc_logmap_se3(Tc, X + 6 * i);
  }
  for (int i = 6 * nkf; i < N; i++) X[i] += DX[i];
}

static void trace_rec(orc_lba_trace* tr, double err, double lambda, double step, int applied, int stop) {
  if (!tr) return;
  if (tr->n < tr->cap) {
    orc_lba_trace_rec* r = tr->rec + tr->n;
    r->err = err; r->lambda = lambda; r->step = step; r->applied = applied; r->stop = stop;
  }
  tr->n++;
}

/* kf index of an observation: >= 0 local keyframe (pose = X block), < 0 fixed keyframe -1 - k (pose fixed_T[k]) */
int orc_local_ba(const orc_camera* cam, const orc_lba_opts* o, int nkf, int npt, int nls, double* X, int n_fixed,
                 const double* fixed_T, int npo, const int* po_lm, const int* po_kf, const double* po_xy, int nlo,
                 const int* lo_lm, const int* lo_kf, const double* lo_le, uint8_t* pt_moved, uint8_t* ls_moved,
                 orc_lba_result* out) {
  return orc_local_ba_trace(cam, o, nkf, npt, nls, X, n_fixed, fixed_T, npo, po_lm, po_kf, po_xy, nlo, lo_lm, lo_kf, lo_le,
                            pt_moved, ls_moved, out, NULL);
}

int orc_local_ba_trace(const orc_camera* cam, const orc_lba_opts* o, int nkf, int npt, int nls, double* X, int n_fixed,
                       const double* fixed_T, int npo, const int* po_lm, const int* po_kf, const double* po_xy, int nlo,
                       const int* lo_lm, const int* lo_kf, const double* lo_le, uint8_t* pt_moved, uint8_t* ls_moved,
                       orc_lba_result* out, orc_lba_trace* tr) {
  const int N = 6 * nkf + 3 * npt + 6 * nls;
  (void)n_fixed;
  if (out) out->zero_lm = -1;
  if (tr) tr->n = 0;
  if (N <= 0 || npo + nlo == 0) return -1;
  double* H = (double*)malloc((size_t)N * N * sizeof(double));
  double* g = (double*)malloc((size_t)N * sizeof(double));
  double* DX = (double*)malloc((size_t)N * sizeof(double));
  double* X0 = (double*)malloc((size_t)N * sizeof(double));
  double* T0inv = (double*)malloc((size_t)(nkf > 0 ? nkf : 1) * 16 * sizeof(double)); /* inverse of the MAP pose of the local keyframes */
  memcpy(X0, X, (size_t)N * sizeof(double));
  for (int i = 0; i < nkf; i++) {
    double T[16];
    orc_expmap_se3(X0 + 6 * i, T);
    orc_inverse_se3(T, T0inv + 16 * i);
  }
  acc_t a = {cam, nkf, npt, nls, N, H, g, 0.0};
  double lambda = o->lambda;
  const double lambda_k = o->lambda_k;
  /* ---- first pass on the map's values ---- */
  memset(H, 0, (size_t)N * N * sizeof(double));
  memset(g, 0, (size_t)N * sizeof(double));
  for (int k = 0; k < npo; k++) {
    double Ti[16];
    if (po_kf[k] >= 0) memcpy(Ti, T0inv + 16 * po_kf[k], sizeof Ti);
    else orc_inverse_se3(fixed_T + 16 * (-1 - po_kf[k]), Ti);
    add_point_row(&a, o->homog_th, Ti, X0 + 6 * nkf + 3 * po_lm[k], po_xy + 2 * k, po_kf[k] >= 0 ? po_kf[k] : -1, po_lm[k]);
  }
  for (int k = 0; k < nlo; k++) {
    double Ti[16];
    if (lo_kf[k] >= 0) memcpy(Ti, T0inv + 16 * lo_kf[k], sizeof Ti);
    else orc_inverse_se3(fixed_T + 16 * (-1 - lo_kf[k]), Ti);
    const double* L = X0 + 6 * nkf + 3 * npt + 6 * lo_lm[k];
    add_line_row(&a, o->homog_th, Ti, L, L + 3, lo_le + 3 * k, lo_kf[k] >= 0 ? lo_kf[k] : -1, lo_lm[k]);
  }
  /* a zero diagonal entry in a landmark's block: refused before any step (see the header) */
  for (int l = 0; l < npt + nls; l++) {
    const int off = l < npt ? 6 * nkf + 3 * l : 6 * nkf + 3 * npt + 6 * (l - npt), dim = l < npt ? 3 : 6;
    for (int i = 0; i < dim; i++)
      if (H[(size_t)(off + i) * N + off + i] == 0.0) {
        if (out) out->zero_lm = l;
        free(H); free(g); free(DX); free(X0); free(T0inv);
        return ORC_LBA_ZERO_BLOCK;
      }
  }
  double err = a.err;
  if (o->ref_quirks) err /= (double)(0 + 0); /* (q1) */
  else err /= (double)(npo + nlo);
  double Hmax = 0.0;
  for (int i = 0; i < N; i++) {
    const double d = H[(size_t)i * N + i];
    if (d > Hmax || d < -Hmax) Hmax = fabs(d);
  }
  lambda *= Hmax;
  for (int i = 0; i < N; i++) H[(size_t)i * N + i] += lambda * H[(size_t)i * N + i];
  ldlt_solve(H, g, DX, N);
  apply_step(X, DX, nkf, N);
  {
    double n2 = 0;
    for (int i = 0; i < N; i++) n2 += DX[i] * DX[i];
    trace_rec(tr, err, lambda, sqrt(n2), 1, ORC_LBA_CONTINUE);
  }
  int stop = ORC_LBA_STOP_MAXIT;
  double err_prev = err;
  /* ---- LM iterations ---- */
  int iters;
  for (iters = 1; iters < o->max_iters; iters++) {
    memset(H, 0, (size_t)N * N * sizeof(double));
    memset(g, 0, (size_t)N * sizeof(double));
    a.err = 0.0;
    for (int k = 0; k < npo; k++) {
      double T[16], Ti[16];
      if (po_kf[k] >= 0) { orc_expmap_se3(X + 6 * po_kf[k], T); orc_inverse_se3(T, Ti); }
      else orc_inverse_se3(fixed_T + 16 * (-1 - po_kf[k]), Ti);
      add_point_row(&a, o->homog_th, Ti, X + 6 * nkf + 3 * po_lm[k], po_xy + 2 * k, po_kf[k] >= 0 ? po_kf[k] : -1, po_lm[k]);
    }
    for (int k = 0; k < nlo; k++) {
      double T[16], Ti[16];
      const double *P, *Q;
      if (o->ref_quirks) {
        if (lo_kf[k] >= 0) memcpy(Ti, T0inv + 16 * lo_kf[k], sizeof Ti);   /* (q3) the map's pose */
        else orc_inverse_se3(fixed_T + 16 * (-1 - lo_kf[k]), Ti);
        P = Q = X + 6 * nkf + 3 * npt + 3 * lo_lm[k];                        /* (q2) */
      } else {
        if (lo_kf[k] >= 0) { orc_expmap_se3(X + 6 * lo_kf[k], T); orc_inverse_se3(T, Ti); }
        else orc_inverse_se3(fixed_T + 16 * (-1 - lo_kf[k]), Ti);
        P = X + 6 * nkf + 3 * npt + 6 * lo_lm[k];
        Q = P + 3;
      }
      add_line_row(&a, o->ref_quirks ? 0.0000001 : o->homog_th /* (q4) */, Ti, P, Q, lo_le + 3 * k, lo_kf[k] >= 0 ? lo_kf[k] : -1, lo_lm[k]);
    }
    err = a.err / (double)(npt + nls);
    if (fabs(err - err_prev) < o->min_error_change || err < o->min_error) {
      stop = fabs(err - err_prev) < o->min_error_change ? ORC_LBA_STOP_CHANGE : ORC_LBA_STOP_MIN_ERROR;
      trace_rec(tr, err, lambda, -1.0, 0, stop);
      break;
    }
    for (int i = 0; i < N; i++) H[(size_t)i * N + i] += lambda * H[(size_t)i * N + i];
    ldlt_solve(H, g, DX, N);
    const double lambda_used = lambda;
    const int grew = err > err_prev;
    if (grew) {
      lambda /= lambda_k;
    } else {
      lambda *= lambda_k;
      apply_step(X, DX, nkf, N);
    }
    double n2 = 0;
    for (int i = 0; i < N; i++) n2 += DX[i] * DX[i];
    const int small = sqrt(n2) < o->min_error_change;
    trace_rec(tr, err, lambda_used, sqrt(n2), !grew, small ? ORC_LBA_STOP_STEP : ORC_LBA_CONTINUE);
    if (small) {
      stop = ORC_LBA_STOP_STEP;
      break;
    }
    err_prev = err;
  }
  /* the loop counter ran out: the last pass made ends the run */
  if (tr && stop == ORC_LBA_STOP_MAXIT && tr->n >= 1 && tr->n <= tr->cap) tr->rec[tr->n - 1].stop = ORC_LBA_STOP_MAXIT;
  /* landmarks that moved more than 1 cm lose their inlier flag (:1826-1851) */
  for (int i = 0; i < npt; i++) {
    double n2 = 0;
    for (int c = 0; c < 3; c++) { const double d = X[6 * nkf + 3 * i + c] - X0[6 * nkf + 3 * i + c]; n2 += d * d; }
    if (pt_moved) pt_moved[i] = sqrt(n2) > 0.01;
  }
  for (int i = 0; i < nls; i++) {
    double n2 = 0;
    for (int c = 0; c < 6; c++) { const double d = X[6 * nkf + 3 * npt + 6 * i + c] - X0[6 * nkf + 3 * npt + 6 * i + c]; n2 += d * d; }
    if (ls_moved) ls_moved[i] = sqrt(n2) > 0.01;
  }
  if (out) { out->iters = iters; out->err = err; out->lambda = lambda; }
  free(H); free(g); free(DX); free(X0); free(T0inv);
  return 0;
}
