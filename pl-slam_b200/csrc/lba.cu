// Local bundle adjustment on the GPU (SURVEY §8(f) row f4).
//
// Replaces MapHandler::levMarquardtOptimizationLBA (src/mapHandler.cpp:1332-1989), the numerical core of
// MapHandler::localBundleAdjustment (:1220-1330): Levenberg-Marquardt over the local keyframes' poses (x_kf_w, se(3)
// vectors), the local 3-D points and the local 3-D line segments (two end points), with Cauchy-weighted scalar residuals
// (the norm of the point reprojection error / of the two end-point distances to the observed line).  The reference
// rebuilds a DENSE N x N Hessian every iteration and factors its sparse view with SimplicialLDLT; here the same normal
// equations are solved through the Schur complement on the landmarks - every observation couples ONE keyframe with ONE
// landmark, so the landmark block is block-diagonal (3x3 / 6x6) and each coupling block is rank one.  Each step is a
// __device__ function of one problem's element, run on every problem of a call by the k_lbb_* kernels below:
//   lba_rows        one thread per observation: residual, weight, the two Jacobian rows (:1384-1400 points, :1441-1503
//                   lines); accumulates the keyframe blocks A (6x6) / g_c and the error
//   lba_lm_accum    one thread per landmark: D = sum w Jx Jx^T, g_l (its observations are contiguous, in the reference's
//                   order), max |diagonal| for the initial lambda (:1543-1550)
//   lba_lm_schur    one thread per landmark: D' = D + lambda diag(D), D'^-1, and the reduced-system contributions
//                   S[a][b] -= w_b (y_a . Jx_b) Jt_a Jt_b^T, g_red[a] -= (y_a . g_l) Jt_a with y_a = w_a D'^-1 Jx_a
//   lba_solve       one CTA: S += A', dense LDL^T (no pivoting, as SimplicialLDLT) and the two triangular solves
//   lba_backsub     one thread per landmark: dx_l = D'^-1 (g_l - sum_a w_a Jx_a (Jt_a . dx_c[a]))
//   lba_apply       T <- T * inverse_se3(expmap_se3(dx)) / X += dx (:1558-1570), |dx|^2
// The reference's control flow (first pass on the map's values, lambda schedule :1785-1803, stop tests :1775,:1805)
// runs on the device too, one thread per problem (k_lbb_first / k_lbb_test / k_lbb_step), so plf_local_ba is
// plf_local_ba_batch's driver with one problem.  opts.ref_quirks selects between the reference as written and its
// evident intent for the four oddities documented in oracle/lba.c (division by the zero counters :1541, both line end
// points read from one block of X at stride 3 :1678-1679, the map's pose for line rows :1681, the literal clamp);
// oracle = oracle/lba.c.
//
// Global bundle adjustment (SURVEY §8(f), after f1-f5): plf_global_ba replaces MapHandler::levMarquardtOptimizationGBA
// (:2101-2699) with the same device functions and driver over every keyframe but keyframe 0 and every landmark.  Its
// quirk set (g1-g6, oracle/gba.py) selects the reference's GBA oddities instead of LBA's, and a reduced system larger
// than 384 (more than 64 keyframes) is factored by the tiled, multi-CTA LDL^T below (gba_*, run by k_gbb_*), whose
// trailing update runs on the FP64 tensor cores (DMMA) and skips the tiles of the panel that are exactly zero.
#include "plf_internal.h"
#include "plf_se3.cuh"

// Which of the reference's oddities the kernels and the host loop reproduce: plf_local_ba's ref_quirks selects q1-q4
// (oracle/lba.c), plf_global_ba's g1-g6 (oracle/gba.py).  0 = the evident intent of both.
enum : int {
  BAQ_FIRST_ERR0 = 1,      // q1 / g1: the first pass divides the error by two counters never incremented
  BAQ_LINE_STRIDE3 = 2,    // q2 / g4: LM line rows read both end points from one block of X at stride 3
  BAQ_LINE_MAP_POSE = 4,   // q3 / g5: LM line rows take the map's pose
  BAQ_LINE_LITERAL = 8,    // q4: LM line rows clamp with the literal 0.0000001
  BAQ_ITER_ERR0 = 16,      // g3: the LM iterations divide the error by the zero counters too
  BAQ_HMAX_INT = 32,       // g2: the first lambda multiplies by the diagonal maximum truncated to int
  BAQ_SWAP_COUPLING = 64,  // g6: the first pass writes the line/keyframe coupling as w Jt Jx^T (landmark row x pose column)
};
constexpr int BAQ_LBA = BAQ_FIRST_ERR0 | BAQ_LINE_STRIDE3 | BAQ_LINE_MAP_POSE | BAQ_LINE_LITERAL;
constexpr int BAQ_GBA = BAQ_FIRST_ERR0 | BAQ_LINE_STRIDE3 | BAQ_LINE_MAP_POSE | BAQ_ITER_ERR0 | BAQ_HMAX_INT | BAQ_SWAP_COUPLING;

struct LbaDev {
  int nkf, npt, nls, N, npo, nlo, nobs, nlm;
  double* X; double* X0; double* T0inv;       // N, N, nkf x 16 (inverse of the map pose of the local keyframes)
  const double* fixedTinv;                     // n_fixed x 16
  const int* obs_lm; const int* obs_kf;        // nobs (points first, then lines)
  const double* obs_z;                         // nobs x 3 (points: x, y, -; lines: the observed line equation)
  const int* lm_start;                         // nlm + 1 (points then lines): first observation of each landmark
  double* Jt; double* Jx; double* Wn;          // nobs x 6, nobs x 6, nobs x 2 {w, r w}
  double* D; double* gl; double* Dinv;         // nlm x 36, nlm x 6, nlm x 36
  double* A; double* gc;                       // nkf x 36, nkf x 6
  double* S; double* gred; double* dxc;        // n x n, n, n   (n = 6 nkf)
  double* DX;                                  // N
  double* scal;                                // [0] err, [1] |dx|^2, [2] Hmax (as ordered bits), [3] Hmax under g2,
                                               // [4] first landmark with a zero diagonal entry in D (lba_lm_accum)
};
struct LbaCam { double fx, fy, cx, cy; };

__device__ __forceinline__ void lba_jac_pose(double gz2, double fxdx, double fydy, double gx, double gy, double gz, double* J) {
  J[0] = +gz2 * fxdx * gz;
  J[1] = +gz2 * fydy * gz;
  J[2] = -gz2 * (fxdx * gx + fydy * gy);
  J[3] = -gz2 * (fxdx * gx * gy + fydy * gy * gy + fydy * gz * gz);
  J[4] = +gz2 * (fxdx * gx * gx + fxdx * gz * gz + fydy * gx * gy);
  J[5] = +gz2 * (fydy * gx * gz - fxdx * gy * gz);
}
__device__ __forceinline__ void lba_rowvec_R(const double* v, const double* T, double* out) {
  for (int j = 0; j < 3; ++j) out[j] = v[0] * T[j] + v[1] * T[4 + j] + v[2] * T[8 + j];
}

// Each step's work for one element (observation k, landmark l, ...) is a __device__ function of the problem's LbaDev,
// which the k_lbb_* kernels below run on each problem of a call.

// mode 0: first pass on the map's values (X0 / T0inv); mode 1: LM iteration on X; quirks: BAQ_* set.  Every lane of the
// warp calls it (the error is reduced over the warp).
__device__ __forceinline__ void lba_rows(const LbaDev& d, const LbaCam& c, int k, int mode, int quirks, double homog_th) {
  double e2w = 0.0;
  if (k < d.nobs) {
    const bool is_line = k >= d.npo;
    const int lm = d.obs_lm[k], kf = d.obs_kf[k];
    const double* X = mode == 0 ? d.X0 : d.X;
    double Ti[16];
    const bool map_pose = mode == 0 || (is_line && (quirks & BAQ_LINE_MAP_POSE));   // (q3, g5)
    if (kf >= 0) {
      if (map_pose) {
        for (int i = 0; i < 16; ++i) Ti[i] = d.T0inv[16 * kf + i];
      } else {
        double T[16];
        d_expmap(X + 6 * kf, T);
        d_inverse_se3(T, Ti);
      }
    } else {
      for (int i = 0; i < 16; ++i) Ti[i] = d.fixedTinv[16 * (-1 - kf) + i];
    }
    double JT[6] = {0, 0, 0, 0, 0, 0}, JX[6] = {0, 0, 0, 0, 0, 0}, nrm;
    const double* z = d.obs_z + 3 * k;
    if (!is_line) {
      double Xwi[3];
      d_transform(Ti, X + 6 * d.nkf + 3 * lm, Xwi);
      const double px = c.cx + c.fx * Xwi[0] / Xwi[2], py = c.cy + c.fy * Xwi[1] / Xwi[2];
      const double dx = z[0] - px, dy = z[1] - py;
      nrm = sqrt(dx * dx + dy * dy);
      const double gx = Xwi[0], gy = Xwi[1], gz = Xwi[2];
      const double gz2 = 1.0 / fmax(homog_th, gz * gz);
      const double fxdx = c.fx * dx, fydy = c.fy * dy;
      lba_jac_pose(gz2, fxdx, fydy, gx, gy, gz, JT);
      const double den = fmax(homog_th, nrm);
      for (int i = 0; i < 6; ++i) JT[i] = JT[i] / den;
      double J3[3] = {+gz2 * fxdx * gz, +gz2 * fydy * gz, -gz2 * (fxdx * gx + fydy * gy)};
      lba_rowvec_R(J3, Ti, JX);
      for (int i = 0; i < 3; ++i) JX[i] = JX[i] / den;
    } else {
      const double hom = (mode == 1 && (quirks & BAQ_LINE_LITERAL)) ? 0.0000001 : homog_th;   // (q4)
      const double *P, *Q;
      if (mode == 1 && (quirks & BAQ_LINE_STRIDE3)) {
        P = Q = X + 6 * d.nkf + 3 * d.npt + 3 * lm;                      // (q2, g4)
      } else {
        P = X + 6 * d.nkf + 3 * d.npt + 6 * lm;
        Q = P + 3;
      }
      double Pwi[3], Qwi[3];
      d_transform(Ti, P, Pwi);
      d_transform(Ti, Q, Qwi);
      const double ppx = c.cx + c.fx * Pwi[0] / Pwi[2], ppy = c.cy + c.fy * Pwi[1] / Pwi[2];
      const double qpx = c.cx + c.fx * Qwi[0] / Qwi[2], qpy = c.cy + c.fy * Qwi[1] / Qwi[2];
      const double e0 = z[0] * ppx + z[1] * ppy + z[2], e1 = z[0] * qpx + z[1] * qpy + z[2];
      nrm = sqrt(e0 * e0 + e1 * e1);
      const double fxlx = c.fx * e0, fyly = c.fy * e1;   // as the reference writes it (:1470-1471)
      const double den = fmax(hom, nrm);
      double JP[6], JQ[6], J3[3], JPw[3], JQw[3];
      {
        const double gx = Pwi[0], gy = Pwi[1], gz = Pwi[2], gz2 = 1.0 / fmax(hom, gz * gz);
        lba_jac_pose(gz2, fxlx, fyly, gx, gy, gz, JP);
        J3[0] = +gz2 * fxlx * gz; J3[1] = +gz2 * fyly * gz; J3[2] = -gz2 * (fxlx * gx + fyly * gy);
        lba_rowvec_R(J3, Ti, JPw);
        for (int i = 0; i < 3; ++i) JPw[i] = JPw[i] * e0 / den;
      }
      {
        const double gx = Qwi[0], gy = Qwi[1], gz = Qwi[2], gz2 = 1.0 / fmax(hom, gz * gz);
        lba_jac_pose(gz2, fxlx, fyly, gx, gy, gz, JQ);
        J3[0] = +gz2 * fxlx * gz; J3[1] = +gz2 * fyly * gz; J3[2] = -gz2 * (fxlx * gx + fyly * gy);
        lba_rowvec_R(J3, Ti, JQw);
        for (int i = 0; i < 3; ++i) JQw[i] = JQw[i] * e1 / den;
      }
      for (int i = 0; i < 6; ++i) JT[i] = (JP[i] * e0 + JQ[i] * e1) / den;
      for (int i = 0; i < 3; ++i) { JX[i] = JPw[i]; JX[3 + i] = JQw[i]; }
    }
    const double w = 1.0 / (1.0 + nrm * nrm);   // robustWeightCauchy
    for (int i = 0; i < 6; ++i) { d.Jt[6 * (size_t)k + i] = JT[i]; d.Jx[6 * (size_t)k + i] = JX[i]; }
    d.Wn[2 * (size_t)k] = w;
    d.Wn[2 * (size_t)k + 1] = nrm * w;
    e2w = nrm * nrm * w;
    if (kf >= 0) {
      for (int i = 0; i < 6; ++i) {
        atomicAdd(&d.gc[6 * kf + i], JT[i] * nrm * w);
        for (int j = 0; j < 6; ++j) atomicAdd(&d.A[36 * kf + 6 * i + j], JT[i] * JT[j] * w);
      }
    }
  }
  // error: warp reduce, one atomic per warp
  for (int off = 16; off > 0; off >>= 1) e2w += __shfl_xor_sync(0xFFFFFFFFu, e2w, off);
  if ((threadIdx.x & 31) == 0 && e2w != 0.0) atomicAdd(&d.scal[0], e2w);
}

__device__ __forceinline__ void lba_atomic_max_pos(double* addr, double v) {   // v >= 0: the bit patterns are ordered
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

__device__ __forceinline__ void lba_lm_accum(const LbaDev& d, int l) {
  if (l >= d.nlm) return;
  const int dim = l < d.npt ? 3 : 6;
  double D[36], g[6];
  for (int i = 0; i < 36; ++i) D[i] = 0.0;
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  for (int k = d.lm_start[l]; k < d.lm_start[l + 1]; ++k) {
    const double* jx = d.Jx + 6 * (size_t)k;
    const double w = d.Wn[2 * (size_t)k], rn = d.Wn[2 * (size_t)k + 1];
    for (int i = 0; i < dim; ++i) {
      g[i] += jx[i] * rn;
      for (int j = 0; j < dim; ++j) D[6 * i + j] += jx[i] * jx[j] * w;
    }
  }
  double mx = 0.0;
  bool zero = false;
  for (int i = 0; i < dim; ++i) { mx = fmax(mx, fabs(D[7 * i])); zero |= D[7 * i] == 0.0; }
  for (int i = 0; i < 36; ++i) d.D[36 * (size_t)l + i] = D[i];
  for (int i = 0; i < 6; ++i) d.gl[6 * (size_t)l + i] = g[i];
  lba_atomic_max_pos(&d.scal[2], mx);
  // a zero diagonal entry: scal[4] (as an integer) keeps nlm - l of the first such landmark, 0 when there is none
  if (zero) atomicMax(reinterpret_cast<unsigned long long*>(&d.scal[4]), (unsigned long long)(d.nlm - l));
}

__device__ __forceinline__ void lba_kf_diagmax(const LbaDev& d, int i) {
  if (i < 6 * d.nkf) lba_atomic_max_pos(&d.scal[2], fabs(d.A[36 * (i / 6) + 7 * (i % 6)]));
}

// in-place inverse of a symmetric positive definite dim x dim matrix (row stride 6) by Gauss-Jordan without pivoting
__device__ void lba_inv_spd(double* M, int dim, double* Minv) {
  for (int i = 0; i < dim; ++i)
    for (int j = 0; j < dim; ++j) Minv[6 * i + j] = i == j ? 1.0 : 0.0;
  for (int p = 0; p < dim; ++p) {
    const double ip = 1.0 / M[7 * p];
    for (int j = 0; j < dim; ++j) { M[6 * p + j] *= ip; Minv[6 * p + j] *= ip; }
    for (int i = 0; i < dim; ++i) {
      if (i == p) continue;
      const double f = M[6 * i + p];
      for (int j = 0; j < dim; ++j) { M[6 * i + j] -= f * M[6 * p + j]; Minv[6 * i + j] -= f * Minv[6 * p + j]; }
    }
  }
}

// swap (g6): for line landmarks the coupling block is w Jt Jx^T, so Jt is the landmark-side vector and Jx the pose side
__device__ __forceinline__ void lba_lm_schur(const LbaDev& d, int l, double lambda, int swap) {
  if (l >= d.nlm) return;
  const int dim = l < d.npt ? 3 : 6, n = 6 * d.nkf;
  const double* U = swap && l >= d.npt ? d.Jt : d.Jx;   // landmark side of the coupling
  const double* V = swap && l >= d.npt ? d.Jx : d.Jt;   // keyframe side
  double D[36], Di[36], g[6];
  for (int i = 0; i < 36; ++i) D[i] = d.D[36 * (size_t)l + i];
  for (int i = 0; i < 6; ++i) g[i] = d.gl[6 * (size_t)l + i];
  for (int i = 0; i < dim; ++i) D[7 * i] += lambda * D[7 * i];
  lba_inv_spd(D, dim, Di);
  for (int i = 0; i < 36; ++i) d.Dinv[36 * (size_t)l + i] = Di[i];
  const int s = d.lm_start[l], e = d.lm_start[l + 1];
  for (int a = s; a < e; ++a) {
    const int ka = d.obs_kf[a];
    if (ka < 0) continue;
    const double* jxa = U + 6 * (size_t)a;
    const double* jta = V + 6 * (size_t)a;
    const double wa = d.Wn[2 * (size_t)a];
    double y[6];
    for (int i = 0; i < dim; ++i) {
      double v = 0.0;
      for (int j = 0; j < dim; ++j) v += Di[6 * i + j] * jxa[j];
      y[i] = wa * v;
    }
    double yg = 0.0;
    for (int i = 0; i < dim; ++i) yg += y[i] * g[i];
    for (int i = 0; i < 6; ++i) atomicAdd(&d.gred[6 * ka + i], -yg * jta[i]);
    for (int b = s; b < e; ++b) {
      const int kb = d.obs_kf[b];
      if (kb < 0) continue;
      const double* jxb = U + 6 * (size_t)b;
      const double* jtb = V + 6 * (size_t)b;
      double cab = 0.0;
      for (int i = 0; i < dim; ++i) cab += y[i] * jxb[i];
      cab *= d.Wn[2 * (size_t)b];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) atomicAdd(&d.S[(size_t)(6 * ka + i) * n + 6 * kb + j], -cab * jta[i] * jtb[j]);
    }
  }
}

// One CTA of 256 threads: S += A' (block diagonal, damped), g_red += g_c, dense LDL^T without pivoting, solve
// S dx_c = g_red.
__device__ __forceinline__ void lba_solve(const LbaDev& d, double lambda) {
  const int n = 6 * d.nkf, tid = threadIdx.x;
  double* S = d.S;
  for (int i = tid; i < 36 * d.nkf; i += 256) {
    const int kf = i / 36, r = (i % 36) / 6, cc = i % 6;
    double v = d.A[i];
    if (r == cc) v += lambda * v;
    S[(size_t)(6 * kf + r) * n + 6 * kf + cc] += v;
  }
  for (int i = tid; i < n; i += 256) d.gred[i] += d.gc[i];
  __syncthreads();
  // right-looking LDL^T on the lower triangle: after column j, S[i][j] = L_ij, S[j][j] = D_j
  for (int j = 0; j < n; ++j) {
    const double dj = S[(size_t)j * n + j];
    __syncthreads();
    for (int i = j + 1 + tid; i < n; i += 256) S[(size_t)i * n + j] /= dj;
    __syncthreads();
    // trailing update: S[i][k] -= L_ij D_j L_kj for j < k <= i
    const int m = n - j - 1;
    for (int t = tid; t < m * m; t += 256) {
      const int i = j + 1 + t / m, k = j + 1 + t % m;
      if (k <= i) S[(size_t)i * n + k] -= S[(size_t)i * n + j] * dj * S[(size_t)k * n + j];
    }
    __syncthreads();
  }
  if (tid == 0) {   // n <= 384: the two triangular solves are a few thousand operations
    double* x = d.dxc;
    for (int i = 0; i < n; ++i) {
      double v = d.gred[i];
      for (int k = 0; k < i; ++k) v -= S[(size_t)i * n + k] * x[k];
      x[i] = v;
    }
    for (int i = 0; i < n; ++i) x[i] /= S[(size_t)i * n + i];
    for (int i = n - 1; i >= 0; --i) {
      double v = x[i];
      for (int k = i + 1; k < n; ++k) v -= S[(size_t)k * n + i] * x[k];
      x[i] = v;
    }
    for (int i = 0; i < n; ++i) d.DX[i] = x[i];
  }
}
__global__ void __launch_bounds__(256) k_lba_solve(LbaDev d, double lambda) { lba_solve(d, lambda); }

__device__ __forceinline__ void lba_backsub(const LbaDev& d, int l, int swap) {
  if (l >= d.nlm) return;
  const int dim = l < d.npt ? 3 : 6;
  const double* U = swap && l >= d.npt ? d.Jt : d.Jx;   // as lba_lm_schur
  const double* V = swap && l >= d.npt ? d.Jx : d.Jt;
  double r[6];
  for (int i = 0; i < 6; ++i) r[i] = d.gl[6 * (size_t)l + i];
  for (int a = d.lm_start[l]; a < d.lm_start[l + 1]; ++a) {
    const int ka = d.obs_kf[a];
    if (ka < 0) continue;
    const double* jt = V + 6 * (size_t)a;
    const double* jx = U + 6 * (size_t)a;
    double s = 0.0;
    for (int i = 0; i < 6; ++i) s += jt[i] * d.dxc[6 * ka + i];
    s *= d.Wn[2 * (size_t)a];
    for (int i = 0; i < dim; ++i) r[i] -= jx[i] * s;
  }
  const double* Di = d.Dinv + 36 * (size_t)l;
  const int off = l < d.npt ? 6 * d.nkf + 3 * l : 6 * d.nkf + 3 * d.npt + 6 * (l - d.npt);
  for (int i = 0; i < dim; ++i) {
    double v = 0.0;
    for (int j = 0; j < dim; ++j) v += Di[6 * i + j] * r[j];
    d.DX[off + i] = v;
  }
}

// |DX|^2 always; the step itself only when `apply`.  Element i: keyframe i (i < nkf), else one landmark coordinate.  Every
// lane of the warp calls it.
__device__ __forceinline__ void lba_apply(const LbaDev& d, int i, int apply) {
  double n2 = 0.0;
  if (i < d.nkf) {
    for (int c = 0; c < 6; ++c) n2 += d.DX[6 * i + c] * d.DX[6 * i + c];
    if (apply) {
      double T[16];
      d_expmap(d.X + 6 * i, T);
      d_update_pose(T, d.DX + 6 * i);   // T <- T * inverse_se3(expmap_se3(dx))
      double x[6];
      d_logmap(T, x);
      for (int c = 0; c < 6; ++c) d.X[6 * i + c] = x[c];
    }
  } else if (i < d.nkf + (d.N - 6 * d.nkf)) {
    const int j = 6 * d.nkf + (i - d.nkf);
    n2 = d.DX[j] * d.DX[j];
    if (apply) d.X[j] += d.DX[j];
  }
  for (int off = 16; off > 0; off >>= 1) n2 += __shfl_xor_sync(0xFFFFFFFFu, n2, off);
  if ((threadIdx.x & 31) == 0 && n2 != 0.0) atomicAdd(&d.scal[1], n2);
}

__device__ __forceinline__ void lba_prep(const LbaDev& d, int i, const double* fixedT, double* fixedTinv, int n_fixed) {
  if (i < d.nkf) {
    double T[16], Ti[16];
    d_expmap(d.X0 + 6 * i, T);
    d_inverse_se3(T, Ti);
    for (int k = 0; k < 16; ++k) d.T0inv[16 * i + k] = Ti[k];
  }
  if (i < n_fixed) {
    double Ti[16];
    d_inverse_se3(fixedT + 16 * i, Ti);
    for (int k = 0; k < 16; ++k) fixedTinv[16 * i + k] = Ti[k];
  }
}

__device__ __forceinline__ void lba_moved(const LbaDev& d, int l, uint8_t* pt_moved, uint8_t* ls_moved) {
  if (l >= d.nlm) return;
  const int dim = l < d.npt ? 3 : 6;
  const int off = l < d.npt ? 6 * d.nkf + 3 * l : 6 * d.nkf + 3 * d.npt + 6 * (l - d.npt);
  double n2 = 0.0;
  for (int c = 0; c < dim; ++c) { const double v = d.X[off + c] - d.X0[off + c]; n2 += v * v; }
  const uint8_t m = sqrt(n2) > 0.01;   // :1829, :1843
  if (l < d.npt) pt_moved[l] = m; else ls_moved[l - d.npt] = m;
}

// (g2) `int Hmax` scanned over the first pass's diagonal in index order (:2359-2364): `d > Hmax` compares with the int,
// `Hmax = fabs(d)` truncates, and a value >= 2^31 converts to INT_MIN (x86-64 cvttsd2si), which the next diagonal entry
// (>= 0) always replaces, unless it is NaN (both comparisons false).  So the result is INT_MIN when an entry is >= 2^31
// and no non-NaN entry follows the last such one, else the truncated maximum of the non-NaN entries after the last one
// >= 2^31 (or of all of them).  One CTA of 1024 threads; leaves the value in scal[3].
__device__ __forceinline__ void gba_hmax_int(const LbaDev& d) {
  __shared__ int last_big, any_after;
  __shared__ unsigned long long mx;
  const int tid = threadIdx.x, nk = 6 * d.nkf, np3 = 3 * d.npt;
  if (tid == 0) { last_big = -1; any_after = 0; mx = 0ull; }
  __syncthreads();
  auto diag = [&](int i) -> double {
    if (i < nk) return d.A[36 * (i / 6) + 7 * (i % 6)];
    i -= nk;
    if (i < np3) return d.D[36 * (size_t)(i / 3) + 7 * (i % 3)];
    i -= np3;
    return d.D[36 * (size_t)(d.npt + i / 6) + 7 * (i % 6)];
  };
  for (int i = tid; i < d.N; i += 1024)
    if (fabs(diag(i)) >= 2147483648.0) atomicMax(&last_big, i);
  __syncthreads();
  for (int i = last_big + 1 + tid; i < d.N; i += 1024) {
    const double v = fabs(diag(i));
    if (v == v) {   // NaN: both comparisons false, skipped
      atomicMax(&mx, (unsigned long long)__double_as_longlong(v));
      any_after = 1;
    }
  }
  __syncthreads();
  if (tid == 0)
    d.scal[3] = last_big >= 0 && !any_after ? -2147483648.0 : trunc(__longlong_as_double((long long)mx));
}

// ---- blocked LDL^T of the reduced system for n = 6 n_kf > 384 (plf_global_ba) -----------------------------------------
// Right-looking over 64 x 64 tiles of S (row-major, leading dimension n; only the lower triangle is read), the same
// factorisation as lba_solve: per tile column k, gba_diag factors the diagonal tile in shared memory, gba_panel solves
// each tile below it (L_ik = S_ik L_kk^-T D_k^-1, keeping W_ik = L_ik D_k) and flags whether it is exactly zero, and
// gba_update subtracts W_ik L_jk^T from every trailing lower tile (i, j) whose two panel tiles are non-zero, on the FP64
// tensor cores.  The substitutions run per tile (gba_fwd / gba_bwd) and skip the same zero tiles.  Tiles past n are
// padded with the identity; n_t = ceil(n / 64).
constexpr int GBA_T = 64, GBA_LD = 65;

__device__ __forceinline__ double gba_S(const LbaDev& d, int r, int c) {   // S[r][c], 0 outside the matrix
  const int n = 6 * d.nkf;
  return r < n && c < n ? d.S[(size_t)r * n + c] : 0.0;
}
// the factored diagonal tile k: strictly lower L into L[64][GBA_LD] (diagonal = D, 1 in the padding)
__device__ __forceinline__ void gba_load_lkk(const LbaDev& d, int k, double* L) {
  const int n = 6 * d.nkf, r0 = GBA_T * k;
  for (int e = threadIdx.x; e < GBA_T * GBA_T; e += blockDim.x) {
    const int r = e >> 6, c = e & 63;
    L[r * GBA_LD + c] = c > r ? 0.0 : (r0 + r < n ? gba_S(d, r0 + r, r0 + c) : (r == c ? 1.0 : 0.0));
  }
}

// Each stage's work for one CTA (or element) of one problem is a __device__ function of the problem's LbaDev, which the
// k_gbb_* kernels run on every large problem of a call.
__device__ __forceinline__ void gba_damp(const LbaDev& d, double lambda, int i) {   // lba_solve's prologue
  const int n = 6 * d.nkf;
  if (i < 36 * d.nkf) {
    const int kf = i / 36, r = (i % 36) / 6, cc = i % 6;
    double v = d.A[i];
    if (r == cc) v += lambda * v;
    d.S[(size_t)(6 * kf + r) * n + 6 * kf + cc] += v;
  } else if (i < 36 * d.nkf + n) {
    d.gred[i - 36 * d.nkf] += d.gc[i - 36 * d.nkf];
  }
}

__device__ __forceinline__ void gba_diag(const LbaDev& d, int k) {
  __shared__ double T[GBA_T * GBA_LD];
  const int n = 6 * d.nkf, r0 = GBA_T * k, tid = threadIdx.x;
  for (int e = tid; e < GBA_T * GBA_T; e += 256) {
    const int r = e >> 6, c = e & 63;
    T[r * GBA_LD + c] = r0 + r < n && r0 + c < n ? d.S[(size_t)(r0 + r) * n + r0 + c] : (r == c ? 1.0 : 0.0);
  }
  __syncthreads();
  for (int j = 0; j < GBA_T; ++j) {   // as lba_solve: after column j, T[i][j] = L_ij, T[j][j] = D_j
    const double dj = T[j * GBA_LD + j];
    for (int i = j + 1 + tid; i < GBA_T; i += 256) T[i * GBA_LD + j] /= dj;
    __syncthreads();
    const int m = GBA_T - j - 1;
    for (int t = tid; t < m * m; t += 256) {
      const int i = j + 1 + t / m, c = j + 1 + t % m;
      if (c <= i) T[i * GBA_LD + c] -= T[i * GBA_LD + j] * dj * T[c * GBA_LD + j];
    }
    __syncthreads();
  }
  for (int e = tid; e < GBA_T * GBA_T; e += 256) {
    const int r = e >> 6, c = e & 63;
    if (c <= r && r0 + r < n) d.S[(size_t)(r0 + r) * n + r0 + c] = T[r * GBA_LD + c];
  }
}

// one CTA per tile row i > k; gsm: dynamic shared memory of 2 x 64 x GBA_LD doubles
__device__ __forceinline__ void gba_panel(const LbaDev& d, double* Wp, uint8_t* nz, int k, int nt, int i, double* gsm) {
  double* L = gsm;
  double* Z = gsm + GBA_T * GBA_LD;
  const int n = 6 * d.nkf, r0 = GBA_T * i, c0 = GBA_T * k, tid = threadIdx.x;
  int any = 0;
  for (int e = tid; e < GBA_T * GBA_T; e += 256) {
    const int r = e >> 6, c = e & 63;
    const double v = gba_S(d, r0 + r, c0 + c);
    Z[r * GBA_LD + c] = v;
    any |= v != 0.0;
  }
  any = __syncthreads_or(any);
  if (tid == 0) nz[(size_t)i * nt + k] = (uint8_t)any;
  if (!any) return;   // L_ik = 0 exactly: nothing to write, nothing to update
  gba_load_lkk(d, k, L);
  __syncthreads();
  // Z = S_ik L_kk^-T, column by column: once column c is final, Z[r][c2] -= Z[r][c] L[c2][c] for c2 > c
  for (int c = 0; c < GBA_T - 1; ++c) {
    const int m = GBA_T - 1 - c;
    for (int t = tid; t < GBA_T * m; t += 256) {
      const int r = t / m, c2 = c + 1 + t % m;
      Z[r * GBA_LD + c2] -= Z[r * GBA_LD + c] * L[c2 * GBA_LD + c];
    }
    __syncthreads();
  }
  for (int e = tid; e < GBA_T * GBA_T; e += 256) {
    const int r = e >> 6, c = e & 63;
    const double z = Z[r * GBA_LD + c];
    Wp[((size_t)i * GBA_T + r) * GBA_T + c] = z;
    if (r0 + r < n && c0 + c < n) d.S[(size_t)(r0 + r) * n + c0 + c] = z / L[c * GBA_LD + c];
  }
}

__device__ __forceinline__ void gba_dmma(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b0) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3) : "d"(a0), "d"(a1), "d"(b0));
}

// S_ij -= W_ik L_jk^T for the trailing lower tiles k < j <= i, one CTA per tile (t enumerates (i, j) row by row).  8 warps; warp w owns rows 16 (w / 2) .. +16 and columns 32 (w % 2) .. +32 of the tile (4 m16n8 accumulators).
constexpr int GBA_KC = 32, GBA_SLD = 36;   // k chunk; shared row stride (conflict-free fragment loads per half warp)
__device__ __forceinline__ void gba_update(const LbaDev& d, const double* Wp, const uint8_t* nz, int k, int nt, int t) {
  int a = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((a + 1) * (a + 2) / 2 <= t) ++a;
  while (a * (a + 1) / 2 > t) --a;
  const int i = k + 1 + a, j = k + 1 + (t - a * (a + 1) / 2);
  if (!nz[(size_t)i * nt + k] || !nz[(size_t)j * nt + k]) return;
  __shared__ double As[GBA_T * GBA_SLD], Bs[GBA_T * GBA_SLD];
  const int n = 6 * d.nkf, tid = threadIdx.x, lane = tid & 31, w = tid >> 5, gid = lane >> 2, tig = lane & 3;
  const int wr = 16 * (w >> 1), wc = 32 * (w & 1);
  double acc[4][4];
  for (int q = 0; q < 4; ++q)
    for (int e = 0; e < 4; ++e) acc[q][e] = 0.0;
  for (int kc = 0; kc < GBA_T; kc += GBA_KC) {
    for (int e = tid; e < GBA_T * GBA_KC; e += 256) {
      const int r = e / GBA_KC, c = e % GBA_KC;
      As[r * GBA_SLD + c] = Wp[((size_t)i * GBA_T + r) * GBA_T + kc + c];
      Bs[r * GBA_SLD + c] = gba_S(d, GBA_T * j + r, GBA_T * k + kc + c);
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < GBA_KC; ks += 4) {
      const double a0 = As[(wr + gid) * GBA_SLD + ks + tig], a1 = As[(wr + gid + 8) * GBA_SLD + ks + tig];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const double b0 = Bs[(wc + 8 * q + gid) * GBA_SLD + ks + tig];
        gba_dmma(acc[q][0], acc[q][1], acc[q][2], acc[q][3], a0, a1, b0);
      }
    }
    __syncthreads();
  }
  for (int q = 0; q < 4; ++q)
    for (int e = 0; e < 4; ++e) {
      const int r = GBA_T * i + wr + gid + (e >> 1) * 8, c = GBA_T * j + wc + 8 * q + 2 * tig + (e & 1);
      if (r < n && c < n) d.S[(size_t)r * n + c] -= acc[q][e];
    }
}

// forward substitution step k: every CTA solves y_k = L_kk^-1 g_k (64 threads, in place of g's tile), CTA 0 stores it in
// dxc, CTA b > 0 subtracts L_ik y_k from g_i (i = k + b) when that tile is non-zero
__device__ __forceinline__ void gba_fwd(const LbaDev& d, const uint8_t* nz, int k, int nt, int b) {
  __shared__ double L[GBA_T * GBA_LD], y[GBA_T];
  const int n = 6 * d.nkf, i = k + b, r0 = GBA_T * k, tid = threadIdx.x;
  if (b > 0 && !nz[(size_t)i * nt + k]) return;
  gba_load_lkk(d, k, L);
  if (tid < GBA_T) y[tid] = r0 + tid < n ? d.gred[r0 + tid] : 0.0;
  __syncthreads();
  for (int c = 0; c < GBA_T - 1; ++c) {
    if (tid > c && tid < GBA_T) y[tid] -= L[tid * GBA_LD + c] * y[c];
    __syncthreads();
  }
  if (b == 0) {
    if (tid < GBA_T && r0 + tid < n) d.dxc[r0 + tid] = y[tid];
    return;
  }
  const int lane = tid & 31, w = tid >> 5;
  for (int rr = 0; rr < 8; ++rr) {   // warp w: rows 8 w .. 8 w + 7 of tile i
    const int r = GBA_T * i + 8 * w + rr;
    double s = gba_S(d, r, r0 + lane) * y[lane] + gba_S(d, r, r0 + 32 + lane) * y[32 + lane];
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, off);
    if (lane == 0 && r < n) d.gred[r] -= s;
  }
}

__device__ __forceinline__ void gba_dscale(const LbaDev& d, int i) {   // z = y / D
  const int n = 6 * d.nkf;
  if (i < n) d.gred[i] = d.dxc[i] / d.S[(size_t)i * n + i];
}

// backward substitution step k (k = n_t - 1 .. 0): every CTA solves x_k = L_kk^-T z_k, CTA 0 stores it in dxc and DX,
// CTA b > 0 subtracts L_kj^T x_k from z_j (j = b - 1) when that tile is non-zero
__device__ __forceinline__ void gba_bwd(const LbaDev& d, const uint8_t* nz, int k, int nt, int b) {
  __shared__ double L[GBA_T * GBA_LD], x[GBA_T], part[4][GBA_T];
  const int n = 6 * d.nkf, r0 = GBA_T * k, tid = threadIdx.x;
  if (b > 0 && !nz[(size_t)k * nt + (b - 1)]) return;
  gba_load_lkk(d, k, L);
  if (tid < GBA_T) x[tid] = r0 + tid < n ? d.gred[r0 + tid] : 0.0;
  __syncthreads();
  for (int c = GBA_T - 1; c > 0; --c) {
    if (tid < c) x[tid] -= L[c * GBA_LD + tid] * x[c];
    __syncthreads();
  }
  if (b == 0) {
    if (tid < GBA_T && r0 + tid < n) { d.dxc[r0 + tid] = x[tid]; d.DX[r0 + tid] = x[tid]; }
    return;
  }
  const int j = b - 1, c = tid & 63, rq = tid >> 6;
  double s = 0.0;
  for (int r = 16 * rq; r < 16 * rq + 16; ++r) s += gba_S(d, r0 + r, GBA_T * j + c) * x[r];
  part[rq][c] = s;
  __syncthreads();
  if (tid < GBA_T && GBA_T * j + tid < n) d.gred[GBA_T * j + tid] -= ((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid];
}

// Test hook (plslam_b200.h): one of the two factorisations on a caller's matrix.  Path 0 is gbb_ldlt with the one system
// by value and no activity flags, as plf_global_ba and plf_pose_graph run it; path 1 is k_lba_solve (lba_solve without
// k_lbb_solve's zeroing, so S comes back factored) with zero keyframe blocks and gradient and lambda = 0, so its prologue
// adds +0.0 to the diagonal 6 x 6 blocks and to g.  The zero flags are cleared first, so the ones the panel kernel never
// sets (i <= k) read 0.
extern "C" plf_status plf_debug_ldlt(plf_ctx* ctx, int path, int n6, double* S, const double* g, double* x, uint8_t* nz) {
  const char* fn = "plf_debug_ldlt";
  if (!ctx || !S || !g || !x) return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  if (path != 0 && path != 1) return plf_fail(ctx, PLF_ERR_INVALID, "%s: path %d (0: tiled, 1: one CTA)", fn, path);
  const int cap = path == 0 ? 4096 : 64;
  if (n6 < 1 || n6 > cap) return plf_fail(ctx, PLF_ERR_INVALID, "%s: n6 = %d outside [1, %d] for path %d", fn, n6, cap, path);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int n = 6 * n6, nt = (n + GBA_T - 1) / GBA_T;
  LbaDev d{};
  d.nkf = n6;
  double* dWp = nullptr;
  uint8_t* dNz = nullptr;
  DevBufList scr;
  scr.add(d.S, (size_t)n * n); scr.add(d.gred, n); scr.add(d.dxc, n); scr.add(d.DX, n);
  if (path == 0) { scr.add(dWp, (size_t)nt * GBA_T * GBA_T); scr.add(dNz, (size_t)nt * nt); }
  else { scr.add(d.A, (size_t)36 * n6); scr.add(d.gc, n); }
  if (plf_status st = scr.carve(ctx, PLF_SCR_BA)) return st;
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(d.S, S, (size_t)n * n * 8, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(d.gred, g, (size_t)n * 8, cudaMemcpyHostToDevice, cs));
  if (path == 0) {
    PLF_CUDA(ctx, cudaMemsetAsync(dNz, 0, (size_t)nt * nt, cs));
    GbbLdlt L{};
    L.S = d.S; L.g = d.gred; L.y = d.dxc; L.x = d.DX; L.Wp = dWp; L.nz = dNz; L.one = GbbBig{0, n6, 0, 0, 0, 0, 0};
    if (plf_status st = gbb_ldlt(ctx, cs, L, 1, n)) return st;
  } else {
    PLF_CUDA(ctx, cudaMemsetAsync(d.A, 0, (size_t)36 * n6 * 8, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(d.gc, 0, (size_t)n * 8, cs));
    k_lba_solve<<<1, 256, 0, cs>>>(d, 0.0);
    PLF_LAUNCH_CHECK(ctx);
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(S, d.S, (size_t)n * n * 8, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(x, d.DX, (size_t)n * 8, cudaMemcpyDeviceToHost, cs));
  if (path == 0 && nz) PLF_CUDA(ctx, cudaMemcpyAsync(nz, dNz, (size_t)nt * nt, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

// The host-side rules of one problem, up to its observations: counts, emptiness, the keyframe limit and NULL arrays.
// Messages start with `fn`.
static plf_status lba_check_shape(plf_ctx* ctx, const char* fn, const plf_lba_problem* p, int kf_cap) {
  if (p->n_kf < 0 || p->n_pt < 0 || p->n_ls < 0 || p->n_pt_obs < 0 || p->n_ls_obs < 0 || p->n_fixed < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  const int nkf = p->n_kf, npt = p->n_pt, nls = p->n_ls, npo = p->n_pt_obs, nlo = p->n_ls_obs;
  if (npo + nlo == 0 || 6 * nkf + 3 * npt + 6 * nls == 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: empty problem (the reference returns -1, :1324-1328)", fn);
  if (nkf > kf_cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d keyframes (limit %d)", fn, nkf, kf_cap);
  if ((nkf && !p->kf_pose) || (npt && !p->pt) || (nls && !p->ls) || (npo && (!p->pt_obs_lm || !p->pt_obs_kf || !p->pt_obs_xy)) ||
      (nlo && (!p->ls_obs_lm || !p->ls_obs_kf || !p->ls_obs_le)) || (p->n_fixed && !p->fixed_T))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: null array", fn);
  return PLF_OK;
}

// The rest of the host-side rules (indices in range, observations grouped, every landmark observed) while gathering the
// observations into the device layout: obs_lm / obs_kf [nobs] (points first, then lines), obs_z [nobs][3] and
// lm_start [nlm + 1] (each landmark's first observation).
static plf_status lba_gather(plf_ctx* ctx, const char* fn, const plf_lba_problem* p, int* lm_start, int* h_lm, int* h_kf,
                             double* h_z) {
  const int nkf = p->n_kf, npt = p->n_pt, nls = p->n_ls, npo = p->n_pt_obs, nobs = npo + p->n_ls_obs, nlm = npt + nls;
  for (int l = 0; l <= nlm; ++l) lm_start[l] = 0;
  // observations are grouped per landmark in non-decreasing landmark order (how the reference builds its lists, :1249-1277)
  for (int k = 0; k < nobs; ++k) {
    const bool is_line = k >= npo;
    const int lm = is_line ? p->ls_obs_lm[k - npo] : p->pt_obs_lm[k], kf = is_line ? p->ls_obs_kf[k - npo] : p->pt_obs_kf[k];
    const int lim = is_line ? nls : npt;
    if (lm < 0 || lm >= lim || kf >= nkf || kf < -p->n_fixed)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: observation %d refers to landmark %d / keyframe %d out of range", fn, k, lm, kf);
    const int prev = k == 0 || k == npo ? -1 : (is_line ? p->ls_obs_lm[k - npo - 1] : p->pt_obs_lm[k - 1]);
    if (lm < prev) return plf_fail(ctx, PLF_ERR_INVALID, "%s: observations must be grouped by landmark in ascending order", fn);
    h_lm[k] = lm; h_kf[k] = kf;
    lm_start[(is_line ? npt : 0) + lm + 1]++;
    if (is_line) for (int c = 0; c < 3; ++c) h_z[3 * (size_t)k + c] = p->ls_obs_le[3 * (size_t)(k - npo) + c];
    else {
      h_z[3 * (size_t)k] = p->pt_obs_xy[2 * (size_t)k]; h_z[3 * (size_t)k + 1] = p->pt_obs_xy[2 * (size_t)k + 1];
      h_z[3 * (size_t)k + 2] = 0.0;
    }
  }
  for (int l = 0; l < nlm; ++l)   // its landmark block would be zero
    if (!lm_start[l + 1])
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s landmark %d has no observation", fn, l < npt ? "point" : "line", l < npt ? l : l - npt);
  for (int l = 0; l < nlm; ++l) lm_start[l + 1] += lm_start[l];
  return PLF_OK;
}

// ---- the driver: one problem or many in one launch chain ---------------------------------------------------------------
// The problems' arrays are concatenated into flat arrays; LbbProb holds problem p's counts, its offsets into each flat
// array and its camera, and lbb_view() builds the LbaDev of its slice, so the kernels below run the single-problem
// functions above on each problem.  They are gridded (problem, chunk): blockIdx.x is the problem and blockIdx.y strides
// over its observations, landmarks or elements, so no warp mixes two problems.  The reference's control flow runs on the
// device in LbbCtrl, one thread per problem (k_lbb_first, k_lbb_test, k_lbb_step).  A problem that has stopped, or was
// refused, is inactive, and every later kernel returns at once for it.  All max_iters rounds are enqueued up front, so
// the call has one host synchronisation, after the download.
struct LbbProb {
  int nkf, npt, nls, npo, nobs, nlm, N, nfix;
  long long xo, oo, lo, ko, fo, go, so;   // offsets into X (doubles), observations, landmarks, keyframes, fixed
                                          // keyframes, rows of the reduced systems and S (doubles)
  LbaCam cam;
};
struct LbbCtrl {
  double lambda, err, err_prev;
  int iters;     // the loop counter at exit: max(max_iters, 1) unless a stop test breaks the loop earlier
  int active;    // 0 once the problem has stopped or was refused
  int apply;     // this round's step is applied (the error did not grow)
  int zero_lm;   // the first landmark whose first-pass block has a zero diagonal entry (the problem is refused), or -1
};
struct LbbDev {
  const LbbProb* prob; LbbCtrl* ctrl; int P;
  double* X; double* X0; double* T0inv; const double* fixedT; double* fixedTinv;
  const int* obs_lm; const int* obs_kf; const double* obs_z; const int* lm_start;   // lm_start: nlm + 1 per problem
  double* Jt; double* Jx; double* Wn; double* D; double* gl; double* Dinv; double* A; double* gc;
  double* S; double* gred; double* dxc; double* DX; double* scal; uint8_t* moved;
};

__device__ __forceinline__ LbaDev lbb_view(const LbbDev& b, const LbbProb& q, int p) {
  LbaDev d;
  d.nkf = q.nkf; d.npt = q.npt; d.nls = q.nls; d.N = q.N; d.npo = q.npo; d.nlo = q.nobs - q.npo; d.nobs = q.nobs; d.nlm = q.nlm;
  d.X = b.X + q.xo; d.X0 = b.X0 + q.xo; d.T0inv = b.T0inv + 16 * q.ko; d.fixedTinv = b.fixedTinv + 16 * q.fo;
  d.obs_lm = b.obs_lm + q.oo; d.obs_kf = b.obs_kf + q.oo; d.obs_z = b.obs_z + 3 * q.oo; d.lm_start = b.lm_start + q.lo + p;
  d.Jt = b.Jt + 6 * q.oo; d.Jx = b.Jx + 6 * q.oo; d.Wn = b.Wn + 2 * q.oo;
  d.D = b.D + 36 * q.lo; d.gl = b.gl + 6 * q.lo; d.Dinv = b.Dinv + 36 * q.lo;
  d.A = b.A + 36 * q.ko; d.gc = b.gc + 6 * q.ko;
  d.S = b.S + q.so; d.gred = b.gred + q.go; d.dxc = b.dxc + q.go; d.DX = b.DX + q.xo;
  d.scal = b.scal + 8 * p;
  return d;
}

// T0inv / fixedTinv, X = X0 and the control state
__global__ void __launch_bounds__(128) k_lbb_prep(LbbDev b, double lambda, int iters) {
  const int p = blockIdx.x;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  for (int i = threadIdx.x; i < max(q.nkf, q.nfix); i += 128) lba_prep(d, i, b.fixedT + 16 * q.fo, b.fixedTinv + 16 * q.fo, q.nfix);
  for (int i = threadIdx.x; i < q.N; i += 128) d.X[i] = d.X0[i];
  if (threadIdx.x == 0) b.ctrl[p] = LbbCtrl{lambda, 0.0, 0.0, iters, 1, 1, -1};
}

__global__ void __launch_bounds__(128) k_lbb_rows(LbbDev b, int mode, int quirks, double homog_th) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  for (int c = blockIdx.y; 128 * c < q.nobs; c += gridDim.y) lba_rows(d, q.cam, 128 * c + threadIdx.x, mode, quirks, homog_th);
}

__global__ void __launch_bounds__(128) k_lbb_lm_accum(LbbDev b) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  for (int c = blockIdx.y; 128 * c < q.nlm; c += gridDim.y) lba_lm_accum(d, 128 * c + threadIdx.x);
}

__global__ void __launch_bounds__(128) k_lbb_kf_diagmax(LbbDev b) {
  const int p = blockIdx.x;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  for (int i = threadIdx.x; i < 6 * q.nkf; i += 128) lba_kf_diagmax(d, i);
}

// swap: (g6), round 0 of plf_global_ba_batch under its quirks
__global__ void __launch_bounds__(128) k_lbb_schur(LbbDev b, int swap) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  const double lambda = b.ctrl[p].lambda;
  for (int c = blockIdx.y; 128 * c < q.nlm; c += gridDim.y) lba_lm_schur(d, 128 * c + threadIdx.x, lambda, swap);
}

// One CTA per problem with n = 6 n_kf <= 384 (lba_solve); then zeroes A, g_c, S and g_red for the next round's
// accumulation.  Larger problems (plf_global_ba) are solved by the k_gbb_* kernels.
__global__ void __launch_bounds__(256) k_lbb_solve(LbbDev b) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  if (!q.nkf || q.nkf > 64) return;
  const LbaDev d = lbb_view(b, q, p);
  lba_solve(d, b.ctrl[p].lambda);
  __syncthreads();
  const int n = 6 * q.nkf;
  for (int i = threadIdx.x; i < n * n; i += 256) d.S[i] = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) d.gred[i] = 0.0;
  for (int i = threadIdx.x; i < 6 * n; i += 256) d.A[i] = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) d.gc[i] = 0.0;
}

__global__ void __launch_bounds__(128) k_lbb_backsub(LbbDev b, int swap) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  for (int c = blockIdx.y; 128 * c < q.nlm; c += gridDim.y) lba_backsub(d, 128 * c + threadIdx.x, swap);
}

__global__ void __launch_bounds__(128) k_lbb_apply(LbbDev b) {
  const int p = blockIdx.x;
  if (!b.ctrl[p].active) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  const int apply = b.ctrl[p].apply, ne = q.nkf + (q.N - 6 * q.nkf);
  for (int c = blockIdx.y; 128 * c < ne; c += gridDim.y) lba_apply(d, 128 * c + threadIdx.x, apply);
}

// The control of both routines: G selects plf_global_ba's over plf_local_ba's.
// After the first pass: the refusal, the error normalisation (q1 / g1: the reference divides by two counters it never
// increments, 0.0 here as there) and lambda *= Hmax (g2: the int-truncated maximum of k_gbb_hmax_int).  The first step
// is applied unconditionally (apply = 1 from k_lbb_prep).
template <bool G>
__device__ __forceinline__ void lbb_first(const LbbDev& b, int quirks) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= b.P) return;
  LbbCtrl& c = b.ctrl[p];
  const LbbProb& q = b.prob[p];
  double* scal = b.scal + 8 * p;
  const unsigned long long zero_flag = (unsigned long long)__double_as_longlong(scal[4]);
  if (zero_flag) { c.zero_lm = q.nlm - (int)zero_flag; c.active = 0; return; }
  double err = scal[0];
  if (quirks & BAQ_FIRST_ERR0) err = __ddiv_rn(err, 0.0);   // (q1) :1541
  else err /= (double)q.nobs;
  // Hmax: under (g2) scal[3], else the double whose bit pattern lba_lm_accum / lba_kf_diagmax maximised
  c.lambda *= G && (quirks & BAQ_HMAX_INT) ? scal[3] : scal[2];
  c.err = err;
  c.err_prev = err;
  scal[0] = 0.0;
}
__global__ void k_lbb_first(LbbDev b, int quirks) { lbb_first<false>(b, quirks); }
__global__ void k_gbb_first(LbbDev b, int quirks) { lbb_first<true>(b, quirks); }

// Round r >= 1 after its accumulation: the error, the change and min-error stops (:1773-1775, :2637) and whether it
// grew.  LBA divides the error by the landmark count (:1773), GBA by the observation count, or under (g3) by the zero
// counters (:2635), so that only max_iters or the |DX| test ends its run.
template <bool G>
__device__ __forceinline__ void lbb_test(const LbbDev& b, int r, int quirks, double min_error, double min_error_change) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= b.P || !b.ctrl[p].active) return;
  LbbCtrl& c = b.ctrl[p];
  const LbbProb& q = b.prob[p];
  double* scal = b.scal + 8 * p;
  const double err = !G ? scal[0] / (double)(q.npt + q.nls)
                        : (quirks & BAQ_ITER_ERR0) ? __ddiv_rn(scal[0], 0.0) : scal[0] / (double)q.nobs;
  scal[0] = 0.0;
  c.err = err;
  if (fabs(err - c.err_prev) < min_error_change || err < min_error) { c.active = 0; c.iters = r; return; }
  c.apply = !(err > c.err_prev);
}
__global__ void k_lbb_test(LbbDev b, int r, double min_error, double min_error_change) {
  lbb_test<false>(b, r, 0, min_error, min_error_change);
}
__global__ void k_gbb_test(LbbDev b, int r, int quirks, double min_error, double min_error_change) {
  lbb_test<true>(b, r, quirks, min_error, min_error_change);
}

// Round r after its step: the lambda schedule (:1785-1803) and the |DX| stop (:1805); round 0 only clears |DX|^2.
__global__ void k_lbb_step(LbbDev b, int r, double lambda_k, double min_error_change) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= b.P || !b.ctrl[p].active) return;
  LbbCtrl& c = b.ctrl[p];
  double* scal = b.scal + 8 * p;
  const double dxn = sqrt(scal[1]);
  scal[1] = 0.0;
  if (r == 0) return;
  if (c.apply) c.lambda *= lambda_k; else c.lambda /= lambda_k;
  if (dxn < min_error_change) { c.active = 0; c.iters = r; return; }
  c.err_prev = c.err;
}

__global__ void __launch_bounds__(128) k_lbb_moved(LbbDev b) {
  const int p = blockIdx.x;
  if (b.ctrl[p].zero_lm >= 0) return;
  const LbbProb q = b.prob[p];
  const LbaDev d = lbb_view(b, q, p);
  uint8_t* m = b.moved + q.lo;
  for (int c = blockIdx.y; 128 * c < q.nlm; c += gridDim.y) lba_moved(d, 128 * c + threadIdx.x, m, m + q.npt);
}

// ---- plf_global_ba: the large problems' tiled LDL^T ----------------------------------------------------------------------
// A problem with n = 6 n_kf > 384 is factored by the tiled LDL^T above, with its own Wp and zero flags.  Per tile column
// there is one launch of each stage over every large problem, gridded (tile, problem) at the largest problem's extent:
// blockIdx.y picks the problem from the GbbBig table (or the one problem passed by value), and a CTA whose problem has
// fewer tiles, has stopped or was refused returns at once.  Each CTA runs the single-problem function of the stage, so a
// problem's factorisation does not depend on the others.  GbbBig and GbbLdlt are declared in plf_internal.h:
// plf_pose_graph factors through gbb_ldlt too.
// The LbaDev fields the tiled kernels read, for problem blockIdx.y, and its tile count; false when it is not active.
__device__ __forceinline__ bool gbb_view(const GbbLdlt& L, LbaDev& d, GbbBig& t, int& nt) {
  t = L.big ? L.big[blockIdx.y] : L.one;
  if (L.active && !L.active[(size_t)t.p * L.active_stride]) return false;
  d.nkf = t.nkf; d.S = L.S + t.so; d.gred = L.g + t.go; d.dxc = L.y + t.go; d.DX = L.x + t.xo;
  nt = (6 * t.nkf + GBA_T - 1) / GBA_T;
  return true;
}

__global__ void __launch_bounds__(256) k_gbb_diag(GbbLdlt L, int k) {
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt) || k >= nt) return;
  gba_diag(d, k);
}
__global__ void __launch_bounds__(256) k_gbb_panel(GbbLdlt L, int k) {
  extern __shared__ double gsm[];
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt) || k + 1 + (int)blockIdx.x >= nt) return;
  gba_panel(d, L.Wp + t.wo, L.nz + t.zo, k, nt, k + 1 + blockIdx.x, gsm);
}
__global__ void __launch_bounds__(256) k_gbb_update(GbbLdlt L, int k) {
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt)) return;
  const int m = nt - k - 1;
  if (m <= 0 || (int)blockIdx.x >= m * (m + 1) / 2) return;
  gba_update(d, L.Wp + t.wo, L.nz + t.zo, k, nt, blockIdx.x);
}
__global__ void __launch_bounds__(256) k_gbb_fwd(GbbLdlt L, int k) {
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt) || k + (int)blockIdx.x >= nt) return;
  gba_fwd(d, L.nz + t.zo, k, nt, blockIdx.x);
}
__global__ void __launch_bounds__(256) k_gbb_dscale(GbbLdlt L) {
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt)) return;
  gba_dscale(d, blockIdx.x * 256 + threadIdx.x);
}
__global__ void __launch_bounds__(256) k_gbb_bwd(GbbLdlt L, int k) {
  LbaDev d{}; GbbBig t; int nt;
  if (!gbb_view(L, d, t, nt) || k >= nt) return;
  gba_bwd(d, L.nz + t.zo, k, nt, blockIdx.x);
}

// The tiled factorisation and the two substitutions of the nb problems in L.big (or of L.one), the largest with n_max
// rows: per tile column k, gba_diag, gba_panel and gba_update; then gba_fwd per tile, gba_dscale and gba_bwd per tile.
plf_status gbb_ldlt(plf_ctx* ctx, cudaStream_t cs, const GbbLdlt& L, int nb, int n_max) {
  static_assert(GBA_T == PLF_LDLT_TILE, "plf_internal.h states the tile size");
  const int nt = (n_max + GBA_T - 1) / GBA_T, smem = 2 * GBA_T * GBA_LD * 8;
  PLF_CUDA(ctx, cudaFuncSetAttribute(k_gbb_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  for (int k = 0; k < nt; ++k) {
    k_gbb_diag<<<dim3(1, nb), 256, 0, cs>>>(L, k);
    PLF_LAUNCH_CHECK(ctx);
    const int m = nt - k - 1;
    if (!m) break;
    k_gbb_panel<<<dim3(m, nb), 256, smem, cs>>>(L, k);
    PLF_LAUNCH_CHECK(ctx);
    k_gbb_update<<<dim3(m * (m + 1) / 2, nb), 256, 0, cs>>>(L, k);
    PLF_LAUNCH_CHECK(ctx);
  }
  for (int k = 0; k < nt; ++k) {
    k_gbb_fwd<<<dim3(nt - k, nb), 256, 0, cs>>>(L, k);
    PLF_LAUNCH_CHECK(ctx);
  }
  k_gbb_dscale<<<dim3((n_max + 255) / 256, nb), 256, 0, cs>>>(L);
  PLF_LAUNCH_CHECK(ctx);
  for (int k = nt - 1; k >= 0; --k) {
    k_gbb_bwd<<<dim3(k + 1, nb), 256, 0, cs>>>(L, k);
    PLF_LAUNCH_CHECK(ctx);
  }
  return PLF_OK;
}

// S += A' and g_red += g_c of every active large problem (gba_damp), gridded (chunk, problem)
__global__ void __launch_bounds__(256) k_gbb_damp(LbbDev b, const GbbBig* big) {
  const GbbBig t = big[blockIdx.y];
  if (!b.ctrl[t.p].active) return;
  const LbaDev d = lbb_view(b, b.prob[t.p], t.p);
  const double lambda = b.ctrl[t.p].lambda;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < 42 * t.nkf; i += gridDim.x * 256) gba_damp(d, lambda, i);
}

// Zeroes S, g_red, A and g_c of every active large problem for the next round's accumulation (k_lbb_solve does it for
// the small ones), across the GPU: S is 288 n_kf^2 bytes, 4.8 GB at 4096 keyframes.
__global__ void __launch_bounds__(256) k_gbb_zero(LbbDev b, const GbbBig* big) {
  const GbbBig t = big[blockIdx.y];
  if (!b.ctrl[t.p].active) return;
  const LbaDev d = lbb_view(b, b.prob[t.p], t.p);
  const size_t n = 6 * (size_t)t.nkf, stride = (size_t)gridDim.x * 256;
  for (size_t i = blockIdx.x * 256 + threadIdx.x; i < n * n; i += stride) d.S[i] = 0.0;
  for (size_t i = blockIdx.x * 256 + threadIdx.x; i < n; i += stride) { d.gred[i] = 0.0; d.gc[i] = 0.0; }
  for (size_t i = blockIdx.x * 256 + threadIdx.x; i < 6 * n; i += stride) d.A[i] = 0.0;
}

// (g2) on the first pass, one CTA of 1024 threads per problem
__global__ void __launch_bounds__(1024) k_gbb_hmax_int(LbbDev b) {
  const int p = blockIdx.x;
  gba_hmax_int(lbb_view(b, b.prob[p], p));
}

// plf_local_ba / plf_global_ba (one problem, batch = false) and their _batch forms: the host-side rules per problem and
// the reference's control on the device (k_lbb_first / k_lbb_test, or k_gbb_first / k_gbb_test with global), one upload,
// every round enqueued, one download.  `global` selects levMarquardtOptimizationGBA (:2101-2699) over
// levMarquardtOptimizationLBA (:1332-1989): its quirk set, its error normalisation in the LM iterations and up to 4096
// keyframes (the tiled factorisation beyond n = 384).  Both refuse a landmark whose first-pass block D has an exactly
// zero diagonal entry, before any step: the reference would factor a zero pivot (its SimplicialLDLT's failure is not
// checked) and the landmark, then every keyframe observing it, would turn NaN.  A landmark without observations is
// refused by name on the host; the rest by one flag per problem set with the first pass.
static plf_status lbb_run(plf_ctx* ctx, const plf_lba_opts* opts, int n_problems, const plf_lba_problem* problems,
                          const int32_t* seq, plf_lba_result* out, plf_status* status, bool global, bool batch) {
  const char* fn = global ? (batch ? "plf_global_ba_batch" : "plf_global_ba") : (batch ? "plf_local_ba_batch" : "plf_local_ba");
  if (!ctx || !opts || n_problems < 0 || (n_problems && (!problems || !status)))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  const int P = n_problems;
  if (!P) return PLF_OK;
  // the large problems are gridded in y, at most 65535 of them; the limit is on the batch so that it does not depend on
  // the problems' sizes
  if (batch && global && P > 65535) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d problems (limit 65535)", fn, P);
  // problem p's messages start with "fn: problem p", or with fn alone in the one-problem calls
  char pfx[64];
  auto prefix = [&](int p) -> const char* {
    if (!batch) return fn;
    snprintf(pfx, sizeof pfx, "%s: problem %d", fn, p);
    return pfx;
  };
  // every refusal before any work: the cameras, then the host-side rules per problem
  std::vector<LbbProb> hp(P);
  std::vector<GbbBig> hb;
  long long tN = 0, tObs = 0, tLm = 0, tKf = 0, tFix = 0, tG = 0, tS = 0, tWp = 0, tNz = 0;
  int mObs = 0, mLm = 0, mEl = 0, mBig = 0;
  for (int p = 0; p < P; ++p) {
    const plf_camera* c;
    if (plf_status st = plf_problem_camera(ctx, fn, seq, p, &c)) return st;
    const plf_lba_problem& pr = problems[p];
    if (plf_status st = lba_check_shape(ctx, prefix(p), &pr, global ? 4096 : 64)) return st;
    LbbProb& q = hp[p];
    q.nkf = pr.n_kf; q.npt = pr.n_pt; q.nls = pr.n_ls; q.npo = pr.n_pt_obs; q.nobs = pr.n_pt_obs + pr.n_ls_obs;
    q.nlm = pr.n_pt + pr.n_ls; q.N = 6 * pr.n_kf + 3 * pr.n_pt + 6 * pr.n_ls; q.nfix = pr.n_fixed;
    q.xo = tN; q.oo = tObs; q.lo = tLm; q.ko = tKf; q.fo = tFix; q.go = tG; q.so = tS;
    q.cam = LbaCam{c->fx, c->fy, c->cx, c->cy};
    if (q.nkf > 64) {   // n > 384: the tiled LDL^T (k_gbb_*)
      const long long nt = (6 * q.nkf + GBA_T - 1) / GBA_T;
      hb.push_back(GbbBig{p, q.nkf, q.so, q.go, q.xo, tWp, tNz});
      tWp += nt * GBA_T * GBA_T; tNz += nt * nt;
      mBig = std::max(mBig, 6 * q.nkf);
    }
    tN += q.N; tObs += q.nobs; tLm += q.nlm; tKf += q.nkf; tFix += q.nfix; tG += 6 * q.nkf; tS += 36LL * q.nkf * q.nkf;
    mObs = std::max(mObs, q.nobs); mLm = std::max(mLm, q.nlm); mEl = std::max(mEl, q.nkf + 3 * q.npt + 6 * q.nls);
  }
  const int nb = (int)hb.size();
  // one staged upload (inputs), one download (X, moved flags, control); the device work after them, the part zeroed
  // before the first pass (A, g_c, S, g_red, scal) last
  StagedLayout L;
  const size_t iProb = L.take_in(sizeof(LbbProb) * P), iX0 = L.take_in(8 * tN), iFT = L.take_in(128 * tFix);
  const size_t iLm = L.take_in(4 * tObs), iKf = L.take_in(4 * tObs), iZ = L.take_in(24 * tObs), iLs = L.take_in(4 * (tLm + P));
  const size_t iBig = L.take_in(sizeof(GbbBig) * nb);
  const size_t oX = L.take_out(8 * tN), oMv = L.take_out(tLm), oCtl = L.take_out(sizeof(LbbCtrl) * P);
  const size_t wT0 = L.take_work(128 * tKf), wFTi = L.take_work(128 * tFix), wJt = L.take_work(48 * tObs),
               wJx = L.take_work(48 * tObs), wWn = L.take_work(16 * tObs), wD = L.take_work(288 * tLm),
               wDi = L.take_work(288 * tLm), wGl = L.take_work(48 * tLm), wDxc = L.take_work(8 * tG), wDX = L.take_work(8 * tN);
  const size_t wWp = L.take_work(8 * tWp), wNz = L.take_work(tNz);
  const size_t wA = L.take_work(288 * tKf), wGc = L.take_work(48 * tKf), wS = L.take_work(8 * tS), wGr = L.take_work(8 * tG),
               wSc = L.take_work(64 * (size_t)P);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *pin, *dev;
  // the one-problem calls share their slot with plf_pose_graph, so that a context running plf_global_ba and
  // plf_pose_graph holds one allocation for the two dense systems, not two
  if (plf_status st = L.acquire(ctx, batch ? PLF_SCR_BA_BATCH : PLF_SCR_BA, &pin, &dev)) return st;
  for (int p = 0; p < P; ++p) {
    const plf_lba_problem& pr = problems[p];
    const LbbProb& q = hp[p];
    if (plf_status st = lba_gather(ctx, prefix(p), &pr, (int*)(pin + iLs) + q.lo + p, (int*)(pin + iLm) + q.oo, (int*)(pin + iKf) + q.oo,
                                   (double*)(pin + iZ) + 3 * q.oo))
      return st;
    double* X0 = (double*)(pin + iX0) + q.xo;
    if (q.nkf) memcpy(X0, pr.kf_pose, 48 * (size_t)q.nkf);
    if (q.npt) memcpy(X0 + 6 * q.nkf, pr.pt, 24 * (size_t)q.npt);
    if (q.nls) memcpy(X0 + 6 * q.nkf + 3 * q.npt, pr.ls, 48 * (size_t)q.nls);
    if (q.nfix) memcpy((double*)(pin + iFT) + 16 * q.fo, pr.fixed_T, 128 * (size_t)q.nfix);
  }
  memcpy(pin + iProb, hp.data(), sizeof(LbbProb) * P);
  if (nb) memcpy(pin + iBig, hb.data(), sizeof(GbbBig) * nb);
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
  uint8_t* const dout = dev + L.in;
  uint8_t* const dwork = dout + L.out;
  PLF_CUDA(ctx, cudaMemsetAsync(dwork + wA, 0, L.work - wA, cs));
  LbbDev b;
  b.prob = (const LbbProb*)(dev + iProb); b.ctrl = (LbbCtrl*)(dout + oCtl); b.P = P;
  b.X = (double*)(dout + oX); b.X0 = (double*)(dev + iX0); b.T0inv = (double*)(dwork + wT0);
  b.fixedT = (const double*)(dev + iFT); b.fixedTinv = (double*)(dwork + wFTi);
  b.obs_lm = (const int*)(dev + iLm); b.obs_kf = (const int*)(dev + iKf); b.obs_z = (const double*)(dev + iZ);
  b.lm_start = (const int*)(dev + iLs);
  b.Jt = (double*)(dwork + wJt); b.Jx = (double*)(dwork + wJx); b.Wn = (double*)(dwork + wWn);
  b.D = (double*)(dwork + wD); b.gl = (double*)(dwork + wGl); b.Dinv = (double*)(dwork + wDi);
  b.A = (double*)(dwork + wA); b.gc = (double*)(dwork + wGc); b.S = (double*)(dwork + wS); b.gred = (double*)(dwork + wGr);
  b.dxc = (double*)(dwork + wDxc); b.DX = (double*)(dwork + wDX); b.scal = (double*)(dwork + wSc); b.moved = dout + oMv;
  const GbbBig* dBig = (const GbbBig*)(dev + iBig);
  static_assert(sizeof(LbbCtrl) % sizeof(int) == 0, "gbb_view reads LbbCtrl::active as a strided int");
  const int* act = (const int*)((const uint8_t*)b.ctrl + offsetof(LbbCtrl, active));
  GbbLdlt gl{dBig, act, (int)(sizeof(LbbCtrl) / sizeof(int)), b.S, b.gred, b.dxc, b.DX, (double*)(dwork + wWp), dwork + wNz, {}};
  // one large problem (every plf_global_ba over 64 keyframes) passes its entry by value: no table load per CTA
  if (nb == 1) { gl.big = nullptr; gl.one = hb[0]; }
  // grids: (problem, chunks of 128 of the largest problem's count); the control kernels: one thread per problem
  auto chunks = [](int n) { return std::max(1, std::min(65535, (n + 127) / 128)); };
  const dim3 gObs(P, chunks(mObs)), gLm(P, chunks(mLm)), gEl(P, chunks(mEl));
  const int gCtl = (P + 127) / 128;
  const int q = opts->ref_quirks ? (global ? BAQ_GBA : BAQ_LBA) : 0;
  // the large problems' damping (42 n_kf elements) and zeroing (36 n_kf^2 + 48 n_kf doubles), gridded (chunk, problem)
  const dim3 gDamp((7 * mBig + 255) / 256, std::max(nb, 1));
  const dim3 gZero((unsigned)std::min<long long>(2048, ((long long)mBig * mBig + 255) / 256), std::max(nb, 1));
  k_lbb_prep<<<P, 128, 0, cs>>>(b, opts->lambda, std::max(opts->max_iters, 1));
  PLF_LAUNCH_CHECK(ctx);
  for (int r = 0; r < std::max(opts->max_iters, 1); ++r) {
    k_lbb_rows<<<gObs, 128, 0, cs>>>(b, r ? 1 : 0, q, opts->homog_th);
    PLF_LAUNCH_CHECK(ctx);
    k_lbb_lm_accum<<<gLm, 128, 0, cs>>>(b);
    PLF_LAUNCH_CHECK(ctx);
    if (r == 0) {
      k_lbb_kf_diagmax<<<P, 128, 0, cs>>>(b);
      PLF_LAUNCH_CHECK(ctx);
      if (q & BAQ_HMAX_INT) {
        k_gbb_hmax_int<<<P, 1024, 0, cs>>>(b);
        PLF_LAUNCH_CHECK(ctx);
      }
      if (global) k_gbb_first<<<gCtl, 128, 0, cs>>>(b, q);
      else k_lbb_first<<<gCtl, 128, 0, cs>>>(b, q);
    } else if (global) {
      k_gbb_test<<<gCtl, 128, 0, cs>>>(b, r, q, opts->min_error, opts->min_error_change);
    } else {
      k_lbb_test<<<gCtl, 128, 0, cs>>>(b, r, opts->min_error, opts->min_error_change);
    }
    PLF_LAUNCH_CHECK(ctx);
    const int swap = r == 0 && (q & BAQ_SWAP_COUPLING) ? 1 : 0;   // (g6)
    k_lbb_schur<<<gLm, 128, 0, cs>>>(b, swap);
    PLF_LAUNCH_CHECK(ctx);
    k_lbb_solve<<<P, 256, 0, cs>>>(b);
    PLF_LAUNCH_CHECK(ctx);
    if (nb) {
      k_gbb_damp<<<gDamp, 256, 0, cs>>>(b, dBig);
      PLF_LAUNCH_CHECK(ctx);
      if (plf_status st = gbb_ldlt(ctx, cs, gl, nb, mBig)) return st;
      k_gbb_zero<<<gZero, 256, 0, cs>>>(b, dBig);
      PLF_LAUNCH_CHECK(ctx);
    }
    k_lbb_backsub<<<gLm, 128, 0, cs>>>(b, swap);
    PLF_LAUNCH_CHECK(ctx);
    k_lbb_apply<<<gEl, 128, 0, cs>>>(b);
    PLF_LAUNCH_CHECK(ctx);
    k_lbb_step<<<gCtl, 128, 0, cs>>>(b, r, opts->lambda_k, opts->min_error_change);
    PLF_LAUNCH_CHECK(ctx);
  }
  k_lbb_moved<<<gLm, 128, 0, cs>>>(b);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in, dout, L.out, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  const LbbCtrl* ctl = (const LbbCtrl*)(pin + L.in + oCtl);
  int refused = -1;
  for (int p = 0; p < P; ++p) {
    const plf_lba_problem& pr = problems[p];
    const LbbProb& qp = hp[p];
    const LbbCtrl& c = ctl[p];
    if (c.zero_lm >= 0) {
      status[p] = PLF_ERR_INVALID;
      if (refused < 0) refused = p;
      continue;
    }
    const double* X = (const double*)(pin + L.in + oX) + qp.xo;
    if (qp.nkf) memcpy(pr.kf_pose, X, 48 * (size_t)qp.nkf);
    if (qp.npt) memcpy(pr.pt, X + 6 * qp.nkf, 24 * (size_t)qp.npt);
    if (qp.nls) memcpy(pr.ls, X + 6 * qp.nkf + 3 * qp.npt, 48 * (size_t)qp.nls);
    const uint8_t* m = pin + L.in + oMv + qp.lo;
    if (pr.pt_moved && qp.npt) memcpy(pr.pt_moved, m, qp.npt);
    if (pr.ls_moved && qp.nls) memcpy(pr.ls_moved, m + qp.npt, qp.nls);
    if (out) { out[p].iters = c.iters; out[p].err = c.err; out[p].lambda = c.lambda; }
    status[p] = PLF_OK;
  }
  if (refused >= 0) {
    const int l = ctl[refused].zero_lm, npt = hp[refused].npt;
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s landmark %d has a zero diagonal entry in its first-pass block (no row constrains it)",
                    prefix(refused), l < npt ? "point" : "line", l < npt ? l : l - npt);
  }
  return PLF_OK;
}

extern "C" plf_status plf_local_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* p, plf_lba_result* out) {
  if (!ctx || !opts || !p) return plf_fail(ctx, PLF_ERR_INVALID, "plf_local_ba: bad arguments");
  plf_status st;
  return lbb_run(ctx, opts, 1, p, nullptr, out, &st, false, false);
}

extern "C" plf_status plf_global_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* p, plf_lba_result* out) {
  if (!ctx || !opts || !p) return plf_fail(ctx, PLF_ERR_INVALID, "plf_global_ba: bad arguments");
  plf_status st;
  return lbb_run(ctx, opts, 1, p, nullptr, out, &st, true, false);
}

extern "C" plf_status plf_local_ba_batch(plf_ctx* ctx, const plf_lba_opts* opts, int n_problems, const plf_lba_problem* problems,
                                         const int32_t* seq, plf_lba_result* out, plf_status* status) {
  return lbb_run(ctx, opts, n_problems, problems, seq, out, status, false, true);
}

extern "C" plf_status plf_global_ba_batch(plf_ctx* ctx, const plf_lba_opts* opts, int n_problems, const plf_lba_problem* problems,
                                          const int32_t* seq, plf_lba_result* out, plf_status* status) {
  return lbb_run(ctx, opts, n_problems, problems, seq, out, status, true, true);
}

// Test hook (plslam_b200.h): the k_gbb_* chain on n caller matrices of mixed sizes, each as plf_debug_ldlt's path 0
extern "C" plf_status plf_debug_ldlt_batch(plf_ctx* ctx, int n, const int* n6, double* const* S, const double* const* g,
                                           double* const* x, uint8_t* const* nz) {
  const char* fn = "plf_debug_ldlt_batch";
  if (!ctx || n < 0 || (n && (!n6 || !S || !g || !x)) || n > 65535) return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  if (!n) return PLF_OK;
  std::vector<GbbBig> hb(n);
  long long tS = 0, tG = 0, tWp = 0, tNz = 0;
  int mx = 0;
  for (int i = 0; i < n; ++i) {
    if (n6[i] < 1 || n6[i] > 4096 || !S[i] || !g[i] || !x[i])
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: matrix %d: n6 = %d outside [1, 4096] or a NULL array", fn, i, n6[i]);
    const long long m = 6LL * n6[i], nt = (m + GBA_T - 1) / GBA_T;
    hb[i] = GbbBig{i, n6[i], tS, tG, tG, tWp, tNz};
    tS += m * m; tG += m; tWp += nt * GBA_T * GBA_T; tNz += nt * nt;
    mx = std::max(mx, (int)m);
  }
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  GbbBig* dBig = nullptr;
  GbbLdlt L{};
  double* dx = nullptr;
  uint8_t* dNz = nullptr;
  DevBufList scr;
  scr.add(dBig, n); scr.add(L.S, tS); scr.add(L.g, tG); scr.add(L.y, tG); scr.add(dx, tG); scr.add(L.Wp, tWp); scr.add(dNz, tNz);
  if (plf_status st = scr.carve(ctx, PLF_SCR_BA)) return st;
  L.big = dBig; L.x = dx; L.nz = dNz;
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dBig, hb.data(), sizeof(GbbBig) * n, cudaMemcpyHostToDevice, cs));
  for (int i = 0; i < n; ++i) {
    const size_t m = 6 * (size_t)n6[i];
    PLF_CUDA(ctx, cudaMemcpyAsync(L.S + hb[i].so, S[i], m * m * 8, cudaMemcpyHostToDevice, cs));
    PLF_CUDA(ctx, cudaMemcpyAsync(L.g + hb[i].go, g[i], m * 8, cudaMemcpyHostToDevice, cs));
  }
  PLF_CUDA(ctx, cudaMemsetAsync(dNz, 0, tNz, cs));
  if (plf_status st = gbb_ldlt(ctx, cs, L, n, mx)) return st;
  for (int i = 0; i < n; ++i) {
    const size_t m = 6 * (size_t)n6[i], nt = (m + GBA_T - 1) / GBA_T;
    PLF_CUDA(ctx, cudaMemcpyAsync(S[i], L.S + hb[i].so, m * m * 8, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaMemcpyAsync(x[i], dx + hb[i].xo, m * 8, cudaMemcpyDeviceToHost, cs));
    if (nz && nz[i]) PLF_CUDA(ctx, cudaMemcpyAsync(nz[i], dNz + hb[i].zo, nt * nt, cudaMemcpyDeviceToHost, cs));
  }
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}
