// Local bundle adjustment on the GPU (SURVEY §8(f) row f4).
//
// Replaces MapHandler::levMarquardtOptimizationLBA (src/mapHandler.cpp:1332-1989), the numerical core of
// MapHandler::localBundleAdjustment (:1220-1330): Levenberg-Marquardt over the local keyframes' poses (x_kf_w, se(3)
// vectors), the local 3-D points and the local 3-D line segments (two end points), with Cauchy-weighted scalar residuals
// (the norm of the point reprojection error / of the two end-point distances to the observed line).  The reference
// rebuilds a DENSE N x N Hessian every iteration and factors its sparse view with SimplicialLDLT; here the same normal
// equations are solved through the Schur complement on the landmarks - every observation couples ONE keyframe with ONE
// landmark, so the landmark block is block-diagonal (3x3 / 6x6) and each coupling block is rank one:
//   k_lba_rows      one thread per observation: residual, weight, the two Jacobian rows (:1384-1400 points, :1441-1503
//                   lines); accumulates the keyframe blocks A (6x6) / g_c and the error
//   k_lba_lm_accum  one thread per landmark: D = sum w Jx Jx^T, g_l (its observations are contiguous, in the reference's
//                   order), max |diagonal| for the initial lambda (:1543-1550)
//   k_lba_lm_schur  one thread per landmark: D' = D + lambda diag(D), D'^-1, and the reduced-system contributions
//                   S[a][b] -= w_b (y_a . Jx_b) Jt_a Jt_b^T, g_red[a] -= (y_a . g_l) Jt_a with y_a = w_a D'^-1 Jx_a
//   k_lba_solve     one CTA: S += A', dense LDL^T (no pivoting, as SimplicialLDLT) and the two triangular solves
//   k_lba_backsub   one thread per landmark: dx_l = D'^-1 (g_l - sum_a w_a Jx_a (Jt_a . dx_c[a]))
//   k_lba_apply     T <- T * inverse_se3(expmap_se3(dx)) / X += dx (:1558-1570), |dx|^2
// The host keeps the reference's control flow (first pass on the map's values, lambda schedule :1785-1803, stop tests
// :1775,:1805).  opts.ref_quirks selects between the reference as written and its evident intent for the four oddities
// documented in oracle/lba.c (division by the zero counters :1541, both line end points read from one block of X at
// stride 3 :1678-1679, the map's pose for line rows :1681, the literal clamp); oracle = oracle/lba.c.
//
// Global bundle adjustment (SURVEY §8(f), after f1-f5): plf_global_ba replaces MapHandler::levMarquardtOptimizationGBA
// (:2101-2699) with the same kernels and host loop over every keyframe but keyframe 0 and every landmark.  Its quirk set
// (g1-g6, oracle/gba.py) selects the reference's GBA oddities instead of LBA's, and a reduced system larger than 384
// (more than 64 keyframes) is factored by the tiled, multi-CTA LDL^T below (k_gba_*), whose trailing update runs on the
// FP64 tensor cores (DMMA) and skips the tiles of the panel that are exactly zero.
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
                                               // [4] first landmark with a zero diagonal entry in D (k_lba_lm_accum)
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
__device__ __forceinline__ void lba_xform(const double* T, const double* P, double* Q) {
  for (int i = 0; i < 3; ++i) Q[i] = T[4 * i] * P[0] + T[4 * i + 1] * P[1] + T[4 * i + 2] * P[2] + T[4 * i + 3];
}

// mode 0: first pass on the map's values (X0 / T0inv); mode 1: LM iteration on X; quirks: BAQ_* set
__global__ void __launch_bounds__(128) k_lba_rows(LbaDev d, LbaCam c, int mode, int quirks, double homog_th) {
  const int k = blockIdx.x * 128 + threadIdx.x;
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
      lba_xform(Ti, X + 6 * d.nkf + 3 * lm, Xwi);
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
      lba_xform(Ti, P, Pwi);
      lba_xform(Ti, Q, Qwi);
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

__global__ void __launch_bounds__(128) k_lba_lm_accum(LbaDev d) {
  const int l = blockIdx.x * 128 + threadIdx.x;
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

__global__ void k_lba_kf_diagmax(LbaDev d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
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
__global__ void __launch_bounds__(128) k_lba_lm_schur(LbaDev d, double lambda, int swap) {
  const int l = blockIdx.x * 128 + threadIdx.x;
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

// One CTA: S += A' (block diagonal, damped), g_red += g_c, dense LDL^T without pivoting, solve S dx_c = g_red.
__global__ void __launch_bounds__(256) k_lba_solve(LbaDev d, double lambda) {
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

__global__ void __launch_bounds__(128) k_lba_backsub(LbaDev d, int swap) {
  const int l = blockIdx.x * 128 + threadIdx.x;
  if (l >= d.nlm) return;
  const int dim = l < d.npt ? 3 : 6;
  const double* U = swap && l >= d.npt ? d.Jt : d.Jx;   // as k_lba_lm_schur
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

// |DX|^2 always; the step itself only when `apply`
__global__ void __launch_bounds__(128) k_lba_apply(LbaDev d, int apply) {
  const int i = blockIdx.x * 128 + threadIdx.x;
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

__global__ void k_lba_prep(LbaDev d, const double* fixedT, double* fixedTinv, int n_fixed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
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

__global__ void k_lba_moved(LbaDev d, uint8_t* pt_moved, uint8_t* ls_moved) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
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
// >= 2^31 (or of all of them).  One CTA; leaves the value in scal[3].
__global__ void __launch_bounds__(1024) k_gba_hmax_int(LbaDev d) {
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
// factorisation as k_lba_solve: per tile column k, k_gba_diag factors the diagonal tile in shared memory, k_gba_panel
// solves each tile below it (L_ik = S_ik L_kk^-T D_k^-1, keeping W_ik = L_ik D_k) and flags whether it is exactly zero,
// and k_gba_update subtracts W_ik L_jk^T from every trailing lower tile (i, j) whose two panel tiles are non-zero, on
// the FP64 tensor cores.  The substitutions run per tile (k_gba_fwd / k_gba_bwd) and skip the same zero tiles.  Tiles
// past n are padded with the identity; n_t = ceil(n / 64).
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

__global__ void __launch_bounds__(256) k_gba_damp(LbaDev d, double lambda) {   // k_lba_solve's prologue
  const int i = blockIdx.x * 256 + threadIdx.x, n = 6 * d.nkf;
  if (i < 36 * d.nkf) {
    const int kf = i / 36, r = (i % 36) / 6, cc = i % 6;
    double v = d.A[i];
    if (r == cc) v += lambda * v;
    d.S[(size_t)(6 * kf + r) * n + 6 * kf + cc] += v;
  } else if (i < 36 * d.nkf + n) {
    d.gred[i - 36 * d.nkf] += d.gc[i - 36 * d.nkf];
  }
}

__global__ void __launch_bounds__(256) k_gba_diag(LbaDev d, int k) {
  __shared__ double T[GBA_T * GBA_LD];
  const int n = 6 * d.nkf, r0 = GBA_T * k, tid = threadIdx.x;
  for (int e = tid; e < GBA_T * GBA_T; e += 256) {
    const int r = e >> 6, c = e & 63;
    T[r * GBA_LD + c] = r0 + r < n && r0 + c < n ? d.S[(size_t)(r0 + r) * n + r0 + c] : (r == c ? 1.0 : 0.0);
  }
  __syncthreads();
  for (int j = 0; j < GBA_T; ++j) {   // as k_lba_solve: after column j, T[i][j] = L_ij, T[j][j] = D_j
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

// one CTA per tile row i > k; dynamic shared memory 2 x 64 x GBA_LD doubles
__global__ void __launch_bounds__(256) k_gba_panel(LbaDev d, double* Wp, uint8_t* nz, int k, int nt) {
  extern __shared__ double gsm[];
  double* L = gsm;
  double* Z = gsm + GBA_T * GBA_LD;
  const int n = 6 * d.nkf, i = k + 1 + blockIdx.x, r0 = GBA_T * i, c0 = GBA_T * k, tid = threadIdx.x;
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

// S_ij -= W_ik L_jk^T for the trailing lower tiles k < j <= i, one CTA per tile (blockIdx.x enumerates (i, j) row by
// row).  8 warps; warp w owns rows 16 (w / 2) .. +16 and columns 32 (w % 2) .. +32 of the tile (4 m16n8 accumulators).
constexpr int GBA_KC = 32, GBA_SLD = 36;   // k chunk; shared row stride (conflict-free fragment loads per half warp)
__global__ void __launch_bounds__(256) k_gba_update(LbaDev d, const double* Wp, const uint8_t* nz, int k, int nt) {
  const int t = blockIdx.x;
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
__global__ void __launch_bounds__(256) k_gba_fwd(LbaDev d, const uint8_t* nz, int k, int nt) {
  __shared__ double L[GBA_T * GBA_LD], y[GBA_T];
  const int n = 6 * d.nkf, b = blockIdx.x, i = k + b, r0 = GBA_T * k, tid = threadIdx.x;
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

__global__ void k_gba_dscale(LbaDev d) {   // z = y / D
  const int i = blockIdx.x * blockDim.x + threadIdx.x, n = 6 * d.nkf;
  if (i < n) d.gred[i] = d.dxc[i] / d.S[(size_t)i * n + i];
}

// backward substitution step k (k = n_t - 1 .. 0): every CTA solves x_k = L_kk^-T z_k, CTA 0 stores it in dxc and DX,
// CTA b > 0 subtracts L_kj^T x_k from z_j (j = b - 1) when that tile is non-zero
__global__ void __launch_bounds__(256) k_gba_bwd(LbaDev d, const uint8_t* nz, int k, int nt) {
  __shared__ double L[GBA_T * GBA_LD], x[GBA_T], part[4][GBA_T];
  const int n = 6 * d.nkf, b = blockIdx.x, r0 = GBA_T * k, tid = threadIdx.x;
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

// The tiled factorisation and the two substitutions (see k_gba_diag), shared by plf_global_ba and plf_pose_graph.  The
// kernels read only the fields of LbaDev set here.
plf_status plf_ldlt_tiled(plf_ctx* ctx, cudaStream_t cs, int n6, double* S, double* g, double* y, double* x, double* Wp,
                          uint8_t* nz) {
  static_assert(GBA_T == PLF_LDLT_TILE, "plf_internal.h states the tile size");
  LbaDev d{};
  d.nkf = n6; d.S = S; d.gred = g; d.dxc = y; d.DX = x;
  const int n = 6 * n6, nt = (n + GBA_T - 1) / GBA_T;
  const int smem = 2 * GBA_T * GBA_LD * 8;
  PLF_CUDA(ctx, cudaFuncSetAttribute(k_gba_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  for (int k = 0; k < nt; ++k) {
    k_gba_diag<<<1, 256, 0, cs>>>(d, k);
    PLF_LAUNCH_CHECK(ctx);
    const int m = nt - k - 1;
    if (!m) break;
    k_gba_panel<<<m, 256, smem, cs>>>(d, Wp, nz, k, nt);
    PLF_LAUNCH_CHECK(ctx);
    k_gba_update<<<m * (m + 1) / 2, 256, 0, cs>>>(d, Wp, nz, k, nt);
    PLF_LAUNCH_CHECK(ctx);
  }
  for (int k = 0; k < nt; ++k) {
    k_gba_fwd<<<nt - k, 256, 0, cs>>>(d, nz, k, nt);
    PLF_LAUNCH_CHECK(ctx);
  }
  k_gba_dscale<<<(n + 255) / 256, 256, 0, cs>>>(d);
  PLF_LAUNCH_CHECK(ctx);
  for (int k = nt - 1; k >= 0; --k) {
    k_gba_bwd<<<k + 1, 256, 0, cs>>>(d, nz, k, nt);
    PLF_LAUNCH_CHECK(ctx);
  }
  return PLF_OK;
}

// The host loop of both routines: the reference's control flow, on the device kernels above.  `global` selects
// levMarquardtOptimizationGBA (:2101-2699) over levMarquardtOptimizationLBA (:1332-1989): its quirk set, its error
// normalisation in the LM iterations and up to 4096 keyframes (the blocked factorisation beyond n = 384).  Both refuse a
// landmark whose first-pass block D has an exactly zero diagonal entry, before any step: the reference would factor a
// zero pivot (its SimplicialLDLT's failure is not checked) and the landmark, then every keyframe observing it, would
// turn NaN.  A landmark without observations is refused by name first; the rest by one flag read with the first pass.
static plf_status ba_run(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* p, plf_lba_result* out, bool global) {
  const char* fn = global ? "plf_global_ba" : "plf_local_ba";
  if (!ctx || !opts || !p || p->n_kf < 0 || p->n_pt < 0 || p->n_ls < 0 || p->n_pt_obs < 0 || p->n_ls_obs < 0 || p->n_fixed < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  const int nkf = p->n_kf, npt = p->n_pt, nls = p->n_ls, npo = p->n_pt_obs, nlo = p->n_ls_obs, nobs = npo + nlo, nlm = npt + nls;
  const int N = 6 * nkf + 3 * npt + 6 * nls, n = 6 * nkf;
  if (nobs == 0 || N == 0) return plf_fail(ctx, PLF_ERR_INVALID, "%s: empty problem (the reference returns -1, :1324-1328)", fn);
  const int kf_cap = global ? 4096 : 64;
  if (nkf > kf_cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d keyframes (limit %d)", fn, nkf, kf_cap);
  if ((nkf && !p->kf_pose) || (npt && !p->pt) || (nls && !p->ls) || (npo && (!p->pt_obs_lm || !p->pt_obs_kf || !p->pt_obs_xy)) ||
      (nlo && (!p->ls_obs_lm || !p->ls_obs_kf || !p->ls_obs_le)) || (p->n_fixed && !p->fixed_T))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: null array", fn);
  // observations are grouped per landmark in non-decreasing landmark order (how the reference builds its lists, :1249-1277)
  std::vector<int> lm_start(nlm + 1, 0), h_lm(nobs), h_kf(nobs);
  std::vector<double> h_z((size_t)nobs * 3, 0.0);
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
    else { h_z[3 * (size_t)k] = p->pt_obs_xy[2 * (size_t)k]; h_z[3 * (size_t)k + 1] = p->pt_obs_xy[2 * (size_t)k + 1]; }
  }
  for (int l = 0; l < nlm; ++l)   // its landmark block would be zero
    if (!lm_start[l + 1])
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s landmark %d has no observation", fn, l < npt ? "point" : "line", l < npt ? l : l - npt);
  for (int l = 0; l < nlm; ++l) lm_start[l + 1] += lm_start[l];
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const bool blocked = n > 384;   // k_lba_solve (one CTA, one launch) up to 64 keyframes, the tiled LDL^T beyond
  const int nt = (n + GBA_T - 1) / GBA_T;
  LbaDev d;
  d.nkf = nkf; d.npt = npt; d.nls = nls; d.N = N; d.npo = npo; d.nlo = nlo; d.nobs = nobs; d.nlm = nlm;
  double *dFT, *dFTi, *dZ, *dWp;
  int *dLm, *dKf, *dLs;
  uint8_t *dPm, *dLmv, *dNz;
  DevBufList scr;
  scr.add(d.X, N); scr.add(d.X0, N); scr.add(d.T0inv, (size_t)std::max(nkf, 1) * 16);
  scr.add(dFT, (size_t)std::max(p->n_fixed, 1) * 16); scr.add(dFTi, (size_t)std::max(p->n_fixed, 1) * 16);
  scr.add(dLm, nobs); scr.add(dKf, nobs); scr.add(dZ, (size_t)nobs * 3); scr.add(dLs, (size_t)nlm + 1);
  scr.add(d.Jt, (size_t)nobs * 6); scr.add(d.Jx, (size_t)nobs * 6); scr.add(d.Wn, (size_t)nobs * 2);
  scr.add(d.D, (size_t)std::max(nlm, 1) * 36); scr.add(d.gl, (size_t)std::max(nlm, 1) * 6); scr.add(d.Dinv, (size_t)std::max(nlm, 1) * 36);
  scr.add(d.A, (size_t)std::max(nkf, 1) * 36); scr.add(d.gc, (size_t)std::max(nkf, 1) * 6);
  scr.add(d.S, std::max((size_t)n * n, (size_t)1)); scr.add(d.gred, (size_t)std::max(n, 1)); scr.add(d.dxc, (size_t)std::max(n, 1));
  scr.add(d.DX, N); scr.add(d.scal, 8);
  scr.add(dPm, std::max(npt, 1)); scr.add(dLmv, std::max(nls, 1));
  scr.add(dWp, blocked ? (size_t)nt * GBA_T * GBA_T : 1); scr.add(dNz, blocked ? (size_t)nt * nt : 1);
  if (plf_status st = scr.carve(ctx, PLF_SCR_BA)) return st;
  d.fixedTinv = dFTi;
  d.obs_lm = dLm; d.obs_kf = dKf; d.obs_z = dZ; d.lm_start = dLs;
  cudaStream_t cs = ctx->stream;
  std::vector<double> hX(N);
  for (int i = 0; i < 6 * nkf; ++i) hX[i] = p->kf_pose[i];
  for (int i = 0; i < 3 * npt; ++i) hX[6 * nkf + i] = p->pt[i];
  for (int i = 0; i < 6 * nls; ++i) hX[6 * nkf + 3 * npt + i] = p->ls[i];
  PLF_CUDA(ctx, cudaMemcpyAsync(d.X, hX.data(), (size_t)N * 8, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(d.X0, hX.data(), (size_t)N * 8, cudaMemcpyHostToDevice, cs));
  if (p->n_fixed) PLF_CUDA(ctx, cudaMemcpyAsync(dFT, p->fixed_T, (size_t)p->n_fixed * 128, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dLm, h_lm.data(), (size_t)nobs * 4, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dKf, h_kf.data(), (size_t)nobs * 4, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dZ, h_z.data(), (size_t)nobs * 24, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dLs, lm_start.data(), (size_t)(nlm + 1) * 4, cudaMemcpyHostToDevice, cs));
  k_lba_prep<<<(std::max(nkf, p->n_fixed) + 63) / 64 + 1, 64, 0, cs>>>(d, dFT, dFTi, p->n_fixed);
  PLF_LAUNCH_CHECK(ctx);
  const LbaCam cam = {ctx->cam.fx, ctx->cam.fy, ctx->cam.cx, ctx->cam.cy};
  const int q = opts->ref_quirks ? (global ? BAQ_GBA : BAQ_LBA) : 0;
  double lambda = opts->lambda;
  double h_scal[5];
  // builds the normal equations of `mode` and leaves err / Hmax in scal
  auto build = [&](int mode) -> plf_status {
    PLF_CUDA(ctx, cudaMemsetAsync(d.A, 0, (size_t)std::max(nkf, 1) * 288, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(d.gc, 0, (size_t)std::max(nkf, 1) * 48, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(d.S, 0, std::max((size_t)n * n, (size_t)1) * 8, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(d.gred, 0, (size_t)std::max(n, 1) * 8, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(d.scal, 0, 64, cs));
    k_lba_rows<<<(nobs + 127) / 128, 128, 0, cs>>>(d, cam, mode, q, opts->homog_th);
    PLF_LAUNCH_CHECK(ctx);
    k_lba_lm_accum<<<(nlm + 127) / 128, 128, 0, cs>>>(d);
    PLF_LAUNCH_CHECK(ctx);
    if (mode == 0 && nkf) {
      k_lba_kf_diagmax<<<(6 * nkf + 63) / 64, 64, 0, cs>>>(d);
      PLF_LAUNCH_CHECK(ctx);
    }
    if (mode == 0 && (q & BAQ_HMAX_INT)) {
      k_gba_hmax_int<<<1, 1024, 0, cs>>>(d);
      PLF_LAUNCH_CHECK(ctx);
    }
    PLF_CUDA(ctx, cudaMemcpyAsync(h_scal, d.scal, 40, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    return PLF_OK;
  };
  // the blocked factorisation and the two substitutions of S dx_c = g_red (see k_gba_diag)
  auto solve_blocked = [&]() -> plf_status {
    k_gba_damp<<<(36 * nkf + n + 255) / 256, 256, 0, cs>>>(d, lambda);
    PLF_LAUNCH_CHECK(ctx);
    return plf_ldlt_tiled(ctx, cs, nkf, d.S, d.gred, d.dxc, d.DX, dWp, dNz);
  };
  // solves the damped system and (optionally) applies the step; leaves |DX| in *dx_norm.  swap: (g6), first pass only
  auto solve = [&](int apply, int swap, double* dx_norm) -> plf_status {
    k_lba_lm_schur<<<(nlm + 127) / 128, 128, 0, cs>>>(d, lambda, swap);
    PLF_LAUNCH_CHECK(ctx);
    if (blocked) {
      plf_status s = solve_blocked();
      if (s) return s;
    } else if (nkf) {
      k_lba_solve<<<1, 256, 0, cs>>>(d, lambda);
      PLF_LAUNCH_CHECK(ctx);
    }
    k_lba_backsub<<<(nlm + 127) / 128, 128, 0, cs>>>(d, swap);
    PLF_LAUNCH_CHECK(ctx);
    k_lba_apply<<<(nkf + (N - 6 * nkf) + 127) / 128, 128, 0, cs>>>(d, apply);
    PLF_LAUNCH_CHECK(ctx);
    PLF_CUDA(ctx, cudaMemcpyAsync(h_scal, d.scal, 32, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    *dx_norm = sqrt(h_scal[1]);
    return PLF_OK;
  };
  plf_status st;
  // ---- first pass on the map's values (LBA :1352-1541, GBA :2117-2356), lambda *= Hmax (:1543-1550, :2358-2365), first
  // step applied unconditionally
  if ((st = build(0))) return st;
  unsigned long long zero_flag;
  memcpy(&zero_flag, &h_scal[4], 8);
  if (zero_flag) {
    const int l = nlm - (int)zero_flag;
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s landmark %d has a zero diagonal entry in its first-pass block (no row constrains it)",
                    fn, l < npt ? "point" : "line", l < npt ? l : l - npt);
  }
  double err = h_scal[0];
  volatile int never_incremented = 0;   // Npt_obs + Nls_obs of the reference
  if (q & BAQ_FIRST_ERR0) err /= (double)never_incremented;   // (q1) :1541, (g1) :2356
  else err /= (double)nobs;
  double Hmax;
  if (q & BAQ_HMAX_INT) Hmax = h_scal[3];   // (g2)
  else { unsigned long long bits; memcpy(&bits, &h_scal[2], 8); memcpy(&Hmax, &bits, 8); }
  lambda *= Hmax;
  double dxn = 0.0;
  if ((st = solve(1, (q & BAQ_SWAP_COUPLING) ? 1 : 0, &dxn))) return st;
  double err_prev = err;
  int iters;
  for (iters = 1; iters < opts->max_iters; ++iters) {
    if ((st = build(1))) return st;
    if (q & BAQ_ITER_ERR0) err = h_scal[0] / (double)never_incremented;                           // (g3) :2635
    else if (global) err = h_scal[0] / (double)nobs;
    else err = h_scal[0] / (double)(npt + nls);                                                  // :1773
    if (fabs(err - err_prev) < opts->min_error_change || err < opts->min_error) break;           // :1775, :2637
    const bool grew = err > err_prev;
    if ((st = solve(grew ? 0 : 1, 0, &dxn))) return st;                                          // :1777-1803, :2639-2665
    if (grew) lambda /= opts->lambda_k; else lambda *= opts->lambda_k;
    if (dxn < opts->min_error_change) break;                                                     // :1805, :2667
    err_prev = err;
  }
  k_lba_moved<<<(nlm + 127) / 128, 128, 0, cs>>>(d, dPm, dLmv);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(hX.data(), d.X, (size_t)N * 8, cudaMemcpyDeviceToHost, cs));
  if (p->pt_moved && npt) PLF_CUDA(ctx, cudaMemcpyAsync(p->pt_moved, dPm, (size_t)npt, cudaMemcpyDeviceToHost, cs));
  if (p->ls_moved && nls) PLF_CUDA(ctx, cudaMemcpyAsync(p->ls_moved, dLmv, (size_t)nls, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  for (int i = 0; i < 6 * nkf; ++i) p->kf_pose[i] = hX[i];
  for (int i = 0; i < 3 * npt; ++i) p->pt[i] = hX[6 * nkf + i];
  for (int i = 0; i < 6 * nls; ++i) p->ls[i] = hX[6 * nkf + 3 * npt + i];
  if (out) { out->iters = iters; out->err = err; out->lambda = lambda; }
  return PLF_OK;
}

extern "C" plf_status plf_local_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* p, plf_lba_result* out) {
  return ba_run(ctx, opts, p, out, false);
}

extern "C" plf_status plf_global_ba(plf_ctx* ctx, const plf_lba_opts* opts, const plf_lba_problem* p, plf_lba_result* out) {
  return ba_run(ctx, opts, p, out, true);
}
