// Robust (Cauchy-weighted) 6-DoF point+line Gauss-Newton pose refinement (SURVEY §8 a8, a9).
//
// Replaces StVO::StereoFrameHandler::optimizePose (app/plslam_dataset.cpp:128, src/mapHandler.cpp:780),
// following its in-tree twin MapHandler::computeRelativePoseRobustGN (src/mapHandler.cpp:3566-3957;
// rows :3331-3426, normalise :3432, stop :3434/:3441, solve :3437-3438, update :3439, gate :3451-3482).
// se(3) helpers: stvo-pl auxiliar (SURVEY Appendix A.4), twist ordering [t; w] (src/mapHandler.cpp:3513-3514).
//
// One CTA (128 threads) per frame pair; many frame pairs per launch (the front-end's batch, plf_gn_pose_batch, the
// loop-closure checks of plf_loop_closure_pose_batch; plf_gn_pose is a batch of one).  Each thread strides over the
// feature rows, accumulates the 21 upper-triangular entries of J^T W J, the 6 of J^T W r, the error and the
// row count in fp64 registers; a warp-shuffle butterfly + one shared-memory hop reduces them; thread 0
// solves the 6x6 system with a column-pivoting Householder QR (same semantics as Eigen's
// ColPivHouseholderQR::solve) and updates T in shared memory.  The work is latency-bound (<= ~2k rows x
// <= 15 iterations); no dense contraction, tensor cores are not applicable.  fp64 throughout, as the
// reference.  Summation order differs from the sequential CPU loop (tree vs sequential), so results agree
// to ~1e-12 relative, not bit-for-bit; the parity bar for this stage is 1e-4 on the se(3) log.
#include <float.h>

#include "plf_internal.h"
#include "plf_se3.cuh"

#define GN_THREADS 128
#define GN_NACC 29  // 21 (H upper) + 6 (g) + e + N

struct GnCam {
  double fx, fy, cx, cy;
};

__device__ __forceinline__ void gn_jac6(double fgz2, double gx, double gy, double gz, double ax, double ay,
                                        double* J) {
  J[0] = +fgz2 * ax * gz;
  J[1] = +fgz2 * ay * gz;
  J[2] = -fgz2 * (gx * ax + gy * ay);
  J[3] = -fgz2 * (gx * gy * ax + gy * gy * ay + gz * gz * ay);
  J[4] = +fgz2 * (gx * gx * ax + gz * gz * ax + gx * gy * ay);
  J[5] = +fgz2 * (gx * gz * ay - gy * gz * ax);
}

__device__ __forceinline__ double gn_point_res(const GnCam& c, const double* T, const double* P,
                                               const double* obs, double* e2, double* Pc) {
  d_transform(T, P, Pc);
  e2[0] = (c.cx + c.fx * Pc[0] / Pc[2]) - obs[0];
  e2[1] = (c.cy + c.fy * Pc[1] / Pc[2]) - obs[1];
  return sqrt(e2[0] * e2[0] + e2[1] * e2[1]);
}

__device__ __forceinline__ double gn_line_res(const GnCam& c, const double* T, const double* sP,
                                              const double* eP, const double* l, double* e2, double* sPc,
                                              double* ePc) {
  d_transform(T, sP, sPc);
  d_transform(T, eP, ePc);
  const double sx = c.cx + c.fx * sPc[0] / sPc[2], sy = c.cy + c.fy * sPc[1] / sPc[2];
  const double ex = c.cx + c.fx * ePc[0] / ePc[2], ey = c.cy + c.fy * ePc[1] / ePc[2];
  e2[0] = l[0] * sx + l[1] * sy + l[2];
  e2[1] = l[0] * ex + l[1] * ey + l[2];
  return sqrt(e2[0] * e2[0] + e2[1] * e2[1]);
}

__device__ __forceinline__ void gn_add_row(double* acc, const double* J, double r, double w) {
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const double ja = J[a] * w;
#pragma unroll
    for (int b = a; b < 6; ++b) acc[k++] += ja * J[b];
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) acc[21 + a] += J[a] * r * w;
  acc[27] += r * r * w;
  acc[28] += 1.0;
}

// ---- small dense helpers (single thread) ---------------------------------------------------------
__device__ void d_colpiv_qr_solve6(const double* Hin, const double* gin, double* x) {
  const int n = 6;
  double A[36], b[6], Rd[6];
  int perm[6];
  for (int i = 0; i < 36; ++i) A[i] = Hin[i];
  for (int i = 0; i < 6; ++i) {
    b[i] = gin[i];
    perm[i] = i;
  }
  double maxpivot = 0;
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double best = -1;
    for (int j = k; j < n; ++j) {
      double s = 0;
      for (int i = k; i < n; ++i) s += A[n * i + j] * A[n * i + j];
      if (s > best) {
        best = s;
        piv = j;
      }
    }
    if (piv != k) {
      for (int i = 0; i < n; ++i) {
        const double t = A[n * i + k];
        A[n * i + k] = A[n * i + piv];
        A[n * i + piv] = t;
      }
      const int t = perm[k];
      perm[k] = perm[piv];
      perm[piv] = t;
    }
    const double c0 = A[n * k + k];
    double tail = 0;
    for (int i = k + 1; i < n; ++i) tail += A[n * i + k] * A[n * i + k];
    double beta, tau, v[6];
    if (tail == 0) {
      tau = 0;
      beta = c0;
      for (int i = k + 1; i < n; ++i) v[i] = 0;
    } else {
      beta = sqrt(c0 * c0 + tail);
      if (c0 >= 0) beta = -beta;
      for (int i = k + 1; i < n; ++i) v[i] = A[n * i + k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    v[k] = 1;
    for (int j = k + 1; j < n; ++j) {
      double s = 0;
      for (int i = k; i < n; ++i) s += v[i] * A[n * i + j];
      s *= tau;
      for (int i = k; i < n; ++i) A[n * i + j] -= s * v[i];
    }
    double s = 0;
    for (int i = k; i < n; ++i) s += v[i] * b[i];
    s *= tau;
    for (int i = k; i < n; ++i) b[i] -= s * v[i];
    A[n * k + k] = beta;
    Rd[k] = beta;
    if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
  }
  int rank = 0;
  for (int k = 0; k < n; ++k)
    if (fabs(Rd[k]) > maxpivot * (DBL_EPSILON * n)) rank++;
  double y[6] = {0, 0, 0, 0, 0, 0};
  for (int i = rank - 1; i >= 0; --i) {
    double s = b[i];
    for (int j = i + 1; j < rank; ++j) s -= A[n * i + j] * y[j];
    y[i] = s / A[n * i + i];
  }
  for (int j = 0; j < n; ++j) x[perm[j]] = (j < rank) ? y[j] : 0.0;
}

__device__ void d_inverse6(const double* Ain, double* I) {
  const int n = 6;
  double A[36];
  for (int i = 0; i < 36; ++i) {
    A[i] = Ain[i];
    I[i] = (i % 7 == 0) ? 1.0 : 0.0;
  }
  for (int k = 0; k < n; ++k) {
    int p = k;
    for (int i = k + 1; i < n; ++i)
      if (fabs(A[n * i + k]) > fabs(A[n * p + k])) p = i;
    if (p != k)
      for (int j = 0; j < n; ++j) {
        double t = A[n * k + j];
        A[n * k + j] = A[n * p + j];
        A[n * p + j] = t;
        t = I[n * k + j];
        I[n * k + j] = I[n * p + j];
        I[n * p + j] = t;
      }
    const double id = 1.0 / A[n * k + k];
    for (int j = 0; j < n; ++j) {
      A[n * k + j] *= id;
      I[n * k + j] *= id;
    }
    for (int i = 0; i < n; ++i) {
      if (i == k) continue;
      const double f = A[n * i + k];
      if (f == 0) continue;
      for (int j = 0; j < n; ++j) {
        A[n * i + j] -= f * A[n * k + j];
        I[n * i + j] -= f * I[n * k + j];
      }
    }
  }
}

// cams: optional per-problem cameras (a batch of several calibrations); null = launch_cam for every problem.
// active: optional per-problem flags; a problem whose flag is 0 is skipped (nothing read or written); null = all run.
// prm: optional per-problem settings, whose gn replaces o.
__global__ void __launch_bounds__(GN_THREADS) k_gn_pose(const GnProblem* __restrict__ probs, GnCam launch_cam,
                                                         const PlfPairCam* __restrict__ cams,
                                                         const int* __restrict__ active, plf_gn_opts o,
                                                         const PlfPairPrm* __restrict__ prm) {
  if (active && !active[blockIdx.x]) return;
  if (prm) o = prm[blockIdx.x].gn;
  const GnProblem P = probs[blockIdx.x];
  GnCam cam = launch_cam;
  if (cams) {
    const PlfPairCam q = cams[blockIdx.x];
    cam = GnCam{q.fx, q.fy, q.cx, q.cy};
  }
  const int np = P.np_ptr ? *P.np_ptr : P.np;
  const int nl = P.nl_ptr ? *P.nl_ptr : P.nl;
  __shared__ double sT[16];
  __shared__ double sred[GN_THREADS / 32][GN_NACC];
  __shared__ double sH[36], sg[6];
  __shared__ double s_e, s_errprev;
  __shared__ int s_stop;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < 16) sT[tid] = P.T_init ? P.T_init[tid] : ((tid % 5 == 0) ? 1.0 : 0.0);
  if (tid == 0) {
    s_errprev = 999999999.9;
    s_e = 0;
    for (int i = 0; i < 36; ++i) sH[i] = 0;
  }
  __syncthreads();
  int iters[2] = {0, 0};
  for (int stage = 0; stage < 2; ++stage) {
    const int max_it = stage == 0 ? o.max_iters : o.max_iters_ref;
    for (int it = 0; it < max_it; ++it) {
      double T[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) T[i] = sT[i];
      double acc[GN_NACC];
#pragma unroll
      for (int i = 0; i < GN_NACC; ++i) acc[i] = 0.0;
      for (int i = tid; i < np; i += GN_THREADS) {
        if (!P.inl_p[i]) continue;
        double e2[2], Pc[3], J[6];
        const double r = gn_point_res(cam, T, P.P + 3 * (size_t)i, P.obs + 2 * (size_t)i, e2, Pc);
        const double fgz2 = cam.fx / fmax(o.homog_th, Pc[2] * Pc[2]);
        gn_jac6(fgz2, Pc[0], Pc[1], Pc[2], e2[0], e2[1], J);
        const double d = fmax(o.homog_th, r);
#pragma unroll
        for (int k = 0; k < 6; ++k) J[k] = J[k] / d;
        gn_add_row(acc, J, r, 1.0 / (1.0 + r * r));
      }
      for (int i = tid; i < nl; i += GN_THREADS) {
        if (!P.inl_l[i]) continue;
        double e2[2], sPc[3], ePc[3], Js[6], Je[6], J[6];
        const double* l = P.le + 3 * (size_t)i;
        const double r = gn_line_res(cam, T, P.sP + 3 * (size_t)i, P.eP + 3 * (size_t)i, l, e2, sPc, ePc);
        gn_jac6(cam.fx / fmax(o.homog_th, sPc[2] * sPc[2]), sPc[0], sPc[1], sPc[2], l[0], l[1], Js);
        gn_jac6(cam.fx / fmax(o.homog_th, ePc[2] * ePc[2]), ePc[0], ePc[1], ePc[2], l[0], l[1], Je);
        const double d = fmax(o.homog_th, r);
#pragma unroll
        for (int k = 0; k < 6; ++k) J[k] = (Js[k] * e2[0] + Je[k] * e2[1]) / d;
        gn_add_row(acc, J, r, 1.0 / (1.0 + r * r));
      }
      // warp butterfly, then across warps through shared memory
#pragma unroll
      for (int i = 0; i < GN_NACC; ++i) {
        double v = acc[i];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, off);
        if (lane == 0) sred[wid][i] = v;
      }
      __syncthreads();
      if (tid == 0) {
        double tot[GN_NACC];
        for (int i = 0; i < GN_NACC; ++i) {
          double v = 0;
          for (int w = 0; w < GN_THREADS / 32; ++w) v += sred[w][i];
          tot[i] = v;
        }
        int k = 0;
        for (int a = 0; a < 6; ++a)
          for (int b = a; b < 6; ++b) {
            sH[6 * a + b] = tot[k];
            sH[6 * b + a] = tot[k];
            ++k;
          }
        for (int a = 0; a < 6; ++a) sg[a] = tot[21 + a];
        const double e = tot[27] / tot[28];
        s_e = e;
        int stop = 0;
        if (fabs(e - s_errprev) < o.eps_change || e < o.eps_err) {
          stop = 1;
        } else {
          double dx[6];
          d_colpiv_qr_solve6(sH, sg, dx);
          d_update_pose(sT, dx);
          double nrm = 0;
          for (int a = 0; a < 6; ++a) nrm += dx[a] * dx[a];
          if (sqrt(nrm) < o.eps_step)
            stop = 2;
          else
            s_errprev = e;
        }
        s_stop = stop;
      }
      __syncthreads();
      const int stop = s_stop;
      if (stop != 1) iters[stage] = it + 1; else iters[stage] = it;
      if (stop) break;
    }
    __syncthreads();
    if (stage == 0) {
      // chi2(2 dof, 95%) gate on the stage-1 pose (:3451-3482)
      double T[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) T[i] = sT[i];
      const double gate = sqrt(7.815);
      for (int i = tid; i < np; i += GN_THREADS) {
        if (!P.inl_p[i]) continue;
        double e2[2], Pc[3];
        if (gn_point_res(cam, T, P.P + 3 * (size_t)i, P.obs + 2 * (size_t)i, e2, Pc) > gate) P.inl_p[i] = 0;
      }
      for (int i = tid; i < nl; i += GN_THREADS) {
        if (!P.inl_l[i]) continue;
        double e2[2], a[3], b[3];
        if (gn_line_res(cam, T, P.sP + 3 * (size_t)i, P.eP + 3 * (size_t)i, P.le + 3 * (size_t)i, e2, a, b) > gate)
          P.inl_l[i] = 0;
      }
      __syncthreads();
    }
  }
  // inlier counts
  int cp = 0, cl = 0;
  for (int i = tid; i < np; i += GN_THREADS) cp += P.inl_p[i] != 0;
  for (int i = tid; i < nl; i += GN_THREADS) cl += P.inl_l[i] != 0;
  for (int off = 16; off > 0; off >>= 1) {
    cp += __shfl_xor_sync(0xFFFFFFFFu, cp, off);
    cl += __shfl_xor_sync(0xFFFFFFFFu, cl, off);
  }
  __shared__ int scnt[GN_THREADS / 32][2];
  if (lane == 0) {
    scnt[wid][0] = cp;
    scnt[wid][1] = cl;
  }
  __syncthreads();
  if (tid == 0) {
    plf_pose_result* out = P.out;
    for (int i = 0; i < 16; ++i) out->T[i] = sT[i];
    d_logmap(sT, out->x);
    d_inverse6(sH, out->cov);
    out->err = s_e;
    out->iters1 = iters[0];
    out->iters2 = iters[1];
    int a = 0, b = 0;
    for (int w = 0; w < GN_THREADS / 32; ++w) {
      a += scnt[w][0];
      b += scnt[w][1];
    }
    out->n_inliers_pt = a;
    out->n_inliers_ls = b;
  }
}

plf_gn_opts plf_gn_opts_from_params(const plf_params& p) {
  plf_gn_opts o;
  o.homog_th = p.homog_th;
  o.max_iters = p.max_iters;
  o.max_iters_ref = p.max_iters_ref;
  o.eps_err = p.min_error;
  o.eps_change = p.min_error_change;
  o.eps_step = DBL_EPSILON;
  return o;
}

plf_status plf_launch_gn(plf_ctx* ctx, cudaStream_t cs, const GnProblem* d_probs, int nprob, const plf_gn_opts& o,
                         const PlfPairCam* d_cams, const int* d_active, const PlfPairPrm* d_prm) {
  if (nprob <= 0) return PLF_OK;
  GnCam c = {ctx->cam.fx, ctx->cam.fy, ctx->cam.cx, ctx->cam.cy};
  k_gn_pose<<<nprob, GN_THREADS, 0, cs>>>(d_probs, c, d_cams, d_active, o, d_prm);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

namespace {

// plf_gn_pose's host-side rules for one problem.
bool gn_args_ok(const plf_gn_problem& q) {
  return q.np >= 0 && q.nl >= 0 && !(q.np > 0 && (!q.P || !q.pl_obs || !q.inlier_pt)) &&
         !(q.nl > 0 && (!q.sP || !q.eP || !q.le_obs || !q.inlier_ls));
}

// The whole call over problems whose host-side rules hold: every problem's rows staged in flat arrays behind a table of
// GnProblem (offsets, counts, T_init) and a table of cameras, one upload, one k_gn_pose launch, one download.  The inlier
// flags are inputs and outputs: they are staged in the output part and uploaded with the inputs.
plf_status gn_run(plf_ctx* ctx, const plf_gn_opts& o, int n, plf_gn_problem* pr, const std::vector<const plf_camera*>& cams) {
  if (n == 0) return PLF_OK;
  std::vector<size_t> po(n), lo(n);
  size_t NP = 0, NL = 0;
  for (int p = 0; p < n; ++p) {
    po[p] = NP; lo[p] = NL;
    NP += (size_t)pr[p].np; NL += (size_t)pr[p].nl;
  }
  StagedLayout L;
  const size_t oprob = L.take_in(n * sizeof(GnProblem)), ocam = L.take_in(n * sizeof(PlfPairCam)), oT = L.take_in(n * 128);
  const size_t oP = L.take_in(NP * 24), oO = L.take_in(NP * 16);
  const size_t osP = L.take_in(NL * 24), oeP = L.take_in(NL * 24), ole = L.take_in(NL * 24);
  const size_t ores = L.take_out(n * sizeof(plf_pose_result)), oip = L.take_out(NP), oil = L.take_out(NL);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_GN, &pin, &dev)) return st;
  uint8_t *pout = pin + L.in, *dout = dev + L.in;
  GnProblem* tab = (GnProblem*)(pin + oprob);
  PlfPairCam* cam = (PlfPairCam*)(pin + ocam);
  for (int p = 0; p < n; ++p) {
    const plf_gn_problem& q = pr[p];
    const size_t a = po[p], b = lo[p];
    if (q.np) {
      memcpy(pin + oP + 24 * a, q.P, (size_t)q.np * 24);
      memcpy(pin + oO + 16 * a, q.pl_obs, (size_t)q.np * 16);
      memcpy(pout + oip + a, q.inlier_pt, (size_t)q.np);
    }
    if (q.nl) {
      memcpy(pin + osP + 24 * b, q.sP, (size_t)q.nl * 24);
      memcpy(pin + oeP + 24 * b, q.eP, (size_t)q.nl * 24);
      memcpy(pin + ole + 24 * b, q.le_obs, (size_t)q.nl * 24);
      memcpy(pout + oil + b, q.inlier_ls, (size_t)q.nl);
    }
    if (q.T_init) memcpy(pin + oT + 128 * (size_t)p, q.T_init, 128);
    tab[p] = {(const double*)(dev + oP) + 3 * a, (const double*)(dev + oO) + 2 * a, dout + oip + a, nullptr, q.np,
              (const double*)(dev + osP) + 3 * b, (const double*)(dev + oeP) + 3 * b, (const double*)(dev + ole) + 3 * b,
              dout + oil + b, nullptr, q.nl, q.T_init ? (const double*)(dev + oT) + 16 * p : nullptr,
              (plf_pose_result*)(dout + ores) + p};
    const plf_camera& c = *cams[p];
    cam[p] = {c.fx, c.fy, c.cx, c.cy, c.b};
  }
  cudaStream_t s = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in + L.out, cudaMemcpyHostToDevice, s));
  if (plf_status st = plf_launch_gn(ctx, s, (const GnProblem*)(dev + oprob), n, o, (const PlfPairCam*)(dev + ocam))) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(pout, dout, L.out, cudaMemcpyDeviceToHost, s));
  PLF_CUDA(ctx, cudaStreamSynchronize(s));
  for (int p = 0; p < n; ++p) {
    plf_gn_problem& q = pr[p];
    memcpy(&q.out, pout + ores + p * sizeof(plf_pose_result), sizeof(plf_pose_result));
    if (q.np) memcpy(q.inlier_pt, pout + oip + po[p], (size_t)q.np);
    if (q.nl) memcpy(q.inlier_ls, pout + oil + lo[p], (size_t)q.nl);
  }
  return PLF_OK;
}

}  // namespace

extern "C" plf_status plf_gn_pose(plf_ctx* ctx, const plf_gn_opts* opts, const double* P, const double* pl_obs,
                                  uint8_t* inlier_pt, int np, const double* sP, const double* eP,
                                  const double* le_obs, uint8_t* inlier_ls, int nl, const double* T_init,
                                  plf_pose_result* out) {
  plf_gn_problem q = {P, pl_obs, inlier_pt, np, sP, eP, le_obs, inlier_ls, nl, T_init, {}};
  if (!ctx || !out || !gn_args_ok(q)) return plf_fail(ctx, PLF_ERR_INVALID, "plf_gn_pose: bad arguments");
  const plf_status st = gn_run(ctx, opts ? *opts : plf_gn_opts_from_params(ctx->params), 1, &q, {&ctx->cam});
  if (st == PLF_OK) *out = q.out;
  return st;
}

extern "C" plf_status plf_gn_pose_batch(plf_ctx* ctx, const plf_gn_opts* opts, int n_problems, plf_gn_problem* problems,
                                        const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = "plf_gn_pose_batch";
  if (n_problems < 0 || (n_problems && !problems))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments (n_problems = %d, problems)", fn, n_problems);
  std::vector<const plf_camera*> cams;
  if (plf_status st = plf_problem_cameras(ctx, fn, n_problems, seq, cams)) return st;
  for (int p = 0; p < n_problems; ++p) {
    const plf_gn_problem& q = problems[p];
    if (!gn_args_ok(q))
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: problem %d: np = %d, nl = %d: a count is negative or an array is NULL while "
                      "its count is > 0", fn, p, q.np, q.nl);
  }
  return gn_run(ctx, opts ? *opts : plf_gn_opts_from_params(ctx->params), n_problems, problems, cams);
}

// se(3) helpers exposed for the C++ shim / parity tests (stvo-pl auxiliar expmap_se3 / logmap_se3 /
// inverse_se3; 28/30/25 uses in src/mapHandler.cpp, e.g. :137-142,:3439).  Tiny: evaluated by one thread.
__global__ void k_se3(int op, const double* in, double* out) {
  if (op == 0) {  // expmap: T = identity updated by inverse(exp(-x))... computed directly below
    double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    double nx[6];
    for (int i = 0; i < 6; ++i) nx[i] = -in[i];
    d_update_pose(T, nx);  // I * inverse(exp(-x)) = exp(x)
    for (int i = 0; i < 16; ++i) out[i] = T[i];
  } else if (op == 1) {
    d_logmap(in, out);
  }
}

extern "C" plf_status plf_se3(plf_ctx* ctx, int op, const double* in, double* out) {
  if (!ctx || !in || !out || op < 0 || op > 1) return plf_fail(ctx, PLF_ERR_INVALID, "plf_se3: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  double *din, *dout;
  DevBufList scr;
  scr.add(din, 16); scr.add(dout, 16);
  if (plf_status st = scr.carve(ctx, PLF_SCR_GN)) return st;
  const int nin = op == 0 ? 6 : 16, nout = op == 0 ? 16 : 6;
  PLF_CUDA(ctx, cudaMemcpyAsync(din, in, nin * 8, cudaMemcpyHostToDevice, ctx->stream));
  k_se3<<<1, 1, 0, ctx->stream>>>(op, din, dout);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(out, dout, nout * 8, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}
