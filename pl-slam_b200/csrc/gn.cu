// Robust (Cauchy-weighted) 6-DoF point+line Gauss-Newton pose refinement (SURVEY §8 a8, a9).
//
// Replaces StVO::StereoFrameHandler::optimizePose (app/plslam_dataset.cpp:128, src/mapHandler.cpp:780),
// following its in-tree twin MapHandler::computeRelativePoseRobustGN (src/mapHandler.cpp:3566-3957;
// rows :3331-3426, normalise :3432, stop :3434/:3441, solve :3437-3438, update :3439, gate :3451-3482).
// se(3) helpers: stvo-pl auxiliar (SURVEY Appendix A.4), twist ordering [t; w] (src/mapHandler.cpp:3513-3514).
//
// One CTA (128 threads) per frame pair; many frame pairs per launch.  Each thread strides over the
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
__global__ void __launch_bounds__(GN_THREADS) k_gn_pose(const GnProblem* __restrict__ probs, GnCam launch_cam,
                                                         const PlfPairCam* __restrict__ cams, plf_gn_opts o) {
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
                         const PlfPairCam* d_cams) {
  if (nprob <= 0) return PLF_OK;
  GnCam c = {ctx->cam.fx, ctx->cam.fy, ctx->cam.cx, ctx->cam.cy};
  k_gn_pose<<<nprob, GN_THREADS, 0, cs>>>(d_probs, c, d_cams, o);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

extern "C" plf_status plf_gn_pose(plf_ctx* ctx, const plf_gn_opts* opts, const double* P, const double* pl_obs,
                                  uint8_t* inlier_pt, int np, const double* sP, const double* eP,
                                  const double* le_obs, uint8_t* inlier_ls, int nl, const double* T_init,
                                  plf_pose_result* out) {
  if (!ctx || !out || np < 0 || nl < 0 || (np > 0 && (!P || !pl_obs || !inlier_pt)) ||
      (nl > 0 && (!sP || !eP || !le_obs || !inlier_ls)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_gn_pose: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const plf_gn_opts o = opts ? *opts : plf_gn_opts_from_params(ctx->params);
  double *dP, *dO, *dsP, *deP, *dle, *dT;
  uint8_t *dIp, *dIl;
  plf_pose_result* dout;
  GnProblem* dprob;
  DevBufList scr;
  scr.add(dP, (size_t)np * 3); scr.add(dO, (size_t)np * 2); scr.add(dIp, np);
  scr.add(dsP, (size_t)nl * 3); scr.add(deP, (size_t)nl * 3); scr.add(dle, (size_t)nl * 3); scr.add(dIl, nl);
  scr.add(dT, 16); scr.add(dout, 1); scr.add(dprob, 1);
  if (plf_status st = scr.carve(ctx, PLF_SCR_GN)) return st;
  cudaStream_t s = ctx->stream;
  if (np) {
    PLF_CUDA(ctx, cudaMemcpyAsync(dP, P, (size_t)np * 24, cudaMemcpyHostToDevice, s));
    PLF_CUDA(ctx, cudaMemcpyAsync(dO, pl_obs, (size_t)np * 16, cudaMemcpyHostToDevice, s));
    PLF_CUDA(ctx, cudaMemcpyAsync(dIp, inlier_pt, (size_t)np, cudaMemcpyHostToDevice, s));
  }
  if (nl) {
    PLF_CUDA(ctx, cudaMemcpyAsync(dsP, sP, (size_t)nl * 24, cudaMemcpyHostToDevice, s));
    PLF_CUDA(ctx, cudaMemcpyAsync(deP, eP, (size_t)nl * 24, cudaMemcpyHostToDevice, s));
    PLF_CUDA(ctx, cudaMemcpyAsync(dle, le_obs, (size_t)nl * 24, cudaMemcpyHostToDevice, s));
    PLF_CUDA(ctx, cudaMemcpyAsync(dIl, inlier_ls, (size_t)nl, cudaMemcpyHostToDevice, s));
  }
  double Tid[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  PLF_CUDA(ctx, cudaMemcpyAsync(dT, T_init ? T_init : Tid, sizeof Tid, cudaMemcpyHostToDevice, s));
  GnProblem hp = {dP, dO, dIp, nullptr, np, dsP, deP, dle, dIl, nullptr, nl, dT, dout};
  PLF_CUDA(ctx, cudaMemcpyAsync(dprob, &hp, sizeof hp, cudaMemcpyHostToDevice, s));
  plf_status st = plf_launch_gn(ctx, s, dprob, 1, o);
  if (st) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(out, dout, sizeof *out, cudaMemcpyDeviceToHost, s));
  if (np) PLF_CUDA(ctx, cudaMemcpyAsync(inlier_pt, dIp, (size_t)np, cudaMemcpyDeviceToHost, s));
  if (nl) PLF_CUDA(ctx, cudaMemcpyAsync(inlier_ls, dIl, (size_t)nl, cudaMemcpyDeviceToHost, s));
  PLF_CUDA(ctx, cudaStreamSynchronize(s));
  return PLF_OK;
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
