// Loop-closure pose-graph optimisation on the GPU (DESIGN.md §1 row f7), one problem (plf_pose_graph) or many at once
// (plf_pose_graph_batch, the same driver).
//
// Replaces the g2o part of MapHandler::loopClosureOptimizationCovGraphG2O (src/mapHandler.cpp:4185-4410):
// computeInitialGuess() and optimize(maxItersPGO) of g2o's OptimizationAlgorithmLevenberg over VertexSE3 / EdgeSE3 with
// identity information.  The host keeps g2o's control flow (oracle/pgo.py restates it), one step function per problem;
// the numerical work runs here, each kernel gridded (item, problem) over the problems still running:
//   k_pgo_linearize   one thread per edge, once per iteration: E = Z^-1 X_i^-1 X_j, e = MQT(E) and the Jacobians J_i, J_j
//                     at the iteration's estimate, reused by every trial of the iteration
//   k_pgo_zero        the dense system S = 0, across the GPU
//   k_pgo_assemble    one CTA per non-zero 6 x 6 block of the lower triangle of H: the block's contributions summed in
//                     ascending edge order (a per-block edge list built once per call), written with + lambda I into
//                     the dense system S; the diagonal blocks also write b = -sum J^T e.  No float atomics: two calls
//                     are bit-identical.
//   gbb_ldlt          the tiled LDL^T and the two substitutions of plf_global_ba (lba.cu), batched (k_gbb_*)
//   k_pgo_step        one thread per vertex: X_t = X (+) x, the pivot check on D and x (lambda x + b) per free vertex
//   k_pgo_edge_chi2   one thread per edge: e^T e at a given estimate
//   k_pgo_reduce      one CTA per problem: chi2, sum x (lambda x + b) and the pivot flag, each summed in a fixed order
// One 4-double copy per problem and trial goes to the host for the trial's decision.
#include <math.h>
#include <stddef.h>

#include <unordered_map>

#include "plf_internal.h"

namespace {

// Poses are isometries stored as 16 doubles, row-major, last row (0, 0, 0, 1).
__host__ __device__ inline void iso_mul(const double* A, const double* B, double* C) {   // C = A B
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) C[4 * r + c] = A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c] + A[4 * r + 2] * B[8 + c];
    C[4 * r + 3] = A[4 * r] * B[3] + A[4 * r + 1] * B[7] + A[4 * r + 2] * B[11] + A[4 * r + 3];
  }
  C[12] = 0.0; C[13] = 0.0; C[14] = 0.0; C[15] = 1.0;
}
__host__ __device__ inline void iso_inv(const double* A, double* B) {   // (R^T, -R^T t)
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) B[4 * r + c] = A[4 * c + r];
    B[4 * r + 3] = -(A[r] * A[3] + A[4 + r] * A[7] + A[8 + r] * A[11]);
  }
  B[12] = 0.0; B[13] = 0.0; B[14] = 0.0; B[15] = 1.0;
}

// Unit quaternion (w, x, y, z) of the rotation block of T, as Eigen's Quaternion(Matrix3) computes it, then normalised
// with w >= 0 (g2o's toCompactQuaternion).
__device__ inline void pgo_quat(const double* T, double* q) {
  // Eigen picks the largest diagonal entry i (j = i + 1, k = j + 1 mod 3) when the trace is not positive; the three cases
  // are written out so that nothing is indexed at run time
  const double R00 = T[0], R01 = T[1], R02 = T[2], R10 = T[4], R11 = T[5], R12 = T[6], R20 = T[8], R21 = T[9], R22 = T[10];
  const double tr = R00 + R11 + R22;
  double w, x, y, z;
  if (tr > 0.0) {
    double t = sqrt(tr + 1.0);
    w = 0.5 * t;
    t = 0.5 / t;
    x = (R21 - R12) * t;
    y = (R02 - R20) * t;
    z = (R10 - R01) * t;
  } else if (R22 > (R11 > R00 ? R11 : R00)) {   // i = 2
    double t = sqrt(R22 - R00 - R11 + 1.0);
    z = 0.5 * t;
    t = 0.5 / t;
    w = (R10 - R01) * t;
    x = (R02 + R20) * t;
    y = (R12 + R21) * t;
  } else if (R11 > R00) {   // i = 1
    double t = sqrt(R11 - R22 - R00 + 1.0);
    y = 0.5 * t;
    t = 0.5 / t;
    w = (R02 - R20) * t;
    z = (R21 + R12) * t;
    x = (R01 + R10) * t;
  } else {   // i = 0
    double t = sqrt(R00 - R11 - R22 + 1.0);
    x = 0.5 * t;
    t = 0.5 / t;
    w = (R21 - R12) * t;
    y = (R10 + R01) * t;
    z = (R20 + R02) * t;
  }
  const double n = sqrt(w * w + x * x + y * y + z * z);
  const double s = w / n < 0.0 ? -1.0 / n : 1.0 / n;
  q[0] = w * s; q[1] = x * s; q[2] = y * s; q[3] = z * s;
}

// e = MQT(Z^-1 (X_i^-1 X_j)); E receives the isometry, q its quaternion
__device__ inline void pgo_error(const double* Xi, const double* Xj, const double* Z, double* E, double* q, double* e) {
  double A[16], B[16], Zi[16];
  iso_inv(Xi, A);
  iso_mul(A, Xj, B);
  iso_inv(Z, Zi);
  iso_mul(Zi, B, E);
  pgo_quat(E, q);
  e[0] = E[3]; e[1] = E[7]; e[2] = E[11]; e[3] = q[1]; e[4] = q[2]; e[5] = q[3];
}

struct PgoDev {
  int nv, ne, nf, nb;
  const int* efrom; const int* eto;       // ne
  const double* Z;                        // ne x 16
  const int* fidx;                        // nv: the vertex's block in the system, -1 when fixed or without edges
  double* X; double* Xt;                  // nv x 16: estimate, trial estimate
  double* e; double* Ji; double* Jj;      // ne x 6, ne x 36, ne x 36 (row-major: error row, increment column)
  double* ce;                             // ne: e^T e
  const int* blk_rc;                      // nb x 2: block row, block column (row >= column; the nf diagonal blocks first)
  const int* blk_start; const int* blk_item;   // items of block k: blk_item[blk_start[k] .. blk_start[k + 1]) = 4 edge + kind
  double* S;                              // n x n, n = 6 nf
  double* b; double* g; double* y; double* x;   // n each: b, the solve's right-hand side (overwritten), work, solution
  double* dotp; uint8_t* bad;             // nf: x (lambda x + b) of the vertex's 6 entries, pivot failure
  double* red;                            // 4: chi2, sum x (lambda x + b), pivot failure
};

// ---- one problem's work: each function is one edge, block, vertex or CTA of the problem d ----------------------------
__device__ __forceinline__ void pgo_linearize(const PgoDev& d, int k) {
  const double* Z = d.Z + 16 * (size_t)k;
  double E[16], q[4], e[6];
  pgo_error(d.X + 16 * (size_t)d.efrom[k], d.X + 16 * (size_t)d.eto[k], Z, E, q, e);
  const double w = q[0], vx = q[1], vy = q[2], vz = q[3];
  // J_j = [R_E 0; 0 wI + [v]x],  J_i = [-R_Z^T  2 [t_E + R_Z^T t_Z]x R_Z^T; 0  (-wI + [v]x) R_Z^T]
  double Jj[36], Ji[36];
  for (int i = 0; i < 36; ++i) { Jj[i] = 0.0; Ji[i] = 0.0; }
  const double Vx[9] = {0.0, -vz, vy, vz, 0.0, -vx, -vy, vx, 0.0};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      Jj[6 * r + c] = E[4 * r + c];
      Jj[6 * (3 + r) + 3 + c] = (r == c ? w : 0.0) + Vx[3 * r + c];
    }
  double RZt[9], p[3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) RZt[3 * r + c] = Z[4 * c + r];
  for (int r = 0; r < 3; ++r) p[r] = E[4 * r + 3] + (RZt[3 * r] * Z[3] + RZt[3 * r + 1] * Z[7] + RZt[3 * r + 2] * Z[11]);
  const double P2[9] = {0.0, -2.0 * p[2], 2.0 * p[1], 2.0 * p[2], 0.0, -2.0 * p[0], -2.0 * p[1], 2.0 * p[0], 0.0};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      Ji[6 * r + c] = -RZt[3 * r + c];
      Ji[6 * r + 3 + c] = P2[3 * r] * RZt[c] + P2[3 * r + 1] * RZt[3 + c] + P2[3 * r + 2] * RZt[6 + c];
      const double m0 = (r == 0 ? -w : 0.0) + Vx[3 * r], m1 = (r == 1 ? -w : 0.0) + Vx[3 * r + 1],
                   m2 = (r == 2 ? -w : 0.0) + Vx[3 * r + 2];
      Ji[6 * (3 + r) + 3 + c] = m0 * RZt[c] + m1 * RZt[3 + c] + m2 * RZt[6 + c];
    }
  for (int i = 0; i < 6; ++i) d.e[6 * (size_t)k + i] = e[i];
  for (int i = 0; i < 36; ++i) { d.Ji[36 * (size_t)k + i] = Ji[i]; d.Jj[36 * (size_t)k + i] = Jj[i]; }
}

// block blk, one CTA of 64 threads; kind 0: J_i^T J_i, 1: J_j^T J_j, 2: J_i^T J_j (the block row is the edge's `from`),
// 3: J_j^T J_i
__device__ __forceinline__ void pgo_assemble(const PgoDev& d, int blk, double lambda) {
  const int t = threadIdx.x, n = 6 * d.nf;
  const int br = d.blk_rc[2 * blk], bc = d.blk_rc[2 * blk + 1], s = d.blk_start[blk], end = d.blk_start[blk + 1];
  if (t < 36) {
    const int r = t / 6, c = t % 6;
    double acc = 0.0;
    for (int it = s; it < end; ++it) {
      const int k = d.blk_item[it] >> 2, kind = d.blk_item[it] & 3;
      const double* L = (kind == 0 || kind == 2 ? d.Ji : d.Jj) + 36 * (size_t)k;
      const double* R = (kind == 0 || kind == 3 ? d.Ji : d.Jj) + 36 * (size_t)k;
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v += L[6 * m + r] * R[6 * m + c];
      acc += v;
    }
    if (br == bc && r == c) acc += lambda;
    d.S[(size_t)(6 * br + r) * n + 6 * bc + c] = acc;
  } else if (t < 42 && br == bc) {
    const int r = t - 36;
    double acc = 0.0;
    for (int it = s; it < end; ++it) {
      const int k = d.blk_item[it] >> 2, kind = d.blk_item[it] & 3;
      const double* J = (kind == 0 ? d.Ji : d.Jj) + 36 * (size_t)k;
      const double* e = d.e + 6 * (size_t)k;
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v += J[6 * m + r] * e[m];
      acc -= v;
    }
    d.b[6 * br + r] = acc;
    d.g[6 * br + r] = acc;
  }
}

// X_t = X Inc(x_v): Inc = (R(q), x_t) with q = (sqrt(1 - |x_q|^2), x_q), the identity rotation when 1 - |x_q|^2 < 0
__device__ __forceinline__ void pgo_step(const PgoDev& d, int v, double lambda) {
  const double* X = d.X + 16 * (size_t)v;
  double* Xt = d.Xt + 16 * (size_t)v;
  const int f = d.fidx[v];
  if (f < 0) {
    for (int i = 0; i < 16; ++i) Xt[i] = X[i];
    return;
  }
  const double* dx = d.x + 6 * f;
  double Inc[16];
  const double qx = dx[3], qy = dx[4], qz = dx[5];
  const double w2 = 1.0 - (qx * qx + qy * qy + qz * qz);
  if (w2 < 0.0) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) Inc[4 * r + c] = r == c ? 1.0 : 0.0;
  } else {   // Eigen's Quaternion::toRotationMatrix
    const double w = sqrt(w2);
    const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * qx, txy = ty * qx, txz = tz * qx, tyy = ty * qy,
                 tyz = tz * qy, tzz = tz * qz;
    Inc[0] = 1.0 - (tyy + tzz); Inc[1] = txy - twz;         Inc[2] = txz + twy;
    Inc[4] = txy + twz;         Inc[5] = 1.0 - (txx + tzz); Inc[6] = tyz - twx;
    Inc[8] = txz - twy;         Inc[9] = tyz + twx;         Inc[10] = 1.0 - (txx + tyy);
  }
  Inc[3] = dx[0]; Inc[7] = dx[1]; Inc[11] = dx[2];
  Inc[12] = 0.0; Inc[13] = 0.0; Inc[14] = 0.0; Inc[15] = 1.0;
  double Y[16];
  iso_mul(X, Inc, Y);
  for (int i = 0; i < 16; ++i) Xt[i] = Y[i];
  const int n = 6 * d.nf;
  double s = 0.0;
  uint8_t bad = 0;
  for (int i = 0; i < 6; ++i) {
    const int j = 6 * f + i;
    s += d.x[j] * (lambda * d.x[j] + d.b[j]);
    const double D = d.S[(size_t)j * n + j];
    bad |= !(D > 0.0 && D <= 1.7976931348623157e308);
  }
  d.dotp[f] = s;
  d.bad[f] = bad;
}

__device__ __forceinline__ void pgo_edge_chi2(const PgoDev& d, const double* X, int k) {
  double E[16], q[4], e[6];
  pgo_error(X + 16 * (size_t)d.efrom[k], X + 16 * (size_t)d.eto[k], d.Z + 16 * (size_t)k, E, q, e);
  double s = 0.0;
  for (int i = 0; i < 6; ++i) s += e[i] * e[i];
  d.ce[k] = s;
}

// Fixed-order sums: thread t adds entries t, t + 1024, ... in turn, then a tree over the threads.
constexpr int PGO_RED = 1024;
__device__ inline double pgo_block_sum(double v, double* sh) {
  const int t = threadIdx.x;
  sh[t] = v;
  __syncthreads();
  for (int h = PGO_RED / 2; h > 0; h >>= 1) {
    if (t < h) sh[t] += sh[t + h];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}
// one CTA of PGO_RED threads: chi2 and the step's two other sums over nf free vertices (0 for the initial chi2)
__device__ __forceinline__ void pgo_reduce(const PgoDev& d, int nf, double* sh) {
  const int t = threadIdx.x;
  double c = 0.0, s = 0.0, b = 0.0;
  for (int i = t; i < d.ne; i += PGO_RED) c += d.ce[i];
  for (int i = t; i < nf; i += PGO_RED) { s += d.dotp[i]; b += d.bad[i]; }
  c = pgo_block_sum(c, sh);
  s = pgo_block_sum(s, sh);
  b = pgo_block_sum(b, sh);
  if (t == 0) { d.red[0] = c; d.red[1] = s; d.red[2] = b; d.red[3] = 0.0; }
}

// ---- the batch: problem p's arrays are slices of flat arrays, at the offsets of its PgoProb -------------------------------
struct PgoProb {
  int nv, ne, nf, nb;
  long long vo, eo, fo, bo, io, so;   // offsets: vertices, edges, free vertices, blocks, block items (blk_start: bo + p),
                                      // S (doubles)
};
// A problem's part of the round, written by the host before each round
struct PgoCtl {
  double lambda;
  int active;   // 0 once the problem has stopped: every kernel returns at once for it
  int start;    // this round's trial starts an iteration: linearise at the estimate
  int cur;      // the pose buffer (0 / 1) that holds the estimate X; the other receives the trial estimate X_t
  int pad;
};
struct PgoBatch {
  const PgoProb* prob; const PgoCtl* ctl;
  const int* efrom; const int* eto; const double* Z; const int* fidx;
  double* X; long long xpar;   // the two pose buffers, xpar doubles apart
  double* e; double* Ji; double* Jj; double* ce;
  const int* blk_rc; const int* blk_start; const int* blk_item;
  double* S; double* b; double* g; double* y; double* x; double* dotp; uint8_t* bad; double* red;
};

__device__ __forceinline__ PgoDev pgo_view(const PgoBatch& B, int p) {
  const PgoProb q = B.prob[p];
  const int cur = B.ctl[p].cur;
  PgoDev d;
  d.nv = q.nv; d.ne = q.ne; d.nf = q.nf; d.nb = q.nb;
  d.efrom = B.efrom + q.eo; d.eto = B.eto + q.eo; d.Z = B.Z + 16 * q.eo; d.fidx = B.fidx + q.vo;
  d.X = B.X + cur * B.xpar + 16 * q.vo; d.Xt = B.X + (cur ^ 1) * B.xpar + 16 * q.vo;
  d.e = B.e + 6 * q.eo; d.Ji = B.Ji + 36 * q.eo; d.Jj = B.Jj + 36 * q.eo; d.ce = B.ce + q.eo;
  d.blk_rc = B.blk_rc + 2 * q.bo; d.blk_start = B.blk_start + q.bo + p; d.blk_item = B.blk_item + q.io;
  d.S = B.S + q.so;
  d.b = B.b + 6 * q.fo; d.g = B.g + 6 * q.fo; d.y = B.y + 6 * q.fo; d.x = B.x + 6 * q.fo;
  d.dotp = B.dotp + q.fo; d.bad = B.bad + q.fo; d.red = B.red + 4 * p;
  return d;
}

// The kernels are gridded (item, problem): blockIdx.y is the problem, blockIdx.x strides over its items at the extent of
// the round's largest active problem.
__global__ void __launch_bounds__(128) k_pgo_linearize(PgoBatch B) {
  const int p = blockIdx.y;
  if (!B.ctl[p].active || !B.ctl[p].start) return;
  const PgoDev d = pgo_view(B, p);
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k < d.ne) pgo_linearize(d, k);
}

// S = 0 across the GPU, for the assembly (which writes only the non-zero blocks)
__global__ void __launch_bounds__(256) k_pgo_zero(PgoBatch B) {
  const int p = blockIdx.y;
  if (!B.ctl[p].active) return;
  const PgoProb q = B.prob[p];
  const size_t n = 6 * (size_t)q.nf, stride = (size_t)gridDim.x * 256;
  double* S = B.S + q.so;
  for (size_t i = blockIdx.x * 256 + threadIdx.x; i < n * n; i += stride) S[i] = 0.0;
}

// one CTA per non-zero block
__global__ void __launch_bounds__(64) k_pgo_assemble(PgoBatch B) {
  const int p = blockIdx.y;
  if (!B.ctl[p].active) return;
  const PgoDev d = pgo_view(B, p);
  if ((int)blockIdx.x < d.nb) pgo_assemble(d, blockIdx.x, B.ctl[p].lambda);
}

__global__ void __launch_bounds__(128) k_pgo_step(PgoBatch B) {
  const int p = blockIdx.y;
  if (!B.ctl[p].active) return;
  const PgoDev d = pgo_view(B, p);
  const int v = blockIdx.x * 128 + threadIdx.x;
  if (v < d.nv) pgo_step(d, v, B.ctl[p].lambda);
}

// e^T e per edge at the estimate (trial 0: the initial chi2) or at the trial estimate
__global__ void __launch_bounds__(128) k_pgo_edge_chi2(PgoBatch B, int trial) {
  const int p = blockIdx.y;
  if (!B.ctl[p].active) return;
  const PgoDev d = pgo_view(B, p);
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k < d.ne) pgo_edge_chi2(d, trial ? d.Xt : d.X, k);
}

__global__ void __launch_bounds__(PGO_RED) k_pgo_reduce(PgoBatch B, int trial) {
  __shared__ double sh[PGO_RED];
  const int p = blockIdx.y;
  if (!B.ctl[p].active) return;
  const PgoDev d = pgo_view(B, p);
  pgo_reduce(d, trial ? d.nf : 0, sh);
}

// ---- host side ---------------------------------------------------------------------------------------------------------
// One problem after its checks: its system's blocks (the free vertices with edges, in id order), the initial guess and
// the blocks of H's lower triangle with their contributions in ascending edge order.
struct PgoHost {
  int nf = 0;
  std::vector<int> fidx, blk_rc, blk_start, blk_item;
  std::vector<double> X;
};

// plf_pose_graph's rules for one problem after its argument checks, in order; pfx starts every message
static plf_status pgo_check(plf_ctx* ctx, const char* pfx, const plf_pgo_problem* p, PgoHost& h) {
  const int nv = p->n_v, ne = p->n_e;
  if ((nv && (!p->T || !p->fixed)) || (ne && (!p->from || !p->to || !p->Z)))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: null array", pfx);
  std::vector<int> deg(nv, 0);
  for (int k = 0; k < ne; ++k) {
    const int a = p->from[k], b = p->to[k];
    if (a < 0 || a >= nv || b < 0 || b >= nv || a == b)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: edge %d joins vertices %d and %d (%d vertices)", pfx, k, a, b, nv);
    deg[a]++; deg[b]++;
  }
  h.fidx.assign(nv, -1);
  int nf = 0;
  for (int v = 0; v < nv; ++v)
    if (!p->fixed[v] && deg[v]) h.fidx[v] = nf++;
  h.nf = nf;
  if (nf > 4096) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d free vertices with edges (limit 4096)", pfx, nf);
  for (size_t i = 0; i < (size_t)nv * 16; ++i)
    if (!isfinite(p->T[i])) return plf_fail(ctx, PLF_ERR_INVALID, "%s: non-finite pose of vertex %d", pfx, (int)(i / 16));
  for (size_t i = 0; i < (size_t)ne * 16; ++i)
    if (!isfinite(p->Z[i])) return plf_fail(ctx, PLF_ERR_INVALID, "%s: non-finite measurement of edge %d", pfx, (int)(i / 16));
  // every connected component with edges holds a fixed vertex (else its system is singular up to the damping)
  std::vector<int> root(nv);
  for (int v = 0; v < nv; ++v) root[v] = v;
  auto find = [&](int v) { while (root[v] != v) v = root[v] = root[root[v]]; return v; };
  for (int k = 0; k < ne; ++k) root[find(p->from[k])] = find(p->to[k]);
  std::vector<uint8_t> anchored(nv, 0);
  for (int v = 0; v < nv; ++v)
    if (p->fixed[v]) anchored[find(v)] = 1;
  for (int k = 0; k < ne; ++k)
    if (!anchored[find(p->from[k])])
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: the component of edge %d has no fixed vertex", pfx, k);
  return PLF_OK;
}

// the initial guess and the block lists of a checked problem
static void pgo_prepare(const plf_pgo_problem* p, PgoHost& h) {
  const int nv = p->n_v, ne = p->n_e, nf = h.nf;
  const std::vector<int>& fidx = h.fidx;
  // ---- initial guess (g2o computeInitialGuess): breadth-first from the fixed vertices in ascending id, each vertex's
  // edges in the order given; a reached free vertex takes parent * Z (parent = from) or parent * Z^-1
  std::vector<double>& X = h.X;
  X.assign(p->T, p->T + (size_t)nv * 16);
  {
    std::vector<int> adj_start(nv + 1, 0), adj((size_t)2 * ne);
    for (int k = 0; k < ne; ++k) { adj_start[p->from[k] + 1]++; adj_start[p->to[k] + 1]++; }
    for (int v = 0; v < nv; ++v) adj_start[v + 1] += adj_start[v];
    std::vector<int> fill(adj_start.begin(), adj_start.end() - 1);
    for (int k = 0; k < ne; ++k) { adj[fill[p->from[k]]++] = k; adj[fill[p->to[k]]++] = k; }
    std::vector<uint8_t> seen(nv);
    std::vector<int> queue;
    queue.reserve(nv);
    for (int v = 0; v < nv; ++v) {
      seen[v] = p->fixed[v] ? 1 : 0;
      if (p->fixed[v]) queue.push_back(v);
    }
    for (size_t hd = 0; hd < queue.size(); ++hd) {
      const int v = queue[hd];
      for (int a = adj_start[v]; a < adj_start[v + 1]; ++a) {
        const int k = adj[a], u = p->from[k] == v ? p->to[k] : p->from[k];
        if (seen[u]) continue;
        seen[u] = 1;
        if (p->from[k] == v) {
          iso_mul(&X[16 * (size_t)v], p->Z + 16 * (size_t)k, &X[16 * (size_t)u]);
        } else {
          double Zi[16];
          iso_inv(p->Z + 16 * (size_t)k, Zi);
          iso_mul(&X[16 * (size_t)v], Zi, &X[16 * (size_t)u]);
        }
        queue.push_back(u);
      }
    }
  }
  // ---- the blocks of H's lower triangle and their contributions, in ascending edge order
  std::vector<int>& blk_rc = h.blk_rc;
  blk_rc.clear();
  blk_rc.reserve((size_t)2 * nf);
  for (int f = 0; f < nf; ++f) { blk_rc.push_back(f); blk_rc.push_back(f); }
  std::unordered_map<long long, int> off;
  std::vector<int> it_blk, it_val;   // (block, 4 edge + kind) in edge order
  for (int k = 0; k < ne; ++k) {
    const int fi = fidx[p->from[k]], fj = fidx[p->to[k]];
    if (fi >= 0) { it_blk.push_back(fi); it_val.push_back(4 * k); }
    if (fj >= 0) { it_blk.push_back(fj); it_val.push_back(4 * k + 1); }
    if (fi >= 0 && fj >= 0) {
      const int r = std::max(fi, fj), c = std::min(fi, fj);
      auto ins = off.emplace((long long)r * 4096 + c, (int)(blk_rc.size() / 2));
      if (ins.second) { blk_rc.push_back(r); blk_rc.push_back(c); }
      it_blk.push_back(ins.first->second);
      it_val.push_back(4 * k + (fi > fj ? 2 : 3));
    }
  }
  const int nb = (int)(blk_rc.size() / 2), nit = (int)it_blk.size();
  h.blk_start.assign(nb + 1, 0);
  h.blk_item.resize(nit);
  for (int i = 0; i < nit; ++i) h.blk_start[it_blk[i] + 1]++;
  for (int b = 0; b < nb; ++b) h.blk_start[b + 1] += h.blk_start[b];
  std::vector<int> fill(h.blk_start.begin(), h.blk_start.end() - 1);
  for (int i = 0; i < nit; ++i) h.blk_item[fill[it_blk[i]]++] = it_val[i];
}

// g2o's OptimizationAlgorithmLevenberg::solve for one problem, between two trials
struct PgoLm {
  int iter = 0, trials = 0;   // the iteration, and the trials it has run so far
  double chi = 0.0, lambda = 0.0;
  double ni = 2.0;            // g2o's _ni is a double: it doubles on every rejected trial and must reach lambda's overflow
  bool running = false;
  int cur = 0;                // the pose buffer holding the estimate
};

// The decision after one trial, from its sums red (chi2 at X_t, sum x (lambda x + b), pivot failure): the trace row,
// g2o's acceptance and lambda / ni schedule, its do ... while (rho < 0 && trials < 10) and the three stop tests that end
// the iteration loop.  The arithmetic stays on the host, in double: the device's pow is not glibc's.
static void pgo_decide(PgoLm& s, const double* red, int max_iters, plf_pgo_result& out) {
  const double chi_t = red[2] != 0.0 ? 1.7976931348623157e308 : red[0];   // failed solve: DBL_MAX
  const double rho = (s.chi - chi_t) / (red[1] + 1e-3);
  const bool accept = rho > 0.0 && isfinite(chi_t);
  if (out.n_trace < out.trace_cap) {
    plf_pgo_trial& tr = out.trace[out.n_trace++];
    tr.iter = s.iter; tr.accepted = accept; tr.lambda = s.lambda; tr.chi = s.chi; tr.chi_t = chi_t; tr.rho = rho;
  }
  if (accept) {
    const double alpha = std::min(1.0 - pow(2.0 * rho - 1.0, 3), 2.0 / 3.0);
    s.lambda *= std::max(1.0 / 3.0, alpha);
    s.ni = 2;
    s.cur ^= 1;
    s.chi = chi_t;
  } else {
    s.lambda *= s.ni;
    s.ni *= 2;
  }
  ++s.trials;
  if (rho < 0.0 && s.trials < 10) return;   // the iteration's next trial
  out.iters = s.iter + 1;
  out.trials += s.trials;
  if (s.trials == 10 || rho == 0.0 || !isfinite(s.lambda)) {
    out.stop = s.trials == 10 ? PLF_PGO_STOP_TRIALS : (rho == 0.0 ? PLF_PGO_STOP_RHO_ZERO : PLF_PGO_STOP_LAMBDA);
    s.running = false;
  } else if (++s.iter == max_iters) {
    s.running = false;
  }
  s.trials = 0;
}

// plf_pose_graph (one problem, batch = false) and plf_pose_graph_batch.  Every refusal comes before any work.  One
// staged upload, then rounds in lockstep: round 0 evaluates every problem's initial chi2, each later round runs one trial
// of every running problem in one launch chain, uploads the problems' lambdas and flags before it and downloads their
// sums after it, with one host synchronisation.  One download of the poses ends the call.
static plf_status pgo_run(plf_ctx* ctx, const plf_pgo_opts* opts, int P, const plf_pgo_problem* problems,
                          plf_pgo_result* out, bool batch) {
  const char* fn = batch ? "plf_pose_graph_batch" : "plf_pose_graph";
  if (!ctx || !opts || P < 0 || (P && (!problems || !out)) || opts->max_iters < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  // g2o takes a non-positive user lambda as "derive one from H"; both call sites pass 1e-10, so anything else is refused
  if (!(opts->lambda_init > 0.0 && opts->lambda_init <= 1.7976931348623157e308))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: lambda_init %g is not a positive finite number", fn, opts->lambda_init);
  if (!P) return PLF_OK;
  // the problems are gridded in y
  if (P > 65535) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d problems (limit 65535)", fn, P);
  std::vector<std::string> pfx(P);
  for (int k = 0; k < P; ++k) {
    char buf[64];
    if (batch) snprintf(buf, sizeof buf, "%s: problem %d", fn, k);
    pfx[k] = batch ? buf : fn;
  }
  // each problem's rules in the single call's order, the problems in turn: the first bad problem is the one named
  std::vector<PgoHost> h(P);
  for (int k = 0; k < P; ++k) {
    const plf_pgo_problem& p = problems[k];
    if (p.n_v < 0 || p.n_e < 0 || out[k].trace_cap < 0 || (out[k].trace_cap && !out[k].trace))
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", pfx[k].c_str());
    if (plf_status st = pgo_check(ctx, pfx[k].c_str(), &p, h[k])) return st;
  }
  // ---- the flat layout
  std::vector<PgoProb> hp(P);
  std::vector<GbbBig> hb(P);
  long long tV = 0, tE = 0, tF = 0, tB = 0, tI = 0, tS = 0, tWp = 0, tNz = 0;
  int mE = 0;
  for (int k = 0; k < P; ++k) {
    pgo_prepare(&problems[k], h[k]);
    PgoProb& q = hp[k];
    q.nv = problems[k].n_v; q.ne = problems[k].n_e; q.nf = h[k].nf; q.nb = (int)(h[k].blk_rc.size() / 2);
    q.vo = tV; q.eo = tE; q.fo = tF; q.bo = tB; q.io = tI; q.so = tS;
    const long long n = 6LL * q.nf, nt = (n + PLF_LDLT_TILE - 1) / PLF_LDLT_TILE;
    hb[k] = GbbBig{k, q.nf, tS, 6 * tF, 6 * tF, tWp, tNz};
    tV += q.nv; tE += q.ne; tF += q.nf; tB += q.nb; tI += (long long)h[k].blk_item.size(); tS += n * n;
    tWp += nt * PLF_LDLT_TILE * PLF_LDLT_TILE; tNz += nt * nt;
    mE = std::max(mE, q.ne);
  }
  // inputs; outputs: the two pose buffers first, so that the initial guess in the first one goes up with the inputs
  StagedLayout L;
  const size_t iProb = L.take_in(sizeof(PgoProb) * P), iBig = L.take_in(sizeof(GbbBig) * P),
               iCtl = L.take_in(sizeof(PgoCtl) * P), iFrom = L.take_in(4 * tE), iTo = L.take_in(4 * tE),
               iZ = L.take_in(128 * tE), iFidx = L.take_in(4 * tV), iRc = L.take_in(8 * tB),
               iStart = L.take_in(4 * (tB + P)), iItem = L.take_in(4 * tI);
  const size_t oX = L.take_out(256 * tV), oRed = L.take_out(32 * (size_t)P);
  const size_t wE = L.take_work(48 * tE), wJi = L.take_work(288 * tE), wJj = L.take_work(288 * tE),
               wCe = L.take_work(8 * tE), wS = L.take_work(8 * tS), wB = L.take_work(48 * tF), wG = L.take_work(48 * tF),
               wY = L.take_work(48 * tF), wX = L.take_work(48 * tF), wDot = L.take_work(8 * tF), wBad = L.take_work(tF),
               wWp = L.take_work(8 * tWp), wNz = L.take_work(tNz);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_BA, &pin, &dev)) return st;
  PgoCtl* ctl = (PgoCtl*)(pin + iCtl);
  double* Xpin = (double*)(pin + L.in + oX);
  const double* red = (const double*)(pin + L.in + oRed);
  for (int k = 0; k < P; ++k) {
    const plf_pgo_problem& p = problems[k];
    const PgoProb& q = hp[k];
    if (q.ne) {
      memcpy((int*)(pin + iFrom) + q.eo, p.from, 4 * (size_t)q.ne);
      memcpy((int*)(pin + iTo) + q.eo, p.to, 4 * (size_t)q.ne);
      memcpy((double*)(pin + iZ) + 16 * q.eo, p.Z, 128 * (size_t)q.ne);
    }
    if (q.nv) {
      memcpy((int*)(pin + iFidx) + q.vo, h[k].fidx.data(), 4 * (size_t)q.nv);
      memcpy(Xpin + 16 * q.vo, h[k].X.data(), 128 * (size_t)q.nv);
    }
    if (q.nb) memcpy((int*)(pin + iRc) + 2 * q.bo, h[k].blk_rc.data(), 8 * (size_t)q.nb);
    memcpy((int*)(pin + iStart) + q.bo + k, h[k].blk_start.data(), 4 * ((size_t)q.nb + 1));
    if (!h[k].blk_item.empty()) memcpy((int*)(pin + iItem) + q.io, h[k].blk_item.data(), 4 * h[k].blk_item.size());
    ctl[k] = PgoCtl{opts->lambda_init, 1, 0, 0, 0};
  }
  memcpy(pin + iProb, hp.data(), sizeof(PgoProb) * P);
  memcpy(pin + iBig, hb.data(), sizeof(GbbBig) * P);
  h.clear();
  cudaStream_t cs = ctx->stream;
  static_assert(sizeof(PgoCtl) % sizeof(int) == 0, "gbb_view reads PgoCtl::active as a strided int");
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in + 128 * tV, cudaMemcpyHostToDevice, cs));   // oX == 0
  uint8_t* const dout = dev + L.in;
  uint8_t* const dwork = dout + L.out;
  PgoBatch B;
  B.prob = (const PgoProb*)(dev + iProb); B.ctl = (const PgoCtl*)(dev + iCtl);
  B.efrom = (const int*)(dev + iFrom); B.eto = (const int*)(dev + iTo); B.Z = (const double*)(dev + iZ);
  B.fidx = (const int*)(dev + iFidx);
  B.X = (double*)(dout + oX); B.xpar = 16 * tV;
  B.e = (double*)(dwork + wE); B.Ji = (double*)(dwork + wJi); B.Jj = (double*)(dwork + wJj); B.ce = (double*)(dwork + wCe);
  B.blk_rc = (const int*)(dev + iRc); B.blk_start = (const int*)(dev + iStart); B.blk_item = (const int*)(dev + iItem);
  B.S = (double*)(dwork + wS); B.b = (double*)(dwork + wB); B.g = (double*)(dwork + wG); B.y = (double*)(dwork + wY);
  B.x = (double*)(dwork + wX); B.dotp = (double*)(dwork + wDot); B.bad = dwork + wBad; B.red = (double*)(dout + oRed);
  const GbbLdlt gl{(const GbbBig*)(dev + iBig), (const int*)(dev + iCtl + offsetof(PgoCtl, active)),
                   (int)(sizeof(PgoCtl) / sizeof(int)), B.S, B.g, B.y, B.x, (double*)(dwork + wWp), dwork + wNz, {}};
  const size_t bytes = L.in + L.out + L.work;
  for (int k = 0; k < P; ++k) out[k].scratch_bytes = bytes;
  auto blocks = [](long long n, int per) { return (unsigned)((n + per - 1) / per); };
  // the round's sums of every problem to the host
  auto sums = [&]() -> plf_status {
    PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in + oRed, B.red, 32 * (size_t)P, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    return PLF_OK;
  };
  // ---- round 0: the initial chi2 of every problem
  if (mE) {
    k_pgo_edge_chi2<<<dim3(blocks(mE, 128), P), 128, 0, cs>>>(B, 0);
    PLF_LAUNCH_CHECK(ctx);
  }
  k_pgo_reduce<<<dim3(1, P), PGO_RED, 0, cs>>>(B, 0);
  PLF_LAUNCH_CHECK(ctx);
  if (plf_status st = sums()) return st;
  std::vector<PgoLm> s(P);
  for (int k = 0; k < P; ++k) {
    s[k].chi = red[4 * k];
    s[k].lambda = opts->lambda_init;
    s[k].running = hp[k].nf && opts->max_iters > 0;   // nothing to optimise without free vertices
    plf_pgo_result& o = out[k];
    o.chi2_init = s[k].chi;
    o.iters = 0; o.stop = PLF_PGO_STOP_MAX_ITERS; o.trials = 0; o.n_trace = 0;
  }
  // ---- one trial of every running problem per round
  for (;;) {
    int rE = 0, rV = 0, rB = 0, rN = 0, running = 0, last = 0;
    bool lin = false;
    for (int k = 0; k < P; ++k) {
      const PgoLm& sk = s[k];
      ctl[k] = PgoCtl{sk.lambda, sk.running, sk.running && sk.trials == 0, sk.cur, 0};
      if (!sk.running) continue;
      ++running;
      last = k;
      lin |= sk.trials == 0;
      rE = std::max(rE, hp[k].ne); rV = std::max(rV, hp[k].nv); rB = std::max(rB, hp[k].nb);
      rN = std::max(rN, 6 * hp[k].nf);
    }
    if (!running) break;
    PLF_CUDA(ctx, cudaMemcpyAsync(dev + iCtl, ctl, sizeof(PgoCtl) * P, cudaMemcpyHostToDevice, cs));
    if (lin) {
      k_pgo_linearize<<<dim3(blocks(rE, 128), P), 128, 0, cs>>>(B);
      PLF_LAUNCH_CHECK(ctx);
    }
    k_pgo_zero<<<dim3((unsigned)std::min<long long>(2048, blocks((long long)rN * rN, 256)), P), 256, 0, cs>>>(B);
    PLF_LAUNCH_CHECK(ctx);
    k_pgo_assemble<<<dim3(rB, P), 64, 0, cs>>>(B);
    PLF_LAUNCH_CHECK(ctx);
    // the factorisation reads a table entry and a flag per CTA only where it must: one running problem passes its entry
    // by value (every round of plf_pose_graph), and a round in which every problem runs needs no flags
    GbbLdlt gr = gl;
    if (running == 1) { gr.big = nullptr; gr.one = hb[last]; gr.active = nullptr; }
    else if (running == P) gr.active = nullptr;
    if (plf_status st = gbb_ldlt(ctx, cs, gr, running == 1 ? 1 : P, rN)) return st;
    k_pgo_step<<<dim3(blocks(rV, 128), P), 128, 0, cs>>>(B);
    PLF_LAUNCH_CHECK(ctx);
    k_pgo_edge_chi2<<<dim3(blocks(rE, 128), P), 128, 0, cs>>>(B, 1);
    PLF_LAUNCH_CHECK(ctx);
    k_pgo_reduce<<<dim3(1, P), PGO_RED, 0, cs>>>(B, 1);
    PLF_LAUNCH_CHECK(ctx);
    if (plf_status st = sums()) return st;
    for (int k = 0; k < P; ++k)
      if (s[k].running) pgo_decide(s[k], red + 4 * k, opts->max_iters, out[k]);
  }
  // ---- the estimates back: both pose buffers in one copy, each problem's from the one holding its estimate
  if (tV) {
    PLF_CUDA(ctx, cudaMemcpyAsync(Xpin, B.X, 256 * (size_t)tV, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  }
  for (int k = 0; k < P; ++k) {
    if (hp[k].nv) memcpy(problems[k].T, Xpin + s[k].cur * 16 * tV + 16 * hp[k].vo, 128 * (size_t)hp[k].nv);
    out[k].chi2 = s[k].chi;
    out[k].lambda = s[k].lambda;
  }
  return PLF_OK;
}

}  // namespace

extern "C" plf_status plf_pose_graph(plf_ctx* ctx, const plf_pgo_opts* opts, const plf_pgo_problem* p, plf_pgo_result* out) {
  if (!ctx || !opts || !p || !out || p->n_v < 0 || p->n_e < 0 || opts->max_iters < 0 || out->trace_cap < 0 ||
      (out->trace_cap && !out->trace))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_pose_graph: bad arguments");
  return pgo_run(ctx, opts, 1, p, out, false);
}

extern "C" plf_status plf_pose_graph_batch(plf_ctx* ctx, const plf_pgo_opts* opts, int n_problems,
                                           const plf_pgo_problem* problems, plf_pgo_result* out) {
  return pgo_run(ctx, opts, n_problems, problems, out, true);
}
