// Loop-closure pose-graph optimisation on the GPU (DESIGN.md §1 row f7).
//
// Replaces the g2o part of MapHandler::loopClosureOptimizationCovGraphG2O (src/mapHandler.cpp:4185-4410):
// computeInitialGuess() and optimize(maxItersPGO) of g2o's OptimizationAlgorithmLevenberg over VertexSE3 / EdgeSE3 with
// identity information.  The host keeps g2o's control flow (oracle/pgo.py restates it); the numerical work runs here:
//   k_pgo_linearize   one thread per edge, once per iteration: E = Z^-1 X_i^-1 X_j, e = MQT(E) and the Jacobians J_i, J_j
//                     at the iteration's estimate, reused by every trial of the iteration
//   k_pgo_assemble    one CTA per non-zero 6 x 6 block of the lower triangle of H: the block's contributions summed in
//                     ascending edge order (a per-block edge list built once per call), written with + lambda I into
//                     the dense system S; the diagonal blocks also write b = -sum J^T e.  No float atomics: two calls
//                     are bit-identical.
//   plf_ldlt_tiled    the tiled LDL^T and the two substitutions of plf_global_ba (lba.cu), unchanged
//   k_pgo_step        one thread per vertex: X_t = X (+) x, the pivot check on D and x (lambda x + b) per free vertex
//   k_pgo_edge_chi2   one thread per edge: e^T e at a given estimate
//   k_pgo_reduce      one CTA: chi2, sum x (lambda x + b) and the pivot flag, each summed in a fixed order
// One 4-double copy per trial goes to the host for the trial's decision.
#include <math.h>

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

__global__ void __launch_bounds__(128) k_pgo_linearize(PgoDev d) {
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k >= d.ne) return;
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

// kind 0: J_i^T J_i, 1: J_j^T J_j, 2: J_i^T J_j (the block row is the edge's `from`), 3: J_j^T J_i
__global__ void __launch_bounds__(64) k_pgo_assemble(PgoDev d, double lambda) {
  const int blk = blockIdx.x, t = threadIdx.x, n = 6 * d.nf;
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
__global__ void __launch_bounds__(128) k_pgo_step(PgoDev d, double lambda) {
  const int v = blockIdx.x * 128 + threadIdx.x;
  if (v >= d.nv) return;
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

__global__ void __launch_bounds__(128) k_pgo_edge_chi2(PgoDev d, const double* X) {
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k >= d.ne) return;
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
__global__ void __launch_bounds__(PGO_RED) k_pgo_reduce(PgoDev d, int nf) {
  __shared__ double sh[PGO_RED];
  const int t = threadIdx.x;
  double c = 0.0, s = 0.0, b = 0.0;
  for (int i = t; i < d.ne; i += PGO_RED) c += d.ce[i];
  for (int i = t; i < nf; i += PGO_RED) { s += d.dotp[i]; b += d.bad[i]; }
  c = pgo_block_sum(c, sh);
  s = pgo_block_sum(s, sh);
  b = pgo_block_sum(b, sh);
  if (t == 0) { d.red[0] = c; d.red[1] = s; d.red[2] = b; d.red[3] = 0.0; }
}

}  // namespace

extern "C" plf_status plf_pose_graph(plf_ctx* ctx, const plf_pgo_opts* opts, const plf_pgo_problem* p, plf_pgo_result* out) {
  const char* fn = "plf_pose_graph";
  if (!ctx || !opts || !p || !out || p->n_v < 0 || p->n_e < 0 || opts->max_iters < 0 || out->trace_cap < 0 ||
      (out->trace_cap && !out->trace))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments", fn);
  // g2o takes a non-positive user lambda as "derive one from H"; both call sites pass 1e-10, so anything else is refused
  if (!(opts->lambda_init > 0.0 && opts->lambda_init <= 1.7976931348623157e308))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: lambda_init %g is not a positive finite number", fn, opts->lambda_init);
  const int nv = p->n_v, ne = p->n_e;
  if ((nv && (!p->T || !p->fixed)) || (ne && (!p->from || !p->to || !p->Z)))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: null array", fn);
  std::vector<int> deg(nv, 0);
  for (int k = 0; k < ne; ++k) {
    const int a = p->from[k], b = p->to[k];
    if (a < 0 || a >= nv || b < 0 || b >= nv || a == b)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: edge %d joins vertices %d and %d (%d vertices)", fn, k, a, b, nv);
    deg[a]++; deg[b]++;
  }
  // the system's blocks: the free vertices with edges, in id order
  std::vector<int> fidx(nv, -1);
  int nf = 0;
  for (int v = 0; v < nv; ++v)
    if (!p->fixed[v] && deg[v]) fidx[v] = nf++;
  if (nf > 4096) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d free vertices with edges (limit 4096)", fn, nf);
  for (size_t i = 0; i < (size_t)nv * 16; ++i)
    if (!isfinite(p->T[i])) return plf_fail(ctx, PLF_ERR_INVALID, "%s: non-finite pose of vertex %d", fn, (int)(i / 16));
  for (size_t i = 0; i < (size_t)ne * 16; ++i)
    if (!isfinite(p->Z[i])) return plf_fail(ctx, PLF_ERR_INVALID, "%s: non-finite measurement of edge %d", fn, (int)(i / 16));
  // every connected component with edges holds a fixed vertex (else its system is singular up to the damping)
  {
    std::vector<int> root(nv);
    for (int v = 0; v < nv; ++v) root[v] = v;
    auto find = [&](int v) { while (root[v] != v) v = root[v] = root[root[v]]; return v; };
    for (int k = 0; k < ne; ++k) root[find(p->from[k])] = find(p->to[k]);
    std::vector<uint8_t> anchored(nv, 0);
    for (int v = 0; v < nv; ++v)
      if (p->fixed[v]) anchored[find(v)] = 1;
    for (int k = 0; k < ne; ++k)
      if (!anchored[find(p->from[k])])
        return plf_fail(ctx, PLF_ERR_INVALID, "%s: the component of edge %d has no fixed vertex", fn, k);
  }
  // ---- initial guess (g2o computeInitialGuess): breadth-first from the fixed vertices in ascending id, each vertex's
  // edges in the order given; a reached free vertex takes parent * Z (parent = from) or parent * Z^-1
  std::vector<double> X(p->T, p->T + (size_t)nv * 16);
  {
    std::vector<int> adj_start(nv + 1, 0), adj((size_t)2 * ne);
    for (int v = 0; v < nv; ++v) adj_start[v + 1] = adj_start[v] + deg[v];
    std::vector<int> fill(adj_start.begin(), adj_start.end() - 1);
    for (int k = 0; k < ne; ++k) { adj[fill[p->from[k]]++] = k; adj[fill[p->to[k]]++] = k; }
    std::vector<uint8_t> seen(nv);
    std::vector<int> queue;
    queue.reserve(nv);
    for (int v = 0; v < nv; ++v) {
      seen[v] = p->fixed[v] ? 1 : 0;
      if (p->fixed[v]) queue.push_back(v);
    }
    for (size_t h = 0; h < queue.size(); ++h) {
      const int v = queue[h];
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
  std::vector<int> blk_rc;
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
  std::vector<int> blk_start(nb + 1, 0), blk_item(nit);
  for (int i = 0; i < nit; ++i) blk_start[it_blk[i] + 1]++;
  for (int b = 0; b < nb; ++b) blk_start[b + 1] += blk_start[b];
  {
    std::vector<int> fill(blk_start.begin(), blk_start.end() - 1);
    for (int i = 0; i < nit; ++i) blk_item[fill[it_blk[i]]++] = it_val[i];
  }
  // ---- device buffers (scratch slot PLF_SCR_BA)
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int n = 6 * nf, nt = (n + PLF_LDLT_TILE - 1) / PLF_LDLT_TILE;
  PgoDev d;
  d.nv = nv; d.ne = ne; d.nf = nf; d.nb = nb;
  int *dFrom, *dTo, *dFidx, *dRc, *dStart, *dItem;
  double *dZ, *dWp;
  uint8_t* dNz;
  const size_t one = 1;
  DevBufList scr;
  scr.add(dFrom, std::max((size_t)ne, one)); scr.add(dTo, std::max((size_t)ne, one));
  scr.add(dZ, std::max((size_t)ne, one) * 16); scr.add(dFidx, std::max((size_t)nv, one));
  scr.add(d.X, std::max((size_t)nv, one) * 16); scr.add(d.Xt, std::max((size_t)nv, one) * 16);
  scr.add(d.e, std::max((size_t)ne, one) * 6); scr.add(d.Ji, std::max((size_t)ne, one) * 36);
  scr.add(d.Jj, std::max((size_t)ne, one) * 36); scr.add(d.ce, std::max((size_t)ne, one));
  scr.add(dRc, std::max((size_t)nb, one) * 2); scr.add(dStart, (size_t)nb + 1); scr.add(dItem, std::max((size_t)nit, one));
  scr.add(d.S, std::max((size_t)n * n, one));
  scr.add(d.b, std::max((size_t)n, one)); scr.add(d.g, std::max((size_t)n, one));
  scr.add(d.y, std::max((size_t)n, one)); scr.add(d.x, std::max((size_t)n, one));
  scr.add(d.dotp, std::max((size_t)nf, one)); scr.add(d.bad, std::max((size_t)nf, one)); scr.add(d.red, 4);
  scr.add(dWp, std::max((size_t)nt, one) * PLF_LDLT_TILE * PLF_LDLT_TILE); scr.add(dNz, std::max((size_t)nt * nt, one));
  if (plf_status st = scr.carve(ctx, PLF_SCR_BA)) return st;
  out->scratch_bytes = scr.bytes();
  d.efrom = dFrom; d.eto = dTo; d.Z = dZ; d.fidx = dFidx; d.blk_rc = dRc; d.blk_start = dStart; d.blk_item = dItem;
  cudaStream_t cs = ctx->stream;
  if (ne) {
    PLF_CUDA(ctx, cudaMemcpyAsync(dFrom, p->from, (size_t)ne * 4, cudaMemcpyHostToDevice, cs));
    PLF_CUDA(ctx, cudaMemcpyAsync(dTo, p->to, (size_t)ne * 4, cudaMemcpyHostToDevice, cs));
    PLF_CUDA(ctx, cudaMemcpyAsync(dZ, p->Z, (size_t)ne * 128, cudaMemcpyHostToDevice, cs));
  }
  if (nv) {
    PLF_CUDA(ctx, cudaMemcpyAsync(dFidx, fidx.data(), (size_t)nv * 4, cudaMemcpyHostToDevice, cs));
    PLF_CUDA(ctx, cudaMemcpyAsync(d.X, X.data(), (size_t)nv * 128, cudaMemcpyHostToDevice, cs));
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(dRc, blk_rc.data(), (size_t)std::max(nb, 1) * 8, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dStart, blk_start.data(), (size_t)(nb + 1) * 4, cudaMemcpyHostToDevice, cs));
  if (nit) PLF_CUDA(ctx, cudaMemcpyAsync(dItem, blk_item.data(), (size_t)nit * 4, cudaMemcpyHostToDevice, cs));
  double h_red[4];
  // chi2 at `Xp` (and, for a trial, the step's two other sums of nf free vertices) into h_red
  auto evaluate = [&](const double* Xp, int nf_sums) -> plf_status {
    if (ne) {
      k_pgo_edge_chi2<<<(ne + 127) / 128, 128, 0, cs>>>(d, Xp);
      PLF_LAUNCH_CHECK(ctx);
    }
    k_pgo_reduce<<<1, PGO_RED, 0, cs>>>(d, nf_sums);
    PLF_LAUNCH_CHECK(ctx);
    PLF_CUDA(ctx, cudaMemcpyAsync(h_red, d.red, 32, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    return PLF_OK;
  };
  plf_status st;
  if ((st = evaluate(d.X, 0))) return st;
  double chi = h_red[0], lambda = opts->lambda_init;
  out->chi2_init = chi;
  out->iters = 0; out->stop = PLF_PGO_STOP_MAX_ITERS; out->trials = 0; out->n_trace = 0;
  // ---- g2o's OptimizationAlgorithmLevenberg::solve, once per iteration (nothing to optimise without free vertices)
  double ni = 2.0;   // g2o's _ni is a double: it doubles on every rejected trial and must reach lambda's overflow
  for (int iter = 0; nf && iter < opts->max_iters; ++iter) {
    k_pgo_linearize<<<(ne + 127) / 128, 128, 0, cs>>>(d);
    PLF_LAUNCH_CHECK(ctx);
    int trials = 0;
    double rho = 0.0;
    do {
      PLF_CUDA(ctx, cudaMemsetAsync(d.S, 0, (size_t)n * n * 8, cs));
      k_pgo_assemble<<<nb, 64, 0, cs>>>(d, lambda);
      PLF_LAUNCH_CHECK(ctx);
      if ((st = plf_ldlt_tiled(ctx, cs, nf, d.S, d.g, d.y, d.x, dWp, dNz))) return st;
      k_pgo_step<<<(nv + 127) / 128, 128, 0, cs>>>(d, lambda);
      PLF_LAUNCH_CHECK(ctx);
      if ((st = evaluate(d.Xt, nf))) return st;
      const double chi_t = h_red[2] != 0.0 ? 1.7976931348623157e308 : h_red[0];   // failed solve: DBL_MAX
      rho = (chi - chi_t) / (h_red[1] + 1e-3);
      const bool accept = rho > 0.0 && isfinite(chi_t);
      if (out->n_trace < out->trace_cap) {
        plf_pgo_trial& tr = out->trace[out->n_trace++];
        tr.iter = iter; tr.accepted = accept; tr.lambda = lambda; tr.chi = chi; tr.chi_t = chi_t; tr.rho = rho;
      }
      if (accept) {
        const double alpha = std::min(1.0 - pow(2.0 * rho - 1.0, 3), 2.0 / 3.0);
        lambda *= std::max(1.0 / 3.0, alpha);
        ni = 2;
        std::swap(d.X, d.Xt);
        chi = chi_t;
      } else {
        lambda *= ni;
        ni *= 2;
      }
      ++trials;
    } while (rho < 0.0 && trials < 10);
    out->iters = iter + 1;
    out->trials += trials;
    if (trials == 10 || rho == 0.0 || !isfinite(lambda)) {
      out->stop = trials == 10 ? PLF_PGO_STOP_TRIALS : (rho == 0.0 ? PLF_PGO_STOP_RHO_ZERO : PLF_PGO_STOP_LAMBDA);
      break;
    }
  }
  if (nv) {
    PLF_CUDA(ctx, cudaMemcpyAsync(p->T, d.X, (size_t)nv * 128, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  }
  out->chi2 = chi;
  out->lambda = lambda;
  return PLF_OK;
}
