// Relative pose between two keyframes for loop closure / keyframe refinement (SURVEY §8(f) f2): the composition
// MapHandler::isLoopClosure (src/mapHandler.cpp:3192-3300) -> computeRelativePoseRobustGN (:3566-3957) performs, on
// the operators of this library: match() twice (points :3223, lines :3249) -> the two-stage robust Gauss-Newton of
// plf_gn_pose (the in-tree twin of optimizePose IS this function, :3566-3872) -> the acceptance tests (:3875-3906) ->
// pose_inc and the surviving correspondences (:3909-3950).
//
// One call checks P candidate pairs (plf_loop_closure_pose_batch; the single call is P = 1): one upload, every kernel on
// ctx->stream, one download, one host synchronisation.  A kind's inputs are concatenated over the problems that match it
// (the kind is enabled and both keyframes have features of it); the problem table (LcProb) holds each problem's offsets,
// counts and pair capacities, a second table its camera.  The chain:
//   k_hamming_knn2_mma  forward and (best_lr_matches) reverse 2-NN of every problem of a kind: match()'s knnMatch
//   k_nnr_mutual        the ratio and mutual checks: match()'s matches_12
//   k_lc_rows           the inlier-ratio pre-condition (:3273-3299) and the order-preserving compaction of the matches into
//                       solver rows in ascending i1, the single call's order (it fixes the solver's summation)
//   k_gn_pose           over the problems that passed the pre-condition (its active flags), each with its camera
//   k_lc_decide         the acceptance tests, the surviving pairs in row order and pose_inc
// The three ratios that are plain quotients of counts (inl_ratio_pt / _ls and ratio_inliers) are recomputed on the host
// from the downloaded counts with the same expressions, so that a 0 / 0 gives the host's NaN, as it always did.
#include <float.h>
#include <math.h>

#include "plf_internal.h"
#include "plf_se3.cuh"

#define LC_MAX_FEATURES 65535   // per kind and keyframe: the kNN keys pack the train index in 16 bits (plf_match's limit)
#define LC_MAX_PROBLEMS 65535   // problems per call: grid.y of the kNN and NNR launches
#define LC_ROWS_THREADS 256
#define LC_ROWS_WARPS (LC_ROWS_THREADS / 32)
#define LC_DECIDE_WARPS 4

// One problem as the kernels read it; kind 0 = points, 1 = lines.
struct LcProb {
  long long qo[2], to[2];   // first kf0 / kf1 row in the kind's flat arrays (a matched kind)
  int n0[2], n1[2];         // kf0 / kf1 feature counts, the pre-condition's denominators
  int matched[2];           // the kind is enabled and both keyframes have features of it
  int has_pairs[2], cap[2]; // the caller's pair array is non-NULL, and its capacity
};

// The flat arrays of one kind over the problems that match it (problem p's rows from qo / to).
struct LcKindDev {
  const double* x0;    // kf0: P [3] (points) / sP [3] (lines)
  const double* x0e;   // kf0: eP [3] (lines)
  const double* x1;    // kf1: pl [2] (points) / le [3] (lines)
  const int32_t* m12;  // [nq] kf1 row or -1
  double* ga;          // solver rows: P / sP [3]
  double* gb;          //              obs [2] / eP [3]
  double* gc;          //              le [3] (lines)
  uint8_t* inl;        // [nq] inlier flags of the rows
  int32_t* idx;        // [nq][2] (i1, i2) of each row
  int32_t* pairs;      // out [nq][2] the surviving pairs in row order
};

struct LcArgs {
  const LcProb* prob;
  int n;
  int has_points, has_lines;
  plf_lc_params lc;
  LcKindDev k[2];
  int* rows;                  // [n][2] solver rows per kind (the solver's np / nl)
  int* active;                // [n] passed the pre-condition
  const plf_pose_result* gn;  // [n]
  plf_lc_result* out;         // [n], zeroed before the chain
  int* info;                  // [n][4] status, rows, inliers, pairs written
};

// max(100 common / n0, 100 common / n1) with std::max's NaN behaviour (x / 0 follows IEEE as in the reference: 0 / 0 when a
// frame is empty, and inf / nan compare false)
__host__ __device__ inline double lc_ratio(int common, int n0, int n1) {
  const double a = 100.0 * common / n0, b = 100.0 * common / n1;
  return a < b ? b : a;
}

// Order-preserving compaction of the rows i of [0, n) with m[i] >= 0 by one CTA of LC_ROWS_THREADS: emit(rank, i, m[i]).
// Returns the count to every thread.
template <class Emit>
__device__ __forceinline__ int lc_compact(const int32_t* __restrict__ m, int n, Emit emit) {
  __shared__ int wsum[LC_ROWS_WARPS];
  __shared__ int base;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += LC_ROWS_THREADS) {
    const int i = c0 + tid;
    const int j = i < n ? m[i] : -1;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, j >= 0);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    if (w == 0) {   // exclusive scan of the warp sums
      const int v = lane < LC_ROWS_WARPS ? wsum[lane] : 0;
      int s = v;
      for (int o = 1; o < LC_ROWS_WARPS; o <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += t;
      }
      if (lane < LC_ROWS_WARPS) wsum[lane] = s - v;
    }
    __syncthreads();
    if (j >= 0) emit(base + wsum[w] + __popc(bal & ((1u << lane) - 1u)), i, j);
    __syncthreads();
    if (tid == LC_ROWS_THREADS - 1) base += wsum[LC_ROWS_WARPS - 1] + __popc(bal);
    __syncthreads();
  }
  const int total = base;
  __syncthreads();   // base is reset by the next call
  return total;
}

// One CTA per problem: the solver rows of both kinds, their counts, the pre-condition (:3277-3299) and common_pt / _ls.
__global__ void __launch_bounds__(LC_ROWS_THREADS) k_lc_rows(LcArgs a) {
  const int p = blockIdx.x;
  const LcProb& q = a.prob[p];
  int cnt[2] = {0, 0};
  for (int kd = 0; kd < 2; ++kd) {
    if (!q.matched[kd]) continue;   // uniform over the CTA
    const LcKindDev& k = a.k[kd];
    const long long qo = q.qo[kd], to = q.to[kd];
    if (kd == 0)
      cnt[0] = lc_compact(k.m12 + qo, q.n0[0], [&](int r, int i, int j) {
        const size_t g = qo + r, s = qo + i, t = to + j;
        for (int c = 0; c < 3; ++c) k.ga[3 * g + c] = k.x0[3 * s + c];
        for (int c = 0; c < 2; ++c) k.gb[2 * g + c] = k.x1[2 * t + c];
        k.inl[g] = 1;
        k.idx[2 * g] = i; k.idx[2 * g + 1] = j;
      });
    else
      cnt[1] = lc_compact(k.m12 + qo, q.n0[1], [&](int r, int i, int j) {
        const size_t g = qo + r, s = qo + i, t = to + j;
        for (int c = 0; c < 3; ++c) {
          k.ga[3 * g + c] = k.x0[3 * s + c];
          k.gb[3 * g + c] = k.x0e[3 * s + c];
          k.gc[3 * g + c] = k.x1[3 * t + c];
        }
        k.inl[g] = 1;
        k.idx[2 * g] = i; k.idx[2 * g + 1] = j;
      });
  }
  if (threadIdx.x == 0) {
    plf_lc_result& o = a.out[p];
    o.common_pt = cnt[0];
    o.common_ls = cnt[1];
    const double rp = lc_ratio(cnt[0], q.n0[0], q.n1[0]), rl = lc_ratio(cnt[1], q.n0[1], q.n1[1]);
    const double th = a.lc.lc_inlier_ratio;
    bool cond = false;
    if (a.has_points && a.has_lines) cond = rp > th && rl > th;
    else if (a.has_points) cond = rp > th;
    else if (a.has_lines) cond = rl > th;
    a.rows[2 * p] = cnt[0];
    a.rows[2 * p + 1] = cnt[1];
    a.active[p] = cond ? 1 : 0;
  }
}

// pose_inc = logmap_se3(inverse_se3(expmap_se3(x_inc))) with plf_se3's expmap.  Out of line: inlined into k_lc_decide,
// its registers would spill around the trigonometric slow paths.
__device__ __noinline__ void lc_pose_inc(const double* x, double* pose_inc) {
  double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, nx[6];
  for (int i = 0; i < 6; ++i) nx[i] = -x[i];
  d_update_pose(T, nx);   // expmap_se3(x_inc) = I * inverse(exp(-x_inc)), as plf_se3 computes it
  d_inverse_se3(T, T);
  d_logmap(T, pose_inc);
}

// One warp per problem that passed the pre-condition: the acceptance block (:3875-3906), then - accepted - the inlier
// correspondences in row order and pose_inc = logmap(inverse(expmap(x_inc))) (:3909-3951).
__global__ void __launch_bounds__(32 * LC_DECIDE_WARPS) k_lc_decide(LcArgs a) {
  const int p = blockIdx.x * LC_DECIDE_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= a.n || !a.active[p]) return;   // uniform over the warp
  const LcProb& q = a.prob[p];
  const plf_pose_result& r = a.gn[p];
  plf_lc_result& o = a.out[p];
  int* info = a.info + 4 * p;
  const int np = a.rows[2 * p], nl = a.rows[2 * p + 1];
  int pass = 0;
  if (lane == 0) {
    o.estimated = 1;
    o.err = r.err;
    for (int i = 0; i < 6; ++i) o.x_inc[i] = r.x[i];
    o.max_cov_eig = plf_sym6_max_eig(r.cov);
    o.t = sqrt(r.x[0] * r.x[0] + r.x[1] * r.x[1] + r.x[2] * r.x[2]);
    o.r = sqrt(r.x[3] * r.x[3] + r.x[4] * r.x[4] + r.x[5] * r.x[5]) * 180.f / 3.1415926535897932384626433832795;
    const bool lc_res = r.err < a.lc.lc_res, lc_unc = o.max_cov_eig < a.lc.lc_unc;
    const bool lc_inl = true;  // the reference overrides its own inlier-ratio test (`lc_inl = true;`, :3900)
    const bool lc_trs = o.t < a.lc.lc_trs, lc_rot = o.r < a.lc.lc_rot;
    pass = lc_res && lc_unc && lc_inl && lc_trs && lc_rot;
    info[1] = np + nl;
    info[2] = r.n_inliers_pt + r.n_inliers_ls;
    info[3] = pass;
  }
  if (!__shfl_sync(0xFFFFFFFFu, pass, 0)) return;
  int kept[2] = {0, 0};
  for (int kd = 0; kd < 2; ++kd) {
    const LcKindDev& k = a.k[kd];
    const long long qo = q.qo[kd];
    const int rows = kd ? nl : np;
    for (int c0 = 0; c0 < rows; c0 += 32) {
      const int i = c0 + lane;
      const bool keep = i < rows && k.inl[qo + i];
      const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
      if (keep) {
        const size_t d = qo + kept[kd] + __popc(bal & ((1u << lane) - 1u));
        k.pairs[2 * d] = k.idx[2 * (qo + i)];
        k.pairs[2 * d + 1] = k.idx[2 * (qo + i) + 1];
      }
      kept[kd] += __popc(bal);
    }
  }
  if (lane) return;
  o.n_pt = kept[0];
  o.n_ls = kept[1];
  if ((q.has_pairs[0] && kept[0] > q.cap[0]) || (q.has_pairs[1] && kept[1] > q.cap[1])) {
    info[0] = PLF_ERR_CAPACITY;
    return;
  }
  lc_pose_inc(r.x, o.pose_inc);
  o.accepted = 1;
}

namespace {

// A kind is matched when it is enabled and both keyframes have features of it (:3220, :3246).
bool lc_matched(const plf_params& P, int kd, const plf_lc_keyframe& a, const plf_lc_keyframe& b) {
  return kd ? P.has_lines && a.n_ls > 0 && b.n_ls > 0 : P.has_points && a.n_pt > 0 && b.n_pt > 0;
}

// The single call's host-side rules for one problem; the messages start with pfx.
plf_status lc_check(plf_ctx* ctx, const char* pfx, const plf_lc_problem& q) {
  const plf_lc_keyframe *a = q.kf0, *b = q.kf1;
  if (!a || !b || a->n_pt < 0 || b->n_pt < 0 || a->n_ls < 0 || b->n_ls < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments (kf0 and kf1 are required, counts must be >= 0)", pfx);
  const plf_params& P = ctx->params;
  if (lc_matched(P, 0, *a, *b) && (!a->pdesc || !b->pdesc || !a->P || !b->pl))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: point arrays missing", pfx);
  if (lc_matched(P, 1, *a, *b) && (!a->ldesc || !b->ldesc || !a->sP || !a->eP || !b->le))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: line arrays missing", pfx);
  for (int kd = 0; kd < 2; ++kd)
    if (lc_matched(P, kd, *a, *b) && std::max(kd ? a->n_ls : a->n_pt, kd ? b->n_ls : b->n_pt) > LC_MAX_FEATURES)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: %d / %d %s in kf0 / kf1 (at most %d per keyframe)", pfx,
                      kd ? a->n_ls : a->n_pt, kd ? b->n_ls : b->n_pt, kd ? "lines" : "points", LC_MAX_FEATURES);
  return PLF_OK;
}

// The staged layout of one kind over the problems that match it.
struct LcKindPlan {
  std::vector<int> probs;   // the call's problems that match the kind, in order
  size_t nq = 0, nt = 0;    // total kf0 / kf1 rows
  int max_n0 = 0, max_n1 = 0;
  size_t knn, nnr, qd, td, x0, x0e, x1;   // in
  size_t pairs;                            // out
  size_t b12, s12, b21, s21, m12, ga, gb, gc, inl, idx;   // work
};

void plan_kind(LcKindPlan& k, StagedLayout& L, bool lines, bool best_lr) {
  const size_t q = k.nq, t = k.nt, P = k.probs.size();
  k.knn = L.take_in((best_lr ? 2 : 1) * P * sizeof(KnnProblem));
  k.nnr = L.take_in(P * sizeof(NnrProblem));
  k.qd = L.take_in(q * 32);
  k.td = L.take_in(t * 32);
  k.x0 = L.take_in(q * 24);
  k.x0e = L.take_in(lines ? q * 24 : 0);
  k.x1 = L.take_in(t * (lines ? 24 : 16));
  k.pairs = L.take_out(q * 8);
  k.b12 = L.take_work(q * 4);
  k.s12 = L.take_work(q * 4);
  k.b21 = L.take_work(t * 4);
  k.s21 = L.take_work(t * 4);
  k.m12 = L.take_work(q * 4);
  k.ga = L.take_work(q * 24);
  k.gb = L.take_work(q * (lines ? 24 : 16));
  k.gc = L.take_work(lines ? q * 24 : 0);
  k.inl = L.take_work(q);
  k.idx = L.take_work(q * 8);
}

// The whole call over problems whose host-side rules hold.  batch: the messages name the problem.
plf_status lc_run(plf_ctx* ctx, const char* fn, bool batch, const plf_lc_params& lc, int n, plf_lc_problem* pr,
                  const std::vector<const plf_camera*>& cams) {
  if (n == 0) return PLF_OK;
  const plf_params& P = ctx->params;
  const bool best_lr = P.best_lr_matches != 0;
  std::vector<LcProb> tab(n);
  LcKindPlan plan[2];
  for (int p = 0; p < n; ++p) {
    const plf_lc_keyframe &a = *pr[p].kf0, &b = *pr[p].kf1;
    LcProb& t = tab[p];
    t = {};
    for (int kd = 0; kd < 2; ++kd) {
      LcKindPlan& k = plan[kd];
      t.n0[kd] = kd ? a.n_ls : a.n_pt;
      t.n1[kd] = kd ? b.n_ls : b.n_pt;
      t.has_pairs[kd] = (kd ? pr[p].ls_pairs : pr[p].pt_pairs) != nullptr;
      t.cap[kd] = kd ? pr[p].cap_ls : pr[p].cap_pt;
      t.matched[kd] = lc_matched(P, kd, a, b);
      if (!t.matched[kd]) continue;
      t.qo[kd] = (long long)k.nq;
      t.to[kd] = (long long)k.nt;
      k.nq += t.n0[kd];
      k.nt += t.n1[kd];
      k.max_n0 = std::max(k.max_n0, t.n0[kd]);
      k.max_n1 = std::max(k.max_n1, t.n1[kd]);
      k.probs.push_back(p);
    }
  }
  StagedLayout L;
  const size_t oprob = L.take_in(n * sizeof(LcProb)), ocam = L.take_in(n * sizeof(PlfPairCam));
  const size_t ognp = L.take_in(n * sizeof(GnProblem));
  for (int kd = 0; kd < 2; ++kd) plan_kind(plan[kd], L, kd == 1, best_lr);
  const size_t ores = L.take_out(n * sizeof(plf_lc_result)), oinfo = L.take_out((size_t)n * 16);
  const size_t orows = L.take_work((size_t)n * 8), oact = L.take_work((size_t)n * 4);
  const size_t ogn = L.take_work(n * sizeof(plf_pose_result));
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_LC, &pin, &dev)) return st;
  uint8_t *pout = pin + L.in, *dout = dev + L.in, *dwork = dev + L.in + L.out;
  // ---- stage: tables, then every matched kind's rows ----
  memcpy(pin + oprob, tab.data(), n * sizeof(LcProb));
  LcArgs args = {};
  args.prob = (const LcProb*)(dev + oprob);
  args.n = n;
  args.has_points = P.has_points ? 1 : 0;
  args.has_lines = P.has_lines ? 1 : 0;
  args.lc = lc;
  args.rows = (int*)(dwork + orows);
  args.active = (int*)(dwork + oact);
  args.gn = (const plf_pose_result*)(dwork + ogn);
  args.out = (plf_lc_result*)(dout + ores);
  args.info = (int*)(dout + oinfo);
  for (int kd = 0; kd < 2; ++kd) {
    const LcKindPlan& k = plan[kd];
    LcKindDev& d = args.k[kd];
    d.x0 = (const double*)(dev + k.x0); d.x0e = (const double*)(dev + k.x0e); d.x1 = (const double*)(dev + k.x1);
    d.m12 = (const int32_t*)(dwork + k.m12);
    d.ga = (double*)(dwork + k.ga); d.gb = (double*)(dwork + k.gb); d.gc = (double*)(dwork + k.gc);
    d.inl = dwork + k.inl;
    d.idx = (int32_t*)(dwork + k.idx);
    d.pairs = (int32_t*)(dout + k.pairs);
    const size_t np = k.probs.size();
    KnnProblem* kn = (KnnProblem*)(pin + k.knn);
    NnrProblem* nr = (NnrProblem*)(pin + k.nnr);
    uint32_t *b12 = (uint32_t*)(dwork + k.b12), *s12 = (uint32_t*)(dwork + k.s12);
    uint32_t *b21 = (uint32_t*)(dwork + k.b21), *s21 = (uint32_t*)(dwork + k.s21);
    const float nnr = kd ? P.min_ratio_12_l : P.min_ratio_12_p;
    for (size_t j = 0; j < np; ++j) {
      const int p = k.probs[j];
      const plf_lc_keyframe &a = *pr[p].kf0, &b = *pr[p].kf1;
      const size_t qo = (size_t)tab[p].qo[kd], to = (size_t)tab[p].to[kd];
      const int n0 = tab[p].n0[kd], n1 = tab[p].n1[kd];
      memcpy(pin + k.qd + 32 * qo, kd ? a.ldesc : a.pdesc, (size_t)n0 * 32);
      memcpy(pin + k.td + 32 * to, kd ? b.ldesc : b.pdesc, (size_t)n1 * 32);
      memcpy(pin + k.x0 + 24 * qo, kd ? a.sP : a.P, (size_t)n0 * 24);
      if (kd) memcpy(pin + k.x0e + 24 * qo, a.eP, (size_t)n0 * 24);
      memcpy(pin + k.x1 + (kd ? 24 : 16) * to, kd ? b.le : b.pl, (size_t)n1 * (kd ? 24 : 16));
      const uint32_t* dq = (const uint32_t*)(dev + k.qd + 32 * qo);
      const uint32_t* dt = (const uint32_t*)(dev + k.td + 32 * to);
      kn[j] = {dq, dt, nullptr, nullptr, n0, n1, b12 + qo, s12 + qo, nullptr};
      if (best_lr) kn[np + j] = {dt, dq, nullptr, nullptr, n1, n0, b21 + to, s21 + to, nullptr};
      nr[j] = {b12 + qo, s12 + qo, b21 + to, s21 + to, nullptr, nullptr, n0, n1, nnr, best_lr ? 1 : 0,
               (int32_t*)(dwork + k.m12) + qo, nullptr};
    }
  }
  GnProblem* gp = (GnProblem*)(pin + ognp);
  PlfPairCam* cam = (PlfPairCam*)(pin + ocam);
  for (int p = 0; p < n; ++p) {
    const size_t qp = (size_t)tab[p].qo[0], ql = (size_t)tab[p].qo[1];
    const LcKindDev &dp = args.k[0], &dl = args.k[1];
    gp[p] = {dp.ga + 3 * qp, dp.gb + 2 * qp, dp.inl + qp, args.rows + 2 * p, 0,
             dl.ga + 3 * ql, dl.gb + 3 * ql, dl.gc + 3 * ql, dl.inl + ql, args.rows + 2 * p + 1, 0,
             nullptr, (plf_pose_result*)(dwork + ogn) + p};
    const plf_camera& c = *cams[p];
    cam[p] = {c.fx, c.fy, c.cx, c.cy, c.b};
  }
  // ---- upload, the chain, download ----
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemsetAsync(dout, 0, L.out, cs));
  plf_status st;
  for (int kd = 0; kd < 2; ++kd) {   // match() (:3223, :3249)
    const LcKindPlan& k = plan[kd];
    const int np = (int)k.probs.size();
    if (!np) continue;
    const KnnProblem* kn = (const KnnProblem*)(dev + k.knn);
    if ((st = plf_launch_knn2(ctx, cs, kn, np, k.max_n0))) return st;
    if (best_lr && (st = plf_launch_knn2(ctx, cs, kn + np, np, k.max_n1))) return st;
    if ((st = plf_launch_nnr(ctx, cs, (const NnrProblem*)(dev + k.nnr), np, k.max_n0))) return st;
  }
  k_lc_rows<<<n, LC_ROWS_THREADS, 0, cs>>>(args);
  PLF_LAUNCH_CHECK(ctx);
  // computeRelativePoseRobustGN (:3566-3872): both stages stop on DBL_EPSILON, iteration counts from the config
  const plf_gn_opts o = {P.homog_th, P.max_iters, P.max_iters_ref, DBL_EPSILON, DBL_EPSILON, DBL_EPSILON};
  if ((st = plf_launch_gn(ctx, cs, (const GnProblem*)(dev + ognp), n, o, (const PlfPairCam*)(dev + ocam), args.active)))
    return st;
  k_lc_decide<<<(n + LC_DECIDE_WARPS - 1) / LC_DECIDE_WARPS, 32 * LC_DECIDE_WARPS, 0, cs>>>(args);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(pout, dout, L.out, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  // ---- outputs ----
  int first = -1;
  for (int p = 0; p < n; ++p) {
    plf_lc_problem& q = pr[p];
    const LcProb& t = tab[p];
    const int* info = (const int*)(pout + oinfo) + 4 * p;
    memcpy(&q.out, pout + ores + p * sizeof(plf_lc_result), sizeof(plf_lc_result));
    q.out.inl_ratio_pt = lc_ratio(q.out.common_pt, t.n0[0], t.n1[0]);
    q.out.inl_ratio_ls = lc_ratio(q.out.common_ls, t.n0[1], t.n1[1]);
    if (q.out.estimated) q.out.ratio_inliers = (double)info[2] / (double)info[1];
    if (info[3]) {   // the acceptance tests passed: the pairs the capacities hold
      int32_t* dst[2] = {q.pt_pairs, q.ls_pairs};
      const int kept[2] = {q.out.n_pt, q.out.n_ls};
      for (int kd = 0; kd < 2; ++kd) {
        const int m = std::min(kept[kd], t.cap[kd]);
        if (dst[kd] && m > 0) memcpy(dst[kd], pout + plan[kd].pairs + 8 * (size_t)t.qo[kd], (size_t)m * 8);
      }
    }
    q.status = info[0];
    if (q.status && first < 0) first = p;
  }
  if (first >= 0) {
    const plf_lc_result& o = pr[first].out;
    if (batch)
      return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: problem %d: %d point / %d line correspondences exceed the caller's capacity",
                      fn, first, o.n_pt, o.n_ls);
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d point / %d line correspondences exceed the caller's capacity", fn, o.n_pt,
                    o.n_ls);
  }
  return PLF_OK;
}

}  // namespace

extern "C" plf_status plf_loop_closure_pose(plf_ctx* ctx, const plf_lc_params* lc, const plf_lc_keyframe* kf0,
                                            const plf_lc_keyframe* kf1, plf_lc_result* out, int32_t* pt_pairs,
                                            int cap_pt, int32_t* ls_pairs, int cap_ls) {
  if (!ctx || !lc || !kf0 || !kf1 || !out || kf0->n_pt < 0 || kf1->n_pt < 0 || kf0->n_ls < 0 || kf1->n_ls < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_loop_closure_pose: bad arguments");
  memset(out, 0, sizeof *out);
  const char* fn = "plf_loop_closure_pose";
  plf_lc_problem q = {kf0, kf1, pt_pairs, cap_pt, ls_pairs, cap_ls, {}, 0};
  if (plf_status st = lc_check(ctx, fn, q)) return st;
  const plf_status st = lc_run(ctx, fn, false, *lc, 1, &q, {&ctx->cam});
  if (st == PLF_OK || q.status) *out = q.out;
  return st;
}

extern "C" plf_status plf_loop_closure_pose_batch(plf_ctx* ctx, const plf_lc_params* lc, int n_problems,
                                                  plf_lc_problem* problems, const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = "plf_loop_closure_pose_batch";
  if (!lc || n_problems < 0 || (n_problems && !problems))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments (lc, n_problems = %d, problems)", fn, n_problems);
  if (n_problems > LC_MAX_PROBLEMS)
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: n_problems = %d exceeds %d", fn, n_problems, LC_MAX_PROBLEMS);
  std::vector<const plf_camera*> cams;
  if (plf_status st = plf_problem_cameras(ctx, fn, n_problems, seq, cams)) return st;
  char pfx[80];
  for (int p = 0; p < n_problems; ++p) {
    snprintf(pfx, sizeof pfx, "%s: problem %d", fn, p);
    if (plf_status st = lc_check(ctx, pfx, problems[p])) return st;
  }
  return lc_run(ctx, fn, true, *lc, n_problems, problems, cams);
}
