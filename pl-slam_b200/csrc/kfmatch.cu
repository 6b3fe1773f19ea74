// Keyframe-to-keyframe and local-map-to-keyframe matching on the device (SURVEY §8(f) f1): the matching and gate parts of
// MapHandler::matchKF2KFPoints / matchKF2KFLines (src/mapHandler.cpp:234-278, :365-426) and matchMap2KFPoints /
// matchMap2KFLines (:532-632, :634-752).  oracle/kfmatching.py restates the same control flow.
//
// One call matches P problems (plf_match_*_batch; the single calls are P = 1): one upload, all kernels on ctx->stream,
// one download, one host synchronisation.  A kind's inputs are concatenated into flat arrays; its device problem table
// (KfProb) holds each problem's offsets, counts, camera, transform, kmin and fallback flag.  The windowed matcher's arrays
// are laid out at a uniform capacity per problem, K (queries) and Kt (train) = the kind's largest counts.  Per kind:
//   k_kf_query_vis      projection of every query (previous-keyframe feature / landmark) with DT / Twf, in f64, and its
//                       visibility flag (map: `use` and the strict image bounds with Z > 0; KF-to-KF: all)
//   k_kf_compact        order-preserving compaction of the visible queries / the unmatched keyframe features (one CTA per
//                       problem and set); the counts stay on the device
//   k_kf_query_gather   compact query rows: grid cells of the projection, descriptors
//   k_kf_train_gather   compact train rows: cells of pl (points), end-point cells + normalised scaled direction (lines)
//   matchGrid           plf_launch_match_grid_batch over the kind's problems, rectangular (queries x train) [fast_matching]
//   match()             plf_launch_knn2 (forward, then reverse) / plf_launch_nnr over the problems whose host-known sizes
//                       allow the fallback, on the device counts
//   k_kf_select         the fallback decision (k_mg_select's rule with each function's own condition), then - map - the
//                       epipolar gate and the scatter back to original indices with an atomic count of the rejects
// Every kernel but k_kf_compact is gridded (chunk, problem), so a CTA never mixes problems.
#include "plf_internal.h"
#include "plf_geom.cuh"
#include "plf_se3.cuh"

#define KF_MAX_LANDMARKS 65535   // 16-bit train index of the kNN keys (the reverse problem's train set is the queries)
#define KF_MAX_FEATURES 8192     // the bound of plf_match_grid_*
#define KF_MAX_PROBLEMS 65535    // problems per batch call: grid.y of the (chunk, problem) grids

struct KfCam { double fx, fy, cx, cy, w, h, iw, ih; };

// One problem of one kind, as the kernels read it.
struct KfProb {
  long long qo, to;   // its first row in the flat query / train arrays
  int nq, nt;         // its query / train counts before compaction
  int bf;             // the brute-force fallback can be taken (host upper bounds)
  int kmin;           // min_pt_matches / min_ls_matches
  int has_lm;         // the train features carry landmark indices (kf_*_lm): only those at -1 are train rows
  KfCam cam;          // the problem's fx, fy, cx, cy; its sequence's image size and grid scales
  double T[16];       // DT / Twf, row-major
};

struct KfKind {
  int lines;
  int map;        // 1: map-to-keyframe (visibility, gate, scatter); 0: keyframe-to-keyframe
  int q_scale;    // 1: query cells in grid units; 0: in pixels (matchKF2KFLines, :392-393)
  int K, Kt;      // per-problem capacity of the [P][K] / [P][Kt] arrays: the kind's largest nq / nt
  const KfProb* prob;
  // inputs, flat (problem p's rows from prob[p].qo / prob[p].to)
  const double* X; int x_stride;        // queries: 3-D points / start points (rows of x_stride doubles)
  const double* XE;                     // lines: end points (same stride)
  const uint8_t* use;                   // [nq] (map) or null
  const uint8_t* qdesc_in;              // [nq][32]
  const double2* t_s; const double2* t_e;   // train: pl (points) / spl, epl (lines)
  const double* t_le;                   // [nt][3] (map lines)
  const int* t_lm;                      // [nt] (rows of problems with has_lm)
  const uint8_t* tdesc_in;              // [nt][32]
  // work, flat
  uint8_t* flag;
  double2* proj;                        // [nq][1|2]
  int* q_orig; int* t_orig;             // compacted row -> the problem's own index
  int32_t* m_bf;
  int* cnt;                             // [P][2] compacted query, train counts
  // work, [P][K] / [P][Kt]
  int* q_geo; int* t_geo; double* t_dir;
  uint8_t* dq; uint8_t* dt;
  int32_t* m_g;
  // outputs
  int32_t* out;                         // flat [nq]
  int* stat;                            // [P][8]: [0] matches before the gate, [1] gate rejects, [2] windowed,
                                        // [3] brute force, [4] fell back
};

__global__ void __launch_bounds__(256) k_kf_query_vis(KfKind k) {
  const KfProb& q = k.prob[blockIdx.y];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= q.nq) return;
  const size_t g = q.qo + i;
  const KfCam& c = q.cam;
  double Ps[3];
  d_transform(q.T, k.X + g * k.x_stride, Ps);
  const double2 ps = plf_project(c.fx, c.fy, c.cx, c.cy, Ps[0], Ps[1], Ps[2]);
  bool vis = ps.x > 0 && ps.x < c.w && ps.y > 0 && ps.y < c.h && Ps[2] > 0.0;   // :551
  if (k.lines) {
    double Pe[3];
    d_transform(q.T, k.XE + g * k.x_stride, Pe);
    const double2 pe = plf_project(c.fx, c.fy, c.cx, c.cy, Pe[0], Pe[1], Pe[2]);
    vis = vis && pe.x > 0 && pe.x < c.w && pe.y > 0 && pe.y < c.h && Pe[2] > 0.0;   // :654-655
    k.proj[2 * g] = ps;
    k.proj[2 * g + 1] = pe;
  } else {
    k.proj[g] = ps;
  }
  if (k.map) vis = vis && (!k.use || k.use[g]);
  else vis = true;
  k.flag[g] = vis ? 1 : 0;
}

// Order-preserving compaction of [0, n) by one CTA of 1024: keep(i) = flag[i] (flag != null), else lm[i] == -1 (lm !=
// null), else 1.
__device__ __forceinline__ void kf_compact(const uint8_t* __restrict__ flag, const int* __restrict__ lm, int n,
                                           int* __restrict__ orig, int* __restrict__ count) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    bool keep = false;
    if (i < n) keep = flag ? flag[i] != 0 : (lm ? lm[i] == -1 : true);
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    if (w == 0) {   // exclusive scan of the 32 warp sums
      const int v = wsum[lane];
      int s = v;
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += t;
      }
      wsum[lane] = s - v;
    }
    __syncthreads();
    if (keep) orig[base + wsum[w] + __popc(bal & ((1u << lane) - 1u))] = i;
    __syncthreads();
    if (tid == 1023) base += wsum[31] + __popc(bal);
    __syncthreads();
  }
  if (tid == 0) *count = base;
}

// grid (problem, set): set 0 compacts the visible queries, set 1 the unmatched train features.
__global__ void __launch_bounds__(1024) k_kf_compact(KfKind k) {
  const int p = blockIdx.x;
  const KfProb& q = k.prob[p];
  if (blockIdx.y == 0) kf_compact(k.flag + q.qo, nullptr, q.nq, k.q_orig + q.qo, k.cnt + 2 * p);
  else kf_compact(nullptr, q.has_lm ? k.t_lm + q.to : nullptr, q.nt, k.t_orig + q.to, k.cnt + 2 * p + 1);
}

__global__ void __launch_bounds__(256) k_kf_query_gather(KfKind k) {
  const int p = blockIdx.y;
  const KfProb& q = k.prob[p];
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= k.cnt[2 * p]) return;
  const size_t i = q.qo + k.q_orig[q.qo + j], r = (size_t)p * k.K + j;
  const double sx = k.q_scale ? q.cam.iw : 1.0, sy = k.q_scale ? q.cam.ih : 1.0;
  if (k.lines) {
    const double2 ps = k.proj[2 * i], pe = k.proj[2 * i + 1];
    int* d = k.q_geo + r * 4;
    d[0] = plf_qcell(ps.x * sx); d[1] = plf_qcell(ps.y * sy); d[2] = plf_qcell(pe.x * sx); d[3] = plf_qcell(pe.y * sy);
  } else {
    const double2 pp = k.proj[i];
    k.q_geo[2 * r] = plf_qcell(pp.x * sx);
    k.q_geo[2 * r + 1] = plf_qcell(pp.y * sy);
  }
  const uint4* s = reinterpret_cast<const uint4*>(k.qdesc_in) + 2 * i;
  uint4* d = reinterpret_cast<uint4*>(k.dq) + 2 * r;
  d[0] = s[0]; d[1] = s[1];
}

__global__ void __launch_bounds__(256) k_kf_train_gather(KfKind k) {
  const int p = blockIdx.y;
  const KfProb& q = k.prob[p];
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= k.cnt[2 * p + 1]) return;
  const size_t i = q.to + k.t_orig[q.to + j], r = (size_t)p * k.Kt + j;
  if (k.lines) {
    plf_train_line(k.t_s[i], k.t_e[i], q.cam.iw, q.cam.ih, k.t_geo + r * 4, k.t_dir + r * 2);
  } else {
    const double2 pp = k.t_s[i];
    k.t_geo[2 * r] = mg_cell(pp.x * q.cam.iw);
    k.t_geo[2 * r + 1] = mg_cell(pp.y * q.cam.ih);
  }
  const uint4* s = reinterpret_cast<const uint4*>(k.tdesc_in) + 2 * i;
  uint4* d = reinterpret_cast<uint4*>(k.dt) + 2 * r;
  d[0] = s[0]; d[1] = s[1];
}

// Fallback: KF-to-KF `n_curr > min && n_prev > min && matches < min` (:274-276, :421-423); map `n_visible > min &&
// n_visible > min && matches < min` (:594-595, :709-710: the visible-landmark count twice).  matches = the windowed count
// with fast_matching, else 0, and then - fallback not taken - matches_12 stays empty.  Map pairs then pass the gate
// (:612-613 points: |pf_map - pl| < max_kf_epip_p; :727-729 lines: le . (p, 1) < max_kf_epip_l at both ends, signed) or
// count as a reject (--matches, :628, :748).
__global__ void __launch_bounds__(256) k_kf_select(KfKind k, int fast, double gate) {
  const int p = blockIdx.y;
  const KfProb& q = k.prob[p];
  int* stat = k.stat + 8 * p;
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int n1 = k.cnt[2 * p], n2 = k.cnt[2 * p + 1], kmin = q.kmin;
  const bool empty = n1 == 0 || n2 == 0;
  const int mg = fast ? stat[2] : 0;
  const bool fall = !empty && q.bf && (k.map ? (n1 > kmin && n1 > kmin) : (n2 > kmin && n1 > kmin)) && mg < kmin;
  if (j == 0) {
    stat[0] = empty ? 0 : (fall ? stat[3] : mg);
    stat[4] = fall ? 1 : 0;
  }
  if (empty || j >= n1) return;
  const int t = fall ? k.m_bf[q.qo + j] : (fast ? k.m_g[(size_t)p * k.K + j] : -1);
  if (t < 0) return;
  const size_t i = q.qo + k.q_orig[q.qo + j];
  const int f = k.t_orig[q.to + t];
  if (k.map) {
    bool pass;
    if (k.lines) {
      const double* le = k.t_le + 3 * (q.to + f);
      const double2 ps = k.proj[2 * i], pe = k.proj[2 * i + 1];
      const double e0 = le[0] * ps.x + le[1] * ps.y + le[2], e1 = le[0] * pe.x + le[1] * pe.y + le[2];
      pass = e0 < gate && e1 < gate;
    } else {
      const double2 pp = k.proj[i], o = k.t_s[q.to + f];
      const double dx = pp.x - o.x, dy = pp.y - o.y;
      pass = sqrt(dx * dx + dy * dy) < gate;
    }
    if (!pass) {
      atomicAdd(&stat[1], 1);
      return;
    }
  }
  k.out[i] = f;
}

namespace {

struct HostKind {   // host arrays of one kind of one problem
  const double* X; const double* XE; bool x_packed;   // x_packed: X holds [n][6] (start | end)
  const uint8_t* use; const uint8_t* qdesc;
  const double* ts; const double* te; const double* tle; const int32_t* tlm; const uint8_t* tdesc;
};

// One problem of a call, on the host.
struct HostProb {
  const double* T;
  const plf_camera* cam;
  bool active[2];        // the kind runs (else it returns 0 and every entry -1)
  int nq[2], nt[2];
  HostKind host[2];
  int32_t* outs[2];      // [nq]
  int* n_out[2];         // the reference's return value, or null
};

// The staged layout and host-known sizes of one kind over the problems where it is active.
struct KindPlan {
  std::vector<int> probs;   // the call's problems where the kind is active, in order
  std::vector<KfProb> tab;
  size_t nq = 0, nt = 0;    // total rows
  int K = 0, Kt = 0;        // largest nq / nt
  std::vector<int> bfp;     // rows of tab that can take the fallback
  int Kbf = 0, Ktbf = 0;    // their largest nq / nt
  // offsets (in: from 0; out: from in; work: from in + out)
  size_t prob, x, use, qd, ts, te, tle, tlm, td, kp, np;
  size_t out, stat;
  size_t flag, proj, qo, to, cnt, qg, tg, tdir, dq, dt, mg, mbf, keys;
};

void plan_kind(KindPlan& p, StagedLayout& L, bool lines, bool map) {
  const size_t q = p.nq, t = p.nt, P = p.probs.size(), K = p.K, Kt = p.Kt, nbf = p.bfp.size();
  p.prob = L.take_in(P * sizeof(KfProb));
  p.x = L.take_in(q * (lines ? 6 : 3) * 8);
  p.use = L.take_in(map ? q : 0);
  p.qd = L.take_in(q * 32);
  p.ts = L.take_in(t * 16);
  p.te = L.take_in(lines ? t * 16 : 0);
  p.tle = L.take_in(map && lines ? t * 24 : 0);
  p.tlm = L.take_in(t * 4);
  p.td = L.take_in(t * 32);
  p.kp = L.take_in(2 * nbf * sizeof(KnnProblem));
  p.np = L.take_in(nbf * sizeof(NnrProblem));
  p.out = L.take_out(q * 4);
  p.stat = L.take_out(P * 8 * 4);
  p.flag = L.take_work(q);
  p.proj = L.take_work(q * (lines ? 32 : 16));
  p.qo = L.take_work(q * 4);
  p.to = L.take_work(t * 4);
  p.cnt = L.take_work(P * 2 * 4);
  p.qg = L.take_work(P * K * (lines ? 16 : 8));
  p.tg = L.take_work(P * Kt * (lines ? 16 : 8));
  p.tdir = L.take_work(lines ? P * Kt * 16 : 0);
  p.dq = L.take_work(P * K * 32);
  p.dt = L.take_work(P * Kt * 32);
  p.mg = L.take_work(P * K * 4);
  p.mbf = L.take_work(q * 4);
  p.keys = L.take_work((2 * q + 2 * t) * 4);
}

// Stages the host inputs of one problem of a planned kind (pinned, same offsets as on the device).
void stage_prob(const KindPlan& p, const KfProb& r, const HostKind& h, uint8_t* pin, bool lines, bool map) {
  const size_t q = r.nq, t = r.nt;
  double* x = (double*)(pin + p.x) + r.qo * (lines ? 6 : 3);
  if (lines) {
    if (h.x_packed) memcpy(x, h.X, q * 48);
    else for (size_t i = 0; i < q; ++i) { memcpy(x + 6 * i, h.X + 3 * i, 24); memcpy(x + 6 * i + 3, h.XE + 3 * i, 24); }
  } else {
    memcpy(x, h.X, q * 24);
  }
  if (map) {   // NULL use = every landmark
    if (h.use) memcpy(pin + p.use + r.qo, h.use, q);
    else memset(pin + p.use + r.qo, 1, q);
  }
  memcpy(pin + p.qd + 32 * r.qo, h.qdesc, q * 32);
  memcpy(pin + p.ts + 16 * r.to, h.ts, t * 16);
  if (lines) memcpy(pin + p.te + 16 * r.to, h.te, t * 16);
  if (h.tle) memcpy(pin + p.tle + 24 * r.to, h.tle, t * 24);
  if (h.tlm) memcpy(pin + p.tlm + 4 * r.to, h.tlm, t * 4);
  memcpy(pin + p.td + 32 * r.to, h.tdesc, t * 32);
}

KfKind kind_args(const KindPlan& p, uint8_t* dev, size_t in, size_t out, bool lines, bool map) {
  uint8_t* o = dev + in;
  uint8_t* w = dev + in + out;
  KfKind k = {};
  k.lines = lines; k.map = map; k.q_scale = map || !lines;
  k.K = p.K; k.Kt = p.Kt;
  k.prob = (const KfProb*)(dev + p.prob);
  k.X = (const double*)(dev + p.x); k.x_stride = lines ? 6 : 3; k.XE = k.X + 3;
  k.use = map ? dev + p.use : nullptr;
  k.qdesc_in = dev + p.qd;
  k.t_s = (const double2*)(dev + p.ts); k.t_e = (const double2*)(dev + p.te);
  k.t_le = (const double*)(dev + p.tle);
  k.t_lm = (const int*)(dev + p.tlm);
  k.tdesc_in = dev + p.td;
  k.flag = w + p.flag; k.proj = (double2*)(w + p.proj);
  k.q_orig = (int*)(w + p.qo); k.t_orig = (int*)(w + p.to);
  k.m_bf = (int32_t*)(w + p.mbf);
  k.cnt = (int*)(w + p.cnt);
  k.q_geo = (int*)(w + p.qg); k.t_geo = (int*)(w + p.tg); k.t_dir = (double*)(w + p.tdir);
  k.dq = w + p.dq; k.dt = w + p.dt;
  k.m_g = (int32_t*)(w + p.mg);
  k.out = (int32_t*)(o + p.out); k.stat = (int*)(o + p.stat);
  return k;
}

// The match() problems of the rows that can take the fallback: the forward kNN [nbf], the reverse [nbf] and the NNR /
// mutual check [nbf], each problem's work rows addressed as its kernels address them.  work: the device work part.
void prepare_bf(const KindPlan& p, const KfKind& k, uint8_t* work, float nnr, int best_lr, KnnProblem* kp, NnrProblem* np) {
  uint32_t *b12 = (uint32_t*)(work + p.keys), *s12 = b12 + p.nq, *b21 = b12 + 2 * p.nq, *s21 = b21 + p.nt;
  const size_t nbf = p.bfp.size();
  for (size_t j = 0; j < nbf; ++j) {
    const int r = p.bfp[j];
    const KfProb& q = p.tab[r];
    const uint32_t* dq = (const uint32_t*)(k.dq + (size_t)r * p.K * 32);
    const uint32_t* dt = (const uint32_t*)(k.dt + (size_t)r * p.Kt * 32);
    const int *nq = k.cnt + 2 * r, *nt = nq + 1;
    kp[j] = {dq, dt, nq, nt, 0, 0, b12 + q.qo, s12 + q.qo, nullptr};
    kp[nbf + j] = {dt, dq, nt, nq, 0, 0, b21 + q.to, s21 + q.to, nullptr};
    np[j] = {b12 + q.qo, s12 + q.qo, b21 + q.to, s21 + q.to, nq, nt, 0, 0, nnr, best_lr, k.m_bf + q.qo, k.stat + 8 * r + 3};
  }
}

// The launches of one kind: 5 + [fast_matching: the windowed matcher's 3 (points) / 4 (lines) per chunk of problems] +
// [some problem can fall back: 2 or 3] + 1.
plf_status run_kind(plf_ctx* ctx, const KindPlan& p, const KfKind& k, uint8_t* dev, int fast, float nnr, double gate,
                    plf_scratch_slot slot) {
  cudaStream_t cs = ctx->stream;
  const plf_params& P = ctx->params;
  const int np = (int)p.probs.size();
  const dim3 gq((p.K + 255) / 256, np), gt((p.Kt + 255) / 256, np);
  PLF_CUDA(ctx, cudaMemsetAsync(k.stat, 0, (size_t)np * 8 * 4, cs));
  k_kf_query_vis<<<gq, 256, 0, cs>>>(k);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_compact<<<dim3(np, 2), 1024, 0, cs>>>(k);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_query_gather<<<gq, 256, 0, cs>>>(k);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_train_gather<<<gt, 256, 0, cs>>>(k);
  PLF_LAUNCH_CHECK(ctx);
  plf_status st;
  if (fast) {
    const int ws = P.matching_f2f_ws;
    MgbArgs a = {};
    a.g = {PLF_GRID_COLS, PLF_GRID_ROWS, ws, ws, ws, ws};
    a.is_lines = k.lines; a.K = p.K; a.Kt = p.Kt; a.best_lr = P.best_lr_matches ? 1 : 0;
    a.clip = k.lines;
    a.nnr = nnr; a.line_sim_th = (double)P.line_sim_th;
    a.q_geo = k.q_geo; a.t_geo = k.t_geo; a.t_dir = k.t_dir;
    a.d1 = k.dq; a.d1_stride = (size_t)p.K * 32; a.d2 = k.dt; a.d2_stride = (size_t)p.Kt * 32;
    a.n1 = k.cnt; a.n2 = k.cnt + 1; a.n1_stride = a.n2_stride = 2;
    a.m12 = k.m_g; a.m12_stride = p.K; a.count = k.stat + 2; a.count_stride = 8;
    if ((st = plf_launch_match_grid_batch(ctx, a, np, p.K, p.Kt, slot, cs))) return st;
  }
  const int nbf = (int)p.bfp.size();
  if (nbf) {
    const KnnProblem* dkp = (const KnnProblem*)(dev + p.kp);
    if ((st = plf_launch_knn2(ctx, cs, dkp, nbf, p.Kbf))) return st;
    if (P.best_lr_matches && (st = plf_launch_knn2(ctx, cs, dkp + nbf, nbf, p.Ktbf))) return st;
    if ((st = plf_launch_nnr(ctx, cs, (const NnrProblem*)(dev + p.np), nbf, p.Kbf))) return st;
  }
  k_kf_select<<<gq, 256, 0, cs>>>(k, fast, gate);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// The whole call over problems whose host-side rules hold: plan, stage, upload, both kinds' launches, download, and the
// outputs of every problem (an inactive kind: 0 and every entry -1).
plf_status kf_run(plf_ctx* ctx, bool map, const plf_kf_match_opts* o, const std::vector<HostProb>& hp) {
  const plf_params& P = ctx->params;
  KindPlan plan[2];
  StagedLayout L;
  for (int kd = 0; kd < 2; ++kd) {
    KindPlan& p = plan[kd];
    const int kmin = kd ? P.min_ls_matches : P.min_pt_matches;
    for (size_t i = 0; i < hp.size(); ++i) {
      const HostProb& h = hp[i];
      if (!h.active[kd]) continue;
      KfProb r = {};
      r.qo = (long long)p.nq; r.to = (long long)p.nt;
      r.nq = h.nq[kd]; r.nt = h.nt[kd];
      // the fallback needs more than kmin queries (and, KF-to-KF, more than kmin train features)
      r.bf = r.nq > kmin && (map || r.nt > kmin);
      r.kmin = kmin;
      r.has_lm = h.host[kd].tlm != nullptr;
      // the grid and the visibility bounds of the problem's own image size (getWidth / getHeight, src/mapHandler.cpp:551)
      const plf_camera& c = *h.cam;
      r.cam = {c.fx, c.fy, c.cx, c.cy, (double)c.width, (double)c.height, PLF_GRID_COLS / (double)c.width,
               PLF_GRID_ROWS / (double)c.height};
      memcpy(r.T, h.T, sizeof r.T);
      if (r.bf) {
        p.bfp.push_back((int)p.tab.size());
        p.Kbf = std::max(p.Kbf, r.nq); p.Ktbf = std::max(p.Ktbf, r.nt);
      }
      p.probs.push_back((int)i);
      p.tab.push_back(r);
      p.nq += r.nq; p.nt += r.nt;
      p.K = std::max(p.K, r.nq); p.Kt = std::max(p.Kt, r.nt);
    }
    if (!p.probs.empty()) plan_kind(p, L, kd == 1, map);
  }
  if (plan[0].probs.size() + plan[1].probs.size()) {
    PLF_CUDA(ctx, cudaSetDevice(ctx->device));
    uint8_t *pin, *dev;
    if (plf_status st = L.acquire(ctx, PLF_SCR_KF, &pin, &dev)) return st;
    cudaStream_t cs = ctx->stream;
    KfKind args[2];
    for (int kd = 0; kd < 2; ++kd) {
      const KindPlan& p = plan[kd];
      if (p.probs.empty()) continue;
      for (size_t j = 0; j < p.probs.size(); ++j) stage_prob(p, p.tab[j], hp[p.probs[j]].host[kd], pin, kd == 1, map);
      memcpy(pin + p.prob, p.tab.data(), p.tab.size() * sizeof(KfProb));
      args[kd] = kind_args(p, dev, L.in, L.out, kd == 1, map);
      prepare_bf(p, args[kd], dev + L.in + L.out, kd ? P.min_ratio_12_l : P.min_ratio_12_p, P.best_lr_matches ? 1 : 0,
                 (KnnProblem*)(pin + p.kp), (NnrProblem*)(pin + p.np));
    }
    PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
    PLF_CUDA(ctx, cudaMemsetAsync(dev + L.in, 0xFF, L.out, cs));
    for (int kd = 0; kd < 2; ++kd) {
      if (plan[kd].probs.empty()) continue;
      plf_status st = run_kind(ctx, plan[kd], args[kd], dev, o->fast_matching ? 1 : 0, kd ? P.min_ratio_12_l : P.min_ratio_12_p,
                               kd ? o->max_kf_epip_l : o->max_kf_epip_p, kd ? PLF_SCR_KF_MGB_LS : PLF_SCR_KF_MGB_PT);
      if (st) return st;
    }
    PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in, dev + L.in, L.out, cudaMemcpyDeviceToHost, cs));
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    for (int kd = 0; kd < 2; ++kd) {
      const KindPlan& p = plan[kd];
      for (size_t j = 0; j < p.probs.size(); ++j) {
        const HostProb& h = hp[p.probs[j]];
        const int* stat = (const int*)(pin + L.in + p.stat) + 8 * j;
        memcpy(h.outs[kd], pin + L.in + p.out + 4 * p.tab[j].qo, (size_t)p.tab[j].nq * 4);
        if (h.n_out[kd]) *h.n_out[kd] = stat[0] - stat[1];
      }
    }
  }
  for (const HostProb& h : hp)
    for (int kd = 0; kd < 2; ++kd) {
      if (h.active[kd]) continue;
      if (h.outs[kd]) for (int i = 0; i < h.nq[kd]; ++i) h.outs[kd][i] = -1;
      if (h.n_out[kd]) *h.n_out[kd] = 0;
    }
  return PLF_OK;
}

bool bad_T(const double* T) {
  for (int i = 0; i < 16; ++i)
    if (!(T[i] == T[i])) return true;
  return false;
}

// plf_match_kf2kf's host-side rules; the messages start with pfx and the first names the required arguments (req).
plf_status kf2kf_check(plf_ctx* ctx, const char* pfx, const char* req, const plf_frame_view* prev, const plf_frame_view* curr,
                       const double* DT, const int32_t* m_pt, const int32_t* m_ls) {
  if (!prev || !curr || !DT || bad_T(DT)) return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s are required", pfx, req);
  const plf_frame_view* f[2] = {prev, curr};
  for (const plf_frame_view* v : f)
    if (v->n_pt < 0 || v->n_ls < 0 || v->n_pt > KF_MAX_FEATURES || v->n_ls > KF_MAX_FEATURES)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: n_pt=%d, n_ls=%d (each must be in [0, %d])", pfx, v->n_pt, v->n_ls,
                      KF_MAX_FEATURES);
  if ((prev->n_pt > 0 && (!prev->pt_P || !prev->pdesc || !m_pt)) || (curr->n_pt > 0 && (!curr->pt_pl || !curr->pdesc)) ||
      (prev->n_ls > 0 && (!prev->ls_sP || !prev->ls_eP || !prev->ldesc || !m_ls)) ||
      (curr->n_ls > 0 && (!curr->ls_spl || !curr->ls_epl || !curr->ldesc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: a feature array is NULL while its count is > 0", pfx);
  return PLF_OK;
}

HostProb kf2kf_prob(const plf_params& P, const plf_camera* cam, const plf_frame_view* prev, const plf_frame_view* curr,
                    const double* DT, int32_t* m_pt, int32_t* m_ls, int* n_pt, int* n_ls) {
  HostProb h = {};
  h.T = DT; h.cam = cam;
  // :243 / :368: a disabled kind, or either keyframe without stereo features of the kind, returns 0
  h.active[0] = P.has_points && prev->n_pt > 0 && curr->n_pt > 0;
  h.active[1] = P.has_lines && prev->n_ls > 0 && curr->n_ls > 0;
  h.nq[0] = prev->n_pt; h.nt[0] = curr->n_pt;
  h.nq[1] = prev->n_ls; h.nt[1] = curr->n_ls;
  h.host[0] = {prev->pt_P, nullptr, false, nullptr, prev->pdesc, curr->pt_pl, nullptr, nullptr, nullptr, curr->pdesc};
  h.host[1] = {prev->ls_sP, prev->ls_eP, false, nullptr, prev->ldesc, curr->ls_spl, curr->ls_epl, nullptr, nullptr, curr->ldesc};
  h.outs[0] = m_pt; h.outs[1] = m_ls;
  h.n_out[0] = n_pt; h.n_out[1] = n_ls;
  return h;
}

// plf_match_map2kf's host-side rules, as kf2kf_check.
plf_status map2kf_check(plf_ctx* ctx, const char* pfx, const char* req, const plf_local_map* map, const double* Twf,
                        const plf_frame_view* kf, const int32_t* lm_pt, const int32_t* lm_ls) {
  if (!map || !kf || !Twf || bad_T(Twf)) return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s are required", pfx, req);
  if (map->n_pt < 0 || map->n_ls < 0 || map->n_pt > KF_MAX_LANDMARKS || map->n_ls > KF_MAX_LANDMARKS)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: map n_pt=%d, n_ls=%d (each must be in [0, %d])", pfx, map->n_pt, map->n_ls,
                    KF_MAX_LANDMARKS);
  if (kf->n_pt < 0 || kf->n_ls < 0 || kf->n_pt > KF_MAX_FEATURES || kf->n_ls > KF_MAX_FEATURES)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: keyframe n_pt=%d, n_ls=%d (each must be in [0, %d])", pfx, kf->n_pt, kf->n_ls,
                    KF_MAX_FEATURES);
  if ((map->n_pt > 0 && (!map->pt_X || !map->pt_desc || !lm_pt)) || (map->n_ls > 0 && (!map->ls_X || !map->ls_desc || !lm_ls)) ||
      (kf->n_pt > 0 && (!kf->pt_pl || !kf->pdesc)) || (kf->n_ls > 0 && (!kf->ls_spl || !kf->ls_epl || !kf->ls_le || !kf->ldesc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: a landmark or feature array is NULL while its count is > 0", pfx);
  return PLF_OK;
}

HostProb map2kf_prob(const plf_params& P, const plf_camera* cam, const plf_local_map* map, const double* Twf,
                     const plf_frame_view* kf, const int32_t* kf_pt_lm, const int32_t* kf_ls_lm, int32_t* lm_pt,
                     int32_t* lm_ls, int* n_pt, int* n_ls) {
  HostProb h = {};
  h.T = Twf; h.cam = cam;
  // :542 / :644: a disabled kind or a keyframe without stereo features of the kind returns 0; so does an empty map (:571)
  h.active[0] = P.has_points && kf->n_pt > 0 && map->n_pt > 0;
  h.active[1] = P.has_lines && kf->n_ls > 0 && map->n_ls > 0;
  h.nq[0] = map->n_pt; h.nt[0] = kf->n_pt;
  h.nq[1] = map->n_ls; h.nt[1] = kf->n_ls;
  h.host[0] = {map->pt_X, nullptr, false, map->pt_use, map->pt_desc, kf->pt_pl, nullptr, nullptr, kf_pt_lm, kf->pdesc};
  h.host[1] = {map->ls_X, nullptr, true, map->ls_use, map->ls_desc, kf->ls_spl, kf->ls_epl, kf->ls_le, kf_ls_lm, kf->ldesc};
  h.outs[0] = lm_pt; h.outs[1] = lm_ls;
  h.n_out[0] = n_pt; h.n_out[1] = n_ls;
  return h;
}

// The batch calls' common argument rules and the camera of each problem (seq as in plf_local_ba_batch).
plf_status batch_cameras(plf_ctx* ctx, const char* fn, const plf_kf_match_opts* opts, int n, const void* problems,
                         const int32_t* seq, std::vector<const plf_camera*>& cams) {
  if (!opts || n < 0 || (n && !problems)) return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments (opts, n_problems = %d, problems)", fn, n);
  if (n > KF_MAX_PROBLEMS)
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: n_problems = %d exceeds %d", fn, n, KF_MAX_PROBLEMS);
  return plf_problem_cameras(ctx, fn, n, seq, cams);
}

}  // namespace

extern "C" plf_status plf_match_kf2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_frame_view* prev,
                                      const plf_frame_view* curr, const double DT[16], int32_t* m_pt, int32_t* m_ls,
                                      int* n_pt, int* n_ls) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_pt) *n_pt = 0;
  if (n_ls) *n_ls = 0;
  const char* fn = "plf_match_kf2kf";
  const char* req = "opts, prev, curr and a finite DT";
  if (!opts) return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s are required", fn, req);
  if (plf_status st = kf2kf_check(ctx, fn, req, prev, curr, DT, m_pt, m_ls)) return st;
  if (m_pt) for (int i = 0; i < prev->n_pt; ++i) m_pt[i] = -1;
  if (m_ls) for (int i = 0; i < prev->n_ls; ++i) m_ls[i] = -1;
  return kf_run(ctx, false, opts, {kf2kf_prob(ctx->params, &ctx->cam, prev, curr, DT, m_pt, m_ls, n_pt, n_ls)});
}

extern "C" plf_status plf_match_map2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_local_map* map, const double Twf[16],
                                       const plf_frame_view* kf, const int32_t* kf_pt_lm, const int32_t* kf_ls_lm, int32_t* lm_pt,
                                       int32_t* lm_ls, int* n_pt, int* n_ls) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_pt) *n_pt = 0;
  if (n_ls) *n_ls = 0;
  const char* fn = "plf_match_map2kf";
  const char* req = "opts, map, kf and a finite Twf";
  if (!opts) return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s are required", fn, req);
  if (plf_status st = map2kf_check(ctx, fn, req, map, Twf, kf, lm_pt, lm_ls)) return st;
  if (lm_pt) for (int i = 0; i < map->n_pt; ++i) lm_pt[i] = -1;
  if (lm_ls) for (int i = 0; i < map->n_ls; ++i) lm_ls[i] = -1;
  return kf_run(ctx, true, opts,
                {map2kf_prob(ctx->params, &ctx->cam, map, Twf, kf, kf_pt_lm, kf_ls_lm, lm_pt, lm_ls, n_pt, n_ls)});
}

extern "C" plf_status plf_match_kf2kf_batch(plf_ctx* ctx, const plf_kf_match_opts* opts, int n_problems,
                                            plf_kf2kf_problem* problems, const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = "plf_match_kf2kf_batch";
  std::vector<const plf_camera*> cams;
  if (plf_status st = batch_cameras(ctx, fn, opts, n_problems, problems, seq, cams)) return st;
  char pfx[80];
  for (int p = 0; p < n_problems; ++p) {
    const plf_kf2kf_problem& q = problems[p];
    snprintf(pfx, sizeof pfx, "%s: problem %d", fn, p);
    if (plf_status st = kf2kf_check(ctx, pfx, "prev, curr and a finite DT", q.prev, q.curr, q.DT, q.m_pt, q.m_ls)) return st;
  }
  std::vector<HostProb> hp(n_problems);
  for (int p = 0; p < n_problems; ++p) {
    plf_kf2kf_problem& q = problems[p];
    hp[p] = kf2kf_prob(ctx->params, cams[p], q.prev, q.curr, q.DT, q.m_pt, q.m_ls, &q.n_pt, &q.n_ls);
  }
  return kf_run(ctx, false, opts, hp);
}

extern "C" plf_status plf_match_map2kf_batch(plf_ctx* ctx, const plf_kf_match_opts* opts, int n_problems,
                                             plf_map2kf_problem* problems, const int32_t* seq) {
  if (!ctx) return PLF_ERR_INVALID;
  const char* fn = "plf_match_map2kf_batch";
  std::vector<const plf_camera*> cams;
  if (plf_status st = batch_cameras(ctx, fn, opts, n_problems, problems, seq, cams)) return st;
  char pfx[80];
  for (int p = 0; p < n_problems; ++p) {
    const plf_map2kf_problem& q = problems[p];
    snprintf(pfx, sizeof pfx, "%s: problem %d", fn, p);
    if (plf_status st = map2kf_check(ctx, pfx, "map, kf and a finite Twf", q.map, q.Twf, q.kf, q.lm_pt, q.lm_ls)) return st;
  }
  std::vector<HostProb> hp(n_problems);
  for (int p = 0; p < n_problems; ++p) {
    plf_map2kf_problem& q = problems[p];
    hp[p] = map2kf_prob(ctx->params, cams[p], q.map, q.Twf, q.kf, q.kf_pt_lm, q.kf_ls_lm, q.lm_pt, q.lm_ls, &q.n_pt, &q.n_ls);
  }
  return kf_run(ctx, true, opts, hp);
}
