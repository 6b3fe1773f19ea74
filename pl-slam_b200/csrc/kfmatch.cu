// Keyframe-to-keyframe and local-map-to-keyframe matching on the device (SURVEY §8(f) f1): the matching and gate parts of
// MapHandler::matchKF2KFPoints / matchKF2KFLines (src/mapHandler.cpp:234-278, :365-426) and matchMap2KFPoints /
// matchMap2KFLines (:532-632, :634-752).  oracle/kfmatching.py restates the same control flow.
//
// One call = one upload, all kernels on ctx->stream, one download.  Per kind (points, lines):
//   k_kf_query_vis      projection of every query (previous-keyframe feature / landmark) with DT / Twf, in f64, and its
//                       visibility flag (map: `use` and the strict image bounds with Z > 0; KF-to-KF: all)
//   k_kf_compact        order-preserving compaction of the visible queries / the unmatched keyframe features (one CTA);
//                       the count stays on the device
//   k_kf_query_gather   compact query rows: grid cells of the projection, descriptors
//   k_kf_train_gather   compact train rows: cells of pl (points), end-point cells + normalised scaled direction (lines)
//   matchGrid           plf_launch_match_grid_batch, one problem, rectangular (queries x train)      [fast_matching]
//   match()             plf_launch_knn2 / plf_launch_nnr on the device counts       [when the fallback can be taken]
//   k_kf_select         the fallback decision (k_mg_select's rule with each function's own condition), then - map - the
//                       epipolar gate and the scatter back to original indices with an atomic count of the rejects
#include "plf_internal.h"
#include "plf_geom.cuh"
#include "plf_se3.cuh"

#define KF_MAX_LANDMARKS 65535   // 16-bit train index of the kNN keys (the reverse problem's train set is the queries)
#define KF_MAX_FEATURES 8192     // the bound of plf_match_grid_*
#define KF_CELL_LIM 268435456.0  // query cells are clamped to +-2^28 (the reference's double -> int is undefined beyond
                                 // int range; the clamp keeps Bresenham differences inside int), NaN -> 0

__device__ __forceinline__ int kf_cell(double v) {
  if (v != v) return 0;
  return mg_cell(fmin(fmax(v, -KF_CELL_LIM), KF_CELL_LIM));
}

struct KfCam { double fx, fy, cx, cy, w, h, iw, ih; };

struct KfKind {
  int lines;
  int map;        // 1: map-to-keyframe (visibility, gate, scatter); 0: keyframe-to-keyframe
  int q_scale;    // 1: query cells in grid units; 0: in pixels (matchKF2KFLines, :392-393)
  int nq_in, nt_in;
  // inputs
  const double* X; int x_stride;        // queries: 3-D points / start points (rows of x_stride doubles)
  const double* XE;                     // lines: end points (same stride)
  const uint8_t* use;                   // [nq_in] or null
  const uint8_t* qdesc_in;              // [nq_in][32]
  const double2* t_s; const double2* t_e;   // train: pl (points) / spl, epl (lines)
  const double* t_le;                   // [nt_in][3] (map lines)
  const int* t_lm;                      // [nt_in] or null
  const uint8_t* tdesc_in;              // [nt_in][32]
  // work
  uint8_t* flag;
  double2* proj;                        // [nq_in][1|2]
  int* q_orig; int* t_orig;
  int* nq; int* nt;
  int* q_geo; int* t_geo; double* t_dir;
  uint8_t* dq; uint8_t* dt;
  int32_t* m_g; int32_t* m_bf;
  uint32_t* keys;                       // best12, second12 [nq_in]; best21, second21 [nt_in]
  // outputs
  int32_t* out;                         // [nq_in]
  int* stat;                            // [0] matches before the gate, [1] gate rejects, [2] windowed, [3] brute force, [4] fell back
};

__global__ void __launch_bounds__(256) k_kf_query_vis(KfKind k, const double* __restrict__ T, KfCam c) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= k.nq_in) return;
  double Ps[3];
  d_transform(T, k.X + (size_t)i * k.x_stride, Ps);
  const double2 ps = plf_project(c.fx, c.fy, c.cx, c.cy, Ps[0], Ps[1], Ps[2]);
  bool vis = ps.x > 0 && ps.x < c.w && ps.y > 0 && ps.y < c.h && Ps[2] > 0.0;   // :551
  if (k.lines) {
    double Pe[3];
    d_transform(T, k.XE + (size_t)i * k.x_stride, Pe);
    const double2 pe = plf_project(c.fx, c.fy, c.cx, c.cy, Pe[0], Pe[1], Pe[2]);
    vis = vis && pe.x > 0 && pe.x < c.w && pe.y > 0 && pe.y < c.h && Pe[2] > 0.0;   // :654-655
    k.proj[2 * (size_t)i] = ps;
    k.proj[2 * (size_t)i + 1] = pe;
  } else {
    k.proj[i] = ps;
  }
  if (k.map) vis = vis && (!k.use || k.use[i]);
  else vis = true;
  k.flag[i] = vis ? 1 : 0;
}

// Order-preserving compaction of [0, n): keep(i) = flag[i] (flag != null), else lm[i] == -1 (lm != null), else 1.
__global__ void __launch_bounds__(1024) k_kf_compact(const uint8_t* __restrict__ flag, const int* __restrict__ lm, int n,
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

__global__ void __launch_bounds__(256) k_kf_query_gather(KfKind k, KfCam c) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= *k.nq) return;
  const int i = k.q_orig[j];
  const double sx = k.q_scale ? c.iw : 1.0, sy = k.q_scale ? c.ih : 1.0;
  if (k.lines) {
    const double2 ps = k.proj[2 * (size_t)i], pe = k.proj[2 * (size_t)i + 1];
    int* d = k.q_geo + (size_t)j * 4;
    d[0] = kf_cell(ps.x * sx); d[1] = kf_cell(ps.y * sy); d[2] = kf_cell(pe.x * sx); d[3] = kf_cell(pe.y * sy);
  } else {
    const double2 p = k.proj[i];
    k.q_geo[2 * (size_t)j] = kf_cell(p.x * sx);
    k.q_geo[2 * (size_t)j + 1] = kf_cell(p.y * sy);
  }
  const uint4* s = reinterpret_cast<const uint4*>(k.qdesc_in) + 2 * (size_t)i;
  uint4* d = reinterpret_cast<uint4*>(k.dq) + 2 * (size_t)j;
  d[0] = s[0]; d[1] = s[1];
}

__global__ void __launch_bounds__(256) k_kf_train_gather(KfKind k, KfCam c) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= *k.nt) return;
  const int i = k.t_orig[j];
  if (k.lines) {
    plf_train_line(k.t_s[i], k.t_e[i], c.iw, c.ih, k.t_geo + (size_t)j * 4, k.t_dir + (size_t)j * 2);
  } else {
    const double2 p = k.t_s[i];
    k.t_geo[2 * (size_t)j] = mg_cell(p.x * c.iw);
    k.t_geo[2 * (size_t)j + 1] = mg_cell(p.y * c.ih);
  }
  const uint4* s = reinterpret_cast<const uint4*>(k.tdesc_in) + 2 * (size_t)i;
  uint4* d = reinterpret_cast<uint4*>(k.dt) + 2 * (size_t)j;
  d[0] = s[0]; d[1] = s[1];
}

// Fallback: KF-to-KF `n_curr > min && n_prev > min && matches < min` (:274-276, :421-423); map `n_visible > min &&
// n_visible > min && matches < min` (:594-595, :709-710: the visible-landmark count twice).  matches = the windowed count
// with fast_matching, else 0, and then - fallback not taken - matches_12 stays empty.  Map pairs then pass the gate
// (:612-613 points: |pf_map - pl| < max_kf_epip_p; :727-729 lines: le . (p, 1) < max_kf_epip_l at both ends, signed) or
// count as a reject (--matches, :628, :748).
__global__ void __launch_bounds__(256) k_kf_select(KfKind k, int fast, int bf, int kmin, double gate) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int n1 = *k.nq, n2 = *k.nt;
  const bool empty = n1 == 0 || n2 == 0;
  const int mg = fast ? k.stat[2] : 0;
  const bool fall = !empty && bf && (k.map ? (n1 > kmin && n1 > kmin) : (n2 > kmin && n1 > kmin)) && mg < kmin;
  if (j == 0) {
    k.stat[0] = empty ? 0 : (fall ? k.stat[3] : mg);
    k.stat[4] = fall ? 1 : 0;
  }
  if (empty || j >= n1) return;
  const int t = fall ? k.m_bf[j] : (fast ? k.m_g[j] : -1);
  if (t < 0) return;
  const int i = k.q_orig[j], f = k.t_orig[t];
  if (k.map) {
    bool pass;
    if (k.lines) {
      const double* le = k.t_le + 3 * (size_t)f;
      const double2 ps = k.proj[2 * (size_t)i], pe = k.proj[2 * (size_t)i + 1];
      const double e0 = le[0] * ps.x + le[1] * ps.y + le[2], e1 = le[0] * pe.x + le[1] * pe.y + le[2];
      pass = e0 < gate && e1 < gate;
    } else {
      const double2 p = k.proj[i], o = k.t_s[f];
      const double dx = p.x - o.x, dy = p.y - o.y;
      pass = sqrt(dx * dx + dy * dy) < gate;
    }
    if (!pass) {
      atomicAdd(&k.stat[1], 1);
      return;
    }
  }
  k.out[i] = f;
}

namespace {

struct KindPlan {
  bool active = false;
  int nq = 0, nt = 0;
  // offsets (in: from 0; out: from in; work: from in + out)
  size_t x, xe, use, qd, ts, te, tle, tlm, td;
  size_t out, stat;
  size_t flag, proj, qo, to, cnt, qg, tg, tdir, dq, dt, mg, mbf, keys, kp, np;
};

struct HostKind {   // host arrays of one kind
  const double* X; const double* XE; int x_stride; bool x_packed;   // x_packed: X holds [n][6] (start | end)
  const uint8_t* use; const uint8_t* qdesc;
  const double* ts; const double* te; const double* tle; const int32_t* tlm; const uint8_t* tdesc;
};

void plan_kind(KindPlan& p, StagedLayout& L, bool lines, bool map_lines_le) {
  const size_t q = p.nq, t = p.nt;
  p.x = L.take_in(q * (lines ? 6 : 3) * 8);
  p.xe = p.x;
  p.use = L.take_in(q);
  p.qd = L.take_in(q * 32);
  p.ts = L.take_in(t * 16);
  p.te = L.take_in(lines ? t * 16 : 0);
  p.tle = L.take_in(map_lines_le ? t * 24 : 0);
  p.tlm = L.take_in(t * 4);
  p.td = L.take_in(t * 32);
  p.kp = L.take_in(2 * sizeof(KnnProblem));
  p.np = L.take_in(sizeof(NnrProblem));
  p.out = L.take_out(q * 4);
  p.stat = L.take_out(8 * 4);
  p.flag = L.take_work(q);
  p.proj = L.take_work(q * (lines ? 32 : 16));
  p.qo = L.take_work(q * 4);
  p.to = L.take_work(t * 4);
  p.cnt = L.take_work(2 * 4);
  p.qg = L.take_work(q * (lines ? 16 : 8));
  p.tg = L.take_work(t * (lines ? 16 : 8));
  p.tdir = L.take_work(lines ? t * 16 : 0);
  p.dq = L.take_work(q * 32);
  p.dt = L.take_work(t * 32);
  p.mg = L.take_work(q * 4);
  p.mbf = L.take_work(q * 4);
  p.keys = L.take_work((2 * q + 2 * t) * 4);
}

// Stages the host inputs of a planned kind (pinned, same offsets as on the device).
void stage_kind(const KindPlan& p, const HostKind& h, uint8_t* pin, bool lines) {
  const size_t q = p.nq, t = p.nt;
  double* x = (double*)(pin + p.x);
  if (lines) {
    if (h.x_packed) memcpy(x, h.X, q * 48);
    else for (size_t i = 0; i < q; ++i) { memcpy(x + 6 * i, h.X + 3 * i, 24); memcpy(x + 6 * i + 3, h.XE + 3 * i, 24); }
  } else {
    memcpy(x, h.X, q * 24);
  }
  if (h.use) memcpy(pin + p.use, h.use, q);
  memcpy(pin + p.qd, h.qdesc, q * 32);
  memcpy(pin + p.ts, h.ts, t * 16);
  if (lines) memcpy(pin + p.te, h.te, t * 16);
  if (h.tle) memcpy(pin + p.tle, h.tle, t * 24);
  if (h.tlm) memcpy(pin + p.tlm, h.tlm, t * 4);
  memcpy(pin + p.td, h.tdesc, t * 32);
}

KfKind kind_args(const KindPlan& p, uint8_t* dev, size_t in, size_t out, bool lines, bool map, const HostKind& h) {
  uint8_t* o = dev + in;
  uint8_t* w = dev + in + out;
  KfKind k = {};
  k.lines = lines; k.map = map; k.q_scale = map || !lines;
  k.nq_in = p.nq; k.nt_in = p.nt;
  k.X = (const double*)(dev + p.x); k.x_stride = lines ? 6 : 3; k.XE = k.X + 3;
  k.use = h.use ? dev + p.use : nullptr;
  k.qdesc_in = dev + p.qd;
  k.t_s = (const double2*)(dev + p.ts); k.t_e = (const double2*)(dev + p.te);
  k.t_le = (const double*)(dev + p.tle);
  k.t_lm = h.tlm ? (const int*)(dev + p.tlm) : nullptr;
  k.tdesc_in = dev + p.td;
  k.flag = w + p.flag; k.proj = (double2*)(w + p.proj);
  k.q_orig = (int*)(w + p.qo); k.t_orig = (int*)(w + p.to);
  k.nq = (int*)(w + p.cnt); k.nt = k.nq + 1;
  k.q_geo = (int*)(w + p.qg); k.t_geo = (int*)(w + p.tg); k.t_dir = (double*)(w + p.tdir);
  k.dq = w + p.dq; k.dt = w + p.dt;
  k.m_g = (int32_t*)(w + p.mg); k.m_bf = (int32_t*)(w + p.mbf);
  k.keys = (uint32_t*)(w + p.keys);
  k.out = (int32_t*)(o + p.out); k.stat = (int*)(o + p.stat);
  return k;
}

// The host-known facts a kind's launches need, beyond its device arguments.
struct KindRun {
  KfKind k;
  bool bf;          // the brute-force fallback can be taken (host upper bounds)
  float nnr;
  int kmin;
  double gate;
  plf_scratch_slot slot;   // of the windowed matcher
  KnnProblem kp[2];
  NnrProblem np;
};

void prepare_bf(KindRun& r, const KindPlan& p, uint8_t* dev, int best_lr) {
  const KfKind& k = r.k;
  uint32_t *b12 = k.keys, *s12 = k.keys + p.nq, *b21 = k.keys + 2 * p.nq, *s21 = b21 + p.nt;
  r.kp[0] = {(const uint32_t*)k.dq, (const uint32_t*)k.dt, k.nq, k.nt, 0, 0, b12, s12, nullptr};
  r.kp[1] = {(const uint32_t*)k.dt, (const uint32_t*)k.dq, k.nt, k.nq, 0, 0, b21, s21, nullptr};
  r.np = {b12, s12, b21, s21, k.nq, k.nt, 0, 0, r.nnr, best_lr, k.m_bf, k.stat + 3};
}

plf_status run_kind(plf_ctx* ctx, KindRun& r, const KindPlan& p, uint8_t* dev, const double* dT, const KfCam& cam, int fast) {
  cudaStream_t cs = ctx->stream;
  const plf_params& P = ctx->params;
  KfKind& k = r.k;
  const int gq = (p.nq + 255) / 256, gt = (p.nt + 255) / 256;
  k_kf_query_vis<<<gq, 256, 0, cs>>>(k, dT, cam);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_compact<<<1, 1024, 0, cs>>>(k.flag, nullptr, p.nq, k.q_orig, k.nq);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_compact<<<1, 1024, 0, cs>>>(nullptr, k.t_lm, p.nt, k.t_orig, k.nt);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_query_gather<<<gq, 256, 0, cs>>>(k, cam);
  PLF_LAUNCH_CHECK(ctx);
  k_kf_train_gather<<<gt, 256, 0, cs>>>(k, cam);
  PLF_LAUNCH_CHECK(ctx);
  plf_status st;
  if (fast) {
    const int ws = P.matching_f2f_ws;
    MgbArgs a = {};
    a.g = {PLF_GRID_COLS, PLF_GRID_ROWS, ws, ws, ws, ws};
    a.is_lines = k.lines; a.K = p.nq; a.Kt = p.nt; a.best_lr = P.best_lr_matches ? 1 : 0;
    a.clip = k.lines;
    a.nnr = r.nnr; a.line_sim_th = (double)P.line_sim_th;
    a.q_geo = k.q_geo; a.t_geo = k.t_geo; a.t_dir = k.t_dir;
    a.d1 = k.dq; a.d2 = k.dt; a.d1_stride = a.d2_stride = 0;
    a.n1 = k.nq; a.n2 = k.nt; a.n1_stride = a.n2_stride = 0;
    a.m12 = k.m_g; a.m12_stride = 0; a.count = k.stat + 2; a.count_stride = 0;
    if ((st = plf_launch_match_grid_batch(ctx, a, 1, p.nq, p.nt, r.slot, cs))) return st;
  }
  if (r.bf) {
    const KnnProblem* dkp = (const KnnProblem*)(dev + p.kp);
    if ((st = plf_launch_knn2(ctx, cs, dkp, P.best_lr_matches ? 2 : 1, std::max(p.nq, p.nt)))) return st;
    if ((st = plf_launch_nnr(ctx, cs, (const NnrProblem*)(dev + p.np), 1, p.nq))) return st;
  }
  k_kf_select<<<gq, 256, 0, cs>>>(k, fast, r.bf ? 1 : 0, r.kmin, r.gate);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// The whole call: plan, stage, upload, the kinds' launches, download.  n_out[kind] = the reference's return value.
plf_status kf_run(plf_ctx* ctx, bool map, const plf_kf_match_opts* o, const double* T, KindPlan plan[2], const HostKind host[2],
                  int32_t* outs[2], int* n_out[2]) {
  const plf_params& P = ctx->params;
  StagedLayout L;
  for (int kd = 0; kd < 2; ++kd)
    if (plan[kd].active) plan_kind(plan[kd], L, kd == 1, map && kd == 1);
  const size_t t_off = L.take_in(16 * 8);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *pin, *dev;
  if (plf_status st = L.acquire(ctx, PLF_SCR_KF, &pin, &dev)) return st;
  cudaStream_t cs = ctx->stream;
  const KfCam cam = {ctx->cam.fx, ctx->cam.fy, ctx->cam.cx, ctx->cam.cy, (double)ctx->cam.width, (double)ctx->cam.height,
                     PLF_GRID_COLS / (double)ctx->cam.width, PLF_GRID_ROWS / (double)ctx->cam.height};
  memcpy(pin + t_off, T, 16 * 8);
  KindRun run[2];
  for (int kd = 0; kd < 2; ++kd) {
    if (!plan[kd].active) continue;
    const KindPlan& p = plan[kd];
    stage_kind(p, host[kd], pin, kd == 1);
    KindRun& r = run[kd];
    r.k = kind_args(p, dev, L.in, L.out, kd == 1, map, host[kd]);
    r.nnr = kd ? P.min_ratio_12_l : P.min_ratio_12_p;
    r.kmin = kd ? P.min_ls_matches : P.min_pt_matches;
    r.gate = kd ? o->max_kf_epip_l : o->max_kf_epip_p;
    r.slot = kd ? PLF_SCR_KF_MGB_LS : PLF_SCR_KF_MGB_PT;
    // the fallback needs more than kmin queries (and, KF-to-KF, more than kmin train features)
    r.bf = p.nq > r.kmin && (map || p.nt > r.kmin);
    prepare_bf(r, p, dev, P.best_lr_matches ? 1 : 0);
    memcpy(pin + p.kp, r.kp, sizeof r.kp);
    memcpy(pin + p.np, &r.np, sizeof r.np);
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(dev, pin, L.in, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemsetAsync(dev + L.in, 0xFF, L.out, cs));
  for (int kd = 0; kd < 2; ++kd) {
    if (!plan[kd].active) continue;
    PLF_CUDA(ctx, cudaMemsetAsync(run[kd].k.stat, 0, 8 * 4, cs));
    plf_status st = run_kind(ctx, run[kd], plan[kd], dev, (const double*)(dev + t_off), cam, o->fast_matching ? 1 : 0);
    if (st) return st;
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(pin + L.in, dev + L.in, L.out, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  for (int kd = 0; kd < 2; ++kd) {
    if (!plan[kd].active) continue;
    const int* stat = (const int*)(pin + L.in + plan[kd].stat);
    memcpy(outs[kd], pin + L.in + plan[kd].out, (size_t)plan[kd].nq * 4);
    if (n_out[kd]) *n_out[kd] = stat[0] - stat[1];
  }
  return PLF_OK;
}

bool bad_T(const double* T) {
  for (int i = 0; i < 16; ++i)
    if (!(T[i] == T[i])) return true;
  return false;
}

}  // namespace

extern "C" plf_status plf_match_kf2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_frame_view* prev,
                                      const plf_frame_view* curr, const double DT[16], int32_t* m_pt, int32_t* m_ls,
                                      int* n_pt, int* n_ls) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_pt) *n_pt = 0;
  if (n_ls) *n_ls = 0;
  if (!opts || !prev || !curr || !DT || bad_T(DT))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_kf2kf: opts, prev, curr and a finite DT are required");
  const plf_frame_view* f[2] = {prev, curr};
  for (const plf_frame_view* v : f)
    if (v->n_pt < 0 || v->n_ls < 0 || v->n_pt > KF_MAX_FEATURES || v->n_ls > KF_MAX_FEATURES)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_kf2kf: n_pt=%d, n_ls=%d (each must be in [0, %d])", v->n_pt, v->n_ls,
                      KF_MAX_FEATURES);
  if ((prev->n_pt > 0 && (!prev->pt_P || !prev->pdesc || !m_pt)) || (curr->n_pt > 0 && (!curr->pt_pl || !curr->pdesc)) ||
      (prev->n_ls > 0 && (!prev->ls_sP || !prev->ls_eP || !prev->ldesc || !m_ls)) ||
      (curr->n_ls > 0 && (!curr->ls_spl || !curr->ls_epl || !curr->ldesc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_kf2kf: a feature array is NULL while its count is > 0");
  const plf_params& P = ctx->params;
  if (m_pt) for (int i = 0; i < prev->n_pt; ++i) m_pt[i] = -1;
  if (m_ls) for (int i = 0; i < prev->n_ls; ++i) m_ls[i] = -1;
  KindPlan plan[2];
  // :243 / :368: a disabled kind, or either keyframe without stereo features of the kind, returns 0
  plan[0].active = P.has_points && prev->n_pt > 0 && curr->n_pt > 0;
  plan[1].active = P.has_lines && prev->n_ls > 0 && curr->n_ls > 0;
  plan[0].nq = prev->n_pt; plan[0].nt = curr->n_pt;
  plan[1].nq = prev->n_ls; plan[1].nt = curr->n_ls;
  if (!plan[0].active && !plan[1].active) return PLF_OK;
  HostKind host[2] = {};
  host[0] = {prev->pt_P, nullptr, 3, false, nullptr, prev->pdesc, curr->pt_pl, nullptr, nullptr, nullptr, curr->pdesc};
  host[1] = {prev->ls_sP, prev->ls_eP, 3, false, nullptr, prev->ldesc, curr->ls_spl, curr->ls_epl, nullptr, nullptr, curr->ldesc};
  int32_t* outs[2] = {m_pt, m_ls};
  int* ns[2] = {n_pt, n_ls};
  return kf_run(ctx, false, opts, DT, plan, host, outs, ns);
}

extern "C" plf_status plf_match_map2kf(plf_ctx* ctx, const plf_kf_match_opts* opts, const plf_local_map* map, const double Twf[16],
                                       const plf_frame_view* kf, const int32_t* kf_pt_lm, const int32_t* kf_ls_lm, int32_t* lm_pt,
                                       int32_t* lm_ls, int* n_pt, int* n_ls) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_pt) *n_pt = 0;
  if (n_ls) *n_ls = 0;
  if (!opts || !map || !kf || !Twf || bad_T(Twf))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_map2kf: opts, map, kf and a finite Twf are required");
  if (map->n_pt < 0 || map->n_ls < 0 || map->n_pt > KF_MAX_LANDMARKS || map->n_ls > KF_MAX_LANDMARKS)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_map2kf: map n_pt=%d, n_ls=%d (each must be in [0, %d])", map->n_pt,
                    map->n_ls, KF_MAX_LANDMARKS);
  if (kf->n_pt < 0 || kf->n_ls < 0 || kf->n_pt > KF_MAX_FEATURES || kf->n_ls > KF_MAX_FEATURES)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_map2kf: keyframe n_pt=%d, n_ls=%d (each must be in [0, %d])", kf->n_pt,
                    kf->n_ls, KF_MAX_FEATURES);
  if ((map->n_pt > 0 && (!map->pt_X || !map->pt_desc || !lm_pt)) || (map->n_ls > 0 && (!map->ls_X || !map->ls_desc || !lm_ls)) ||
      (kf->n_pt > 0 && (!kf->pt_pl || !kf->pdesc)) || (kf->n_ls > 0 && (!kf->ls_spl || !kf->ls_epl || !kf->ls_le || !kf->ldesc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match_map2kf: a landmark or feature array is NULL while its count is > 0");
  const plf_params& P = ctx->params;
  if (lm_pt) for (int i = 0; i < map->n_pt; ++i) lm_pt[i] = -1;
  if (lm_ls) for (int i = 0; i < map->n_ls; ++i) lm_ls[i] = -1;
  KindPlan plan[2];
  // :542 / :644: a disabled kind or a keyframe without stereo features of the kind returns 0; so does an empty map (:571)
  plan[0].active = P.has_points && kf->n_pt > 0 && map->n_pt > 0;
  plan[1].active = P.has_lines && kf->n_ls > 0 && map->n_ls > 0;
  plan[0].nq = map->n_pt; plan[0].nt = kf->n_pt;
  plan[1].nq = map->n_ls; plan[1].nt = kf->n_ls;
  if (!plan[0].active && !plan[1].active) return PLF_OK;
  HostKind host[2] = {};
  host[0] = {map->pt_X, nullptr, 3, false, map->pt_use, map->pt_desc, kf->pt_pl, nullptr, nullptr, kf_pt_lm, kf->pdesc};
  host[1] = {map->ls_X, nullptr, 6, true, map->ls_use, map->ls_desc, kf->ls_spl, kf->ls_epl, kf->ls_le, kf_ls_lm, kf->ldesc};
  int32_t* outs[2] = {lm_pt, lm_ls};
  int* ns[2] = {n_pt, n_ls};
  return kf_run(ctx, true, opts, Twf, plan, host, outs, ns);
}
