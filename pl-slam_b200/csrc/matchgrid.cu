// Windowed greedy matcher: stvo-pl `matchGrid` (points and lines overloads) over a `GridStructure`, as pl-slam calls it
// at src/mapHandler.cpp:251-271 (points), :382-418 (lines), :580-591, :686-706 (SURVEY §8 a5 / (f) f1).
//
// stvo-pl is not on disk: the semantics restate SURVEY Appendix A.3 and the published sources from memory (see
// oracle/matchgrid.py for the full statement; "parity unpinned").  Candidates are visited in ascending index order
// (stvo-pl iterates a std::unordered_set, whose order is implementation-defined and only matters for ties).
//
// The reference loop is sequential over the queries: with best_lr_matches a candidate i2 counts for query i1 only if
// d(i1,i2) beats the smallest distance any EARLIER query achieved on i2.  That is an exclusive prefix-minimum down each
// column of the (query x train) candidate matrix, so the work splits into
//   k_mg_columns : one thread per train feature walks the queries in order, evaluates the candidate predicate (is one
//                  of the grid cells the feature was pushed into inside the GridStructure::get window of the query's
//                  cell - for lines: of one of the query's Bresenham cells - plus, for lines, the direction gate),
//                  computes the Hamming distance of the candidates and writes d or "not considered" to a dense u16
//                  matrix (the grid arrives as cell -> items lists, the host wrapper inverts it to item -> cells);
//   k_mg_rows    : one thread per query scans its row in ascending train index with the reference's strict '<' updates,
//                  applies the f32 ratio test and records matches_12; matches_21 comes from the column pass;
//   k_mg_mutual  : drops i1 unless matches_21[matches_12[i1]] == i1, counts the matches.
#include "plf_internal.h"
#include <algorithm>
#include <vector>

#define MG_NONE 0xFFFFu


__device__ __forceinline__ int mg_hamming(const uint4* a, const uint4* b) {
  const uint4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
         __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// 8-connected Bresenham walk over the cells of (x1,y1)-(x2,y2), end points included (used as a set).
struct MgLine {
  bool steep; int x, x_end, y, dx, dy, err, ystep;
  __device__ void start(int x1, int y1, int x2, int y2) {
    steep = abs(y2 - y1) > abs(x2 - x1);
    if (steep) { int t = x1; x1 = y1; y1 = t; t = x2; x2 = y2; y2 = t; }
    if (x1 > x2) { int t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    dx = x2 - x1; dy = abs(y2 - y1); err = dx / 2; ystep = y1 < y2 ? 1 : -1; y = y1; x = x1; x_end = x2;
  }
  __device__ bool next(int* cx, int* cy) {
    if (x > x_end) return false;
    *cx = steep ? y : x; *cy = steep ? x : y;
    err -= dy;
    if (err < 0) { y += ystep; err += dx; }
    ++x;
    return true;
  }
};

// is one of the cells (packed x * rows + y) the train feature sits in returned by get(cx, cy, w)?
__device__ __forceinline__ bool mg_cells_in_window(const MgGrid& g, int cx, int cy, const int* cells, int nc) {
  const int x0 = max(0, cx - g.w_lo), x1 = min(g.cols, cx + g.w_hi + 1), y0 = max(0, cy - g.h_lo), y1 = min(g.rows, cy + g.h_hi + 1);
  if (x0 >= x1 || y0 >= y1) return false;
  for (int k = 0; k < nc; ++k) {
    const int x = cells[k] / g.rows, y = cells[k] - x * g.rows;
    if (x >= x0 && x < x1 && y >= y0 && y < y1) return true;
  }
  return false;
}

__global__ void __launch_bounds__(128) k_mg_columns(MgGrid g, int is_lines, const int* __restrict__ q_geo,
                                                    const int* __restrict__ t_cell_start, const int* __restrict__ t_cells,
                                                    const double* __restrict__ t_dir, double line_sim_th,
                                                    const uint32_t* __restrict__ d1, int n1,
                                                    const uint32_t* __restrict__ d2, int n2, int best_lr,
                                                    unsigned short* __restrict__ D, int* __restrict__ m21) {
  const int i2 = blockIdx.x * 128 + threadIdx.x;
  if (i2 >= n2) return;
  const uint4* b = reinterpret_cast<const uint4*>(d2) + 2 * (size_t)i2;
  const int* cells = t_cells + t_cell_start[i2];
  const int nc = t_cell_start[i2 + 1] - t_cell_start[i2];  // 0: the feature is in no cell of the grid -> never a candidate
  double tdx = 0, tdy = 0;
  if (is_lines) { tdx = t_dir[2 * i2]; tdy = t_dir[2 * i2 + 1]; }
  int run = 0x7FFFFFFF, who = -1;
  for (int i1 = 0; i1 < n1; ++i1) {
    bool cand = false;
    if (nc > 0) {
      if (is_lines) {
        const int* q = q_geo + 4 * i1;
        MgLine lq; lq.start(q[0], q[1], q[2], q[3]);
        int cx, cy;
        while (!cand && lq.next(&cx, &cy)) cand = mg_cells_in_window(g, cx, cy, cells, nc);
        if (cand) {  // direction gate, before the distance (and before the best-so-far record) as in the reference
          double vx = (double)(q[2] - q[0]), vy = (double)(q[3] - q[1]);
          const double nrm = sqrt(vx * vx + vy * vy);
          vx /= nrm; vy /= nrm;  // unguarded like the reference's normalize(): 0/0 = NaN fails the '<' below -> kept
          if (fabs(vx * tdx + vy * tdy) < line_sim_th) cand = false;
        }
      } else {
        cand = mg_cells_in_window(g, q_geo[2 * i1], q_geo[2 * i1 + 1], cells, nc);
      }
    }
    unsigned short out = MG_NONE;
    if (cand) {
      const int d = mg_hamming(reinterpret_cast<const uint4*>(d1) + 2 * (size_t)i1, b);
      if (best_lr) {
        if (d < run) { run = d; who = i1; out = (unsigned short)d; }
      } else {
        out = (unsigned short)d;
      }
    }
    D[(size_t)i1 * n2 + i2] = out;
  }
  m21[i2] = who;
}

__global__ void __launch_bounds__(128) k_mg_rows(const unsigned short* __restrict__ D, int n1, int n2, float nnr,
                                                 int32_t* __restrict__ m12) {
  const int i1 = blockIdx.x * 128 + threadIdx.x;
  if (i1 >= n1) return;
  int best_d = 0x7FFFFFFF, best_d2 = 0x7FFFFFFF, best_idx = -1;
  const unsigned short* row = D + (size_t)i1 * n2;
  for (int i2 = 0; i2 < n2; ++i2) {
    const int d = row[i2];
    if (d == MG_NONE) continue;
    if (d < best_d) { best_d2 = best_d; best_d = d; best_idx = i2; }
    else if (d < best_d2) best_d2 = d;
  }
  // `best_d < best_d2 * nnr`: int * float -> f32 product, int -> f32 comparison (INT_MAX when there is one candidate)
  m12[i1] = ((float)best_d < __fmul_rn((float)best_d2, nnr)) ? best_idx : -1;
}

__global__ void __launch_bounds__(128) k_mg_mutual(int32_t* __restrict__ m12, const int* __restrict__ m21, int n1,
                                                   int best_lr, int* __restrict__ count) {
  const int i1 = blockIdx.x * 128 + threadIdx.x;
  bool ok = false;
  if (i1 < n1) {
    const int i2 = m12[i1];
    ok = i2 >= 0;
    if (ok && best_lr && m21[i2] != i1) { m12[i1] = -1; ok = false; }
  }
  const unsigned bal = __ballot_sync(0xFFFFFFFFu, ok);
  if ((threadIdx.x & 31) == 0 && bal) atomicAdd(count, __popc(bal));
}

static size_t mg_align(size_t x) { return (x + 255) & ~size_t(255); }

static plf_status mg_run(plf_ctx* ctx, const char* who, int is_lines, const int* q_geo, const uint8_t* d1, int n1,
                         const int* cell_start, const int* cell_items, const double* t_dir, const uint8_t* d2, int n2,
                         int cols, int rows, plf_grid_window w, float nnr, double line_sim_th, int best_lr,
                         int32_t* matches_12, int* n_matches) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_matches) *n_matches = 0;
  if (n1 < 0 || n2 < 0 || n1 > 8192 || n2 > 8192 || cols <= 0 || rows <= 0 || cols > 4096 || rows > 4096 || !cell_start ||
      (n1 > 0 && (!q_geo || !d1 || !matches_12)) || (n2 > 0 && (!d2 || (is_lines && !t_dir))))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: bad arguments (n1=%d, n2=%d, each <= 8192; grid %dx%d)", who, n1, n2, cols, rows);
  const int ncell = cols * rows, nitems = cell_start[ncell];
  if (cell_start[0] != 0 || nitems < 0 || (nitems > 0 && !cell_items))
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: cell_start must start at 0 and be non-decreasing", who);
  if (n1 == 0) return PLF_OK;
  for (int i = 0; i < n1; ++i) matches_12[i] = -1;
  if (n2 == 0) return PLF_OK;
  // invert the grid: cell -> items (what GridStructure holds) to item -> cells (what a per-feature thread scans);
  // items outside [0, n2) are dropped as the reference's `if (i2 < 0 || i2 >= desc2.rows) continue;` does
  std::vector<int> tstart(n2 + 1, 0);
  for (int c = 0; c < ncell; ++c) {
    if (cell_start[c + 1] < cell_start[c]) return plf_fail(ctx, PLF_ERR_INVALID, "%s: cell_start must be non-decreasing", who);
    for (int k = cell_start[c]; k < cell_start[c + 1]; ++k)
      if (cell_items[k] >= 0 && cell_items[k] < n2) tstart[cell_items[k] + 1]++;
  }
  for (int i = 0; i < n2; ++i) tstart[i + 1] += tstart[i];
  std::vector<int> tcells(std::max(tstart[n2], 1)), fill(tstart.begin(), tstart.end() - 1);
  for (int c = 0; c < ncell; ++c)
    for (int k = cell_start[c]; k < cell_start[c + 1]; ++k)
      if (cell_items[k] >= 0 && cell_items[k] < n2) tcells[fill[cell_items[k]]++] = c;  // cell id = x * rows + y
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int gq = is_lines ? 4 : 2;
  const size_t bq = mg_align((size_t)n1 * gq * 4), bts = mg_align((size_t)(n2 + 1) * 4), btc = mg_align(tcells.size() * 4),
               bdir = mg_align((size_t)n2 * 16), b1 = mg_align((size_t)n1 * 32), b2 = mg_align((size_t)n2 * 32),
               bD = mg_align((size_t)n1 * n2 * 2), bm12 = mg_align((size_t)n1 * 4), bm21 = mg_align((size_t)n2 * 4);
  uint8_t* base = (uint8_t*)plf_scratch(ctx, 0, bq + bts + btc + bdir + b1 + b2 + bD + bm12 + bm21 + 256);
  if (!base) return PLF_ERR_CUDA;
  uint8_t* p = base;
  int* dq = (int*)p; p += bq;
  int* dts = (int*)p; p += bts;
  int* dtc = (int*)p; p += btc;
  double* ddir = (double*)p; p += bdir;
  uint8_t* dd1 = p; p += b1;
  uint8_t* dd2 = p; p += b2;
  unsigned short* D = (unsigned short*)p; p += bD;
  int32_t* dm12 = (int32_t*)p; p += bm12;
  int* dm21 = (int*)p; p += bm21;
  int* dcount = (int*)p;
  cudaStream_t cs = ctx->stream;
  ctx->cur = cs;
  PLF_CUDA(ctx, cudaMemcpyAsync(dq, q_geo, (size_t)n1 * gq * 4, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dts, tstart.data(), (size_t)(n2 + 1) * 4, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dtc, tcells.data(), tcells.size() * 4, cudaMemcpyHostToDevice, cs));
  if (is_lines) PLF_CUDA(ctx, cudaMemcpyAsync(ddir, t_dir, (size_t)n2 * 16, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dd1, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dd2, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemsetAsync(dcount, 0, sizeof(int), cs));
  const MgGrid g = {cols, rows, w.width_lo, w.width_hi, w.height_lo, w.height_hi};
  k_mg_columns<<<(n2 + 127) / 128, 128, 0, cs>>>(g, is_lines, dq, dts, dtc, ddir, line_sim_th, (const uint32_t*)dd1, n1,
                                                 (const uint32_t*)dd2, n2, best_lr ? 1 : 0, D, dm21);
  PLF_LAUNCH_CHECK(ctx);
  k_mg_rows<<<(n1 + 127) / 128, 128, 0, cs>>>(D, n1, n2, nnr, dm12);
  PLF_LAUNCH_CHECK(ctx);
  k_mg_mutual<<<(n1 + 127) / 128, 128, 0, cs>>>(dm12, dm21, n1, best_lr ? 1 : 0, dcount);
  PLF_LAUNCH_CHECK(ctx);
  int cnt = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(matches_12, dm12, (size_t)n1 * 4, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(&cnt, dcount, sizeof(int), cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));  // (the host vectors above are pageable: their copies completed at enqueue)
  if (n_matches) *n_matches = cnt;
  return PLF_OK;
}

extern "C" plf_status plf_match_grid_points(plf_ctx* ctx, const int* q_cell, const uint8_t* d1, int n1, const int* cell_start,
                                            const int* cell_items, const uint8_t* d2, int n2, int grid_cols, int grid_rows,
                                            plf_grid_window w, float nnr, int best_lr, int32_t* matches_12, int* n_matches) {
  return mg_run(ctx, "plf_match_grid_points", 0, q_cell, d1, n1, cell_start, cell_items, nullptr, d2, n2, grid_cols, grid_rows, w,
                nnr, 0.0, best_lr, matches_12, n_matches);
}

extern "C" plf_status plf_match_grid_lines(plf_ctx* ctx, const int* q_line, const uint8_t* d1, int n1, const int* cell_start,
                                           const int* cell_items, const double* t_dir, const uint8_t* d2, int n2,
                                           int grid_cols, int grid_rows, plf_grid_window w, float nnr, double line_sim_th,
                                           int best_lr, int32_t* matches_12, int* n_matches) {
  return mg_run(ctx, "plf_match_grid_lines", 1, q_line, d1, n1, cell_start, cell_items, t_dir, d2, n2, grid_cols, grid_rows, w,
                nnr, line_sim_th, best_lr, matches_12, n_matches);
}

// =====================================================================================================================
// Batched, device-resident form used by plf_batch_run when plf_params.matching_strategy != 0 (SURVEY §8 a5 / a7):
// the same three passes over MANY problems at once (grid.y = problem), with the geometry produced on the device from
// the frame's own feature arrays - no host hop.  A problem's arrays are addressed base + problem * stride.
//   k_mgb_qmask   (lines) per query line: bit mask over the grid cells of "some cell of the query's Bresenham walk has
//                 this cell inside its GridStructure::get window" (the window dilation of the walk)
//   k_mgb_columns one thread per train feature: candidate test (points: its cell inside the query's window; lines: one of
//                 its own Bresenham cells set in the query's mask, then the direction gate), Hamming distance, exclusive
//                 prefix-minimum down the column (best_lr_matches), dense u16 row-major matrix D
//   k_mgb_rows / k_mgb_mutual: as k_mg_rows / k_mg_mutual
// D costs 2 * K * K bytes per problem, so the problems are processed in chunks that share one scratch buffer.
#define MGB_MASK_WORDS 128   // >= cols * rows / 32 for the 64 x 48 grid (96 words)

__global__ void __launch_bounds__(128) k_mgb_qmask(MgbArgs a, int p0) {
  const int pl = blockIdx.y, p = p0 + pl;
  const int i1 = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n1 = min(a.n1[(size_t)p * a.n1_stride], a.K);
  if (i1 >= n1) return;
  uint32_t* m = a.qmask + ((size_t)pl * a.K + i1) * MGB_MASK_WORDS;
  for (int k = lane; k < MGB_MASK_WORDS; k += 32) m[k] = 0u;
  __syncwarp();
  const int* q = a.q_geo + ((size_t)p * a.K + i1) * 4;
  MgLine lq; lq.start(q[0], q[1], q[2], q[3]);
  int cx, cy;
  const MgGrid& g = a.g;
  while (lq.next(&cx, &cy)) {   // warp-uniform walk; the window's cells are spread over the lanes
    const int x0 = max(0, cx - g.w_lo), x1 = min(g.cols, cx + g.w_hi + 1), y0 = max(0, cy - g.h_lo), y1 = min(g.rows, cy + g.h_hi + 1);
    const int nx = x1 - x0, ny = y1 - y0;
    if (nx <= 0 || ny <= 0) continue;
    for (int k = lane; k < nx * ny; k += 32) {
      const int c = (x0 + k / ny) * g.rows + (y0 + k % ny);
      atomicOr(&m[c >> 5], 1u << (c & 31));
    }
  }
}

// The same mask, walking only the steps of the Bresenham line whose window can reach the grid: along the major axis a
// cell further than the window from the grid contributes nothing, so the walk starts at the first step that can and
// stops after the last one.  The state of the walk at step n is closed-form - err_n = (dx/2 - n dy) mod dx and the minor
// coordinate advanced by (err_n - dx/2 + n dy) / dx - so the cells visited are exactly those of the full walk.  Used for
// queries in pixel units (KF-to-KF lines), whose walk would otherwise cross thousands of cells outside the grid.
__global__ void __launch_bounds__(128) k_mgb_qmask_clip(MgbArgs a, int p0) {
  const int pl = blockIdx.y, p = p0 + pl;
  const int i1 = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n1 = min(a.n1[(size_t)p * a.n1_stride], a.K);
  if (i1 >= n1) return;
  uint32_t* m = a.qmask + ((size_t)pl * a.K + i1) * MGB_MASK_WORDS;
  for (int k = lane; k < MGB_MASK_WORDS; k += 32) m[k] = 0u;
  __syncwarp();
  const int* q = a.q_geo + ((size_t)p * a.K + i1) * 4;
  const MgGrid& g = a.g;
  long long x1 = q[0], y1 = q[1], x2 = q[2], y2 = q[3];
  const bool steep = llabs(y2 - y1) > llabs(x2 - x1);
  if (steep) { long long t = x1; x1 = y1; y1 = t; t = x2; x2 = y2; y2 = t; }
  if (x1 > x2) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
  const long long dx = x2 - x1, dy = llabs(y2 - y1), e0 = dx / 2, ystep = y1 < y2 ? 1 : -1;
  // major-axis range whose window reaches the grid
  const long long lo = steep ? -(long long)g.h_hi : -(long long)g.w_hi;
  const long long hi = steep ? (long long)g.rows - 1 + g.h_lo : (long long)g.cols - 1 + g.w_lo;
  const long long n0 = max(0ll, lo - x1), n_end = min(x2, hi) - x1;
  if (n0 > n_end) return;
  long long err = e0, y = y1;
  if (n0 > 0) {   // dx > 0 here (n0 <= n_end <= dx)
    err = (e0 - n0 * dy) % dx;
    if (err < 0) err += dx;
    y = y1 + ystep * ((err - e0 + n0 * dy) / dx);
  }
  for (long long n = n0; n <= n_end; ++n) {   // warp-uniform walk; the window's cells are spread over the lanes
    const long long xx = x1 + n;
    const int cx = (int)(steep ? y : xx), cy = (int)(steep ? xx : y);   // y may be far outside: its window is then empty
    err -= dy;
    if (err < 0) { y += ystep; err += dx; }
    const long long fx0 = (long long)cx - g.w_lo, fy0 = (long long)cy - g.h_lo;
    const int x0 = (int)max(0ll, fx0), xe = (int)min((long long)g.cols, (long long)cx + g.w_hi + 1);
    const int y0 = (int)max(0ll, fy0), ye = (int)min((long long)g.rows, (long long)cy + g.h_hi + 1);
    const int nx = xe - x0, ny = ye - y0;
    if (nx <= 0 || ny <= 0) continue;
    for (int k = lane; k < nx * ny; k += 32) {
      const int c = (x0 + k / ny) * g.rows + (y0 + k % ny);
      atomicOr(&m[c >> 5], 1u << (c & 31));
    }
  }
}

template <int IS_LINES>
__global__ void __launch_bounds__(128) k_mgb_columns(MgbArgs a, int p0) {
  const int pl = blockIdx.y, p = p0 + pl;
  const int i2 = blockIdx.x * 128 + threadIdx.x;
  const int n1 = min(a.n1[(size_t)p * a.n1_stride], a.K), n2 = min(a.n2[(size_t)p * a.n2_stride], a.Kt);
  if (i2 >= n2) return;
  const MgGrid& g = a.g;
  const uint4* b = reinterpret_cast<const uint4*>(a.d2 + (size_t)p * a.d2_stride) + 2 * (size_t)i2;
  const uint4* q1 = reinterpret_cast<const uint4*>(a.d1 + (size_t)p * a.d1_stride);
  const int* tg = a.t_geo + ((size_t)p * a.Kt + i2) * (IS_LINES ? 4 : 2);
  const int* qg = a.q_geo + (size_t)p * a.K * (IS_LINES ? 4 : 2);
  unsigned short* D = a.D + (size_t)pl * a.K * a.Kt;
  int tx = 0, ty = 0, t4[4] = {0, 0, 0, 0};
  double tdx = 0, tdy = 0;
  bool t_in = false;
  if (IS_LINES) {
    t4[0] = tg[0]; t4[1] = tg[1]; t4[2] = tg[2]; t4[3] = tg[3];
    tdx = a.t_dir[((size_t)p * a.Kt + i2) * 2]; tdy = a.t_dir[((size_t)p * a.Kt + i2) * 2 + 1];
  } else {
    tx = tg[0]; ty = tg[1];
    t_in = tx >= 0 && tx < g.cols && ty >= 0 && ty < g.rows;   // pushed outside the grid: never returned
  }
  int run = 0x7FFFFFFF, who = -1;
  for (int i1 = 0; i1 < n1; ++i1) {
    bool cand = false;
    if (IS_LINES) {
      const uint32_t* m = a.qmask + ((size_t)pl * a.K + i1) * MGB_MASK_WORDS;
      MgLine lt; lt.start(t4[0], t4[1], t4[2], t4[3]);
      int cx, cy;
      while (!cand && lt.next(&cx, &cy)) {
        if (cx < 0 || cx >= g.cols || cy < 0 || cy >= g.rows) continue;   // a cell outside the grid is never returned
        const int c = cx * g.rows + cy;
        cand = (m[c >> 5] >> (c & 31)) & 1u;
      }
      if (cand) {
        const int* q = qg + 4 * i1;
        double vx = (double)(q[2] - q[0]), vy = (double)(q[3] - q[1]);
        const double nrm = sqrt(vx * vx + vy * vy);
        vx /= nrm; vy /= nrm;
        if (fabs(vx * tdx + vy * tdy) < a.line_sim_th) cand = false;
      }
    } else if (t_in) {
      const int qx = qg[2 * i1], qy = qg[2 * i1 + 1];
      cand = tx >= qx - g.w_lo && tx <= qx + g.w_hi && ty >= qy - g.h_lo && ty <= qy + g.h_hi;
    }
    unsigned short out = MG_NONE;
    if (cand) {
      const int d = mg_hamming(q1 + 2 * (size_t)i1, b);
      if (a.best_lr) {
        if (d < run) { run = d; who = i1; out = (unsigned short)d; }
      } else {
        out = (unsigned short)d;
      }
    }
    D[(size_t)i1 * a.Kt + i2] = out;
  }
  a.m21[(size_t)pl * a.Kt + i2] = who;
}

__global__ void __launch_bounds__(128) k_mgb_rows(MgbArgs a, int p0) {
  const int pl = blockIdx.y, p = p0 + pl;
  const int i1 = blockIdx.x * 128 + threadIdx.x;
  const int n1 = min(a.n1[(size_t)p * a.n1_stride], a.K), n2 = min(a.n2[(size_t)p * a.n2_stride], a.Kt);
  if (i1 >= n1) return;
  int best_d = 0x7FFFFFFF, best_d2 = 0x7FFFFFFF, best_idx = -1;
  const unsigned short* row = a.D + (size_t)pl * a.K * a.Kt + (size_t)i1 * a.Kt;
  for (int i2 = 0; i2 < n2; ++i2) {
    const int d = row[i2];
    if (d == MG_NONE) continue;
    if (d < best_d) { best_d2 = best_d; best_d = d; best_idx = i2; }
    else if (d < best_d2) best_d2 = d;
  }
  a.m12[(size_t)p * a.m12_stride + i1] = ((float)best_d < __fmul_rn((float)best_d2, a.nnr)) ? best_idx : -1;
}

__global__ void __launch_bounds__(128) k_mgb_mutual(MgbArgs a, int p0) {
  const int pl = blockIdx.y, p = p0 + pl;
  const int i1 = blockIdx.x * 128 + threadIdx.x;
  const int n1 = min(a.n1[(size_t)p * a.n1_stride], a.K);
  bool ok = false;
  if (i1 < n1) {
    int32_t* m12 = a.m12 + (size_t)p * a.m12_stride;
    const int i2 = m12[i1];
    ok = i2 >= 0;
    if (ok && a.best_lr && a.m21[(size_t)pl * a.Kt + i2] != i1) { m12[i1] = -1; ok = false; }
  }
  const unsigned bal = __ballot_sync(0xFFFFFFFFu, ok);
  if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&a.count[(size_t)p * a.count_stride], __popc(bal));
}

// Runs nprob windowed matching problems.  scratch: MGB scratch of the context (slot `slot`), sized here.
plf_status plf_launch_match_grid_batch(plf_ctx* ctx, MgbArgs a, int nprob, int max_n1, int max_n2, int slot) {
  if (nprob <= 0) return PLF_OK;
  if (a.g.cols * a.g.rows > 32 * MGB_MASK_WORDS) return plf_fail(ctx, PLF_ERR_INVALID, "match grid: %dx%d cells exceed the mask", a.g.cols, a.g.rows);
  const int K = a.K, Kt = a.Kt;
  const size_t perD = (size_t)K * Kt * 2, perM = a.is_lines ? (size_t)K * MGB_MASK_WORDS * 4 : 0, per21 = (size_t)Kt * 4;
  const size_t per = mg_align(perD) + mg_align(perM) + mg_align(per21);
  int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)nprob, (size_t(1) << 31) / per));   // <= 2 GB of scratch
  uint8_t* base = (uint8_t*)plf_scratch(ctx, slot, per * chunk);
  if (!base) return PLF_ERR_CUDA;
  a.D = (unsigned short*)base;
  a.qmask = (uint32_t*)(base + mg_align(perD) * chunk);
  a.m21 = (int*)(base + (mg_align(perD) + mg_align(perM)) * chunk);
  cudaStream_t cs = ctx->cur;
  const int gx1 = (max_n1 + 127) / 128, gx2 = (max_n2 + 127) / 128;
  if (gx1 == 0 || gx2 == 0) return PLF_OK;
  for (int p0 = 0; p0 < nprob; p0 += chunk) {
    const int np = std::min(chunk, nprob - p0);
    if (a.is_lines) {
      if (a.clip) k_mgb_qmask_clip<<<dim3((max_n1 + 3) / 4, np), 128, 0, cs>>>(a, p0);
      else k_mgb_qmask<<<dim3((max_n1 + 3) / 4, np), 128, 0, cs>>>(a, p0);
      PLF_LAUNCH_CHECK(ctx);
      k_mgb_columns<1><<<dim3(gx2, np), 128, 0, cs>>>(a, p0);
    } else {
      k_mgb_columns<0><<<dim3(gx2, np), 128, 0, cs>>>(a, p0);
    }
    PLF_LAUNCH_CHECK(ctx);
    k_mgb_rows<<<dim3(gx1, np), 128, 0, cs>>>(a, p0);
    PLF_LAUNCH_CHECK(ctx);
    k_mgb_mutual<<<dim3(gx1, np), 128, 0, cs>>>(a, p0);
    PLF_LAUNCH_CHECK(ctx);
  }
  return PLF_OK;
}
