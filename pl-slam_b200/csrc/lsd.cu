// LSD line segment detector, batched over images (SURVEY §8 a2), and the LSDDetectorC KeyLine stage.
//
// Replaces LSDDetectorC::detect -> detectImpl (3rdparty/line_descriptor/src/LSDDetector_custom.cpp:218-324):
//   cv::createLineSegmentDetector(refine=0, scale, sigma_scale, quant, ang_th, log_eps, density_th, n_bins)
//   ->detect(img)  (:246-264; OpenCV imgproc lsd.cpp, not vendored by the reference — arithmetic pinned bit-exact
//   against cv2 4.13 by oracle/lsd.c), endpoint clamp (:76-102), min-length filter (:280-281), KeyLine fill
//   (:284-303), and stvo-pl's "sort by response, keep lsd_nfeatures" (SURVEY Appendix A.2).
//
// With refine = LSD_REFINE_NONE the detector is: Gaussian pre-blur (CV_8U fixed-point) + INTER_LINEAR_EXACT resample
// -> level-line angle / gradient magnitude -> 1024-bin pseudo-ordering of the seeds (bins descending, raster order
// inside a bin) -> greedy region growing -> rectangle fit.  No NFA validation runs at refine 0.
//
// Kernels
//   k_lsd_build_lut  once per context: the gradient lookup tables (LsdTables)
//   k_lsd_fill_notdef
//                    once per state: every record of the record maps set to "undefined"
//   k_lsd_pre        one tile kernel from the source image to the gradient records: separable Q8.8 Gaussian pre-blur
//                    (DP4A row pass, one rounding), INTER_LINEAR_EXACT resample to scale, 2x2 gradient, staged by TMA box
//                    loads with no blurred or resampled map in global memory.  For the DEFINED pixels only (|grad| > rho,
//                    ~12 %) it writes the 8-byte record {angle (cv::fastAtan2 = plf_fast_atan2, degrees, f32, from a table
//                    keyed by (gx,gy)), table index} and one packed entry (column, |grad|^2) of the raster-ordered seed list
//                    of the pixel's row segment; and the per-image max of |grad|^2.  Nothing dense leaves the kernel (the
//                    record map restores itself to "undefined", see k_lsd_fill_notdef)
//   k_lsd_seed_order stable counting sort of the seed lists by magnitude bin (descending), raster order inside a
//                    bin == OpenCV's ordered_points; one CTA per image, bin counts in shared memory
//   k_lsd_grow       region growing.  The algorithm is a sequential greedy partition (each accepted pixel updates the
//                    region angle that the next test uses, and regions compete through the `used` map), so it is run by
//                    ONE WARP PER IMAGE with thousands of images in flight: lanes 9e..9e+8 hold the 3x3 neighbourhood
//                    records of queue entry r+e, e < 3 (fetched one round ahead, L1-resident through a look-ahead
//                    prefetch), the alignment tests run lane-parallel in the reference order, and the
//                    region angle is only evaluated when a decision depends on it (see the kernel's comment; bit-exact).
//                    The (cosf, sinf) a member adds to the region's sums comes from a table keyed by the record's index,
//                    staged in a shared-memory ring by cp.async and added, in the reference's order, when the sums are read.
//                    `used` is folded into the angle (a used pixel gets the NOTDEF sentinel).
//   k_lsd_rect_order / k_lsd_rects
//                    one thread per region, regions permuted into size classes: weighted centroid, inertia-matrix
//                    angle, extent - sequential fp64 sums in region order (bit-exact with the CPU loop)
//   k_keylines       clamp + length filter + KeyLine fill with ordered compaction, optional top-K by response
// Roofline: region growing is latency-bound by construction and is reported as time, not as a roofline fraction (SURVEY §8d);
// the rest in DESIGN.md §4.
#include <float.h>
#include <stdlib.h>

#include "glibc_atan2f.cuh"
#include "glibc_sincosf.cuh"
#include "plf_internal.h"
#include "plf_tma.cuh"

#define LSD_NOTDEF (-1024.0f)
#define LSD_PI 3.1415926535897932384626433832795
#define LSD_3_2_PI ((3 * LSD_PI) / 2)
#define LSD_2PI (2 * LSD_PI)
#define LSD_DEG2RAD (LSD_PI / 180)
#define LSD_BINS_MAX 1024
#define LSD_QCAP 256   // shared-memory window of the region queue (entries)

// The launch of k_lsd_pre for one image size at the context's parameters (lsd_pre_geom): the pre-blur's KS Q8 taps (KS = 1:
// no blur, at scale 1 or when the centre tap is 256), TH scaled rows per CTA, and each CTA's 512-column row segment cut
// into NP pieces of PW scaled columns, one TMA box each.
struct LsdPreGeom {
  int ks = 1, th = 0, np = 0, pw = 0;
  bool packed = true;            // the resample takes four scaled columns per thread (plf_resize_packed_ok); else one
  uint4 taps = {0u, 0u, 0u, 0u}; // tap k in byte k % 4 of word k / 4
};

// What LSD derives from the context's parameters alone, built once per context and read by every LSD state.
struct LsdTables {
  double prec = 0, p = 0, rho = 0;
  int m2_min = 0;           // smallest gx^2+gy^2 whose gradient norm exceeds rho (defined pixel)
  float* angle_lut = nullptr;   // [1021*1021] gradient (gx,gy) -> level-line angle (degrees) of a defined pixel
  float2* cs_lut = nullptr;     // [1021*1021] gradient (gx,gy) -> (cosf, sinf) of float(angle in radians): a member's term of the region sums
  float2* seed_lut = nullptr;   // [1021*1021] gradient (gx,gy) -> unit vector of a region seed
  DevBufList bufs;
};

struct LsdState {
  int w = 0, h = 0, nimg = 0;
  int ws = 0, hs = 0;       // scaled size
  int n_bins = 1024;
  double scale = 1.2;
  int min_reg_size = 0;
  int max_regions = 0, max_lines = 0;
  bool two_parities = false;
  LsdPreGeom pre;             // k_lsd_pre's launch (lsd_pre_geom)
  uint32_t* rect_perm = nullptr;  // [nimg][max_regions] regions in size-class order (k_lsd_rect_order)
  struct LsdPix* pix_raw[2] = {nullptr, nullptr};  // allocation (pix + look-ahead slack on both sides)
  struct LsdPix* pix[2] = {nullptr, nullptr};  // [nimg][guard + hs*ws]  {angle (deg, f32) | NOTDEF = undefined/used, table index}
  size_t pix_stride = 0;      // entries per image = guard (ws+1, permanently NOTDEF) + hs*ws
  // seed lists per row segment (LSD_SEG columns): segment (y, xb) owns the entries [y * ws + LSD_SEG * xb, ...);
  // an entry is column-in-segment | gx^2+gy^2 << LSD_COL_BITS (k_lsd_pre)
  uint32_t* seedlist = nullptr; // [nimg][hs*ws]
  int* segcnt = nullptr;        // [nimg][hs][nxb] entries per segment
  int nxb = 0;                  // segments per row
  int* maxmag2 = nullptr;     // [nimg]
  // per batch parity: what crosses from the pre-grow phase to the growing (pix, order, nseeds) and what the match phase
  // reads (kls, nlines).  One copy: what only the growing / rectangle / KeyLine kernels of one batch write and read.
  int* nseeds[2] = {nullptr, nullptr};      // [nimg]
  uint32_t* order[2] = {nullptr, nullptr};  // [nimg][hs*ws]
  plf_keyline* kls[2] = {nullptr, nullptr}; // [nimg][max_lines]  final KeyLines (after top-K)
  int* nlines[2] = {nullptr, nullptr};      // [nimg]
  uint32_t* regpts = nullptr;   // [nimg][hs*ws]
  uint4* regions = nullptr;     // [nimg][max_regions] {start, count, angle_lo, angle_hi}
  int* nregions = nullptr;      // [nimg]
  float4* segs = nullptr;       // [nimg][max_regions]
  plf_keyline* kls_all = nullptr; // [nimg][max_regions] before top-K
  int* overflow = nullptr;    // [1]
  int* rs_tab = nullptr;      // resize tables
  size_t rs_x_off = 0, rs_y_off = 0, rs_xp_off = 0;
  DevBufList bufs;   // every buffer but rs_tab; empty in a state that borrows them (plf_lsd_create_sizes)
  DevBufList tabs;   // rs_tab, the state's own
};

// ---- gradient ---------------------------------------------------------------------------------------------
// Per-pixel record read by the region-growing kernel: one 8-byte load per neighbour.
struct __align__(8) LsdPix {
  float a;    // level-line angle in DEGREES exactly as cv::fastAtan2(gx,-gy) returns it (OpenCV stores a * DEG_TO_RADS as
              // f64; that product is re-formed where the f64 value is needed) or LSD_NOTDEF_F = undefined / used
  uint32_t li; // index of the pixel's gradient in the (gx,gy) tables: a member's (cosf, sinf) is lut_cs[li], a seed's unit
               // vector lut_seed[li], and the rectangle fit recovers (gx, gy) from it
};
#define LSD_NOTDEF_F (-1024.f)

// Gradient lookup tables.  The 2x2 gradient (gx, gy) takes 1021 x 1021 integer values; the level-line angle, the NOTDEF
// decision (|grad| <= rho) and cosf/sinf of float(angle) are functions of (gx, gy) only.  They are tabulated once per
// context with exactly the device functions used elsewhere (4 + 8 + 8 MB, L2-resident), which turns ~200 dependent
// instructions per defined pixel into table loads.
#define LSD_LUT_DIM 1021
// lut_angle: the angle of a defined gradient (NOTDEF otherwise; k_lsd_pre only looks up defined ones);
// lut_cs: (cos(float(angle)), sin(float(angle))) as region_grow adds them, host libm -> glibc port;
// lut_seed: the unit vector region_grow starts its sums from, float(cos(angle)), float(sin(angle)) of the f64 angle.
__global__ void __launch_bounds__(256) k_lsd_build_lut(double rho, float* __restrict__ lut_angle, float2* __restrict__ lut_cs,
                                                       float2* __restrict__ lut_seed) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= LSD_LUT_DIM * LSD_LUT_DIM) return;
  const int gx = i / LSD_LUT_DIM - 510, gy = i % LSD_LUT_DIM - 510;
  float a = LSD_NOTDEF_F;
  float2 cs = make_float2(0.f, 0.f), sv = make_float2(0.f, 0.f);
  const double norm = sqrt((double)(gx * gx + gy * gy) / 4.0);
  if (!(norm <= rho)) {
    const float adeg = plf_fast_atan2((float)gx, (float)(-gy));
    a = adeg;
    const float af = (float)((double)adeg * LSD_DEG2RAD);
    cs = make_float2(glibc_cosf(af), glibc_sinf(af));
    const double ad = (double)adeg * LSD_DEG2RAD;
    sv = make_float2((float)cos(ad), (float)sin(ad));
  }
  lut_angle[i] = a;
  lut_cs[i] = cs;
  lut_seed[i] = sv;
}

// Every record of the map (guards included) starts as "undefined".  From then on the map returns to that state by itself:
// the growing kernel visits every defined pixel - as a seed or as a member of a region - and marks it used (= NOTDEF), so
// when a batch's region growing has finished, all records of its images read NOTDEF again.  The gradient kernel therefore
// writes records for the DEFINED pixels only (~12 % of them).
__global__ void k_lsd_fill_notdef(LsdPix* __restrict__ pix, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  LsdPix e;
  e.a = LSD_NOTDEF_F; e.li = 0u;
  pix[i] = e;
}

// ---- pre-blur + resample + gradient ----------------------------------------------------------------------------
// k_lsd_pre: from the source image to the records, seed lists, segcnt and maxmag2, with no blurred or resampled map in
// between.  A CTA owns one 512-column row segment (LSD_SEG) of TH <= LSD_PRE_TH scaled rows.  The segment is cut into NP
// pieces of scaled columns; a piece's source footprint - the blurred rows and columns the resample of its scaled columns
// and of the scaled rows TH + 1 reads, plus the blur halo - arrives as ONE TMA box (LSD_PRE_BOXH rows of LSD_PRE_BOXW
// bytes, wider than the 256 elements a box dimension holds: plf_tma_encode_u8_blocks); border CTAs rebuild
// BORDER_REFLECT_101 in shared memory.  Per piece:
//   blur     : a PRMT + DP4A row pass into u16 (four sums of a row per group, the taps packed as bytes), then the column
//              pass and its one rounding, over the footprint only (KS = 1: no blur, the box is the blurred tile)
//   resample : the integer INTER_LINEAR_EXACT blend from the state's tables into the segment's scaled tile: four scaled
//              columns of one row per thread (k_resize_exact4's form) where four span at most 8 blurred bytes, else one
// Then, once over the tile:
//   gradient : a warp per scaled row, four 128-column chunks of 4 columns per lane; the records of the defined pixels and
//              the ordered compaction of the row segment's seed list (per chunk: one warp scan; the row is the segment, so
//              no barrier)
// pix points at pixel (0,0) of image 0 (i.e. past the guard); image stride pix_stride.  Only the DEFINED pixels (gradient
// norm above rho, ~12 %) leave the kernel: their 8-byte record (the map's other records already read "undefined", see
// k_lsd_fill_notdef) and one entry (column in the segment, gx^2 + gy^2) of the raster-ordered SEED LIST of their row
// segment; segment (y, xb) stores its entries at the segment's own pixel offset y * W + LSD_SEG * xb of the list array, so
// it can never overflow, and its length in segcnt.  Nothing dense is written: the seed ordering works on the lists, and the
// rectangle fit reads the gradient of a region point back from its record (li).
// The blur, resample and gradient are exact integer arithmetic: the records and lists are those of cv::GaussianBlur,
// cv::resize(INTER_LINEAR_EXACT) and the 2x2 gradient run one after the other.
// Measured on an H100 80GB HBM3 (700 W power limit), KITTI shape, 2048 images, default parameters (KS 7, TH 16, one
// piece): 5.42 ms against 8.26 ms for separate blur, resample and gradient kernels; 8 scaled rows per CTA took 6.69 ms.
#define LSD_SEG 512
// list entry: the low LSD_COL_BITS hold the column inside the segment, the high bits gx^2 + gy^2 (<= 2 * 510^2 over the
// table's gradient range)
#define LSD_COL_BITS 9
static_assert(LSD_SEG <= (1 << LSD_COL_BITS), "seed list: a segment column must fit the column field");
static_assert(2u * 510u * 510u < (1u << (32 - LSD_COL_BITS)), "seed list: gx^2 + gy^2 must fit above the column field");
#define LSD_PRE_TH 16         // scaled rows per CTA, at most
#define LSD_PRE_THREADS 256   // 8 warps: the gradient takes rows wrp, wrp + 8
#define LSD_PRE_BOXW 544      // TMA box width, bytes (34 blocks of 16)
#define LSD_PRE_BOXH 24       // TMA box rows
#define LSD_PRE_HW 528        // blurred columns a piece can produce (132 groups of 4: the row pass reads < LSD_PRE_BOXW)
#define LSD_PRE_SP 528        // row pitch of the staged scaled tile (>= LSD_SEG + 4)
#define LSD_PRE_KS_MAX 15
// The image-size sweep the front-end's geometry tests run every detector at (tests/test_frontend_geometry.py) keeps the
// edges of the two LSD blur tile grids this kernel replaced - 64 x 32 tiles placed at 64 bx - (16 - R), and 64 x 16 tiles
// - and reads their sizes here, so that the sweep and the tests written against it stay as they are.  No kernel uses them.
#define BF_TW 64
#define BF_TH 32
#define BQ_TW 64
#define BQ_TH 16
static_assert(LSD_PRE_HW % 4 == 0 && 4 * (LSD_PRE_HW / 4 - 1) + 4 * ((LSD_PRE_KS_MAX + 3) / 4 + 1) <= LSD_PRE_BOXW,
              "row pass: a group reads (KS + 3) / 4 + 1 words");
static_assert(LSD_PRE_HW + LSD_PRE_KS_MAX - 1 <= LSD_PRE_BOXW, "blur: the halo of the blurred columns lies in the box");
static_assert(LSD_PRE_BOXW % 16 == 0 && LSD_PRE_BOXW / 16 <= 256, "box: 16-byte blocks, at most 256 of them");
static_assert((LSD_PRE_TH + 1) * LSD_PRE_SP <= LSD_PRE_BOXH * LSD_PRE_HW * 2, "one piece: the scaled tile reuses the u16 row-pass tile");

// The source footprint of scaled columns [xa, xl] and rows [ya, yl], from the resample tables (ox / oy non-decreasing,
// at most the source size - 2): blurred columns [bxc, sx1] and rows [sy0, sy1]; the box starts at column bxc - R (on a
// 16-byte boundary) and row sy0 - R.
struct LsdPreFoot { int bxc, sx1, sy0, sy1; };
__host__ __device__ __forceinline__ LsdPreFoot lsd_pre_foot(const int* ox, const int* oy, int xa, int xl, int ya, int yl, int R) {
  LsdPreFoot f;
  f.bxc = ((ox[xa] - R) & ~15) + R;   // floor to a 16-byte boundary (two's complement: also below column 0)
  f.sx1 = ox[xl] + 1;
  f.sy0 = oy[ya];
  f.sy1 = oy[yl] + 1;
  return f;
}

// tabx = [ox(W) | cx(W)], taby = [oy(H) | cy(H)] (plf_linear_coeffs_host), tabxp = the packed x table of k_resize_exact4
// (plf_resize_pack_x); g = the state's LsdPreGeom; dynamic shared memory: the scaled tile ((TH + 1) x LSD_PRE_SP) when
// NP > 1, none otherwise.
template <int KS>
__global__ void __launch_bounds__(LSD_PRE_THREADS, 5) k_lsd_pre(const __grid_constant__ CUtensorMap tmap, int w, int h, int W, int H,
                                                             const LsdPreGeom g, const int* __restrict__ tabx,
                                                             const int4* __restrict__ tabxp, const int* __restrict__ taby,
                                                             const float* __restrict__ lut_angle,
                                                             int m2_min, size_t stride, LsdPix* __restrict__ pix, size_t pix_stride,
                                                             uint32_t* __restrict__ list, int* __restrict__ segcnt, int nxb,
                                                             int* __restrict__ maxmag2) {
  constexpr int R = KS / 2, NW = (KS + 3) / 4;   // NW tap words
  constexpr int BP = LSD_PRE_BOXW;
  __shared__ __align__(128) uint8_t raw[LSD_PRE_BOXH][BP];        // the box; then the blurred tile (pitch BP)
  __shared__ __align__(16) uint16_t hrow[LSD_PRE_BOXH][LSD_PRE_HW]; // row-pass sums; with one piece then the scaled tile
  __shared__ __align__(8) uint64_t bar;
  __shared__ int s_max[LSD_PRE_THREADS / 32];
  extern __shared__ __align__(16) uint8_t sc_own[];
  uint8_t* blur = &raw[0][0];
  uint8_t* sc = g.np > 1 ? sc_own : reinterpret_cast<uint8_t*>(&hrow[0][0]);   // pitch LSD_PRE_SP
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int xb = blockIdx.x, im = blockIdx.z, TH = g.th;
  const int X0 = xb * LSD_SEG, Y0 = blockIdx.y * TH;
  const int nsc = min(LSD_SEG + 1, W - X0), nsr = min(TH + 1, H - Y0);   // scaled columns / rows of the tile that exist
  uint32_t tw[NW];
#pragma unroll
  for (int k = 0; k < NW; ++k) tw[k] = k == 0 ? g.taps.x : k == 1 ? g.taps.y : k == 2 ? g.taps.z : g.taps.w;
  if (tid == 0) plf_mbar_init(&bar);
  __syncthreads();
  for (int p = 0; p < g.np && p * g.pw < nsc; ++p) {
    const int u0 = p * g.pw, u1 = min(u0 + g.pw, nsc);   // the piece's scaled columns, from X0
    const LsdPreFoot f = lsd_pre_foot(tabx, taby, X0 + u0, X0 + u1 - 1, Y0, min(Y0 + TH, H - 1), R);
    const int gx0 = f.bxc - R, gy0 = f.sy0 - R;   // source pixel of raw[0][0]
    if (p > 0) {   // the previous piece's blurred tile is read
      plf_fence_proxy_async();
      __syncthreads();
    }
    if (tid == 0) plf_tma_load_4d(&raw[0][0], &tmap, 0, gx0 >> 4, gy0, im, &bar, LSD_PRE_BOXH * BP);
    const int ncol = f.sx1 - f.bxc + 1, nrow = f.sy1 - f.sy0 + 1;   // blurred tile: nrow x ncol
    const int need_w = ncol + 2 * R, need_h = nrow + 2 * R;        // box cells the blur reads
    plf_mbar_wait(&bar, p & 1);
    // BORDER_REFLECT_101: the cells outside the image among those read, from their mirror pixel (inside this box: the
    // footprint reaches at most R + 15 columns / R rows past an edge, and its tables end at the source size - 2).
    // In-image rows first, then whole rows.  Cells past the image's last column hold the pitch padding or zeros; rows
    // outside it zeros.
    if (gx0 < 0 || gx0 + need_w > w || gy0 < 0 || gy0 + need_h > h) {
      const int ry_lo = max(0, -gy0), ry_hi = min(need_h, h - gy0);
      const int nl = min(need_w, max(0, -gx0)), rx_r = max(0, w - gx0), nr = max(0, need_w - rx_r);
      if (nl + nr > 0)
        for (int i = tid; i < (ry_hi - ry_lo) * (nl + nr); i += LSD_PRE_THREADS) {
          const int k = i / (nl + nr), j = i - k * (nl + nr);
          const int rx = j < nl ? j : rx_r + (j - nl);
          raw[ry_lo + k][rx] = raw[ry_lo + k][plf_reflect101(gx0 + rx, w) - gx0];
        }
      __syncthreads();
      const int nw = (need_w + 3) >> 2;
      for (int i = tid; i < (ry_lo + need_h - ry_hi) * nw; i += LSD_PRE_THREADS) {
        const int k = i / nw, j = i - k * nw;
        const int ry = k < ry_lo ? k : ry_hi + (k - ry_lo);
        const int m = plf_reflect101(gy0 + ry, h) - gy0;
        reinterpret_cast<uint32_t*>(raw[ry])[j] = reinterpret_cast<const uint32_t*>(raw[m])[j];
      }
    }
    __syncthreads();
    if (KS > 1) {
      // row pass: 4 adjacent sums of a row per group (sum of column c: box columns c .. c + 2R); output i of tap word k is
      // the byte window 4k + i .. 4k + i + 3, one PRMT of words k, k + 1, reduced by one DP4A (taps <= 255, exact in 32 bits,
      // result < 2^16)
      const int ngrp = (ncol + 3) >> 2;
      for (int ry = wrp; ry < need_h; ry += LSD_PRE_THREADS / 32)
        for (int j = lane; j < ngrp; j += 32) {
          const uint32_t* wp = reinterpret_cast<const uint32_t*>(&raw[ry][4 * j]);
          uint32_t wv[NW + 1];
#pragma unroll
          for (int k = 0; k <= NW; ++k) wv[k] = wp[k];
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            o[i] = 0u;
#pragma unroll
            for (int k = 0; k < NW; ++k) o[i] = __dp4a(__byte_perm(wv[k], wv[k + 1], 0x3210 + 0x1111 * i), tw[k], o[i]);
          }
          *reinterpret_cast<uint2*>(&hrow[ry][4 * j]) = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
        }
      __syncthreads();
      // column pass: one column per thread, the taps in registers, one rounding (the box is dead: the blurred tile replaces it)
      uint32_t t[KS];
#pragma unroll
      for (int k = 0; k < KS; ++k) t[k] = (tw[k >> 2] >> (8 * (k & 3))) & 0xFFu;
      for (int c = tid; c < ncol; c += LSD_PRE_THREADS) {
        uint32_t v[LSD_PRE_BOXH];
#pragma unroll
        for (int k = 0; k < LSD_PRE_BOXH; ++k) v[k] = hrow[k][c];
#pragma unroll
        for (int r = 0; r < LSD_PRE_BOXH - 2 * R; ++r)
          if (r < nrow) {
            uint32_t a = 0;
#pragma unroll
            for (int k = 0; k < KS; ++k) a += t[k] * v[r + k];
            const uint32_t o = (a + (1u << 15)) >> 16;
            blur[r * BP + c] = (uint8_t)(o > 255 ? 255 : o);
          }
      }
      __syncthreads();
    }
    // resample of the piece's scaled columns [u0, u1) and the rows Y0 .. Y0 + TH that exist.  Packed form: four adjacent
    // columns per thread from three words per blurred row, each output's byte pair by one PRMT, the horizontal blend by one
    // IDP.2A on the packed weight pair; thread = (4-column group tid % 128, row parity tid / 128).  Column LSD_SEG (the
    // right neighbour of the segment's last column), and every column where the packed form does not apply, by the scalar
    // form.
    if (g.packed) {
      const int gi = tid & 127, x = X0 + 4 * gi;
      if (4 * gi >= u0 && 4 * gi < min(u1, LSD_SEG)) {
        const int4 t0 = __ldg(&tabxp[2 * (x >> 2)]), t1 = __ldg(&tabxp[2 * (x >> 2) + 1]);
        const int ox0 = t0.x - f.bxc, mis = ox0 & 3, s8 = 8 * mis;
        const int ofs[4] = {t0.x, t0.z, t1.x, t1.z};
        const uint32_t wx[4] = {(uint32_t)t0.y, (uint32_t)t0.w, (uint32_t)t1.y, (uint32_t)t1.w};
        for (int r = tid >> 7; r < nsr; r += 2) {
          const int oy = __ldg(&taby[Y0 + r]) - f.sy0, cy = __ldg(&taby[H + Y0 + r]);
          const uint32_t* pa = reinterpret_cast<const uint32_t*>(blur + oy * BP + ox0 - mis);
          const uint32_t* pb = pa + BP / 4;
          const uint32_t alo = __funnelshift_r(pa[0], pa[1], s8), ahi = __funnelshift_r(pa[1], pa[2], s8);
          const uint32_t blo = __funnelshift_r(pb[0], pb[1], s8), bhi = __funnelshift_r(pb[1], pb[2], s8);
          const uint32_t wy0 = (uint32_t)(256 - cy), wy1 = (uint32_t)cy;
          uint32_t v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t sel = (uint32_t)(ofs[i] - ofs[0]) * 0x11u + 0x10u;
            const uint32_t h0 = __dp2a_lo(wx[i], __byte_perm(alo, ahi, sel), 0u);
            const uint32_t h1 = __dp2a_lo(wx[i], __byte_perm(blo, bhi, sel), 0u);
            v[i] = (h0 * wy0 + h1 * wy1 + 32768u) >> 16;
          }
          *reinterpret_cast<uint32_t*>(sc + r * LSD_PRE_SP + 4 * gi) = (v[0] | (v[1] << 8)) | ((v[2] | (v[3] << 8)) << 16);
        }
      }
    }
    const int us = g.packed ? max(u0, LSD_SEG) : u0, nu = u1 - us;
    for (int i = tid; i < nu * nsr; i += LSD_PRE_THREADS) {
      const int r = i / nu, u = us + (i - r * nu);
      const int ox = __ldg(&tabx[X0 + u]) - f.bxc, cx = __ldg(&tabx[W + X0 + u]);
      const int oy = __ldg(&taby[Y0 + r]) - f.sy0, cy = __ldg(&taby[H + Y0 + r]);
      const uint8_t* b0 = blur + oy * BP + ox;
      const uint32_t h0 = (uint32_t)b0[0] * (uint32_t)(256 - cx) + (uint32_t)b0[1] * (uint32_t)cx;
      const uint32_t h1 = (uint32_t)b0[BP] * (uint32_t)(256 - cx) + (uint32_t)b0[BP + 1] * (uint32_t)cx;
      sc[r * LSD_PRE_SP + u] = (uint8_t)((h0 * (uint32_t)(256 - cy) + h1 * (uint32_t)cy + 32768u) >> 16);
    }
  }
  __syncthreads();
  // gradient: warp wrp takes scaled rows y = Y0 + t, t = wrp, wrp + 8, ... (cells of the tile outside the image are never
  // read into a defined pixel)
  int mag2 = -1;
  for (int t = wrp; t < TH && Y0 + t < H; t += LSD_PRE_THREADS / 32) {
    const int y = Y0 + t;
    const uint32_t* s0 = reinterpret_cast<const uint32_t*>(sc + t * LSD_PRE_SP);
    const uint32_t* s1 = reinterpret_cast<const uint32_t*>(sc + (t + 1) * LSD_PRE_SP);
    const bool rok = y < H - 1;
    LsdPix* prow = pix + (size_t)im * pix_stride + (size_t)y * W + X0;
    uint32_t* lrow = list + (size_t)im * stride + (size_t)y * W + X0;
    int base = 0;   // entries of the row segment so far (chunks in x order)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int wi = 32 * k + lane, x4 = X0 + 4 * wi;
      const uint32_t a0 = s0[wi], a1 = s0[wi + 1], c0 = s1[wi], c1 = s1[wi + 1];
      int li[4], m2v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        li[c] = -1; m2v[c] = 0;
        // pixel (x, y): A = (x, y), B = (x+1, y), C = (x, y+1), D = (x+1, y+1)
        const int A = (a0 >> (8 * c)) & 0xFF, C = (c0 >> (8 * c)) & 0xFF;
        const int B = c < 3 ? (int)((a0 >> (8 * c + 8)) & 0xFF) : (int)(a1 & 0xFF);
        const int D = c < 3 ? (int)((c0 >> (8 * c + 8)) & 0xFF) : (int)(c1 & 0xFF);
        if (rok && x4 + c < W - 1) {
          const int DA = D - A, BC = B - C, gx = DA + BC, gy = DA - BC, m2 = gx * gx + gy * gy;
          if (m2 >= m2_min) { li[c] = (gx + 510) * LSD_LUT_DIM + (gy + 510); m2v[c] = m2; mag2 = max(mag2, m2); }
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (li[c] >= 0)
          *reinterpret_cast<uint2*>(&prow[4 * wi + c]) = make_uint2(__float_as_uint(__ldg(&lut_angle[li[c]])), (uint32_t)li[c]);
      // ordered compaction: one warp scan per chunk
      const int cnt = (li[0] >= 0) + (li[1] >= 0) + (li[2] >= 0) + (li[3] >= 0);
      int incl = cnt;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += v;
      }
      int o = base + incl - cnt;
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (li[c] >= 0) lrow[o++] = (uint32_t)(4 * wi + c) | ((uint32_t)m2v[c] << LSD_COL_BITS);
      base += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0) segcnt[(size_t)im * ((size_t)H * nxb) + (size_t)y * nxb + xb] = base;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mag2 = max(mag2, __shfl_xor_sync(0xFFFFFFFFu, mag2, off));
  if (lane == 0) s_max[wrp] = mag2;
  __syncthreads();
  if (tid == 0) {
    int m = s_max[0];
#pragma unroll
    for (int k = 1; k < LSD_PRE_THREADS / 32; ++k) m = max(m, s_max[k]);
    if (m >= 0 && m > __ldcg(&maxmag2[im])) atomicMax(&maxmag2[im], m);
  }
}

// ---- pseudo-ordering (stable counting sort, bins descending) ---------------------------------------------------
__device__ __forceinline__ double lsd_bin_coef(int maxmag2, int n_bins) {
  if (maxmag2 < 0) return 0.0;
  const double max_grad = sqrt((double)maxmag2 / 4.0);
  return max_grad > 0 ? (double)(n_bins - 1) / max_grad : 0.0;
}

// One CTA orders the seeds of one image.  The image's list entries, in raster order, are cut into LSD_SO_WARPS contiguous
// ranges of equal length (by an entry-count prefix over segcnt, so a band of edge-dense rows is shared by all warps); each
// warp counts the bins of its range into its own row of a shared [warp][bin] table, one scan turns the table into each
// warp's first slot per bin (bins descending, then warps in range order), and each warp walks its range again in raster
// order and stores every seed at its slot (match.any ranks inside 32 entries).  The bin is recomputed from gx^2 + gy^2 in
// both walks: nothing is written back to the lists and no count leaves the CTA.
#ifndef LSD_SO_WARPS
#define LSD_SO_WARPS 16
#endif
#define LSD_SO_THREADS (32 * LSD_SO_WARPS)
#define LSD_SO_AHEAD 4   // runs of 32 entries whose loads are in flight ahead of the one being processed
#define LSD_SO_BPT ((LSD_BINS_MAX + LSD_SO_THREADS - 1) / LSD_SO_THREADS)   // bins per thread in the scan over the bins
static size_t lsd_seed_order_smem(int n_bins) { return (size_t)LSD_SO_WARPS * n_bins * sizeof(uint32_t); }

// Hands out one warp's range of list entries as runs of at most 32 entries of one row segment, in raster order.  Every
// lane holds the same state; the lengths of 32 segments at a time sit one per lane, so runs of empty segments are
// skipped with one ballot.
struct LsdSegWalk {
  const int* sc;        // segment lengths of the image
  int nseg, nxb, W;
  int seg, i, n;        // current segment, its next entry, its length
  uint32_t p0;          // pixel offset of the current segment = where its list starts
  uint32_t left;        // entries of the range not handed out yet
  int cbase, c32;       // this lane's length: segment cbase + lane
  unsigned nz;          // lanes whose segment is not empty

  __device__ __forceinline__ void load_lengths(int base) {
    const int lane = threadIdx.x & 31;
    cbase = base;
    c32 = base + lane < nseg ? __ldg(&sc[base + lane]) : 0;
    nz = __ballot_sync(0xFFFFFFFFu, c32 > 0);
  }
  __device__ __forceinline__ void enter(int s) {
    seg = s;
    const int y = s / nxb;
    p0 = (uint32_t)(y * W + (s - y * nxb) * LSD_SEG);
  }
  __device__ __forceinline__ void init(const int* sc_, int nseg_, int nxb_, int W_, int seg0, int off, uint32_t count) {
    sc = sc_; nseg = nseg_; nxb = nxb_; W = W_;
    left = count;
    i = off;
    if (count) {
      enter(seg0);
      load_lengths(seg0);
      n = __shfl_sync(0xFFFFFFFFu, c32, 0);
    }
  }
  // the next run: its first list index (from the image's list start) and its length (0: the range is done); *q0 = the
  // pixel offset of its segment
  __device__ __forceinline__ int next(uint32_t* q0, uint32_t* l0) {
    if (left == 0) return 0;
    const int m = min(min(32, n - i), (int)left);
    *q0 = p0;
    *l0 = p0 + (uint32_t)i;
    i += m;
    left -= (uint32_t)m;
    if (left && i == n) {   // on to the next segment with entries (one exists: entries are left)
      for (;;) {
        const int d = seg + 1 - cbase;
        const unsigned ahead = d < 32 ? nz & (0xFFFFFFFFu << d) : 0u;
        if (ahead) {
          const int s = cbase + __ffs(ahead) - 1;
          n = __shfl_sync(0xFFFFFFFFu, c32, s - cbase);
          enter(s);
          i = 0;
          break;
        }
        load_lengths(cbase + 32);
        seg = cbase - 1;
      }
    }
    return m;
  }
};

// Walks a warp's range with the entries of LSD_SO_AHEAD runs loaded ahead; f(entry, pixel offset of its segment, run
// length) is called once per run, in raster order, by the whole warp (lanes >= run length hold no entry).
template <class F>
__device__ __forceinline__ void lsd_walk_range(LsdSegWalk wk, const uint32_t* __restrict__ lst, F f) {
  const int lane = threadIdx.x & 31;
  uint32_t e[LSD_SO_AHEAD], p0[LSD_SO_AHEAD];
  int m[LSD_SO_AHEAD];
  auto fetch = [&](int j) {
    uint32_t l0 = 0;
    m[j] = wk.next(&p0[j], &l0);
    e[j] = lane < m[j] ? __ldg(&lst[l0 + lane]) : 0u;
  };
#pragma unroll
  for (int j = 0; j < LSD_SO_AHEAD; ++j) fetch(j);
  for (;;) {
#pragma unroll
    for (int j = 0; j < LSD_SO_AHEAD; ++j) {
      if (m[j] == 0) return;
      f(e[j], p0[j], m[j]);
      fetch(j);
    }
  }
}

// Block-wide inclusive prefix of v over the CTA's threads; *total = the sum.  s_w: LSD_SO_WARPS words of shared memory.
__device__ __forceinline__ uint32_t lsd_so_scan(uint32_t v, uint32_t* s_w, uint32_t* total) {
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, v, off);
    if (lane >= off) v += u;
  }
  if (lane == 31) s_w[wrp] = v;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < LSD_SO_WARPS; ++k) {
    const uint32_t x = s_w[k];
    if (k < wrp) base += x;
    tot += x;
  }
  __syncthreads();   // s_w is free again
  *total = tot;
  return base + v;
}

// list / order: image stride `stride` entries; segcnt: nseg = (H - 1) * nxb lengths per image (the last row holds no
// seed).  Dynamic shared memory: LSD_SO_WARPS * n_bins words.
__global__ void __launch_bounds__(LSD_SO_THREADS) k_lsd_seed_order(const uint32_t* __restrict__ list, const int* __restrict__ segcnt,
                                                                   size_t stride, int W, int H, int nxb, int n_bins,
                                                                   const int* __restrict__ maxmag2, uint32_t* __restrict__ order,
                                                                   int* __restrict__ nseeds) {
  extern __shared__ uint32_t s_cnt[];   // [warp][bin]: counts, then the warp's first slot per bin
  __shared__ uint32_t s_w[LSD_SO_WARPS];
  __shared__ int s_seg[LSD_SO_WARPS], s_off[LSD_SO_WARPS];
  const int im = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int nseg = (H - 1) * nxb;
  const int* sc = segcnt + (size_t)im * ((size_t)H * nxb);
  const uint32_t* lst = list + (size_t)im * stride;
  for (int k = tid; k < LSD_SO_WARPS * n_bins; k += LSD_SO_THREADS) s_cnt[k] = 0;
  // the image's entry count, and the segment and offset at which each warp's range starts
  uint32_t t = 0, total;
  for (int s = tid; s < nseg; s += LSD_SO_THREADS) t += (uint32_t)__ldg(&sc[s]);
  lsd_so_scan(t, s_w, &total);
  uint32_t carry = 0;
  for (int s0 = 0; s0 < nseg; s0 += LSD_SO_THREADS) {
    const int s = s0 + tid;
    const uint32_t n = s < nseg ? (uint32_t)__ldg(&sc[s]) : 0u;
    uint32_t tile;
    const uint32_t pre = carry + lsd_so_scan(n, s_w, &tile) - n;
#pragma unroll
    for (int k = 0; k < LSD_SO_WARPS; ++k) {
      const uint32_t b = (uint32_t)((unsigned long long)k * total / LSD_SO_WARPS);
      if (b - pre < n) { s_seg[k] = s; s_off[k] = (int)(b - pre); }
    }
    carry += tile;
  }
  __syncthreads();
  const uint32_t r0 = (uint32_t)((unsigned long long)wrp * total / LSD_SO_WARPS);
  const uint32_t r1 = (uint32_t)((unsigned long long)(wrp + 1) * total / LSD_SO_WARPS);
  LsdSegWalk wk;
  wk.init(sc, nseg, nxb, W, r1 > r0 ? s_seg[wrp] : 0, r1 > r0 ? s_off[wrp] : 0, r1 - r0);
  const double coef = lsd_bin_coef(maxmag2[im], n_bins);
  auto bin_of = [&](uint32_t e) { return (int)(sqrt((double)(e >> LSD_COL_BITS) / 4.0) * coef); };
  uint32_t* cw = s_cnt + wrp * n_bins;
  // count
  lsd_walk_range(wk, lst, [&](uint32_t e, uint32_t, int m) {
    if (lane < m) atomicAdd(&cw[bin_of(e)], 1u);
  });
  __syncthreads();
  // slots: per bin, a prefix over the warps; over the bins, a prefix in descending bin order (thread tid holds the
  // LSD_SO_BPT bins at descending positions LSD_SO_BPT * tid ...)
  uint32_t bt[LSD_SO_BPT], sum = 0;
#pragma unroll
  for (int h = 0; h < LSD_SO_BPT; ++h) {
    const int b = n_bins - 1 - (LSD_SO_BPT * tid + h);
    bt[h] = 0;
    if (b >= 0)
      for (int w = 0; w < LSD_SO_WARPS; ++w) {
        const uint32_t c = s_cnt[w * n_bins + b];
        s_cnt[w * n_bins + b] = bt[h];
        bt[h] += c;
      }
    sum += bt[h];
  }
  uint32_t all;
  uint32_t base = lsd_so_scan(sum, s_w, &all) - sum;
#pragma unroll
  for (int h = 0; h < LSD_SO_BPT; ++h) {
    const int b = n_bins - 1 - (LSD_SO_BPT * tid + h);
    if (b >= 0)
      for (int w = 0; w < LSD_SO_WARPS; ++w) s_cnt[w * n_bins + b] += base;
    base += bt[h];
  }
  if (tid == 0) nseeds[im] = (int)all;
  __syncthreads();
  // scatter, in raster order: stable ranks among the run's lanes of one bin
  uint32_t* ord = order + (size_t)im * stride;
  lsd_walk_range(wk, lst, [&](uint32_t e, uint32_t p0, int m) {
    if (lane < m) {
      const int b = bin_of(e);
      const unsigned peers = __match_any_sync(0xFFFFFFFFu >> (32 - m), b);
      const int leader = __ffs(peers) - 1;
      uint32_t slot = 0;
      if (lane == leader) {
        slot = cw[b];
        cw[b] = slot + __popc(peers);
      }
      slot = __shfl_sync(peers, slot, leader) + __popc(peers & ((1u << lane) - 1u));
      ord[slot] = p0 + (e & ((1u << LSD_COL_BITS) - 1u));
    }
    __syncwarp();
  });
}

// ---- region growing ----------------------------------------------------------------------------------------
__device__ __forceinline__ bool lsd_aligned_rad(double a, double theta, double prec) {
  double n_theta = theta - a;
  if (n_theta < 0) n_theta = -n_theta;
  if (n_theta > LSD_3_2_PI) {
    n_theta -= LSD_2PI;
    if (n_theta < 0) n_theta = -n_theta;
  }
  return n_theta <= prec;
}

// The warp that grows an image is the only reader and writer of that image's records while the kernel runs, and a CTA
// never leaves its SM, so L1-cached loads (ld.ca) are coherent with the warp's own stores.
struct LsdRec { float a; uint32_t li; };
__device__ __forceinline__ LsdRec lsd_load_pix(const LsdPix* p) {
  const uint2 v = __ldca(reinterpret_cast<const uint2*>(p));
  LsdRec r;
  r.a = __uint_as_float(v.x);
  r.li = v.y;
  return r;
}
__device__ __forceinline__ void lsd_prefetch(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
#define LSD_REC_BYTES 8   // sizeof(LsdPix), as the byte stride of the growing kernel's address arithmetic
static_assert(sizeof(LsdPix) == LSD_REC_BYTES, "LSD record size");

// One warp per image.  Pixels are addressed by their linear index i = y*W + x; the 8 neighbours are i + {-W-1 .. W+1}.
// No bounds tests are needed: the last column and last row of the map are always NOTDEF (ll_angle), so x-1 / x+1 wrap
// onto NOTDEF pixels, y+1 stays inside, and a guard of W+1 permanently-NOTDEF records precedes pixel 0 for y-1.
// Three queue entries per round: lane 9e + kk holds the 8-byte record of neighbour kk (row-major 3x3) of entry r + e, for
// the E = min(3, nreg - r) entries that exist when the round starts; cells accepted in the round join the queue for a
// later round.  Lane order is (entry, neighbour), the reference's order of tests, and the candidates are re-decided after
// every acceptance, which reproduces the reference's sequential semantics (each test sees the region angle and the used
// state left by the acceptances before it).  Two entries of a round share neighbours: accepting a cell also decides the
// lanes that hold it for a later entry (match.any mask).  The next round's records are loaded one round ahead - at the
// round's start for the entries that exist, at its acceptance for an entry added during the round - and a cell accepted
// after its record was loaded is patched to "used" in the look-ahead registers.
//
// Region sums off the decision chain.  A member adds (cosf, sinf) of its angle to the sums S; that pair is lut_cs[li].
// No acceptance decision reads S (see below: only an evaluation of the region angle and the region's end do), so an
// accepted cell's lane copies its table entry into a shared-memory ring (cp.async: no register waits on the load), and
// the staged terms are added in acceptance order only when S is about to be read - one wait per evaluation, not one per
// acceptance.  A plain load would not do: its register is read by the next addition, which waits for it.
#define LSD_CSQ 256   // staged terms (ring of float2; a full ring is summed early)
//
// Deferred region angle.  The reference recomputes theta_i = fastAtan2(S_i) after every acceptance (S_i = running sum of
// the members' unit vectors).  Most decisions do not need it: with th = the last angle that WAS evaluated (at sum S_0),
//   |theta_i - th| <= m_i,   m_0 = 2E + slack,   m_{i+1} = m_i + min(d_k + m_i, prec + E) / |S_0|       (degrees)
// because adding a unit vector at angle phi to S turns it by at most phi / |S| (tan(delta) = sin(phi) / (|S| + cos(phi))),
// phi <= d_k + m_i for the accepted cell k, |S_i| never shrinks (every member is within prec + E < 90 deg of S), and
// E = 0.02 deg bounds the error of the fastAtan2 polynomial (measured maximum 0.0096 deg).  A neighbour whose distance
// to th is below prec - m_i is aligned under theta_i whatever theta_i is, one above prec + m_i is not; only when the FIRST
// undecided neighbour falls inside the band is theta_i evaluated (th <- fastAtan2(S_i), m <- m_0), and if it is still
// inside the (now 0.05 deg) band the reference's own f64 test decides.  The float sums S_i are accumulated in the
// reference's order either way, so every accepted/rejected decision - and the final angle - is the reference's.
#define LSD_MARGIN0 0.05f
__device__ __forceinline__ void lsd_grow_body(LsdPix* __restrict__ pix_all, size_t pix_stride, size_t stride, int W,
                                                 const uint32_t* __restrict__ order_all, const float2* __restrict__ lut_seed,
                                                 const float2* __restrict__ lut_cs,
                                                 const int* __restrict__ nseeds, double prec, float prec_deg,
                                                 int min_reg_size, uint32_t* __restrict__ regpts_all,
                                                 uint4* __restrict__ regions_all, int max_regions,
                                                 int* __restrict__ nregions, int* __restrict__ overflow) {
  __shared__ uint32_t q[LSD_QCAP];
  __shared__ __align__(8) float2 s_cs[LSD_CSQ];   // lut_cs of accepted cells, by acceptance count (qpos)
  const int im = blockIdx.x, lane = threadIdx.x;
  LsdPix* pix = pix_all + (size_t)im * pix_stride;
  const uint32_t* order = order_all + (size_t)im * stride;
  uint32_t* regpts = regpts_all + (size_t)im * stride;
  uint4* regions = regions_all + (size_t)im * max_regions;
  // keep the per-image base pointers (and the queue's shared-window address) in registers: without these barriers ptxas
  // re-derives them with 64-bit multiplies / special-register reads at every access of the serial loop
  uint32_t qs = (uint32_t)__cvta_generic_to_shared(q);
  asm volatile("" : "+l"(pix));
  asm volatile("" : "+l"(regpts));
  asm volatile("" : "+l"(regions));
  asm volatile("" : "+r"(qs));
  const int ns = nseeds[im];
  const int grp = lane < 27 ? lane / 9 : 3;           // entry of the round served by this lane (lanes 27..31 idle)
  const int kk = lane < 27 ? lane - 9 * grp : 4;      // and the neighbour slot (row-major 3x3: the reference order)
  const int noff = (kk / 3 - 1) * W + (kk % 3 - 1);   // linear offset of that neighbour (row-major 3x3: reference order)
  // look-ahead window fetched into L1/L2 whenever a pixel joins the region: 7 rows x 8 records around it (the cells the
  // next two breadth-first layers will examine), one address per lane
  const int poff = lane < 28 ? (lane / 4 - 3) * W + (lane % 4) * 2 - 3 : 0;
  const int pmin = -(W + 1);  // first record of this image (the guard); smaller values mean "nothing fetched"
  const char* const pb = reinterpret_cast<const char*>(pix);
  const int l0 = lane == 0 ? 1 : 0;
  // ang_th close to 90 deg would break the "sum never shrinks" argument: fall back to evaluating every angle
  const float margin0 = prec_deg <= 60.f ? LSD_MARGIN0 : 1e30f;
  const float dmax = prec_deg + LSD_MARGIN0;
  uint32_t cursor = 0;
  int nreg_out = 0;
  const uint32_t csb = (uint32_t)__cvta_generic_to_shared(&s_cs[0]);
  // terms staged so far by this warp (ring slot = qpos % LSD_CSQ), and qpos at the last wait for all of them: a slot is
  // reused only after its copy has been waited for (two outstanding copies to one address would be unordered)
  uint32_t qpos = 0, qwait = 0;
  uint32_t seed_next = lane < ns ? order[lane] : 0u;
  for (int s0 = 0; s0 < ns; s0 += 32) {
    const int si = s0 + lane;
    const uint32_t seed = seed_next;
    // angle + index of the seed's gradient in the (gx,gy) tables: the region's sums start from lut_seed[li] =
    // (float(cos(double angle)), float(sin(double angle))) - tabulated once per context with the very expressions this
    // kernel used to evaluate per region (130 f64 instructions at 10 k region starts per frame: 15 % of the kernel)
    const uint2 ali = si < ns ? __ldcg(reinterpret_cast<const uint2*>(&pix[seed])) : make_uint2(__float_as_uint(LSD_NOTDEF_F), 0u);
    float a0 = __uint_as_float(ali.x);
    const uint32_t seed_li = ali.y;
    seed_next = si + 32 < ns ? order[si + 32] : 0u;   // next group of seeds: index now, record into L2 while this group runs
    if (si + 32 < ns) asm volatile("prefetch.global.L2 [%0];" ::"l"(&pix[seed_next]));
    unsigned pending = __ballot_sync(0xFFFFFFFFu, a0 != LSD_NOTDEF_F);
    while (pending) {
      const int src = __ffs(pending) - 1;
      const uint32_t sidx = __shfl_sync(0xFFFFFFFFu, seed, src);
      float th = __shfl_sync(0xFFFFFFFFu, a0, src);      // region angle (degrees) at the last evaluation
      const double th_seed = (double)th * LSD_DEG2RAD;    // the reference's f64 angle of the seed
      const float2 sv = __ldg(&lut_seed[__shfl_sync(0xFFFFFFFFu, seed_li, src)]);
      float sumdx = sv.x, sumdy = sv.y;                   // = (float)cos(th_seed), (float)sin(th_seed)
      float margin = margin0, inv0 = 1.02f;               // m_i and an upper bound of 1/|S_0|
      float lo = prec_deg - margin, hi = prec_deg + margin;
      bool fresh = true;                                  // th is the reference's current angle
      if (lane == 0) {
        pix[sidx].a = LSD_NOTDEF_F;
        regpts[cursor] = sidx;
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(qs), "r"(sidx) : "memory");
      }
      lsd_prefetch(pb + (long long)((int)sidx + poff) * LSD_REC_BYTES);
      __syncwarp();
      uint32_t nreg = 1;
      // records of the next round's entries on their lanes (nxt, cell ni; ni < pmin: nothing loaded): the seed's now,
      // later ones one round ahead or when their cell is accepted.  A cell accepted meanwhile is patched to "used".
      int ni = grp == 0 ? (int)sidx + noff : pmin - 1;
      asm volatile("" : "+r"(ni));  // keep the index 32-bit: one IMAD.WIDE forms the address
      LsdRec nxt;
      nxt.a = LSD_NOTDEF_F; nxt.li = 0u;
      if (grp == 0) nxt = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)ni * LSD_REC_BYTES));
      // the region's members whose terms are staged but not yet in S: ring positions [qsum, qpos), in acceptance order
      uint32_t qsum = qpos;
      auto add_staged = [&]() {
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncwarp();
        for (; qsum != qpos; ++qsum) {
          const float2 e = s_cs[qsum & (LSD_CSQ - 1)];
          sumdx = __fadd_rn(sumdx, e.x);
          sumdy = __fadd_rn(sumdy, e.y);
        }
        qwait = qpos;
      };
      for (uint32_t r = 0; r < nreg;) {
        const uint32_t ne = min(3u, nreg - r);   // entries of this round: the ones that exist now
        const uint32_t rn = r + ne;              // first entry of the next round
        const LsdRec cur = nxt;
        const int ci = ni;
        // lanes that see the same cell (neighbours shared by two entries): accepting it decides all of them
        const unsigned same = __match_any_sync(0xFFFFFFFFu, ci);
        nxt.a = LSD_NOTDEF_F;
        ni = pmin - 1;
        const uint32_t nx = rn + (uint32_t)grp;  // the next round's entries that already exist: load them now
        if (grp < 3 && nx < nreg) {
          uint32_t pt;
          if (nreg - nx <= LSD_QCAP) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(pt) : "r"(qs + ((nx & (LSD_QCAP - 1)) << 2)) : "memory");
          else pt = __ldcg(&regpts[cursor + nx]);
          ni = (int)pt + noff;
          asm volatile("" : "+r"(ni));
          nxt = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)ni * LSD_REC_BYTES));
        }
        // kk != 4: the centre is the entry itself (already used); with lane < 9 ne it also keeps the idle lanes out
        unsigned rem = __ballot_sync(0xFFFFFFFFu, lane < 9 * (int)ne && kk != 4 && cur.a != LSD_NOTDEF_F);
        // Off the decision chain: each lane's distance to th (changes only when th is evaluated) and the margin the
        // region would have after accepting this lane's cell (the margin update of the reference order, done by every
        // lane ahead of the decision; the accepted lane's value is taken by one shuffle)
        auto lane_dist = [&]() {
          float dd = fabsf(__fsub_rn(cur.a, th));
          return dd > 180.f ? __fsub_rn(360.f, dd) : dd;
        };
        float d = lane_dist();
        float mn = __fmaf_rn(fminf(__fadd_rn(d, margin), dmax), inv0, margin);
        while (rem) {
          const bool mine = (rem >> lane) & 1u;
          const unsigned mm = __ballot_sync(0xFFFFFFFFu, mine && d <= hi);  // aligned or undecided
          if (!mm) break;                                                    // everything left is clearly not aligned
          const int k = __ffs(mm) - 1;
          const unsigned mi = __ballot_sync(0xFFFFFFFFu, mine && d < lo);   // certainly aligned
          if (!((mi >> k) & 1u)) {  // the first candidate sits in the band
            if (!fresh) {
              add_staged();
              th = plf_fast_atan2(sumdy, sumdx);
              inv0 = __fmul_rn(rsqrtf(__fadd_rn(__fmul_rn(sumdx, sumdx), __fmul_rn(sumdy, sumdy))), 1.02f);
              margin = margin0;
              lo = prec_deg - margin; hi = prec_deg + margin;
              fresh = true;
              d = lane_dist();
              mn = __fmaf_rn(fminf(__fadd_rn(d, margin), dmax), inv0, margin);
              continue;
            }
            float av = cur.a;
            asm volatile("" : "+f"(av));  // the f64 form of the angle is only needed here: keep it out of the hot loop
            const bool ex = lsd_aligned_rad((double)av * LSD_DEG2RAD, (double)th * LSD_DEG2RAD, prec);
            if (!((__ballot_sync(0xFFFFFFFFu, ex) >> k) & 1u)) {
              rem &= ~((2u << k) - 1u);  // k rejected by the exact test; the cells before it were clearly not aligned
              continue;
            }
          }
          const int ai = __shfl_sync(0xFFFFFFFFu, ci, k);
          margin = __shfl_sync(0xFFFFFFFFu, mn, k);
          lo = prec_deg - margin; hi = prec_deg + margin;
          rem &= ~(((2u << k) - 1u) | __shfl_sync(0xFFFFFFFFu, same, k));  // k, everything before it and k's cell: decided
          // lane 0 marks the cell used and appends it to the region / the queue (predicated: no divergent branch)
          asm volatile(
              "{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %0, 0;\n\t"
              "@p st.global.f32 [%1], %2;\n\t@p st.global.u32 [%3], %4;\n\t@p st.shared.u32 [%5], %4;\n\t}"
              ::"r"(l0), "l"(pb + (long long)ai * LSD_REC_BYTES), "f"(LSD_NOTDEF_F), "l"(regpts + (cursor + nreg)), "r"(ai),
                "r"(qs + ((nreg & (LSD_QCAP - 1)) << 2))
              : "memory");
          const uint32_t en = nreg - rn;   // the new entry's place in the next round
          ++nreg;
          lsd_prefetch(pb + (long long)(ai + poff) * LSD_REC_BYTES);
          if (ni == ai) nxt.a = LSD_NOTDEF_F;  // a look-ahead copy of this cell is stale
          if (en < 3) {                      // the new entry is one of the next round's: load its neighbourhood now
            if (grp == (int)en) ni = ai + noff;
            __syncwarp();                    // after lane 0's store of this round's acceptances
            if (grp == (int)en) nxt = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)ni * LSD_REC_BYTES));
          }
          // stage the member's term: lane k holds its record (landed: its angle was just tested)
          if (qpos - qwait == LSD_CSQ) add_staged();   // ring full: its oldest slot is about to be reused
          if (lane == k)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(csb + ((qpos & (LSD_CSQ - 1)) << 3)),
                         "l"(lut_cs + cur.li) : "memory");
          ++qpos;
          mn = __fmaf_rn(fminf(__fadd_rn(d, margin), dmax), inv0, margin);
          fresh = false;
        }
        __syncwarp();
        r = rn;
      }
      if ((int)nreg >= min_reg_size) {
        if (nreg_out < max_regions) {
          if (!fresh) add_staged();   // the members accepted since S was last read (fresh: none)
          if (lane == 0) {
            // region angle handed to the rectangle fit: the seed's own angle for a 1-pixel region, else the angle of the sum
            const double reg_angle = nreg == 1 ? th_seed : (double)(fresh ? th : plf_fast_atan2(sumdy, sumdx)) * LSD_DEG2RAD;
            const unsigned long long bits = (unsigned long long)__double_as_longlong(reg_angle);
            regions[nreg_out] = make_uint4(cursor, nreg, (uint32_t)bits, (uint32_t)(bits >> 32));
          }
          ++nreg_out;
          cursor += nreg;
        } else if (lane == 0) {
          atomicOr(overflow, PLF_LSD_OVF_SEGMENTS);
        }
      }
      pending &= ~((2u << src) - 1u);
      if (pending) {
        a0 = (pending >> lane) & 1u ? __ldcg(&pix[seed].a) : LSD_NOTDEF_F;
        pending = __ballot_sync(0xFFFFFFFFu, a0 != LSD_NOTDEF_F);
      }
    }
  }
  if (lane == 0) nregions[im] = nreg_out;
}

#define LSD_GROW_ARGS LsdPix* __restrict__ pix_all, size_t pix_stride, size_t stride, int W, const uint32_t* __restrict__ order_all, \
    const float2* __restrict__ lut_seed, const float2* __restrict__ lut_cs, const int* __restrict__ nseeds, double prec, float prec_deg, \
    int min_reg_size, uint32_t* __restrict__ regpts_all, uint4* __restrict__ regions_all, int max_regions, int* __restrict__ nregions,   \
    int* __restrict__ overflow
#define LSD_GROW_PASS pix_all, pix_stride, stride, W, order_all, lut_seed, lut_cs, nseeds, prec, prec_deg, min_reg_size, regpts_all, regions_all, max_regions, nregions, overflow
__global__ void __launch_bounds__(32) k_lsd_grow(LSD_GROW_ARGS) { lsd_grow_body(LSD_GROW_PASS); }

// ---- rectangle fit -------------------------------------------------------------------------------------------
__device__ __forceinline__ double lsd_angle_diff(double a, double b) {
  double diff = a - b;
  while (diff <= -LSD_PI) diff += LSD_2PI;
  while (diff > LSD_PI) diff -= LSD_2PI;
  if (diff < 0.0) diff = -diff;
  return diff;
}

// The rectangle fit runs one THREAD per region (three sequential f64 passes over its points, in the reference's
// order), so a warp takes as long as its largest region; region sizes span 17 .. several thousand pixels in detection
// order.  k_lsd_rect_order permutes each image's regions into power-of-two size classes, largest first, so that the 32
// regions of a warp have similar lengths (outputs stay indexed by the original region number).
#define LSD_SIZE_BINS 20
__global__ void __launch_bounds__(256) k_lsd_rect_order(const uint4* __restrict__ regions_all, int max_regions,
                                                        const int* __restrict__ nregions, uint32_t* __restrict__ perm_all) {
  __shared__ int cnt[LSD_SIZE_BINS], pos[LSD_SIZE_BINS];
  const int im = blockIdx.x, n = min(nregions[im], max_regions);
  const uint4* regions = regions_all + (size_t)im * max_regions;
  uint32_t* perm = perm_all + (size_t)im * max_regions;
  if (threadIdx.x < LSD_SIZE_BINS) cnt[threadIdx.x] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += 256) atomicAdd(&cnt[min(31 - __clz((int)regions[i].y | 1), LSD_SIZE_BINS - 1)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int b = LSD_SIZE_BINS - 1; b >= 0; --b) { pos[b] = run; run += cnt[b]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += 256)
    perm[atomicAdd(&pos[min(31 - __clz((int)regions[i].y | 1), LSD_SIZE_BINS - 1)], 1)] = (uint32_t)i;
}

__global__ void __launch_bounds__(128) k_lsd_rects(const LsdPix* __restrict__ pix_all, size_t pix_stride, size_t stride, int W,
                                                   const uint32_t* __restrict__ regpts_all,
                                                   const uint4* __restrict__ regions_all, int max_regions,
                                                   const int* __restrict__ nregions, const uint32_t* __restrict__ perm_all,
                                                   double prec, double scale, float4* __restrict__ segs_all) {
  const int im = blockIdx.y, slot = blockIdx.x * 128 + threadIdx.x;
  if (slot >= nregions[im]) return;
  const int ri = (int)perm_all[(size_t)im * max_regions + slot];
  const uint4 R = regions_all[(size_t)im * max_regions + ri];
  const uint32_t* pts = regpts_all + (size_t)im * stride + R.x;
  // the gradient of a region point comes back from its record: li = (gx + 510) * 1021 + (gy + 510) (region growing only
  // overwrites the record's angle)
  const LsdPix* recs = pix_all + (size_t)im * pix_stride;
  const int n = (int)R.y;
  const double reg_angle = __longlong_as_double((long long)(((unsigned long long)R.w << 32) | R.z));
  // The sums run in the region's point order (bit-exact with the CPU loop); what is batched is the LOADS: the point
  // indices and the gradients of 8 points are fetched before their terms are added, so the dependent pts[k] -> record
  // round trips overlap instead of serialising (the thread is otherwise one L2 / DRAM latency per point).
  constexpr int PF = 8;
  double x = 0, y = 0, sum = 0;
  for (int k0 = 0; k0 < n; k0 += PF) {
    uint32_t pp[PF];
    short2 gg[PF];
#pragma unroll
    for (int j = 0; j < PF; ++j) pp[j] = k0 + j < n ? pts[k0 + j] : 0u;
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      const uint32_t li = k0 + j < n ? __ldg(&recs[pp[j]].li) : 0u;
      const int gxv = (int)(li / (uint32_t)LSD_LUT_DIM);
      gg[j] = make_short2((short)(gxv - 510), (short)((int)li - gxv * LSD_LUT_DIM - 510));
    }
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      if (k0 + j < n) {
        const uint32_t p = pp[j];
        const int py = (int)(p / (uint32_t)W), px = (int)p - py * W;
        const double wgt = sqrt((double)(gg[j].x * gg[j].x + gg[j].y * gg[j].y) / 4.0);
        x += (double)px * wgt;
        y += (double)py * wgt;
        sum += wgt;
      }
    }
  }
  x /= sum;
  y /= sum;
  double Ixx = 0, Iyy = 0, Ixy = 0;
  for (int k0 = 0; k0 < n; k0 += PF) {
    uint32_t pp[PF];
    short2 gg[PF];
#pragma unroll
    for (int j = 0; j < PF; ++j) pp[j] = k0 + j < n ? pts[k0 + j] : 0u;
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      const uint32_t li = k0 + j < n ? __ldg(&recs[pp[j]].li) : 0u;
      const int gxv = (int)(li / (uint32_t)LSD_LUT_DIM);
      gg[j] = make_short2((short)(gxv - 510), (short)((int)li - gxv * LSD_LUT_DIM - 510));
    }
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      if (k0 + j < n) {
        const uint32_t p = pp[j];
        const int py = (int)(p / (uint32_t)W), px = (int)p - py * W;
        const double wgt = sqrt((double)(gg[j].x * gg[j].x + gg[j].y * gg[j].y) / 4.0);
        const double dx = (double)px - x, dy = (double)py - y;
        Ixx += dy * dy * wgt;
        Iyy += dx * dx * wgt;
        Ixy -= dx * dy * wgt;
      }
    }
  }
  const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
  double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)plf_fast_atan2((float)(lambda - Ixx), (float)Ixy)
                                         : (double)plf_fast_atan2((float)Ixy, (float)(lambda - Iyy));
  theta *= LSD_DEG2RAD;
  if (lsd_angle_diff(theta, reg_angle) > prec) theta += LSD_PI;
  const double dx = cos(theta), dy = sin(theta);
  double l_min = 0, l_max = 0;
  for (int k0 = 0; k0 < n; k0 += PF) {
    uint32_t pp[PF];
#pragma unroll
    for (int j = 0; j < PF; ++j) pp[j] = k0 + j < n ? pts[k0 + j] : 0u;
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      if (k0 + j < n) {
        const uint32_t p = pp[j];
        const int py = (int)(p / (uint32_t)W), px = (int)p - py * W;
        const double regdx = (double)px - x, regdy = (double)py - y;
        const double l = regdx * dx + regdy * dy;
        if (l > l_max) l_max = l;
        else if (l < l_min) l_min = l;
      }
    }
  }
  double x1 = x + l_min * dx, y1 = y + l_min * dy, x2 = x + l_max * dx, y2 = y + l_max * dy;
  x1 += 0.5; y1 += 0.5; x2 += 0.5; y2 += 0.5;
  if (scale != 1) { x1 /= scale; y1 /= scale; x2 /= scale; y2 /= scale; }
  segs_all[(size_t)im * max_regions + ri] = make_float4((float)x1, (float)y1, (float)x2, (float)y2);
}

// ---- KeyLines (LSDDetector_custom.cpp:267-308) + stvo-pl top-K ---------------------------------------------------
// MASKED (plf_set_sequence_mask, plf_detect_lines_masked): masks[im] is image im's mask (plf_pitch16(w) bytes per row) or
// NULL.  A KeyLine whose two end points both truncate onto a 0 of the mask is deleted after the length filter and before
// the top-K, keeping the class_id it was given among the lines of sufficient length (LSDDetector_custom.cpp:310-322 runs
// after :299 numbers them).  The unmasked instantiation ignores masks.
// prm (plf_lsd_grow): image im keeps the top lsd_nfeatures of the lines longer than min_line_length min(w, h), its pair's
// settings prm[im / 2].
#define KL_SORT_CAP 4096
template <bool MASKED>
__global__ void __launch_bounds__(1024) k_keylines(const float4* __restrict__ segs_all, const int* __restrict__ nsegs,
                                                   int max_regions, int w, int h,
                                                   plf_keyline* __restrict__ kls_all, plf_keyline* __restrict__ kls_out,
                                                   int max_lines, int* __restrict__ nlines, int* __restrict__ overflow,
                                                   const uint8_t* const* __restrict__ masks, const PlfPairPrm* __restrict__ prm) {
  __shared__ unsigned long long keys[KL_SORT_CAP];  // (response desc, index asc) for the top-K
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int im = blockIdx.x, tid = threadIdx.x;
  const int nfeatures = prm[im >> 1].lsd_nfeatures;
  const double min_length = (double)prm[im >> 1].min_line_length * (double)min(w, h);
  const int n = min(nsegs[im], max_regions);
  const float4* segs = segs_all + (size_t)im * max_regions;
  plf_keyline* all = kls_all + (size_t)im * max_regions;
  plf_keyline* out = kls_out + (size_t)im * max_lines;
  // pass 1: accept flags + ordered compaction (class_id = running counter of accepted lines, :299)
  int base = 0;
  const uint8_t* mk = nullptr;
  const int mp = (w + 15) & ~15;
  int cbase = 0;   // MASKED: lines of sufficient length so far (the class_id counter), base counting those the mask keeps
  if constexpr (MASKED) mk = masks[im];
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    bool ok = false, len_ok = false;   // len_ok: MASKED only
    plf_keyline kl;
    if (i < n) {
      float4 e = segs[i];
      if (e.x < 0) e.x = 0;
      if (e.x >= w) e.x = (float)w - 1.0f;
      if (e.z < 0) e.z = 0;
      if (e.z >= w) e.z = (float)w - 1.0f;
      if (e.y < 0) e.y = 0;
      if (e.y >= h) e.y = (float)h - 1.0f;
      if (e.w < 0) e.w = 0;
      if (e.w >= h) e.w = (float)h - 1.0f;
      const double ddx = (double)__fsub_rn(e.x, e.z), ddy = (double)__fsub_rn(e.y, e.w);
      const double length = (double)(float)sqrt(ddx * ddx + ddy * ddy);
      ok = length > min_length;
      if constexpr (MASKED) {
        len_ok = ok;
        if (ok && mk)   // the end points are clamped into the image above: (int) truncates onto one of its pixels
          ok = mk[(size_t)(int)e.y * mp + (int)e.x] != 0 || mk[(size_t)(int)e.w * mp + (int)e.z] != 0;
      }
      if (ok) {
        kl.startPointX = e.x; kl.startPointY = e.y; kl.endPointX = e.z; kl.endPointY = e.w;  // octaveScale = 1
        kl.sPointInOctaveX = e.x; kl.sPointInOctaveY = e.y; kl.ePointInOctaveX = e.z; kl.ePointInOctaveY = e.w;
        kl.lineLength = (float)length;
        const int x1 = __float2int_rn(e.x), y1 = __float2int_rn(e.y), x2 = __float2int_rn(e.z), y2 = __float2int_rn(e.w);
        kl.numOfPixels = max(abs(x2 - x1), abs(y2 - y1)) + 1;  // LineIterator(8-connected).count
        // atan2(float, float) at LSDDetector_custom.cpp:286 is glibc's atan2f in the reference build (bit-exact port)
        kl.angle = glibc_atan2f(__fsub_rn(kl.endPointY, kl.startPointY), __fsub_rn(kl.endPointX, kl.startPointX));
        kl.octave = 0;
        kl.size = __fmul_rn(__fsub_rn(kl.endPointX, kl.startPointX), __fsub_rn(kl.endPointY, kl.startPointY));
        kl.response = __fdiv_rn(kl.lineLength, (float)max(w, h));
        kl.ptx = __fdiv_rn(__fadd_rn(kl.endPointX, kl.startPointX), 2.f);
        kl.pty = __fdiv_rn(__fadd_rn(kl.endPointY, kl.startPointY), 2.f);
      }
    }
    // block exclusive scan of ok flags (MASKED: the length flags counted in the high half-word, ok in the low one)
    if constexpr (MASKED) {
      s_scan[tid] = (len_ok ? 0x10000 : 0) | (ok ? 1 : 0);
    } else {
      s_scan[tid] = ok ? 1 : 0;
    }
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      const int v = tid >= off ? s_scan[tid - off] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    const int incl = s_scan[tid];
    if (tid == 1023) s_total = incl;
    if constexpr (MASKED) {
      if (ok) {
        kl.class_id = cbase + (incl >> 16) - 1;
        all[base + (incl & 0xFFFF) - 1] = kl;
      }
      __syncthreads();
      base += s_total & 0xFFFF;
      cbase += s_total >> 16;
    } else {
      if (ok) {
        kl.class_id = base + incl - 1;
        all[base + incl - 1] = kl;
      }
      __syncthreads();
      base += s_total;
    }
    __syncthreads();
  }
  const int m = base;
  int keep = m;
  if (nfeatures != 0 && m > nfeatures) {
    // stvo-pl: sort by response (descending), keep nfeatures, class_id = rank.  Ties: detection order.
    if (m > KL_SORT_CAP) {
      if (tid == 0) atomicOr(overflow, PLF_LSD_OVF_SORT);
    }
    const int mm = min(m, KL_SORT_CAP);
    int p2 = 1;
    while (p2 < mm) p2 <<= 1;
    for (int i = tid; i < p2; i += 1024) {
      if (i < mm) {
        const uint32_t rb = __float_as_uint(all[i].response);  // responses are positive floats: bit order == value order
        keys[i] = ((unsigned long long)(~rb) << 32) | (uint32_t)i;
      } else {
        keys[i] = ~0ull;
      }
    }
    __syncthreads();
    for (int k = 2; k <= p2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < p2; i += 1024) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = keys[i], b = keys[ixj];
            const bool up = (i & k) == 0;
            if ((a > b) == up) {
              keys[i] = b;
              keys[ixj] = a;
            }
          }
        }
        __syncthreads();
      }
    keep = nfeatures;
    if (keep > max_lines) {
      if (tid == 0) atomicOr(overflow, PLF_LSD_OVF_LINES);
      keep = max_lines;
    }
    for (int i = tid; i < keep; i += 1024) {
      plf_keyline kl = all[(uint32_t)(keys[i] & 0xFFFFFFFFu)];
      kl.class_id = i;
      out[i] = kl;
    }
  } else {
    if (keep > max_lines) {
      if (tid == 0) atomicOr(overflow, PLF_LSD_OVF_LINES);
      keep = max_lines;
    }
    for (int i = tid; i < keep; i += 1024) out[i] = all[i];
  }
  if (tid == 0) nlines[im] = keep;
}

// ---- host side -------------------------------------------------------------------------------------------------
void plf_lsd_free(LsdState* s) {
  if (!s) return;
  s->bufs.release();
  s->tabs.release();
  delete s;
}

// getGaussianKernelBitExact + fixed-point error diffusion (see oracle/lbd.c orc_gaussian_kernel_q8)
static void gaussian_taps_q8(int ksize, double sigma, int* taps) {
  double k[33], sum = 0;
  const double scale2x = -0.5 / (sigma * sigma);
  for (int i = 0; i < ksize; i++) {
    const double x = i - (ksize - 1) * 0.5;
    k[i] = exp(scale2x * x * x);
    sum += k[i];
  }
  sum = 1. / sum;
  double err = 0;
  int s = 0;
  for (int i = 0; i < ksize / 2; i++) {
    const double adj = k[i] * sum * 256.0 + err;
    const int v0 = (int)nearbyint(adj);
    err = adj - v0;
    taps[i] = taps[ksize - 1 - i] = v0;
    s += v0;
  }
  taps[ksize / 2] = 256 - 2 * s;
}

// The Gaussian pre-blur of scale != 1: its size (0 at scale 1) and, up to LSD_PRE_KS_MAX, its Q8 taps.
static void lsd_blur_taps(const plf_params& P, int* ksize, int* taps) {
  *ksize = 0;
  if (P.lsd_scale == 1.0) return;
  const double scale = P.lsd_scale;
  const double sigma = (scale < 1) ? (P.lsd_sigma_scale / scale) : P.lsd_sigma_scale;
  const unsigned hk = (unsigned)(ceil(sigma * sqrt(2 * 3.0 * log(10.0))));
  *ksize = 1 + 2 * (int)hk;
  if (*ksize <= LSD_PRE_KS_MAX) gaussian_taps_q8(*ksize, sigma, taps);
}

// k_lsd_pre's launch for a w x h image resampled to ws x hs, from the resize tables ox, oy:
//   KS      the pre-blur's taps; 1 at scale 1 and where the centre tap is 256.  gaussian_taps_q8 makes the side taps
//           non-negative and below 128, so a 256 centre (the one tap a byte cannot hold) means every side tap is 0 and
//           the blur is a copy;
//   TH      the most scaled rows (<= LSD_PRE_TH) whose footprint plus the blur halo fits the box's rows in every band;
//   NP, PW  the fewest pieces of PW scaled columns (a multiple of 4) per segment whose footprints fit LSD_PRE_HW blurred
//           columns in every segment;
//   packed  plf_resize_packed_ok.
// false where even one scaled row does not fit the box (downsampling by more than about 1 / (22 - 2R)).
static bool lsd_pre_geom(const plf_params& P, int w, int ws, int hs, const int* ox, const int* oy, LsdPreGeom* g) {
  int ks, taps[LSD_PRE_KS_MAX];
  lsd_blur_taps(P, &ks, taps);
  *g = LsdPreGeom();
  if (ks > LSD_PRE_KS_MAX) return false;
  if (ks > 1 && taps[ks / 2] < 256) {
    uint32_t tw[4] = {0u, 0u, 0u, 0u};
    for (int k = 0; k < ks; ++k) tw[k >> 2] |= (uint32_t)taps[k] << (8 * (k & 3));
    g->ks = ks;
    g->taps = make_uint4(tw[0], tw[1], tw[2], tw[3]);
  }
  const int R = g->ks / 2;
  for (g->th = LSD_PRE_TH; g->th > 0; --g->th) {
    bool fits = true;
    for (int y0 = 0; y0 < hs && fits; y0 += g->th) {
      const LsdPreFoot f = lsd_pre_foot(ox, oy, 0, 0, y0, std::min(y0 + g->th, hs - 1), R);
      fits = f.sy1 - f.sy0 + 1 + 2 * R <= LSD_PRE_BOXH;
    }
    if (fits) break;
  }
  if (g->th == 0) return false;
  for (g->np = 1;; ++g->np) {
    g->pw = ((LSD_SEG + g->np) / g->np + 3) & ~3;   // ceil((LSD_SEG + 1) / np), whole groups of four
    bool fits = true;
    for (int x0 = 0; x0 < ws && fits; x0 += LSD_SEG) {
      const int nsc = std::min(LSD_SEG + 1, ws - x0);
      for (int u0 = 0; u0 < nsc && fits; u0 += g->pw) {
        const LsdPreFoot f = lsd_pre_foot(ox, oy, x0 + u0, x0 + std::min(u0 + g->pw, nsc) - 1, 0, 0, R);
        fits = f.sx1 - f.bxc + 1 <= LSD_PRE_HW;
      }
    }
    if (fits) break;
    if (g->pw == 4) return false;
  }
  g->packed = plf_resize_packed_ok(w, ws);
  return true;
}

// The sizes an LSD state for nimg images of w x h takes from the context's parameters and limits.
static void lsd_set_sizes(const plf_ctx* ctx, LsdState* s, int w, int h, int nimg, bool two_parities) {
  s->w = w; s->h = h; s->nimg = nimg;
  s->two_parities = two_parities;
  s->scale = ctx->params.lsd_scale;
  s->n_bins = ctx->params.lsd_n_bins;
  s->ws = s->scale != 1.0 ? (int)nearbyint(w * s->scale) : w;
  s->hs = s->scale != 1.0 ? (int)nearbyint(h * s->scale) : h;
  s->max_regions = ctx->limits.max_segments;
  s->max_lines = ctx->limits.max_lines;
}

// Records of one record map: nimg images of pix_stride records, plus 3 rows + 8 records of slack on both sides (the
// look-ahead prefetches need no clamping).
static size_t lsd_pix_pad(const LsdState* s) { return 3 * (size_t)s->ws + 8; }
static size_t lsd_pix_records(const LsdState* s) { return s->pix_stride * s->nimg + 2 * lsd_pix_pad(s); }

// The device buffers of an LSD state whose sizes are set (lsd_set_sizes), and the layout derived from those sizes.
static void lsd_buffers(LsdState* s, DevBufList& b) {
  const size_t N = (size_t)s->nimg, As = (size_t)s->ws * s->hs, R = (size_t)s->max_regions;
  s->nxb = (s->ws + LSD_SEG - 1) / LSD_SEG;
  s->pix_stride = As + (size_t)s->ws + 1;
  b.add(s->seedlist, As * N);
  b.add(s->segcnt, N * s->hs * s->nxb);
  b.add(s->rect_perm, N * R);
  b.add(s->maxmag2, N);
  b.add(s->regpts, As * N);
  b.add(s->regions, N * R);
  b.add(s->nregions, N);
  b.add(s->segs, N * R);
  b.add(s->kls_all, N * R);
  // buffers that cross from the pre-grow phase to the growing (or to the match phase) exist twice (parity of the batch),
  // so that batch i+1 can be extracted while batch i is still growing regions
  for (int p = 0; p < (s->two_parities ? 2 : 1); ++p) {
    b.add(s->pix_raw[p], lsd_pix_records(s));
    b.add(s->nseeds[p], N);
    b.add(s->order[p], As * N);
    b.add(s->kls[p], N * s->max_lines);
    b.add(s->nlines[p], N);
  }
  b.add(s->overflow, 1);
  s->rs_x_off = 0;
  s->rs_y_off = 2 * (size_t)s->ws;
  s->rs_xp_off = (s->rs_y_off + 2 * (size_t)s->hs + 3) & ~(size_t)3;   // 16-byte aligned: read with 128-bit loads
  s->tabs.add(s->rs_tab, s->rs_xp_off + plf_resize_packed_len(s->ws));
}

// The resize tables of s (identity at scale 1), laid out as rs_tab (lsd_buffers).
static std::vector<int> lsd_resize_tables(const LsdState* s) {
  std::vector<int> tab(s->rs_xp_off + plf_resize_packed_len(s->ws));
  plf_linear_coeffs_host(s->w, s->ws, 1.0 / s->scale, &tab[s->rs_x_off], &tab[s->rs_x_off + s->ws]);
  plf_linear_coeffs_host(s->h, s->hs, 1.0 / s->scale, &tab[s->rs_y_off], &tab[s->rs_y_off + s->hs]);
  plf_resize_pack_x(&tab[s->rs_x_off], &tab[s->rs_x_off + s->ws], s->ws, &tab[s->rs_xp_off]);
  return tab;
}

size_t plf_lsd_footprint(const plf_ctx* ctx, int n, const int* wh, int nimg, bool two_parities) {
  std::vector<LsdState> z(n);
  size_t tabs = 0;
  for (int i = 0; i < n; ++i) {
    lsd_set_sizes(ctx, &z[i], wh[2 * i], wh[2 * i + 1], nimg, two_parities);
    lsd_buffers(&z[i], z[i].bufs);
    z[0].bufs.grow(z[i].bufs);
    tabs += z[i].tabs.bytes();
  }
  return z[0].bufs.bytes() + tabs;
}

static plf_status lsd_tables_build(plf_ctx* ctx, LsdTables* t) {
  const plf_params& P = ctx->params;
  if (P.lsd_refine != 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: only lsd_refine = 0 (LSD_REFINE_NONE, the reference configs) is supported");
  if (P.lsd_n_bins < 1 || P.lsd_n_bins > LSD_BINS_MAX)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: lsd_n_bins must be in [1,%d]", LSD_BINS_MAX);
  t->prec = LSD_PI * P.lsd_ang_th / 180;
  t->p = P.lsd_ang_th / 180;
  t->rho = P.lsd_quant / sin(t->prec);
  int ksize, taps[LSD_PRE_KS_MAX];
  lsd_blur_taps(P, &ksize, taps);
  if (ksize > LSD_PRE_KS_MAX)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: Gaussian kernel %d > %d unsupported", ksize, LSD_PRE_KS_MAX);
  for (t->m2_min = 0; t->m2_min <= 2 * 510 * 510; ++t->m2_min)  // same double expression as the kernels
    if (!(sqrt((double)t->m2_min / 4.0) <= t->rho)) break;
  const size_t LUT = (size_t)LSD_LUT_DIM * LSD_LUT_DIM;
  t->bufs.add(t->angle_lut, LUT);
  t->bufs.add(t->cs_lut, LUT);
  t->bufs.add(t->seed_lut, LUT);
  plf_status st = t->bufs.alloc(ctx, "LSD tables");
  if (st) return st;
  k_lsd_build_lut<<<(LSD_LUT_DIM * LSD_LUT_DIM + 255) / 256, 256, 0, ctx->stream>>>(t->rho, t->angle_lut, t->cs_lut, t->seed_lut);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// Once per context, before any LSD state.
plf_status plf_lsd_tables(plf_ctx* ctx) {
  if (ctx->lsd_tables) return PLF_OK;
  LsdTables* t = new LsdTables();
  const plf_status st = lsd_tables_build(ctx, t);
  if (st) {
    t->bufs.release();
    delete t;
    return st;
  }
  ctx->lsd_tables = t;
  return PLF_OK;
}

void plf_lsd_tables_free(plf_ctx* ctx) {
  if (!ctx->lsd_tables) return;
  ctx->lsd_tables->bufs.release();
  delete ctx->lsd_tables;
  ctx->lsd_tables = nullptr;
}

// The sizes of s for nimg images of w x h, checked, its pre-grow launch chosen and its buffers listed (not allocated).
// Host only.
static plf_status lsd_layout(plf_ctx* ctx, LsdState* s, int w, int h, int nimg, bool two_parities) {
  lsd_set_sizes(ctx, s, w, h, nimg, two_parities);
  if (s->ws >= 65536 || s->hs >= 65536 || s->ws < 3 || s->hs < 3)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: scaled image %dx%d out of range", s->ws, s->hs);
  lsd_buffers(s, s->bufs);
  const std::vector<int> tab = lsd_resize_tables(s);
  if (!lsd_pre_geom(ctx->params, w, s->ws, s->hs, &tab[s->rs_x_off], &tab[s->rs_y_off], &s->pre))
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: lsd_scale %g with lsd_sigma_scale %g: one scaled row of %dx%d needs more source rows "
                    "than the pre-grow tile holds", s->scale, ctx->params.lsd_sigma_scale, w, h);
  return PLF_OK;
}

plf_status plf_lsd_check_size(plf_ctx* ctx, int w, int h, int* ws, int* hs) {
  LsdState s;
  const plf_status st = lsd_layout(ctx, &s, w, h, 1, false);
  if (!st && ws) { *ws = s.ws; *hs = s.hs; }
  return st;
}

// s's own resize tables and record map pointers, once its buffers exist.
static plf_status lsd_ready(plf_ctx* ctx, LsdState* s) {
  const double LOG_NT = 5 * (log10((double)s->ws) + log10((double)s->hs)) / 2 + log10(11.0);
  s->min_reg_size = (int)(size_t)(-LOG_NT / log10(ctx->lsd_tables->p));
  plf_status st = s->tabs.alloc(ctx, "LSD");
  if (st) return st;
  for (int p = 0; p < (s->two_parities ? 2 : 1); ++p) s->pix[p] = s->pix_raw[p] + lsd_pix_pad(s);
  const std::vector<int> tab = lsd_resize_tables(s);
  PLF_CUDA(ctx, cudaMemcpyAsync(s->rs_tab, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// The states of n image sizes share one set of buffers, each sized for the largest of them.  Every record map is filled
// with NOTDEF whole, guards and slack of every size's layout included; k_lsd_fill_notdef says why it stays so whichever
// size the next batch has (DESIGN.md section 8).
plf_status plf_lsd_create_sizes(plf_ctx* ctx, int n, const int* wh, int nimg, bool two_parities, LsdState** out) {
  plf_status st = plf_lsd_tables(ctx);
  if (st) return st;
  std::vector<LsdState*> v(n, nullptr);
  size_t records = 0;
  for (int i = 0; i < n && !st; ++i) {
    v[i] = new LsdState();
    st = lsd_layout(ctx, v[i], wh[2 * i], wh[2 * i + 1], nimg, two_parities);
    if (!st) records = std::max(records, lsd_pix_records(v[i]));
  }
  if (!st) {
    for (int i = 1; i < n; ++i) v[0]->bufs.grow(v[i]->bufs);
    st = v[0]->bufs.alloc(ctx, "LSD");
  }
  if (!st) {
    for (int i = 1; i < n; ++i) v[0]->bufs.lend(v[i]->bufs);
    for (int p = 0; p < (two_parities ? 2 : 1) && !st; ++p) {
      k_lsd_fill_notdef<<<(unsigned)((records + 255) / 256), 256, 0, ctx->stream>>>(v[0]->pix_raw[p], records);
      ctx->launches++;
      if (cudaGetLastError() != cudaSuccess) st = plf_fail(ctx, PLF_ERR_CUDA, "LSD: filling the record maps failed");
    }
    if (!st && cudaMemsetAsync(v[0]->overflow, 0, sizeof(int), ctx->stream) != cudaSuccess)
      st = plf_fail(ctx, PLF_ERR_CUDA, "LSD: clearing the overflow flag failed");
  }
  for (int i = 0; i < n && !st; ++i) st = lsd_ready(ctx, v[i]);
  if (st) {
    for (LsdState* s : v) plf_lsd_free(s);
    return st;
  }
  std::copy(v.begin(), v.end(), out);
  return PLF_OK;
}

plf_status plf_lsd_create(plf_ctx* ctx, int w, int h, int nimg, bool two_parities, LsdState** out) {
  const int wh[2] = {w, h};
  return plf_lsd_create_sizes(ctx, 1, wh, nimg, two_parities, out);
}

// LSD on images [0, n) of a batch resident on the device, in two phases so that callers can overlap them with other
// work: `pre` = blur, resample, gradient and seed ordering (bandwidth-bound), `grow` = region growing, rectangle fit and
// the KeyLine stage (latency-bound).  `par` selects the buffer set that carries data from pre to grow.  The state must
// hold >= n images.  Enqueued on cs; results stay on the device.
plf_status plf_lsd_pre(plf_ctx* ctx, cudaStream_t cs, LsdState* s, const uint8_t* d_imgs, size_t img_stride, int pitch, int par, int n) {
  if (s->nimg < n) return plf_fail(ctx, PLF_ERR_STATE, "plf_lsd_pre: %d images > the state's %d", n, s->nimg);
  const LsdTables& T = *ctx->lsd_tables;
  const LsdPreGeom& g = s->pre;
  const int W = s->ws, H = s->hs;
  const size_t As = (size_t)W * H;
  LsdPix* pix = s->pix[par] + (s->ws + 1);  // pixel (0,0) of the first image
  // the tensor map is encoded per call (host only, a few microseconds per batch)
  CUtensorMap tm;
  if (!plf_tma_encode_u8_blocks(&tm, d_imgs, s->w, s->h, n, pitch, img_stride, LSD_PRE_BOXW / 16, LSD_PRE_BOXH))
    return plf_fail(ctx, PLF_ERR_CUDA, "LSD: cuTensorMapEncodeTiled failed for the source images (pitch %d, stride %zu)", pitch, img_stride);
  PLF_CUDA(ctx, cudaMemsetAsync(s->maxmag2, 0xFF, (size_t)n * sizeof(int), cs));  // -1
  // no 3-tap kernel: its side tap (sigma <= 0.27) rounds to 0, so it is the copy KS = 1 runs
  static const decltype(&k_lsd_pre<1>) kern[] = {k_lsd_pre<1>, nullptr, k_lsd_pre<5>, k_lsd_pre<7>,
                                                 k_lsd_pre<9>, k_lsd_pre<11>, k_lsd_pre<13>, k_lsd_pre<15>};
  static_assert(sizeof kern / sizeof kern[0] == LSD_PRE_KS_MAX / 2 + 1, "one entry per odd KS");
  const size_t smem = g.np > 1 ? (size_t)(g.th + 1) * LSD_PRE_SP : 0;
  kern[g.ks / 2]<<<dim3(s->nxb, (H + g.th - 1) / g.th, n), LSD_PRE_THREADS, smem, cs>>>(
      tm, s->w, s->h, W, H, g, s->rs_tab + s->rs_x_off, reinterpret_cast<const int4*>(s->rs_tab + s->rs_xp_off),
      s->rs_tab + s->rs_y_off, T.angle_lut, T.m2_min, As, pix, s->pix_stride, s->seedlist, s->segcnt, s->nxb, s->maxmag2);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "lsd.k_lsd_pre");
  k_lsd_seed_order<<<n, LSD_SO_THREADS, lsd_seed_order_smem(s->n_bins), cs>>>(s->seedlist, s->segcnt, As, W, H, s->nxb, s->n_bins,
                                                                              s->maxmag2, s->order[par], s->nseeds[par]);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "lsd.k_lsd_seed_order");
  return PLF_OK;
}

plf_status plf_lsd_grow(plf_ctx* ctx, cudaStream_t cs, LsdState* s, int par, int n, cudaEvent_t keylines_wait,
                        const uint8_t* const* masks, const PlfPairPrm* prm) {
  if (s->nimg < n) return plf_fail(ctx, PLF_ERR_STATE, "plf_lsd_grow: %d images > the state's %d", n, s->nimg);
  const LsdTables& T = *ctx->lsd_tables;
  const int w = s->w, h = s->h;
  const int W = s->ws, H = s->hs;
  const size_t As = (size_t)W * H;
  LsdPix* pix = s->pix[par] + (s->ws + 1);
  // one copy of regpts, regions, segs, kls_all: the growing, rectangle and KeyLine kernels of a batch run in stream order
  // before those of the next
  // (thread / lane per image, register-capped and unrolled variants and an angle-map layout were all bit-exact and were
  // not kept; DESIGN.md section 5 lists them)
  k_lsd_grow<<<n, 32, 0, cs>>>(pix, s->pix_stride, As, W, s->order[par], T.seed_lut, T.cs_lut, s->nseeds[par], T.prec, (float)(T.p * 180.0),
                               s->min_reg_size, s->regpts, s->regions, s->max_regions, s->nregions, s->overflow);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "lsd.k_lsd_grow");
  k_lsd_rect_order<<<n, 256, 0, cs>>>(s->regions, s->max_regions, s->nregions, s->rect_perm);
  PLF_LAUNCH_CHECK(ctx);
  k_lsd_rects<<<dim3((s->max_regions + 127) / 128, n), 128, 0, cs>>>(pix, s->pix_stride, As, W, s->regpts, s->regions, s->max_regions, s->nregions,
                                                                     s->rect_perm, T.prec, s->scale, s->segs);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "lsd.k_lsd_rects");
  if (keylines_wait) PLF_CUDA(ctx, cudaStreamWaitEvent(cs, keylines_wait, 0));
  if (masks)
    k_keylines<true><<<n, 1024, 0, cs>>>(s->segs, s->nregions, s->max_regions, w, h, s->kls_all,
                                         s->kls[par], s->max_lines, s->nlines[par], s->overflow, masks, prm);
  else
    k_keylines<false><<<n, 1024, 0, cs>>>(s->segs, s->nregions, s->max_regions, w, h, s->kls_all,
                                          s->kls[par], s->max_lines, s->nlines[par], s->overflow, nullptr, prm);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "lsd.k_keylines");
  return PLF_OK;
}

int* plf_lsd_overflow_flag(const LsdState* s) { return s->overflow; }

// Names every limit in `causes`.  max_segments and max_lines are plf_limits fields; KL_SORT_CAP is a fixed capacity of
// k_keylines that raising plf_limits does not move (lsd_nfeatures = 0 does not rank and has no such bound).
void plf_lsd_overflow_text(const LsdState* s, int causes, char* buf, size_t len) {
  char seg[96] = "", lines[96] = "", sort[160] = "";
  if (causes & PLF_LSD_OVF_SEGMENTS)
    snprintf(seg, sizeof seg, "more segments in an image than plf_limits.max_segments=%d; ", s->max_regions);
  if (causes & PLF_LSD_OVF_LINES)
    snprintf(lines, sizeof lines, "more lines to return from an image than plf_limits.max_lines=%d; ", s->max_lines);
  if (causes & PLF_LSD_OVF_SORT)
    snprintf(sort, sizeof sort, "more than KL_SORT_CAP=%d lines to rank for the top lsd_nfeatures (internal, not a plf_limits "
             "field); ", KL_SORT_CAP);
  snprintf(buf, len, "%s%s%s", seg, lines, sort);
  const size_t n = strlen(buf);
  if (n >= 2) buf[n - 2] = 0;   // the last "; "
}

void plf_lsd_outputs(const LsdState* s, int par, plf_keyline** kls, int** nlines, int* max_lines) {
  *kls = s->kls[par]; *nlines = s->nlines[par]; *max_lines = s->max_lines;
}

// LSD of the standalone operators on one w x h image at dimg, in ctx->lsd_standalone (rebuilt when the size changes).  prm:
// a one-entry device table of the context's settings.
static plf_status lsd_standalone(plf_ctx* ctx, const uint8_t* dimg, int pitch, int w, int h, const uint8_t* const* masks,
                                 const PlfPairPrm* prm) {
  LsdState*& s = ctx->lsd_standalone;
  plf_status st;
  if (s && (s->w != w || s->h != h)) {
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    plf_lsd_free(s);
    s = nullptr;
  }
  if (!s && (st = plf_lsd_create(ctx, w, h, 1, false, &s))) return st;
  if ((st = plf_lsd_pre(ctx, ctx->stream, s, dimg, (size_t)pitch * h, pitch, 0, 1))) return st;
  return plf_lsd_grow(ctx, ctx->stream, s, 0, 1, nullptr, masks, prm);
}

// `causes`: the ones that spoil what the caller returns.  plf_lsd returns the raw segments, which the KeyLine stage's
// capacities (it runs all the same) do not touch.
static plf_status lsd_check_overflow(plf_ctx* ctx, const LsdState* s, const char* what, int causes) {
  int ovf = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&ovf, s->overflow, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ovf) cudaMemsetAsync(s->overflow, 0, sizeof(int), ctx->stream);
  ovf &= causes;
  if (ovf) {
    char why[400];
    plf_lsd_overflow_text(s, ovf, why, sizeof why);
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: segment/line capacity exceeded: %s", what, why);
  }
  return PLF_OK;
}

extern "C" plf_status plf_lsd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, float* segs, int cap,
                              int* n_out) {
  if (!ctx || !img || !n_out || w < 3 || h < 3 || stride < w || cap < 0 || (cap > 0 && !segs))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_lsd: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  uint8_t* dimg;
  PlfPairPrm* dprm;
  DevBufList scr;
  scr.add(dimg, (size_t)pitch * h); scr.add(dprm, 1);
  if (plf_status st = scr.carve(ctx, PLF_SCR_LSD)) return st;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dprm, &ctx->pair, sizeof(PlfPairPrm), cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = lsd_standalone(ctx, dimg, pitch, w, h, nullptr, dprm);
  if (st) return st;
  const LsdState* s = ctx->lsd_standalone;
  int n = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&n, s->nregions, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  st = lsd_check_overflow(ctx, s, "plf_lsd", PLF_LSD_OVF_SEGMENTS);
  if (st) return st;
  *n_out = n;
  if (n > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_lsd: %d segments > caller capacity %d", n, cap);
  if (n > 0) {
    PLF_CUDA(ctx, cudaMemcpyAsync(segs, s->segs,(size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
}

// plf_detect_lines and plf_detect_lines_masked (mask NULL: unmasked).  The one-entry settings table (the context's), and the
// mask (level 0 of the pyramid layout, one plane) and its one-entry table, live in PLF_SCR_LSD beside the image.
static plf_status detect_lines(plf_ctx* ctx, const char* fn, const uint8_t* img, int w, int h, int stride, const uint8_t* mask,
                               int mask_stride, plf_keyline* keylines, uint8_t* desc, int cap, int* n_out) {
  const int pitch = plf_pitch16(w);
  uint8_t *dimg, *ddesc, *dmask = nullptr;
  const uint8_t** dtab = nullptr;
  short2* dgrad;
  PlfPairPrm* dprm;
  DevBufList scr;
  scr.add(dimg, (size_t)pitch * h); scr.add(dgrad, (size_t)w * h); scr.add(ddesc, (size_t)ctx->limits.max_lines * 32);
  scr.add(dprm, 1);
  if (mask) { scr.add(dmask, (size_t)pitch * h); scr.add(dtab, 1); }
  if (plf_status st = scr.carve(ctx, PLF_SCR_LSD)) return st;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dprm, &ctx->pair, sizeof(PlfPairPrm), cudaMemcpyHostToDevice, ctx->stream));
  if (mask) {
    const uint8_t* hp = dmask;
    PLF_CUDA(ctx, cudaMemcpy2DAsync(dmask, pitch, mask, mask_stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
    PLF_CUDA(ctx, cudaMemcpyAsync(dtab, &hp, sizeof hp, cudaMemcpyHostToDevice, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // hp is on this stack frame
  }
  plf_status st = lsd_standalone(ctx, dimg, pitch, w, h, dtab, dprm);
  if (st) return st;
  const LsdState* s = ctx->lsd_standalone;
  PlfTmaCache tm;
  st = plf_launch_blur5_sobel(ctx, ctx->stream, &tm, dimg, pitch, (size_t)pitch * h, w, h, 1, dgrad, 0);
  if (st) return st;
  st = plf_launch_lbd(ctx, ctx->stream, dgrad, 0, w, h, 1, s->kls[0], s->nlines[0], s->max_lines, ddesc, nullptr);
  if (st) return st;
  int n = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&n, s->nlines[0], sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  st = lsd_check_overflow(ctx, s, fn, PLF_LSD_OVF_SEGMENTS | PLF_LSD_OVF_LINES | PLF_LSD_OVF_SORT);
  if (st) return st;
  *n_out = n;
  if (n > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: %d lines > caller capacity %d", fn, n, cap);
  if (n > 0) {
    PLF_CUDA(ctx, cudaMemcpyAsync(keylines, s->kls[0], (size_t)n * sizeof(plf_keyline), cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaMemcpyAsync(desc, ddesc, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
}

extern "C" plf_status plf_detect_lines(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                                       plf_keyline* keylines, uint8_t* desc, int cap, int* n_out) {
  if (!ctx || !img || !n_out || w < 3 || h < 3 || stride < w || cap < 0 || (cap > 0 && (!keylines || !desc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_detect_lines: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  return detect_lines(ctx, "plf_detect_lines", img, w, h, stride, nullptr, 0, keylines, desc, cap, n_out);
}

extern "C" plf_status plf_detect_lines_masked(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, const uint8_t* mask,
                                              int mask_stride, plf_keyline* keylines, uint8_t* desc, int cap, int* n_out) {
  if (!ctx || !img || !n_out || w < 3 || h < 3 || stride < w || cap < 0 || (cap > 0 && (!keylines || !desc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_detect_lines_masked: bad arguments");
  if (!mask || mask_stride < w)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_detect_lines_masked: mask %s, need a w x h mask of stride >= w = %d",
                    mask ? "stride too small" : "is NULL", w);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  return detect_lines(ctx, "plf_detect_lines_masked", img, w, h, stride, mask, mask_stride, keylines, desc, cap, n_out);
}

// glibc sinf/cosf port check hook (tests only exercise it through this entry point)
__global__ void k_sincosf_probe(const float* in, float* s, float* c, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    s[i] = glibc_sinf(in[i]);
    c[i] = glibc_cosf(in[i]);
  }
}

extern "C" plf_status plf_debug_sincosf(plf_ctx* ctx, const float* in, float* s, float* c, int n) {
  if (!ctx || n <= 0) return PLF_ERR_INVALID;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  float *din, *ds, *dc;
  DevBufList scr;
  scr.add(din, n); scr.add(ds, n); scr.add(dc, n);
  if (plf_status st = scr.carve(ctx, PLF_SCR_LSD)) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(din, in, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  k_sincosf_probe<<<(n + 255) / 256, 256, 0, ctx->stream>>>(din, ds, dc, n);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(s, ds, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(c, dc, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// The gradient stage of LSD (records, seed lists, segcnt, maxmag2) of n source images by k_lsd_pre, in a state of its
// own: tests compare it byte for byte with a CPU reference.
extern "C" plf_status plf_debug_lsd_pre(plf_ctx* ctx, const uint8_t* imgs, int n, int w, int h, int pitch, size_t img_stride,
                                        int* sizes, uint32_t* pix, uint32_t* seedlist, int* segcnt, int* maxmag2) {
  if (!ctx || n < 1 || w < 3 || h < 3 || pitch < w || (pitch & 15) || img_stride < (size_t)pitch * h || (img_stride & 15) || !sizes)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_debug_lsd_pre: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  LsdState* s = nullptr;
  const int wh[2] = {w, h};
  plf_status st = plf_lsd_create_sizes(ctx, 1, wh, n, false, &s);
  if (st) return st;
  const int sz[6] = {s->ws, s->hs, s->nxb, s->pre.ks, s->pre.th, s->pre.np};
  std::copy(sz, sz + 6, sizes);
  if (!imgs || !pix || !seedlist || !segcnt || !maxmag2) {   // sizes only
    plf_lsd_free(s);
    return PLF_OK;
  }
  const size_t As = (size_t)s->ws * s->hs, nseg = (size_t)n * s->hs * s->nxb;
  uint8_t* dimg = nullptr;
  DevBufList ib;
  ib.add(dimg, (size_t)n * img_stride);
  st = ib.alloc(ctx, "plf_debug_lsd_pre");
  if (!st && (cudaMemcpyAsync(dimg, imgs, (size_t)n * img_stride, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess ||
              cudaMemsetAsync(s->seedlist, 0, As * n * sizeof(uint32_t), ctx->stream) != cudaSuccess ||
              cudaMemsetAsync(s->segcnt, 0, nseg * sizeof(int), ctx->stream) != cudaSuccess))
    st = plf_fail(ctx, PLF_ERR_CUDA, "plf_debug_lsd_pre: upload failed");
  if (!st) st = plf_lsd_pre(ctx, ctx->stream, s, dimg, img_stride, pitch, 0, n);
  if (!st && (cudaMemcpy2DAsync(pix, As * sizeof(LsdPix), s->pix[0] + (s->ws + 1), s->pix_stride * sizeof(LsdPix), As * sizeof(LsdPix), n,
                                cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
              cudaMemcpyAsync(seedlist, s->seedlist, As * n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
              cudaMemcpyAsync(segcnt, s->segcnt, nseg * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
              cudaMemcpyAsync(maxmag2, s->maxmag2, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
              cudaStreamSynchronize(ctx->stream) != cudaSuccess))
    st = plf_fail(ctx, PLF_ERR_CUDA, "plf_debug_lsd_pre: %s", cudaGetErrorString(cudaGetLastError()));
  cudaStreamSynchronize(ctx->stream);
  ib.release();
  plf_lsd_free(s);
  return st;
}

// The region-growing kernel stays resident for tens of milliseconds while the next batch's extraction kernels are
// co-scheduled on the same SMs.  The L1 / shared-memory split of an SM can only change while it is empty, so the split
// this kernel is launched with is the one those kernels have to live with: ask for a large shared-memory carve-out
// (164 KB) so that their CTAs (up to 17 KB of shared memory each) still fit at full occupancy.  Measured: k_orb_blur7 of
// the overlapped batch 28 ms -> 7 ms, step 83.3 -> 81.9 ms.
void plf_configure_lsd() {
  cudaFuncSetAttribute((const void*)k_lsd_grow, cudaFuncAttributePreferredSharedMemoryCarveout, 72);
  cudaFuncSetAttribute((const void*)k_lsd_seed_order, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)lsd_seed_order_smem(LSD_BINS_MAX));
}
