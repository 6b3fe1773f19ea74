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
//   k_lsd_build_lut / k_lsd_fill_notdef
//                    once per state: the gradient lookup tables, and every record of the record maps set to "undefined"
//   k_blur_q8_fast   separable Q8.8 Gaussian of 5 or 7 taps <= 255 (tile + halo staged by one TMA bulk-tensor copy, DP4A
//                    row pass), one rounding (k_blur_q8: generic variant for the other kernels, up to 15 taps)
//   k_resize_exact4  (orb.cu) INTER_LINEAR_EXACT resample to scale
//   k_lsd_grad       2x2 gradient; for the DEFINED pixels only (|grad| > rho, ~12 %): the 8-byte record {angle
//                    (cv::fastAtan2, degrees, f32, from a table keyed by (gx,gy)), table index}, and one packed entry
//                    (column, |grad|^2) of the raster-ordered seed list of the pixel's row segment; per-image max of |grad|^2.
//                    Nothing dense leaves the kernel (the record map restores itself to "undefined", see k_lsd_fill_notdef)
//   k_lsd_rowhist / k_lsd_binscan / k_lsd_scatter
//                    stable counting sort of the seed lists by magnitude bin (descending), raster order inside a
//                    bin == OpenCV's ordered_points
//   k_lsd_grow       region growing.  The algorithm is a sequential greedy partition (each accepted pixel updates the
//                    region angle that the next test uses, and regions compete through the `used` map), so it is run by
//                    ONE WARP PER IMAGE with thousands of images in flight: lanes 0..8 hold the 3x3 neighbourhood
//                    records of the current region point (fetched two queue entries ahead, L1-resident through a
//                    look-ahead prefetch), the alignment tests run lane-parallel in the reference order, and the
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

struct LsdState {
  int w = 0, h = 0, nimg = 0;
  int ws = 0, hs = 0;       // scaled size
  int ksize = 0;
  int taps[16];
  bool taps_u8 = false;     // every tap <= 255: the packed-byte fast blur applies (a 256 centre tap at small sigma does not)
  int n_bins = 1024;
  double scale = 1.2, prec = 0, p = 0, rho = 0;
  int min_reg_size = 0;
  int max_regions = 0, max_lines = 0;
  bool two_parities = false;
  uint8_t* blur = nullptr;    // [nimg][h][bp]   bp = plf_pitch16(w)
  uint8_t* scaled = nullptr;  // [nimg][hs][sp]  sp = plf_pitch16(ws)
  int bp = 0, sp = 0;
  PlfTmaCache tm_blur;        // source images of k_blur_q8_fast
  uint32_t* rect_perm = nullptr;  // [nimg][max_regions] regions in size-class order (k_lsd_rect_order)
  struct LsdPix* pix_raw[2] = {nullptr, nullptr};  // allocation (pix + look-ahead slack on both sides)
  struct LsdPix* pix[2] = {nullptr, nullptr};  // [nimg][guard + hs*ws]  {angle (deg, f32) | NOTDEF = undefined/used, table index}
  size_t pix_stride = 0;      // entries per image = guard (ws+1, permanently NOTDEF) + hs*ws
  int m2_min = 0;             // smallest gx^2+gy^2 whose gradient norm exceeds rho (defined pixel)
  // seed lists per row segment (LSD_SEG columns): segment (y, xb) owns the entries [y * ws + LSD_SEG * xb, ...);
  // an entry is column-in-segment | gx^2+gy^2 << LSD_COL_BITS (k_lsd_grad), then column | bin << LSD_COL_BITS (k_lsd_rowhist)
  uint32_t* seedlist = nullptr; // [nimg][hs*ws]
  int* segcnt = nullptr;        // [nimg][hs][nxb] entries per segment
  int nxb = 0;                  // segments per row
  int* maxmag2 = nullptr;     // [nimg]
  uint32_t* rowcnt = nullptr; // [nimg][nchunks][n_bins]  per-chunk bin counts -> prefixes
  uint32_t* binstart = nullptr; // [nimg][n_bins]
  // per batch parity: what crosses from the pre-grow chain to the growing (pix, order, nseeds) and what the match phase
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
  float* angle_lut = nullptr;   // [1021*1021] gradient (gx,gy) -> level-line angle (degrees) of a defined pixel
  float2* cs_lut = nullptr;     // [1021*1021] gradient (gx,gy) -> (cosf, sinf) of float(angle in radians): a member's term of the region sums
  float2* seed_lut = nullptr;   // [1021*1021] gradient (gx,gy) -> unit vector of a region seed
  DevBufList bufs;
};

__constant__ int c_lsd_taps[16];

// ---- fixed-point Gaussian (ksize <= 15) ------------------------------------------------------------------
#define BQ_TW 64
#define BQ_TH 16
#define BQ_R 7
__global__ void __launch_bounds__(256) k_blur_q8(const uint8_t* __restrict__ src, size_t src_stride, int pitch,
                                                 int w, int h, int r, uint8_t* __restrict__ dst, size_t dst_stride, int dpitch) {
  __shared__ uint8_t raw[BQ_TH + 2 * BQ_R][BQ_TW + 2 * BQ_R + 2];
  __shared__ uint16_t hrow[BQ_TH + 2 * BQ_R][BQ_TW];
  const uint8_t* s = src + (size_t)blockIdx.z * src_stride;
  uint8_t* d = dst + (size_t)blockIdx.z * dst_stride;
  const int x0 = blockIdx.x * BQ_TW, y0 = blockIdx.y * BQ_TH, tid = threadIdx.x;
  const int RW = BQ_TW + 2 * r, RH = BQ_TH + 2 * r;
  const int lane = tid & 31, wrp = tid >> 5;
  const bool interior = x0 >= r && x0 + BQ_TW + r <= w && y0 >= r && y0 + BQ_TH + r <= h;
  for (int ry = wrp; ry < RH; ry += 8) {  // one warp per row, lanes along x
    const int gy = interior ? y0 - r + ry : plf_reflect101(y0 - r + ry, h);
    const uint8_t* row = s + (size_t)gy * pitch;
    for (int rx = lane; rx < RW; rx += 32) raw[ry][rx] = row[interior ? x0 - r + rx : plf_reflect101(x0 - r + rx, w)];
  }
  __syncthreads();
  const int ks = 2 * r + 1;
  const int tx = tid & (BQ_TW - 1), rg = tid >> 6;  // BQ_TW == 64
  for (int ry = rg; ry < RH; ry += 4) {
    uint32_t a = 0;
    for (int k = 0; k < ks; ++k) a += (uint32_t)c_lsd_taps[k] * raw[ry][tx + k];
    hrow[ry][tx] = (uint16_t)a;
  }
  __syncthreads();
  const int gx = x0 + tx;
  if (gx < w) {
    for (int ty = rg; ty < BQ_TH; ty += 4) {
      const int gy = y0 + ty;
      if (gy >= h) break;
      uint32_t a = 0;
      for (int k = 0; k < ks; ++k) a += (uint32_t)c_lsd_taps[k] * hrow[ty + k][tx];
      const uint32_t v = (a + (1u << 15)) >> 16;
      d[(size_t)gy * dpitch + gx] = (uint8_t)(v > 255 ? 255 : v);
    }
  }
}

// Fast path for KS <= 8 taps (7x7 at the reference's scale 1.2 / 0.8): 64x32 output tile staged by ONE TMA bulk-tensor
// copy (plf_tma.cuh; border CTAs rebuild BORDER_REFLECT_101 inside shared memory), DP4A row pass.
//   row pass : a thread produces 4 adjacent outputs of one row from three aligned 32-bit words of the staged tile;
//              the KS byte window of each output is assembled with PRMT (byte_perm) and reduced with two DP4As against
//              the packed u8 taps (taps <= 255, products summed exactly in 32 bits, result < 2^16);
//   col pass : a thread slides down 8 rows of one column with the KS taps in registers.
// ~30 thread-instructions per pixel instead of ~200 for the generic kernel; bit-identical results.
#define BF_TW 64
#define BF_TH 32
template <int KS>
__global__ void __launch_bounds__(256) k_blur_q8_fast(const __grid_constant__ CUtensorMap tmap, int z0, int w, int h,
                                                      uint32_t tapsA, uint32_t tapsB, uint8_t* __restrict__ dst,
                                                      size_t dst_stride, int dpitch) {
  constexpr int R = KS / 2;
  constexpr int RH = BF_TH + 2 * R;
  constexpr int RP = 80;     // TMA box width (bytes, multiple of 16)
  constexpr int NEED = 72;   // columns the row pass reads (64 outputs + 2R taps, whole 32-bit words)
  __shared__ __align__(128) uint8_t raw[RH][RP];
  __shared__ __align__(16) uint16_t hrow[RH][BF_TW];
  __shared__ __align__(8) uint64_t bar;
  uint8_t* d = dst + (size_t)blockIdx.z * dst_stride;
  const int x0 = blockIdx.x * BF_TW - (16 - R), y0 = blockIdx.y * BF_TH, tid = threadIdx.x;   // x0 - R on a 16-byte boundary (TMA)
  if (tid == 0) plf_mbar_init(&bar);
  __syncthreads();
  if (tid == 0) plf_tma_load_3d(&raw[0][0], &tmap, x0 - R, y0 - R, z0 + (int)blockIdx.z, &bar, RH * RP);
  plf_mbar_wait(&bar, 0);
  if (!(x0 >= R && x0 - R + NEED <= w && y0 >= R && y0 + BF_TH + R <= h))   // border tile: BORDER_REFLECT_101 in place
    plf_tma_reflect_fix<RH, RP>(raw, x0 - R, y0 - R, w, h, NEED);
  __syncthreads();
  for (int it = tid; it < RH * (BF_TW / 4); it += 256) {
    const int ry = it >> 4, j = it & 15;  // BF_TW / 4 == 16 groups per row
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(&raw[ry][4 * j]);
    const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = __byte_perm(w0, w1, 0x3210 + 0x1111 * i);
      const uint32_t hi = __byte_perm(w1, w2, 0x3210 + 0x1111 * i);
      o[i] = __dp4a(hi, tapsB, __dp4a(lo, tapsA, 0u));
    }
    uint2 pk = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
    *reinterpret_cast<uint2*>(&hrow[ry][4 * j]) = pk;
  }
  __syncthreads();
  const int c = tid & 63, q = tid >> 6;
  const int gx = x0 + c;
  if (gx >= 0 && gx < w) {
    uint32_t t[KS];
#pragma unroll
    for (int k = 0; k < KS; ++k) t[k] = k < 4 ? ((tapsA >> (8 * k)) & 0xFFu) : ((tapsB >> (8 * (k - 4))) & 0xFFu);
    uint32_t v[8 + KS - 1];
#pragma unroll
    for (int k = 0; k < 8 + KS - 1; ++k) v[k] = hrow[q * 8 + k][c];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int gy = y0 + q * 8 + r;
      if (gy < h) {
        uint32_t a = 0;
#pragma unroll
        for (int k = 0; k < KS; ++k) a += t[k] * v[r + k];
        const uint32_t o = (a + (1u << 15)) >> 16;
        d[(size_t)gy * dpitch + gx] = (uint8_t)(o > 255 ? 255 : o);
      }
    }
  }
}

// ---- gradient ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float lsd_fast_atan2(float y, float x) {  // cv::fastAtan2, see orb.cu
  const float p1 = 0.9997878412794807f * (float)(180 / 3.14159265358979323846);
  const float p3 = -0.3258083974640975f * (float)(180 / 3.14159265358979323846);
  const float p5 = 0.1555786518463281f * (float)(180 / 3.14159265358979323846);
  const float p7 = -0.04432655554792128f * (float)(180 / 3.14159265358979323846);
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, (float)2.2204460492503131e-16));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, (float)2.2204460492503131e-16));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

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
// lut_angle: the angle of a defined gradient (NOTDEF otherwise; k_lsd_grad only looks up defined ones);
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
    const float adeg = lsd_fast_atan2((float)gx, (float)(-gy));
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

// pix points at pixel (0,0) of image 0 (i.e. past the guard); image stride pix_stride.
// Only the DEFINED pixels (gradient norm above rho, ~12 %) leave the kernel: their 8-byte record (the map's other records
// already read "undefined", see k_lsd_fill_notdef) and one entry (column in the segment, gx^2 + gy^2) of the raster-ordered
// SEED LIST of their row segment - the LSD_SEG columns of this block; segment (y, xb) stores its entries at the segment's own
// pixel offset y * W + LSD_SEG * xb of the list array, so it can never overflow, and its length in segcnt.  Nothing dense is
// written: the seed ordering works on the lists, and the rectangle fit reads the gradient of a region point back from its
// record (li).
#define LSD_SEG 512
#define LSD_GRAD_THREADS (LSD_SEG / 4)
// list entry: the low LSD_COL_BITS hold the column inside the segment, the high bits gx^2 + gy^2 (<= 2 * 510^2 over the
// table's gradient range) and, after k_lsd_rowhist, the bin (< LSD_BINS_MAX)
#define LSD_COL_BITS 9
static_assert(LSD_SEG <= (1 << LSD_COL_BITS), "seed list: a segment column must fit the column field");
static_assert(2u * 510u * 510u < (1u << (32 - LSD_COL_BITS)), "seed list: gx^2 + gy^2 must fit above the column field");
static_assert(LSD_BINS_MAX <= (1 << (32 - LSD_COL_BITS)), "seed list: the bin must fit above the column field");
// A thread produces FOUR adjacent columns of two rows from three aligned 32-bit words of the (16-byte pitched) image - the
// fifth column of each row comes from the neighbour lane's word (lane 31 loads it) - so a warp issues 3 (+3) load instructions
// for 256 pixels instead of 6 for 64.
__global__ void __launch_bounds__(LSD_GRAD_THREADS) k_lsd_grad(const uint8_t* __restrict__ img, size_t img_stride, int IP, int W, int H,
                                                               const float* __restrict__ lut_angle, int m2_min, size_t stride,
                                                               LsdPix* __restrict__ pix, size_t pix_stride,
                                                               uint32_t* __restrict__ list, int* __restrict__ segcnt, int nxb,
                                                               int* __restrict__ maxmag2) {
  const int x4 = blockIdx.x * LSD_SEG + threadIdx.x * 4, y0 = blockIdx.y * 2, im = blockIdx.z;
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  // words of rows y0 .. y0+2 at columns x4 .. x4+3 (rows / words beyond the image read as 0: those pixels are never defined -
  // the last column and the last row of the map are excluded below)
  uint32_t w[3] = {0u, 0u, 0u}, wn[3] = {0u, 0u, 0u};
  const uint8_t* p = img + (size_t)im * img_stride + (size_t)y0 * IP + x4;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    if (x4 < W && y0 + r < H) w[r] = __ldg(reinterpret_cast<const uint32_t*>(p + (size_t)r * IP));   // IP is a multiple of 16, x4 of 4
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    wn[r] = __shfl_down_sync(0xFFFFFFFFu, w[r], 1);
    if (lane == 31) wn[r] = (x4 + 4 < IP && y0 + r < H) ? __ldg(reinterpret_cast<const uint32_t*>(p + (size_t)r * IP + 4)) : 0u;
  }
  int mag2 = -1;
  int li[2][4], m2v[2][4];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const bool rok = y0 + r < H - 1;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      li[r][c] = -1; m2v[r][c] = 0;
      // pixel (x, y) = (x4 + c, y0 + r): A = (x, y), B = (x+1, y), C = (x, y+1), D = (x+1, y+1)
      const int A = (w[r] >> (8 * c)) & 0xFF, C = (w[r + 1] >> (8 * c)) & 0xFF;
      const int B = c < 3 ? (int)((w[r] >> (8 * c + 8)) & 0xFF) : (int)(wn[r] & 0xFF);
      const int D = c < 3 ? (int)((w[r + 1] >> (8 * c + 8)) & 0xFF) : (int)(wn[r + 1] & 0xFF);
      if (rok && x4 + c < W - 1) {
        const int DA = D - A, BC = B - C, gx = DA + BC, gy = DA - BC, m2 = gx * gx + gy * gy;
        if (m2 >= m2_min) { li[r][c] = (gx + 510) * LSD_LUT_DIM + (gy + 510); m2v[r][c] = m2; mag2 = max(mag2, m2); }  // defined angle
      }
    }
  }
  // records of the defined pixels
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (li[r][c] >= 0)
        *reinterpret_cast<uint2*>(&pix[(size_t)im * pix_stride + (size_t)(y0 + r) * W + x4 + c]) =
            make_uint2(__float_as_uint(__ldg(&lut_angle[li[r][c]])), (uint32_t)li[r][c]);
  // ordered compaction of the two row segments (x ascending) + the per-image maximum: one barrier
  __shared__ int s_max[4], s_c[2][4];
  int cnt[2], incl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    cnt[r] = (li[r][0] >= 0) + (li[r][1] >= 0) + (li[r][2] >= 0) + (li[r][3] >= 0);
    incl[r] = cnt[r];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xFFFFFFFFu, incl[r], off);
      if (lane >= off) incl[r] += v;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mag2 = max(mag2, __shfl_xor_sync(0xFFFFFFFFu, mag2, off));
  if (lane == 31) { s_c[0][wrp] = incl[0]; s_c[1][wrp] = incl[1]; }
  if (lane == 0) s_max[wrp] = mag2;
  __syncthreads();
  const size_t lbase = (size_t)im * stride + (size_t)blockIdx.x * LSD_SEG;
  int tot[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    int woff = 0;
    tot[r] = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < wrp) woff += s_c[r][k];
      tot[r] += s_c[r][k];
    }
    size_t o = lbase + (size_t)(y0 + r) * W + woff + incl[r] - cnt[r];
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (li[r][c] >= 0) {
        list[o] = (uint32_t)(threadIdx.x * 4 + c) | ((uint32_t)m2v[r][c] << LSD_COL_BITS);
        ++o;
      }
  }
  if (threadIdx.x == 0) {
    int* sc = segcnt + (size_t)im * ((size_t)H * nxb);
    sc[(size_t)y0 * nxb + blockIdx.x] = tot[0];
    if (y0 + 1 < H) sc[(size_t)(y0 + 1) * nxb + blockIdx.x] = tot[1];
    const int m = max(max(s_max[0], s_max[1]), max(s_max[2], s_max[3]));
    if (m >= 0 && m > __ldcg(&maxmag2[im])) atomicMax(&maxmag2[im], m);   // only touch the (contended) address when it would grow
  }
}

// ---- pseudo-ordering (stable counting sort, bins descending) ---------------------------------------------------
__device__ __forceinline__ double lsd_bin_coef(int maxmag2, int n_bins) {
  if (maxmag2 < 0) return 0.0;
  const double max_grad = sqrt((double)maxmag2 / 4.0);
  return max_grad > 0 ? (double)(n_bins - 1) / max_grad : 0.0;
}

// The image is cut into chunks of LSD_CHUNK rows.  One CTA bins a chunk: its warps walk the chunk's row-segment lists (written
// by the gradient kernel: only the defined pixels, ~12 %), turn gx^2 + gy^2 into the bin of the 1024-bin pseudo-ordering
// (the per-image maximum is known by now), store the bin in its place and count the bins; one warp then scatters the
// chunk's lists in raster order.
#define LSD_CHUNK 16
__global__ void __launch_bounds__(256) k_lsd_rowhist(size_t stride, int W, int H, int n_bins, int nchunks, int nxb,
                                                     const int* __restrict__ maxmag2, uint32_t* __restrict__ list,
                                                     const int* __restrict__ segcnt, uint32_t* __restrict__ chunkcnt) {
  __shared__ uint32_t hist[LSD_BINS_MAX];
  const int ch = blockIdx.x, im = blockIdx.y, tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  for (int i = tid; i < n_bins; i += 256) hist[i] = 0;
  __syncthreads();
  const double coef = lsd_bin_coef(maxmag2[im], n_bins);
  const int ya = ch * LSD_CHUNK, y1 = min((ch + 1) * LSD_CHUNK, H - 1);
  const int nseg = (y1 - ya) * nxb;
  const int* sc = segcnt + (size_t)im * ((size_t)H * nxb);
  for (int sg = wrp; sg < nseg; sg += 8) {
    const int y = ya + sg / nxb, xb = sg - (sg / nxb) * nxb;
    const int n = sc[(size_t)y * nxb + xb];
    const size_t o = (size_t)im * stride + (size_t)y * W + (size_t)xb * LSD_SEG;
    for (int i = lane; i < n; i += 32) {
      const uint32_t e = list[o + i];
      const double norm = sqrt((double)(e >> LSD_COL_BITS) / 4.0);
      const int b = (int)(norm * coef);
      list[o + i] = (e & ((1u << LSD_COL_BITS) - 1u)) | ((uint32_t)b << LSD_COL_BITS);
      atomicAdd(&hist[b], 1u);
    }
  }
  __syncthreads();
  uint32_t* out = chunkcnt + ((size_t)im * nchunks + ch) * n_bins;
  for (int i = tid; i < n_bins; i += 256) out[i] = hist[i];
}

// one block (n_bins threads, <= 1024) per image: per-bin prefix over chunks, then start of each bin (bins descending).
// The chunk counts of a bin are loaded 8 at a time before their prefixes are stored back (the loads of a plain
// read-modify-write loop serialise behind the stores to the same array); the scan over the bins is two levels of warp shuffles.
__global__ void __launch_bounds__(1024) k_lsd_binscan(uint32_t* __restrict__ chunkcnt, int nchunks, int n_bins,
                                                      uint32_t* __restrict__ binstart, int* __restrict__ nseeds) {
  __shared__ uint32_t tot[LSD_BINS_MAX];
  __shared__ uint32_t wsum[32];
  const int im = blockIdx.x, b = threadIdx.x, lane = b & 31, wrp = b >> 5;
  uint32_t run = 0;
  if (b < n_bins) {
    uint32_t* c = chunkcnt + (size_t)im * nchunks * n_bins + b;
    for (int k0 = 0; k0 < nchunks; k0 += 8) {
      uint32_t v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = k0 + j < nchunks ? __ldcg(&c[(size_t)(k0 + j) * n_bins]) : 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (k0 + j < nchunks) {
          c[(size_t)(k0 + j) * n_bins] = run;
          run += v[j];
        }
    }
    tot[b] = run;
  }
  __syncthreads();
  // exclusive scan over bins in DESCENDING bin order: thread b holds reversed element b = bin (n_bins - 1 - b)
  const int rb = n_bins - 1 - b;
  const uint32_t mine = b < n_bins ? tot[rb] : 0u;
  uint32_t incl = mine;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) wsum[wrp] = incl;
  __syncthreads();
  if (wrp == 0) {
    uint32_t w = wsum[lane], wi = w;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, wi, off);
      if (lane >= off) wi += v;
    }
    wsum[lane] = wi - w;   // exclusive prefix of the warp totals
  }
  __syncthreads();
  const uint32_t excl = wsum[wrp] + incl - mine;
  if (b < n_bins) binstart[(size_t)im * n_bins + rb] = excl;
  if (b == n_bins - 1) nseeds[im] = (int)(excl + mine);
}

// one warp per (chunk, image): walks the chunk's row-segment lists in raster order, stable ranks via match_any
__global__ void __launch_bounds__(128) k_lsd_scatter(const uint32_t* __restrict__ list,
                                                     const int* __restrict__ segcnt, size_t stride, int W, int H, int n_bins,
                                                     int nchunks, int nxb, const uint32_t* __restrict__ chunkcnt,
                                                     const uint32_t* __restrict__ binstart, uint32_t* __restrict__ order) {
  __shared__ uint32_t cnt[4][LSD_BINS_MAX];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ch = blockIdx.x * 4 + wid, im = blockIdx.y;
  if (ch >= nchunks) return;
  uint32_t* c = cnt[wid];
  const uint32_t* rc = chunkcnt + ((size_t)im * nchunks + ch) * n_bins;
  const uint32_t* bs = binstart + (size_t)im * n_bins;
  for (int i = lane; i < n_bins; i += 32) c[i] = rc[i] + bs[i];
  __syncwarp();
  uint32_t* ord = order + (size_t)im * stride;
  const int ya = ch * LSD_CHUNK, y1 = min((ch + 1) * LSD_CHUNK, H - 1);
  const int nseg = (y1 - ya) * nxb;
  const int* sc = segcnt + (size_t)im * ((size_t)H * nxb) + (size_t)ya * nxb;   // the chunk's segments are contiguous, row-major
  int n_next = nseg > 0 ? sc[0] : 0;
  for (int sg = 0; sg < nseg; ++sg) {
    const int n = n_next;
    n_next = sg + 1 < nseg ? sc[sg + 1] : 0;
    const int y = ya + sg / nxb, xb = sg - (sg / nxb) * nxb;
    const uint32_t seg0 = (uint32_t)(y * W + xb * LSD_SEG);   // pixel index of the segment's first column
    const size_t o = (size_t)im * stride + seg0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const bool valid = i < n;
      const uint32_t e = valid ? list[o + i] : 0u;
      const uint32_t idx = seg0 + (e & ((1u << LSD_COL_BITS) - 1u));
      const int b = valid ? (int)(e >> LSD_COL_BITS) : -1;
      const unsigned vm = __ballot_sync(0xFFFFFFFFu, valid);
      if (valid) {
        const unsigned peers = __match_any_sync(vm, b);
        const int rank = __popc(peers & ((1u << lane) - 1));
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == leader) {
          base = c[b];
          c[b] = base + __popc(peers);
        }
        base = __shfl_sync(peers, base, leader);
        ord[base + rank] = idx;
      }
      __syncwarp();
    }
  }
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
// Per region point: lanes 0..8 hold the 8-byte records of the 3x3 neighbourhood, fetched two queue entries AHEAD; cells
// accepted meanwhile are patched to "used" in the prefetched registers.  The neighbours are decided lane-parallel and
// re-decided after every acceptance, which reproduces the reference's sequential semantics (each test sees the region
// angle left by the previous acceptance).
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
  const int kk = lane < 9 ? lane : 4;                  // neighbour slot served by this lane (lanes >= 9 idle on the centre)
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
      // neighbourhood records of queue entries r+1 (pf1) and r+2 (pf2), fetched while earlier entries are processed;
      // a cell accepted meanwhile is patched to "used" in both prefetched copies (i < pmin: nothing fetched)
      LsdRec pf1, pf2;
      pf1.a = pf2.a = LSD_NOTDEF_F; pf1.li = pf2.li = 0u;
      int i1 = pmin - 1, i2 = pmin - 1;
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
      for (uint32_t r = 0; r < nreg; ++r) {
        LsdRec cur;
        int ci;
        if (i1 >= pmin) {
          cur = pf1;
          ci = i1;
        } else {
          uint32_t pt;
          if (nreg - r <= LSD_QCAP) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(pt) : "r"(qs + ((r & (LSD_QCAP - 1)) << 2)) : "memory");
          else pt = __ldcg(&regpts[cursor + r]);
          ci = (int)pt + noff;
          asm volatile("" : "+r"(ci));  // keep the index 32-bit: one IMAD.WIDE forms the address
          cur = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)ci * LSD_REC_BYTES));
        }
        pf1 = pf2; i1 = i2;
        i2 = pmin - 1;
        if (i1 < pmin && r + 1 < nreg) {
          uint32_t pt;
          if (nreg - (r + 1) <= LSD_QCAP) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(pt) : "r"(qs + (((r + 1) & (LSD_QCAP - 1)) << 2)) : "memory");
          else pt = __ldcg(&regpts[cursor + r + 1]);
          i1 = (int)pt + noff;
          asm volatile("" : "+r"(i1));
          pf1 = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)i1 * LSD_REC_BYTES));
        }
        if (r + 2 < nreg) {
          uint32_t pt;
          if (nreg - (r + 2) <= LSD_QCAP) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(pt) : "r"(qs + (((r + 2) & (LSD_QCAP - 1)) << 2)) : "memory");
          else pt = __ldcg(&regpts[cursor + r + 2]);
          i2 = (int)pt + noff;
          asm volatile("" : "+r"(i2));
          pf2 = lsd_load_pix(reinterpret_cast<const LsdPix*>(pb + (long long)i2 * LSD_REC_BYTES));
        }
        unsigned rem = __ballot_sync(0xFFFFFFFFu, lane < 9 && cur.a != LSD_NOTDEF_F);
        while (rem) {
          float d = fabsf(__fsub_rn(cur.a, th));
          if (d > 180.f) d = __fsub_rn(360.f, d);
          const bool mine = (rem >> lane) & 1u;
          const unsigned mm = __ballot_sync(0xFFFFFFFFu, mine && d <= hi);  // aligned or undecided
          if (!mm) break;                                                    // everything left is clearly not aligned
          const int k = __ffs(mm) - 1;
          const unsigned mi = __ballot_sync(0xFFFFFFFFu, mine && d < lo);   // certainly aligned
          if (!((mi >> k) & 1u)) {  // the first candidate sits in the band
            if (!fresh) {
              add_staged();
              th = lsd_fast_atan2(sumdy, sumdx);
              inv0 = __fmul_rn(rsqrtf(__fadd_rn(__fmul_rn(sumdx, sumdx), __fmul_rn(sumdy, sumdy))), 1.02f);
              margin = margin0;
              lo = prec_deg - margin; hi = prec_deg + margin;
              fresh = true;
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
          rem &= ~((2u << k) - 1u);  // k and everything before it have been decided
          const int ai = __shfl_sync(0xFFFFFFFFu, ci, k);
          const float dk = __shfl_sync(0xFFFFFFFFu, d, k);
          // lane 0 marks the cell used and appends it to the region / the queue (predicated: no divergent branch)
          asm volatile(
              "{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %0, 0;\n\t"
              "@p st.global.f32 [%1], %2;\n\t@p st.global.u32 [%3], %4;\n\t@p st.shared.u32 [%5], %4;\n\t}"
              ::"r"(l0), "l"(pb + (long long)ai * LSD_REC_BYTES), "f"(LSD_NOTDEF_F), "l"(regpts + (cursor + nreg)), "r"(ai),
                "r"(qs + ((nreg & (LSD_QCAP - 1)) << 2))
              : "memory");
          ++nreg;
          lsd_prefetch(pb + (long long)(ai + poff) * LSD_REC_BYTES);
          if (i1 == ai) pf1.a = LSD_NOTDEF_F;  // prefetched copies of this cell are stale
          if (i2 == ai) pf2.a = LSD_NOTDEF_F;
          // stage the member's term: lane k holds its record (landed: its angle was just tested)
          if (qpos - qwait == LSD_CSQ) add_staged();   // ring full: its oldest slot is about to be reused
          if (lane == k)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(csb + ((qpos & (LSD_CSQ - 1)) << 3)),
                         "l"(lut_cs + cur.li) : "memory");
          ++qpos;
          margin = __fmaf_rn(fminf(__fadd_rn(dk, margin), dmax), inv0, margin);
          lo = prec_deg - margin; hi = prec_deg + margin;
          fresh = false;
        }
        __syncwarp();
      }
      if ((int)nreg >= min_reg_size) {
        if (nreg_out < max_regions) {
          if (!fresh) add_staged();   // the members accepted since S was last read (fresh: none)
          if (lane == 0) {
            // region angle handed to the rectangle fit: the seed's own angle for a 1-pixel region, else the angle of the sum
            const double reg_angle = nreg == 1 ? th_seed : (double)(fresh ? th : lsd_fast_atan2(sumdy, sumdx)) * LSD_DEG2RAD;
            const unsigned long long bits = (unsigned long long)__double_as_longlong(reg_angle);
            regions[nreg_out] = make_uint4(cursor, nreg, (uint32_t)bits, (uint32_t)(bits >> 32));
          }
          ++nreg_out;
          cursor += nreg;
        } else if (lane == 0) {
          *overflow = 1;
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
  double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)lsd_fast_atan2((float)(lambda - Ixx), (float)Ixy)
                                         : (double)lsd_fast_atan2((float)Ixy, (float)(lambda - Iyy));
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
#define KL_SORT_CAP 4096
__global__ void __launch_bounds__(1024) k_keylines(const float4* __restrict__ segs_all, const int* __restrict__ nsegs,
                                                   int max_regions, int w, int h, double min_length, int nfeatures,
                                                   plf_keyline* __restrict__ kls_all, plf_keyline* __restrict__ kls_out,
                                                   int max_lines, int* __restrict__ nlines, int* __restrict__ overflow) {
  __shared__ unsigned long long keys[KL_SORT_CAP];  // (response desc, index asc) for the top-K
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int im = blockIdx.x, tid = threadIdx.x;
  const int n = min(nsegs[im], max_regions);
  const float4* segs = segs_all + (size_t)im * max_regions;
  plf_keyline* all = kls_all + (size_t)im * max_regions;
  plf_keyline* out = kls_out + (size_t)im * max_lines;
  // pass 1: accept flags + ordered compaction (class_id = running counter of accepted lines, :299)
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    bool ok = false;
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
    // block exclusive scan of ok flags
    s_scan[tid] = ok ? 1 : 0;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      const int v = tid >= off ? s_scan[tid - off] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    const int incl = s_scan[tid];
    if (tid == 1023) s_total = incl;
    if (ok) {
      kl.class_id = base + incl - 1;
      all[base + incl - 1] = kl;
    }
    __syncthreads();
    base += s_total;
    __syncthreads();
  }
  const int m = base;
  int keep = m;
  if (nfeatures != 0 && m > nfeatures) {
    // stvo-pl: sort by response (descending), keep nfeatures, class_id = rank.  Ties: detection order.
    if (m > KL_SORT_CAP) {
      if (tid == 0) *overflow = 1;
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
      if (tid == 0) *overflow = 1;
      keep = max_lines;
    }
    for (int i = tid; i < keep; i += 1024) {
      plf_keyline kl = all[(uint32_t)(keys[i] & 0xFFFFFFFFu)];
      kl.class_id = i;
      out[i] = kl;
    }
  } else {
    if (keep > max_lines) {
      if (tid == 0) *overflow = 1;
      keep = max_lines;
    }
    for (int i = tid; i < keep; i += 1024) out[i] = all[i];
  }
  if (tid == 0) nlines[im] = keep;
}

// ---- host side -------------------------------------------------------------------------------------------------
extern "C" void plf_lsd_free(plf_ctx* ctx) {
  if (ctx->lsd) {
    ctx->lsd->bufs.release();
    delete ctx->lsd;
    ctx->lsd = nullptr;
  }
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
  const size_t N = (size_t)s->nimg, As = (size_t)s->ws * s->hs, R = (size_t)s->max_regions, LUT = (size_t)LSD_LUT_DIM * LSD_LUT_DIM;
  s->bp = plf_pitch16(s->w); s->sp = plf_pitch16(s->ws);
  s->nxb = (s->ws + LSD_SEG - 1) / LSD_SEG;
  s->pix_stride = As + (size_t)s->ws + 1;
  b.add(s->blur, (size_t)s->bp * s->h * N);
  b.add(s->scaled, (size_t)s->sp * s->hs * N);
  b.add(s->seedlist, As * N);
  b.add(s->segcnt, N * s->hs * s->nxb);
  b.add(s->rect_perm, N * R);
  b.add(s->maxmag2, N);
  b.add(s->rowcnt, N * ((s->hs + LSD_CHUNK - 1) / LSD_CHUNK) * s->n_bins);
  b.add(s->binstart, N * s->n_bins);
  b.add(s->regpts, As * N);
  b.add(s->regions, N * R);
  b.add(s->nregions, N);
  b.add(s->segs, N * R);
  b.add(s->kls_all, N * R);
  // buffers that cross from the pre-grow phase to the growing (or to the match phase) exist twice (parity of the batch),
  // so that batch i+1 can be extracted while batch i is still growing regions; standalone operators use parity 0 only
  for (int p = 0; p < (s->two_parities ? 2 : 1); ++p) {
    b.add(s->pix_raw[p], lsd_pix_records(s));
    b.add(s->nseeds[p], N);
    b.add(s->order[p], As * N);
    b.add(s->kls[p], N * s->max_lines);
    b.add(s->nlines[p], N);
  }
  b.add(s->overflow, 1);
  b.add(s->angle_lut, LUT);
  b.add(s->cs_lut, LUT);
  b.add(s->seed_lut, LUT);
  if (s->scale != 1.0) {
    s->rs_x_off = 0;
    s->rs_y_off = 2 * (size_t)s->ws;
    s->rs_xp_off = (s->rs_y_off + 2 * (size_t)s->hs + 3) & ~(size_t)3;   // 16-byte aligned: read with 128-bit loads
    b.add(s->rs_tab, s->rs_xp_off + plf_resize_packed_len(s->ws));
  }
}

size_t plf_lsd_footprint(const plf_ctx* ctx, int w, int h, int nimg, bool two_parities) {
  LsdState z;
  lsd_set_sizes(ctx, &z, w, h, nimg, two_parities);
  DevBufList b;
  lsd_buffers(&z, b);
  return b.bytes();
}

static plf_status lsd_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities) {
  LsdState* s = ctx->lsd;
  if (s && s->w == w && s->h == h && s->nimg >= nimg && (s->two_parities || !two_parities)) return PLF_OK;
  if (s && s->two_parities) two_parities = true;
  if (s) {
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s->bufs.release();
    *s = LsdState();
  } else {
    s = ctx->lsd = new LsdState();
  }
  const plf_params& P = ctx->params;
  if (P.lsd_refine != 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: only lsd_refine = 0 (LSD_REFINE_NONE, the reference configs) is supported");
  if (P.lsd_n_bins < 1 || P.lsd_n_bins > LSD_BINS_MAX)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: lsd_n_bins must be in [1,%d]", LSD_BINS_MAX);
  lsd_set_sizes(ctx, s, w, h, nimg, two_parities);
  s->prec = LSD_PI * P.lsd_ang_th / 180;
  s->p = P.lsd_ang_th / 180;
  s->rho = P.lsd_quant / sin(s->prec);
  if (s->scale != 1.0) {
    const double sigma = (s->scale < 1) ? (P.lsd_sigma_scale / s->scale) : P.lsd_sigma_scale;
    const unsigned hk = (unsigned)(ceil(sigma * sqrt(2 * 3.0 * log(10.0))));
    s->ksize = 1 + 2 * (int)hk;
    if (s->ksize > 15) return plf_fail(ctx, PLF_ERR_INVALID, "LSD: Gaussian kernel %d > 15 unsupported", s->ksize);
    gaussian_taps_q8(s->ksize, sigma, s->taps);
    s->taps_u8 = true;
    for (int k = 0; k < s->ksize; ++k) s->taps_u8 = s->taps_u8 && s->taps[k] <= 255;
  } else {
    s->ksize = 0;
  }
  if (s->ws >= 65536 || s->hs >= 65536 || s->ws < 3 || s->hs < 3)
    return plf_fail(ctx, PLF_ERR_INVALID, "LSD: scaled image %dx%d out of range", s->ws, s->hs);
  const double LOG_NT = 5 * (log10((double)s->ws) + log10((double)s->hs)) / 2 + log10(11.0);
  s->min_reg_size = (int)(size_t)(-LOG_NT / log10(s->p));
  for (s->m2_min = 0; s->m2_min <= 2 * 510 * 510; ++s->m2_min)  // same double expression as the kernels
    if (!(sqrt((double)s->m2_min / 4.0) <= s->rho)) break;
  lsd_buffers(s, s->bufs);
  plf_status st = s->bufs.alloc(ctx, "LSD");
  if (st) return st;
  for (int p = 0; p < (s->two_parities ? 2 : 1); ++p) {
    s->pix[p] = s->pix_raw[p] + lsd_pix_pad(s);
    k_lsd_fill_notdef<<<(unsigned)((lsd_pix_records(s) + 255) / 256), 256, 0, ctx->stream>>>(s->pix_raw[p], lsd_pix_records(s));
    PLF_LAUNCH_CHECK(ctx);
  }
  PLF_CUDA(ctx, cudaMemsetAsync(s->overflow, 0, sizeof(int), ctx->stream));
  k_lsd_build_lut<<<(LSD_LUT_DIM * LSD_LUT_DIM + 255) / 256, 256, 0, ctx->stream>>>(s->rho, s->angle_lut, s->cs_lut, s->seed_lut);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (s->scale != 1.0) {
    PLF_CUDA(ctx, cudaMemcpyToSymbolAsync(c_lsd_taps, s->taps, sizeof(int) * 16, 0, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<int> tab(s->rs_xp_off + plf_resize_packed_len(s->ws));
    plf_linear_coeffs_host(w, s->ws, 1.0 / s->scale, &tab[0], &tab[s->ws]);
    plf_linear_coeffs_host(h, s->hs, 1.0 / s->scale, &tab[s->rs_y_off], &tab[s->rs_y_off + s->hs]);
    plf_resize_pack_x(&tab[0], &tab[s->ws], s->ws, &tab[s->rs_xp_off]);
    PLF_CUDA(ctx, cudaMemcpyAsync(s->rs_tab, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
}

// A failed (re)build leaves no state behind (see plf_orb_prepare).
plf_status plf_lsd_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities) {
  const plf_status st = lsd_prepare(ctx, w, h, nimg, two_parities);
  if (st && ctx->lsd) {
    ctx->lsd->bufs.release();
    *ctx->lsd = LsdState();
  }
  return st;
}

// LSD on images [0, n) of a batch resident on the device, in two phases so that callers can overlap them with other
// work: `pre` = blur, resample, gradient and seed ordering (bandwidth-bound), `grow` = region growing, rectangle fit and
// the KeyLine stage (latency-bound).  `par` selects the buffer set that carries data from pre to grow.  State must be
// prepared for >= n images.  Enqueued on ctx->cur; results stay on the device.
plf_status plf_lsd_pre(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int par, int n) {
  LsdState* s = ctx->lsd;
  if (!s || s->w != w || s->h != h || s->nimg < n || (par && !s->two_parities))
    return plf_fail(ctx, PLF_ERR_STATE, "plf_lsd_pre: state not prepared for these images");
  cudaStream_t cs = ctx->cur;
  const int W = s->ws, H = s->hs;
  const size_t As = (size_t)W * H, A = (size_t)s->bp * h, Asp = (size_t)s->sp * H;
  LsdPix* pix = s->pix[par] + (s->ws + 1);  // pixel (0,0) of the first image
  const int nchunks = (H - 1 + LSD_CHUNK - 1) / LSD_CHUNK;
  plf_status st;
  const uint8_t* scaled = d_imgs;
  size_t scaled_stride = img_stride;
  int scaled_pitch = pitch;
  if (s->scale != 1.0) {
    if ((s->ksize == 7 || s->ksize == 5) && s->taps_u8) {
      const CUtensorMap* tm = s->tm_blur.get(d_imgs, w, h, n, pitch, img_stride, 80, BF_TH + s->ksize - 1);
      if (!tm)
        return plf_fail(ctx, PLF_ERR_CUDA, "LSD: cuTensorMapEncodeTiled failed for the source images (pitch %d, stride %zu)", pitch, img_stride);
      uint32_t tA = 0, tB = 0;
      for (int k = 0; k < s->ksize; ++k) (k < 4 ? tA : tB) |= (uint32_t)s->taps[k] << (8 * (k & 3));
      dim3 gf(plf_tma_tiles_x(w, s->ksize / 2), (h + BF_TH - 1) / BF_TH, n);
      if (s->ksize == 7) k_blur_q8_fast<7><<<gf, 256, 0, cs>>>(*tm, 0, w, h, tA, tB, s->blur, A, s->bp);
      else k_blur_q8_fast<5><<<gf, 256, 0, cs>>>(*tm, 0, w, h, tA, tB, s->blur, A, s->bp);
    } else {
      dim3 gb((w + BQ_TW - 1) / BQ_TW, (h + BQ_TH - 1) / BQ_TH, n);
      k_blur_q8<<<gb, 256, 0, cs>>>(d_imgs, img_stride, pitch, w, h, s->ksize / 2, s->blur, A, s->bp);
    }
    PLF_LAUNCH_CHECK(ctx);
    plf_mark(ctx, "lsd.k_blur_q8");
    st = plf_launch_resize_exact(ctx, s->blur, A, s->bp, w, h, s->scaled, Asp, s->sp, W, H, s->rs_tab + s->rs_x_off, s->rs_tab + s->rs_xp_off, s->rs_tab + s->rs_y_off, n);
    if (st) return st;
    plf_mark(ctx, "lsd.k_resize_exact");
    scaled = s->scaled;
    scaled_stride = Asp;
    scaled_pitch = s->sp;
  }
  PLF_CUDA(ctx, cudaMemsetAsync(s->maxmag2, 0xFF, (size_t)n * sizeof(int), cs));  // -1
  k_lsd_grad<<<dim3(s->nxb, (H + 1) / 2, n), LSD_GRAD_THREADS, 0, cs>>>(scaled, scaled_stride, scaled_pitch, W, H, s->angle_lut, s->m2_min, As, pix, s->pix_stride,
                                                               s->seedlist, s->segcnt, s->nxb, s->maxmag2);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_grad");
  k_lsd_rowhist<<<dim3(nchunks, n), 256, 0, cs>>>(As, W, H, s->n_bins, nchunks, s->nxb, s->maxmag2, s->seedlist, s->segcnt, s->rowcnt);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_rowhist");
  k_lsd_binscan<<<n, 1024, 0, cs>>>(s->rowcnt, nchunks, s->n_bins, s->binstart, s->nseeds[par]);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_binscan");
  k_lsd_scatter<<<dim3((nchunks + 3) / 4, n), 128, 0, cs>>>(s->seedlist, s->segcnt, As, W, H, s->n_bins, nchunks, s->nxb, s->rowcnt, s->binstart,
                                                            s->order[par]);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_scatter");
  return PLF_OK;
}

plf_status plf_lsd_grow(plf_ctx* ctx, int w, int h, int par, int n) {
  LsdState* s = ctx->lsd;
  if (!s || s->w != w || s->h != h || s->nimg < n || (par && !s->two_parities))
    return plf_fail(ctx, PLF_ERR_STATE, "plf_lsd_grow: state not prepared for these images");
  cudaStream_t cs = ctx->cur;
  const int W = s->ws, H = s->hs;
  const size_t As = (size_t)W * H;
  LsdPix* pix = s->pix[par] + (s->ws + 1);
  // one copy of regpts, regions, segs, kls_all: the growing, rectangle and KeyLine kernels of a batch run in stream order
  // before those of the next
  // (thread / lane per image, register-capped and unrolled variants and an angle-map layout were all bit-exact and were
  // not kept; DESIGN.md section 5 lists them)
  k_lsd_grow<<<n, 32, 0, cs>>>(pix, s->pix_stride, As, W, s->order[par], s->seed_lut, s->cs_lut, s->nseeds[par], s->prec, (float)(s->p * 180.0),
                               s->min_reg_size, s->regpts, s->regions, s->max_regions, s->nregions, s->overflow);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_grow");
  k_lsd_rect_order<<<n, 256, 0, cs>>>(s->regions, s->max_regions, s->nregions, s->rect_perm);
  PLF_LAUNCH_CHECK(ctx);
  k_lsd_rects<<<dim3((s->max_regions + 127) / 128, n), 128, 0, cs>>>(pix, s->pix_stride, As, W, s->regpts, s->regions, s->max_regions, s->nregions,
                                                                     s->rect_perm, s->prec, s->scale, s->segs);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_lsd_rects");
  const double min_length = (double)ctx->params.min_line_length * (double)std::min(w, h);
  if (ctx->lsd_keylines_wait) PLF_CUDA(ctx, cudaStreamWaitEvent(cs, ctx->lsd_keylines_wait, 0));
  k_keylines<<<n, 1024, 0, cs>>>(s->segs, s->nregions, s->max_regions, w, h, min_length, ctx->params.lsd_nfeatures, s->kls_all, s->kls[par],
                                 s->max_lines, s->nlines[par], s->overflow);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "lsd.k_keylines");
  return PLF_OK;
}

plf_status plf_lsd_run(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int nimg) {
  plf_status st = plf_lsd_prepare(ctx, w, h, nimg, false);
  if (st) return st;
  if ((st = plf_lsd_pre(ctx, d_imgs, img_stride, pitch, w, h, 0, nimg))) return st;
  return plf_lsd_grow(ctx, w, h, 0, nimg);
}

int* plf_lsd_overflow_flag(plf_ctx* ctx) { return ctx->lsd->overflow; }

void plf_lsd_outputs(plf_ctx* ctx, int par, plf_keyline** kls, int** nlines, int* max_lines) {
  LsdState* s = ctx->lsd;
  *kls = s->kls[par]; *nlines = s->nlines[par]; *max_lines = s->max_lines;
}

static plf_status lsd_check_overflow(plf_ctx* ctx, const char* what) {
  LsdState* s = ctx->lsd;
  int ovf = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&ovf, s->overflow, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ovf) {
    cudaMemsetAsync(s->overflow, 0, sizeof(int), ctx->stream);
    return plf_fail(ctx, PLF_ERR_CAPACITY, "%s: segment/line capacity exceeded (max_segments=%d, max_lines=%d)", what,
                    s->max_regions, s->max_lines);
  }
  return PLF_OK;
}

extern "C" plf_status plf_lsd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, float* segs, int cap,
                              int* n_out) {
  if (!ctx || !img || !n_out || w < 3 || h < 3 || stride < w || cap < 0 || (cap > 0 && !segs))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_lsd: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  uint8_t* dimg = (uint8_t*)plf_scratch(ctx, 4, (size_t)pitch * h);
  if (!dimg) return PLF_ERR_CUDA;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_lsd_run(ctx, dimg, (size_t)pitch * h, pitch, w, h, 1);
  if (st) return st;
  LsdState* s = ctx->lsd;
  int n = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&n, s->nregions, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  st = lsd_check_overflow(ctx, "plf_lsd");
  if (st) return st;
  *n_out = n;
  if (n > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_lsd: %d segments > caller capacity %d", n, cap);
  if (n > 0) {
    PLF_CUDA(ctx, cudaMemcpyAsync(segs, s->segs,(size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
}

extern "C" plf_status plf_detect_lines(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                                       plf_keyline* keylines, uint8_t* desc, int cap, int* n_out) {
  if (!ctx || !img || !n_out || w < 3 || h < 3 || stride < w || cap < 0 || (cap > 0 && (!keylines || !desc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_detect_lines: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  const size_t A = ((size_t)pitch * h + 255) & ~size_t(255);
  uint8_t* base = (uint8_t*)plf_scratch(ctx, 4, A + A * 4 + (size_t)ctx->limits.max_lines * 32 + 256);
  if (!base) return PLF_ERR_CUDA;
  uint8_t* dimg = base;
  short2* dgrad = (short2*)(base + A);
  uint8_t* ddesc = base + A + A * 4;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_lsd_run(ctx, dimg, (size_t)pitch * h, pitch, w, h, 1);
  if (st) return st;
  LsdState* s = ctx->lsd;
  st = plf_launch_blur5_sobel(ctx, dimg, pitch, (size_t)pitch * h, w, h, 1, dgrad, 0);
  if (st) return st;
  st = plf_launch_lbd(ctx, dgrad, 0, w, h, 1, s->kls[0], s->nlines[0], s->max_lines, ddesc, nullptr);
  if (st) return st;
  int n = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&n, s->nlines[0], sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  st = lsd_check_overflow(ctx, "plf_detect_lines");
  if (st) return st;
  *n_out = n;
  if (n > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_detect_lines: %d lines > caller capacity %d", n, cap);
  if (n > 0) {
    PLF_CUDA(ctx, cudaMemcpyAsync(keylines, s->kls[0], (size_t)n * sizeof(plf_keyline), cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaMemcpyAsync(desc, ddesc, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
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
  float* d = (float*)plf_scratch(ctx, 4, (size_t)n * 12);
  if (!d) return PLF_ERR_CUDA;
  PLF_CUDA(ctx, cudaMemcpyAsync(d, in, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  k_sincosf_probe<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d, d + n, d + 2 * (size_t)n, n);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(s, d + n, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(c, d + 2 * (size_t)n, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// The region-growing kernel stays resident for tens of milliseconds while the next batch's extraction kernels are
// co-scheduled on the same SMs.  The L1 / shared-memory split of an SM can only change while it is empty, so the split
// this kernel is launched with is the one those kernels have to live with: ask for a large shared-memory carve-out
// (164 KB) so that their CTAs (up to 17 KB of shared memory each) still fit at full occupancy.  Measured: k_orb_blur7 of
// the overlapped batch 28 ms -> 7 ms, step 83.3 -> 81.9 ms.
void plf_configure_lsd() {
  cudaFuncSetAttribute((const void*)k_lsd_grow, cudaFuncAttributePreferredSharedMemoryCarveout, 72);
}
