// ORB keypoints + rBRIEF-256 descriptors, batched over images (SURVEY §8 a1).
//
// Replaces stvo-pl StereoFrame::detectPointFeatures -> cv::ORB::create(nfeatures, scaleFactor, nlevels, edgeTh, 0,
// wtaK=2, FAST_SCORE, patchSize, fastTh)->detectAndCompute (parameters config/config/config_euroc.yaml:59-67; rows
// consumed as pdesc_l at src/mapHandler.cpp:86-88,302).  OpenCV is not vendored by the reference; the arithmetic
// mirrored here is OpenCV's published ORB (features2d orb.cpp / fast.cpp / fast_score.cpp, imgproc resize
// INTER_LINEAR_EXACT and the float sepFilter2D Gaussian), pinned integer-for-integer against cv2 4.13 by oracle/orb.c.
//
// Kernels (all gridded [tile or feature, image]; one launch covers every image of the batch)
//   k_resize_exact4  pyramid level l from level l-1: Q8.8 x Q8.8 bilinear, one rounding (bit-exact INTER_LINEAR_EXACT),
//                    four outputs per thread from two unaligned 32-bit reads per source row (k_resize_exact: scalar
//                    variant for scale factors above 1.9)
//   k_fast_nms       FAST-9/16 corner score + 3x3 non-max suppression + border filter on a 62x30 tile staged in
//                    shared memory by one TMA box (halo 4): 4-pair rejection, survivors compacted, full ring + score
//                    on dense warps; corners are appended to a per-(image,level) candidate list and a 256-bin
//                    response histogram
//   k_select_sort    KeyPointsFilter::retainBest: per-level response threshold from the histogram (n-th largest,
//                    ties kept), compaction, in-shared-memory bitonic sort to the canonical (octave, y, x) order
//   k_ic_angle       intensity-centroid orientation: integer moments over the 31-px circular patch, one warp per
//                    keypoint, cv::fastAtan2 polynomial
//   k_orb_blur7_fast 7x7 sigma-2 Gaussian in float with FMA (OpenCV takes its sepFilter2D path for the pyramid ROI), 64x32
//                    outputs per CTA, 4 per thread
//   k_orb_trig       (float) cos / sin of each keypoint angle, one thread per keypoint
//   k_rbrief         256 rotated pair tests from a 37x37 shared-memory patch, one warp per keypoint (lane = byte)
// Per-image algorithmic bytes are A0 + 2*sum(A_k>=1) + 2*S + 56*N (SURVEY §8d); what bounds each kernel (issue rate,
// latency - none is HBM-bound) is discussed in DESIGN.md §4.
#include "orb_pattern.h"
#include "plf_internal.h"
#include "plf_tma.cuh"

#define ORB_MAX_LEVELS 8
#define ORB_MIN_EDGE 19   // smallest orb_edge_th: keypoint to level border >= the 18-pixel reach of the 37 x 37 window
#define ORB_TW 64
#define ORB_TH 16
#define ORB_SORT_CAP 4096

struct OrbGeom {
  int nlevels;
  int w[ORB_MAX_LEVELS], h[ORB_MAX_LEVELS];
  int pitch[ORB_MAX_LEVELS];        // row pitch (bytes, multiple of 16) of level l; level 0 = the caller's image pitch
  int bpitch[ORB_MAX_LEVELS];       // row pitch of the blurred level l
  float scale[ORB_MAX_LEVELS];
  int nfeat[ORB_MAX_LEVELS];
  int umax[20];
  size_t pyr_off[ORB_MAX_LEVELS];   // byte offset of level l (l>=1) inside one image's pyramid block
  size_t pyr_stride;                // bytes of levels 1.. per image
  size_t blur_off[ORB_MAX_LEVELS];  // blurred levels 0..
  size_t blur_stride;
  int cand_cap[ORB_MAX_LEVELS];
  size_t cand_off[ORB_MAX_LEVELS];  // in entries
  size_t cand_stride;
  int tile_start[ORB_MAX_LEVELS + 1];  // FAST tiles: prefix over levels
  int tiles_x[ORB_MAX_LEVELS];
  int edge, fast_th, patch, half_patch;
  int max_kp;
};

struct OrbState {
  int w = 0, h = 0, nimg = 0;
  bool two_parities = false;
  OrbGeom g;
  uint8_t* pyr = nullptr;    // levels 1..n-1, all images
  uint8_t* blur = nullptr;   // blurred levels 0..n-1
  uint32_t* cand = nullptr;  // candidate keys
  int* cand_count = nullptr; // [nimg][levels]
  int* hist = nullptr;       // [nimg][levels][256]
  // resize tables per level l>=1: x: ofs (int), c1 (int); y likewise
  int* rs_tab = nullptr;
  size_t rs_x_off[ORB_MAX_LEVELS], rs_y_off[ORB_MAX_LEVELS], rs_xp_off[ORB_MAX_LEVELS];
  // outputs
  plf_keypoint* kps[2] = {nullptr, nullptr};  // [nimg][max_kp]
  short2* kp_lxy[2] = {nullptr, nullptr};     // level coordinates
  uint8_t* desc[2] = {nullptr, nullptr};      // [nimg][max_kp][32]
  int* kp_count[2] = {nullptr, nullptr};      // [nimg]
  int* overflow = nullptr;      // [1]
  float2* trig = nullptr;       // [nimg][max_kp] (cos, sin) of the keypoint angle (k_orb_trig -> k_rbrief)
  float blur_k[7];
  // TMA descriptors (plf_tma.cuh): halo boxes of the FAST tile (96 x 38) and of the blur tile (80 x 38) per level; level 0
  // is the caller's image buffer
  CUtensorMap tm_fast[ORB_MAX_LEVELS], tm_blur[ORB_MAX_LEVELS];
  PlfTmaCache tm_fast0, tm_blur0;
  DevBufList bufs;
};

__constant__ float c_blur7[7];

// ---- pyramid ---------------------------------------------------------------------------------------
// tab layout per level: [ox(dw) | cx(dw) | oy(dh) | cy(dh) | packed x (k_resize_exact4)]
__global__ void __launch_bounds__(256) k_resize_exact(const uint8_t* __restrict__ src, size_t src_stride, int sp, int sw,
                                                      int sh, uint8_t* __restrict__ dst, size_t dst_stride, int dp, int dw,
                                                      int dh, const int* __restrict__ tabx,
                                                      const int* __restrict__ taby) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= dw) return;
  const uint8_t* s = src + (size_t)blockIdx.z * src_stride;
  const int ox = tabx[x], cx = tabx[dw + x], oy = taby[y], cy = taby[dh + y];
  const uint8_t* r0 = s + (size_t)oy * sp + ox;
  const uint8_t* r1 = r0 + sp;
  const uint32_t h0 = r0[0] * (256 - cx) + r0[1] * cx;
  const uint32_t h1 = r1[0] * (256 - cx) + r1[1] * cx;
  const uint32_t v = (h0 * (256 - cy) + h1 * cy + 32768u) >> 16;
  dst[(size_t)blockIdx.z * dst_stride + (size_t)y * dp + x] = (uint8_t)(v > 255 ? 255 : v);
}

// Four adjacent outputs per thread.  For scale factors up to 1.9 the four outputs read source columns ox0 .. ox0+7 at
// most: three aligned 32-bit words per source row, funnel-shifted to start at ox0.  Each output then takes its byte pair
// with one PRMT and forms the horizontal blend p0*(256-cx) + p1*cx with one IDP.2A (the 16-bit weight pair comes packed
// from the table: tabxp[e] = {ofs, (256-cx) | cx << 16}, padded to a multiple of four entries, two 128-bit loads per
// thread).  Same integer arithmetic as k_resize_exact (bit-identical; v <= 255 by construction, so no clamp), half the
// instructions of the shift-and-mask form.
__global__ void __launch_bounds__(256) k_resize_exact4(const uint8_t* __restrict__ src, size_t src_stride, int sp, int sw,
                                                       int sh, uint8_t* __restrict__ dst, size_t dst_stride, int dp, int dw,
                                                       int dh, const int4* __restrict__ tabxp,
                                                       const int* __restrict__ taby) {
  const int xq = blockIdx.x * 64 + threadIdx.x;  // block = 64 x 4 threads = 256 x 4 outputs
  const int x = xq * 4;
  const int y = blockIdx.y * 4 + threadIdx.y;
  if (x >= dw || y >= dh) return;
  const int4 t0 = __ldg(&tabxp[2 * xq]), t1 = __ldg(&tabxp[2 * xq + 1]);  // {ofs, weights} of outputs x .. x+3
  const int oy = __ldg(&taby[y]), cy = __ldg(&taby[dh + y]);
  // source bytes ox0 .. ox0+7 of rows oy and oy+1.  The second row is clamped to the image (its weight cy is 0 there), so
  // every byte wanted lies inside the image or within 7 bytes of its end: unclamped loads (allocation slack).  Pitches and
  // image strides are multiples of 16, so both rows have the same misalignment.
  const uint8_t* r0 = src + (size_t)blockIdx.z * src_stride + (size_t)oy * sp + t0.x;
  const int mis = (int)((uintptr_t)r0 & 3);
  const uint32_t* pa = reinterpret_cast<const uint32_t*>(r0 - mis);
  const uint32_t* pb = oy + 1 < sh ? reinterpret_cast<const uint32_t*>(r0 - mis + sp) : pa;
  const uint32_t a0 = __ldg(pa), a1 = __ldg(pa + 1), a2 = __ldg(pa + 2);
  const uint32_t b0 = __ldg(pb), b1 = __ldg(pb + 1), b2 = __ldg(pb + 2);
  const int s8 = 8 * mis;
  const uint32_t alo = __funnelshift_r(a0, a1, s8), ahi = __funnelshift_r(a1, a2, s8);
  const uint32_t blo = __funnelshift_r(b0, b1, s8), bhi = __funnelshift_r(b1, b2, s8);
  const uint32_t wy0 = (uint32_t)(256 - cy), wy1 = (uint32_t)cy;
  const int ofs[4] = {t0.x, t0.z, t1.x, t1.z};
  const uint32_t wx[4] = {(uint32_t)t0.y, (uint32_t)t0.w, (uint32_t)t1.y, (uint32_t)t1.w};
  uint32_t v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t sel = (uint32_t)(ofs[i] - ofs[0]) * 0x11u + 0x10u;  // bytes k, k+1 of the 8-byte window
    const uint32_t h0 = __dp2a_lo(wx[i], __byte_perm(alo, ahi, sel), 0u);
    const uint32_t h1 = __dp2a_lo(wx[i], __byte_perm(blo, bhi, sel), 0u);
    v[i] = (h0 * wy0 + h1 * wy1 + 32768u) >> 16;
  }
  // rows are 16-byte aligned (pitch) and x is a multiple of 4: one 32-bit store (bytes past dw land in the row's padding)
  uint8_t* d = dst + (size_t)blockIdx.z * dst_stride + (size_t)y * dp + x;
  *reinterpret_cast<uint32_t*>(d) = (v[0] | (v[1] << 8)) | ((v[2] | (v[3] << 8)) << 16);
}

// Packed x table of k_resize_exact4 from (ofs, c1): 2 ints per output column, padded to a multiple of 4 columns with the
// last column's entry.  `out` has plf_resize_packed_len(dw) ints and must start on a 16-byte boundary.
size_t plf_resize_packed_len(int dw) { return 2 * (size_t)((dw + 3) & ~3); }
void plf_resize_pack_x(const int* ofs, const int* c1, int dw, int* out) {
  const int dw4 = (dw + 3) & ~3;
  for (int e = 0; e < dw4; ++e) {
    const int v = e < dw ? e : dw - 1;
    out[2 * e] = ofs[v];
    out[2 * e + 1] = (256 - c1[v]) | (c1[v] << 16);
  }
}

plf_status plf_launch_resize_exact(plf_ctx* ctx, const uint8_t* src, size_t src_stride, int sp, int sw, int sh, uint8_t* dst,
                                   size_t dst_stride, int dp, int dw, int dh, const int* tabx, const int* tabxp, const int* taby, int nimg) {
  if ((double)sw <= 1.9 * (double)dw) {  // four outputs span at most 3 * 1.9 + 2 < 8 source columns
    dim3 grid((dw + 255) / 256, (dh + 3) / 4, nimg);
    k_resize_exact4<<<grid, dim3(64, 4), 0, ctx->cur>>>(src, src_stride, sp, sw, sh, dst, dst_stride, dp, dw, dh,
                                                        reinterpret_cast<const int4*>(tabxp), taby);
  } else {
    dim3 grid((dw + 255) / 256, dh, nimg);
    k_resize_exact<<<grid, 256, 0, ctx->cur>>>(src, src_stride, sp, sw, sh, dst, dst_stride, dp, dw, dh, tabx, taby);
  }
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// ---- FAST + NMS ------------------------------------------------------------------------------------
__device__ __forceinline__ bool has_run9(uint32_t m16) {
  uint32_t m = m16 | (m16 << 16);  // circular
  uint32_t r = m & (m >> 1);       // runs of 2
  r &= r >> 2;                     // 4
  r &= r >> 4;                     // 8
  r &= m >> 8;                     // 9
  return (r & 0xFFFFu) != 0;
}

// exact cornerScore<16>: (max over 9-arcs of min signed difference, either polarity) - 1
__device__ int fast_corner_score(const int* d /*16*/) {
  int best = 0;
#pragma unroll
  for (int pol = 0; pol < 2; ++pol) {
    int m2[16], m4[16], m8[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int a = pol ? -d[i] : d[i], b = pol ? -d[(i + 1) & 15] : d[(i + 1) & 15];
      m2[i] = min(a, b);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) m4[i] = min(m2[i], m2[(i + 2) & 15]);
#pragma unroll
    for (int i = 0; i < 16; ++i) m8[i] = min(m4[i], m4[(i + 4) & 15]);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int last = pol ? -d[(i + 8) & 15] : d[(i + 8) & 15];
      best = max(best, min(m8[i], last));
    }
  }
  return best - 1;
}

// Tile = 62 x 30 output pixels; scores are needed on a 64 x 32 region (1-px halo for the NMS) and pixels on a 70 x 38
// region (3-px ring), which arrives as one TMA box (96 x 38 bytes from the 16-byte boundary at or below x0 - 4).
//   pass A  rejection, FOUR pixels per step on the aligned 32-bit words of the box: |v - p0| and |v - p8| of four adjacent
//           centres are two VABSDIFF4 on the words of rows y-3 / y / y+3, and "some difference exceeds the threshold" is a
//           3-instruction SWAR compare - a 9-arc of the 16-ring always contains one pixel of every opposite pair (k, k+8)
//           (OpenCV's FAST_t uses the same test), so a group whose four bytes all fail is dropped after ~5 instructions per
//           pixel; groups that survive get the pairs (4,12), (2,10), (6,14) the same way (neighbour words by funnel shift);
//           the bytes left go through the exact polarity-consistent pair tests one pixel at a time and are compacted
//           (measured: the extra SWAR stages leave time and instruction count where they were - pass B dominates);
//   pass B  full ring test + exact cornerScore on the compacted candidates (dense warps);
//   NMS     3x3 strict maximum + border filter + append, over the candidates only (nothing else has a score).
#define FN_OW 62
#define FN_OH 30
// bit 7 of every byte of d that is greater than th (bytes are unsigned; k7 = (0x7f - (th & 0x7f)) * 0x01010101)
__device__ __forceinline__ uint32_t fast_gt4(uint32_t d, uint32_t k7, bool th_small) {
  const uint32_t low = (d & 0x7f7f7f7fu) + k7;           // bit 7 <=> (d & 0x7f) > (th & 0x7f); no carry crosses a byte
  return (th_small ? (low | d) : (low & d)) & 0x80808080u;
}
__global__ void __launch_bounds__(256, 5) k_fast_nms(const __grid_constant__ CUtensorMap tmap, OrbGeom g, int l, int tiles_x,
                                                  uint32_t* __restrict__ cand, int* __restrict__ cand_count,
                                                  int* __restrict__ hist, int* __restrict__ overflow) {
  const int W = g.w[l], H = g.h[l];
  const int x0 = (blockIdx.x % tiles_x) * FN_OW, y0 = (blockIdx.x / tiles_x) * FN_OH;
  const int img = blockIdx.y;
  __shared__ __align__(128) uint8_t pxb[38][96];  // the TMA box (96 x 38 bytes) from the 16-byte boundary at or below x0 - 4
  __shared__ __align__(16) uint8_t sc[32][64];    // score of pixel (x0 - 1 + sx, y0 - 1 + sy)
  __shared__ unsigned short clist[32 * 64];
  __shared__ int ccount;
  __shared__ __align__(8) uint64_t bar;
  const int tid = threadIdx.x;
  if (tid == 0) {
    ccount = 0;
    plf_mbar_init(&bar);
  }
  reinterpret_cast<uint2*>(&sc[0][0])[tid] = make_uint2(0u, 0u);   // 256 x 8 bytes = the whole score tile
  __syncthreads();
  // The tile + halo arrives as ONE bulk-tensor copy (TMA).  Positions outside the image come back as zeros - they are
  // never used by a valid score (gx in [3, W-3), gy in [3, H-3)).
  const int xs = (x0 - 4) & ~15;   // (two's complement: also the boundary below a negative origin)
  if (tid == 0) plf_tma_load_3d(&pxb[0][0], &tmap, xs, y0 - 4, img, &bar, 38 * 96);
  const int boxoff = (x0 - 4) - xs;   // box column of pixel x0 - 4
  // px[ry][rx] = pixel (x0 - 4 + rx, y0 - 4 + ry)
  const uint8_t (*px)[96] = reinterpret_cast<const uint8_t (*)[96]>(&pxb[0][boxoff]);
  const int th = g.fast_th;
  const uint32_t k7 = (uint32_t)(0x7f - (th & 0x7f)) * 0x01010101u;
  const bool th_small = th < 128;
  plf_mbar_wait(&bar, 0);
  // ---- pass A: score pixel (sy, sx) sits at box row sy + 3, box column c_first + sx
  const int c_first = boxoff + 3, w_first = c_first >> 2, nwords = ((c_first + 63) >> 2) - w_first + 1;   // 16 or 17 words
  for (int gi = tid; gi < 32 * 17; gi += 256) {
    const int sy = gi / 17, wi = gi - sy * 17;
    const int gy = y0 - 1 + sy;
    if (wi >= nwords || gy < 3 || gy >= H - 3) continue;
    const int wcol = w_first + wi;
    const uint32_t wc = reinterpret_cast<const uint32_t*>(&pxb[sy + 3][0])[wcol];
    const uint32_t wd = reinterpret_cast<const uint32_t*>(&pxb[sy + 6][0])[wcol];   // ring pixel 0: (x, y + 3)
    const uint32_t wu = reinterpret_cast<const uint32_t*>(&pxb[sy][0])[wcol];       // ring pixel 8: (x, y - 3)
    uint32_t t = fast_gt4(__vabsdiffu4(wc, wd), k7, th_small) | fast_gt4(__vabsdiffu4(wc, wu), k7, th_small);
    if (t) {
      // the other three opposite pairs, still four centres at a time: (4, 12) = (x +- 3, y) from the neighbour words of the
      // centre row, (2, 10) / (6, 14) = (x +- 2, y +- 2) from rows y +- 2, each neighbour word a funnel shift of two aligned
      // words.  |difference| > th for one pixel of EVERY pair is necessary for either polarity, so this only rejects; the
      // byte loop below stays the exact (polarity-consistent) test.  Words beside the row's ends only feed bytes that are
      // not score pixels (sx < 0 or sx >= 64).
      const uint32_t* rc = reinterpret_cast<const uint32_t*>(&pxb[sy + 3][0]) + wcol;
      const uint32_t cl = rc[-1], cr = rc[1];
      t &= fast_gt4(__vabsdiffu4(wc, __funnelshift_r(wc, cr, 24)), k7, th_small) |
           fast_gt4(__vabsdiffu4(wc, __funnelshift_r(cl, wc, 8)), k7, th_small);
    }
    if (t) {
      const uint32_t* rp = reinterpret_cast<const uint32_t*>(&pxb[sy + 5][0]) + wcol;   // row y + 2
      const uint32_t* rm = reinterpret_cast<const uint32_t*>(&pxb[sy + 1][0]) + wcol;   // row y - 2
      const uint32_t p0 = rp[-1], p1 = rp[0], p2 = rp[1], m0 = rm[-1], m1 = rm[0], m2 = rm[1];
      const uint32_t pr = __funnelshift_r(p1, p2, 16), pl = __funnelshift_r(p0, p1, 16);   // (x + 2, y + 2), (x - 2, y + 2)
      const uint32_t mr = __funnelshift_r(m1, m2, 16), ml = __funnelshift_r(m0, m1, 16);   // (x + 2, y - 2), (x - 2, y - 2)
      t &= (fast_gt4(__vabsdiffu4(wc, pr), k7, th_small) | fast_gt4(__vabsdiffu4(wc, ml), k7, th_small)) &
           (fast_gt4(__vabsdiffu4(wc, mr), k7, th_small) | fast_gt4(__vabsdiffu4(wc, pl), k7, th_small));
    }
    while (t) {
      const int b = (__ffs(t) - 1) >> 3;   // byte whose pair (0, 8) does not rule it out
      t &= ~(0x80u << (8 * b));
      const int sx = 4 * wcol + b - c_first;
      const int gx = x0 - 1 + sx;
      if (sx < 0 || sx >= 64 || gx < 3 || gx >= W - 3) continue;
      const int cy = sy + 3, cx = sx + 3;
      const int v = (wc >> (8 * b)) & 0xFF;
      const int q0 = v - (int)((wd >> (8 * b)) & 0xFF), q8 = v - (int)((wu >> (8 * b)) & 0xFF);
      bool pd = (q0 > th) | (q8 > th), pb = (q0 < -th) | (q8 < -th);
      const int q4 = v - px[cy][cx + 3], q12 = v - px[cy][cx - 3];
      pd &= (q4 > th) | (q12 > th);
      pb &= (q4 < -th) | (q12 < -th);
      if (pd | pb) {
        const int q2 = v - px[cy + 2][cx + 2], q10 = v - px[cy - 2][cx - 2];
        const int q6 = v - px[cy - 2][cx + 2], q14 = v - px[cy + 2][cx - 2];
        pd &= ((q2 > th) | (q10 > th)) & ((q6 > th) | (q14 > th));
        pb &= ((q2 < -th) | (q10 < -th)) & ((q6 < -th) | (q14 < -th));
        if (pd | pb) clist[atomicAdd(&ccount, 1)] = (unsigned short)(sy * 64 + sx);
      }
    }
  }
  __syncthreads();
  // ---- pass B: full ring test + score on the candidates
  const int nc = ccount;
  for (int c = tid; c < nc; c += 256) {
    const int i = clist[c];
    const int sy = i >> 6, sx = i & 63;
    const int cy = sy + 3, cx = sx + 3;
    const int v = px[cy][cx];
    int d[16];
    d[0] = v - px[cy + 3][cx];      d[1] = v - px[cy + 3][cx + 1];  d[2] = v - px[cy + 2][cx + 2];
    d[3] = v - px[cy + 1][cx + 3];  d[4] = v - px[cy][cx + 3];      d[5] = v - px[cy - 1][cx + 3];
    d[6] = v - px[cy - 2][cx + 2];  d[7] = v - px[cy - 3][cx + 1];  d[8] = v - px[cy - 3][cx];
    d[9] = v - px[cy - 3][cx - 1];  d[10] = v - px[cy - 2][cx - 2]; d[11] = v - px[cy - 1][cx - 3];
    d[12] = v - px[cy][cx - 3];     d[13] = v - px[cy + 1][cx - 3]; d[14] = v - px[cy + 2][cx - 2];
    d[15] = v - px[cy + 3][cx - 1];
    uint32_t md = 0, mb = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      md |= (d[k] > th ? 1u : 0u) << k;   // neighbour darker than centre by more than th
      mb |= (d[k] < -th ? 1u : 0u) << k;  // brighter
    }
    if (has_run9(md) || has_run9(mb)) sc[sy][sx] = (uint8_t)fast_corner_score(d);
  }
  __syncthreads();
  // ---- NMS over the 62 x 30 interior of the score region + border filter + append: only candidates carry a score
  for (int c = tid; c < nc; c += 256) {
    const int i = clist[c];
    const int sy = i >> 6, sx = i & 63;
    if (sy < 1 || sy > FN_OH || sx < 1 || sx > FN_OW) continue;
    const int s = sc[sy][sx];
    if (s == 0) continue;
    const int gx = x0 - 1 + sx, gy = y0 - 1 + sy;
    if (gx < g.edge || gx >= W - g.edge || gy < g.edge || gy >= H - g.edge) continue;  // runByImageBorder
    if (!(s > sc[sy][sx - 1] && s > sc[sy][sx + 1] && s > sc[sy - 1][sx - 1] && s > sc[sy - 1][sx] &&
          s > sc[sy - 1][sx + 1] && s > sc[sy + 1][sx - 1] && s > sc[sy + 1][sx] && s > sc[sy + 1][sx + 1]))
      continue;
    const int slot = atomicAdd(&cand_count[img * ORB_MAX_LEVELS + l], 1);
    if (slot < g.cand_cap[l])
      cand[(size_t)img * g.cand_stride + g.cand_off[l] + slot] = ((uint32_t)gy << 20) | ((uint32_t)gx << 8) | (uint32_t)s;
    else
      *overflow = 1;
    atomicAdd(&hist[(img * ORB_MAX_LEVELS + l) * 256 + s], 1);
  }
}

// ---- retainBest + canonical ordering -----------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_select_sort(OrbGeom g, const uint32_t* __restrict__ cand,
                                                      const int* __restrict__ cand_count,
                                                      const int* __restrict__ hist, plf_keypoint* __restrict__ kps,
                                                      short2* __restrict__ kp_lxy, int* __restrict__ kp_count,
                                                      int* __restrict__ overflow) {
  __shared__ uint32_t keys[ORB_SORT_CAP];
  __shared__ int s_cnt, s_thr;
  const int img = blockIdx.x, tid = threadIdx.x;
  int base = 0;
  for (int l = 0; l < g.nlevels; ++l) {
    const int n = min(cand_count[img * ORB_MAX_LEVELS + l], g.cand_cap[l]);
    if (tid == 0) {
      s_cnt = 0;
      int thr = 0;
      const int want = g.nfeat[l];
      if (want < n) {
        if (want == 0) {
          thr = 256;
        } else {
          const int* hh = hist + (img * ORB_MAX_LEVELS + l) * 256;
          int acc = 0;
          for (int s = 255; s >= 0; --s) {
            acc += hh[s];
            if (acc >= want) {
              thr = s;
              break;
            }
          }
        }
      }
      s_thr = thr;
    }
    __syncthreads();
    const int thr = s_thr;
    const uint32_t* c = cand + (size_t)img * g.cand_stride + g.cand_off[l];
    for (int i = tid; i < n; i += 1024) {
      const uint32_t k = c[i];
      if ((int)(k & 0xFFu) >= thr) {
        const int pos = atomicAdd(&s_cnt, 1);
        if (pos < ORB_SORT_CAP) keys[pos] = k;
      }
    }
    __syncthreads();
    int m = s_cnt;
    if (m > ORB_SORT_CAP) {
      if (tid == 0) *overflow = 1;
      m = ORB_SORT_CAP;
    }
    int p2 = 1;
    while (p2 < m) p2 <<= 1;
    for (int i = m + tid; i < p2; i += 1024) keys[i] = 0xFFFFFFFFu;
    __syncthreads();
    for (int k = 2; k <= p2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < p2; i += 1024) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const uint32_t a = keys[i], b = keys[ixj];
            const bool up = (i & k) == 0;
            if ((a > b) == up) {
              keys[i] = b;
              keys[ixj] = a;
            }
          }
        }
        __syncthreads();
      }
    for (int i = tid; i < m; i += 1024) {
      const int o = base + i;
      if (o < g.max_kp) {
        const uint32_t k = keys[i];
        const int y = k >> 20, x = (k >> 8) & 0xFFF, s = k & 0xFF;
        plf_keypoint kp;
        kp.x = __fmul_rn((float)x, g.scale[l]);
        kp.y = __fmul_rn((float)y, g.scale[l]);
        kp.size = __fmul_rn((float)g.patch, g.scale[l]);
        kp.angle = -1.f;
        kp.response = (float)s;
        kp.octave = l;
        kp.class_id = -1;
        kps[(size_t)img * g.max_kp + o] = kp;
        kp_lxy[(size_t)img * g.max_kp + o] = make_short2((short)x, (short)y);
      } else if (i == m - 1) {
        *overflow = 1;
      }
    }
    base = min(base + m, g.max_kp);
    __syncthreads();
  }
  if (tid == 0) kp_count[img] = base;
}

// ---- orientation -------------------------------------------------------------------------------------
// cv::fastAtan2 scalar path (degrees); unfused float ops in OpenCV's order.
__device__ __forceinline__ float orb_fast_atan2(float y, float x) {
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

__global__ void __launch_bounds__(256) k_ic_angle(const uint8_t* __restrict__ img0, size_t img0_stride,
                                                  const uint8_t* __restrict__ pyr, OrbGeom g,
                                                  plf_keypoint* __restrict__ kps, const short2* __restrict__ kp_lxy,
                                                  const int* __restrict__ kp_count) {
  const int img = blockIdx.y;
  const int ki = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (ki >= kp_count[img]) return;
  plf_keypoint* kp = &kps[(size_t)img * g.max_kp + ki];
  const int l = kp->octave;
  const short2 p = kp_lxy[(size_t)img * g.max_kp + ki];
  const int W = g.pitch[l];   // row pitch
  const uint8_t* src = (l == 0) ? img0 + (size_t)img * img0_stride
                                : pyr + (size_t)img * g.pyr_stride + g.pyr_off[l];
  const uint8_t* center = src + (size_t)p.y * W + p.x;
  const int hp = g.half_patch;
  int m01 = 0, m10 = 0;
  const int u = lane - hp;  // lanes 0..2*hp cover u = -hp..hp (hp = 15 -> 31 lanes)
  if (lane <= 2 * hp) {
    m10 += u * center[u];
    for (int v = 1; v <= hp; ++v) {
      const int d = g.umax[v];
      if (u >= -d && u <= d) {
        const int vp = center[u + v * W], vm = center[u - v * W];
        m01 += v * (vp - vm);
        m10 += u * (vp + vm);
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    m01 += __shfl_xor_sync(0xFFFFFFFFu, m01, off);
    m10 += __shfl_xor_sync(0xFFFFFFFFu, m10, off);
  }
  if (lane == 0) kp->angle = orb_fast_atan2((float)m01, (float)m10);
}

// ---- descriptor-stage blur -----------------------------------------------------------------------------
// float row pass (sequential, FMA), symmetric float column pass (FMA), round-half-even saturate: OpenCV's sepFilter2D
// path for the pyramid ROI on FMA-capable hosts (see oracle/orb.c orc_orb_blur7).
// 64x32 outputs per CTA; the (tile + halo) box is staged by ONE TMA bulk-tensor copy (13 KB of shared memory per CTA in all, so
// 8 CTAs fit beside co-resident kernels; border CTAs rebuild BORDER_REFLECT_101 inside shared memory), the row pass produces 4
// adjacent outputs per thread from 10 pixels (k0*p0, fma(k1,p1,.) ... order), the column pass slides down 8 rows.
#define OBF_TW 64
#define OBF_TH 32
__global__ void __launch_bounds__(256) k_orb_blur7_fast(const __grid_constant__ CUtensorMap tmap, OrbGeom g,
                                                        uint8_t* __restrict__ blur, int l, int tiles_x) {
  constexpr int RH = OBF_TH + 6, RP = 80, NEED = 72;  // 70 pixels needed per row (72: whole words); box pitch 80
  __shared__ __align__(128) uint8_t raw[RH][RP];
  __shared__ __align__(16) float hrow[RH][OBF_TW];
  __shared__ __align__(8) uint64_t bar;
  const int W = g.w[l], H = g.h[l], BP = g.bpitch[l];
  const int x0 = (blockIdx.x % tiles_x) * OBF_TW - 13, y0 = (blockIdx.x / tiles_x) * OBF_TH;   // x0 - 3 on a 16-byte boundary (TMA)
  const int img = blockIdx.y;
  uint8_t* dst = blur + (size_t)img * g.blur_stride + g.blur_off[l];
  const int tid = threadIdx.x;
  if (tid == 0) plf_mbar_init(&bar);
  __syncthreads();
  if (tid == 0) plf_tma_load_3d(&raw[0][0], &tmap, x0 - 3, y0 - 3, img, &bar, RH * RP);
  plf_mbar_wait(&bar, 0);
  if (!(x0 >= 3 && x0 - 3 + NEED <= W && y0 >= 3 && y0 + OBF_TH + 3 <= H))   // border tile: BORDER_REFLECT_101 in place
    plf_tma_reflect_fix<RH, RP>(raw, x0 - 3, y0 - 3, W, H, NEED);
  __syncthreads();
  const float k0 = c_blur7[0], k1 = c_blur7[1], k2 = c_blur7[2], k3 = c_blur7[3], k4 = c_blur7[4], k5 = c_blur7[5], k6 = c_blur7[6];
  for (int it = tid; it < RH * (OBF_TW / 4); it += 256) {
    const int ry = it >> 4, j = it & 15;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(&raw[ry][4 * j]);
    const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
    const float p[10] = {(float)(w0 & 0xFFu), (float)((w0 >> 8) & 0xFFu), (float)((w0 >> 16) & 0xFFu), (float)(w0 >> 24),
                         (float)(w1 & 0xFFu), (float)((w1 >> 8) & 0xFFu), (float)((w1 >> 16) & 0xFFu), (float)(w1 >> 24),
                         (float)(w2 & 0xFFu), (float)((w2 >> 8) & 0xFFu)};
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a = __fmul_rn(k0, p[i]);
      a = __fmaf_rn(k1, p[i + 1], a); a = __fmaf_rn(k2, p[i + 2], a); a = __fmaf_rn(k3, p[i + 3], a);
      a = __fmaf_rn(k4, p[i + 4], a); a = __fmaf_rn(k5, p[i + 5], a); a = __fmaf_rn(k6, p[i + 6], a);
      o[i] = a;
    }
    *reinterpret_cast<float4*>(&hrow[ry][4 * j]) = make_float4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();
  const int c = tid & 63, q = tid >> 6;
  const int gx = x0 + c;
  if (gx >= 0 && gx < W) {
    float v[14];
#pragma unroll
    for (int k = 0; k < 14; ++k) v[k] = hrow[q * 8 + k][c];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int gy = y0 + q * 8 + r;
      if (gy < H) {
        float a = __fmul_rn(k3, v[r + 3]);
        a = __fmaf_rn(k4, __fadd_rn(v[r + 4], v[r + 2]), a);
        a = __fmaf_rn(k5, __fadd_rn(v[r + 5], v[r + 1]), a);
        a = __fmaf_rn(k6, __fadd_rn(v[r + 6], v[r]), a);
        uint32_t o;   // round half to even, saturated to [0, 255]: one conversion instruction
        asm("cvt.rni.u8.f32 %0, %1;" : "=r"(o) : "f"(a));
        dst[(size_t)gy * BP + gx] = (uint8_t)o;
      }
    }
  }
}

// ---- rBRIEF --------------------------------------------------------------------------------------------
// Rotation of the sampling pattern: (float)cos / sin of the keypoint angle in double, as OpenCV's computeOrbDescriptors
// evaluates it.  One THREAD per keypoint here - inside the warp-per-keypoint descriptor kernel the 32 lanes each paid the
// two f64 evaluations for the same value.
__global__ void __launch_bounds__(256) k_orb_trig(OrbGeom g, const plf_keypoint* __restrict__ kps,
                                                  const int* __restrict__ kp_count, float2* __restrict__ trig) {
  const int img = blockIdx.y, ki = blockIdx.x * 256 + threadIdx.x;
  if (ki >= kp_count[img]) return;
  const float angle = __fmul_rn(kps[(size_t)img * g.max_kp + ki].angle, (float)(3.14159265358979323846 / 180.f));
  trig[(size_t)img * g.max_kp + ki] = make_float2((float)cos((double)angle), (float)sin((double)angle));
}

// One warp per keypoint.  The 37x37 neighbourhood of the (blurred) keypoint that the 512 rotated samples can reach
// (|offset| <= 18) is first copied to shared memory with row-contiguous loads; the 16 samples of each lane then come
// from shared memory instead of 16 scattered global sectors.
#define RB_R 18
#define RB_D (2 * RB_R + 1)
#define RB_P 40
__global__ void __launch_bounds__(256) k_rbrief(const uint8_t* __restrict__ blur, OrbGeom g,
                                                const plf_keypoint* __restrict__ kps,
                                                const int* __restrict__ kp_count, const float2* __restrict__ trig,
                                                const int8_t* __restrict__ pattern, uint8_t* __restrict__ desc) {
  // the pattern as floats, transposed so that the 32 lanes of a warp read consecutive float4s for their j-th test:
  // test tt = lane * 8 + j lives at patf[j * 32 + lane]
  __shared__ __align__(16) float4 patf[256];
  __shared__ __align__(16) uint8_t patch[8][RB_D][RB_P];
  {
    const uint32_t w = reinterpret_cast<const uint32_t*>(pattern)[threadIdx.x];  // 4 x int8 of test threadIdx.x
    patf[(threadIdx.x & 7) * 32 + (threadIdx.x >> 3)] =
        make_float4((float)(int8_t)(w & 0xFF), (float)(int8_t)((w >> 8) & 0xFF), (float)(int8_t)((w >> 16) & 0xFF), (float)(int8_t)(w >> 24));
  }
  __syncthreads();
  const int img = blockIdx.y;
  const int wrp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ki = blockIdx.x * 8 + wrp;
  if (ki >= kp_count[img]) return;
  const plf_keypoint kp = kps[(size_t)img * g.max_kp + ki];
  const int l = kp.octave, W = g.bpitch[l];   // row pitch of the blurred level
  const float scale = __fdiv_rn(1.f, g.scale[l]);
  const float2 cs = __ldg(&trig[(size_t)img * g.max_kp + ki]);
  const float a = cs.x, b = cs.y;
  const int cyi = __float2int_rn(__fmul_rn(kp.y, scale)), cxi = __float2int_rn(__fmul_rn(kp.x, scale));
  // keypoints are >= edge (19) pixels inside the level, so the 37x37 window never leaves it
  const uint8_t* base = blur + (size_t)img * g.blur_stride + g.blur_off[l] + (size_t)(cyi - RB_R) * W + (cxi - RB_R);
  uint8_t (*P)[RB_P] = patch[wrp];
  {  // 37 rows x 10 words, four pixels per load step (plf_load4): 12 steps per lane instead of 74 byte loads
    // (keypoints are >= 19 pixels inside the level: rows y-18 .. y+18 and columns x-18 .. x+21 are inside the image)
    uint32_t* Pw = reinterpret_cast<uint32_t*>(&P[0][0]);
#pragma unroll 4
    for (int i = lane; i < RB_D * (RB_P / 4); i += 32) {
      const int r = i / (RB_P / 4), j = i - r * (RB_P / 4);
      Pw[i] = plf_load4_fast(base + (size_t)r * W + 4 * j);
    }
  }
  __syncwarp();
  unsigned val = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 q = patf[j * 32 + lane];
    const float qx0 = q.x, qy0 = q.y, qx1 = q.z, qy1 = q.w;
    const int ix0 = __float2int_rn(__fsub_rn(__fmul_rn(qx0, a), __fmul_rn(qy0, b)));
    const int iy0 = __float2int_rn(__fadd_rn(__fmul_rn(qx0, b), __fmul_rn(qy0, a)));
    const int ix1 = __float2int_rn(__fsub_rn(__fmul_rn(qx1, a), __fmul_rn(qy1, b)));
    const int iy1 = __float2int_rn(__fadd_rn(__fmul_rn(qx1, b), __fmul_rn(qy1, a)));
    const int t0 = P[RB_R + iy0][RB_R + ix0], t1 = P[RB_R + iy1][RB_R + ix1];
    val |= (t0 < t1 ? 1u : 0u) << j;
  }
  desc[((size_t)img * g.max_kp + ki) * 32 + lane] = (uint8_t)val;
}

// ---- host side -----------------------------------------------------------------------------------------
static int cv_round_f(float v) { return (int)nearbyintf(v); }

void plf_linear_coeffs_host(int srcsize, int dstsize, double scale, int* ofs, int* c1) {
  // interpolationLinear::getCoeffs (resize.cpp, bit-exact path); clamped cases folded into (ofs, c1)
  int mn = 0, mx = dstsize;
  for (int v = 0; v < dstsize; v++) {
    const double fval = scale * ((double)v + 0.5) - 0.5;
    const int ival = (int)floor(fval);
    ofs[v] = 0;
    c1[v] = 0;
    if (ival >= 0 && srcsize > 1) {
      if (ival < srcsize - 1) {
        ofs[v] = ival;
        c1[v] = (int)nearbyint((fval - ival) * 256.0);
      } else if (v < mx) {
        mx = v;
      }
    } else if (v + 1 > mn) {
      mn = v + 1;
    }
  }
  for (int v = 0; v < dstsize; v++) {
    if (v < mn) {
      ofs[v] = 0;
      c1[v] = 0;
    } else if (v >= mx) {
      ofs[v] = srcsize >= 2 ? srcsize - 2 : 0;
      c1[v] = srcsize >= 2 ? 256 : 0;
    }
  }
}

extern "C" void plf_orb_free(plf_ctx* ctx) {
  if (ctx->orb) {
    ctx->orb->bufs.release();
    delete ctx->orb;
    ctx->orb = nullptr;
  }
}

static int8_t* g_dev_pattern = nullptr;  // shared by all contexts on a device (read-only)
static int g_dev_pattern_device = -1;

// (Re)builds the ORB state for images of w x h and up to nimg images per launch.
static plf_status orb_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities) {
  OrbState* s = ctx->orb;
  if (s && s->w == w && s->h == h && s->nimg >= nimg && (s->two_parities || !two_parities)) return PLF_OK;
  if (s && s->two_parities) two_parities = true;
  if (s) {
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s->bufs.release();
    *s = OrbState();
  } else {
    s = ctx->orb = new OrbState();
  }
  const plf_params& P = ctx->params;
  if (P.orb_nlevels < 1 || P.orb_nlevels > ORB_MAX_LEVELS || P.orb_wta_k != 2 || P.orb_score != 1 ||
      P.orb_patch_size != 31)
    return plf_fail(ctx, PLF_ERR_INVALID,
                    "ORB: supported configuration is 1..8 levels, WTA_K=2, FAST score, patch 31 (got levels=%d "
                    "wta_k=%d score=%d patch=%d)", P.orb_nlevels, P.orb_wta_k, P.orb_score, P.orb_patch_size);
  // keypoints lie >= edge pixels inside their level and the orientation / rBRIEF window (37 x 37) is read without border
  // handling (k_ic_angle, k_rbrief), where OpenCV reads a border-reflected level padded by max(edge, 22): below 19 the
  // window would cross the level's border (and, on level 0, the image buffer)
  if (P.orb_edge_th < ORB_MIN_EDGE)
    return plf_fail(ctx, PLF_ERR_INVALID, "ORB: orb_edge_th %d < %d unsupported (the 31-pixel patch needs that border)",
                    P.orb_edge_th, ORB_MIN_EDGE);
  if (w >= 4096 || h >= 4096) return plf_fail(ctx, PLF_ERR_INVALID, "ORB: image larger than 4095 px");
  s->w = w; s->h = h; s->nimg = nimg;
  s->two_parities = two_parities;
  OrbGeom& g = s->g;
  memset(&g, 0, sizeof g);
  g.nlevels = P.orb_nlevels;
  g.edge = P.orb_edge_th; g.fast_th = min(max(P.orb_fast_th, 0), 255);
  g.patch = P.orb_patch_size; g.half_patch = P.orb_patch_size / 2;
  g.max_kp = ctx->limits.max_keypoints;
  const double scaleFactor = (double)P.orb_scale_factor;
  size_t pyr = 0, blur = 0, cand = 0;
  int tiles = 0;
  for (int l = 0; l < g.nlevels; ++l) {
    const float sc = (float)pow(scaleFactor, (double)l);
    g.scale[l] = sc;
    const float inv = 1.0f / sc;
    g.w[l] = cv_round_f(w * inv);
    g.h[l] = cv_round_f(h * inv);
    if (g.w[l] < 2 * g.edge + 8 || g.h[l] < 2 * g.edge + 8)
      return plf_fail(ctx, PLF_ERR_INVALID, "ORB: level %d (%dx%d) too small for edge threshold %d", l, g.w[l],
                      g.h[l], g.edge);
    g.pitch[l] = g.bpitch[l] = plf_pitch16(g.w[l]);   // level 0's source pitch is the caller's (set per run)
    const size_t a = ((size_t)g.pitch[l] * g.h[l] + 255) & ~size_t(255);
    if (l >= 1) { g.pyr_off[l] = pyr; pyr += a; }
    g.blur_off[l] = blur; blur += a;
    g.cand_cap[l] = (int)std::min<size_t>((size_t)g.w[l] * g.h[l] / 9 + 64, 32768);
    g.cand_off[l] = cand; cand += g.cand_cap[l];
    g.tiles_x[l] = (g.w[l] + ORB_TW - 1) / ORB_TW;
    g.tile_start[l] = tiles;
    tiles += g.tiles_x[l] * ((g.h[l] + ORB_TH - 1) / ORB_TH);
  }
  g.tile_start[g.nlevels] = tiles;
  for (int l = g.nlevels + 1; l <= ORB_MAX_LEVELS; ++l) g.tile_start[l] = tiles;
  g.pyr_stride = pyr; g.blur_stride = blur; g.cand_stride = cand;
  {  // nfeaturesPerLevel (orb.cpp computeKeyPoints)
    const float factor = (float)(1.0 / scaleFactor);
    float nd = P.orb_nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)g.nlevels));
    int sum = 0;
    for (int l = 0; l < g.nlevels - 1; ++l) {
      g.nfeat[l] = cv_round_f(nd);
      sum += g.nfeat[l];
      nd *= factor;
    }
    g.nfeat[g.nlevels - 1] = std::max(P.orb_nfeatures - sum, 0);
  }
  {  // umax
    const int hp = g.half_patch;
    int v, v0, vmax = (int)floor(hp * sqrt(2.f) / 2 + 1), vmin = (int)ceil(hp * sqrt(2.f) / 2);
    for (v = 0; v <= vmax; ++v) g.umax[v] = (int)nearbyint(sqrt((double)hp * hp - v * v));
    for (v = hp, v0 = 0; v >= vmin; --v) {
      while (g.umax[v0] == g.umax[v0 + 1]) ++v0;
      g.umax[v] = v0;
      ++v0;
    }
  }
  // resize tables
  std::vector<int> tab;
  for (int l = 1; l < g.nlevels; ++l) {
    const int sw = g.w[l - 1], sh = g.h[l - 1], dw = g.w[l], dh = g.h[l];
    s->rs_x_off[l] = tab.size();
    tab.resize(tab.size() + 2 * dw);
    plf_linear_coeffs_host(sw, dw, 1.0 / ((double)dw / sw), &tab[s->rs_x_off[l]], &tab[s->rs_x_off[l] + dw]);
    s->rs_y_off[l] = tab.size();
    tab.resize(tab.size() + 2 * dh);
    plf_linear_coeffs_host(sh, dh, 1.0 / ((double)dh / sh), &tab[s->rs_y_off[l]], &tab[s->rs_y_off[l] + dh]);
    tab.resize((tab.size() + 3) & ~(size_t)3);   // the packed x table is read with 128-bit loads
    s->rs_xp_off[l] = tab.size();
    tab.resize(tab.size() + plf_resize_packed_len(dw));
    plf_resize_pack_x(&tab[s->rs_x_off[l]], &tab[s->rs_x_off[l] + dw], dw, &tab[s->rs_xp_off[l]]);
  }
  const size_t N = (size_t)nimg, M = (size_t)g.max_kp;
  DevBufList& b = s->bufs;
  b.add(s->pyr, std::max<size_t>(pyr, 256) * N);
  b.add(s->blur, blur * N);
  b.add(s->cand, cand * N);
  b.add(s->cand_count, N * ORB_MAX_LEVELS);
  b.add(s->hist, N * ORB_MAX_LEVELS * 256);
  b.add(s->rs_tab, std::max<size_t>(tab.size(), 1));
  for (int p = 0; p < (two_parities ? 2 : 1); ++p) {  // outputs exist per batch parity (read by the match phase of batch i
    b.add(s->kps[p], N * M);                           // while batch i+1 is being extracted)
    b.add(s->kp_lxy[p], N * M);
    b.add(s->desc[p], N * M * 32);
    b.add(s->kp_count[p], N);
  }
  b.add(s->overflow, 1);
  b.add(s->trig, N * M);
  plf_status st = b.alloc(ctx, "ORB");
  if (st) return st;
  PLF_CUDA(ctx, cudaMemsetAsync(s->overflow, 0, sizeof(int), ctx->stream));
  if (!tab.empty())
    PLF_CUDA(ctx, cudaMemcpyAsync(s->rs_tab, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  {  // getGaussianKernel(7, 2, CV_32F): host doubles -> float (pinned equal to cv2 in tests)
    double d[7], sum = 0;
    for (int i = 0; i < 7; ++i) {
      const double x = i - 3.0;
      d[i] = exp(-0.5 / (2.0 * 2.0) * x * x);
      sum += d[i];
    }
    sum = 1. / sum;
    for (int i = 0; i < 7; ++i) s->blur_k[i] = (float)(d[i] * sum);
    PLF_CUDA(ctx, cudaMemcpyToSymbolAsync(c_blur7, s->blur_k, sizeof s->blur_k, 0, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (!g_dev_pattern || g_dev_pattern_device != ctx->device) {
    int8_t hp[1024];
    for (int i = 0; i < 1024; ++i) hp[i] = (int8_t)h_orb_bit_pattern_31[i];
    PLF_CUDA(ctx, cudaMalloc(&g_dev_pattern, 1024));
    PLF_CUDA(ctx, cudaMemcpyAsync(g_dev_pattern, hp, 1024, cudaMemcpyHostToDevice, ctx->stream));
    g_dev_pattern_device = ctx->device;
  }
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // tensor maps of the pyramid levels (fixed addresses); level 0 = the caller's image buffer, cached per run
  for (int l = 1; l < g.nlevels; ++l) {
    if (!plf_tma_encode_u8(&s->tm_fast[l], s->pyr + g.pyr_off[l], g.w[l], g.h[l], nimg, g.pitch[l], g.pyr_stride, 96, 38) ||
        !plf_tma_encode_u8(&s->tm_blur[l], s->pyr + g.pyr_off[l], g.w[l], g.h[l], nimg, g.pitch[l], g.pyr_stride, 80, OBF_TH + 6))
      return plf_fail(ctx, PLF_ERR_CUDA, "ORB: cuTensorMapEncodeTiled failed for pyramid level %d", l);
  }
  return PLF_OK;
}

// A failed (re)build leaves no state behind: the next call starts from scratch and fails the same way, instead of finding
// a size that matches the request and buffers that were released.
plf_status plf_orb_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities) {
  const plf_status st = orb_prepare(ctx, w, h, nimg, two_parities);
  if (st && ctx->orb) {
    ctx->orb->bufs.release();
    *ctx->orb = OrbState();
  }
  return st;
}

// Runs ORB on nimg images resident at d_imgs ([nimg][h][pitch], pitch a multiple of 16, stride img_stride bytes).
// Results stay on the device.
plf_status plf_orb_run(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int nimg, int par) {
  plf_status st = plf_orb_prepare(ctx, w, h, nimg, par != 0);
  if (st) return st;
  OrbState* s = ctx->orb;
  OrbGeom g = s->g;
  g.pitch[0] = pitch;
  cudaStream_t cs = ctx->cur;
  const CUtensorMap* tm_fast0 = s->tm_fast0.get(d_imgs, w, h, nimg, pitch, img_stride, 96, 38);
  const CUtensorMap* tm_blur0 = s->tm_blur0.get(d_imgs, w, h, nimg, pitch, img_stride, 80, OBF_TH + 6);
  if (!tm_fast0 || !tm_blur0)
    return plf_fail(ctx, PLF_ERR_CUDA, "ORB: cuTensorMapEncodeTiled failed for the source images (pitch %d, stride %zu)", pitch, img_stride);
  PLF_CUDA(ctx, cudaMemsetAsync(s->cand_count, 0, (size_t)nimg * ORB_MAX_LEVELS * sizeof(int), cs));
  PLF_CUDA(ctx, cudaMemsetAsync(s->hist, 0, (size_t)nimg * ORB_MAX_LEVELS * 256 * sizeof(int), cs));
  for (int l = 1; l < g.nlevels; ++l) {
    const uint8_t* src = (l == 1) ? d_imgs : s->pyr + g.pyr_off[l - 1];
    const size_t sstride = (l == 1) ? img_stride : g.pyr_stride;
    st = plf_launch_resize_exact(ctx, src, sstride, g.pitch[l - 1], g.w[l - 1], g.h[l - 1], s->pyr + g.pyr_off[l], g.pyr_stride,
                                 g.pitch[l], g.w[l], g.h[l], s->rs_tab + s->rs_x_off[l], s->rs_tab + s->rs_xp_off[l],
                                 s->rs_tab + s->rs_y_off[l], nimg);
    if (st) return st;
  }
  plf_mark(ctx, "orb.k_resize_exact");
  for (int l = 0; l < g.nlevels; ++l) {
    const int tx_ = (g.w[l] + FN_OW - 1) / FN_OW, ty_ = (g.h[l] + FN_OH - 1) / FN_OH;
    k_fast_nms<<<dim3(tx_ * ty_, nimg), 256, 0, cs>>>(l == 0 ? *tm_fast0 : s->tm_fast[l], g, l, tx_, s->cand, s->cand_count,
                                                      s->hist, s->overflow);
    PLF_LAUNCH_CHECK(ctx);
  }
  plf_mark(ctx, "orb.k_fast_nms");
  k_select_sort<<<nimg, 1024, 0, cs>>>(g, s->cand, s->cand_count, s->hist, s->kps[par], s->kp_lxy[par], s->kp_count[par], s->overflow);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "orb.k_select_sort");
  k_ic_angle<<<dim3((g.max_kp + 7) / 8, nimg), 256, 0, cs>>>(d_imgs, img_stride, s->pyr, g, s->kps[par], s->kp_lxy[par], s->kp_count[par]);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "orb.k_ic_angle");
  for (int l = 0; l < g.nlevels; ++l) {
    const int tx_ = plf_tma_tiles_x(g.w[l], 3), ty_ = (g.h[l] + OBF_TH - 1) / OBF_TH;
    k_orb_blur7_fast<<<dim3(tx_ * ty_, nimg), 256, 0, cs>>>(l == 0 ? *tm_blur0 : s->tm_blur[l], g, s->blur, l, tx_);
    PLF_LAUNCH_CHECK(ctx);
  }
  plf_mark(ctx, "orb.k_orb_blur7");
  k_orb_trig<<<dim3((g.max_kp + 255) / 256, nimg), 256, 0, cs>>>(g, s->kps[par], s->kp_count[par], s->trig);
  PLF_LAUNCH_CHECK(ctx);
  k_rbrief<<<dim3((g.max_kp + 7) / 8, nimg), 256, 0, cs>>>(s->blur, g, s->kps[par], s->kp_count[par], s->trig, g_dev_pattern, s->desc[par]);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "orb.k_rbrief");
  return PLF_OK;
}

int* plf_orb_overflow_flag(plf_ctx* ctx) { return ctx->orb->overflow; }

// device-side accessors for the pipeline
void plf_orb_outputs(plf_ctx* ctx, int par, plf_keypoint** kps, uint8_t** desc, int** counts, int* max_kp) {
  OrbState* s = ctx->orb;
  *kps = s->kps[par]; *desc = s->desc[par]; *counts = s->kp_count[par]; *max_kp = s->g.max_kp;
}

extern "C" plf_status plf_orb(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride, plf_keypoint* kps,
                              uint8_t* desc, int cap, int* n_out) {
  if (!ctx || !img || !n_out || w < 8 || h < 8 || stride < w || cap < 0 || (cap > 0 && (!kps || !desc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_orb: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  uint8_t* dimg = (uint8_t*)plf_scratch(ctx, 3, (size_t)pitch * h);
  if (!dimg) return PLF_ERR_CUDA;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_orb_run(ctx, dimg, (size_t)pitch * h, pitch, w, h, 1, 0);
  if (st) return st;
  OrbState* s = ctx->orb;
  int n = 0, ovf = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&n, s->kp_count[0], sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(&ovf, s->overflow, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ovf) {
    cudaMemsetAsync(s->overflow, 0, sizeof(int), ctx->stream);
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_orb: keypoint capacity exceeded (max_keypoints=%d)", s->g.max_kp);
  }
  *n_out = n;
  if (n > cap) return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_orb: %d keypoints > caller capacity %d", n, cap);
  if (n > 0) {
    PLF_CUDA(ctx, cudaMemcpyAsync(kps, s->kps[0], (size_t)n * sizeof(plf_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaMemcpyAsync(desc, s->desc[0], (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return PLF_OK;
}
