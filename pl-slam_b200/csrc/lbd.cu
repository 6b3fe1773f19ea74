// LBD line band descriptor (SURVEY §8 a3): 5x5 Gaussian + 3x3 Sobel prelude and the 9-band
// descriptor with its 256-bit packing.
//
// Replaces BinaryDescriptor::compute -> computeImpl -> computeSobel/computeGaussianPyramid/computeLBD
// (3rdparty/line_descriptor/src/binary_descriptor_custom.cpp:524-528, :539-687, :350-398, :1026-1372,
// packing :401-412 over combinations :74-107).
//
// Kernels
//   k_blur5_sobel_fast
//                  u8 image -> interleaved int16 (dx,dy) gradient map.  One 64x32 tile per CTA staged by 32-bit words
//                  in shared memory with a 3-pixel BORDER_REFLECT_101 halo; the 5x5 sigma-1 blur is OpenCV's
//                  CV_8U fixed-point path (Q8.8 taps 14,62,104,62,14; DP4A row pass, one rounding), Sobel is exact
//                  integer.  HBM traffic: 1 B/px read + 4 B/px written (the algorithmic minimum for this stage).
//                  (k_blur5_sobel: generic variant for tiny images)
//   k_lbd          one CTA (64 threads) per line.  Bit-exactness fixes the mapping (SURVEY Appendix B): thread h
//                  (0..62) replays the h row-steps of the LSR origin in f32, then walks its row serially with
//                  the reference's repeated f32 additions and sequential f32 row sums; 72 threads-worth of band
//                  accumulators are then evaluated in row order by the same threads; the three normalisations keep their
//                  sums sequential on one thread (their f32 order is part of the result) and run everything
//                  element-wise on all threads; 32 byte-compares pack the bits.  No tree/shuffle reductions.
// All float arithmetic is unfused (--fmad=false) in the reference's source order.
#include "plf_internal.h"
#include "plf_tma.cuh"

#define LBD_TW 64
#define LBD_TH 16
#define LBD_NB 9
#define LBD_WB 7
#define LBD_ROWS 63

plf_status plf_lbd_init(plf_ctx* ctx);

struct LbdState {
  PlfTmaCache tm;   // source images of k_blur5_sobel_fast
};

__constant__ float c_gaussL[21];  // (float)gaussCoefL_[i]
__constant__ float c_gaussG[63];  // (float)gaussCoefG_[i]
__constant__ int c_comb[32][2];

static const int h_comb[32][2] = {
    {0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6},
    {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7}, {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8},
    {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};

// grid: (ceil(w/64), ceil(h/16), nimg); block 256
__global__ void __launch_bounds__(256) k_blur5_sobel(const uint8_t* __restrict__ imgs, int pitch,
                                                      size_t img_stride, int w, int h,
                                                      short2* __restrict__ grad, size_t grad_stride) {
  __shared__ uint8_t raw[LBD_TH + 6][LBD_TW + 8];       // halo 3
  __shared__ uint16_t hrow[LBD_TH + 6][LBD_TW + 2];     // horizontal pass, Q8.8, halo 1 in x
  __shared__ uint8_t blur[LBD_TH + 2][LBD_TW + 2];      // blurred, halo 1
  const uint8_t* img = imgs + (size_t)blockIdx.z * img_stride;
  short2* out = grad + (size_t)blockIdx.z * grad_stride;
  const int x0 = blockIdx.x * LBD_TW, y0 = blockIdx.y * LBD_TH;
  const int tid = threadIdx.x;
  // stage raw tile with reflect-101 on load: one warp per row, lanes along x
  const int lane = tid & 31, wrp = tid >> 5;
  const bool interior = x0 >= 3 && x0 + LBD_TW + 3 <= w && y0 >= 3 && y0 + LBD_TH + 3 <= h;
  for (int ry = wrp; ry < LBD_TH + 6; ry += 8) {
    const int gy = interior ? y0 - 3 + ry : plf_reflect101(y0 - 3 + ry, h);
    const uint8_t* row = img + (size_t)gy * pitch;
    for (int rx = lane; rx < LBD_TW + 6; rx += 32) raw[ry][rx] = row[interior ? x0 - 3 + rx : plf_reflect101(x0 - 3 + rx, w)];
  }
  __syncthreads();
  // horizontal 5-tap pass for halo-1 columns, all halo-3 rows (66 columns: lanes 0..31 take cx, cx+32, and 64/65)
  for (int ry = wrp; ry < LBD_TH + 6; ry += 8)
    for (int cx = lane; cx < LBD_TW + 2; cx += 32) {
      const uint8_t* p = &raw[ry][cx];  // taps at coords (x0-1+cx) + {-2..2} = raw offsets cx..cx+4
      hrow[ry][cx] = (uint16_t)(14 * p[0] + 62 * p[1] + 104 * p[2] + 62 * p[3] + 14 * p[4]);
    }
  __syncthreads();
  // vertical pass -> blurred (halo 1)
  for (int by = wrp; by < LBD_TH + 2; by += 8)
    for (int bx = lane; bx < LBD_TW + 2; bx += 32) {
      const uint32_t a = 14u * hrow[by][bx] + 62u * hrow[by + 1][bx] + 104u * hrow[by + 2][bx] +
                         62u * hrow[by + 3][bx] + 14u * hrow[by + 4][bx];
      const uint32_t v = (a + (1u << 15)) >> 16;
      blur[by][bx] = (uint8_t)(v > 255 ? 255 : v);
    }
  __syncthreads();
  // Sobel's own BORDER_REFLECT_101 acts on the *blurred* image (blurred(-1) = blurred(1)).  The raw tile was staged
  // with reflect-101, and the 5-tap window is symmetric, so blur computed at coordinate -1 from reflected pixels equals
  // the blur at coordinate 1 exactly (mirror-image taps): no fix-up needed at the image border.
  const int tx = tid & (LBD_TW - 1), rg = tid >> 6;  // LBD_TW == 64
  const int gx = x0 + tx;
  if (gx < w) {
    for (int ty = rg; ty < LBD_TH; ty += 4) {
      const int gy = y0 + ty;
      if (gy >= h) break;
      const int a00 = blur[ty][tx], a01 = blur[ty][tx + 1], a02 = blur[ty][tx + 2];
      const int a10 = blur[ty + 1][tx], a12 = blur[ty + 1][tx + 2];
      const int a20 = blur[ty + 2][tx], a21 = blur[ty + 2][tx + 1], a22 = blur[ty + 2][tx + 2];
      const int dx = (a02 - a00) + 2 * (a12 - a10) + (a22 - a20);
      const int dy = (a20 - a00) + 2 * (a21 - a01) + (a22 - a02);
      out[(size_t)gy * w + gx] = make_short2((short)dx, (short)dy);
    }
  }
}

// Fast variant: 64x32 outputs per CTA, the (tile + halo) box staged by ONE TMA bulk-tensor copy (plf_tma.cuh; border CTAs
// rebuild BORDER_REFLECT_101 inside shared memory), DP4A row pass (taps 14,62,104,62 | 14 packed as u8), 4-column vertical
// pass, register-sliding Sobel.  Same integer arithmetic as k_blur5_sobel (bit-identical), ~4x fewer instructions per pixel.
#define LBF_TW 64
#define LBF_TH 32
__global__ void __launch_bounds__(256) k_blur5_sobel_fast(const __grid_constant__ CUtensorMap tmap, int w, int h,
                                                           short2* __restrict__ grad, size_t grad_stride) {
  constexpr int RH = LBF_TH + 6;   // raw rows: halo 3 (blur 2 + sobel 1)
  constexpr int RP = 80;           // TMA box width (bytes, multiple of 16)
  constexpr int NEED = 76;         // columns read: 68 blurred columns + 4 taps + word slack
  constexpr int BW = 68;           // blurred columns computed (66 needed, rounded to groups of 4)
  __shared__ __align__(128) uint8_t raw[RH][RP];
  __shared__ __align__(16) uint16_t hrow[RH][BW];
  __shared__ __align__(16) uint8_t blur[LBF_TH + 2][BW + 4];
  __shared__ __align__(8) uint64_t bar;
  short2* out = grad + (size_t)blockIdx.z * grad_stride;
  const int x0 = blockIdx.x * LBF_TW - 13, y0 = blockIdx.y * LBF_TH, tid = threadIdx.x;   // x0 - 3 on a 16-byte boundary (TMA)
  if (tid == 0) plf_mbar_init(&bar);
  __syncthreads();
  if (tid == 0) plf_tma_load_3d(&raw[0][0], &tmap, x0 - 3, y0 - 3, (int)blockIdx.z, &bar, RH * RP);
  plf_mbar_wait(&bar, 0);
  if (!(x0 >= 3 && x0 - 3 + NEED <= w && y0 >= 3 && y0 + LBF_TH + 3 <= h))   // border tile: BORDER_REFLECT_101 in place
    plf_tma_reflect_fix<RH, RP>(raw, x0 - 3, y0 - 3, w, h, NEED);
  __syncthreads();
  const uint32_t tapsA = 14u | (62u << 8) | (104u << 16) | (62u << 24), tapsB = 14u;
  // horizontal pass: blurred column b (coordinate x0-1+b) uses raw offsets b..b+4
  for (int it = tid; it < RH * (BW / 4); it += 256) {
    const int ry = it / (BW / 4), j = it - ry * (BW / 4);
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(&raw[ry][4 * j]);
    const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = __byte_perm(w0, w1, 0x3210 + 0x1111 * i);
      const uint32_t hi = __byte_perm(w1, w2, 0x3210 + 0x1111 * i);
      o[i] = __dp4a(hi, tapsB, __dp4a(lo, tapsA, 0u));
    }
    *reinterpret_cast<uint2*>(&hrow[ry][4 * j]) = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
  }
  __syncthreads();
  // vertical pass -> blurred bytes (rows y0-1 .. y0+32, columns x0-1 .. x0+66)
  for (int it = tid; it < (LBF_TH + 2) * (BW / 4); it += 256) {
    const int by = it / (BW / 4), j = it - by * (BW / 4);
    uint32_t acc[4] = {0, 0, 0, 0};
    const uint32_t tp[5] = {14u, 62u, 104u, 62u, 14u};
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const uint2 v = *reinterpret_cast<const uint2*>(&hrow[by + k][4 * j]);
      acc[0] += tp[k] * (v.x & 0xFFFFu); acc[1] += tp[k] * (v.x >> 16);
      acc[2] += tp[k] * (v.y & 0xFFFFu); acc[3] += tp[k] * (v.y >> 16);
    }
    uint32_t pk = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t v = (acc[i] + (1u << 15)) >> 16;
      pk |= (v > 255 ? 255u : v) << (8 * i);
    }
    *reinterpret_cast<uint32_t*>(&blur[by][4 * j]) = pk;
  }
  __syncthreads();
  // Sobel (BORDER_REFLECT_101 on the blurred image is reproduced by the reflect-staged raw tile, see k_blur5_sobel)
  const int tx = tid & 63, q = tid >> 6;
  const int gx = x0 + tx;
  if (gx >= 0 && gx < w) {
    int a0[3], a1[3], a2[3];
    const int by0 = q * 8;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      a0[i] = blur[by0][tx + i];
      a1[i] = blur[by0 + 1][tx + i];
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int i = 0; i < 3; ++i) a2[i] = blur[by0 + r + 2][tx + i];
      const int gy = y0 + by0 + r;
      if (gy < h) {
        const int dx = (a0[2] - a0[0]) + 2 * (a1[2] - a1[0]) + (a2[2] - a2[0]);
        const int dy = (a2[0] - a0[0]) + 2 * (a2[1] - a0[1]) + (a2[2] - a0[2]);
        out[(size_t)gy * w + gx] = make_short2((short)dx, (short)dy);
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        a0[i] = a1[i];
        a1[i] = a2[i];
      }
    }
  }
}

plf_status plf_launch_blur5_sobel(plf_ctx* ctx, const uint8_t* imgs, int pitch, size_t img_stride,
                                  int w, int h, int nimg, short2* grad, size_t grad_stride) {
  if (nimg <= 0) return PLF_OK;
  if (w >= 8 && h >= 8 && (pitch & 15) == 0 && (img_stride & 15) == 0 && ((uintptr_t)imgs & 15) == 0) {
    plf_status st0 = plf_lbd_init(ctx);
    if (st0) return st0;
    const CUtensorMap* tm = ctx->lbd->tm.get(imgs, w, h, nimg, pitch, img_stride ? img_stride : (size_t)pitch * h, 80, LBF_TH + 6);
    if (!tm) return plf_fail(ctx, PLF_ERR_CUDA, "LBD: cuTensorMapEncodeTiled failed (pitch %d, stride %zu)", pitch, img_stride);
    dim3 grid(plf_tma_tiles_x(w, 3), (h + LBF_TH - 1) / LBF_TH, nimg);
    k_blur5_sobel_fast<<<grid, 256, 0, ctx->cur>>>(*tm, w, h, grad, grad_stride);
  } else {  // tiny images / unpadded rows: generic kernel
    dim3 grid((w + LBD_TW - 1) / LBD_TW, (h + LBD_TH - 1) / LBD_TH, nimg);
    k_blur5_sobel<<<grid, 256, 0, ctx->cur>>>(imgs, pitch, img_stride, w, h, grad, grad_stride);
  }
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// One CTA per (image, line slot).  kls: [nimg][max_lines]; counts: [nimg]; desc: [nimg][max_lines][32].
__global__ void __launch_bounds__(64, 12) k_lbd(const short2* __restrict__ grad, size_t grad_stride, int w,
                                            int h, const plf_keyline* __restrict__ kls,
                                            const int* __restrict__ counts, int max_lines,
                                            uint8_t* __restrict__ desc, float* __restrict__ desc_f) {
  const int img = blockIdx.y, li = blockIdx.x;
  if (li >= counts[img]) return;
  const plf_keyline kl = kls[(size_t)img * max_lines + li];
  const short2* g = grad + (size_t)img * grad_stride;
  __shared__ float rowv[LBD_ROWS][8];  // pgdL, ngdL, pgdO, ngdO, then their squares
  __shared__ float bandv[LBD_NB][8];   // pgdL, ngdL, pgdL2, ngdL2, pgdO, ngdO, pgdO2, ngdO2
  __shared__ float des[72];
  const int hID = threadIdx.x;
  const int lengthOfLSP = (short)kl.numOfPixels;
  const int halfWidth = (lengthOfLSP - 1) / 2;
  const int halfHeight = (LBD_ROWS - 1) / 2;
  const int imageWidth = w - 1, imageHeight = h - 1;
  const float midX = (float)(0.5 * (double)__fadd_rn(kl.sPointInOctaveX, kl.ePointInOctaveX));
  const float midY = (float)(0.5 * (double)__fadd_rn(kl.sPointInOctaveY, kl.ePointInOctaveY));
  const float dL0 = (float)cos((double)kl.angle), dL1 = (float)sin((double)kl.angle);
  const float dO0 = -dL1, dO1 = dL0;
  if (hID < LBD_ROWS) {
    float sCorX0 = __fadd_rn(__fadd_rn(__fmul_rn(-dL0, (float)halfWidth), __fmul_rn(dL1, (float)halfHeight)), midX);
    float sCorY0 = __fadd_rn(__fsub_rn(__fmul_rn(-dL1, (float)halfWidth), __fmul_rn(dL0, (float)halfHeight)), midY);
    for (int k = 0; k < hID; ++k) {  // replay the row steps in f32 (:1186-1187)
      sCorX0 = __fsub_rn(sCorX0, dL1);
      sCorY0 = __fadd_rn(sCorY0, dL0);
    }
    float sCorX = sCorX0, sCorY = sCorY0;
    float pL = 0.f, nL = 0.f, pO = 0.f, nO = 0.f;
    for (int wID = 0; wID < lengthOfLSP; ++wID) {
      int tx = (int)roundf(sCorX);
      int ty = (int)roundf(sCorY);
      tx = tx < 0 ? 0 : (tx > imageWidth ? imageWidth : tx);
      ty = ty < 0 ? 0 : (ty > imageHeight ? imageHeight : ty);
      const short2 d = __ldg(&g[(size_t)ty * w + tx]);
      const float fx = (float)d.x, fy = (float)d.y;
      const float gDL = __fadd_rn(__fmul_rn(fx, dL0), __fmul_rn(fy, dL1));
      const float gDO = __fadd_rn(__fmul_rn(fx, dO0), __fmul_rn(fy, dO1));
      if (gDL > 0) pL = __fadd_rn(pL, gDL); else nL = __fsub_rn(nL, gDL);
      if (gDO > 0) pO = __fadd_rn(pO, gDO); else nO = __fsub_rn(nO, gDO);
      sCorX = __fadd_rn(sCorX, dL0);
      sCorY = __fadd_rn(sCorY, dL1);
    }
    const float cg = c_gaussG[hID];
    pL = __fmul_rn(cg, pL); nL = __fmul_rn(cg, nL); pO = __fmul_rn(cg, pO); nO = __fmul_rn(cg, nO);
    rowv[hID][0] = pL; rowv[hID][1] = nL;
    rowv[hID][2] = __fmul_rn(pL, pL); rowv[hID][3] = __fmul_rn(nL, nL);
    rowv[hID][4] = pO; rowv[hID][5] = nO;
    rowv[hID][6] = __fmul_rn(pO, pO); rowv[hID][7] = __fmul_rn(nO, nO);
  }
  __syncthreads();
  // 72 band accumulators, each sequential over the rows that feed it, in row order (:1203-1239).
  for (int a = threadIdx.x; a < 72; a += 64) {
    const int b = a >> 3, q = a & 7;
    const bool sq = (q == 2 || q == 3 || q == 6 || q == 7);
    float acc = 0.f;
    const int h0 = max(0, LBD_WB * (b - 1)), h1 = min(LBD_ROWS, LBD_WB * (b + 2));
    for (int hh = h0; hh < h1; ++hh) {
      const int rb = hh / LBD_WB;
      // own band: weights [7..13]; row of band b+1 feeds b as "band above": [14..20]; row of band b-1: [0..6]
      const int wi = (hh % LBD_WB) + (rb == b ? LBD_WB : (rb == b + 1 ? 2 * LBD_WB : 0));
      const float c = c_gaussL[wi];
      const float v = rowv[hh][q];
      acc = __fadd_rn(acc, sq ? __fmul_rn(__fmul_rn(c, c), v) : __fmul_rn(c, v));
    }
    bandv[b][q] = acc;
  }
  __syncthreads();
  // Mean / standard deviation per band (:1253-1280), the two L2 normalisations (:1283-1315), the 0.4 clamp (:1322-1328)
  // and the final L2 normalisation (:1331-1341).  The element-wise parts (36 sqrtf, scalings, clamp) run on all
  // threads; only the three sums, whose f32 order is part of the result, stay sequential on thread 0.
  __shared__ float s_scale[2];
  {
    const float invN2 = (float)(1.0 / (LBD_WB * 2.0)), invN3 = (float)(1.0 / (LBD_WB * 3.0));
    for (int e = threadIdx.x; e < 36; e += 64) {   // e = band * 4 + q, q: pgdL, ngdL, pgdO, ngdO
      const int b = e >> 2, q = e & 3;
      const float invN = (b == 0 || b == LBD_NB - 1) ? invN2 : invN3;
      const int src = q < 2 ? q : q + 2;           // bandv column of the sum (0, 1, 4, 5); its square sum is at +2
      const float t = __fmul_rn(bandv[b][src], invN);
      des[b * 8 + q] = t;
      des[b * 8 + 4 + q] = sqrtf(__fsub_rn(__fmul_rn(bandv[b][src + 2], invN), __fmul_rn(t, t)));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tempM = 0.f, tempS = 0.f;
    for (int b = 0; b < LBD_NB; ++b) {
      const float* v = des + 8 * b;
      for (int k = 0; k < 4; ++k) tempM = __fadd_rn(tempM, __fmul_rn(v[k], v[k]));
      for (int k = 4; k < 8; ++k) tempS = __fadd_rn(tempS, __fmul_rn(v[k], v[k]));
    }
    s_scale[0] = __fdiv_rn(1.0f, sqrtf(tempM));
    s_scale[1] = __fdiv_rn(1.0f, sqrtf(tempS));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 72; i += 64) {
    float v = __fmul_rn(des[i], s_scale[(i & 7) < 4 ? 0 : 1]);
    if ((double)v > 0.4) v = (float)0.4;
    des[i] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 72; ++i) t = __fadd_rn(t, __fmul_rn(des[i], des[i]));
    s_scale[0] = __fdiv_rn(1.0f, sqrtf(t));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 72; i += 64) des[i] = __fmul_rn(des[i], s_scale[0]);
  __syncthreads();
  uint8_t* o = desc + ((size_t)img * max_lines + li) * 32;
  if (threadIdx.x < 32) {
    const float* f1 = des + 8 * c_comb[threadIdx.x][0];
    const float* f2 = des + 8 * c_comb[threadIdx.x][1];
    unsigned r = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (f1[i] > f2[i]) r |= 1u << i;
    o[threadIdx.x] = (uint8_t)r;
  }
  if (desc_f) {
    float* of = desc_f + ((size_t)img * max_lines + li) * 72;
    for (int i = threadIdx.x; i < 72; i += 64) of[i] = des[i];
  }
}

plf_status plf_lbd_init(plf_ctx* ctx) {
  if (ctx->lbd) return PLF_OK;
  // BinaryDescriptor ctor, binary_descriptor_custom.cpp:217-259 (host doubles, narrowed at use sites)
  float gl[21], gg[63];
  {
    double u = (LBD_WB * 3 - 1) / 2, sigma = (LBD_WB * 2 + 1) / 2, inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 21; ++i) {
      double dis = i - u;
      gl[i] = (float)exp(dis * dis * inv);
    }
    u = (LBD_NB * LBD_WB - 1) / 2;
    sigma = u;
    inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < 63; ++i) {
      double dis = i - u;
      gg[i] = (float)exp(dis * dis * inv);
    }
  }
  PLF_CUDA(ctx, cudaMemcpyToSymbolAsync(c_gaussL, gl, sizeof gl, 0, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyToSymbolAsync(c_gaussG, gg, sizeof gg, 0, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyToSymbolAsync(c_comb, h_comb, sizeof h_comb, 0, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->lbd = new LbdState();
  return PLF_OK;
}

plf_status plf_launch_lbd(plf_ctx* ctx, const short2* grad, size_t grad_stride, int w, int h, int nimg,
                          const plf_keyline* kls, const int* counts, int max_lines, uint8_t* desc,
                          float* desc_f) {
  if (nimg <= 0 || max_lines <= 0) return PLF_OK;
  plf_status st = plf_lbd_init(ctx);
  if (st) return st;
  dim3 grid(max_lines, nimg);
  k_lbd<<<grid, 64, 0, ctx->cur>>>(grad, grad_stride, w, h, kls, counts, max_lines, desc, desc_f);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

extern "C" void plf_lbd_free(plf_ctx* ctx) {
  delete ctx->lbd;
  ctx->lbd = nullptr;
}

static size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

extern "C" plf_status plf_lbd_gradients(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                                        int16_t* dxdy) {
  if (!ctx || !img || !dxdy || w < 2 || h < 2 || stride < w)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_lbd_gradients: bad arguments");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  const size_t ib = al256((size_t)pitch * h), gb = al256((size_t)w * h * 4);
  uint8_t* base = (uint8_t*)plf_scratch(ctx, 1, ib + gb);
  if (!base) return PLF_ERR_CUDA;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(base, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_launch_blur5_sobel(ctx, base, pitch, (size_t)pitch * h, w, h, 1, (short2*)(base + ib), 0);
  if (st) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(dxdy, base + ib, (size_t)w * h * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

extern "C" plf_status plf_lbd(plf_ctx* ctx, const uint8_t* img, int w, int h, int stride,
                              const plf_keyline* keylines, int n, uint8_t* desc, float* desc_float) {
  if (!ctx || !img || w < 2 || h < 2 || stride < w || n < 0 || (n > 0 && (!keylines || !desc)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_lbd: bad arguments");
  if (n == 0) {
    // reference: "Error: keypoint list is empty" + silent return (binary_descriptor_custom.cpp:556-560)
    return PLF_OK;
  }
  if (n > 32767)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_lbd: %d lines (reference numOfFinalLine is a short, :1029)", n);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int pitch = plf_pitch16(w);
  const size_t ib = al256((size_t)pitch * h), gb = al256((size_t)w * h * 4),
               kb = al256((size_t)n * sizeof(plf_keyline)), db = al256((size_t)n * 32),
               fb = al256((size_t)n * 72 * 4);
  uint8_t* base = (uint8_t*)plf_scratch(ctx, 1, ib + gb + kb + db + fb + 256);
  if (!base) return PLF_ERR_CUDA;
  uint8_t* dimg = base;
  short2* dgrad = (short2*)(base + ib);
  plf_keyline* dkl = (plf_keyline*)(base + ib + gb);
  uint8_t* ddesc = base + ib + gb + kb;
  float* dfl = (float*)(base + ib + gb + kb + db);
  int* dcount = (int*)(base + ib + gb + kb + db + fb);
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dimg, pitch, img, stride, w, h, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dkl, keylines, (size_t)n * sizeof(plf_keyline), cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dcount, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_launch_blur5_sobel(ctx, dimg, pitch, (size_t)pitch * h, w, h, 1, dgrad, 0);
  if (st) return st;
  st = plf_launch_lbd(ctx, dgrad, 0, w, h, 1, dkl, dcount, n, ddesc, desc_float ? dfl : nullptr);
  if (st) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(desc, ddesc, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
  if (desc_float)
    PLF_CUDA(ctx, cudaMemcpyAsync(desc_float, dfl, (size_t)n * 72 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}
