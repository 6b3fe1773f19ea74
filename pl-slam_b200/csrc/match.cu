// Hamming 2-NN brute-force matcher + NNR / mutual-consistency filter (SURVEY §8 a4, a5).
//
// Replaces cv::BFMatcher(NORM_HAMMING).knnMatch(k=2) + the ratio / mutual logic of stvo-pl
// match()/matchNNR() (call sites src/mapHandler.cpp:277,424,597,712,3223,3249) and the popcount
// distance of 3rdparty/line_descriptor/src/bitops_custom.hpp:83-96.
//
// Layout: descriptors are 32 bytes = 8 x u32 = 2 x uint4, row-major, 16-byte aligned.
// (best, second) are packed u32 keys (distance << 16 | train index), so the (distance, index)
// lexicographic order of OpenCV's batch-distance kNN is a plain unsigned min; partial results are
// merged with warp shuffles.  The distances come from the int8 tensor-core MMA (see k_hamming_knn2_mma);
// DRAM traffic is the two descriptor sets once (they sit in L2 for the other query blocks).
#include "plf_internal.h"

#define KNN_NONE 0xFFFFFFFFu

// ---- the kNN kernel: tensor-core formulation ------------------------------------------------------------------------
// (round 1 started with an XOR+POPC kernel - 64 queries x 4 lanes per CTA over a shared train tile - that ran at the
//  POPC issue roofline, 13.1 ms per 3072 images; this formulation does the same work in 6.0 ms)
// Hamming(a, b) = popc(a) + popc(b) - 2 popc(a & b), and popc(a & b) over 256 bits is a dot product of 0/1 vectors: an
// integer GEMM.  Descriptors are expanded to one byte per bit and the dot products come from the int8 tensor-core MMA
// (mma.sync m16n8k32 u8 x u8 -> s32, 8 k-steps per 256 bits), which replaces 24 XOR/POPC/ADD instructions per pair and
// lane by 8 MMAs per 128 pairs and warp; what is left per pair is the (distance, index) key and the two-smallest update.
// Layout: a warp owns 16 queries (one m16 tile), kept expanded in registers for the whole kernel (A fragments, 32
// registers); a CTA of 8 warps shares a tile of 64 train descriptors expanded in shared memory in natural order (byte b
// = bit b, 320-byte row pitch: conflict-free 16-byte reads).  Because a dot product does not care about the order of
// k, lane (g, t) simply takes the 16-bit pieces t, t+4, t+8, t+12 of a descriptor for its 64 k-positions, for A and B
// alike, so B fragments are four 16-byte shared loads per group of 8 train rows.
#define KM_WARPS 8
#define KM_QPB (KM_WARPS * 16)
#define KM_TILE 64
#define KM_PITCH 320

__device__ __forceinline__ uint32_t km_expand4(uint32_t nibble) {  // 4 bits -> 4 bytes of 0 / 1
  return (nibble * 0x00204081u) & 0x01010101u;
}

__global__ void __launch_bounds__(KM_WARPS * 32) k_hamming_knn2_mma(const KnnProblem* __restrict__ probs) {
  const KnnProblem P = probs[blockIdx.y];
  const int nq = P.nq_ptr ? *P.nq_ptr : P.nq;
  const int nt = P.nt_ptr ? *P.nt_ptr : P.nt;
  const int q0 = blockIdx.x * KM_QPB;
  if (q0 >= nq) return;
  __shared__ __align__(16) uint8_t tb[KM_TILE * KM_PITCH];
  __shared__ __align__(8) int tpop[KM_TILE];
  const int tid = threadIdx.x, wrp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int qa = q0 + wrp * 16 + g, qb = qa + 8;
  const bool va = qa < nq, vb = qb < nq;
  const int rowa = va ? (P.qlist ? P.qlist[qa] : qa) : 0, rowb = vb ? (P.qlist ? P.qlist[qb] : qb) : 0;
  // A fragments: pieces t, t+4, t+8, t+12 of the two query rows, one byte per bit; popcounts of the whole rows
  uint32_t A[8][4];
  int pqa = 0, pqb = 0;
  {
    const uint4* pa = reinterpret_cast<const uint4*>(P.q) + 2 * (size_t)rowa;
    const uint4* pb = reinterpret_cast<const uint4*>(P.q) + 2 * (size_t)rowb;
    uint32_t wa[8] = {0, 0, 0, 0, 0, 0, 0, 0}, wb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (va) { const uint4 x = pa[0], y = pa[1]; wa[0] = x.x; wa[1] = x.y; wa[2] = x.z; wa[3] = x.w; wa[4] = y.x; wa[5] = y.y; wa[6] = y.z; wa[7] = y.w; }
    if (vb) { const uint4 x = pb[0], y = pb[1]; wb[0] = x.x; wb[1] = x.y; wb[2] = x.z; wb[3] = x.w; wb[4] = y.x; wb[5] = y.y; wb[6] = y.z; wb[7] = y.w; }
#pragma unroll
    for (int k = 0; k < 8; ++k) { pqa += __popc(wa[k]); pqb += __popc(wb[k]); }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int h = 4 * j + t;                         // 16-bit piece h = bits 16h .. 16h+15 = half (h & 1) of word h >> 1
      uint32_t ha = 0, hb = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {                    // (select without dynamic register indexing)
        ha = (h >> 1) == k ? wa[k] : ha;
        hb = (h >> 1) == k ? wb[k] : hb;
      }
      ha = (h & 1) ? ha >> 16 : ha & 0xFFFFu;
      hb = (h & 1) ? hb >> 16 : hb & 0xFFFFu;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 4 * j + i;                       // register r of the lane's 64 k-positions: step r/2, half r%2
        A[r >> 1][(r & 1) ? 2 : 0] = km_expand4((ha >> (4 * i)) & 0xFu);
        A[r >> 1][(r & 1) ? 3 : 1] = km_expand4((hb >> (4 * i)) & 0xFu);
      }
    }
  }
  uint32_t besta = KNN_NONE, seconda = KNN_NONE, bestb = KNN_NONE, secondb = KNN_NONE;
  const uint16_t* tp16 = reinterpret_cast<const uint16_t*>(P.t);
  const uint4* tp = reinterpret_cast<const uint4*>(P.t);
  for (int t0 = 0; t0 < nt; t0 += KM_TILE) {
    const int cnt = min(KM_TILE, nt - t0);
    __syncthreads();
    // expand the tile: 64 rows x 16 pieces, 4 pieces per thread; rows past the end are zero
    for (int i = tid; i < KM_TILE * 16; i += KM_WARPS * 32) {
      const int col = i >> 4, h = i & 15;
      const uint32_t hw = col < cnt ? (uint32_t)tp16[(size_t)(t0 + col) * 16 + h] : 0u;
      *reinterpret_cast<uint4*>(&tb[col * KM_PITCH + 16 * h]) =
          make_uint4(km_expand4(hw & 0xFu), km_expand4((hw >> 4) & 0xFu), km_expand4((hw >> 8) & 0xFu), km_expand4(hw >> 12));
    }
    if (tid < KM_TILE) {
      int pc = 0;
      if (tid < cnt) {
        const uint4 x = tp[2 * (size_t)(t0 + tid)], y = tp[2 * (size_t)(t0 + tid) + 1];
        pc = __popc(x.x) + __popc(x.y) + __popc(x.z) + __popc(x.w) + __popc(y.x) + __popc(y.y) + __popc(y.z) + __popc(y.w);
      }
      tpop[tid] = pc;
    }
    __syncthreads();
    const bool partial = cnt < KM_TILE;
    for (int grp = 0; grp < (cnt + 7) / 8; ++grp) {
      const uint8_t* brow = &tb[(grp * 8 + g) * KM_PITCH + 16 * t];
      uint32_t B[16];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 v = *reinterpret_cast<const uint4*>(brow + 64 * j);
        B[4 * j] = v.x; B[4 * j + 1] = v.y; B[4 * j + 2] = v.z; B[4 * j + 3] = v.w;
      }
      int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
#pragma unroll
      for (int st = 0; st < 8; ++st)
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3)
                     : "r"(A[st][0]), "r"(A[st][1]), "r"(A[st][2]), "r"(A[st][3]), "r"(B[2 * st]), "r"(B[2 * st + 1]));
      // c0, c1: row g x columns 2t, 2t+1 of the group; c2, c3: row g+8
      const int2 pt = *reinterpret_cast<const int2*>(&tpop[grp * 8 + 2 * t]);
      const uint32_t idx = (uint32_t)(t0 + grp * 8 + 2 * t);
      uint32_t k00 = ((uint32_t)(pqa + pt.x - 2 * c0) << 16) | idx, k01 = ((uint32_t)(pqa + pt.y - 2 * c1) << 16) | (idx + 1);
      uint32_t k10 = ((uint32_t)(pqb + pt.x - 2 * c2) << 16) | idx, k11 = ((uint32_t)(pqb + pt.y - 2 * c3) << 16) | (idx + 1);
      if (partial) {  // columns past the end of the train set do not exist
        if ((int)idx >= nt) { k00 = KNN_NONE; k10 = KNN_NONE; }
        if ((int)idx + 1 >= nt) { k01 = KNN_NONE; k11 = KNN_NONE; }
      }
      seconda = min(seconda, max(besta, k00)); besta = min(besta, k00);
      seconda = min(seconda, max(besta, k01)); besta = min(besta, k01);
      secondb = min(secondb, max(bestb, k10)); bestb = min(bestb, k10);
      secondb = min(secondb, max(bestb, k11)); bestb = min(bestb, k11);
    }
  }
  // the four lanes t = 0..3 of a row hold disjoint column subsets: merge
#pragma unroll
  for (int off = 1; off < 4; off <<= 1) {
    uint32_t ob = __shfl_xor_sync(0xFFFFFFFFu, besta, off), os = __shfl_xor_sync(0xFFFFFFFFu, seconda, off);
    seconda = min(min(seconda, os), max(besta, ob)); besta = min(besta, ob);
    ob = __shfl_xor_sync(0xFFFFFFFFu, bestb, off); os = __shfl_xor_sync(0xFFFFFFFFu, secondb, off);
    secondb = min(min(secondb, os), max(bestb, ob)); bestb = min(bestb, ob);
  }
  if (t == 0) {
    if (va) { P.best[rowa] = besta; P.second[rowa] = seconda; }
    if (vb) { P.best[rowb] = bestb; P.second[rowb] = secondb; }
  }
}

plf_status plf_launch_knn2(plf_ctx* ctx, cudaStream_t cs, const KnnProblem* d_probs, int nprob, int max_nq) {
  if (nprob <= 0 || max_nq <= 0) return PLF_OK;
  dim3 grid((max_nq + KM_QPB - 1) / KM_QPB, nprob);
  k_hamming_knn2_mma<<<grid, KM_WARPS * 32, 0, cs>>>(d_probs);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// matches_[i][0].distance < matches_[i][1].distance * nnr, evaluated in f32 exactly as the
// reference writes it (DMatch.distance is float; the product is rounded to f32 before the compare).
__device__ __forceinline__ bool nnr_accept(uint32_t best, uint32_t second, float nnr) {
  if (best == KNN_NONE || second == KNN_NONE) return false;  // fewer than 2 train rows: no match
  const float d1 = (float)(best >> 16), d2 = (float)(second >> 16);
  return d1 < __fmul_rn(d2, nnr);
}

__global__ void __launch_bounds__(256) k_nnr_mutual(const NnrProblem* __restrict__ probs) {
  const NnrProblem P = probs[blockIdx.y];
  const int n1 = P.n1_ptr ? *P.n1_ptr : P.n1;
  const int n2 = P.n2_ptr ? *P.n2_ptr : P.n2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int m = -1;
  if (i < n1 && n2 > 0) {
    const uint32_t b = P.best12[i], s = P.second12[i];
    if (nnr_accept(b, s, P.nnr)) {
      m = (int)(b & 0xFFFFu);
      if (P.best_lr) {
        const uint32_t b2 = P.best21[m], s2 = P.second21[m];
        if (!(nnr_accept(b2, s2, P.nnr) && (int)(b2 & 0xFFFFu) == i)) m = -1;
      }
    }
  }
  if (i < n1) P.matches12[i] = m;
  const unsigned ball = __ballot_sync(0xFFFFFFFFu, m >= 0);
  if ((threadIdx.x & 31) == 0 && ball && P.count) atomicAdd(P.count, __popc(ball));
}

// The mutual check of k_nnr_mutual reads the reverse 2-NN only at rows that are the accepted best match of some query;
// this kernel lists those rows (each once, any order) so the reverse kNN runs on them alone.
__global__ void __launch_bounds__(256) k_nnr_mark(const NnrProblem* __restrict__ probs, int* __restrict__ flags,
                                                  int* __restrict__ qlist, int* __restrict__ qcount, int stride) {
  const NnrProblem P = probs[blockIdx.y];
  const int n1 = P.n1_ptr ? *P.n1_ptr : P.n1;
  const int n2 = P.n2_ptr ? *P.n2_ptr : P.n2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1 || n2 <= 0 || !P.best_lr) return;
  const uint32_t b = P.best12[i], s = P.second12[i];
  if (!nnr_accept(b, s, P.nnr)) return;
  const int m = (int)(b & 0xFFFFu);
  if (atomicExch(&flags[(size_t)blockIdx.y * stride + m], 1) == 0)
    qlist[(size_t)blockIdx.y * stride + atomicAdd(&qcount[blockIdx.y], 1)] = m;
}

plf_status plf_launch_nnr_mark(plf_ctx* ctx, cudaStream_t cs, const NnrProblem* d_probs, int nprob, int max_n1, int* flags, int* qlist,
                               int* qcount, int stride) {
  if (nprob <= 0 || max_n1 <= 0) return PLF_OK;
  dim3 grid((max_n1 + 255) / 256, nprob);
  k_nnr_mark<<<grid, 256, 0, cs>>>(d_probs, flags, qlist, qcount, stride);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

plf_status plf_launch_nnr(plf_ctx* ctx, cudaStream_t cs, const NnrProblem* d_probs, int nprob, int max_n1) {
  if (nprob <= 0 || max_n1 <= 0) return PLF_OK;
  dim3 grid((max_n1 + 255) / 256, nprob);
  k_nnr_mutual<<<grid, 256, 0, cs>>>(d_probs);
  PLF_LAUNCH_CHECK(ctx);
  return PLF_OK;
}

// ---- host-pointer operator entry points ---------------------------------------------------------

extern "C" plf_status plf_hamming_knn2(plf_ctx* ctx, const uint8_t* d1, int n1, const uint8_t* d2,
                                       int n2, int32_t* idx1, int32_t* dist1, int32_t* idx2,
                                       int32_t* dist2) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n1 < 0 || n2 < 0 || n2 > 65535 || (n1 > 0 && !d1) || (n2 > 0 && !d2))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_hamming_knn2: bad sizes n1=%d n2=%d (n2 <= 65535)", n1,
                    n2);
  if (n1 == 0) return PLF_OK;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *dq, *dt;
  uint32_t *dbest, *dsec;
  KnnProblem* dprob;
  DevBufList scr;
  scr.add(dq, (size_t)n1 * 32); scr.add(dt, (size_t)std::max(n2, 1) * 32);
  scr.add(dbest, n1); scr.add(dsec, n1); scr.add(dprob, 1);
  if (plf_status st = scr.carve(ctx, PLF_SCR_MATCH)) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(dq, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, ctx->stream));
  if (n2 > 0)
    PLF_CUDA(ctx, cudaMemcpyAsync(dt, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, ctx->stream));
  KnnProblem hp = {(const uint32_t*)dq, (const uint32_t*)dt, nullptr, nullptr, n1, n2, dbest, dsec};
  PLF_CUDA(ctx, cudaMemcpyAsync(dprob, &hp, sizeof hp, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_launch_knn2(ctx, ctx->stream, dprob, 1, n1);
  if (st) return st;
  std::vector<uint32_t> hb(n1), hs(n1);
  PLF_CUDA(ctx, cudaMemcpyAsync(hb.data(), dbest, (size_t)n1 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(hs.data(), dsec, (size_t)n1 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n1; ++i) {
    const bool vb = hb[i] != KNN_NONE, vs = hs[i] != KNN_NONE;
    if (idx1) idx1[i] = vb ? (int32_t)(hb[i] & 0xFFFF) : -1;
    if (dist1) dist1[i] = vb ? (int32_t)(hb[i] >> 16) : -1;
    if (idx2) idx2[i] = vs ? (int32_t)(hs[i] & 0xFFFF) : -1;
    if (dist2) dist2[i] = vs ? (int32_t)(hs[i] >> 16) : -1;
  }
  return PLF_OK;
}

extern "C" plf_status plf_match(plf_ctx* ctx, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                                float nnr, int best_lr, int32_t* matches_12, int* n_matches) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n1 < 0 || n2 < 0 || n1 > 65535 || n2 > 65535 || (n1 > 0 && (!d1 || !matches_12)) ||
      (n2 > 0 && !d2))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_match: bad arguments n1=%d n2=%d (each <= 65535)", n1,
                    n2);
  if (n_matches) *n_matches = 0;
  if (n1 == 0) return PLF_OK;
  if (n2 == 0) {
    for (int i = 0; i < n1; ++i) matches_12[i] = -1;
    return PLF_OK;
  }
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t *dq, *dt;
  uint32_t *b12, *s12, *b21, *s21;
  int32_t* dm;
  int* dcount;
  KnnProblem* dkp;
  NnrProblem* dnp;
  DevBufList scr;
  scr.add(dq, (size_t)n1 * 32); scr.add(dt, (size_t)n2 * 32);
  scr.add(b12, n1); scr.add(s12, n1); scr.add(dm, n1);
  scr.add(b21, n2); scr.add(s21, n2);
  scr.add(dcount, 1); scr.add(dkp, 2); scr.add(dnp, 1);
  if (plf_status st = scr.carve(ctx, PLF_SCR_MATCH)) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(dq, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dt, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemsetAsync(dcount, 0, sizeof(int), ctx->stream));
  KnnProblem hk[2] = {
      {(const uint32_t*)dq, (const uint32_t*)dt, nullptr, nullptr, n1, n2, b12, s12},
      {(const uint32_t*)dt, (const uint32_t*)dq, nullptr, nullptr, n2, n1, b21, s21}};
  NnrProblem hn = {b12, s12, b21, s21, nullptr, nullptr, n1, n2, nnr, best_lr ? 1 : 0, dm, dcount};
  const int nk = best_lr ? 2 : 1;
  PLF_CUDA(ctx, cudaMemcpyAsync(dkp, hk, sizeof(KnnProblem) * nk, cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(dnp, &hn, sizeof hn, cudaMemcpyHostToDevice, ctx->stream));
  plf_status st = plf_launch_knn2(ctx, ctx->stream, dkp, nk, n1 > n2 ? n1 : n2);
  if (st) return st;
  st = plf_launch_nnr(ctx, ctx->stream, dnp, 1, n1);
  if (st) return st;
  int hcount = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(matches_12, dm, (size_t)n1 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaMemcpyAsync(&hcount, dcount, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (n_matches) *n_matches = hcount;
  return PLF_OK;
}

// ---- landmark descriptor maintenance (SURVEY 8(f) f3) ---------------------------------------------------------
// MapPoint::updateAverageDescDir / MapLine::updateAverageDescDir (src/mapFeatures.cpp:51-93, 121-163): among the n
// descriptors observed for a landmark, the representative is the one whose sorted row of Hamming distances to all of
// them (its own 0 included) has the smallest element at position int(1 + 0.5 (n - 1)); ties keep the first.  The mean
// observation direction is the plain f64 sum in observation order divided by n (the reference accumulates into an
// uninitialised Vector3d, :88-90 / :158-160 - started from zero here, deliberately).
// One warp per landmark.  Distances d(i,j) (<= 256) go to shared memory; the k-th smallest of row i is found by rank
// counting under the (value, column) order, which is what std::sort's result looks like position-wise.
#define MED_MAX_OBS 64
__global__ void __launch_bounds__(128) k_median_desc(const uint32_t* __restrict__ desc, const int* __restrict__ offsets,
                                                     const double* __restrict__ dirs, int n_landmarks,
                                                     int* __restrict__ med_idx, double* __restrict__ med_dir) {
  __shared__ unsigned short dist[4][MED_MAX_OBS][MED_MAX_OBS + 1];
  const int wrp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = blockIdx.x * 4 + wrp;
  if (L >= n_landmarks) return;
  const int o = offsets[L], n = offsets[L + 1] - o;
  if (n <= 0 || n > MED_MAX_OBS) {
    if (lane == 0) med_idx[L] = n <= 0 ? -1 : -2;  // -2: more observations than one warp pass handles
    return;
  }
  unsigned short (*D)[MED_MAX_OBS + 1] = dist[wrp];
  const uint4* dp = reinterpret_cast<const uint4*>(desc) + 2 * (size_t)o;
  for (int pr = lane; pr < n * n; pr += 32) {
    const int i = pr / n, j = pr - i * n;
    const uint4 a0 = dp[2 * i], a1 = dp[2 * i + 1], b0 = dp[2 * j], b1 = dp[2 * j + 1];
    D[i][j] = (unsigned short)plf_hamming256(a0, a1, b0, b1);
  }
  __syncwarp();
  const int k = (int)(1 + 0.5 * (n - 1));  // position read by the reference; k <= n - 1 for n >= 2
  unsigned best = 0xFFFFFFFFu;             // (median << 16 | row): smallest median, first row on ties
  for (int i = lane; i < n; i += 32) {
    int med = 0;
    if (k < n) {
      for (int j = 0; j < n; ++j) {
        const int v = D[i][j];
        int rank = 0;
        for (int m = 0; m < n; ++m) {
          const int u = D[i][m];
          rank += (u < v || (u == v && m < j)) ? 1 : 0;
        }
        if (rank == k) med = v;
      }
    }
    best = min(best, ((unsigned)med << 16) | (unsigned)i);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, off));
  if (lane == 0) {
    med_idx[L] = (int)(best & 0xFFFFu);
    if (dirs && med_dir) {
      double sx = 0.0, sy = 0.0, sz = 0.0;
      for (int i = 0; i < n; ++i) {
        sx += dirs[3 * (size_t)(o + i)]; sy += dirs[3 * (size_t)(o + i) + 1]; sz += dirs[3 * (size_t)(o + i) + 2];
      }
      med_dir[3 * (size_t)L] = sx / n; med_dir[3 * (size_t)L + 1] = sy / n; med_dir[3 * (size_t)L + 2] = sz / n;
    }
  }
}

extern "C" plf_status plf_median_descriptors(plf_ctx* ctx, const uint8_t* desc, const int* offsets, const double* dirs,
                                             int n_landmarks, int* med_idx, double* med_dir) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n_landmarks < 0 || (n_landmarks > 0 && (!desc || !offsets || !med_idx)))
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_median_descriptors: bad arguments");
  if (n_landmarks == 0) return PLF_OK;
  const int total = offsets[n_landmarks];
  if (offsets[0] != 0 || total < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_median_descriptors: offsets must start at 0 and be non-decreasing");
  for (int l = 0; l < n_landmarks; ++l) {
    const int n = offsets[l + 1] - offsets[l];
    if (n < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_median_descriptors: offsets must be non-decreasing");
    if (n == 1) return plf_fail(ctx, PLF_ERR_INVALID, "plf_median_descriptors: landmark %d has one observation (the reference reads past its row, src/mapFeatures.cpp:76; a landmark's first observation sets med_desc directly, :25-38)", l);
    if (n > MED_MAX_OBS) return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_median_descriptors: landmark %d has %d observations (max %d)", l, n, MED_MAX_OBS);
  }
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  uint8_t* dd;
  int *dofs, *didx;
  double *ddir, *dmed;
  DevBufList scr;
  scr.add(dd, (size_t)total * 32); scr.add(dofs, (size_t)n_landmarks + 1); scr.add(ddir, (size_t)total * 3);
  scr.add(didx, n_landmarks); scr.add(dmed, (size_t)n_landmarks * 3);
  if (plf_status st = scr.carve(ctx, PLF_SCR_MATCH)) return st;
  cudaStream_t cs = ctx->stream;
  if (total > 0) PLF_CUDA(ctx, cudaMemcpyAsync(dd, desc, (size_t)total * 32, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dofs, offsets, (size_t)(n_landmarks + 1) * 4, cudaMemcpyHostToDevice, cs));
  const bool want_dir = dirs && med_dir;
  if (want_dir && total > 0) PLF_CUDA(ctx, cudaMemcpyAsync(ddir, dirs, (size_t)total * 24, cudaMemcpyHostToDevice, cs));
  k_median_desc<<<(n_landmarks + 3) / 4, 128, 0, cs>>>((const uint32_t*)dd, dofs, want_dir ? ddir : nullptr, n_landmarks, didx,
                                                       want_dir ? dmed : nullptr);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(med_idx, didx, (size_t)n_landmarks * 4, cudaMemcpyDeviceToHost, cs));
  if (want_dir) PLF_CUDA(ctx, cudaMemcpyAsync(med_dir, dmed, (size_t)n_landmarks * 24, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}
