// Internal declarations shared by the CUDA translation units of libplslam_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "plslam_b200.h"

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

// The device buffers of one subsystem, declared once as (pointer slot, bytes): the same list gives the footprint, the
// allocation (one cudaMalloc per buffer, each with 64 bytes of slack for plf_load4, see plf_image_span) and the release.
struct DevBufList {
  struct Entry { void** slot; size_t bytes; };
  std::vector<Entry> entries;
  template <typename T>
  void add(T*& p, size_t n) { entries.push_back({reinterpret_cast<void**>(&p), n * sizeof(T)}); }
  size_t bytes() const;
  plf_status alloc(plf_ctx* ctx, const char* owner);   // on failure the buffers allocated so far stay listed
  void release();                                      // frees every buffer and nulls its slot
};

struct plf_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;  // main stream: copies, the serial part of the pipeline, standalone operators
  cudaStream_t cur = nullptr;     // stream the launch helpers enqueue on (== stream except inside forked sections)
  cudaStream_t aux[3] = {nullptr, nullptr, nullptr};  // streams of the extraction (E), LSD growing (G) and LSD pre-grow (P) phases of plf_batch_run
  cudaEvent_t lsd_keylines_wait = nullptr;  // if set: plf_lsd_grow waits for it before it overwrites the KeyLine outputs
  plf_params params;
  plf_camera cam;
  plf_limits limits;
  std::string err;
  long long launches = 0;
  // generic scratch slots (device) used by the host-pointer operator entry points
  DevBuf scratch[16];
  // pinned host staging
  void* pinned = nullptr;
  size_t pinned_bytes = 0;
  // subsystem state (owned by the respective .cu)
  struct OrbState* orb = nullptr;
  struct LsdState* lsd = nullptr;
  struct LbdState* lbd = nullptr;
  struct PipeState* pipe = nullptr;
  // optional per-stage timing (plf_profile_enable): events recorded after each kernel of plf_batch_run
  bool profile = false;
  bool profile_piped = false;  // marks recorded while the E/G/M software pipeline stays enabled (durations under overlap)
  std::vector<cudaEvent_t> prof_ev;
  std::vector<std::string> prof_names;
  size_t prof_used = 0;
};
// Records a timing mark on ctx->stream after the work named `name` (no-op unless profiling is enabled).
void plf_mark(plf_ctx* ctx, const char* name);

plf_status plf_fail(plf_ctx* ctx, plf_status code, const char* fmt, ...);
// Ensures scratch slot `slot` holds at least `bytes`; returns device pointer or nullptr (error set).
void* plf_scratch(plf_ctx* ctx, int slot, size_t bytes);
void* plf_pinned(plf_ctx* ctx, size_t bytes);

#define PLF_CUDA(ctx, call)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (call);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return plf_fail((ctx), PLF_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call,        \
                      cudaGetErrorString(_e));                                               \
  } while (0)

#define PLF_LAUNCH_CHECK(ctx)                                                                \
  do {                                                                                       \
    (ctx)->launches++;                                                                       \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess)                                                                   \
      return plf_fail((ctx), PLF_ERR_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__,    \
                      cudaGetErrorString(_e));                                               \
  } while (0)

// ---- matcher (match.cu) -----------------------------------------------------------------------
// One kNN problem: queries q[nq][8 x u32] against train t[nt][8 x u32]. If nq_ptr/nt_ptr are
// non-null the counts are read on the device (pipeline use), else nq/nt are used.
struct KnnProblem {
  const uint32_t* q;
  const uint32_t* t;
  const int* nq_ptr;
  const int* nt_ptr;
  int nq, nt;
  uint32_t* best;    // [nq] packed (dist << 16 | idx), 0xFFFFFFFF if none
  uint32_t* second;  // [nq]
  const int* qlist;  // optional: the query rows to process (nq / *nq_ptr = its length); results stored at best[row]
};
// Launches the kNN kernel over `nprob` problems (device array), max_nq = upper bound of nq.
plf_status plf_launch_knn2(plf_ctx* ctx, const KnnProblem* d_probs, int nprob, int max_nq);

struct NnrProblem {
  const uint32_t* best12;
  const uint32_t* second12;
  const uint32_t* best21;  // may be null when !best_lr
  const uint32_t* second21;
  const int* n1_ptr;
  const int* n2_ptr;
  int n1, n2;
  float nnr;
  int best_lr;
  int32_t* matches12;  // [n1]
  int* count;          // device counter (accumulated with atomicAdd; caller zeroes)
};
plf_status plf_launch_nnr(plf_ctx* ctx, const NnrProblem* d_probs, int nprob, int max_n1);
// Marks, per problem, the train rows that are the NNR-accepted best match of some query: the only rows whose reverse
// 2-NN the mutual-consistency check will read.  flags/qlist: [nprob][stride] (flags zeroed by the caller), qcount: [nprob].
plf_status plf_launch_nnr_mark(plf_ctx* ctx, const NnrProblem* d_probs, int nprob, int max_n1, int* flags, int* qlist,
                               int* qcount, int stride);

// ---- windowed greedy matcher, batched device-resident form (matchgrid.cu) ------------------------------------
struct MgGrid { int cols, rows, w_lo, w_hi, h_lo, h_hi; };
struct MgbArgs {
  MgGrid g;
  int is_lines, K, best_lr;
  int Kt;                // train capacity per problem (K: query capacity); D is K x Kt per problem
  int clip;              // lines: walk only the part of a query's Bresenham line whose window can reach the grid (for
                         // queries far outside it, e.g. pixel-unit projections); 0 walks every cell
  float nnr;
  double line_sim_th;
  const int* q_geo;      // [P][K][2|4]  query cells (points) / integer end points in grid units (lines)
  const int* t_geo;      // [P][Kt][2|4]
  const double* t_dir;   // [P][Kt][2] (lines) unit directions of the train lines
  const uint8_t* d1; size_t d1_stride;   // descriptor rows of problem p: d1 + p * d1_stride
  const uint8_t* d2; size_t d2_stride;
  const int* n1; int n1_stride;          // counts: n1[p * n1_stride]
  const int* n2; int n2_stride;
  unsigned short* D;     // scratch (set by the launcher)
  uint32_t* qmask;
  int* m21;
  int32_t* m12; size_t m12_stride;       // output rows of problem p: m12 + p * m12_stride
  int* count; int count_stride;          // matches of problem p (accumulated; zeroed by the caller)
};
// max_n1 / max_n2: upper bounds of the query / train counts; slot: the scratch slot D, the query masks and m21 live in.
plf_status plf_launch_match_grid_batch(plf_ctx* ctx, MgbArgs a, int nprob, int max_n1, int max_n2, int slot);

// ---- LBD (lbd.cu) ------------------------------------------------------------------------------
plf_status plf_launch_blur5_sobel(plf_ctx* ctx, const uint8_t* imgs, int pitch, size_t img_stride,
                                  int w, int h, int nimg, short2* grad, size_t grad_stride);
plf_status plf_launch_lbd(plf_ctx* ctx, const short2* grad, size_t grad_stride, int w, int h, int nimg,
                          const plf_keyline* kls, const int* counts, int max_lines, uint8_t* desc,
                          float* desc_f);

// ---- Gauss-Newton (gn.cu) -----------------------------------------------------------------------
struct GnProblem {
  const double* P;    // [np][3]
  const double* obs;  // [np][2]
  uint8_t* inl_p;     // [np]
  const int* np_ptr;
  int np;
  const double* sP;   // [nl][3]
  const double* eP;
  const double* le;
  uint8_t* inl_l;
  const int* nl_ptr;
  int nl;
  const double* T_init;  // 16 or null
  plf_pose_result* out;
};
plf_gn_opts plf_gn_opts_from_params(const plf_params& p);
plf_status plf_launch_gn(plf_ctx* ctx, const GnProblem* d_probs, int nprob, const plf_gn_opts& o);

// ---- ORB (orb.cu) --------------------------------------------------------------------------------
plf_status plf_orb_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities);
plf_status plf_orb_run(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int nimg, int par);
void plf_orb_outputs(plf_ctx* ctx, int par, plf_keypoint** kps, uint8_t** desc, int** counts, int* max_kp);
void plf_linear_coeffs_host(int srcsize, int dstsize, double scale, int* ofs, int* c1);
plf_status plf_launch_resize_exact(plf_ctx* ctx, const uint8_t* src, size_t src_stride, int sp, int sw, int sh, uint8_t* dst,
                                   size_t dst_stride, int dp, int dw, int dh, const int* tabx, const int* tabxp, const int* taby, int nimg);
size_t plf_resize_packed_len(int dw);                                 // ints of the packed x table of k_resize_exact4
void plf_resize_pack_x(const int* ofs, const int* c1, int dw, int* out);   // out: 16-byte aligned

// ---- LSD (lsd.cu) --------------------------------------------------------------------------------
plf_status plf_lsd_prepare(plf_ctx* ctx, int w, int h, int nimg, bool two_parities);
size_t plf_lsd_footprint(const plf_ctx* ctx, int w, int h, int nimg, bool two_parities);   // bytes plf_lsd_prepare allocates
plf_status plf_lsd_run(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int nimg);
plf_status plf_lsd_pre(plf_ctx* ctx, const uint8_t* d_imgs, size_t img_stride, int pitch, int w, int h, int par, int n);
plf_status plf_lsd_grow(plf_ctx* ctx, int w, int h, int par, int n);
void plf_lsd_outputs(plf_ctx* ctx, int par, plf_keyline** kls, int** nlines, int* max_lines);
int* plf_orb_overflow_flag(plf_ctx* ctx);
int* plf_lsd_overflow_flag(plf_ctx* ctx);

void plf_configure_lsd();

#ifdef __CUDACC__
// Four consecutive pixels starting at an arbitrary byte address, as two aligned 32-bit loads + a funnel shift (image
// rows are not 4-byte aligned for odd widths).  Word addresses are clamped to [lo, hi] - the aligned words that hold
// the first and the last byte of the image - so a halo word beyond the image's edge stays inside the allocation (the
// bytes it then returns lie outside the image and are never used).  The word at hi may extend up to 3 bytes past the
// image: every image buffer is allocated with 64 bytes of slack for that.
struct plf_span { uintptr_t lo, hi; };
__device__ __forceinline__ plf_span plf_image_span(const uint8_t* base, size_t bytes) {
  plf_span s;
  s.lo = (uintptr_t)base & ~(uintptr_t)3;
  s.hi = ((uintptr_t)(base + bytes) - 1) & ~(uintptr_t)3;
  return s;
}
__device__ __forceinline__ uint32_t plf_load4(const uint8_t* p, plf_span sp) {
  const uintptr_t a = (uintptr_t)p & ~(uintptr_t)3;
  const uintptr_t a0 = a < sp.lo ? sp.lo : (a > sp.hi ? sp.hi : a);
  const uintptr_t b = a + 4;
  const uintptr_t a1 = b < sp.lo ? sp.lo : (b > sp.hi ? sp.hi : b);
  const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(a0)), w1 = __ldg(reinterpret_cast<const uint32_t*>(a1));
  return __funnelshift_r(w0, w1, 8 * (int)((uintptr_t)p & 3));
}
// The same without the clamps, for callers whose four bytes are known to lie inside the image: the two aligned words
// then reach at most 3 bytes before the first / after the last of them, i.e. stay inside the image or - at its very end
// - inside the 64 bytes of slack every image buffer is allocated with.
__device__ __forceinline__ uint32_t plf_load4_fast(const uint8_t* p) {
  const uint32_t* a = reinterpret_cast<const uint32_t*>((uintptr_t)p & ~(uintptr_t)3);
  return __funnelshift_r(__ldg(a), __ldg(a + 1), 8 * (int)((uintptr_t)p & 3));
}
#endif
