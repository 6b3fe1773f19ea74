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

// Every buffer carved out of a larger block starts on a 256-byte boundary.
inline size_t plf_align256(size_t x) { return (x + 255) & ~size_t(255); }

// The scratch slots of a context: device buffers that grow on demand (plf_scratch) and live until plf_destroy.  A slot
// belongs to the operators named beside it and to nothing else.  An entry point must not call anything that uses its own
// slot while pointers it carved from that slot are live: the call may reallocate the slot.
enum plf_scratch_slot {
  PLF_SCR_MATCH,       // plf_hamming_knn2, plf_match, plf_median_descriptors, plf_match_grid_points / _lines
  PLF_SCR_LBD,         // plf_lbd_gradients, plf_lbd
  PLF_SCR_GN,          // plf_gn_pose, plf_gn_pose_batch, plf_se3, plf_debug_motion_prior
  PLF_SCR_ORB,         // plf_orb
  PLF_SCR_LSD,         // plf_lsd, plf_detect_lines, plf_debug_sincosf
  PLF_SCR_MGB_PIPE,    // the windowed matcher of plf_batch_run (matching_strategy != 0)
  PLF_SCR_BA,          // plf_local_ba, plf_global_ba, plf_pose_graph, plf_pose_graph_batch: their staged layout;
                       // plf_debug_ldlt, plf_debug_ldlt_batch
  PLF_SCR_KF,          // plf_match_kf2kf, plf_match_map2kf and their _batch forms: their staged layout;
                       // plf_debug_match_grid_batch's inputs and outputs
  PLF_SCR_KF_MGB_PT,   // plf_match_kf2kf, plf_match_map2kf and their _batch forms, plf_debug_match_grid_batch: the
  PLF_SCR_KF_MGB_LS,   //   windowed matcher of points ... and of lines
  PLF_SCR_BOW,         // plf_bow_insert, plf_bow_insert_batch
  PLF_SCR_BA_BATCH,    // plf_local_ba_batch and plf_global_ba_batch: their staged layout
  PLF_SCR_LC,          // plf_loop_closure_pose and plf_loop_closure_pose_batch: their staged layout
  PLF_SCR_RECT_PIPE,   // the rectification of a grey batch in plf_batch_run_sequences (plf_set_sequence_rectification):
                       // its remapped pairs, sized for max_batch pairs once, so that it never grows under batches in flight
  PLF_SCR_COLOR_PIPE,  // plf_batch_upload_color and the conversion of plf_batch_run_sequences: the colour landing buffer
                       // of max_batch pairs (color_scratch in pipeline.cu)
  PLF_SCR_MASK_PIPE,   // plf_batch_upload_masks and the mask build of plf_batch_run_sequences: the pair masks' pyramids,
                       // 2 max_batch per upload slot at the largest image size (mask_scratch in pipeline.cu)
  PLF_SCR_COUNT
};

// The device buffers of one subsystem or call, declared once as (pointer, bytes).  For persistent buffers the same list
// gives the footprint, the allocation (one cudaMalloc per buffer, each with 64 bytes of slack for plf_load4, see
// plf_image_span) and the release; for per-call scratch it gives the carve from a scratch slot.
struct DevBufList {
  struct Entry { void** ptr; size_t bytes; };
  std::vector<Entry> entries;
  template <typename T>
  void add(T*& p, size_t n) { entries.push_back({reinterpret_cast<void**>(&p), n * sizeof(T)}); }
  size_t bytes() const;
  plf_status alloc(plf_ctx* ctx, const char* owner);   // on failure the buffers allocated so far stay listed
  void release();                                      // frees every buffer and nulls its pointer
  // Points every entry into one block of scratch slot `slot`, each at a 256-byte boundary.  On failure returns
  // PLF_ERR_CUDA (error set) and leaves the pointers untouched.
  plf_status carve(plf_ctx* ctx, plf_scratch_slot slot) const;
  // Buffers shared by states of several image sizes (plf_orb_create_sizes, plf_lsd_create_sizes): o lists the same
  // entries in the same order for another size.  Before alloc, grow takes each entry to the larger of the two sizes;
  // after, lend points o's entries at these buffers and empties o, so that only this list frees them.
  void grow(const DevBufList& o);
  void lend(DevBufList& o) const;
};

// The staged layout of one call: the host inputs [0, in), the outputs [in, in + out) and the device-only work after them,
// with a pinned mirror of inputs and outputs at the same offsets, so one copy uploads and one copy downloads.
// take_in / take_out / take_work return an offset from the start of their part.
struct StagedLayout {
  size_t in = 0, out = 0, work = 0;
  size_t take_in(size_t b) { const size_t o = in; in += plf_align256(b); return o; }
  size_t take_out(size_t b) { const size_t o = out; out += plf_align256(b); return o; }
  size_t take_work(size_t b) { const size_t o = work; work += plf_align256(b); return o; }
  // Fetches the pinned mirror (in + out bytes) and the device block (in + out + work bytes, scratch slot `slot`).
  plf_status acquire(plf_ctx* ctx, plf_scratch_slot slot, uint8_t** pin, uint8_t** dev) const;
};

// Upper bound of plf_set_max_sequences: keeps every slot index of the pipeline an int.
#define PLF_MAX_SEQUENCES (1 << 20)
// Upper bound of plf_set_image_sizes' n.
#define PLF_MAX_IMAGE_SIZES 8

struct OrbState;      // orb.cu
struct LsdState;      // lsd.cu
struct PlfTmaCache;   // plf_tma.cuh
struct BowDbs;        // dbow.cu

#define PLF_ORB_MAX_LEVELS 8
// The front-end settings of one pair of a batch (plf_set_sequence_params): its sequence's plf_params, or the context's, as
// the consumers read them, resolved when the batch was run.  The standalone detectors read a one-entry table of the
// context's.
struct PlfPairPrm {
  int orb_nlevels;                       // <= the context's: the levels the pair's images detect on
  int orb_nfeat[PLF_ORB_MAX_LEVELS];     // nfeaturesPerLevel of orb_nfeatures over orb_nlevels (plf_orb_level_features)
  int fast_th;                           // orb_fast_th clamped to [0, 255], the first frame's FAST threshold
  int lsd_nfeatures;
  float min_line_length;
  float max_dist_epip, min_disp, line_horiz_th, stereo_overlap_th, ls_min_disp_ratio;
  float min_ratio_12_p, min_ratio_12_l, line_sim_th;
  int best_lr;
  int matching_strategy, matching_s_ws, matching_f2f_ws, min_pt_matches, min_ls_matches, min_features;
  plf_gn_opts gn;                        // plf_gn_opts_from_params
};
PlfPairPrm plf_pair_prm(const plf_params& p);   // orb_nfeat stays 0 for an orb_nlevels no ORB state accepts

// What one sequence of a batched context has of its own; plf_reset_sequence keeps it, plf_drop_sequences frees it.
struct PlfSequence {
  bool own_prm = false;     // plf_set_sequence_params: prm (and pair, its device form) are the sequence's settings
  plf_params prm = {};
  PlfPairPrm pair = {};
  bool own_cam = false;     // plf_set_sequence_camera: cam is the sequence's calibration, else it uses the context's
  plf_camera cam = {};
  uint8_t* rect = nullptr;  // plf_set_sequence_rectification: device block of 12 w h bytes (PLF_RECT_* layout, pipeline.cu)
  uint8_t* mask[2] = {nullptr, nullptr};   // plf_set_sequence_mask: the left / right image's mask pyramid (plf_orb_mask_build)
  BowDbs* bow = nullptr;    // its bag-of-words databases (dbow.cu), from its first insert
};

struct plf_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;  // main stream: copies, the serial part of the pipeline, standalone operators
  cudaStream_t aux[3] = {nullptr, nullptr, nullptr};  // streams of the extraction (E), LSD growing (G) and LSD pre-grow (P) phases of plf_batch_run
  plf_params params;
  PlfPairPrm pair;                // plf_pair_prm(params), built by plf_create: params do not change after it
  plf_camera cam;
  plf_limits limits;
  int max_sequences = 1;          // plf_set_max_sequences: fixed once the pipeline exists
  // [max_sequences] once a sequence has something of its own (plf_sequence), else empty: every sequence at its defaults
  std::vector<PlfSequence> seqs;
  bool afast_on = false;          // plf_set_adaptive_fast: per-sequence FAST thresholds in the batched pipeline
  plf_adaptive_fast afast = {};
  bool motion_on = false;         // plf_set_motion_model: per-sequence pose predictions in the batched pipeline
  // plf_set_image_sizes: (w, h) of each image size the batched pipeline accepts besides cam's, none equal to it or to
  // another; fixed once the pipeline exists
  std::vector<int> image_sizes;
  std::string err;
  long long launches = 0;
  // scratch slots (device) of the host-pointer operator entry points
  DevBuf scratch[PLF_SCR_COUNT];
  // pinned host staging
  void* pinned = nullptr;
  size_t pinned_bytes = 0;
  // subsystem state (owned by the respective .cu)
  struct OrbState* orb_standalone = nullptr;   // plf_orb's working state: one image, rebuilt when the image size changes
  struct LsdState* lsd_standalone = nullptr;   // plf_lsd's and plf_detect_lines': likewise
  struct LsdTables* lsd_tables = nullptr;      // the LSD lookup tables of the parameters, read by every LSD state
  struct PipeState* pipe = nullptr;            // the batched pipeline, with its own ORB and LSD states
  struct BowState* bow = nullptr;   // DBoW2 vocabularies and keyframe database (dbow.cu)
  // optional per-stage timing (plf_profile_enable): events recorded after each kernel of plf_batch_run
  bool profile = false;
  bool profile_piped = false;  // marks recorded while the E/G/M software pipeline stays enabled (durations under overlap)
  std::vector<cudaEvent_t> prof_ev;
  std::vector<std::string> prof_names;
  size_t prof_used = 0;
};
// Records a timing mark on cs, the stream of the work named `name`, after that work (no-op unless profiling is enabled).
void plf_mark(plf_ctx* ctx, cudaStream_t cs, const char* name);

plf_status plf_fail(plf_ctx* ctx, plf_status code, const char* fmt, ...);
// Refuses a sequence index s outside [0, max_sequences), naming fn and s, or entry k of a seq array when k >= 0.
plf_status plf_check_sequence(plf_ctx* ctx, const char* fn, int s, int k = -1);
// Sequence s's record, sizing the records to max_sequences on the first call: call it to give s something of its own.
inline PlfSequence& plf_sequence(plf_ctx* ctx, int s) {
  if (ctx->seqs.empty()) ctx->seqs.resize(ctx->max_sequences);
  return ctx->seqs[s];
}
// The camera of sequence s (-1: the context's): its own calibration if it has one, else the context's.
inline const plf_camera& plf_sequence_camera(const plf_ctx* ctx, int s) {
  return s >= 0 && !ctx->seqs.empty() && ctx->seqs[s].own_cam ? ctx->seqs[s].cam : ctx->cam;
}
// The settings of sequence s as the front-end reads them: its own if it has them, else the context's.
inline const PlfPairPrm& plf_sequence_pair(const plf_ctx* ctx, int s) {
  const bool own = !ctx->seqs.empty() && ctx->seqs[s].own_prm;
  return own ? ctx->seqs[s].pair : ctx->pair;
}
// The index of image size w x h in the batched pipeline's list: 0 for the context's (cam), 1 + i for image_sizes' i-th,
// -1 for a size it does not accept.
inline int plf_image_size_index(const plf_ctx* ctx, int w, int h) {
  if (w == ctx->cam.width && h == ctx->cam.height) return 0;
  for (size_t i = 0; i < ctx->image_sizes.size(); i += 2)
    if (ctx->image_sizes[i] == w && ctx->image_sizes[i + 1] == h) return 1 + (int)(i / 2);
  return -1;
}
// Problem p of a batch call: its sequence to *s (seq NULL or seq[p] = -1: the context's) and that sequence's camera now
// to *cam, each if given.  An entry outside [-1, max_sequences) returns PLF_ERR_INVALID naming fn, the problem and entry.
plf_status plf_problem_camera(plf_ctx* ctx, const char* fn, const int32_t* seq, int p, const plf_camera** cam, int* s = nullptr);
plf_status plf_problem_cameras(plf_ctx* ctx, const char* fn, int n, const int32_t* seq, std::vector<const plf_camera*>& cams);
// Frees every sequence's maps, masks and databases and empties the records.
void plf_drop_sequences(plf_ctx* ctx);
// Frees one sequence's bag-of-words databases (dbow.cu); NULL is a no-op.
void plf_bow_dbs_free(BowDbs* d);
// Ensures scratch slot `slot` holds at least `bytes`; returns device pointer or nullptr (error set).
void* plf_scratch(plf_ctx* ctx, plf_scratch_slot slot, size_t bytes);
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
plf_status plf_launch_knn2(plf_ctx* ctx, cudaStream_t cs, const KnnProblem* d_probs, int nprob, int max_nq);

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
plf_status plf_launch_nnr(plf_ctx* ctx, cudaStream_t cs, const NnrProblem* d_probs, int nprob, int max_n1);
// Marks, per problem, the train rows that are the NNR-accepted best match of some query: the only rows whose reverse
// 2-NN the mutual-consistency check will read.  flags/qlist: [nprob][stride] (flags zeroed by the caller), qcount: [nprob].
plf_status plf_launch_nnr_mark(plf_ctx* ctx, cudaStream_t cs, const NnrProblem* d_probs, int nprob, int max_n1, int* flags,
                               int* qlist, int* qcount, int stride);

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
  const int* q_slot;     // optional [P]: problem p reads the query rows and count of slot q_slot[p] instead of slot p
  const uint8_t* d1; size_t d1_stride;   // query descriptor rows of problem p: d1 + slot * d1_stride (slot: see q_slot)
  const uint8_t* d2; size_t d2_stride;   // train rows: d2 + p * d2_stride
  const int* n1; int n1_stride;          // counts: n1[slot * n1_stride], n2[p * n2_stride]
  const int* n2; int n2_stride;
  unsigned short* D;     // scratch (set by the launcher)
  uint32_t* qmask;
  int* m21;
  int32_t* m12; size_t m12_stride;       // output rows of problem p: m12 + p * m12_stride
  int* count; int count_stride;          // matches of problem p (accumulated; zeroed by the caller)
  // optional [P]: problem p takes its window (matching_f2f_ws on every side when f2f, else (matching_s_ws, 0) x (0, 0)),
  // nnr, best_lr and line_sim_th from prm[p] instead of the fields above (the batched front-end's pairs)
  const struct PlfPairPrm* prm;
  int f2f;
};
// max_n1 / max_n2: upper bounds of the query / train counts; slot: the scratch slot D, the query masks and m21 live in;
// cs: the stream the launches are enqueued on.
plf_status plf_launch_match_grid_batch(plf_ctx* ctx, MgbArgs a, int nprob, int max_n1, int max_n2, plf_scratch_slot slot,
                                       cudaStream_t cs);

// ---- LBD (lbd.cu) ------------------------------------------------------------------------------
// tm: the caller's tensor-map cache over its source images (plf_tma.cuh)
plf_status plf_launch_blur5_sobel(plf_ctx* ctx, cudaStream_t cs, PlfTmaCache* tm, const uint8_t* imgs, int pitch,
                                  size_t img_stride, int w, int h, int nimg, short2* grad, size_t grad_stride);
plf_status plf_launch_lbd(plf_ctx* ctx, cudaStream_t cs, const short2* grad, size_t grad_stride, int w, int h, int nimg,
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
// The calibration of one pair of a batch: its sequence's camera when the batch was run (plf_set_sequence_camera).
struct PlfPairCam { double fx, fy, cx, cy, b; };
plf_gn_opts plf_gn_opts_from_params(const plf_params& p);
// d_cams: optional [nprob] device array, the camera of each problem (b unused); null = the context's camera.
// d_active: optional [nprob] device flags; a problem whose flag is 0 is not solved (its out and flags are not written).
// d_prm: optional [nprob] device array; problem p solves with d_prm[p].gn instead of o.
plf_status plf_launch_gn(plf_ctx* ctx, cudaStream_t cs, const GnProblem* d_probs, int nprob, const plf_gn_opts& o,
                         const PlfPairCam* d_cams = nullptr, const int* d_active = nullptr, const PlfPairPrm* d_prm = nullptr);

// ---- tiled LDL^T (lba.cu) ------------------------------------------------------------------------
// Factors each symmetric n x n matrix S (n = 6 nkf; row-major, leading dimension n; only its lower triangle is read) in
// place as L D L^T without pivoting, over 64 x 64 tiles, skipping the tiles of L that are exactly zero, and solves
// S x = g.  Afterwards S's diagonal holds D, y and x both hold the solution, and g has been overwritten.  Wp
// (n_t x 64 x 64 doubles) and nz (n_t x n_t bytes) are work, n_t = ceil(n / 64).  Enqueued on cs.
// Used by plf_global_ba, plf_pose_graph, their _batch forms and the plf_debug_ldlt hooks: one launch per stage and tile
// column over the nb systems of `big`, gridded (tile, system) at the largest one's n_max rows.  Each system is factored
// and solved with its own Wp and zero flags, bit for bit as it would be alone.  System i is skipped when
// active[big[i].p * active_stride] is 0 (active NULL: none is).  With big NULL the one system is `one` (nb = 1), read
// from the kernels' parameters: nothing is loaded before the factorisation's own data.
constexpr int PLF_LDLT_TILE = 64;
struct GbbBig {
  int p, nkf;                     // the system's problem index in its batch and its block count (n = 6 nkf rows)
  long long so, go, xo, wo, zo;   // offsets into S, g / y, x (doubles), Wp (doubles) and the zero flags (bytes)
};
struct GbbLdlt {
  const GbbBig* big;
  const int* active; int active_stride;   // the problems' activity flags, every active_stride ints, or NULL
  double* S; double* g; double* y; double* x; double* Wp; uint8_t* nz;
  GbbBig one;   // the system when big is NULL
};
plf_status gbb_ldlt(plf_ctx* ctx, cudaStream_t cs, const GbbLdlt& L, int nb, int n_max);

// ---- ORB (orb.cu) --------------------------------------------------------------------------------
// A working state for up to nimg images of w x h, with outputs once or per batch parity (two_parities).  On failure
// nothing is left allocated and *out is untouched.
plf_status plf_orb_create(plf_ctx* ctx, int w, int h, int nimg, bool two_parities, OrbState** out);
// out[i]: a state for images of size (wh[2i], wh[2i+1]), i < n.  They share one set of buffers, sized for the largest
// requirement of any of the sizes and owned by out[0]; each has its own geometry, resize tables and tensor maps.  So
// only one of them may run at a time, and out[0] is freed last or with the others.
plf_status plf_orb_create_sizes(plf_ctx* ctx, int n, const int* wh, int nimg, bool two_parities, OrbState** out);
// What plf_orb_create would refuse for w x h, with its message, allocating nothing; the level sizes when nlevels is given.
plf_status plf_orb_check_size(plf_ctx* ctx, int w, int h, int* nlevels = nullptr, int* lw = nullptr, int* lh = nullptr);
void plf_orb_free(OrbState* s);
// prm: a device table of pair settings, prm[z / 2] for image z: its level count (at most the state's), per-level counts and
// FAST threshold.
// img_th: the FAST threshold of each image, on the device (plf_set_adaptive_fast), or NULL for prm's.
// masks: a device table of each image's mask pyramid (plf_orb_mask_build), an entry NULL for an unmasked image, or NULL
// for no mask at all (the unmasked FAST kernel).
plf_status plf_orb_run(plf_ctx* ctx, cudaStream_t cs, OrbState* s, const uint8_t* d_imgs, size_t img_stride, int pitch, int nimg, int par,
                       const int* img_th, const uint8_t* const* masks, const PlfPairPrm* prm);
// nfeaturesPerLevel of cv::ORB (orb.cpp computeKeyPoints): nfeat[l] for l < nlevels.
void plf_orb_level_features(int nfeatures, float scale_factor, int nlevels, int* nfeat);
// One image's mask pyramid in s's level layout: its bytes (allocate 64 more, as every image buffer), and its build from a
// host mask of s->w x s->h, stride bytes per row, on cs.  Its first plf_pitch16(w) * h bytes are the mask itself.
size_t plf_orb_mask_bytes(const OrbState* s);
plf_status plf_orb_mask_build(plf_ctx* ctx, cudaStream_t cs, const OrbState* s, const uint8_t* mask, int stride, uint8_t* dst);
// One mask pyramid of a batched build (plf_orb_mask_pyramids): dst holds the caller's mask as its level 0 (any non-zero
// value allowed), and the build ANDs in the pyramid and_with (its level 0), or nothing when that is NULL.
struct PlfMaskBuild {
  uint8_t* dst;
  const uint8_t* and_with;
};
// Builds n mask pyramids of s's level layout in place from their level 0, one launch per level on cs: entries tab[0 .. n)
// of a device table, or the one entry `one` when tab is NULL.  Level 0 becomes 255 where the mask and and_with are both
// non-zero, else 0; level l >= 1 is resize(level l-1, INTER_LINEAR_EXACT) thresholded at 254, as plf_orb_mask_build.
plf_status plf_orb_mask_pyramids(plf_ctx* ctx, cudaStream_t cs, const OrbState* s, const PlfMaskBuild* tab, PlfMaskBuild one, int n);
void plf_orb_outputs(const OrbState* s, int par, plf_keypoint** kps, uint8_t** desc, int** counts, int* max_kp);
// The overflow flag is a set of causes (one bit each, OR-ed in by the kernel that met it); plf_orb_overflow_text words them,
// naming the limit that was actually hit: only max_keypoints is the caller's to raise.
enum { PLF_ORB_OVF_KEYPOINTS = 1,    // an image has more keypoints than plf_limits.max_keypoints (k_select_sort)
       PLF_ORB_OVF_SORT = 2,         // one pyramid level keeps more than ORB_SORT_CAP keypoints (k_select_sort)
       PLF_ORB_OVF_CANDIDATES = 4 }; // one pyramid level has more FAST corners than its candidate list holds (k_fast_nms)
int* plf_orb_overflow_flag(const OrbState* s);
void plf_orb_overflow_text(const OrbState* s, int causes, char* buf, size_t len);
void plf_linear_coeffs_host(int srcsize, int dstsize, double scale, int* ofs, int* c1);
plf_status plf_launch_resize_exact(plf_ctx* ctx, cudaStream_t cs, const uint8_t* src, size_t src_stride, int sp, int sw, int sh, uint8_t* dst,
                                   size_t dst_stride, int dp, int dw, int dh, const int* tabx, const int* tabxp, const int* taby, int nimg);
size_t plf_resize_packed_len(int dw);                                 // ints of the packed x table of k_resize_exact4
// k_resize_exact4's form (four outputs from an 8-byte source window) applies: four outputs span at most 3 * 1.9 + 2 < 8
// source columns
static inline bool plf_resize_packed_ok(int sw, int dw) { return (double)sw <= 1.9 * (double)dw; }
void plf_resize_pack_x(const int* ofs, const int* c1, int dw, int* out);   // out: 16-byte aligned

// ---- LSD (lsd.cu) --------------------------------------------------------------------------------
// Builds ctx->lsd_tables, once per context (plf_lsd_create calls it too).
plf_status plf_lsd_tables(plf_ctx* ctx);
void plf_lsd_tables_free(plf_ctx* ctx);
// A working state for up to nimg images of w x h, with the hand-off buffers once or per batch parity (two_parities).
// On failure nothing is left allocated and *out is untouched.
plf_status plf_lsd_create(plf_ctx* ctx, int w, int h, int nimg, bool two_parities, LsdState** out);
// n states of the sizes wh, sharing their buffers, as plf_orb_create_sizes.
plf_status plf_lsd_create_sizes(plf_ctx* ctx, int n, const int* wh, int nimg, bool two_parities, LsdState** out);
// What plf_lsd_create would refuse for w x h, allocating nothing; the scaled size when ws is given.
plf_status plf_lsd_check_size(plf_ctx* ctx, int w, int h, int* ws = nullptr, int* hs = nullptr);
void plf_lsd_free(LsdState* s);
// bytes plf_lsd_create_sizes allocates
size_t plf_lsd_footprint(const plf_ctx* ctx, int n, const int* wh, int nimg, bool two_parities);
plf_status plf_lsd_pre(plf_ctx* ctx, cudaStream_t cs, LsdState* s, const uint8_t* d_imgs, size_t img_stride, int pitch, int par, int n);
// keylines_wait: if set, the KeyLine outputs are overwritten only after this event.  masks: as for plf_orb_run; the KeyLine
// stage reads level 0 (plf_pitch16(w) bytes per row) of each listed image.  prm: as for plf_orb_run, image z's
// lsd_nfeatures and min_line_length from prm[z / 2].
plf_status plf_lsd_grow(plf_ctx* ctx, cudaStream_t cs, LsdState* s, int par, int n, cudaEvent_t keylines_wait,
                        const uint8_t* const* masks, const PlfPairPrm* prm);
void plf_lsd_outputs(const LsdState* s, int par, plf_keyline** kls, int** nlines, int* max_lines);
// Causes of the LSD overflow flag, one bit each (as the ORB flag above)
enum { PLF_LSD_OVF_SEGMENTS = 1,   // an image grows more regions than plf_limits.max_segments (k_lsd_grow)
       PLF_LSD_OVF_LINES = 2,      // more KeyLines to return than plf_limits.max_lines (k_keylines)
       PLF_LSD_OVF_SORT = 4 };     // more KeyLines to rank for the top lsd_nfeatures than KL_SORT_CAP (k_keylines)
int* plf_lsd_overflow_flag(const LsdState* s);
void plf_lsd_overflow_text(const LsdState* s, int causes, char* buf, size_t len);

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

// cv::fastAtan2 scalar path (degrees); unfused float ops in OpenCV's order.
__device__ __forceinline__ float plf_fast_atan2(float y, float x) {
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

// Hamming distance of two 256-bit descriptors, each as two uint4 halves (a0, a1) and (b0, b1).
__device__ __forceinline__ int plf_hamming256(uint4 a0, uint4 a1, uint4 b0, uint4 b1) {
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
         __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}
#endif
