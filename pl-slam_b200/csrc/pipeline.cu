// Batched stereo front-end: extraction -> L/R stereo association -> frame-to-frame tracking -> pose refinement
// (SURVEY §8 a6, a7, a10 and the call pattern of app/plslam_dataset.cpp:111-163).
//
// Replaces, per stereo pair: StereoFrameHandler::insertStereoPair (app/plslam_dataset.cpp:127) = new StereoFrame +
// extractStereoFeatures (ORB + LSD/LBD on both images, matchStereoPoints / matchStereoLines) + f2fTracking, and
// StereoFrameHandler::optimizePose (app/plslam_dataset.cpp:128).  stvo-pl is not vendored by the reference; the
// association rules restate SURVEY.md Appendix A.2/A.3 (see oracle/frontend.py, which this file must match
// bit-for-bit on features / matches and to 1e-4 on the pose).
//
// One call processes B stereo pairs of up to max_sequences sequences.  Everything except the final SE(3) chaining is
// independent per pair (extraction, stereo association) or per pair and its previous frame of the same sequence
// (tracking and the pose increment start from identity, or with plf_set_motion_model from the sequence's prediction,
// which the previous batch's match phase left on the device), so all B
// pairs run in the same launches: images [2B][H][W] (2k = left, 2k+1 = right) -> ORB / LSD / LBD over 2B images ->
// per-pair kernels.  Pair k's previous frame is the slot prev[k] of the batch's sequence table; the last frame of each
// sequence in the batch is carried to that sequence's carry slot for the next call.
#include <cmath>
#include <cstddef>

#include "plf_internal.h"
#include "plf_geom.cuh"
#include "plf_se3.cuh"
#include "plf_tma.cuh"

// Stereo-valid features per frame slot, [slots][cap][per]: one row per array, (name = its plf_frame_view member, element
// type, capacity per slot: K = max_keypoints or Ln = max_lines, elements per feature).  The counts (one int per slot)
// follow the arrays of their kind.
#define PLF_PT_FIELDS(X) \
  X(pt_pl, double2, K, 1) X(pt_disp, double, K, 1) X(pt_P, double, K, 3) X(pt_octave, int, K, 1) X(pdesc, uint8_t, K, 32)
#define PLF_LS_FIELDS(X)                                                                                              \
  X(ls_spl, double2, Ln, 1) X(ls_epl, double2, Ln, 1) X(ls_sdisp, double, Ln, 1) X(ls_edisp, double, Ln, 1)         \
  X(ls_sP, double, Ln, 3) X(ls_eP, double, Ln, 3) X(ls_le, double, Ln, 3) X(ls_angle, float, Ln, 1) X(ldesc, uint8_t, Ln, 32)

struct FrameSlots {
#define PLF_FS_MEMBER(name, T, cap, per) T* name = nullptr;
  PLF_PT_FIELDS(PLF_FS_MEMBER) int* pt_count = nullptr;
  PLF_LS_FIELDS(PLF_FS_MEMBER) int* ls_count = nullptr;
#undef PLF_FS_MEMBER
};
#define PLF_FS_ONE(name, T, cap, per) +1
constexpr int PLF_FS_NFIELDS = 0 PLF_PT_FIELDS(PLF_FS_ONE) PLF_LS_FIELDS(PLF_FS_ONE);
#undef PLF_FS_ONE

// ---- rectification (plf_set_sequence_rectification, DESIGN.md section 8) ----
// A sequence's maps, one device block of 12 w h bytes: map1 (x, y) of the left then the right image (short2 [2][h][w]),
// then map2 of the left then the right image (uint16 [2][h][w]).
#define PLF_RECT_MAP1(base, A, side) (reinterpret_cast<const short2*>(base) + (size_t)(side) * (A))
#define PLF_RECT_MAP2(base, A, side) (reinterpret_cast<const uint16_t*>((base) + 8 * (A)) + (size_t)(side) * (A))
// One pair of a batch's input table: its index and its sequence's maps (NULL: the pair is not rectified).
struct PlfRectPair { const uint8_t* maps; int pair; int pad; };

// One entry of the batch table ring, for max_batch pairs B: the sequence table (prev[B] = the frame slot of pair k's
// previous frame, then the carry list [B][2] of (frame slot, carry slot)), the pairs' cameras [B] and settings [B]
// (plf_set_sequence_camera, plf_set_sequence_params, else the context's), then the input table [B], the mask table [2B]
// (image z's mask pyramid: its pair mask's, plf_batch_upload_masks, else its sequence's, plf_set_sequence_mask, else
// NULL) and the build list [2B] of the pair masks' pyramids.  Every batch uses the parts before the input table: they are
// one copy.  The pinned and the device ring use the same layout.
struct BatchTab {
  int32_t* prev;
  int32_t* carry;
  PlfPairCam* cams;
  PlfPairPrm* prm;
  PlfRectPair* in;
  const uint8_t** masks;
  PlfMaskBuild* build;
};
static size_t batch_tab_bytes(int B) {
  return plf_align256(3 * sizeof(int32_t) * B) + plf_align256(sizeof(PlfPairCam) * B) + plf_align256(sizeof(PlfPairPrm) * B) +
         plf_align256(sizeof(PlfRectPair) * B) + plf_align256(sizeof(uint8_t*) * 2 * B) + plf_align256(sizeof(PlfMaskBuild) * 2 * B);
}
static BatchTab batch_tab(uint8_t* base, int B) {
  uint8_t* cams = base + plf_align256(3 * sizeof(int32_t) * B);
  uint8_t* prm = cams + plf_align256(sizeof(PlfPairCam) * B);
  uint8_t* in = prm + plf_align256(sizeof(PlfPairPrm) * B);
  uint8_t* masks = in + plf_align256(sizeof(PlfRectPair) * B);
  uint8_t* build = masks + plf_align256(sizeof(uint8_t*) * 2 * B);
  return {reinterpret_cast<int32_t*>(base), reinterpret_cast<int32_t*>(base) + B, reinterpret_cast<PlfPairCam*>(cams),
          reinterpret_cast<PlfPairPrm*>(prm), reinterpret_cast<PlfRectPair*>(in), reinterpret_cast<const uint8_t**>(masks),
          reinterpret_cast<PlfMaskBuild*>(build)};
}

// What each sequence carries to its next pair besides its frame slot: the pose prediction (row-major 4x4) and whether it
// came from a good solution (plf_set_motion_model), and the FAST threshold (plf_set_adaptive_fast).  Only the fields of
// the features that are on are kept up to date.
struct SeqRecord {
  double T[16];
  int valid;
  int th;
};

// One image size of the pipeline (plf_set_image_sizes; record 0 is the context's size), built once by pipe_build: its
// row pitch, and ORB and LSD states of its own geometry, tables and tensor maps over buffers that every size shares
// (plf_orb_create_sizes, plf_lsd_create_sizes).  A batch runs every phase with the record of its upload's size.
struct PipeGeo {
  int w = 0, h = 0;
  int pitch = 0;               // row pitch of the device images: plf_pitch16(w) (16-byte rows: every halo tile is a legal TMA box)
  OrbState* orb = nullptr;     // ORB of 2B images, outputs per batch parity
  LsdState* lsd = nullptr;     // LSD of 2B images, hand-off buffers per batch parity if lsd2
  PlfTmaCache lbd_tm;          // tensor maps of the LBD gradient prelude over imgs2
};

struct PipeState {
  int B = 0, max_kp = 0, max_ln = 0;
  std::vector<PipeGeo> geo;    // [1 + plf_ctx::image_sizes / 2], in plf_image_size_index's order
  // Sequences: frame slots 0 .. B-1 hold the pairs of the running batch, B + s carries sequence s's last frame and
  // B + nseq is a slot whose counts stay 0, the "previous frame" of a first frame.
  int nseq = 1;
  std::vector<uint8_t> carried;  // [nseq] sequence s has a frame in its carry slot
  std::vector<int> last_pair;    // [nseq] scratch of plf_batch_run_sequences: the batch's last pair of each sequence, or -1
  std::vector<int> pair_seq;     // [B] scratch of plf_batch_run_sequences: the sequence of each pair of the batch
  // The batch tables (BatchTab), rings indexed like h_results (up to three batches in flight): one pinned block h_tab[rp]
  // per entry, device tab [3][batch_tab_bytes].  The copy goes on the copy stream at the start of the run, in order behind
  // the batch's own images, ahead of its input conversion and of the next batch's upload; ev_tab marks it for the E and M
  // phases.
  uint8_t* h_tab[3] = {nullptr, nullptr, nullptr};
  uint8_t* tab = nullptr;
  cudaEvent_t ev_tab[3] = {nullptr, nullptr, nullptr};
  // Every image buffer holds 2B images of any of the sizes, laid out at that size's h and pitch.
  uint8_t* imgs2[2] = {nullptr, nullptr};  // double-buffered [2B][h][pitch]: upload of batch i+1 overlaps the run of batch i
  uint8_t* stage = nullptr;    // dense [2B][h][w] landing buffer of the H2D copy (one contiguous DMA per side), repacked to the padded pitch on the device
  int up_slot = 0;             // slot written by the last plf_batch_upload
  int up_geo = 0;              // size (geo record) of the last upload
  // channels of the last upload: 1 for plf_batch_upload (its images are in imgs2[up_slot]), 3 or 4 for
  // plf_batch_upload_color (its images are in the colour landing buffer until the run converts them into imgs2[up_slot])
  int up_ch = 1;
  bool uploaded = false;       // an upload was made, or device_images handed out a slot
  cudaStream_t copy = nullptr; // H2D stream
  cudaEvent_t ev_up[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr}, ev_free2[2] = {nullptr, nullptr};
  // Pair masks (plf_batch_upload_masks): mpyr[slot] holds the mask pyramids of images 0 .. 2 max_batch - 1 of the upload
  // in that slot, one every mask_stride(size) bytes (PLF_SCR_MASK_PIPE, carved at the first mask upload).  mask_B pairs of
  // the most recent upload have masks on the sides mask_side (0: none); the run that consumes the upload takes them.
  // ev_mfree[slot]: the KeyLine stage of the last run with pair masks in that slot has read them.
  uint8_t* mpyr[2] = {nullptr, nullptr};
  int mask_B = 0;
  bool mask_side[2] = {false, false};
  cudaEvent_t ev_mfree[2] = {nullptr, nullptr};
  short2* lbd_grad[2] = {nullptr, nullptr};  // [parity][2B][h*w]
  uint8_t* ldesc_raw = nullptr;  // [2B][max_ln][32]  LBD of every kept KeyLine
  FrameSlots fs;               // B + nseq + 1 slots
  // seq_rec[s]: what sequence s's next pair starts from unless that pair is a first frame, written by k_seq_update on the
  // M stream (ev_th marks the thresholds for the next E phase).  img_th = the FAST threshold of each image of the running
  // batch (plf_set_adaptive_fast); pair_T = the prediction of each pair of the running batch (plf_set_motion_model), read
  // by the f2f geometry and, through gn_probs_mm (the pose problems with T_init = pair_T + 16 k), by the pose solver
  SeqRecord* seq_rec = nullptr;   // [nseq]
  int* img_th = nullptr;       // [2B]
  cudaEvent_t ev_th = nullptr;
  double* pair_T = nullptr;    // [B][16]
  GnProblem* gn_probs_mm = nullptr;   // [B]
  // matching scratch
  uint32_t* knn_keys = nullptr;   // [B][8][2][max_kp]
  int32_t* m12 = nullptr;         // [B][4][max_kp]  stereo pts, stereo lines, f2f pts, f2f lines
  int* mcount = nullptr;          // [B][4]
  // match-phase copies of the extraction outputs (taken right after the LBD kernel, so that the extraction buffers of
  // this parity are released to batch i+2 early): keypoints, ORB descriptors, KeyLines and their counts for 2B images
  plf_keypoint* kpsM = nullptr; uint8_t* descM = nullptr; int* kcntM = nullptr;
  plf_keyline* klsM = nullptr; int* lcntM = nullptr;
  KnnProblem* knn_stereo = nullptr;  // [B*4]: [0,2B) forward L->R (points, lines per pair), [2B,4B) reverse R->L on listed rows
  int* rev_flags = nullptr; int* rev_list = nullptr; int* rev_count = nullptr;  // [2B][max_kp], [2B][max_kp], [2B]
  KnnProblem* knn_f2f = nullptr;     // [B*4]
  NnrProblem* nnr_stereo = nullptr;  // [B*2]
  NnrProblem* nnr_f2f = nullptr;     // [B*2]
  // GN inputs / outputs
  double* gnP = nullptr; double* gnObs = nullptr; uint8_t* gnInlP = nullptr; int* gnNp = nullptr;
  double* gn_sP = nullptr; double* gn_eP = nullptr; double* gn_le = nullptr; uint8_t* gnInlL = nullptr; int* gnNl = nullptr;
  GnProblem* gn_probs = nullptr;
  plf_pose_result* gn_out = nullptr;
  plf_frame_result* results = nullptr;                  // [3][B] device, ring indexed like h_results (plf_batch_device_poses reads it)
  plf_frame_result* h_results[3] = {nullptr, nullptr, nullptr};  // pinned host mirrors, ring of PIPE_DEPTH (filled at the end of M)
  int* h_ovf[3] = {nullptr, nullptr, nullptr};                   // pinned overflow flags {orb, lsd}
  int* d_ovf = nullptr;         // [3][2] per-batch snapshots of the two global overflow flags (taken at the end of E and G)
  // windowed matching (plf_params.matching_strategy != 0): grid geometry of the four problem kinds per pair
  // (0 stereo points, 1 stereo lines, 2 f2f points, 3 f2f lines), train-line directions, f2f grid results and counts
  int* mg_q[4] = {nullptr, nullptr, nullptr, nullptr};
  int* mg_t[4] = {nullptr, nullptr, nullptr, nullptr};
  double* mg_dir[2] = {nullptr, nullptr};   // [B][Ln][2]: stereo lines, f2f lines
  int32_t* m12g = nullptr;                  // [B][2][K]  f2f matchGrid results (points, lines)
  int* mgcount = nullptr;                   // [B][2]
  // Batches are software-pipelined over three streams: E (extract: ORB, LSD pre-grow, LBD prelude) -> G (LSD region
  // growing, latency-bound) -> M (LBD, stereo, tracking, pose).  Buffers that cross E -> G -> M exist per batch parity.
  // M starts with the LBD kernel and a device copy of the (small) extraction outputs it still needs, then records evX:
  // from there on batch i+2 may overwrite the parity's extraction buffers, so E(i+2) overlaps the rest of M(i) and
  // G(i+1).  Up to PIPE_DEPTH = 3 batches may be in flight (run, run, run, download, ...).
  cudaEvent_t evE[2] = {nullptr, nullptr}, evG[2] = {nullptr, nullptr}, evX[2] = {nullptr, nullptr};
  cudaEvent_t evP[2] = {nullptr, nullptr};   // end of the LSD pre-grow phase (stream P)
  bool lsd2 = false;            // LSD hand-off buffers exist per batch parity: pre-grow of batch i+1 overlaps the growing of batch i
  cudaEvent_t evM[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t tE0[2] = {nullptr, nullptr}, tG0[2] = {nullptr, nullptr}, tM0[3] = {nullptr, nullptr, nullptr};  // phase starts (timeline)
  long long seq = 0;            // batches issued
  int pend_slot[3] = {0, 0, 0}, pend_B[3] = {0, 0, 0}, n_pending = 0;
  int rp_geo[3] = {0, 0, 0};    // size (geo record) of the batch in each slot of the result ring
  DevBufList bufs;
  // the largest image of any size: pixels w h, and bytes pitch h
  size_t max_area() const { size_t a = 0; for (const PipeGeo& g : geo) a = std::max(a, (size_t)g.w * g.h); return a; }
  size_t max_image() const { size_t a = 0; for (const PipeGeo& g : geo) a = std::max(a, (size_t)g.pitch * g.h); return a; }
};

// The device buffers of the pipeline for B pairs of K keypoints / Ln lines per image.
// Image buffers are sized for the largest image of any size.
static void pipe_buffers(PipeState* s, bool windowed, DevBufList& b) {
  const size_t B = s->B, K = s->max_kp, Ln = s->max_ln, A = s->max_area(), AP = s->max_image();
  const size_t S = B + s->nseq + 1;   // frame slots, carry slots, the empty slot
  b.add(s->imgs2[0], 2 * B * AP);
  b.add(s->imgs2[1], 2 * B * AP);
  bool padded = false;   // a size's rows are padded: its dense uploads land in stage
  for (const PipeGeo& g : s->geo) padded |= g.pitch != g.w;
  if (padded) b.add(s->stage, 2 * B * A);
  b.add(s->lbd_grad[0], 2 * B * A);
  b.add(s->lbd_grad[1], 2 * B * A);
  b.add(s->ldesc_raw, 2 * B * Ln * 32);
  FrameSlots& f = s->fs;
#define PLF_FS_ALLOC(name, T, cap, per) b.add(f.name, S * cap * per);
  PLF_PT_FIELDS(PLF_FS_ALLOC) b.add(f.pt_count, S);
  PLF_LS_FIELDS(PLF_FS_ALLOC) b.add(f.ls_count, S);
#undef PLF_FS_ALLOC
  b.add(s->seq_rec, s->nseq);
  b.add(s->img_th, 2 * B);
  b.add(s->pair_T, B * 16);
  b.add(s->gn_probs_mm, B);
  b.add(s->knn_keys, B * 8 * 2 * K);
  b.add(s->m12, B * 4 * K);
  b.add(s->mcount, B * 4);
  b.add(s->knn_stereo, B * 4); b.add(s->knn_f2f, B * 4);
  b.add(s->nnr_stereo, B * 2); b.add(s->nnr_f2f, B * 2);
  b.add(s->rev_flags, 2 * B * K); b.add(s->rev_list, 2 * B * K); b.add(s->rev_count, 2 * B);
  b.add(s->kpsM, 2 * B * K); b.add(s->descM, 2 * B * K * 32); b.add(s->kcntM, 2 * B);
  b.add(s->klsM, 2 * B * Ln); b.add(s->lcntM, 2 * B);
  b.add(s->gnP, B * K * 3); b.add(s->gnObs, B * K * 2); b.add(s->gnInlP, B * K); b.add(s->gnNp, B);
  b.add(s->gn_sP, B * Ln * 3); b.add(s->gn_eP, B * Ln * 3); b.add(s->gn_le, B * Ln * 3); b.add(s->gnInlL, B * Ln); b.add(s->gnNl, B);
  b.add(s->gn_probs, B); b.add(s->gn_out, B); b.add(s->results, 3 * B);
  b.add(s->d_ovf, 6);
  b.add(s->tab, 3 * batch_tab_bytes(s->B));
  if (windowed) {
    for (int kind = 0; kind < 4; ++kind) {   // points: 2 cells per feature, lines: 2 end points
      b.add(s->mg_q[kind], B * (kind & 1 ? Ln * 4 : K * 2));
      b.add(s->mg_t[kind], B * (kind & 1 ? Ln * 4 : K * 2));
    }
    b.add(s->mg_dir[0], B * Ln * 2); b.add(s->mg_dir[1], B * Ln * 2);
    b.add(s->m12g, B * 2 * K);
    b.add(s->mgcount, B * 2);
  }
}

// Every event of the pipeline: (array, count, creation flags).  plf_debug_timeline reads the timed ones.  evM uses
// blocking sync: a host thread waiting in plf_batch_download sleeps instead of spinning, which matters when several ranks
// share a fraction of a machine's CPUs.
struct PipeEvents { cudaEvent_t* ev; int n; unsigned flags; };
static std::vector<PipeEvents> pipe_events(PipeState* s) {
  return {{s->ev_up, 2, cudaEventDisableTiming}, {s->ev_free, 2, cudaEventDisableTiming}, {s->ev_free2, 2, cudaEventDisableTiming},
          {s->evM, 3, cudaEventBlockingSync},    {s->tM0, 3, cudaEventDefault},           {s->evE, 2, cudaEventDefault},
          {s->evG, 2, cudaEventDefault},         {s->evX, 2, cudaEventDisableTiming},     {s->evP, 2, cudaEventDisableTiming},
          {s->tE0, 2, cudaEventDefault},         {s->tG0, 2, cudaEventDefault},           {s->ev_tab, 3, cudaEventDisableTiming},
          {&s->ev_th, 1, cudaEventDisableTiming}, {s->ev_mfree, 2, cudaEventDisableTiming}};
}

extern "C" void plf_pipe_free(plf_ctx* ctx) {
  PipeState* s = ctx->pipe;
  if (!s) return;
  for (PipeGeo& g : s->geo) {
    plf_orb_free(g.orb);
    plf_lsd_free(g.lsd);
  }
  s->bufs.release();
  for (int i = 0; i < 3; ++i) {
    if (s->h_results[i]) cudaFreeHost(s->h_results[i]);
    if (s->h_ovf[i]) cudaFreeHost(s->h_ovf[i]);
    if (s->h_tab[i]) cudaFreeHost(s->h_tab[i]);
  }
  for (const PipeEvents& a : pipe_events(s))
    for (int i = 0; i < a.n; ++i)
      if (a.ev[i]) cudaEventDestroy(a.ev[i]);
  if (s->copy) { cudaStreamSynchronize(s->copy); cudaStreamDestroy(s->copy); }
  delete s;
  ctx->pipe = nullptr;
}

__device__ __forceinline__ void back_projection(const PlfPairCam& c, double u, double v, double disp, double* P) {
  const double Z = c.fx * c.b / disp;  // PinholeStereoCamera::backProjection (SURVEY A.4)
  P[0] = Z * (u - c.cx) / c.fx;
  P[1] = Z * (v - c.cy) / c.fy;
  P[2] = Z;
}

// block-wide inclusive scan of 0/1 flags (1024 threads); returns inclusive prefix, total in *total
__device__ __forceinline__ int block_scan_flags(bool flag, int* s_scan, int* s_total) {
  const int tid = threadIdx.x;
  s_scan[tid] = flag ? 1 : 0;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const int v = tid >= off ? s_scan[tid - off] : 0;
    __syncthreads();
    s_scan[tid] += v;
    __syncthreads();
  }
  const int incl = s_scan[tid];
  if (tid == 1023) *s_total = incl;
  __syncthreads();
  return incl;
}

// matchStereoPoints: epipolar + disparity gates, back-projection, compaction in left-index order, with pair k's camera
// cams[k] and gates prm[k].
__global__ void __launch_bounds__(1024) k_stereo_points(const plf_keypoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                                         const int* __restrict__ kp_count, int max_kp,
                                                         const int32_t* __restrict__ m12_all, int m12_stride,
                                                         const PlfPairCam* __restrict__ cams, const PlfPairPrm* __restrict__ prm,
                                                         FrameSlots fs) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int il = 2 * k, ir = 2 * k + 1, slot = k;
  const PlfPairCam cam = cams[k];
  const PlfPairPrm& q = prm[k];
  const plf_keypoint* kl = kps + (size_t)il * max_kp;
  const plf_keypoint* kr = kps + (size_t)ir * max_kp;
  const int32_t* m12 = m12_all + (size_t)k * m12_stride;
  const int n = min(kp_count[il], max_kp);
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    bool ok = false;
    float xl = 0, yl = 0;
    double d = 0;
    int oct = 0;
    if (i < n) {
      const int j = m12[i];
      if (j >= 0) {
        const plf_keypoint a = kl[i], b = kr[j];
        xl = a.x; yl = a.y; oct = a.octave;
        if (fabsf(__fsub_rn(a.y, b.y)) <= q.max_dist_epip) {
          d = (double)__fsub_rn(a.x, b.x);
          ok = d >= (double)q.min_disp;
        }
      }
    }
    const int incl = block_scan_flags(ok, s_scan, &s_total);
    if (ok) {
      const size_t o = (size_t)slot * max_kp + base + incl - 1;
      fs.pt_pl[o] = make_double2((double)xl, (double)yl);
      fs.pt_disp[o] = d;
      back_projection(cam, (double)xl, (double)yl, d, fs.pt_P + 3 * o);
      fs.pt_octave[o] = oct;
      const uint4* src = reinterpret_cast<const uint4*>(desc + ((size_t)il * max_kp + i) * 32);
      uint4* dst = reinterpret_cast<uint4*>(fs.pdesc + o * 32);
      dst[0] = src[0];
      dst[1] = src[1];
    }
    base += s_total;
    __syncthreads();
  }
  if (tid == 0) fs.pt_count[slot] = base;
}

__device__ __forceinline__ double line_overlap_stereo(double spl_obs, double epl_obs, double spl_proj, double epl_proj,
                                                      double line_horiz_th) {
  double overlap = 1.0;
  if (fabs(epl_obs - spl_obs) > line_horiz_th) {
    const double sln = fmin(spl_obs, epl_obs), eln = fmax(spl_obs, epl_obs);
    const double spn = fmin(spl_proj, epl_proj), epn = fmax(spl_proj, epl_proj);
    const double length = eln - spn;
    if (epn < sln || spn > eln) overlap = 0.0;
    else if (epn > eln && spn < sln) overlap = eln - sln;
    else overlap = fmin(eln, epn) - fmax(sln, spn);
    overlap = (length > (double)0.01f) ? overlap / length : 0.0;
    if (overlap > 1.0) overlap = 1.0;
  }
  return overlap;
}

// matchStereoLines (camera and gates: as k_stereo_points)
__global__ void __launch_bounds__(1024) k_stereo_lines(const plf_keyline* __restrict__ kls, const uint8_t* __restrict__ ldesc,
                                                        const int* __restrict__ nlines, int max_ln,
                                                        const int32_t* __restrict__ m12_all, int m12_stride,
                                                        const PlfPairCam* __restrict__ cams, const PlfPairPrm* __restrict__ prm,
                                                        FrameSlots fs) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int il = 2 * k, ir = 2 * k + 1, slot = k;
  const PlfPairCam cam = cams[k];
  const PlfPairPrm& q = prm[k];
  const plf_keyline* L = kls + (size_t)il * max_ln;
  const plf_keyline* R = kls + (size_t)ir * max_ln;
  const int32_t* m12 = m12_all + (size_t)k * m12_stride;
  const int n = min(nlines[il], max_ln);
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + tid;
    bool ok = false;
    double spl[2] = {0, 0}, epl[2] = {0, 0}, le_l[3] = {0, 0, 0}, disp_s = 0, disp_e = 0;
    float angle = 0;
    if (i < n) {
      const int j = m12[i];
      if (j >= 0) {
        const plf_keyline a = L[i], b = R[j];
        const double sxl = a.startPointX, syl = a.startPointY, exl = a.endPointX, eyl = a.endPointY;
        const double sxr = b.startPointX, syr = b.startPointY, exr = b.endPointX, eyr = b.endPointY;
        // le = sp x ep with homogeneous 1
        double l0 = syl * 1.0 - 1.0 * eyl, l1 = 1.0 * exl - sxl * 1.0, l2 = sxl * eyl - syl * exl;
        const double nrm = sqrt(l0 * l0 + l1 * l1);
        le_l[0] = l0 / nrm; le_l[1] = l1 / nrm; le_l[2] = l2 / nrm;
        const double r0 = syr * 1.0 - 1.0 * eyr, r1 = 1.0 * exr - sxr * 1.0, r2 = sxr * eyr - syr * exr;
        const double overlap = line_overlap_stereo(syl, eyl, syr, eyr, (double)q.line_horiz_th);
        const double sx_on_r = -(r2 + r1 * syl) / r0;
        const double ex_on_r = -(r2 + r1 * eyl) / r0;
        disp_s = sxl - sx_on_r;
        disp_e = exl - ex_on_r;
        if (!(fmin(disp_s, disp_e) / fmax(disp_s, disp_e) >= (double)q.ls_min_disp_ratio)) disp_s = disp_e = -1.0;
        ok = disp_s >= (double)q.min_disp && disp_e >= (double)q.min_disp &&
             fabsf((float)r0) > q.line_horiz_th && overlap > (double)q.stereo_overlap_th;
        spl[0] = sxl; spl[1] = syl; epl[0] = exl; epl[1] = eyl;
        angle = a.angle;
      }
    }
    const int incl = block_scan_flags(ok, s_scan, &s_total);
    if (ok) {
      const size_t o = (size_t)slot * max_ln + base + incl - 1;
      fs.ls_spl[o] = make_double2(spl[0], spl[1]);
      fs.ls_epl[o] = make_double2(epl[0], epl[1]);
      fs.ls_sdisp[o] = disp_s;
      fs.ls_edisp[o] = disp_e;
      back_projection(cam, spl[0], spl[1], disp_s, fs.ls_sP + 3 * o);
      back_projection(cam, epl[0], epl[1], disp_e, fs.ls_eP + 3 * o);
      fs.ls_le[3 * o] = le_l[0]; fs.ls_le[3 * o + 1] = le_l[1]; fs.ls_le[3 * o + 2] = le_l[2];
      fs.ls_angle[o] = angle;
      const uint4* src = reinterpret_cast<const uint4*>(ldesc + ((size_t)il * max_ln + i) * 32);
      uint4* dst = reinterpret_cast<uint4*>(fs.ldesc + o * 32);
      dst[0] = src[0];
      dst[1] = src[1];
    }
    base += s_total;
    __syncthreads();
  }
  if (tid == 0) fs.ls_count[slot] = base;
}

// The matching problems of pair k that depend on the batch, with its ratios and best_lr from prm[k].  f2fTracking: the
// previous frame (slot prev[k]) against the current one (slot k), 2-NN both ways for points and lines, then the mutual NNR
// check; the forward best / second keys of problem kind c (4 = points, 6 = lines) and the reverse ones (c + 1) live in the
// pair's knn_keys rows.  Stereo: the NNR check of the static kNN problems (pipe_build) over the left (kinds 0, 2) and right
// (1, 3) images' counts kcnt, lcnt.  A windowed pair (matching_strategy != 0) gets its stereo matches from the windowed
// matcher: its stereo problems read their query count at zero, an int that stays 0, so they write no row.
__global__ void k_f2f_problems(FrameSlots fs, const int* __restrict__ prev, int B, int K, int Ln, uint32_t* __restrict__ knn_keys,
                               int32_t* __restrict__ m12, int* __restrict__ mcount, const int* kcnt, const int* lcnt,
                               const int* zero, const PlfPairPrm* __restrict__ prm, KnnProblem* __restrict__ kf,
                               NnrProblem* __restrict__ nf, NnrProblem* __restrict__ ns) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= B) return;
  const PlfPairPrm& q = prm[k];
  const int ps = prev[k], cs = k;
  auto key = [&](int prob, int which) { return knn_keys + (((size_t)k * 8 + prob) * 2 + which) * K; };
  const uint32_t* pp = (const uint32_t*)(fs.pdesc + (size_t)ps * K * 32);
  const uint32_t* pc = (const uint32_t*)(fs.pdesc + (size_t)cs * K * 32);
  const uint32_t* lp = (const uint32_t*)(fs.ldesc + (size_t)ps * Ln * 32);
  const uint32_t* lc = (const uint32_t*)(fs.ldesc + (size_t)cs * Ln * 32);
  const int *np = fs.pt_count + ps, *nc = fs.pt_count + cs, *lnp = fs.ls_count + ps, *lnc = fs.ls_count + cs;
  kf[4 * k + 0] = KnnProblem{pp, pc, np, nc, 0, 0, key(4, 0), key(4, 1), nullptr};
  kf[4 * k + 1] = KnnProblem{pc, pp, nc, np, 0, 0, key(5, 0), key(5, 1), nullptr};
  kf[4 * k + 2] = KnnProblem{lp, lc, lnp, lnc, 0, 0, key(6, 0), key(6, 1), nullptr};
  kf[4 * k + 3] = KnnProblem{lc, lp, lnc, lnp, 0, 0, key(7, 0), key(7, 1), nullptr};
  nf[2 * k + 0] = NnrProblem{key(4, 0), key(4, 1), key(5, 0), key(5, 1), np, nc, 0, 0, q.min_ratio_12_p, q.best_lr,
                             m12 + ((size_t)k * 4 + 2) * K, mcount + 4 * k + 2};
  nf[2 * k + 1] = NnrProblem{key(6, 0), key(6, 1), key(7, 0), key(7, 1), lnp, lnc, 0, 0, q.min_ratio_12_l, q.best_lr,
                             m12 + ((size_t)k * 4 + 3) * K, mcount + 4 * k + 3};
  ns[2 * k + 0] = NnrProblem{key(0, 0), key(0, 1), key(1, 0), key(1, 1), q.matching_strategy ? zero : kcnt + 2 * k, kcnt + 2 * k + 1,
                             0, 0, q.min_ratio_12_p, q.best_lr, m12 + (size_t)k * 4 * K, mcount + 4 * k};
  ns[2 * k + 1] = NnrProblem{key(2, 0), key(2, 1), key(3, 0), key(3, 1), q.matching_strategy ? zero : lcnt + 2 * k, lcnt + 2 * k + 1,
                             0, 0, q.min_ratio_12_l, q.best_lr, m12 + ((size_t)k * 4 + 1) * K, mcount + 4 * k + 1};
}

// Copies `rows` rows of row_bytes (a multiple of 4) from slot `from` to slot `to` of an array of `cap` rows per slot.
__device__ __forceinline__ void carry_rows(void* base, size_t row_bytes, size_t cap, int from, int to, int rows) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(base) + (size_t)from * cap * row_bytes);
  uint32_t* dst = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(base) + (size_t)to * cap * row_bytes);
  const size_t words = (size_t)rows * row_bytes / 4;
  for (size_t i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
}

// Carries the batch's last frame of each sequence to its carry slot: block (field, j) copies the stereo-valid rows of one
// FrameSlots array for carry[j] = (frame slot, carry slot); the counts go with the first field.
__global__ void __launch_bounds__(256) k_carry(FrameSlots fs, const int* __restrict__ carry, int K, int Ln) {
  const int from = carry[2 * blockIdx.y], to = carry[2 * blockIdx.y + 1];
  const int np = fs.pt_count[from], nl = fs.ls_count[from];
  const int field = blockIdx.x;
  if (field == 0 && threadIdx.x == 0) { fs.pt_count[to] = np; fs.ls_count[to] = nl; }
  int f = 0;
#define PLF_PT_CARRY(name, T, cap, per) if (field == f++) carry_rows(fs.name, sizeof(T) * (per), (size_t)(cap), from, to, min(np, cap));
#define PLF_LS_CARRY(name, T, cap, per) if (field == f++) carry_rows(fs.name, sizeof(T) * (per), (size_t)(cap), from, to, min(nl, cap));
  PLF_PT_FIELDS(PLF_PT_CARRY)
  PLF_LS_FIELDS(PLF_LS_CARRY)
#undef PLF_LS_CARRY
#undef PLF_PT_CARRY
}

// f2fTracking: gather the matched rows into the GN problem of pair k (previous frame: slot prev[k], current: slot k)
__global__ void __launch_bounds__(1024) k_f2f_build(FrameSlots fs, const int* __restrict__ prev, int max_kp, int max_ln,
                                                    const int32_t* __restrict__ m_pt_all, const int32_t* __restrict__ m_ls_all,
                                                    int m_stride, double* __restrict__ gnP, double* __restrict__ gnObs,
                                                    uint8_t* __restrict__ gnInlP, int* __restrict__ gnNp,
                                                    double* __restrict__ gn_sP, double* __restrict__ gn_eP,
                                                    double* __restrict__ gn_le, uint8_t* __restrict__ gnInlL,
                                                    int* __restrict__ gnNl) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int ps = prev[k], cs = k;
  {  // points
    const int32_t* m = m_pt_all + (size_t)k * m_stride;
    const int n = min(fs.pt_count[ps], max_kp);
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += 1024) {
      const int i = c0 + tid;
      const int j = i < n ? m[i] : -1;
      const bool ok = j >= 0;
      const int incl = block_scan_flags(ok, s_scan, &s_total);
      if (ok) {
        const size_t o = (size_t)k * max_kp + base + incl - 1;
        const double* P = fs.pt_P + 3 * ((size_t)ps * max_kp + i);
        gnP[3 * o] = P[0]; gnP[3 * o + 1] = P[1]; gnP[3 * o + 2] = P[2];
        const double2 q = fs.pt_pl[(size_t)cs * max_kp + j];
        gnObs[2 * o] = q.x; gnObs[2 * o + 1] = q.y;
        gnInlP[o] = 1;
      }
      base += s_total;
      __syncthreads();
    }
    if (tid == 0) gnNp[k] = base;
  }
  {  // lines
    const int32_t* m = m_ls_all + (size_t)k * m_stride;
    const int n = min(fs.ls_count[ps], max_ln);
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += 1024) {
      const int i = c0 + tid;
      const int j = i < n ? m[i] : -1;
      const bool ok = j >= 0;
      const int incl = block_scan_flags(ok, s_scan, &s_total);
      if (ok) {
        const size_t o = (size_t)k * max_ln + base + incl - 1;
        const size_t pi = (size_t)ps * max_ln + i, ci = (size_t)cs * max_ln + j;
        for (int c = 0; c < 3; ++c) {
          gn_sP[3 * o + c] = fs.ls_sP[3 * pi + c];
          gn_eP[3 * o + c] = fs.ls_eP[3 * pi + c];
          gn_le[3 * o + c] = fs.ls_le[3 * ci + c];
        }
        gnInlL[o] = 1;
      }
      base += s_total;
      __syncthreads();
    }
    if (tid == 0) gnNl[k] = base;
  }
}

// optimizePose epilogue: curr.DT = inverse_se3(T_inc); identity when there were too few correspondences; a pair whose
// previous frame is the empty slot is a first frame (initialize())
__global__ void k_finalize(const plf_pose_result* __restrict__ gn, const int* __restrict__ gnNp, const int* __restrict__ gnNl,
                           const int* __restrict__ kp_count, const int* __restrict__ nlines, FrameSlots fs,
                           const int* __restrict__ prev, int empty_slot, int B, plf_frame_result* __restrict__ out,
                           const PlfPairPrm* __restrict__ prm) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= B) return;
  const int min_features = prm[k].min_features;
  plf_frame_result r;
  for (int i = 0; i < 16; ++i) r.DT[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 36; ++i) r.DT_cov[i] = 0.0;
  r.err = -1.0;
  r.n_kp_l = kp_count[2 * k]; r.n_kp_r = kp_count[2 * k + 1];
  r.n_lines_l = nlines[2 * k]; r.n_lines_r = nlines[2 * k + 1];
  r.n_stereo_pt = fs.pt_count[k]; r.n_stereo_ls = fs.ls_count[k];
  r.n_matched_pt = r.n_matched_ls = r.n_inliers_pt = r.n_inliers_ls = r.iters1 = r.iters2 = 0;
  if (prev[k] == empty_slot) {
    r.status = 2;
  } else {
    const plf_pose_result& g = gn[k];
    r.n_matched_pt = gnNp[k]; r.n_matched_ls = gnNl[k];
    if (r.n_matched_pt + r.n_matched_ls < min_features) {
      r.status = 1;
    } else {
      r.status = 0;
      d_inverse_se3(g.T, r.DT);
      for (int i = 0; i < 36; ++i) r.DT_cov[i] = g.cov[i];
      r.err = g.err;
      r.n_inliers_pt = g.n_inliers_pt; r.n_inliers_ls = g.n_inliers_ls;
      r.iters1 = g.iters1; r.iters2 = g.iters2;
    }
  }
  out[k] = r;
}

// ---- what each sequence carries to its next pair: adaptative_fast (plf_set_adaptive_fast) and use_motion_model
// (plf_set_motion_model), DESIGN.md §8.  With either on a batch holds at most one pair of each sequence, so prev[k] is the
// empty slot (a first frame) or pair k's carry slot carry0 + s, and every pair is in the carry list. ----

// The FAST threshold of both images of pair k: its sequence's, or its settings' first-frame one for a first frame.
__global__ void k_fast_th_images(const int* __restrict__ prev, int B, int carry0, int empty, const SeqRecord* __restrict__ rec,
                                 const PlfPairPrm* __restrict__ prm, int* __restrict__ img_th) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= B) return;
  const int p = prev[k];
  const int th = p != empty ? rec[p - carry0].th : prm[k].fast_th;
  img_th[2 * k] = th;
  img_th[2 * k + 1] = th;
}

// StereoFrameHandler::updateFrame's threshold step after pair k, detected at th with result r.  stvo-pl goes on with
// "else if n_inliers_pt > 4 feat_th: th + 2 inc_th", which the "> 3 feat_th" test before it leaves unreachable.
__device__ __forceinline__ int fast_th_next(int th, const plf_frame_result& r, const plf_adaptive_fast& a) {
  if (r.status == 2) return th;   // initialize() runs no updateFrame
  bool ident = true;
  for (int i = 0; i < 16; ++i) ident &= r.DT[i] == ((i % 5 == 0) ? 1.0 : 0.0);
  const long long n = r.n_inliers_pt, f = a.feat_th, t = th;
  if (ident || r.err > a.err_th || n < f) return (int)max((long long)a.min_th, t - 2ll * a.inc_th);
  if (n < 2 * f) return (int)max((long long)a.min_th, t - a.inc_th);
  if (n > 3 * f) return (int)min((long long)a.max_th, t + a.inc_th);
  return th;
}

PlfPairPrm plf_pair_prm(const plf_params& P) {
  PlfPairPrm q = {};
  q.orb_nlevels = P.orb_nlevels;
  if (P.orb_nlevels >= 1 && P.orb_nlevels <= PLF_ORB_MAX_LEVELS)
    plf_orb_level_features(P.orb_nfeatures, P.orb_scale_factor, P.orb_nlevels, q.orb_nfeat);
  q.fast_th = std::min(std::max(P.orb_fast_th, 0), 255);
  q.lsd_nfeatures = P.lsd_nfeatures;
  q.min_line_length = P.min_line_length;
  q.max_dist_epip = P.max_dist_epip; q.min_disp = P.min_disp; q.line_horiz_th = P.line_horiz_th;
  q.stereo_overlap_th = P.stereo_overlap_th; q.ls_min_disp_ratio = P.ls_min_disp_ratio;
  q.min_ratio_12_p = P.min_ratio_12_p; q.min_ratio_12_l = P.min_ratio_12_l; q.line_sim_th = P.line_sim_th;
  q.best_lr = P.best_lr_matches ? 1 : 0;
  q.matching_strategy = P.matching_strategy; q.matching_s_ws = P.matching_s_ws; q.matching_f2f_ws = P.matching_f2f_ws;
  q.min_pt_matches = P.min_pt_matches; q.min_ls_matches = P.min_ls_matches; q.min_features = P.min_features;
  q.gn = plf_gn_opts_from_params(P);
  return q;
}

// stvo-pl's isGoodSolution on a pair's result, each of its tests a rejection: so a NaN err or eigenvalue passes.  A
// covariance with a non-finite entry has NaN eigenvalues (the library's definition; the solver gives such a covariance
// whole, e.g. on rows at infinity).
__device__ __forceinline__ bool motion_good(int status, const double* DT, const double* cov, double err) {
  if (status != 0) return false;
  for (int i = 0; i < 16; ++i)
    if (!isfinite(DT[i])) return false;
  if (err < 0.0 || err > 1.0) return false;
  for (int i = 0; i < 36; ++i)
    if (!isfinite(cov[i])) return true;
  double A[36];
  plf_sym6_jacobi(cov, A);
  double lo = A[0], hi = A[0];
  for (int i = 1; i < 6; ++i) {
    lo = A[7 * i] < lo ? A[7 * i] : lo;
    hi = A[7 * i] > hi ? A[7 * i] : hi;
  }
  return !(lo < 0.0 || hi > 1.0);
}

// The prediction a pair's result gives its sequence's next pair: the optimiser's transform inverse_se3(DT) (previous frame
// into current) after a good solution, else the identity.  Returns the valid flag.
__device__ __forceinline__ int motion_prior(int status, const double* DT, const double* cov, double err, double* T) {
  const bool good = motion_good(status, DT, cov, err);
  if (good) d_inverse_se3(DT, T);
  else
    for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  return good ? 1 : 0;
}

// Carry entry j = (pair k, carry slot carry0 + s): sequence s's record from pair k's result, its next threshold (img_th
// set: adaptive FAST, from the threshold pair k was detected at) and its next prediction (motion set).
__global__ void k_seq_update(const plf_frame_result* __restrict__ res, const int* __restrict__ carry, int ncarry, int carry0,
                             const int* __restrict__ img_th, plf_adaptive_fast a, int motion, SeqRecord* __restrict__ rec) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ncarry) return;
  const int k = carry[2 * j];
  const plf_frame_result& r = res[k];
  SeqRecord& q = rec[carry[2 * j + 1] - carry0];
  if (img_th) q.th = fast_th_next(img_th[2 * k], r, a);
  if (motion) q.valid = motion_prior(r.status, r.DT, r.DT_cov, r.err, q.T);
}

// Block k, thread i: entry i of pair k's prediction, its sequence's or the identity for a first frame.
__global__ void k_motion_pairs(const int* __restrict__ prev, int carry0, int empty, const SeqRecord* __restrict__ rec,
                               double* __restrict__ pair_T) {
  const int k = blockIdx.x, i = threadIdx.x, p = prev[k];
  pair_T[16 * k + i] = p == empty ? ((i % 5 == 0) ? 1.0 : 0.0) : rec[p - carry0].T[i];
}

// plf_debug_motion_prior: the rule on n caller results.
__global__ void k_motion_debug(int n, const double* __restrict__ DT, const double* __restrict__ cov, const double* __restrict__ err,
                               const int32_t* __restrict__ status, double* __restrict__ T, int32_t* __restrict__ valid) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  valid[j] = motion_prior(status[j], DT + 16 * (size_t)j, cov + 36 * (size_t)j, err[j], T + 16 * (size_t)j);
}

// Every sequence's record back to a first frame's, in the fields of the features named (no batch in flight): the
// threshold to orb_fast_th, the prediction to the identity (not valid).  The fields T, valid, th are contiguous, so the
// named ones are one column range of the record array.
static plf_status pipe_seq_reset(plf_ctx* ctx, bool fast_th, bool motion) {
  PipeState* s = ctx->pipe;
  SeqRecord r = {};
  for (int i = 0; i < 16; i += 5) r.T[i] = 1.0;
  r.th = ctx->pair.fast_th;
  const std::vector<SeqRecord> v(s->nseq, r);
  const size_t lo = motion ? 0 : offsetof(SeqRecord, th), hi = fast_th ? sizeof(SeqRecord) : offsetof(SeqRecord, th);
  if (lo >= hi) return PLF_OK;
  PLF_CUDA(ctx, cudaMemcpy2DAsync(reinterpret_cast<uint8_t*>(s->seq_rec) + lo, sizeof(SeqRecord),
                                  reinterpret_cast<const uint8_t*>(v.data()) + lo, sizeof(SeqRecord), hi - lo, v.size(),
                                  cudaMemcpyHostToDevice, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// Sequence s's record, behind the updates of every batch in flight (M stream).
static plf_status pipe_seq_read(plf_ctx* ctx, int s, SeqRecord* out) {
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  PLF_CUDA(ctx, cudaMemcpyAsync(out, ctx->pipe->seq_rec + s, sizeof(SeqRecord), cudaMemcpyDeviceToHost, ctx->stream));
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

// ---- windowed matching: grid geometry on the device (oracle/frontend.py grid_match_points / grid_match_lines) ----
// (cells and projection: plf_geom.cuh)

// stereo: queries = left key points / KeyLines of pair k (image 2k), train = the right ones (image 2k+1)
__global__ void __launch_bounds__(256) k_mg_geom_stereo(const plf_keypoint* __restrict__ kps, const int* __restrict__ kcnt, int K,
                                                        const plf_keyline* __restrict__ kls, const int* __restrict__ lcnt, int Ln,
                                                        double iw, double ih, int* __restrict__ qp, int* __restrict__ tp,
                                                        int* __restrict__ ql, int* __restrict__ tl, double* __restrict__ tdir) {
  const int img = blockIdx.y, k = img >> 1, right = img & 1, i = blockIdx.x * 256 + threadIdx.x;
  if (i < min(kcnt[img], K)) {
    const plf_keypoint kp = kps[(size_t)img * K + i];
    int* d = (right ? tp : qp) + ((size_t)k * K + i) * 2;
    d[0] = mg_cell((double)kp.x * iw);
    d[1] = mg_cell((double)kp.y * ih);
  }
  if (i < min(lcnt[img], Ln)) {
    const plf_keyline kl = kls[(size_t)img * Ln + i];
    const double sx = kl.startPointX, sy = kl.startPointY, ex = kl.endPointX, ey = kl.endPointY;
    int* d = (right ? tl : ql) + ((size_t)k * Ln + i) * 4;
    d[0] = mg_cell(sx * iw); d[1] = mg_cell(sy * ih); d[2] = mg_cell(ex * iw); d[3] = mg_cell(ey * ih);
    if (right) {
      const double vx = (ex - sx) * iw, vy = (ey - sy) * ih, nrm = sqrt(vx * vx + vy * vy);
      tdir[((size_t)k * Ln + i) * 2] = vx / nrm;        // unguarded like the reference's normalize()
      tdir[((size_t)k * Ln + i) * 2 + 1] = vy / nrm;
    }
  }
}

// frame-to-frame: queries = the previous frame's 3-D features (slot prev[k]) projected with DT = identity, or through pair
// k's motion prediction T_pred[k] with the motion model on (src/mapHandler.cpp:254-256, :384-389 project through DT);
// train = the current frame's image features (slot k).  The projection uses pair k's camera: both frames belong to one
// sequence, and a new camera restarts its sequence, so the previous frame was triangulated with the same one.
__global__ void __launch_bounds__(256) k_mg_geom_f2f(FrameSlots fs, const int* __restrict__ prev, int K, int Ln,
                                                     const PlfPairCam* __restrict__ cams, const double* __restrict__ T_pred,
                                                     double iw, double ih, int* __restrict__ qp, int* __restrict__ tp,
                                                     int* __restrict__ ql, int* __restrict__ tl, double* __restrict__ tdir) {
  const int k = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  const int ps = prev[k], cs = k;
  const PlfPairCam c = cams[k];
  const double* T = T_pred ? T_pred + 16 * k : nullptr;
  // the query point X of the previous frame, moved into the current frame when there is a prediction
  auto moved = [&](const double* X, double* Y) -> const double* {
    if (!T) return X;
    d_transform(T, X, Y);
    return Y;
  };
  if (i < min(fs.pt_count[ps], K)) {
    double Q[3];
    const double* P = moved(fs.pt_P + 3 * ((size_t)ps * K + i), Q);
    const double2 u = plf_project(c.fx, c.fy, c.cx, c.cy, P[0], P[1], P[2]);
    qp[((size_t)k * K + i) * 2] = plf_qcell(u.x * iw);
    qp[((size_t)k * K + i) * 2 + 1] = plf_qcell(u.y * ih);
  }
  if (i < min(fs.pt_count[cs], K)) {
    const double2 p = fs.pt_pl[(size_t)cs * K + i];
    tp[((size_t)k * K + i) * 2] = mg_cell(p.x * iw);
    tp[((size_t)k * K + i) * 2 + 1] = mg_cell(p.y * ih);
  }
  if (i < min(fs.ls_count[ps], Ln)) {
    double QS[3], QE[3];
    const double* S = moved(fs.ls_sP + 3 * ((size_t)ps * Ln + i), QS);
    const double* E = moved(fs.ls_eP + 3 * ((size_t)ps * Ln + i), QE);
    int* d = ql + ((size_t)k * Ln + i) * 4;
    d[0] = plf_qcell(plf_project_u(c.fx, c.cx, S[0], S[2]) * iw); d[1] = plf_qcell(plf_project_v(c.fy, c.cy, S[1], S[2]) * ih);
    d[2] = plf_qcell(plf_project_u(c.fx, c.cx, E[0], E[2]) * iw); d[3] = plf_qcell(plf_project_v(c.fy, c.cy, E[1], E[2]) * ih);
  }
  if (i < min(fs.ls_count[cs], Ln))
    plf_train_line(fs.ls_spl[(size_t)cs * Ln + i], fs.ls_epl[(size_t)cs * Ln + i], iw, ih, tl + ((size_t)k * Ln + i) * 4,
                   tdir + ((size_t)k * Ln + i) * 2);
}

// src/mapHandler.cpp:274-278 / :421-425: keep the windowed result unless both frames hold more than `kmin` features and
// fewer than `kmin` matches survived - then the brute-force match() result (already in m12) stands.  kmin is the pair's
// min_pt_matches / min_ls_matches, and a pair at matching_strategy 0 keeps its match() result.
__global__ void __launch_bounds__(256) k_mg_select(const int32_t* __restrict__ m12g, const int* __restrict__ mgcount,
                                                   const int* __restrict__ cnt, const int* __restrict__ prev, int cap, int K,
                                                   int which, int32_t* __restrict__ m12, const PlfPairPrm* __restrict__ prm) {
  const int k = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  if (!prm[k].matching_strategy) return;
  const int kmin = which ? prm[k].min_ls_matches : prm[k].min_pt_matches;
  const int n1 = min(cnt[prev[k]], cap), n2 = min(cnt[k], cap);
  if (i >= n1) return;
  const bool fall_back = n2 > kmin && n1 > kmin && mgcount[2 * k + which] < kmin;
  if (!fall_back) m12[((size_t)k * 4 + 2 + which) * K + i] = m12g[((size_t)k * 2 + which) * K + i];
}

// The LSD hand-off maps (8-byte record and seed order: 12 bytes per scaled pixel) exist once or per batch parity.  Per
// parity the pre-grow chain of batch i+1 (blur, resample, gradient, seed ordering) runs on its own stream while batch i is
// still growing regions, which takes the pre-grow kernels off the LSD chain.  The second copy costs 12 bytes per scaled
// pixel of every image of a batch (about 16 MB per KITTI-shape pair); it is made whenever it fits the free device memory
// with LSD_PARITY_MARGIN to spare.  PLF_LSD_PARITIES = 1 or 2 forces either layout.
#define LSD_PARITY_MARGIN (4ull << 30)   // room left for what is allocated after the pipeline is prepared (the standalone
                                         // operators' scratch, the caller's own buffers) and for allocation granularity
// (the footprint of every image size's LSD state: one set of buffers, each the largest any size needs)
static bool lsd_want_two_parities(const plf_ctx* ctx, int n, const int* wh, int nimg) {
  const char* e = getenv("PLF_LSD_PARITIES");
  if (e && *e) return atoi(e) >= 2;
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return plf_lsd_footprint(ctx, n, wh, nimg, true) + LSD_PARITY_MARGIN <= free_b;
}

static plf_status pipe_build(plf_ctx* ctx) {
  PipeState* s = ctx->pipe = new PipeState();
  const int B = ctx->limits.max_batch, K = ctx->limits.max_keypoints, Ln = ctx->limits.max_lines;
  if (Ln > K || K > 65535)
    return plf_fail(ctx, PLF_ERR_INVALID, "limits: need max_lines <= max_keypoints <= 65535 (got %d, %d)", Ln, K);
  s->B = B; s->max_kp = K; s->max_ln = Ln;
  std::vector<int> wh = {ctx->cam.width, ctx->cam.height};   // the sizes, in plf_image_size_index's order
  wh.insert(wh.end(), ctx->image_sizes.begin(), ctx->image_sizes.end());
  const int ngeo = (int)wh.size() / 2;
  s->geo.resize(ngeo);
  for (int i = 0; i < ngeo; ++i) {
    s->geo[i].w = wh[2 * i]; s->geo[i].h = wh[2 * i + 1];
    s->geo[i].pitch = plf_pitch16(wh[2 * i]);
  }
  s->nseq = ctx->max_sequences;
  s->carried.assign(s->nseq, 0);
  s->last_pair.assign(s->nseq, -1);
  const plf_params& P = ctx->params;
  pipe_buffers(s, P.matching_strategy != 0, s->bufs);
  plf_status st = s->bufs.alloc(ctx, "pipeline");
  if (st) return st;
  PLF_CUDA(ctx, cudaStreamCreateWithFlags(&s->copy, cudaStreamNonBlocking));
  for (const PipeEvents& a : pipe_events(s))
    for (int i = 0; i < a.n; ++i) PLF_CUDA(ctx, cudaEventCreateWithFlags(&a.ev[i], a.flags));
  for (int i = 0; i < 3; ++i) {
    PLF_CUDA(ctx, cudaHostAlloc(&s->h_results[i], sizeof(plf_frame_result) * B, cudaHostAllocDefault));
    PLF_CUDA(ctx, cudaHostAlloc(&s->h_ovf[i], 2 * sizeof(int), cudaHostAllocDefault));
    PLF_CUDA(ctx, cudaHostAlloc(&s->h_tab[i], batch_tab_bytes(B), cudaHostAllocDefault));
  }
  FrameSlots& f = s->fs;
  cudaStream_t cs = ctx->stream;
  const size_t nslots = (size_t)B + s->nseq + 1;   // the empty slot's counts stay 0 from here on
  PLF_CUDA(ctx, cudaMemsetAsync(f.pt_count, 0, nslots * sizeof(int), cs));
  PLF_CUDA(ctx, cudaMemsetAsync(f.ls_count, 0, nslots * sizeof(int), cs));
  // sub-systems sized for 2B images; the LSD tables come first, so that the parity decision sees the memory they take
  std::vector<OrbState*> orb(ngeo, nullptr);
  std::vector<LsdState*> lsd(ngeo, nullptr);
  if ((st = plf_orb_create_sizes(ctx, ngeo, wh.data(), 2 * B, true, orb.data()))) return st;
  for (int i = 0; i < ngeo; ++i) s->geo[i].orb = orb[i];
  if ((st = plf_lsd_tables(ctx))) return st;
  s->lsd2 = lsd_want_two_parities(ctx, ngeo, wh.data(), 2 * B);
  if ((st = plf_lsd_create_sizes(ctx, ngeo, wh.data(), 2 * B, s->lsd2, lsd.data()))) return st;
  for (int i = 0; i < ngeo; ++i) s->geo[i].lsd = lsd[i];
  // static problem descriptors over the pipeline's own buffers (pointers never change; counts are read on the device):
  // the stereo problems read the match phase's copies of the extraction outputs.  The NNR problems depend on the batch's
  // sequence table and settings and are built on the device per batch (k_f2f_problems).
  const int* kcnt = s->kcntM;
  const int* lcnt = s->lcntM;
  std::vector<KnnProblem> ks(B * 4);
  std::vector<GnProblem> gp(B);
  for (int k = 0; k < B; ++k) {
    auto key = [&](int prob, int which) { return s->knn_keys + (((size_t)k * 8 + prob) * 2 + which) * K; };
    const uint32_t* dl = (const uint32_t*)(s->descM + (size_t)(2 * k) * K * 32);
    const uint32_t* dr = (const uint32_t*)(s->descM + (size_t)(2 * k + 1) * K * 32);
    const uint32_t* ll = (const uint32_t*)(s->ldesc_raw + (size_t)(2 * k) * Ln * 32);
    const uint32_t* lr = (const uint32_t*)(s->ldesc_raw + (size_t)(2 * k + 1) * Ln * 32);
    // forward problems (all left rows), then reverse problems restricted to the right rows the mutual check will read
    ks[2 * k + 0] = {dl, dr, kcnt + 2 * k, kcnt + 2 * k + 1, 0, 0, key(0, 0), key(0, 1), nullptr};
    ks[2 * k + 1] = {ll, lr, lcnt + 2 * k, lcnt + 2 * k + 1, 0, 0, key(2, 0), key(2, 1), nullptr};
    ks[2 * B + 2 * k + 0] = {dr, dl, s->rev_count + 2 * k, kcnt + 2 * k, 0, 0, key(1, 0), key(1, 1), s->rev_list + (size_t)(2 * k) * K};
    ks[2 * B + 2 * k + 1] = {lr, ll, s->rev_count + 2 * k + 1, lcnt + 2 * k, 0, 0, key(3, 0), key(3, 1), s->rev_list + (size_t)(2 * k + 1) * K};
    gp[k] ={s->gnP + (size_t)k * K * 3, s->gnObs + (size_t)k * K * 2, s->gnInlP + (size_t)k * K, s->gnNp + k, 0,
             s->gn_sP + (size_t)k * Ln * 3, s->gn_eP + (size_t)k * Ln * 3, s->gn_le + (size_t)k * Ln * 3,
             s->gnInlL + (size_t)k * Ln, s->gnNl + k, 0, nullptr, s->gn_out + k};
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(s->knn_stereo, ks.data(), ks.size() * sizeof(KnnProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->gn_probs, gp.data(), gp.size() * sizeof(GnProblem), cudaMemcpyHostToDevice, cs));
  for (int k = 0; k < B; ++k) gp[k].T_init = s->pair_T + 16 * (size_t)k;   // the same problems seeded with the prediction
  PLF_CUDA(ctx, cudaMemcpyAsync(s->gn_probs_mm, gp.data(), gp.size() * sizeof(GnProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return pipe_seq_reset(ctx, ctx->afast_on, ctx->motion_on);
}

// Builds the pipeline for the camera's image size and the declared ones on first use; a failed setup leaves no state
// behind.
static plf_status pipe_prepare(plf_ctx* ctx) {
  if (ctx->pipe) return PLF_OK;
  const plf_status st = pipe_build(ctx);
  if (st) plf_pipe_free(ctx);
  return st;
}

// One plf_batch_run call: its pairs, buffer parities and slots, and the streams of its phases.
struct BatchRun {
  int B;
  int g;         // the batch's image size: record s->geo[g], the size of the upload it consumes
  int ncarry;    // entries of the carry list in batch table rp: the sequences the batch holds
  int nin;       // entries of the input table in batch table rp (0: none, every pair is converted as it is)
  bool masked;   // batch table rp holds the images' masks (a pair or a sequence of the batch has one); else no image is masked
  int nbuild;    // entries of the build list in batch table rp: the images with a pair mask (plf_batch_upload_masks)
  int nwin;      // pairs at matching_strategy != 0
  bool best_lr;  // some pair matches with best_lr_matches
  bool afast;    // adaptive FAST thresholds (plf_set_adaptive_fast): pair thresholds in the E phase, the next ones behind k_finalize
  bool motion;   // motion model (plf_set_motion_model): pair predictions at the start of M, the next ones behind k_finalize
  int par;       // parity of the E -> G -> M hand-off buffers
  int lp;        // parity of the LSD hand-off buffers (0 when they exist once)
  int rp;        // slot of the result ring
  int run_slot;  // upload slot consumed: the most recently uploaded batch
  bool piped, lsd2;
  cudaStream_t sM, sE, sG, sP;
};

// Entry rp of the pinned and of the device batch table ring.
static BatchTab host_tab(const PipeState* s, int rp) { return batch_tab(s->h_tab[rp], s->B); }
static BatchTab dev_tab(const PipeState* s, int rp) { return batch_tab(s->tab + rp * batch_tab_bytes(s->B), s->B); }

// The parts of the batch's table that it uses, to ring entry rp of the device on the copy stream: the sequence table, the
// cameras and the settings always (one copy, up to the batch's last settings), the input table, the masks and the build
// list when it has them.  ev_tab[rp] marks them.
static plf_status send_tab(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const BatchTab h = host_tab(s, r.rp), d = dev_tab(s, r.rp);
  cudaStream_t cs = s->copy;
  const size_t head = reinterpret_cast<const uint8_t*>(h.prm + r.B) - reinterpret_cast<const uint8_t*>(h.prev);
  PLF_CUDA(ctx, cudaMemcpyAsync(d.prev, h.prev, head, cudaMemcpyHostToDevice, cs));
  if (r.nin) PLF_CUDA(ctx, cudaMemcpyAsync(d.in, h.in, sizeof(PlfRectPair) * r.nin, cudaMemcpyHostToDevice, cs));
  if (r.masked) PLF_CUDA(ctx, cudaMemcpyAsync(d.masks, h.masks, sizeof(uint8_t*) * 2 * r.B, cudaMemcpyHostToDevice, cs));
  if (r.nbuild) PLF_CUDA(ctx, cudaMemcpyAsync(d.build, h.build, sizeof(PlfMaskBuild) * r.nbuild, cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaEventRecord(s->ev_tab[r.rp], cs));
  return PLF_OK;
}

// cv::remap(src, dst, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) at one output pixel of one channel: map1 = (sx, sy),
// map2 & 1023 = 32 fy + fx selects OpenCV's weights 32 (32 - fx) (32 - fy), 32 fx (32 - fy), 32 (32 - fx) fy and 32 fx fy of
// the taps (x, y), (x+1, y), (x, y+1), (x+1, y+1) (exact: no rounding excess to move), so (sum w p + 2^14) >> 15 is
// (sum (w / 32) p + 2^9) >> 10.  src points at the channel's byte of pixel (0, 0) of a w x h image of `row` bytes per row
// and `px` bytes per pixel (cv::remap of a multi-channel image is this per channel).  Taps outside the image read 0.
__device__ __forceinline__ int remap_px(const uint8_t* __restrict__ src, int row, int px, int w, int h, int sx, int sy, int fx,
                                        int fy) {
  auto tap = [&](int u, int v) -> int {
    return (unsigned)u < (unsigned)w && (unsigned)v < (unsigned)h ? __ldg(src + (size_t)v * row + u * px) : 0;
  };
  const int acc = (32 - fx) * (32 - fy) * tap(sx, sy) + fx * (32 - fy) * tap(sx + 1, sy) + (32 - fx) * fy * tap(sx, sy + 1) +
                  fx * fy * tap(sx + 1, sy + 1);
  return (acc + 512) >> 10;
}

// cv::cvtColor(COLOR_BGR2GRAY) of 8-bit B, G, R as OpenCV 4 computes it (15-bit fixed point; COLOR_BGRA2GRAY ignores alpha)
__device__ __forceinline__ int bgr_gray(int b, int g, int r) { return (3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15; }

// Grey image z = 2 j + side of a batch's input: entry j of tab gives the pair and its maps (tab NULL: pair j, not
// rectified).  src holds image 2k + side of pair k `img` bytes after image 0, w x h pixels of `row` bytes per row and CH
// interleaved bytes per pixel (1: grey, 3: BGR, 4: BGRA).  A pair with maps is remapped per channel first and converted
// after, as stvo-pl's reader remaps the colour image it read and the detectors convert it; every other pair is converted
// as it is.
template <int CH>
__global__ void __launch_bounds__(256) k_input(const PlfRectPair* __restrict__ tab, const uint8_t* __restrict__ src, size_t img,
                                               int row, int w, int h, size_t AP, int pitch, uint8_t* __restrict__ out) {
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= w || y >= h) return;
  const int j = blockIdx.z >> 1, side = blockIdx.z & 1;
  const PlfRectPair e = tab ? tab[j] : PlfRectPair{nullptr, j, 0};
  const uint8_t* im = src + (size_t)(2 * e.pair + side) * img;
  constexpr int NC = CH == 1 ? 1 : 3;   // the channels read: alpha is not
  int v[3] = {0, 0, 0};
  if (e.maps) {
    const size_t A = (size_t)w * h, i = (size_t)y * w + x;
    const short2 m = PLF_RECT_MAP1(e.maps, A, side)[i];
    const int f = PLF_RECT_MAP2(e.maps, A, side)[i] & 1023, fx = f & 31, fy = f >> 5;
    for (int c = 0; c < NC; ++c) v[c] = remap_px(im + c, row, CH, w, h, m.x, m.y, fx, fy);
  } else {
    for (int c = 0; c < NC; ++c) v[c] = __ldg(im + (size_t)y * row + x * CH + c);
  }
  out[(size_t)blockIdx.z * AP + (size_t)y * pitch + x] = (uint8_t)(CH == 1 ? v[0] : bgr_gray(v[0], v[1], v[2]));
}

// The colour landing buffer of ch channels, [2 max_batch][h][w][ch] (image 2k = left k, 2k+1 = right k) at the largest
// image size (any size's upload lands there), carved from
// PLF_SCR_COLOR_PIPE.  Only the copy stream touches it: the uploads land there and the runs' conversions read it in call
// order, so one buffer serves every batch in flight.  To grow (the first colour upload, or 4 channels after 3) the block
// waits for the copy stream, and the new block is allocated before the old one is freed: a failed allocation leaves the
// last upload as it was.
static plf_status color_scratch(plf_ctx* ctx, PipeState* s, int ch, uint8_t** land) {
  DevBufList b;
  b.add(*land, 2 * (size_t)s->B * s->max_area() * ch);
  size_t need = 0;
  for (const DevBufList::Entry& e : b.entries) need += plf_align256(e.bytes);
  DevBuf& slot = ctx->scratch[PLF_SCR_COLOR_PIPE];
  if (slot.bytes < need) {
    PLF_CUDA(ctx, cudaStreamSynchronize(s->copy));
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, need + 64);   // + the slack plf_scratch gives every slot
    if (e != cudaSuccess) {
      cudaGetLastError();
      return plf_fail(ctx, PLF_ERR_CUDA, "plf_batch_upload_color: cudaMalloc(%zu) of the colour landing buffer: %s", need,
                      cudaGetErrorString(e));
    }
    cudaFree(slot.p);
    slot.p = p;
    slot.bytes = need;
  }
  return b.carve(ctx, PLF_SCR_COLOR_PIPE);
}

// Turns the upload the run consumes into the grey images of its slot, before any stream of the run reads them: on the
// copy stream, behind the upload and the batch table, once the runs that read the slot before have finished with it;
// ev_up[run_slot] is recorded again, so the E and P phases (which wait for it) read the result.  A colour upload
// (plf_batch_upload_color) is converted from the landing buffer into the slot, the pairs of rectified sequences remapped
// in the same pass.  A grey upload landed in the slot before the run knew its sequences: its rectified pairs are remapped
// into scratch and copied back in place (the copy stream orders one batch's scratch use before the next's), and a grey
// batch without one enqueues nothing.
static plf_status run_input(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const bool color = s->up_ch > 1;
  if (!color && r.nin == 0) return PLF_OK;
  const PipeGeo& G = s->geo[r.g];
  const int w = G.w, h = G.h, pitch = G.pitch;
  const size_t AP = (size_t)pitch * h;
  uint8_t* imgs = s->imgs2[r.run_slot];
  const PlfRectPair* tab = r.nin ? dev_tab(s, r.rp).in : nullptr;
  uint8_t* land = nullptr;    // colour: the landing buffer
  uint8_t* pairs = nullptr;   // grey: the remapped pairs
  if (color) {
    if (plf_status st = color_scratch(ctx, s, s->up_ch, &land)) return st;
  } else {
    DevBufList b;
    b.add(pairs, 2 * (size_t)s->B * s->max_image());
    if (b.carve(ctx, PLF_SCR_RECT_PIPE)) return PLF_ERR_CUDA;
  }
  cudaStream_t cs = s->copy;
  // a run that read this slot before (a slot run twice) has finished with it
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->ev_free[r.run_slot], 0));
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->ev_free2[r.run_slot], 0));
  const dim3 grid((w + 31) / 32, (h + 7) / 8, 2 * (color ? r.B : r.nin)), block(32, 8);
  if (color) {
    const int row = s->up_ch * w;
    plf_mark(ctx, cs, "color.start");
    if (s->up_ch == 3) k_input<3><<<grid, block, 0, cs>>>(tab, land, (size_t)row * h, row, w, h, AP, pitch, imgs);
    else k_input<4><<<grid, block, 0, cs>>>(tab, land, (size_t)row * h, row, w, h, AP, pitch, imgs);
    PLF_LAUNCH_CHECK(ctx);
    plf_mark(ctx, cs, "color.k_color");
  } else {
    k_input<1><<<grid, block, 0, cs>>>(tab, imgs, AP, pitch, w, h, AP, pitch, pairs);
    PLF_LAUNCH_CHECK(ctx);
    // back in runs of consecutive pairs, w bytes of each row (the slot's row padding stays as the upload left it)
    const PlfRectPair* in = host_tab(s, r.rp).in;
    for (int j0 = 0, j1; j0 < r.nin; j0 = j1) {
      for (j1 = j0 + 1; j1 < r.nin && in[j1].pair == in[j1 - 1].pair + 1;) ++j1;
      PLF_CUDA(ctx, cudaMemcpy2DAsync(imgs + 2 * (size_t)in[j0].pair * AP, (size_t)pitch, pairs + 2 * (size_t)j0 * AP,
                                      (size_t)pitch, (size_t)w, 2 * (size_t)(j1 - j0) * h, cudaMemcpyDeviceToDevice, cs));
    }
  }
  PLF_CUDA(ctx, cudaEventRecord(s->ev_up[r.run_slot], cs));
  return PLF_OK;
}

// Bytes between two images' mask pyramids in a block of PLF_SCR_MASK_PIPE at image size G: a multiple of the row pitch,
// so that one 3-D copy per side lands an upload's level 0 planes.
static size_t mask_stride(const PipeGeo& G) {
  const size_t b = plf_orb_mask_bytes(G.orb);
  return (b + G.pitch - 1) / G.pitch * G.pitch;
}

// The pair masks' pyramid blocks, one per upload slot, each of 2 max_batch pyramids at the largest mask_stride of any
// size: carved from PLF_SCR_MASK_PIPE, which is allocated at the first call and never grows after it.
static plf_status mask_scratch(plf_ctx* ctx, PipeState* s) {
  size_t img = 0;
  for (const PipeGeo& G : s->geo) img = std::max(img, mask_stride(G));
  DevBufList b;
  b.add(s->mpyr[0], 2 * (size_t)s->B * img);
  b.add(s->mpyr[1], 2 * (size_t)s->B * img);
  return b.carve(ctx, PLF_SCR_MASK_PIPE);
}

// Builds the pair masks' pyramids of the upload the run consumes (plf_batch_upload_masks landed their level 0): on the
// copy stream, behind the upload, the mask copy and the batch table, each ANDed with its sequence's mask as the build list
// gives it; ev_up[run_slot] is recorded again, so the E and P phases (which wait for it) read the result.
static plf_status run_masks(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  if (r.nbuild == 0) return PLF_OK;
  cudaStream_t cs = s->copy;
  plf_mark(ctx, cs, "masks.start");
  if (plf_status st = plf_orb_mask_pyramids(ctx, cs, s->geo[r.g].orb, dev_tab(s, r.rp).build, PlfMaskBuild{}, r.nbuild)) return st;
  plf_mark(ctx, cs, "masks.k_mask_pyramid");
  PLF_CUDA(ctx, cudaEventRecord(s->ev_up[r.run_slot], cs));
  return PLF_OK;
}

// ---- E phase: ORB + LBD gradient prelude (bandwidth / ALU bound); outputs per batch parity ----
static plf_status run_extract(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  PipeGeo& G = s->geo[r.g];
  const int w = G.w, h = G.h, B = r.B, par = r.par;
  const size_t A = (size_t)w * h, AP = (size_t)G.pitch * h;   // dense maps / padded images
  const uint8_t* imgs = s->imgs2[r.run_slot];
  cudaStream_t sE = r.sE;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->ev_up[r.run_slot], 0));  // images uploaded
  PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->evX[par], 0));           // batch i-2 (same parity) no longer reads these buffers
  plf_mark(ctx, sE, "start");
  PLF_CUDA(ctx, cudaEventRecord(s->tE0[par], sE));
  const BatchTab tab = dev_tab(s, r.rp);
  const int* img_th = nullptr;   // without adaptive FAST each image detects at its pair's settings' threshold
  const uint8_t* const* masks = r.masked ? tab.masks : nullptr;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->ev_tab[r.rp], 0));   // the settings, sequence and mask tables
  if (r.afast) {
    // the thresholds of the batch's images: the sequence table, and the previous batch's threshold update (which has
    // also read img_th for the last time)
    PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->ev_th, 0));
    k_fast_th_images<<<(B + 127) / 128, 128, 0, sE>>>(tab.prev, B, s->B, s->B + s->nseq, s->seq_rec, tab.prm, s->img_th);
    PLF_LAUNCH_CHECK(ctx);
    img_th = s->img_th;
  }
  plf_status st = plf_orb_run(ctx, sE, G.orb, imgs, AP, G.pitch, 2 * B, par, img_th, masks, tab.prm);
  if (!st) st = plf_launch_blur5_sobel(ctx, sE, &G.lbd_tm, imgs, G.pitch, AP, w, h, 2 * B, s->lbd_grad[par], A);
  if (st) return st;
  plf_mark(ctx, sE, "lbd.k_blur5_sobel");
  // this batch's ORB overflow flag (one for every size): snapshot + clear on the E stream, so that a flag raised by batch
  // i+1's extraction is not reported on batch i's download
  PLF_CUDA(ctx, cudaMemcpyAsync(s->d_ovf + 2 * r.rp, plf_orb_overflow_flag(G.orb), sizeof(int), cudaMemcpyDeviceToDevice, sE));
  PLF_CUDA(ctx, cudaMemsetAsync(plf_orb_overflow_flag(G.orb), 0, sizeof(int), sE));
  PLF_CUDA(ctx, cudaEventRecord(s->evE[par], sE));
  PLF_CUDA(ctx, cudaEventRecord(s->ev_free[r.run_slot], sE));  // the image buffer may be overwritten by the next upload
  return PLF_OK;
}

// ---- P / G phases: the LSD chain.  P = blur / resize / gradient / seed ordering (bandwidth-bound), G = region growing
// (latency bound, one warp per image), rectangle fit and KeyLines.  With the hand-off maps per batch parity (lsd2, the
// default where they fit) P runs on its own stream: P(i+1) overlaps G(i), and the chain on the critical path is G alone;
// with one copy P and G share a stream and LSD(i+1) starts when LSD(i) ends.  The buffers only G writes and reads
// (region points, regions, segments) exist once either way: G(i+1) follows G(i) on its stream. ----
static plf_status run_lsd(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const int par = r.par;
  const PipeGeo& G = s->geo[r.g];
  const size_t AP = (size_t)G.pitch * G.h;
  cudaStream_t sP = r.sP, sG = r.sG;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sP, s->ev_up[r.run_slot], 0));
  PLF_CUDA(ctx, cudaStreamWaitEvent(sP, s->ev_tab[r.rp], 0));   // the settings and mask tables, read by G's KeyLine stage
  if (r.lsd2) PLF_CUDA(ctx, cudaStreamWaitEvent(sP, s->evG[par], 0));   // batch i-2 (same parity) has finished growing / fitting on these maps
  PLF_CUDA(ctx, cudaEventRecord(s->tG0[par], sP));
  plf_status st = plf_lsd_pre(ctx, sP, G.lsd, s->imgs2[r.run_slot], AP, G.pitch, r.lp, 2 * r.B);
  if (st) return st;
  PLF_CUDA(ctx, cudaEventRecord(s->ev_free2[r.run_slot], sP));
  PLF_CUDA(ctx, cudaEventRecord(s->evP[par], sP));
  PLF_CUDA(ctx, cudaStreamWaitEvent(sG, s->evP[par], 0));
  // the KeyLine outputs are overwritten: the match phase that read them last (batch i-2 with two parities, batch i-1 with one)
  // has taken its copy
  const BatchTab tab = dev_tab(s, r.rp);
  st = plf_lsd_grow(ctx, sG, G.lsd, r.lp, 2 * r.B, r.piped ? s->evX[r.lsd2 ? par : par ^ 1] : nullptr, r.masked ? tab.masks : nullptr,
                    tab.prm);
  if (st) return st;
  // the KeyLine stage has read the pair masks' level 0: the next mask upload into the slot may overwrite them
  if (r.nbuild) PLF_CUDA(ctx, cudaEventRecord(s->ev_mfree[r.run_slot], sG));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->d_ovf + 2 * r.rp + 1, plf_lsd_overflow_flag(G.lsd), sizeof(int), cudaMemcpyDeviceToDevice, sG));
  PLF_CUDA(ctx, cudaMemsetAsync(plf_lsd_overflow_flag(G.lsd), 0, sizeof(int), sG));
  PLF_CUDA(ctx, cudaEventRecord(s->evG[par], sG));
  return PLF_OK;
}

// One windowed-matching launch over B problems of one kind (points: cap = K, lines: cap = Ln).  Problem p matches the
// descriptor rows of image / slot q_slot[p] * step of `desc` (p * step without q_slot; cnt[...] of them) against those of
// image / slot p * step + t_off.  Problem p takes its window, ratio, best_lr and direction gate from the pair's settings
// prm[p] (f2f: the frame-to-frame window, else the stereo one).
static MgbArgs mgb_args(bool lines, int cap, int step, const int* q_slot, int t_off, const int* q_geo, const int* t_geo,
                        const double* t_dir, const uint8_t* desc, const int* cnt, int32_t* m12, size_t m12_stride, int* count,
                        int count_stride, const PlfPairPrm* prm, int f2f) {
  MgbArgs a = {};
  a.g.cols = PLF_GRID_COLS; a.g.rows = PLF_GRID_ROWS;
  a.is_lines = lines ? 1 : 0; a.K = a.Kt = cap;
  a.q_geo = q_geo; a.t_geo = t_geo; a.t_dir = t_dir;
  a.q_slot = q_slot;
  a.d1 = desc; a.d2 = desc + (size_t)t_off * cap * 32; a.d1_stride = a.d2_stride = (size_t)step * cap * 32;
  a.n1 = cnt; a.n2 = cnt + t_off; a.n1_stride = a.n2_stride = step;
  a.m12 = m12; a.m12_stride = m12_stride; a.count = count; a.count_stride = count_stride;
  a.prm = prm; a.f2f = f2f;
  return a;
}

// ---- M phase: LBD, stereo association, frame-to-frame tracking, pose (needs the previous batch's M phase) ----
static plf_status run_match(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const PipeGeo& G = s->geo[r.g];
  const int w = G.w, h = G.h, B = r.B, par = r.par, rp = r.rp;
  const size_t A = (size_t)w * h;
  const int K = s->max_kp, Ln = s->max_ln;
  const plf_params& P = ctx->params;
  plf_keypoint* kps; uint8_t* odesc; int* kcnt; int mk;
  plf_keyline* kls; int* lcnt; int ml;
  plf_orb_outputs(G.orb, par, &kps, &odesc, &kcnt, &mk);
  plf_lsd_outputs(G.lsd, r.lp, &kls, &lcnt, &ml);
  cudaStream_t cs = r.sM;
  plf_status st;
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->evG[par], 0));
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->evE[par], 0));
  PLF_CUDA(ctx, cudaEventRecord(s->tM0[rp], cs));
  // the batch's sequence table, and the pairs' cameras and settings
  const BatchTab tab = dev_tab(s, rp);
  const int32_t* prev = tab.prev;
  const int32_t* carry = tab.carry;
  const PlfPairCam* pcam = tab.cams;
  const PlfPairPrm* prm = tab.prm;
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->ev_tab[rp], 0));
  k_f2f_problems<<<(B + 127) / 128, 128, 0, cs>>>(s->fs, prev, B, K, Ln, s->knn_keys, s->m12, s->mcount, s->kcntM, s->lcntM,
                                                  s->fs.pt_count + s->B + s->nseq, prm, s->knn_f2f, s->nnr_f2f, s->nnr_stereo);
  PLF_LAUNCH_CHECK(ctx);
  // the pairs' motion predictions, when the model is on (null: the f2f geometry and the pose solver start from identity).
  // The previous batch wrote its sequences' ones behind its k_finalize on this stream.
  const double* T_pred = nullptr;
  if (r.motion) {
    k_motion_pairs<<<B, 16, 0, cs>>>(prev, s->B, s->B + s->nseq, s->seq_rec, s->pair_T);
    PLF_LAUNCH_CHECK(ctx);
    T_pred = s->pair_T;
  }
  if ((st = plf_launch_lbd(ctx, cs, s->lbd_grad[par], A, w, h, 2 * B, kls, lcnt, Ln, s->ldesc_raw, nullptr))) return st;
  plf_mark(ctx, cs, "lbd.k_lbd");
  // the rest of the match phase works on its own copy of the extraction outputs; evX releases this parity to batch i+2
  PLF_CUDA(ctx, cudaMemcpyAsync(s->kpsM, kps, sizeof(plf_keypoint) * 2 * (size_t)B * K, cudaMemcpyDeviceToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->descM, odesc, 32 * 2 * (size_t)B * K, cudaMemcpyDeviceToDevice, cs));
  // has_points / has_lines = 0 (stvo-pl skips the disabled kind in extraction and f2fTracking): its counts are zero from
  // here on, so it has no stereo rows, no matches, no pose rows and reports 0 detected features
  if (P.has_points) PLF_CUDA(ctx, cudaMemcpyAsync(s->kcntM, kcnt, sizeof(int) * 2 * (size_t)B, cudaMemcpyDeviceToDevice, cs));
  else PLF_CUDA(ctx, cudaMemsetAsync(s->kcntM, 0, sizeof(int) * 2 * (size_t)B, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->klsM, kls, sizeof(plf_keyline) * 2 * (size_t)B * Ln, cudaMemcpyDeviceToDevice, cs));
  if (P.has_lines) PLF_CUDA(ctx, cudaMemcpyAsync(s->lcntM, lcnt, sizeof(int) * 2 * (size_t)B, cudaMemcpyDeviceToDevice, cs));
  else PLF_CUDA(ctx, cudaMemsetAsync(s->lcntM, 0, sizeof(int) * 2 * (size_t)B, cs));
  PLF_CUDA(ctx, cudaEventRecord(s->evX[par], cs));
  kps = s->kpsM; odesc = s->descM; kcnt = s->kcntM; kls = s->klsM; lcnt = s->lcntM;
  plf_mark(ctx, cs, "copy extraction outputs");
  PLF_CUDA(ctx, cudaMemsetAsync(s->mcount, 0, (size_t)B * 4 * sizeof(int), cs));
  const double mg_iw = PLF_GRID_COLS / (double)w, mg_ih = PLF_GRID_ROWS / (double)h;   // StereoFrame::inv_width / inv_height
  // The windowed matcher runs over every pair when one of them is windowed; then match() over every pair when one is not
  // (its problems of windowed pairs write nothing, k_f2f_problems), so each pair keeps the association of its own strategy.
  const bool windowed = r.nwin > 0, brute = r.nwin < B;
  if (windowed) {
    // stereo association through matchGrid(): window (matching_s_ws, 0) x (0, 0) over the right image's grid
    k_mg_geom_stereo<<<dim3((std::max(K, Ln) + 255) / 256, 2 * B), 256, 0, cs>>>(kps, kcnt, K, kls, lcnt, Ln, mg_iw, mg_ih, s->mg_q[0],
                                                                                 s->mg_t[0], s->mg_q[1], s->mg_t[1], s->mg_dir[0]);
    PLF_LAUNCH_CHECK(ctx);
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(false, K, 2, nullptr, 1, s->mg_q[0], s->mg_t[0], nullptr, odesc, kcnt,
                                                        s->m12, 4 * (size_t)K, s->mcount, 4, prm, 0), B, K, K, PLF_SCR_MGB_PIPE, cs))) return st;
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(true, Ln, 2, nullptr, 1, s->mg_q[1], s->mg_t[1], s->mg_dir[0], s->ldesc_raw,
                                                        lcnt, s->m12 + K, 4 * (size_t)K, s->mcount + 1, 4, prm, 0), B, Ln, Ln, PLF_SCR_MGB_PIPE, cs))) return st;
    plf_mark(ctx, cs, "stereo.k_mgb (matchGrid)");
  }
  if (brute) {
    // L->R 2-NN for every left feature; R->L only for the right features that are somebody's accepted best match
    // (k_nnr_mutual reads nothing else of the reverse direction): the same matches for ~2/3 of the popcounts
    if ((st = plf_launch_knn2(ctx, cs, s->knn_stereo, 2 * B, std::max(K, Ln)))) return st;
    if (r.best_lr) {
      PLF_CUDA(ctx, cudaMemsetAsync(s->rev_flags, 0, 2 * (size_t)B * K * sizeof(int), cs));
      PLF_CUDA(ctx, cudaMemsetAsync(s->rev_count, 0, 2 * (size_t)B * sizeof(int), cs));
      if ((st = plf_launch_nnr_mark(ctx, cs, s->nnr_stereo, 2 * B, std::max(K, Ln), s->rev_flags, s->rev_list, s->rev_count, K))) return st;
      // the reverse problems are laid out after the forward problems of ALL max_batch pairs (pipe_prepare), not of this
      // call's B pairs: a partial batch (B < max_batch) must still start at 2 * max_batch
      if ((st = plf_launch_knn2(ctx, cs, s->knn_stereo + 2 * s->B, 2 * B, std::max(K, Ln)))) return st;
    }
    plf_mark(ctx, cs, "stereo.k_hamming_knn2");
    if ((st = plf_launch_nnr(ctx, cs, s->nnr_stereo, 2 * B, std::max(K, Ln)))) return st;
    plf_mark(ctx, cs, "stereo.k_nnr_mutual");
  }
  k_stereo_points<<<B, 1024, 0, cs>>>(kps, odesc, kcnt, K, s->m12, 4 * K, pcam, prm, s->fs);
  PLF_LAUNCH_CHECK(ctx);
  k_stereo_lines<<<B, 1024, 0, cs>>>(kls, s->ldesc_raw, lcnt, Ln, s->m12 + K, 4 * K, pcam, prm, s->fs);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "stereo.k_stereo_points+lines");
  if ((st = plf_launch_knn2(ctx, cs, s->knn_f2f, 4 * B, std::max(K, Ln)))) return st;
  plf_mark(ctx, cs, "f2f.k_hamming_knn2");
  if ((st = plf_launch_nnr(ctx, cs, s->nnr_f2f, 2 * B, std::max(K, Ln)))) return st;
  if (windowed) {
    // frame-to-frame: matchGrid() in a +-matching_f2f_ws window around the projected feature; the match() result above
    // stands where the window search found fewer than min_pt_matches / min_ls_matches
    PLF_CUDA(ctx, cudaMemsetAsync(s->mgcount, 0, (size_t)B * 2 * sizeof(int), cs));
    k_mg_geom_f2f<<<dim3((std::max(K, Ln) + 255) / 256, B), 256, 0, cs>>>(s->fs, prev, K, Ln, pcam, T_pred, mg_iw, mg_ih,
                                                                          s->mg_q[2], s->mg_t[2], s->mg_q[3], s->mg_t[3],
                                                                          s->mg_dir[1]);
    PLF_LAUNCH_CHECK(ctx);
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(false, K, 1, prev, 0, s->mg_q[2], s->mg_t[2], nullptr, s->fs.pdesc,
                                                        s->fs.pt_count, s->m12g, 2 * (size_t)K, s->mgcount, 2, prm, 1), B, K, K, PLF_SCR_MGB_PIPE, cs))) return st;
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(true, Ln, 1, prev, 0, s->mg_q[3], s->mg_t[3], s->mg_dir[1], s->fs.ldesc,
                                                        s->fs.ls_count, s->m12g + K, 2 * (size_t)K, s->mgcount + 1, 2, prm, 1), B, Ln, Ln, PLF_SCR_MGB_PIPE, cs))) return st;
    k_mg_select<<<dim3((K + 255) / 256, B), 256, 0, cs>>>(s->m12g, s->mgcount, s->fs.pt_count, prev, K, K, 0, s->m12, prm);
    PLF_LAUNCH_CHECK(ctx);
    k_mg_select<<<dim3((Ln + 255) / 256, B), 256, 0, cs>>>(s->m12g, s->mgcount, s->fs.ls_count, prev, Ln, K, 1, s->m12, prm);
    PLF_LAUNCH_CHECK(ctx);
    plf_mark(ctx, cs, "f2f.k_mgb (matchGrid)");
  }
  k_f2f_build<<<B, 1024, 0, cs>>>(s->fs, prev, K, Ln, s->m12 + 2 * K, s->m12 + 3 * K, 4 * K, s->gnP, s->gnObs, s->gnInlP, s->gnNp,
                                  s->gn_sP, s->gn_eP, s->gn_le, s->gnInlL, s->gnNl);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, cs, "f2f.k_nnr_mutual+k_f2f_build");
  if ((st = plf_launch_gn(ctx, cs, T_pred ? s->gn_probs_mm : s->gn_probs, B, plf_gn_opts_from_params(P), pcam, nullptr, prm))) return st;
  plf_mark(ctx, cs, "gn.k_gn_pose");
  k_finalize<<<(B + 127) / 128, 128, 0, cs>>>(s->gn_out, s->gnNp, s->gnNl, kcnt, lcnt, s->fs, prev, s->B + s->nseq, B,
                                               s->results + (size_t)rp * s->B, prm);
  PLF_LAUNCH_CHECK(ctx);
  k_carry<<<dim3(PLF_FS_NFIELDS, r.ncarry), 256, 0, cs>>>(s->fs, carry, K, Ln);   // the next batch tracks against these
  PLF_LAUNCH_CHECK(ctx);
  if (r.afast || r.motion) {
    // the next batch's E phase waits on ev_th for its sequences' thresholds; its M phase, on this stream, reads their
    // predictions
    k_seq_update<<<(r.ncarry + 127) / 128, 128, 0, cs>>>(s->results + (size_t)rp * s->B, carry, r.ncarry, s->B,
                                                         r.afast ? s->img_th : nullptr, ctx->afast, r.motion ? 1 : 0, s->seq_rec);
    PLF_LAUNCH_CHECK(ctx);
    if (r.afast) PLF_CUDA(ctx, cudaEventRecord(s->ev_th, cs));
  }
  plf_mark(ctx, cs, "k_finalize+carry");
  // results + overflow flags to pinned memory as part of this batch's stream work; evM marks them ready
  PLF_CUDA(ctx, cudaMemcpyAsync(s->h_results[rp], s->results + (size_t)rp * s->B, sizeof(plf_frame_result) * B, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->h_ovf[rp], s->d_ovf + 2 * rp, 2 * sizeof(int), cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaEventRecord(s->evM[rp], cs));
  return PLF_OK;
}

// Sequence s (-1: every sequence) restarts: its next pair in a run is a first frame (the batches run keep their tables).
static void restart_sequence(plf_ctx* ctx, int s) {
  if (!ctx->pipe) return;
  std::vector<uint8_t>& c = ctx->pipe->carried;
  if (s < 0) std::fill(c.begin(), c.end(), 0);
  else c[s] = 0;
}

// B pairs of w x h images of `row` bytes per row, read from left / right at `stride` bytes per row, to dst as images
// 2k = left k, 2k+1 = right k of h rows at dpitch bytes per row, on stream cs.  Dense rows (stride = dpitch = row) are one
// 2-D copy per side of B contiguous images ("rows" = images, pitch 2 images interleaving left and right); otherwise one
// 3-D copy per side (B images of h rows, the destination "height" of 2h rows skipping the other side's image of each pair).
static plf_status upload_pairs(plf_ctx* ctx, cudaStream_t cs, uint8_t* dst, int dpitch, int B, const uint8_t* left,
                               const uint8_t* right, int stride, int row, int h) {
  const size_t img = (size_t)dpitch * h;
  for (int side = 0; side < 2; ++side) {
    const uint8_t* src = side ? right : left;
    if (stride == row && dpitch == row) {
      PLF_CUDA(ctx, cudaMemcpy2DAsync(dst + side * img, 2 * img, src, img, img, B, cudaMemcpyHostToDevice, cs));
    } else {
      cudaMemcpy3DParms cp = {};
      cp.srcPtr = make_cudaPitchedPtr(const_cast<uint8_t*>(src), (size_t)stride, (size_t)row, (size_t)h);
      cp.dstPtr = make_cudaPitchedPtr(dst + side * img, (size_t)dpitch, (size_t)row, 2 * (size_t)h);
      cp.extent = make_cudaExtent((size_t)row, (size_t)h, (size_t)B);
      cp.kind = cudaMemcpyHostToDevice;
      PLF_CUDA(ctx, cudaMemcpy3DAsync(&cp, cs));
    }
  }
  return PLF_OK;
}

// ---- plf_set_sequence_params: the classification of plf_params' fields, the one place the library and the binding read
// it from (plf_sequence_param_fields).  SEQUENCE: read per pair or per image by the batched front-end; CONTEXT: fixes
// buffer geometry, lookup tables, tensor maps or which launch chains exist; IGNORED: has no effect for the context either.
struct ParamField {
  const char* name;
  size_t off;
  char type;   // 'i' int, 'f' float, 'd' double
  int cls;
};
#define PLF_PF(f, t, c) {#f, offsetof(plf_params, f), t, PLF_PARAM_##c}
static const ParamField kParamFields[] = {
    PLF_PF(has_points, 'i', CONTEXT),       PLF_PF(has_lines, 'i', CONTEXT),          PLF_PF(best_lr_matches, 'i', SEQUENCE),
    PLF_PF(max_dist_epip, 'f', SEQUENCE),   PLF_PF(min_disp, 'f', SEQUENCE),          PLF_PF(min_ratio_12_p, 'f', SEQUENCE),
    PLF_PF(line_sim_th, 'f', SEQUENCE),     PLF_PF(stereo_overlap_th, 'f', SEQUENCE), PLF_PF(f2f_overlap_th, 'f', IGNORED),
    PLF_PF(min_line_length, 'f', SEQUENCE), PLF_PF(line_horiz_th, 'f', SEQUENCE),     PLF_PF(min_ratio_12_l, 'f', SEQUENCE),
    PLF_PF(ls_min_disp_ratio, 'f', SEQUENCE), PLF_PF(homog_th, 'd', SEQUENCE),        PLF_PF(min_features, 'i', SEQUENCE),
    PLF_PF(max_iters, 'i', SEQUENCE),       PLF_PF(max_iters_ref, 'i', SEQUENCE),     PLF_PF(min_error, 'd', SEQUENCE),
    PLF_PF(min_error_change, 'd', SEQUENCE), PLF_PF(inlier_k, 'd', IGNORED),          PLF_PF(orb_nfeatures, 'i', SEQUENCE),
    PLF_PF(orb_scale_factor, 'f', CONTEXT), PLF_PF(orb_nlevels, 'i', SEQUENCE),       PLF_PF(orb_edge_th, 'i', CONTEXT),
    PLF_PF(orb_wta_k, 'i', CONTEXT),        PLF_PF(orb_score, 'i', CONTEXT),          PLF_PF(orb_patch_size, 'i', CONTEXT),
    PLF_PF(orb_fast_th, 'i', SEQUENCE),     PLF_PF(lsd_nfeatures, 'i', SEQUENCE),     PLF_PF(lsd_refine, 'i', CONTEXT),
    PLF_PF(lsd_scale, 'd', CONTEXT),        PLF_PF(lsd_sigma_scale, 'd', CONTEXT),    PLF_PF(lsd_quant, 'd', CONTEXT),
    PLF_PF(lsd_ang_th, 'd', CONTEXT),       PLF_PF(lsd_log_eps, 'd', CONTEXT),        PLF_PF(lsd_density_th, 'd', CONTEXT),
    PLF_PF(lsd_n_bins, 'i', CONTEXT),       PLF_PF(matching_strategy, 'i', SEQUENCE), PLF_PF(matching_s_ws, 'i', SEQUENCE),
    PLF_PF(matching_f2f_ws, 'i', SEQUENCE), PLF_PF(min_pt_matches, 'i', SEQUENCE),    PLF_PF(min_ls_matches, 'i', SEQUENCE),
};
#undef PLF_PF

static double param_value(const plf_params& p, const ParamField& f) {
  const uint8_t* a = reinterpret_cast<const uint8_t*>(&p) + f.off;
  if (f.type == 'i') return *reinterpret_cast<const int*>(a);
  if (f.type == 'f') return *reinterpret_cast<const float*>(a);
  return *reinterpret_cast<const double*>(a);
}

// What plf_set_sequence_params refuses in p for a context of settings c, naming the field; PLF_OK if nothing.
static plf_status check_sequence_params(plf_ctx* ctx, const plf_params& p) {
  const plf_params& c = ctx->params;
  for (const ParamField& f : kParamFields) {
    const double v = param_value(p, f), cv = param_value(c, f);
    if (f.cls == PLF_PARAM_CONTEXT) {
      if (v != cv && !(std::isnan(v) && std::isnan(cv)))
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_params: %s = %.17g, the context's is %.17g; it fixes the context's "
                        "buffers, tables or launches and must equal it", f.name, v, cv);
    } else if (f.cls == PLF_PARAM_SEQUENCE) {
      // counts and integer thresholds >= 0, real thresholds finite
      if (f.type == 'i' && v < 0)
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_params: %s = %d, need %s >= 0", f.name, (int)v, f.name);
      if (f.type != 'i' && !std::isfinite(v))
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_params: %s = %g, need a finite value", f.name, v);
    }
  }
  // the ORB buffers, tables and tensor maps hold the context's levels; a level does not depend on those after it
  if (p.orb_nlevels < 1 || p.orb_nlevels > c.orb_nlevels)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_params: orb_nlevels = %d, need 1 <= orb_nlevels <= the context's %d",
                    p.orb_nlevels, c.orb_nlevels);
  // the windowed matcher's buffers exist only in a context created windowed
  if (p.matching_strategy != 0 && c.matching_strategy == 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_params: matching_strategy = %d, and the context's is 0: a sequence may "
                    "be windowed only in a context created with matching_strategy != 0", p.matching_strategy);
  return PLF_OK;
}

// The image sizes the context accepts, its own first: "1242x375, 1226x370".
static std::string image_size_list(const plf_ctx* ctx) {
  std::string out = std::to_string(ctx->cam.width) + "x" + std::to_string(ctx->cam.height);
  for (size_t i = 0; i < ctx->image_sizes.size(); i += 2)
    out += ", " + std::to_string(ctx->image_sizes[i]) + "x" + std::to_string(ctx->image_sizes[i + 1]);
  return out;
}

extern "C" {

plf_status plf_reset_sequence(plf_ctx* ctx) {
  if (!ctx) return PLF_ERR_INVALID;
  if (ctx->pipe && ctx->pipe->n_pending)
    return plf_fail(ctx, PLF_ERR_STATE, "plf_reset_sequence: %d batch(es) still in flight; download them first", ctx->pipe->n_pending);
  restart_sequence(ctx, -1);
  return PLF_OK;
}

plf_status plf_set_max_sequences(plf_ctx* ctx, int n) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n < 1 || n > PLF_MAX_SEQUENCES)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_max_sequences: n = %d, need 1 <= n <= %d", n, PLF_MAX_SEQUENCES);
  if (ctx->pipe) return plf_fail(ctx, PLF_ERR_STATE, "plf_set_max_sequences: the pipeline exists (a batch call was made)");
  plf_drop_sequences(ctx);
  ctx->max_sequences = n;
  return PLF_OK;
}

plf_status plf_set_sequence_camera(plf_ctx* ctx, int s, const plf_camera* cam) {
  if (!ctx) return PLF_ERR_INVALID;
  if (plf_status st = plf_check_sequence(ctx, "plf_set_sequence_camera", s)) return st;
  if (cam) {
    if (ctx->image_sizes.empty()) {
      if (cam->width != ctx->cam.width)
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_camera: width = %d, the context's is %d", cam->width, ctx->cam.width);
      if (cam->height != ctx->cam.height)
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_camera: height = %d, the context's is %d", cam->height, ctx->cam.height);
    } else if (plf_image_size_index(ctx, cam->width, cam->height) < 0) {
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_camera: size %dx%d is not one of the context's image sizes (%s)",
                      cam->width, cam->height, image_size_list(ctx).c_str());
    }
    const struct { const char* name; double v; bool positive; } f[] = {
        {"fx", cam->fx, true}, {"fy", cam->fy, true}, {"cx", cam->cx, false}, {"cy", cam->cy, false}, {"b", cam->b, true}};
    for (const auto& e : f)
      if (!std::isfinite(e.v) || (e.positive && !(e.v > 0.0)))
        return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_camera: %s = %g, need a finite value%s", e.name, e.v,
                        e.positive ? " > 0" : "");
  }
  // the maps and mask pyramids of s were built for its present size
  const plf_camera& now = plf_sequence_camera(ctx, s);
  const plf_camera& next = cam ? *cam : ctx->cam;
  if ((next.width != now.width || next.height != now.height) && !ctx->seqs.empty()) {
    const PlfSequence& o = ctx->seqs[s];
    const bool maps = o.rect != nullptr, masks = o.mask[0] || o.mask[1];
    if (maps || masks)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_camera: sequence %d has %s%s%s of %dx%d; clear %s before changing "
                      "its image size to %dx%d", s, maps ? "rectification maps" : "", maps && masks ? " and " : "",
                      masks ? "masks" : "", now.width, now.height, maps && masks ? "them" : "it", next.width, next.height);
  }
  PlfSequence& q = plf_sequence(ctx, s);
  q.own_cam = cam != nullptr;
  q.cam = cam ? *cam : ctx->cam;
  restart_sequence(ctx, s);
  return PLF_OK;
}

plf_status plf_set_sequence_rectification(plf_ctx* ctx, int s, const int16_t* map1_l, const uint16_t* map2_l,
                                          const int16_t* map1_r, const uint16_t* map2_r) {
  if (!ctx) return PLF_ERR_INVALID;
  if (plf_status st = plf_check_sequence(ctx, "plf_set_sequence_rectification", s)) return st;
  const int given = !!map1_l + !!map2_l + !!map1_r + !!map2_r;
  if (given != 0 && given != 4)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_rectification: %d of the four maps given, need all four or none (NULL clears)",
                    given);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  // the copy stream runs every rectification: once it is idle, no batch run so far reads sequence s's old maps
  cudaStream_t cs = ctx->pipe ? ctx->pipe->copy : ctx->stream;
  uint8_t* old = ctx->seqs.empty() ? nullptr : ctx->seqs[s].rect;
  const plf_camera& sc = plf_sequence_camera(ctx, s);   // the maps are of the sequence's image size
  const size_t A = (size_t)sc.width * sc.height;
  if (given) {
    uint8_t* d = old;
    if (!d) {
      const cudaError_t e = cudaMalloc(&d, 12 * A);
      if (e != cudaSuccess) {
        cudaGetLastError();
        return plf_fail(ctx, PLF_ERR_CUDA, "plf_set_sequence_rectification: cudaMalloc(%zu): %s", 12 * A, cudaGetErrorString(e));
      }
    }
    const void* src[4] = {map1_l, map1_r, map2_l, map2_r};
    const size_t off[4] = {0, 4 * A, 8 * A, 10 * A}, len[4] = {4 * A, 4 * A, 2 * A, 2 * A};
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaMemcpyAsync(d + off[i], src[i], len[i], cudaMemcpyHostToDevice, cs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
    if (e != cudaSuccess) {
      if (!old) cudaFree(d);
      return plf_fail(ctx, PLF_ERR_CUDA, "plf_set_sequence_rectification: copying the maps: %s", cudaGetErrorString(e));
    }
    plf_sequence(ctx, s).rect = d;
  } else if (old) {
    PLF_CUDA(ctx, cudaStreamSynchronize(cs));
    cudaFree(old);
    ctx->seqs[s].rect = nullptr;
  }
  // its carried frame was extracted from other images
  restart_sequence(ctx, s);
  return PLF_OK;
}

plf_status plf_set_sequence_mask(plf_ctx* ctx, int s, const uint8_t* mask_l, const uint8_t* mask_r, int stride) {
  if (!ctx) return PLF_ERR_INVALID;
  if (plf_status st = plf_check_sequence(ctx, "plf_set_sequence_mask", s)) return st;
  const int w = plf_sequence_camera(ctx, s).width, h = plf_sequence_camera(ctx, s).height;   // the sequence's image size
  if ((mask_l || mask_r) && stride < w)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_sequence_mask: stride = %d, need stride >= width = %d", stride, w);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  // the new pyramids, built into fresh blocks on the main stream with the pipeline's ORB geometry of the sequence's size
  // (or, before the pipeline exists, that of a one-image ORB state of the same size and parameters)
  uint8_t* fresh[2] = {nullptr, nullptr};
  if (mask_l || mask_r) {
    OrbState* tmp = nullptr;
    plf_status st = ctx->pipe ? PLF_OK : plf_orb_create(ctx, w, h, 1, false, &tmp);
    if (st) return st;
    const OrbState* geo = ctx->pipe ? ctx->pipe->geo[plf_image_size_index(ctx, w, h)].orb : tmp;
    const size_t bytes = plf_orb_mask_bytes(geo) + 64;
    const uint8_t* src[2] = {mask_l, mask_r};
    for (int side = 0; side < 2 && !st; ++side) {
      if (!src[side]) continue;
      const cudaError_t e = cudaMalloc(&fresh[side], bytes);
      if (e != cudaSuccess) {
        cudaGetLastError();
        fresh[side] = nullptr;
        st = plf_fail(ctx, PLF_ERR_CUDA, "plf_set_sequence_mask: cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
      } else {
        st = plf_orb_mask_build(ctx, ctx->stream, geo, src[side], stride, fresh[side]);
      }
    }
    if (!st && cudaStreamSynchronize(ctx->stream) != cudaSuccess)
      st = plf_fail(ctx, PLF_ERR_CUDA, "plf_set_sequence_mask: building the mask pyramids: %s", cudaGetErrorString(cudaGetLastError()));
    plf_orb_free(tmp);
    if (st) {
      cudaFree(fresh[0]);
      cudaFree(fresh[1]);
      return st;
    }
  }
  // Batches in flight read the old pyramids in their extraction (ORB) and LSD (KeyLine) phases, on the E and G streams, or
  // all on the main stream when profiling serialises them: the call waits for those streams before it frees them.
  uint8_t** cur = ctx->seqs.empty() ? nullptr : ctx->seqs[s].mask;
  if (cur && (cur[0] || cur[1]) && ctx->pipe) {
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->aux[0]));
    PLF_CUDA(ctx, cudaStreamSynchronize(ctx->aux[1]));
  }
  if (cur) {
    cudaFree(cur[0]);
    cudaFree(cur[1]);
  }
  if (fresh[0] || fresh[1] || cur) {
    PlfSequence& q = plf_sequence(ctx, s);
    q.mask[0] = fresh[0];
    q.mask[1] = fresh[1];
  }
  return PLF_OK;
}

plf_status plf_get_sequence_mask_set(plf_ctx* ctx, int s, int* left, int* right) {
  if (!ctx) return PLF_ERR_INVALID;
  if (!left || !right) return plf_fail(ctx, PLF_ERR_INVALID, "plf_get_sequence_mask_set: left and right are required");
  if (plf_status st = plf_check_sequence(ctx, "plf_get_sequence_mask_set", s)) return st;
  const bool any = !ctx->seqs.empty();
  *left = any && ctx->seqs[s].mask[0] != nullptr;
  *right = any && ctx->seqs[s].mask[1] != nullptr;
  return PLF_OK;
}

plf_status plf_get_sequence_camera(const plf_ctx* ctx, int s, plf_camera* out) {
  if (!ctx) return PLF_ERR_INVALID;
  plf_ctx* c = const_cast<plf_ctx*>(ctx);   // the error text is the only state a failed call writes
  if (!out) return plf_fail(c, PLF_ERR_INVALID, "plf_get_sequence_camera: out is NULL");
  if (plf_status st = plf_check_sequence(c, "plf_get_sequence_camera", s)) return st;
  *out = plf_sequence_camera(ctx, s);
  return PLF_OK;
}

int plf_sequence_param_fields(const char** names, int* classes, int cap) {
  const int n = (int)(sizeof kParamFields / sizeof kParamFields[0]);
  for (int i = 0; i < n && i < cap; ++i) {
    if (names) names[i] = kParamFields[i].name;
    if (classes) classes[i] = kParamFields[i].cls;
  }
  return n;
}

plf_status plf_set_sequence_params(plf_ctx* ctx, int s, const plf_params* p) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_set_sequence_params: ctx is NULL");
  if (plf_status st = plf_check_sequence(ctx, "plf_set_sequence_params", s)) return st;
  if (p) {
    if (plf_status st = check_sequence_params(ctx, *p)) return st;
    PlfSequence& q = plf_sequence(ctx, s);
    q.own_prm = true;
    q.prm = *p;
    q.pair = plf_pair_prm(*p);
  } else if (!ctx->seqs.empty()) {
    ctx->seqs[s].own_prm = false;
  }
  // its carried frame was extracted and matched under the old settings
  restart_sequence(ctx, s);
  return PLF_OK;
}

plf_status plf_get_sequence_params(const plf_ctx* ctx, int s, plf_params* out) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_get_sequence_params: ctx is NULL");
  plf_ctx* c = const_cast<plf_ctx*>(ctx);   // the error text is the only state a failed call writes
  if (!out) return plf_fail(c, PLF_ERR_INVALID, "plf_get_sequence_params: out is NULL");
  if (plf_status st = plf_check_sequence(c, "plf_get_sequence_params", s)) return st;
  const bool own = !ctx->seqs.empty() && ctx->seqs[s].own_prm;
  *out = own ? ctx->seqs[s].prm : ctx->params;
  return PLF_OK;
}

plf_status plf_set_adaptive_fast(plf_ctx* ctx, const plf_adaptive_fast* cfg) {
  if (cfg) {   // checked first, so that a NULL context reports the field too (plf_last_error(NULL))
    const plf_adaptive_fast& a = *cfg;
    if (a.min_th < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: min_th = %d, need 0 <= min_th", a.min_th);
    if (a.max_th > 255) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: max_th = %d, need max_th <= 255", a.max_th);
    if (a.min_th > a.max_th)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: min_th = %d > max_th = %d, need min_th <= max_th", a.min_th, a.max_th);
    if (a.inc_th < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: inc_th = %d, need inc_th >= 0", a.inc_th);
    if (a.feat_th < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: feat_th = %d, need feat_th >= 0", a.feat_th);
    if (!std::isfinite(a.err_th)) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_adaptive_fast: err_th = %g, need a finite value", a.err_th);
  }
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_set_adaptive_fast: ctx is NULL");
  if (ctx->pipe && ctx->pipe->n_pending)
    return plf_fail(ctx, PLF_ERR_STATE, "plf_set_adaptive_fast: %d batch(es) still in flight; download them first", ctx->pipe->n_pending);
  if (cfg && ctx->pipe) {
    PLF_CUDA(ctx, cudaSetDevice(ctx->device));
    const plf_status st = pipe_seq_reset(ctx, true, false);
    if (st) return st;
  }
  ctx->afast_on = cfg != nullptr;
  ctx->afast = cfg ? *cfg : plf_adaptive_fast{};
  return PLF_OK;
}

plf_status plf_get_sequence_fast_th(plf_ctx* ctx, int s, int* th) {
  if (!ctx) return PLF_ERR_INVALID;
  if (!th) return plf_fail(ctx, PLF_ERR_INVALID, "plf_get_sequence_fast_th: th is NULL");
  if (plf_status st = plf_check_sequence(ctx, "plf_get_sequence_fast_th", s)) return st;
  *th = plf_sequence_pair(ctx, s).fast_th;
  if (!ctx->afast_on || !ctx->pipe || !ctx->pipe->carried[s]) return PLF_OK;   // the next pair is detected at orb_fast_th
  SeqRecord q;
  if (plf_status st = pipe_seq_read(ctx, s, &q)) return st;
  *th = q.th;
  return PLF_OK;
}

plf_status plf_set_motion_model(plf_ctx* ctx, int on) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_set_motion_model: ctx is NULL");
  if (ctx->pipe && ctx->pipe->n_pending)
    return plf_fail(ctx, PLF_ERR_STATE, "plf_set_motion_model: %d batch(es) still in flight; download them first", ctx->pipe->n_pending);
  if (on && ctx->pipe) {
    PLF_CUDA(ctx, cudaSetDevice(ctx->device));
    const plf_status st = pipe_seq_reset(ctx, false, true);
    if (st) return st;
  }
  ctx->motion_on = on != 0;
  return PLF_OK;
}

plf_status plf_get_sequence_motion(plf_ctx* ctx, int s, double T[16], int* valid) {
  if (!ctx) return PLF_ERR_INVALID;
  if (!T || !valid) return plf_fail(ctx, PLF_ERR_INVALID, "plf_get_sequence_motion: T and valid are required");
  if (plf_status st = plf_check_sequence(ctx, "plf_get_sequence_motion", s)) return st;
  for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  *valid = 0;
  if (!ctx->motion_on || !ctx->pipe || !ctx->pipe->carried[s]) return PLF_OK;   // the next pair starts from identity
  SeqRecord q;
  if (plf_status st = pipe_seq_read(ctx, s, &q)) return st;
  memcpy(T, q.T, sizeof q.T);
  *valid = q.valid;
  return PLF_OK;
}

plf_status plf_debug_motion_prior(plf_ctx* ctx, int n, const double* DT, const double* DT_cov, const double* err,
                                  const int32_t* status, double* T_out, int32_t* valid_out) {
  if (!ctx) return PLF_ERR_INVALID;
  if (n < 0) return plf_fail(ctx, PLF_ERR_INVALID, "plf_debug_motion_prior: n = %d < 0", n);
  if (n == 0) return PLF_OK;
  if (!DT || !DT_cov || !err || !status || !T_out || !valid_out)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_debug_motion_prior: every array is required");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t N = n;
  double *dDT, *dcov, *derr, *dT;
  int32_t *dst, *dvalid;
  DevBufList b;
  b.add(dDT, 16 * N); b.add(dcov, 36 * N); b.add(derr, N); b.add(dst, N); b.add(dT, 16 * N); b.add(dvalid, N);
  if (b.carve(ctx, PLF_SCR_GN)) return PLF_ERR_CUDA;
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemcpyAsync(dDT, DT, 16 * N * sizeof(double), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dcov, DT_cov, 36 * N * sizeof(double), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(derr, err, N * sizeof(double), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(dst, status, N * sizeof(int32_t), cudaMemcpyHostToDevice, cs));
  k_motion_debug<<<(n + 127) / 128, 128, 0, cs>>>(n, dDT, dcov, derr, dst, dT, dvalid);
  PLF_LAUNCH_CHECK(ctx);
  PLF_CUDA(ctx, cudaMemcpyAsync(T_out, dT, 16 * N * sizeof(double), cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(valid_out, dvalid, N * sizeof(int32_t), cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

// The grey pairs of an upload of image size s->geo[g] (arguments checked) into the slot the GPU is not reading.
static plf_status upload_grey(plf_ctx* ctx, int g, int B, const uint8_t* left, const uint8_t* right, int stride) {
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  plf_status st = pipe_prepare(ctx);
  if (st) return st;
  PipeState* s = ctx->pipe;
  const PipeGeo& G = s->geo[g];
  const int w = G.w, h = G.h;
  // H2D on the copy stream into the slot the GPU is not reading, so the copy of batch i+1 overlaps the run of batch i.
  // Device layout interleaves the pair: image 2k = left k, 2k+1 = right k; rows are padded to a 16-byte pitch.
  const int slot = s->up_slot ^ 1;
  uint8_t* dst = s->imgs2[slot];
  PLF_CUDA(ctx, cudaStreamWaitEvent(s->copy, s->ev_free[slot], 0));   // the last run that read this slot has finished with it
  PLF_CUDA(ctx, cudaStreamWaitEvent(s->copy, s->ev_free2[slot], 0));  // (ORB / LBD prelude on one stream, LSD on another)
  if (stride == w && G.pitch != w) {
    // densely packed input: ONE contiguous H2D copy per side into the dense landing buffer, then a device-to-device 2-D
    // copy widens the rows to the 16-byte pitch (the DMA engines move 1242-byte rows from host memory at a fraction of
    // the contiguous rate: measured 8.9 k vs 12.7 k pairs/s end to end)
    if ((st = upload_pairs(ctx, s->copy, s->stage, w, B, left, right, stride, w, h))) return st;
    PLF_CUDA(ctx, cudaMemcpy2DAsync(dst, (size_t)G.pitch, s->stage, (size_t)w, (size_t)w, 2 * (size_t)B * h, cudaMemcpyDeviceToDevice, s->copy));
  } else if ((st = upload_pairs(ctx, s->copy, dst, G.pitch, B, left, right, stride, w, h))) {   // pitch == w: dense rows
    return st;
  }
  PLF_CUDA(ctx, cudaEventRecord(s->ev_up[slot], s->copy));
  s->up_slot = slot;
  s->up_ch = 1;
  s->up_geo = g;
  s->uploaded = true;
  s->mask_B = 0;
  return PLF_OK;
}

// The colour pairs of an upload of image size s->geo[g] (arguments checked) into the landing buffer.
static plf_status upload_color(plf_ctx* ctx, int g, int B, const uint8_t* left, const uint8_t* right, int stride, int channels) {
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  plf_status st = pipe_prepare(ctx);
  if (st) return st;
  PipeState* s = ctx->pipe;
  uint8_t* land;
  if ((st = color_scratch(ctx, s, channels, &land))) return st;
  // H2D on the copy stream into the landing buffer; the run converts it into the image slot the GPU is not reading.
  // Dense rows of ch w bytes are one contiguous block per image (no short-row DMA to avoid, unlike the grey path's stage).
  const int row = channels * s->geo[g].w;
  if ((st = upload_pairs(ctx, s->copy, land, row, B, left, right, stride, row, s->geo[g].h))) return st;
  s->up_slot ^= 1;
  s->up_ch = channels;
  s->up_geo = g;
  s->uploaded = true;
  s->mask_B = 0;
  return PLF_OK;
}

// The refusals of the colour and sized uploads, fn naming the call: channels first when the call takes grey too.
static plf_status check_upload(plf_ctx* ctx, const char* fn, int B, int w, const uint8_t* left, const uint8_t* right,
                               int stride, int channels) {
  if (B < 1 || B > ctx->limits.max_batch)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: B = %d, need 1 <= B <= max_batch = %d", fn, B, ctx->limits.max_batch);
  if (!left || !right) return plf_fail(ctx, PLF_ERR_INVALID, "%s: left and right are required", fn);
  if ((long long)stride < (long long)channels * w)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: stride = %d, need at least channels * width = %d", fn, stride, channels * w);
  return PLF_OK;
}

plf_status plf_batch_upload(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride) {
  if (!ctx || !left || !right || B < 1 || B > ctx->limits.max_batch || stride < ctx->cam.width)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_upload: bad arguments (B=%d, max_batch=%d)", B, ctx ? ctx->limits.max_batch : 0);
  return upload_grey(ctx, 0, B, left, right, stride);
}

plf_status plf_batch_upload_color(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride, int channels) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_batch_upload_color: ctx is NULL");
  if (channels != 3 && channels != 4)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_upload_color: channels = %d, need 3 (BGR) or 4 (BGRA)", channels);
  if (plf_status st = check_upload(ctx, "plf_batch_upload_color", B, ctx->cam.width, left, right, stride, channels)) return st;
  return upload_color(ctx, 0, B, left, right, stride, channels);
}

plf_status plf_batch_upload_sized(plf_ctx* ctx, int B, int w, int h, const uint8_t* left, const uint8_t* right, int stride,
                                  int channels) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_batch_upload_sized: ctx is NULL");
  if (channels != 1 && channels != 3 && channels != 4)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_upload_sized: channels = %d, need 1 (grey), 3 (BGR) or 4 (BGRA)", channels);
  const int g = plf_image_size_index(ctx, w, h);
  if (g < 0)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_upload_sized: size %dx%d is not one of the context's image sizes (%s)", w, h,
                    image_size_list(ctx).c_str());
  if (plf_status st = check_upload(ctx, "plf_batch_upload_sized", B, w, left, right, stride, channels)) return st;
  return channels == 1 ? upload_grey(ctx, g, B, left, right, stride) : upload_color(ctx, g, B, left, right, stride, channels);
}

void* plf_batch_device_images(plf_ctx* ctx) {
  if (!ctx) return nullptr;
  if (pipe_prepare(ctx)) return nullptr;
  ctx->pipe->uploaded = true;
  return ctx->pipe->imgs2[ctx->pipe->up_slot];
}

plf_status plf_batch_upload_masks(plf_ctx* ctx, int B, const uint8_t* mask_l, const uint8_t* mask_r, int stride) {
  const char* fn = "plf_batch_upload_masks";
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "%s: ctx is NULL", fn);
  PipeState* s = ctx->pipe;
  if (!s || !s->uploaded)
    return plf_fail(ctx, PLF_ERR_STATE, "%s: no upload yet; the masks belong to the most recent upload, so upload the images first", fn);
  if (B < 1 || B > s->B) return plf_fail(ctx, PLF_ERR_INVALID, "%s: B = %d, need 1 <= B <= max_batch = %d", fn, B, s->B);
  if (!mask_l && !mask_r) return plf_fail(ctx, PLF_ERR_INVALID, "%s: mask_l and mask_r are both NULL; give at least one", fn);
  const PipeGeo& G = s->geo[s->up_geo];
  if (stride < G.w)
    return plf_fail(ctx, PLF_ERR_INVALID, "%s: stride = %d, need stride >= width = %d of the upload's images", fn, stride, G.w);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const uint8_t* src[2] = {mask_l, mask_r};
  const char* name[2] = {"mask_l", "mask_r"};
  for (int side = 0; side < 2; ++side) {
    if (!src[side]) continue;
    cudaPointerAttributes a = {};
    if (cudaPointerGetAttributes(&a, src[side]) != cudaSuccess) {
      cudaGetLastError();
      a.type = cudaMemoryTypeUnregistered;   // pageable host memory
    }
    if (a.type == cudaMemoryTypeDevice && a.device != ctx->device)
      return plf_fail(ctx, PLF_ERR_INVALID, "%s: %s is memory of device %d, and the context runs on device %d", fn, name[side], a.device,
                      ctx->device);
  }
  if (plf_status st = mask_scratch(ctx, s)) return st;
  // level 0 of image 2k + side's pyramid: mask k of that side, one 3-D copy per side (the destination "height" spans two
  // pyramids, skipping the other side's).  The copy waits for the runs that read the slot's pyramids before: their ORB
  // (ev_free) and KeyLine (ev_mfree) stages.
  const int slot = s->up_slot;
  const size_t img = mask_stride(G);
  cudaStream_t cs = s->copy;
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->ev_free[slot], 0));
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->ev_mfree[slot], 0));
  for (int side = 0; side < 2; ++side) {
    if (!src[side]) continue;
    cudaMemcpy3DParms cp = {};
    cp.srcPtr = make_cudaPitchedPtr(const_cast<uint8_t*>(src[side]), (size_t)stride, (size_t)G.w, (size_t)G.h);
    cp.dstPtr = make_cudaPitchedPtr(s->mpyr[slot] + side * img, (size_t)G.pitch, (size_t)G.w, 2 * img / G.pitch);
    cp.extent = make_cudaExtent((size_t)G.w, (size_t)G.h, (size_t)B);
    cp.kind = cudaMemcpyDefault;
    PLF_CUDA(ctx, cudaMemcpy3DAsync(&cp, cs));
  }
  s->mask_B = B;
  s->mask_side[0] = mask_l != nullptr;
  s->mask_side[1] = mask_r != nullptr;
  return PLF_OK;
}

plf_status plf_batch_device_layout(plf_ctx* ctx, int* w, int* h, int* pitch) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_batch_device_layout: ctx is NULL");
  if (!w || !h || !pitch) return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_device_layout: w, h and pitch are required");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  if (plf_status st = pipe_prepare(ctx)) return st;
  const PipeGeo& G = ctx->pipe->geo[ctx->pipe->up_geo];
  *w = G.w; *h = G.h; *pitch = G.pitch;
  return PLF_OK;
}

plf_status plf_set_image_sizes(plf_ctx* ctx, int n, const int32_t* wh) {
  if (!ctx) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_set_image_sizes: ctx is NULL");
  if (ctx->pipe) return plf_fail(ctx, PLF_ERR_STATE, "plf_set_image_sizes: the pipeline exists (a batch call was made)");
  if (n < 0 || n > PLF_MAX_IMAGE_SIZES)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_image_sizes: n = %d, need 0 <= n <= %d", n, PLF_MAX_IMAGE_SIZES);
  if (n > 0 && !wh) return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_image_sizes: wh is NULL");
  std::vector<int> sizes;
  for (int i = 0; i < n; ++i) {
    const int w = wh[2 * i], h = wh[2 * i + 1];
    if (w <= 0 || h <= 0)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_image_sizes: size %d is %dx%d, need a positive width and height", i, w, h);
    plf_status st = plf_orb_check_size(ctx, w, h);
    if (!st) st = plf_lsd_check_size(ctx, w, h);
    if (st) {
      const std::string why = ctx->err;
      return plf_fail(ctx, st, "plf_set_image_sizes: size %d (%dx%d): %s", i, w, h, why.c_str());
    }
    bool dup = w == ctx->cam.width && h == ctx->cam.height;
    for (size_t j = 0; j < sizes.size(); j += 2) dup |= sizes[j] == w && sizes[j + 1] == h;
    if (!dup) { sizes.push_back(w); sizes.push_back(h); }
  }
  // a sequence keeps its camera: its size stays one the context accepts
  for (size_t q = 0; q < ctx->seqs.size(); ++q) {
    const plf_camera& c = ctx->seqs[q].cam;
    if (!ctx->seqs[q].own_cam || (c.width == ctx->cam.width && c.height == ctx->cam.height)) continue;
    bool kept = false;
    for (size_t j = 0; j < sizes.size(); j += 2) kept |= sizes[j] == c.width && sizes[j + 1] == c.height;
    if (!kept)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_set_image_sizes: sequence %zu has a camera of %dx%d, which the new sizes do not "
                      "hold; give it another camera first", q, c.width, c.height);
  }
  ctx->image_sizes = sizes;
  return PLF_OK;
}

plf_status plf_get_image_geometry(const plf_params* params, int w, int h, plf_image_geometry* out) {
  if (!out) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_get_image_geometry: out is NULL");
  plf_ctx c;   // host only: the parameters and the limits are all the checks read
  if (params) c.params = *params;
  else plf_default_params(&c.params);
  plf_default_limits(&c.limits);
  memset(out, 0, sizeof *out);
  plf_status st = w > 0 && h > 0 ? PLF_OK : plf_fail(&c, PLF_ERR_INVALID, "size %dx%d, need a positive width and height", w, h);
  if (!st) st = plf_orb_check_size(&c, w, h, &out->orb_nlevels, out->orb_w, out->orb_h);
  if (!st) st = plf_lsd_check_size(&c, w, h, &out->lsd_w, &out->lsd_h);
  if (st) return plf_fail(nullptr, st, "plf_get_image_geometry: %s", c.err.c_str());
  out->pitch = plf_pitch16(w);
  out->grid_iw = PLF_GRID_COLS / (double)w;
  out->grid_ih = PLF_GRID_ROWS / (double)h;
  return PLF_OK;
}

plf_status plf_batch_run(plf_ctx* ctx, int B) { return plf_batch_run_sequences(ctx, B, nullptr, nullptr); }

plf_status plf_batch_run_sequences(plf_ctx* ctx, int B, const int32_t* seq, const uint8_t* restart) {
  if (!ctx || B < 1 || B > ctx->limits.max_batch) return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_run: bad B");
  if (seq)
    for (int k = 0; k < B; ++k)
      if (plf_status st = plf_check_sequence(ctx, "plf_batch_run_sequences", seq[k], k)) return st;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  plf_status st = pipe_prepare(ctx);
  if (st) return st;
  PipeState* s = ctx->pipe;
  if (s->n_pending >= 3)
    return plf_fail(ctx, PLF_ERR_STATE, "plf_batch_run: three batches already in flight; call plf_batch_download first");
  if (seq) s->pair_seq.assign(seq, seq + B);
  else s->pair_seq.assign(B, 0);
  const int* q = s->pair_seq.data();
  if (s->mask_B && B != s->mask_B)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_run_sequences: B = %d, and the masks of the upload it runs (plf_batch_upload_masks) "
                    "are of %d pairs", B, s->mask_B);
  // a batch is of one image size, its upload's
  const PipeGeo& G = s->geo[s->up_geo];
  for (int k = 0; k < B; ++k) {
    const plf_camera& c = plf_sequence_camera(ctx, q[k]);
    if (c.width != G.w || c.height != G.h)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_run_sequences: pair %d is of sequence %d, of %dx%d images, and the upload it "
                      "runs is of %dx%d; a batch holds pairs of one image size", k, q[k], c.width, c.height, G.w, G.h);
  }
  // pair k of a sequence is detected at the threshold pair k-1's pose gives, or starts from the prediction pair k-1's pose
  // gives: one pair per sequence
  if (ctx->afast_on || ctx->motion_on) {
    int first = -1, dup = -1;
    for (int k = 0; k < B && dup < 0; ++k) {
      int& last = s->last_pair[q[k]];
      if (last >= 0) { first = last; dup = k; }
      else last = k;
    }
    for (int k = 0; k < B; ++k) s->last_pair[q[k]] = -1;
    if (dup >= 0)
      return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_run_sequences: pairs %d and %d are both of sequence %d; with %s a batch "
                      "holds at most one pair of each sequence", first, dup, q[dup],
                      ctx->afast_on ? "adaptive FAST thresholds (plf_set_adaptive_fast)" : "the motion model (plf_set_motion_model)");
  }
  BatchRun r;
  r.B = B;
  r.g = s->up_geo;
  r.par = (int)(s->seq & 1);
  r.rp = (int)(s->seq % 3);
  // The batch's table, into its ring entry (the batch that used it last has been downloaded, and its input conversion
  // ran before its ev_up).  Pair k tracks against the batch's previous pair of its sequence, else the sequence's carried
  // frame, else (and on a restart) nothing
  const BatchTab tab = host_tab(s, r.rp);
  int32_t* prev = tab.prev;
  int32_t* carry = tab.carry;
  const int empty = s->B + s->nseq;
  for (int k = 0; k < B; ++k) {
    if (restart && restart[k]) prev[k] = empty;
    else if (s->last_pair[q[k]] >= 0) prev[k] = s->last_pair[q[k]];
    else prev[k] = s->carried[q[k]] ? s->B + q[k] : empty;
    s->last_pair[q[k]] = k;
  }
  r.ncarry = 0;
  for (int k = 0; k < B; ++k) {
    if (s->last_pair[q[k]] != k) continue;
    carry[2 * r.ncarry] = k;
    carry[2 * r.ncarry + 1] = s->B + q[k];
    r.ncarry++;
  }
  // the cameras, settings, maps and masks of the pairs, resolved now: a later plf_set_sequence_camera, _params,
  // _rectification or _mask does not reach this batch.  The input table of a grey batch lists its rectified pairs; a colour
  // batch, converted whole, lists every pair when one of them is rectified.
  r.nin = 0;
  r.masked = false;
  r.nbuild = 0;
  r.nwin = 0;
  r.best_lr = false;
  bool rect = false;
  for (int k = 0; k < B; ++k) {
    const plf_camera& c = plf_sequence_camera(ctx, q[k]);
    tab.cams[k] = PlfPairCam{c.fx, c.fy, c.cx, c.cy, c.b};
    tab.prm[k] = plf_sequence_pair(ctx, q[k]);
    r.nwin += tab.prm[k].matching_strategy != 0;
    r.best_lr |= tab.prm[k].best_lr != 0;
    const PlfSequence* sq = ctx->seqs.empty() ? nullptr : &ctx->seqs[q[k]];
    const uint8_t* maps = sq ? sq->rect : nullptr;
    if (maps || s->up_ch > 1) tab.in[r.nin++] = PlfRectPair{maps, k, 0};
    rect |= maps != nullptr;
    for (int side = 0; side < 2; ++side) {
      const int z = 2 * k + side;
      const uint8_t* seq_mask = sq ? sq->mask[side] : nullptr;
      if (s->mask_B && s->mask_side[side]) {
        uint8_t* pyr = s->mpyr[s->up_slot] + z * mask_stride(G);
        tab.build[r.nbuild++] = PlfMaskBuild{pyr, seq_mask};
        tab.masks[z] = pyr;
      } else {
        tab.masks[z] = seq_mask;
      }
      r.masked |= tab.masks[z] != nullptr;
    }
  }
  if (!rect) r.nin = 0;
  r.run_slot = s->up_slot;
  // With profiling on everything is serialised on the main stream so that the per-kernel marks are meaningful.
  r.piped = !ctx->profile || ctx->profile_piped;
  r.lsd2 = s->lsd2;
  r.lp = r.lsd2 ? r.par : 0;
  r.sM = ctx->stream;
  r.sE = r.piped ? ctx->aux[0] : r.sM;
  r.sG = r.piped ? ctx->aux[1] : r.sM;
  r.sP = (r.piped && r.lsd2) ? ctx->aux[2] : r.sG;   // LSD pre-grow chain: own stream when its outputs exist per parity
  r.afast = ctx->afast_on;
  r.motion = ctx->motion_on;
  st = send_tab(ctx, s, r);
  if (!st) st = run_input(ctx, s, r);
  if (!st) st = run_masks(ctx, s, r);
  if (!st) st = run_extract(ctx, s, r);
  if (!st) st = run_lsd(ctx, s, r);
  if (!st) st = run_match(ctx, s, r);
  for (int k = 0; k < B; ++k) {
    s->last_pair[q[k]] = -1;
    if (!st) s->carried[q[k]] = 1;
  }
  if (st) return st;
  s->mask_B = 0;   // the run has taken the upload's masks
  s->pend_slot[s->n_pending] = r.rp;
  s->pend_B[s->n_pending] = B;
  s->rp_geo[r.rp] = r.g;
  s->n_pending++;
  s->seq++;
  return PLF_OK;
}

// Results of the OLDEST batch in flight (FIFO): waits for its match phase only, so a later batch keeps running.
plf_status plf_batch_download(plf_ctx* ctx, int B, plf_frame_result* out) {
  if (!ctx || !ctx->pipe || !out || B < 1 || B > ctx->limits.max_batch)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_download: bad arguments");
  PipeState* s = ctx->pipe;
  if (s->n_pending == 0) return plf_fail(ctx, PLF_ERR_STATE, "plf_batch_download: no batch in flight");
  const int par = s->pend_slot[0];
  if (B != s->pend_B[0])
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_download: B=%d but the oldest batch in flight has %d pairs", B, s->pend_B[0]);
  PLF_CUDA(ctx, cudaEventSynchronize(s->evM[par]));
  s->pend_slot[0] = s->pend_slot[1]; s->pend_slot[1] = s->pend_slot[2];
  s->pend_B[0] = s->pend_B[1]; s->pend_B[1] = s->pend_B[2];
  s->n_pending--;
  memcpy(out, s->h_results[par], sizeof(plf_frame_result) * B);
  // an overflow of a disabled kind's extraction buffers does not reach the results
  const int o0 = ctx->params.has_points ? s->h_ovf[par][0] : 0, o1 = ctx->params.has_lines ? s->h_ovf[par][1] : 0;
  if (o0 || o1) {
    char why0[400] = "", why1[400] = "";
    const PipeGeo& G = s->geo[s->rp_geo[par]];   // the capacities of the batch's own image size
    if (o0) plf_orb_overflow_text(G.orb, o0, why0, sizeof why0);
    if (o1) plf_lsd_overflow_text(G.lsd, o1, why1, sizeof why1);
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_batch_download: a fixed-capacity buffer overflowed in this batch (%s%s%s%s%s)",
                    o0 ? "ORB keypoints: " : "", why0, o0 && o1 ? "; " : "", o1 ? "LSD segments/lines: " : "", why1);
  }
  return PLF_OK;
}

// Device-resident poses of the OLDEST batch in flight: copies DT (16 f64, row-major) of its B frames into the caller's
// DEVICE buffer dst[B][16] on the CALLER's stream, behind that batch's end-of-match-phase event - what a multi-GPU
// caller hands to its NCCL all-gather (issued on the same stream) without a host round trip and without queueing behind
// the later batches already enqueued on the library's own streams.  Does not retire the batch.
plf_status plf_batch_device_poses(plf_ctx* ctx, int B, double* dst_device, void* stream) {
  if (!ctx || !ctx->pipe || !dst_device || B < 1) return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_device_poses: bad arguments");
  PipeState* s = ctx->pipe;
  if (s->n_pending == 0) return plf_fail(ctx, PLF_ERR_STATE, "plf_batch_device_poses: no batch in flight");
  if (B != s->pend_B[0]) return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_device_poses: B=%d but the oldest batch has %d pairs", B, s->pend_B[0]);
  const int rp = s->pend_slot[0];
  cudaStream_t cs = stream ? (cudaStream_t)stream : s->copy;
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->evM[rp], 0));
  PLF_CUDA(ctx, cudaMemcpy2DAsync(dst_device, 16 * sizeof(double), s->results + (size_t)rp * s->B, sizeof(plf_frame_result),
                                  16 * sizeof(double), B, cudaMemcpyDeviceToDevice, cs));
  if (!stream) PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

// Timeline of the two most recent batches (device clock, ms): for parity p = 0,1 the start and end of the E, G and M
// phases relative to the earlier of the two E starts.  Call with nothing in flight.
plf_status plf_debug_timeline(plf_ctx* ctx, float out[12]) {
  if (!ctx || !ctx->pipe || !out) return plf_fail(ctx, PLF_ERR_INVALID, "plf_debug_timeline: bad arguments");
  PipeState* s = ctx->pipe;
  if (s->n_pending) return plf_fail(ctx, PLF_ERR_STATE, "plf_debug_timeline: batches in flight");
  if (s->seq < 2) return plf_fail(ctx, PLF_ERR_STATE, "plf_debug_timeline: needs two completed batches");
  PLF_CUDA(ctx, cudaDeviceSynchronize());
  const int p0 = (int)(s->seq & 1);  // parity of the older of the last two batches
  cudaEvent_t ref = s->tE0[p0];
  for (int k = 0; k < 2; ++k) {
    const int p = k == 0 ? p0 : p0 ^ 1;
    const int r = (int)((s->seq - 2 + k) % 3);
    cudaEvent_t ev[6] = {s->tE0[p], s->evE[p], s->tG0[p], s->evG[p], s->tM0[r], s->evM[r]};
    for (int j = 0; j < 6; ++j) PLF_CUDA(ctx, cudaEventElapsedTime(&out[k * 6 + j], ref, ev[j]));
  }
  return PLF_OK;
}

plf_status plf_process_batch(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride,
                             plf_frame_result* out) {
  plf_status st = plf_batch_upload(ctx, B, left, right, stride);
  if (st) return st;
  if ((st = plf_batch_run(ctx, B))) return st;
  return plf_batch_download(ctx, B, out);
}

// Copies the stereo-valid features of frame k of the last batch to host arrays (any pointer may be NULL).
plf_status plf_get_frame(plf_ctx* ctx, int k, plf_frame_view* v) {
  if (!ctx || !ctx->pipe || !v || k < 0 || k >= ctx->limits.max_batch)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_get_frame: bad arguments");
  PipeState* s = ctx->pipe;
  FrameSlots& f = s->fs;
  const int slot = k;
  const size_t K = s->max_kp, Ln = s->max_ln;
  cudaStream_t cs = ctx->stream;
  int np = 0, nl = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&np, f.pt_count + slot, 4, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(&nl, f.ls_count + slot, 4, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  v->n_pt = np; v->n_ls = nl;
  if (np > v->cap_pt || nl > v->cap_ls)
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_get_frame: %d points / %d lines exceed the view capacity", np, nl);
#define GET(name, n, cap, per)                                                                                       \
  if (v->name && (n) > 0)                                                                                            \
    PLF_CUDA(ctx, cudaMemcpyAsync(v->name, f.name + (size_t)slot * cap * per, (size_t)(n) * per * sizeof(*f.name),   \
                                  cudaMemcpyDeviceToHost, cs));
#define GET_PT(name, T, cap, per) GET(name, np, cap, per)
#define GET_LS(name, T, cap, per) GET(name, nl, cap, per)
  PLF_PT_FIELDS(GET_PT)
  PLF_LS_FIELDS(GET_LS)
#undef GET_LS
#undef GET_PT
#undef GET
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

// Frame-to-frame correspondences of pair k of the last batch: what f2fTracking leaves in matched_pt / matched_ls
// (P / sP,eP from the previous frame, pl_obs / le_obs from the current one, inlier flags after optimizePose).
plf_status plf_get_matches(plf_ctx* ctx, int k, plf_match_view* v) {
  if (!ctx || !ctx->pipe || !v || k < 0 || k >= ctx->limits.max_batch)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_get_matches: bad arguments");
  PipeState* s = ctx->pipe;
  const size_t K = s->max_kp, Ln = s->max_ln;
  cudaStream_t cs = ctx->stream;
  int np = 0, nl = 0;
  PLF_CUDA(ctx, cudaMemcpyAsync(&np, s->gnNp + k, 4, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(&nl, s->gnNl + k, 4, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  v->n_pt = np; v->n_ls = nl;
  if (np > v->cap_pt || nl > v->cap_ls)
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_get_matches: %d points / %d lines exceed the view capacity", np, nl);
#define GETM(dst, src, per, n, base) if ((dst) && (n) > 0) PLF_CUDA(ctx, cudaMemcpyAsync((dst), (const char*)(src) + (size_t)k * (base) * (per), (size_t)(n) * (per), cudaMemcpyDeviceToHost, cs))
  GETM(v->P, s->gnP, 24, np, K); GETM(v->pl_obs, s->gnObs, 16, np, K); GETM(v->inlier_pt, s->gnInlP, 1, np, K);
  GETM(v->sP, s->gn_sP, 24, nl, Ln); GETM(v->eP, s->gn_eP, 24, nl, Ln); GETM(v->le_obs, s->gn_le, 24, nl, Ln);
  GETM(v->inlier_ls, s->gnInlL, 1, nl, Ln);
#undef GETM
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

}  // extern "C"
