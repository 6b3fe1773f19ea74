// Batched stereo front-end: extraction -> L/R stereo association -> frame-to-frame tracking -> pose refinement
// (SURVEY §8 a6, a7, a10 and the call pattern of app/plslam_dataset.cpp:111-163).
//
// Replaces, per stereo pair: StereoFrameHandler::insertStereoPair (app/plslam_dataset.cpp:127) = new StereoFrame +
// extractStereoFeatures (ORB + LSD/LBD on both images, matchStereoPoints / matchStereoLines) + f2fTracking, and
// StereoFrameHandler::optimizePose (app/plslam_dataset.cpp:128).  stvo-pl is not vendored by the reference; the
// association rules restate SURVEY.md Appendix A.2/A.3 (see oracle/frontend.py, which this file must match
// bit-for-bit on features / matches and to 1e-4 on the pose).
//
// One call processes B consecutive stereo pairs of ONE sequence.  Everything except the final SE(3) chaining is
// independent per pair (extraction, stereo association) or per consecutive pair (tracking and the pose increment
// start from identity: use_motion_model = false, config_euroc.yaml:18), so all B pairs run in the same launches:
// images [2B][H][W] (2k = left, 2k+1 = right) -> ORB / LSD / LBD over 2B images -> per-pair kernels.  The last
// frame's stereo features are carried to the next call (slot 0).
#include "plf_internal.h"
#include "plf_geom.cuh"
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

struct PipeState {
  int w = 0, h = 0, B = 0, max_kp = 0, max_ln = 0;
  int pitch = 0;               // row pitch of the device images: plf_pitch16(w) (16-byte rows: every halo tile is a legal TMA box)
  bool has_prev = false;
  uint8_t* imgs2[2] = {nullptr, nullptr};  // double-buffered [2B][h][pitch]: upload of batch i+1 overlaps the run of batch i
  uint8_t* stage = nullptr;    // dense [2B][h][w] landing buffer of the H2D copy (one contiguous DMA per side), repacked to the padded pitch on the device
  int up_slot = 0;             // slot written by the last plf_batch_upload
  cudaStream_t copy = nullptr; // H2D stream
  cudaEvent_t ev_up[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr}, ev_free2[2] = {nullptr, nullptr};
  short2* lbd_grad[2] = {nullptr, nullptr};  // [parity][2B][h*w]
  uint8_t* ldesc_raw = nullptr;  // [2B][max_ln][32]  LBD of every kept KeyLine
  FrameSlots fs;               // B+1 slots
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
  DevBufList bufs;
};

// The device buffers of the pipeline for B pairs of K keypoints / Ln lines per image.
static void pipe_buffers(PipeState* s, bool windowed, DevBufList& b) {
  const size_t B = s->B, K = s->max_kp, Ln = s->max_ln, A = (size_t)s->w * s->h, AP = (size_t)s->pitch * s->h, S = B + 1;
  b.add(s->imgs2[0], 2 * B * AP);
  b.add(s->imgs2[1], 2 * B * AP);
  if (s->pitch != s->w) b.add(s->stage, 2 * B * A);
  b.add(s->lbd_grad[0], 2 * B * A);
  b.add(s->lbd_grad[1], 2 * B * A);
  b.add(s->ldesc_raw, 2 * B * Ln * 32);
  FrameSlots& f = s->fs;
#define PLF_FS_ALLOC(name, T, cap, per) b.add(f.name, S * cap * per);
  PLF_PT_FIELDS(PLF_FS_ALLOC) b.add(f.pt_count, S);
  PLF_LS_FIELDS(PLF_FS_ALLOC) b.add(f.ls_count, S);
#undef PLF_FS_ALLOC
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
          {s->tE0, 2, cudaEventDefault},         {s->tG0, 2, cudaEventDefault}};
}

extern "C" void plf_pipe_free(plf_ctx* ctx) {
  PipeState* s = ctx->pipe;
  if (!s) return;
  s->bufs.release();
  for (int i = 0; i < 3; ++i) {
    if (s->h_results[i]) cudaFreeHost(s->h_results[i]);
    if (s->h_ovf[i]) cudaFreeHost(s->h_ovf[i]);
  }
  for (const PipeEvents& a : pipe_events(s))
    for (int i = 0; i < a.n; ++i)
      if (a.ev[i]) cudaEventDestroy(a.ev[i]);
  if (s->copy) { cudaStreamSynchronize(s->copy); cudaStreamDestroy(s->copy); }
  delete s;
  ctx->pipe = nullptr;
}

struct StereoPrm {
  float max_dist_epip, min_disp, line_horiz_th, stereo_overlap_th, ls_min_disp_ratio;
  double fx, fy, cx, cy, b;
};

__device__ __forceinline__ void back_projection(const StereoPrm& c, double u, double v, double disp, double* P) {
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

// matchStereoPoints: epipolar + disparity gates, back-projection, compaction in left-index order.
__global__ void __launch_bounds__(1024) k_stereo_points(const plf_keypoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                                         const int* __restrict__ kp_count, int max_kp,
                                                         const int32_t* __restrict__ m12_all, int m12_stride, StereoPrm prm,
                                                         FrameSlots fs, int slot0) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int il = 2 * k, ir = 2 * k + 1, slot = slot0 + k;
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
        if (fabsf(__fsub_rn(a.y, b.y)) <= prm.max_dist_epip) {
          d = (double)__fsub_rn(a.x, b.x);
          ok = d >= (double)prm.min_disp;
        }
      }
    }
    const int incl = block_scan_flags(ok, s_scan, &s_total);
    if (ok) {
      const size_t o = (size_t)slot * max_kp + base + incl - 1;
      fs.pt_pl[o] = make_double2((double)xl, (double)yl);
      fs.pt_disp[o] = d;
      back_projection(prm, (double)xl, (double)yl, d, fs.pt_P + 3 * o);
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

// matchStereoLines
__global__ void __launch_bounds__(1024) k_stereo_lines(const plf_keyline* __restrict__ kls, const uint8_t* __restrict__ ldesc,
                                                        const int* __restrict__ nlines, int max_ln,
                                                        const int32_t* __restrict__ m12_all, int m12_stride, StereoPrm prm,
                                                        FrameSlots fs, int slot0) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int il = 2 * k, ir = 2 * k + 1, slot = slot0 + k;
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
        const double overlap = line_overlap_stereo(syl, eyl, syr, eyr, (double)prm.line_horiz_th);
        const double sx_on_r = -(r2 + r1 * syl) / r0;
        const double ex_on_r = -(r2 + r1 * eyl) / r0;
        disp_s = sxl - sx_on_r;
        disp_e = exl - ex_on_r;
        if (!(fmin(disp_s, disp_e) / fmax(disp_s, disp_e) >= (double)prm.ls_min_disp_ratio)) disp_s = disp_e = -1.0;
        ok = disp_s >= (double)prm.min_disp && disp_e >= (double)prm.min_disp &&
             fabsf((float)r0) > prm.line_horiz_th && overlap > (double)prm.stereo_overlap_th;
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
      back_projection(prm, spl[0], spl[1], disp_s, fs.ls_sP + 3 * o);
      back_projection(prm, epl[0], epl[1], disp_e, fs.ls_eP + 3 * o);
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

// f2fTracking: gather the matched rows into the GN problem of pair k (prev slot = slot0+k-1 ... see host code)
__global__ void __launch_bounds__(1024) k_f2f_build(FrameSlots fs, int prev_slot0, int max_kp, int max_ln,
                                                    const int32_t* __restrict__ m_pt_all, const int32_t* __restrict__ m_ls_all,
                                                    int m_stride, double* __restrict__ gnP, double* __restrict__ gnObs,
                                                    uint8_t* __restrict__ gnInlP, int* __restrict__ gnNp,
                                                    double* __restrict__ gn_sP, double* __restrict__ gn_eP,
                                                    double* __restrict__ gn_le, uint8_t* __restrict__ gnInlL,
                                                    int* __restrict__ gnNl) {
  __shared__ int s_scan[1024];
  __shared__ int s_total;
  const int k = blockIdx.x, tid = threadIdx.x;
  const int ps = prev_slot0 + k, cs = ps + 1;
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

// optimizePose epilogue: curr.DT = inverse_se3(T_inc); identity when there were too few correspondences
__global__ void k_finalize(const plf_pose_result* __restrict__ gn, const int* __restrict__ gnNp, const int* __restrict__ gnNl,
                           const int* __restrict__ kp_count, const int* __restrict__ nlines, FrameSlots fs, int slot0,
                           int min_features, int first_is_init, int B, plf_frame_result* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= B) return;
  plf_frame_result r;
  for (int i = 0; i < 16; ++i) r.DT[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 36; ++i) r.DT_cov[i] = 0.0;
  r.err = -1.0;
  r.n_kp_l = kp_count[2 * k]; r.n_kp_r = kp_count[2 * k + 1];
  r.n_lines_l = nlines[2 * k]; r.n_lines_r = nlines[2 * k + 1];
  r.n_stereo_pt = fs.pt_count[slot0 + k]; r.n_stereo_ls = fs.ls_count[slot0 + k];
  r.n_matched_pt = r.n_matched_ls = r.n_inliers_pt = r.n_inliers_ls = r.iters1 = r.iters2 = 0;
  if (k == 0 && first_is_init) {
    r.status = 2;
  } else {
    const plf_pose_result& g = gn[k];
    r.n_matched_pt = gnNp[k]; r.n_matched_ls = gnNl[k];
    if (r.n_matched_pt + r.n_matched_ls < min_features) {
      r.status = 1;
    } else {
      r.status = 0;
      const double* T = g.T;
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) r.DT[4 * i + j] = T[4 * j + i];
        r.DT[4 * i + 3] = -(T[i] * T[3] + T[4 + i] * T[7] + T[8 + i] * T[11]);
      }
      for (int i = 0; i < 36; ++i) r.DT_cov[i] = g.cov[i];
      r.err = g.err;
      r.n_inliers_pt = g.n_inliers_pt; r.n_inliers_ls = g.n_inliers_ls;
      r.iters1 = g.iters1; r.iters2 = g.iters2;
    }
  }
  out[k] = r;
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

// frame-to-frame: queries = the previous frame's 3-D features projected with DT = identity (slot k), train = the
// current frame's image features (slot k+1)
__global__ void __launch_bounds__(256) k_mg_geom_f2f(FrameSlots fs, int K, int Ln, StereoPrm c, double iw, double ih,
                                                     int* __restrict__ qp, int* __restrict__ tp, int* __restrict__ ql,
                                                     int* __restrict__ tl, double* __restrict__ tdir) {
  const int k = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  const int ps = k, cs = k + 1;
  if (i < min(fs.pt_count[ps], K)) {
    const double* P = fs.pt_P + 3 * ((size_t)ps * K + i);
    const double2 u = plf_project(c.fx, c.fy, c.cx, c.cy, P[0], P[1], P[2]);
    qp[((size_t)k * K + i) * 2] = mg_cell(u.x * iw);
    qp[((size_t)k * K + i) * 2 + 1] = mg_cell(u.y * ih);
  }
  if (i < min(fs.pt_count[cs], K)) {
    const double2 p = fs.pt_pl[(size_t)cs * K + i];
    tp[((size_t)k * K + i) * 2] = mg_cell(p.x * iw);
    tp[((size_t)k * K + i) * 2 + 1] = mg_cell(p.y * ih);
  }
  if (i < min(fs.ls_count[ps], Ln)) {
    const double* S = fs.ls_sP + 3 * ((size_t)ps * Ln + i);
    const double* E = fs.ls_eP + 3 * ((size_t)ps * Ln + i);
    int* d = ql + ((size_t)k * Ln + i) * 4;
    d[0] = mg_cell(plf_project_u(c.fx, c.cx, S[0], S[2]) * iw); d[1] = mg_cell(plf_project_v(c.fy, c.cy, S[1], S[2]) * ih);
    d[2] = mg_cell(plf_project_u(c.fx, c.cx, E[0], E[2]) * iw); d[3] = mg_cell(plf_project_v(c.fy, c.cy, E[1], E[2]) * ih);
  }
  if (i < min(fs.ls_count[cs], Ln))
    plf_train_line(fs.ls_spl[(size_t)cs * Ln + i], fs.ls_epl[(size_t)cs * Ln + i], iw, ih, tl + ((size_t)k * Ln + i) * 4,
                   tdir + ((size_t)k * Ln + i) * 2);
}

// src/mapHandler.cpp:274-278 / :421-425: keep the windowed result unless both frames hold more than `kmin` features and
// fewer than `kmin` matches survived - then the brute-force match() result (already in m12) stands.
__global__ void __launch_bounds__(256) k_mg_select(const int32_t* __restrict__ m12g, const int* __restrict__ mgcount,
                                                   const int* __restrict__ cnt, int cap, int K, int which, int kmin,
                                                   int32_t* __restrict__ m12) {
  const int k = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  const int n1 = min(cnt[k], cap), n2 = min(cnt[k + 1], cap);
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
static bool lsd_want_two_parities(const plf_ctx* ctx, int w, int h, int nimg) {
  const char* e = getenv("PLF_LSD_PARITIES");
  if (e && *e) return atoi(e) >= 2;
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return plf_lsd_footprint(ctx, w, h, nimg, true) + LSD_PARITY_MARGIN <= free_b;
}

static plf_status pipe_build(plf_ctx* ctx, int w, int h) {
  PipeState* s = ctx->pipe = new PipeState();
  const int B = ctx->limits.max_batch, K = ctx->limits.max_keypoints, Ln = ctx->limits.max_lines;
  if (Ln > K || K > 65535)
    return plf_fail(ctx, PLF_ERR_INVALID, "limits: need max_lines <= max_keypoints <= 65535 (got %d, %d)", Ln, K);
  s->w = w; s->h = h; s->B = B; s->max_kp = K; s->max_ln = Ln;
  s->pitch = plf_pitch16(w);
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
  }
  FrameSlots& f = s->fs;
  cudaStream_t cs = ctx->stream;
  PLF_CUDA(ctx, cudaMemsetAsync(f.pt_count, 0, (B + 1) * sizeof(int), cs));
  PLF_CUDA(ctx, cudaMemsetAsync(f.ls_count, 0, (B + 1) * sizeof(int), cs));
  // sub-systems sized for 2B images
  if ((st = plf_orb_prepare(ctx, w, h, 2 * B, true))) return st;
  s->lsd2 = lsd_want_two_parities(ctx, w, h, 2 * B);
  if ((st = plf_lsd_prepare(ctx, w, h, 2 * B, s->lsd2))) return st;
  // static problem descriptors over the pipeline's own buffers (pointers never change; counts are read on the device):
  // the stereo problems read the match phase's copies of the extraction outputs
  const int* kcnt = s->kcntM;
  const int* lcnt = s->lcntM;
  const int best_lr = P.best_lr_matches ? 1 : 0;
  std::vector<KnnProblem> ks(B * 4), kf(B * 4);
  std::vector<NnrProblem> ns(B * 2), nf(B * 2);
  std::vector<GnProblem> gp(B);
  for (int k = 0; k < B; ++k) {
    auto key = [&](int prob, int which) { return s->knn_keys + (((size_t)k * 8 + prob) * 2 + which) * K; };
    auto m12 = [&](int kind) { return s->m12 + ((size_t)k * 4 + kind) * K; };
    const uint32_t* dl = (const uint32_t*)(s->descM + (size_t)(2 * k) * K * 32);
    const uint32_t* dr = (const uint32_t*)(s->descM + (size_t)(2 * k + 1) * K * 32);
    const uint32_t* ll = (const uint32_t*)(s->ldesc_raw + (size_t)(2 * k) * Ln * 32);
    const uint32_t* lr = (const uint32_t*)(s->ldesc_raw + (size_t)(2 * k + 1) * Ln * 32);
    // forward problems (all left rows), then reverse problems restricted to the right rows the mutual check will read
    ks[2 * k + 0] = {dl, dr, kcnt + 2 * k, kcnt + 2 * k + 1, 0, 0, key(0, 0), key(0, 1), nullptr};
    ks[2 * k + 1] = {ll, lr, lcnt + 2 * k, lcnt + 2 * k + 1, 0, 0, key(2, 0), key(2, 1), nullptr};
    ks[2 * B + 2 * k + 0] = {dr, dl, s->rev_count + 2 * k, kcnt + 2 * k, 0, 0, key(1, 0), key(1, 1), s->rev_list + (size_t)(2 * k) * K};
    ks[2 * B + 2 * k + 1] = {lr, ll, s->rev_count + 2 * k + 1, lcnt + 2 * k, 0, 0, key(3, 0), key(3, 1), s->rev_list + (size_t)(2 * k + 1) * K};
    ns[2 * k + 0] = {key(0, 0), key(0, 1), key(1, 0), key(1, 1), kcnt + 2 * k, kcnt + 2 * k + 1, 0, 0, P.min_ratio_12_p, best_lr, m12(0), s->mcount + 4 * k + 0};
    ns[2 * k + 1] = {key(2, 0), key(2, 1), key(3, 0), key(3, 1), lcnt + 2 * k, lcnt + 2 * k + 1, 0, 0, P.min_ratio_12_l, best_lr, m12(1), s->mcount + 4 * k + 1};
    // f2f: prev slot k, curr slot k+1
    const uint32_t* pp = (const uint32_t*)(f.pdesc + (size_t)k * K * 32);
    const uint32_t* pc = (const uint32_t*)(f.pdesc + (size_t)(k + 1) * K * 32);
    const uint32_t* lp = (const uint32_t*)(f.ldesc + (size_t)k * Ln * 32);
    const uint32_t* lc = (const uint32_t*)(f.ldesc + (size_t)(k + 1) * Ln * 32);
    kf[4 * k + 0] = {pp, pc, f.pt_count + k, f.pt_count + k + 1, 0, 0, key(4, 0), key(4, 1)};
    kf[4 * k + 1] = {pc, pp, f.pt_count + k + 1, f.pt_count + k, 0, 0, key(5, 0), key(5, 1)};
    kf[4 * k + 2] = {lp, lc, f.ls_count + k, f.ls_count + k + 1, 0, 0, key(6, 0), key(6, 1)};
    kf[4 * k + 3] = {lc, lp, f.ls_count + k + 1, f.ls_count + k, 0, 0, key(7, 0), key(7, 1)};
    nf[2 * k + 0] = {key(4, 0), key(4, 1), key(5, 0), key(5, 1), f.pt_count + k, f.pt_count + k + 1, 0, 0, P.min_ratio_12_p, best_lr, m12(2), s->mcount + 4 * k + 2};
    nf[2 * k + 1] = {key(6, 0), key(6, 1), key(7, 0), key(7, 1), f.ls_count + k, f.ls_count + k + 1, 0, 0, P.min_ratio_12_l, best_lr, m12(3), s->mcount + 4 * k + 3};
    gp[k] = {s->gnP + (size_t)k * K * 3, s->gnObs + (size_t)k * K * 2, s->gnInlP + (size_t)k * K, s->gnNp + k, 0,
             s->gn_sP + (size_t)k * Ln * 3, s->gn_eP + (size_t)k * Ln * 3, s->gn_le + (size_t)k * Ln * 3,
             s->gnInlL + (size_t)k * Ln, s->gnNl + k, 0, nullptr, s->gn_out + k};
  }
  PLF_CUDA(ctx, cudaMemcpyAsync(s->knn_stereo, ks.data(), ks.size() * sizeof(KnnProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->nnr_stereo, ns.data(), ns.size() * sizeof(NnrProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->knn_f2f, kf.data(), kf.size() * sizeof(KnnProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->nnr_f2f, nf.data(), nf.size() * sizeof(NnrProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->gn_probs, gp.data(), gp.size() * sizeof(GnProblem), cudaMemcpyHostToDevice, cs));
  PLF_CUDA(ctx, cudaStreamSynchronize(cs));
  return PLF_OK;
}

static plf_status pipe_prepare(plf_ctx* ctx, int w, int h) {
  PipeState* s = ctx->pipe;
  if (s && s->w == w && s->h == h) {
    // a standalone operator call on another image size may have rebuilt the ORB / LSD state meanwhile: rebuild it again.
    // No pipeline buffer or problem descriptor points into that state, so the sequence goes on where it was.
    const plf_status st = plf_orb_prepare(ctx, w, h, 2 * s->B, true);
    return st ? st : plf_lsd_prepare(ctx, w, h, 2 * s->B, s->lsd2);
  }
  plf_pipe_free(ctx);
  const plf_status st = pipe_build(ctx, w, h);
  if (st) plf_pipe_free(ctx);   // a failed setup leaves no state behind (see plf_orb_prepare)
  return st;
}

static plf_status copy_slot(plf_ctx* ctx, PipeState* s, int from, int to) {
  FrameSlots& f = s->fs;
  const size_t K = s->max_kp, Ln = s->max_ln;
  cudaStream_t cs = ctx->stream;
#define CP(ptr, per) PLF_CUDA(ctx, cudaMemcpyAsync((ptr) + (size_t)to * (per), (ptr) + (size_t)from * (per), (per) * sizeof(*(ptr)), cudaMemcpyDeviceToDevice, cs));
#define PLF_FS_COPY(name, T, cap, per) CP(f.name, cap * per)
  PLF_PT_FIELDS(PLF_FS_COPY) CP(f.pt_count, 1)
  PLF_LS_FIELDS(PLF_FS_COPY) CP(f.ls_count, 1)
#undef PLF_FS_COPY
#undef CP
  return PLF_OK;
}

// One plf_batch_run call: its pairs, buffer parities and slots, and the streams of its phases.
struct BatchRun {
  int B;
  int par;       // parity of the E -> G -> M hand-off buffers
  int lp;        // parity of the LSD hand-off buffers (0 when they exist once)
  int rp;        // slot of the result ring
  int run_slot;  // upload slot consumed: the most recently uploaded batch
  bool piped, lsd2;
  cudaStream_t sM, sE, sG, sP;
};

// ---- E phase: ORB + LBD gradient prelude (bandwidth / ALU bound); outputs per batch parity ----
static plf_status run_extract(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const int w = s->w, h = s->h, B = r.B, par = r.par;
  const size_t A = (size_t)w * h, AP = (size_t)s->pitch * h;   // dense maps / padded images
  const uint8_t* imgs = s->imgs2[r.run_slot];
  cudaStream_t sE = r.sE;
  ctx->cur = sE;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->ev_up[r.run_slot], 0));  // images uploaded
  PLF_CUDA(ctx, cudaStreamWaitEvent(sE, s->evX[par], 0));           // batch i-2 (same parity) no longer reads these buffers
  plf_mark(ctx, "start");
  PLF_CUDA(ctx, cudaEventRecord(s->tE0[par], sE));
  plf_status st = plf_orb_run(ctx, imgs, AP, s->pitch, w, h, 2 * B, par);
  if (!st) st = plf_launch_blur5_sobel(ctx, imgs, s->pitch, AP, w, h, 2 * B, s->lbd_grad[par], A);
  if (st) return st;
  plf_mark(ctx, "lbd.k_blur5_sobel");
  // this batch's ORB overflow flag: snapshot + clear on the E stream, so that a flag raised by batch i+1's extraction is
  // not reported on batch i's download
  PLF_CUDA(ctx, cudaMemcpyAsync(s->d_ovf + 2 * r.rp, plf_orb_overflow_flag(ctx), sizeof(int), cudaMemcpyDeviceToDevice, sE));
  PLF_CUDA(ctx, cudaMemsetAsync(plf_orb_overflow_flag(ctx), 0, sizeof(int), sE));
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
  const int w = s->w, h = s->h, par = r.par;
  const size_t AP = (size_t)s->pitch * h;
  cudaStream_t sP = r.sP, sG = r.sG;
  ctx->cur = sP;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sP, s->ev_up[r.run_slot], 0));
  if (r.lsd2) PLF_CUDA(ctx, cudaStreamWaitEvent(sP, s->evG[par], 0));   // batch i-2 (same parity) has finished growing / fitting on these maps
  PLF_CUDA(ctx, cudaEventRecord(s->tG0[par], sP));
  plf_status st = plf_lsd_pre(ctx, s->imgs2[r.run_slot], AP, s->pitch, w, h, r.lp, 2 * r.B);
  if (st) return st;
  PLF_CUDA(ctx, cudaEventRecord(s->ev_free2[r.run_slot], sP));
  PLF_CUDA(ctx, cudaEventRecord(s->evP[par], sP));
  ctx->cur = sG;
  PLF_CUDA(ctx, cudaStreamWaitEvent(sG, s->evP[par], 0));
  // the KeyLine outputs are overwritten: the match phase that read them last (batch i-2 with two parities, batch i-1 with one)
  // has taken its copy
  ctx->lsd_keylines_wait = r.piped ? s->evX[r.lsd2 ? par : par ^ 1] : nullptr;
  st = plf_lsd_grow(ctx, w, h, r.lp, 2 * r.B);
  ctx->lsd_keylines_wait = nullptr;
  if (st) return st;
  PLF_CUDA(ctx, cudaMemcpyAsync(s->d_ovf + 2 * r.rp + 1, plf_lsd_overflow_flag(ctx), sizeof(int), cudaMemcpyDeviceToDevice, sG));
  PLF_CUDA(ctx, cudaMemsetAsync(plf_lsd_overflow_flag(ctx), 0, sizeof(int), sG));
  PLF_CUDA(ctx, cudaEventRecord(s->evG[par], sG));
  return PLF_OK;
}

// One windowed-matching launch over B problems of one kind (points: cap = K, lines: cap = Ln).  Problem p matches the
// descriptor rows of image / slot p * step of `desc` (n1[p * step] of them) against those of the next image / slot.
static MgbArgs mgb_args(const plf_params& P, MgGrid g, bool lines, int cap, int step, const int* q_geo, const int* t_geo,
                        const double* t_dir, const uint8_t* desc, const int* cnt, int32_t* m12, size_t m12_stride, int* count,
                        int count_stride) {
  MgbArgs a = {};
  a.g = g;
  a.is_lines = lines ? 1 : 0; a.K = a.Kt = cap; a.best_lr = P.best_lr_matches ? 1 : 0;
  a.nnr = lines ? P.min_ratio_12_l : P.min_ratio_12_p;
  a.line_sim_th = (double)P.line_sim_th;
  a.q_geo = q_geo; a.t_geo = t_geo; a.t_dir = t_dir;
  a.d1 = desc; a.d2 = desc + (size_t)cap * 32; a.d1_stride = a.d2_stride = (size_t)step * cap * 32;
  a.n1 = cnt; a.n2 = cnt + 1; a.n1_stride = a.n2_stride = step;
  a.m12 = m12; a.m12_stride = m12_stride; a.count = count; a.count_stride = count_stride;
  return a;
}

// ---- M phase: LBD, stereo association, frame-to-frame tracking, pose (needs the previous batch's M phase) ----
static plf_status run_match(plf_ctx* ctx, PipeState* s, const BatchRun& r) {
  const int w = s->w, h = s->h, B = r.B, par = r.par, rp = r.rp;
  const size_t A = (size_t)w * h;
  const int K = s->max_kp, Ln = s->max_ln;
  const plf_params& P = ctx->params;
  plf_keypoint* kps; uint8_t* odesc; int* kcnt; int mk;
  plf_keyline* kls; int* lcnt; int ml;
  plf_orb_outputs(ctx, par, &kps, &odesc, &kcnt, &mk);
  plf_lsd_outputs(ctx, r.lp, &kls, &lcnt, &ml);
  cudaStream_t cs = r.sM;
  ctx->cur = cs;
  plf_status st;
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->evG[par], 0));
  PLF_CUDA(ctx, cudaStreamWaitEvent(cs, s->evE[par], 0));
  PLF_CUDA(ctx, cudaEventRecord(s->tM0[rp], cs));
  if (!s->has_prev) {  // initialize(): no previous frame to track against
    PLF_CUDA(ctx, cudaMemsetAsync(s->fs.pt_count, 0, sizeof(int), cs));
    PLF_CUDA(ctx, cudaMemsetAsync(s->fs.ls_count, 0, sizeof(int), cs));
  }
  if ((st = plf_launch_lbd(ctx, s->lbd_grad[par], A, w, h, 2 * B, kls, lcnt, Ln, s->ldesc_raw, nullptr))) return st;
  plf_mark(ctx, "lbd.k_lbd");
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
  plf_mark(ctx, "copy extraction outputs");
  PLF_CUDA(ctx, cudaMemsetAsync(s->mcount, 0, (size_t)B * 4 * sizeof(int), cs));
  const double mg_iw = PLF_GRID_COLS / (double)w, mg_ih = PLF_GRID_ROWS / (double)h;   // StereoFrame::inv_width / inv_height
  if (P.matching_strategy) {
    // stereo association through matchGrid(): window (matching_s_ws, 0) x (0, 0) over the right image's grid
    k_mg_geom_stereo<<<dim3((std::max(K, Ln) + 255) / 256, 2 * B), 256, 0, cs>>>(kps, kcnt, K, kls, lcnt, Ln, mg_iw, mg_ih, s->mg_q[0],
                                                                                 s->mg_t[0], s->mg_q[1], s->mg_t[1], s->mg_dir[0]);
    PLF_LAUNCH_CHECK(ctx);
    const MgGrid g = {PLF_GRID_COLS, PLF_GRID_ROWS, P.matching_s_ws, 0, 0, 0};
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(P, g, false, K, 2, s->mg_q[0], s->mg_t[0], nullptr, odesc, kcnt, s->m12,
                                                        4 * (size_t)K, s->mcount, 4), B, K, K, 9))) return st;
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(P, g, true, Ln, 2, s->mg_q[1], s->mg_t[1], s->mg_dir[0], s->ldesc_raw, lcnt,
                                                        s->m12 + K, 4 * (size_t)K, s->mcount + 1, 4), B, Ln, Ln, 9))) return st;
    plf_mark(ctx, "stereo.k_mgb (matchGrid)");
  } else {
    // L->R 2-NN for every left feature; R->L only for the right features that are somebody's accepted best match
    // (k_nnr_mutual reads nothing else of the reverse direction): the same matches for ~2/3 of the popcounts
    if ((st = plf_launch_knn2(ctx, s->knn_stereo, 2 * B, std::max(K, Ln)))) return st;
    if (P.best_lr_matches) {
      PLF_CUDA(ctx, cudaMemsetAsync(s->rev_flags, 0, 2 * (size_t)B * K * sizeof(int), cs));
      PLF_CUDA(ctx, cudaMemsetAsync(s->rev_count, 0, 2 * (size_t)B * sizeof(int), cs));
      if ((st = plf_launch_nnr_mark(ctx, s->nnr_stereo, 2 * B, std::max(K, Ln), s->rev_flags, s->rev_list, s->rev_count, K))) return st;
      // the reverse problems are laid out after the forward problems of ALL max_batch pairs (pipe_prepare), not of this
      // call's B pairs: a partial batch (B < max_batch) must still start at 2 * max_batch
      if ((st = plf_launch_knn2(ctx, s->knn_stereo + 2 * s->B, 2 * B, std::max(K, Ln)))) return st;
    }
    plf_mark(ctx, "stereo.k_hamming_knn2");
    if ((st = plf_launch_nnr(ctx, s->nnr_stereo, 2 * B, std::max(K, Ln)))) return st;
    plf_mark(ctx, "stereo.k_nnr_mutual");
  }
  StereoPrm sp = {P.max_dist_epip, P.min_disp, P.line_horiz_th, P.stereo_overlap_th, P.ls_min_disp_ratio,
                  ctx->cam.fx, ctx->cam.fy, ctx->cam.cx, ctx->cam.cy, ctx->cam.b};
  k_stereo_points<<<B, 1024, 0, cs>>>(kps, odesc, kcnt, K, s->m12, 4 * K, sp, s->fs, 1);
  PLF_LAUNCH_CHECK(ctx);
  k_stereo_lines<<<B, 1024, 0, cs>>>(kls, s->ldesc_raw, lcnt, Ln, s->m12 + K, 4 * K, sp, s->fs, 1);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "stereo.k_stereo_points+lines");
  if ((st = plf_launch_knn2(ctx, s->knn_f2f, 4 * B, std::max(K, Ln)))) return st;
  plf_mark(ctx, "f2f.k_hamming_knn2");
  if ((st = plf_launch_nnr(ctx, s->nnr_f2f, 2 * B, std::max(K, Ln)))) return st;
  if (P.matching_strategy) {
    // frame-to-frame: matchGrid() in a +-matching_f2f_ws window around the projected feature; the match() result above
    // stands where the window search found fewer than min_pt_matches / min_ls_matches
    PLF_CUDA(ctx, cudaMemsetAsync(s->mgcount, 0, (size_t)B * 2 * sizeof(int), cs));
    k_mg_geom_f2f<<<dim3((std::max(K, Ln) + 255) / 256, B), 256, 0, cs>>>(s->fs, K, Ln, sp, mg_iw, mg_ih, s->mg_q[2], s->mg_t[2],
                                                                          s->mg_q[3], s->mg_t[3], s->mg_dir[1]);
    PLF_LAUNCH_CHECK(ctx);
    const int ws = P.matching_f2f_ws;
    const MgGrid g = {PLF_GRID_COLS, PLF_GRID_ROWS, ws, ws, ws, ws};
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(P, g, false, K, 1, s->mg_q[2], s->mg_t[2], nullptr, s->fs.pdesc, s->fs.pt_count,
                                                        s->m12g, 2 * (size_t)K, s->mgcount, 2), B, K, K, 9))) return st;
    if ((st = plf_launch_match_grid_batch(ctx, mgb_args(P, g, true, Ln, 1, s->mg_q[3], s->mg_t[3], s->mg_dir[1], s->fs.ldesc, s->fs.ls_count,
                                                        s->m12g + K, 2 * (size_t)K, s->mgcount + 1, 2), B, Ln, Ln, 9))) return st;
    k_mg_select<<<dim3((K + 255) / 256, B), 256, 0, cs>>>(s->m12g, s->mgcount, s->fs.pt_count, K, K, 0, P.min_pt_matches, s->m12);
    PLF_LAUNCH_CHECK(ctx);
    k_mg_select<<<dim3((Ln + 255) / 256, B), 256, 0, cs>>>(s->m12g, s->mgcount, s->fs.ls_count, Ln, K, 1, P.min_ls_matches, s->m12);
    PLF_LAUNCH_CHECK(ctx);
    plf_mark(ctx, "f2f.k_mgb (matchGrid)");
  }
  k_f2f_build<<<B, 1024, 0, cs>>>(s->fs, 0, K, Ln, s->m12 + 2 * K, s->m12 + 3 * K, 4 * K, s->gnP, s->gnObs, s->gnInlP, s->gnNp,
                                  s->gn_sP, s->gn_eP, s->gn_le, s->gnInlL, s->gnNl);
  PLF_LAUNCH_CHECK(ctx);
  plf_mark(ctx, "f2f.k_nnr_mutual+k_f2f_build");
  if ((st = plf_launch_gn(ctx, s->gn_probs, B, plf_gn_opts_from_params(P)))) return st;
  plf_mark(ctx, "gn.k_gn_pose");
  k_finalize<<<(B + 127) / 128, 128, 0, cs>>>(s->gn_out, s->gnNp, s->gnNl, kcnt, lcnt, s->fs, 1, P.min_features,
                                               s->has_prev ? 0 : 1, B, s->results + (size_t)rp * s->B);
  PLF_LAUNCH_CHECK(ctx);
  if ((st = copy_slot(ctx, s, B, 0))) return st;  // carry the last frame to the next batch
  plf_mark(ctx, "k_finalize+carry");
  // results + overflow flags to pinned memory as part of this batch's stream work; evM marks them ready
  PLF_CUDA(ctx, cudaMemcpyAsync(s->h_results[rp], s->results + (size_t)rp * s->B, sizeof(plf_frame_result) * B, cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaMemcpyAsync(s->h_ovf[rp], s->d_ovf + 2 * rp, 2 * sizeof(int), cudaMemcpyDeviceToHost, cs));
  PLF_CUDA(ctx, cudaEventRecord(s->evM[rp], cs));
  return PLF_OK;
}

extern "C" {

plf_status plf_reset_sequence(plf_ctx* ctx) {
  if (!ctx) return PLF_ERR_INVALID;
  if (ctx->pipe) {
    if (ctx->pipe->n_pending)
      return plf_fail(ctx, PLF_ERR_STATE, "plf_reset_sequence: %d batch(es) still in flight; download them first", ctx->pipe->n_pending);
    ctx->pipe->has_prev = false;
  }
  return PLF_OK;
}

plf_status plf_batch_upload(plf_ctx* ctx, int B, const uint8_t* left, const uint8_t* right, int stride) {
  if (!ctx || !left || !right || B < 1 || B > ctx->limits.max_batch || stride < ctx->cam.width)
    return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_upload: bad arguments (B=%d, max_batch=%d)", B, ctx ? ctx->limits.max_batch : 0);
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  const int w = ctx->cam.width, h = ctx->cam.height;
  plf_status st = pipe_prepare(ctx, w, h);
  if (st) return st;
  PipeState* s = ctx->pipe;
  const size_t A = (size_t)s->pitch * h;
  // H2D on the copy stream into the slot the GPU is not reading, so the copy of batch i+1 overlaps the run of batch i.
  // Device layout interleaves the pair: image 2k = left k, 2k+1 = right k; rows are padded to a 16-byte pitch.
  const int slot = s->up_slot ^ 1;
  uint8_t* dst = s->imgs2[slot];
  PLF_CUDA(ctx, cudaStreamWaitEvent(s->copy, s->ev_free[slot], 0));   // the last run that read this slot has finished with it
  PLF_CUDA(ctx, cudaStreamWaitEvent(s->copy, s->ev_free2[slot], 0));  // (ORB / LBD prelude on one stream, LSD on another)
  const size_t A0 = (size_t)w * h;
  if (stride == w && s->stage) {
    // densely packed input: ONE contiguous H2D copy per side into the dense landing buffer ("rows" = images, pitch 2 A0
    // interleaves left and right), then a device-to-device 2-D copy widens the rows to the 16-byte pitch (the DMA engines
    // move 1242-byte rows from host memory at a fraction of the contiguous rate: measured 8.9 k vs 12.7 k pairs/s end to end)
    PLF_CUDA(ctx, cudaMemcpy2DAsync(s->stage, 2 * A0, left, A0, A0, B, cudaMemcpyHostToDevice, s->copy));
    PLF_CUDA(ctx, cudaMemcpy2DAsync(s->stage + A0, 2 * A0, right, A0, A0, B, cudaMemcpyHostToDevice, s->copy));
    PLF_CUDA(ctx, cudaMemcpy2DAsync(dst, (size_t)s->pitch, s->stage, (size_t)w, (size_t)w, 2 * (size_t)B * h, cudaMemcpyDeviceToDevice, s->copy));
  } else if (stride == w) {   // pitch == w: the dense layout is the device layout
    PLF_CUDA(ctx, cudaMemcpy2DAsync(dst, 2 * A, left, A, A, B, cudaMemcpyHostToDevice, s->copy));
    PLF_CUDA(ctx, cudaMemcpy2DAsync(dst + A, 2 * A, right, A, A, B, cudaMemcpyHostToDevice, s->copy));
  } else {
    // strided input: one 3-D copy per side (rows of w bytes, h rows per image, B images; the destination "height" of 2h
    // rows skips the other side's image of each pair)
    for (int side = 0; side < 2; ++side) {
      cudaMemcpy3DParms cp = {};
      cp.srcPtr = make_cudaPitchedPtr(const_cast<uint8_t*>(side ? right : left), (size_t)stride, (size_t)w, (size_t)h);
      cp.dstPtr = make_cudaPitchedPtr(dst + (size_t)side * A, (size_t)s->pitch, (size_t)w, 2 * (size_t)h);
      cp.extent = make_cudaExtent((size_t)w, (size_t)h, (size_t)B);
      cp.kind = cudaMemcpyHostToDevice;
      PLF_CUDA(ctx, cudaMemcpy3DAsync(&cp, s->copy));
    }
  }
  PLF_CUDA(ctx, cudaEventRecord(s->ev_up[slot], s->copy));
  s->up_slot = slot;
  return PLF_OK;
}

void* plf_batch_device_images(plf_ctx* ctx) {
  if (!ctx) return nullptr;
  if (pipe_prepare(ctx, ctx->cam.width, ctx->cam.height)) return nullptr;
  return ctx->pipe->imgs2[ctx->pipe->up_slot];
}

plf_status plf_batch_run(plf_ctx* ctx, int B) {
  if (!ctx || B < 1 || B > ctx->limits.max_batch) return plf_fail(ctx, PLF_ERR_INVALID, "plf_batch_run: bad B");
  PLF_CUDA(ctx, cudaSetDevice(ctx->device));
  plf_status st = pipe_prepare(ctx, ctx->cam.width, ctx->cam.height);
  if (st) return st;
  PipeState* s = ctx->pipe;
  if (s->n_pending >= 3)
    return plf_fail(ctx, PLF_ERR_STATE, "plf_batch_run: three batches already in flight; call plf_batch_download first");
  BatchRun r;
  r.B = B;
  r.par = (int)(s->seq & 1);
  r.rp = (int)(s->seq % 3);
  r.run_slot = s->up_slot;
  // With profiling on everything is serialised on the main stream so that the per-kernel marks are meaningful.
  r.piped = !ctx->profile || ctx->profile_piped;
  r.lsd2 = s->lsd2;
  r.lp = r.lsd2 ? r.par : 0;
  r.sM = ctx->stream;
  r.sE = r.piped ? ctx->aux[0] : r.sM;
  r.sG = r.piped ? ctx->aux[1] : r.sM;
  r.sP = (r.piped && r.lsd2) ? ctx->aux[2] : r.sG;   // LSD pre-grow chain: own stream when its outputs exist per parity
  st = run_extract(ctx, s, r);
  if (!st) st = run_lsd(ctx, s, r);
  if (!st) st = run_match(ctx, s, r);
  ctx->cur = r.sM;
  if (st) return st;
  s->has_prev = true;
  s->pend_slot[s->n_pending] = r.rp;
  s->pend_B[s->n_pending] = B;
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
    return plf_fail(ctx, PLF_ERR_CAPACITY, "plf_batch_download: a fixed-capacity buffer overflowed (%s%s); raise plf_limits",
                    o0 ? "ORB keypoints " : "", o1 ? "LSD segments/lines" : "");
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
  const int slot = k + 1;
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
