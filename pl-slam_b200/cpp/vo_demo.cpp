// vo_demo — the VO part of the reference's frame loop (app/plslam_dataset.cpp:111-163) on top of the C++ shim.
// Usage: vo_demo <frames.bin> [orb_nfeatures lsd_nfeatures] [--grid-selftest | --kf-match-selftest]
// frames.bin: int32 n, w, h; double fx, fy, cx, cy, b; then n x (left h*w bytes, right h*w bytes).
// Prints one line per frame: idx status n_stereo_pt n_stereo_ls n_inliers newKF Tfw(16 values, row-major).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "stvo_shim.h"

// The fast-matching branch of MapHandler::matchKF2KFPoints / matchKF2KFLines (src/mapHandler.cpp:251-271, :382-418)
// written against the shim: grid filled with grid.at(x, y).push_back(idx), GridWindow of +-ws cells, matchGrid.
// `vo_demo --grid-selftest` runs it on the features of one synthetic frame against themselves (every feature must then
// find itself) - a build-time check that the overloads instantiate and a usage example for INTEGRATION.md.
static int grid_selftest(StVO::StereoFrameHandler* h, const StVO::StereoFrame* fr, float nnr) {
  using namespace StVO;
  const double inv_w = fr->inv_width, inv_h = fr->inv_height;  // = GRID_COLS / width, GRID_ROWS / height
  std::vector<point_2d> pj_points;
  GridStructure grid(GRID_ROWS, GRID_COLS);
  for (size_t idx = 0; idx < fr->stereo_pt.size(); ++idx) {
    const PointFeature* pt = fr->stereo_pt[idx];
    pj_points.push_back(std::make_pair((int)(pt->pl[0] * inv_w), (int)(pt->pl[1] * inv_h)));
    grid.at((int)(pt->pl[0] * inv_w), (int)(pt->pl[1] * inv_h)).push_back((int)idx);
  }
  GridWindow w;
  w.width = std::make_pair(1, 1);
  w.height = std::make_pair(1, 1);
  std::vector<int> m12;
  const int np = matchGrid(h->ctx(), pj_points, fr->pdesc_l, grid, fr->pdesc_l, w, m12, nnr);
  int self = 0;
  for (size_t i = 0; i < m12.size(); ++i) self += m12[i] == (int)i;
  std::vector<line_2d> pj_lines;
  std::vector<std::pair<double, double>> directions(fr->stereo_ls.size());
  GridStructure lgrid(GRID_ROWS, GRID_COLS);
  std::list<point_2d> cells;
  for (size_t idx = 0; idx < fr->stereo_ls.size(); ++idx) {
    const LineFeature* ls = fr->stereo_ls[idx];
    std::pair<double, double>& v = directions[idx];
    v = std::make_pair((ls->epl[0] - ls->spl[0]) * inv_w, (ls->epl[1] - ls->spl[1]) * inv_h);
    normalize(v);
    getLineCoords(ls->spl[0] * inv_w, ls->spl[1] * inv_h, ls->epl[0] * inv_w, ls->epl[1] * inv_h, cells);
    for (const point_2d& p : cells) lgrid.at(p.first, p.second).push_back((int)idx);
    pj_lines.push_back(std::make_pair(std::make_pair((int)(ls->spl[0] * inv_w), (int)(ls->spl[1] * inv_h)),
                                      std::make_pair((int)(ls->epl[0] * inv_w), (int)(ls->epl[1] * inv_h))));
  }
  std::vector<int> l12;
  const int nl = matchGrid(h->ctx(), pj_lines, fr->ldesc_l, lgrid, fr->ldesc_l, directions, w, l12, nnr, 0.75);
  std::printf("grid-selftest points %zu matched %d self %d lines %zu matched %d\n", fr->stereo_pt.size(), np, self,
              fr->stereo_ls.size(), nl);
  return 0;
}

// A keyframe's stereo features as KeyFrame deep-copies them (src/keyFrame.cpp:39-53), flattened for plf_frame_view.
struct KfArrays {
  std::vector<double> pl, P, spl, epl, sP, eP, le;
  std::vector<uint8_t> pdesc, ldesc;
  StVO::Matrix4d T_kf_w;   // KeyFrame::T_kf_w (= the frame's Tfw)
  explicit KfArrays(const StVO::StereoFrame* fr) : pdesc(fr->pdesc_l.data), ldesc(fr->ldesc_l.data), T_kf_w(fr->Tfw) {
    for (const StVO::PointFeature* p : fr->stereo_pt) {
      pl.insert(pl.end(), {p->pl[0], p->pl[1]});
      P.insert(P.end(), {p->P[0], p->P[1], p->P[2]});
    }
    for (const StVO::LineFeature* l : fr->stereo_ls) {
      spl.insert(spl.end(), {l->spl[0], l->spl[1]});
      epl.insert(epl.end(), {l->epl[0], l->epl[1]});
      sP.insert(sP.end(), {l->sP[0], l->sP[1], l->sP[2]});
      eP.insert(eP.end(), {l->eP[0], l->eP[1], l->eP[2]});
      le.insert(le.end(), {l->le[0], l->le[1], l->le[2]});
    }
  }
  plf_frame_view view() {
    plf_frame_view v{};
    v.n_pt = (int)pl.size() / 2; v.n_ls = (int)spl.size() / 2;
    v.pt_pl = pl.data(); v.pt_P = P.data(); v.pdesc = pdesc.data();
    v.ls_spl = spl.data(); v.ls_epl = epl.data(); v.ls_sP = sP.data(); v.ls_eP = eP.data(); v.ls_le = le.data();
    v.ldesc = ldesc.data();
    return v;
  }
};

// The C ABI takes row-major 4x4 poses.  MapHandler's DT / Twf are Eigen::Matrix4d (column-major storage), so copy them
// element by element rather than passing .data(); the shim's Matrix4d is read the same way.
static void row_major(const StVO::Matrix4d& M, double out[16]) {
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[4 * r + c] = M(r, c);
}

// X in the keyframe's camera frame -> world: T_kf_w X, each row ((r0 x + r1 y) + r2 z) + t (src/mapHandler.cpp:297)
static void to_world(const StVO::Matrix4d& T, const double* X, double* out) {
  for (int r = 0; r < 3; ++r) out[r] = ((T(r, 0) * X[0] + T(r, 1) * X[1]) + T(r, 2) * X[2]) + T(r, 3);
}

static void print_ints(const char* name, const std::vector<int32_t>& v) {
  std::printf("kfm %s", name);
  for (int32_t x : v) std::printf(" %d", x);
  std::printf("\n");
}

// lookForCommonMatches (src/mapHandler.cpp:754-821) on the device: matchKF2KFPoints / Lines between two keyframes, then
// matchMap2KFPoints / Lines of the current keyframe against a local map.  The local map is the previous keyframe's
// features moved into the world (what the KF-to-KF bookkeeping of :290-318 creates), in feature order; a landmark the
// current keyframe has just observed is not used (:547 kf_obs_list.back() != kf_idx), and the current keyframe's features
// matched to it carry its index (:294, :334).  `vo_demo frames.bin ... --kf-match-selftest` prints the poses and every
// output array, which the Python binding must reproduce.
static int kf_match_selftest(plf_ctx* ctx, KfArrays& prev_kf, KfArrays& curr_kf) {
  using namespace StVO;
  const plf_kf_match_opts o = {1, 1.0, 1.0};   // SlamConfig::fastMatching(), maxKFEpipP(), maxKFEpipL() (config_*.yaml)
  const Matrix4d Twf = plf::inverse_se3(curr_kf.T_kf_w);   // MapHandler::Twf, :804
  const Matrix4d DT = Twf * prev_kf.T_kf_w;               // MapHandler::DT, :805
  double DT_rm[16], Twf_rm[16];
  row_major(DT, DT_rm);
  row_major(Twf, Twf_rm);
  plf_frame_view prev = prev_kf.view(), curr = curr_kf.view();
  std::vector<int32_t> m_pt(prev.n_pt), m_ls(prev.n_ls);
  int common_pt = 0, common_ls = 0;
  if (plf_match_kf2kf(ctx, &o, &prev, &curr, DT_rm, m_pt.data(), m_ls.data(), &common_pt, &common_ls) != PLF_OK) {
    std::fprintf(stderr, "plf_match_kf2kf: %s\n", plf_last_error(ctx));
    return 2;
  }
  // the local map and the current keyframe's landmark indices after the KF-to-KF bookkeeping
  std::vector<double> pt_X(3 * (size_t)prev.n_pt), ls_X(6 * (size_t)prev.n_ls);
  std::vector<uint8_t> pt_use(prev.n_pt), ls_use(prev.n_ls);
  std::vector<int32_t> kf_pt_lm(curr.n_pt, -1), kf_ls_lm(curr.n_ls, -1);
  for (int i = 0; i < prev.n_pt; ++i) {
    to_world(prev_kf.T_kf_w, &prev_kf.P[3 * (size_t)i], &pt_X[3 * (size_t)i]);
    pt_use[i] = m_pt[i] < 0;
    if (m_pt[i] >= 0) kf_pt_lm[m_pt[i]] = i;
  }
  for (int i = 0; i < prev.n_ls; ++i) {
    to_world(prev_kf.T_kf_w, &prev_kf.sP[3 * (size_t)i], &ls_X[6 * (size_t)i]);
    to_world(prev_kf.T_kf_w, &prev_kf.eP[3 * (size_t)i], &ls_X[6 * (size_t)i + 3]);
    ls_use[i] = m_ls[i] < 0;
    if (m_ls[i] >= 0) kf_ls_lm[m_ls[i]] = i;
  }
  const plf_local_map map = {prev.n_pt, pt_X.data(), prev_kf.pdesc.data(), pt_use.data(),
                             prev.n_ls, ls_X.data(), prev_kf.ldesc.data(), ls_use.data()};
  std::vector<int32_t> lm_pt(prev.n_pt), lm_ls(prev.n_ls);
  int map_pt = 0, map_ls = 0;
  if (plf_match_map2kf(ctx, &o, &map, Twf_rm, &curr, kf_pt_lm.data(), kf_ls_lm.data(), lm_pt.data(), lm_ls.data(), &map_pt,
                       &map_ls) != PLF_OK) {
    std::fprintf(stderr, "plf_match_map2kf: %s\n", plf_last_error(ctx));
    return 2;
  }
  std::printf("kfm DT");
  for (double v : DT_rm) std::printf(" %.17g", v);
  std::printf("\nkfm Twf");
  for (double v : Twf_rm) std::printf(" %.17g", v);
  std::printf("\nkfm kf2kf %d %d\n", common_pt, common_ls);
  print_ints("m_pt", m_pt);
  print_ints("m_ls", m_ls);
  std::printf("kfm map2kf %d %d\n", map_pt, map_ls);
  print_ints("lm_pt", lm_pt);
  print_ints("lm_ls", lm_ls);
  return 0;
}

int main(int argc, char** argv) {
  bool grid_test = false, kf_test = false;
  if (argc >= 2 && std::string(argv[argc - 1]) == "--grid-selftest") { grid_test = true; --argc; }
  if (argc >= 2 && std::string(argv[argc - 1]) == "--kf-match-selftest") { kf_test = true; --argc; }
  if (argc < 2) {
    std::fprintf(stderr, "usage: %s frames.bin [orb_nfeatures lsd_nfeatures]\n", argv[0]);
    return 1;
  }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) { std::perror("open"); return 1; }
  int32_t hdr[3];
  double cam[5];
  if (std::fread(hdr, 4, 3, f) != 3 || std::fread(cam, 8, 5, f) != 5) { std::fprintf(stderr, "bad header\n"); return 1; }
  const int n = hdr[0], w = hdr[1], h = hdr[2];
  std::vector<uint8_t> buf((size_t)2 * w * h);
  try {
    StVO::PinholeStereoCamera cam_pin(w, h, cam[0], cam[1], cam[2], cam[3], cam[4]);
    plf_params prm;
    plf_default_params(&prm);
    if (argc >= 4) { prm.orb_nfeatures = std::atoi(argv[2]); prm.lsd_nfeatures = std::atoi(argv[3]); }
    StVO::StereoFrameHandler* StVO_ = new StVO::StereoFrameHandler(&cam_pin, &prm);   // app:109
    KfArrays* first_kf = nullptr;   // --kf-match-selftest: frame 0 against the last frame
    int rc = 0;
    for (int frame_counter = 0; frame_counter < n; ++frame_counter) {                   // app:111
      if (std::fread(buf.data(), 1, buf.size(), f) != buf.size()) { std::fprintf(stderr, "short read\n"); return 1; }
      plf::Image img_l{buf.data(), w, h, w}, img_r{buf.data() + (size_t)w * h, w, h, w};
      bool new_kf = false;
      StVO::StereoFrame* cur;
      if (frame_counter == 0) {
        StVO_->initialize(img_l, img_r, 0);                                             // app:115
        cur = StVO_->prev_frame;
        if (grid_test) return grid_selftest(StVO_, cur, prm.min_ratio_12_p);
      } else {
        StVO_->insertStereoPair(img_l, img_r, frame_counter);                           // app:127
        StVO_->optimizePose();                                                          // app:128
        cur = StVO_->curr_frame;
        if (StVO_->needNewKF()) {                                                       // app:135
          new_kf = true;
          StVO_->currFrameIsKF();                                                       // app:145
        }
      }
      const plf_frame_result& r = StVO_->last_result();
      std::printf("%d %d %zu %zu %d %d", frame_counter, r.status, cur->stereo_pt.size(), cur->stereo_ls.size(),
                  StVO_->n_inliers, new_kf ? 1 : 0);
      for (int i = 0; i < 16; ++i) std::printf(" %.17g", cur->Tfw.v[i]);
      std::printf("\n");
      if (kf_test && frame_counter == 0) first_kf = new KfArrays(cur);
      if (kf_test && frame_counter == n - 1 && first_kf) {
        KfArrays last_kf(cur);
        rc = kf_match_selftest(StVO_->ctx(), *first_kf, last_kf);
      }
      if (frame_counter > 0) StVO_->updateFrame();                                      // app:159
    }
    delete first_kf;
    delete StVO_;
    if (rc) return rc;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "error: %s\n", e.what());
    return 2;
  }
  std::fclose(f);
  return 0;
}
