// vo_demo — the VO part of the reference's frame loop (app/plslam_dataset.cpp:111-163) on top of the C++ shim.
// Usage: vo_demo <frames.bin> [orb_nfeatures lsd_nfeatures] [--grid-selftest | --kf-match-selftest |
//                                                            --bow-selftest <voc_p.yml> <voc_l.yml> |
//                                                            --lc-detect-selftest <voc_p.yml> <voc_l.yml>]
//        vo_demo --gba-selftest <problem.bin>
//        vo_demo --pgo-selftest <map.bin>
// frames.bin: int32 n, w, h; double fx, fy, cx, cy, b; then n x (left h*w bytes, right h*w bytes).
// Prints one line per frame: idx status n_stereo_pt n_stereo_ls n_inliers newKF Tfw(16 values, row-major).
#include <algorithm>
#include <array>
#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <unordered_map>
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

// ---- INTEGRATION.md §4 f5: DBoW2 place recognition (the text between the two markers is the snippet shown there) ----
// What MapHandler's BoW code reads: KeyFrame::kf_idx and KeyFrame::stereo_frame (include/keyFrame.h), the map_keyframes
// list (NULL once removeRedundantKFs deleted a keyframe) and conf_matrix (include/mapHandler.h:147).  The global BA
// (f6 below) reads x_kf_w and writes T_kf_w.
struct KeyFrame {
  int kf_idx;
  StVO::StereoFrame* stereo_frame;
  StVO::Vector6d x_kf_w;
  StVO::Matrix4d T_kf_w;
};
struct BowMap {
  plf_ctx* ctx;
  bool has_points, has_lines;   // SlamConfig::hasPoints() / hasLines()
  std::vector<KeyFrame*> map_keyframes;
  std::vector<std::vector<float>> conf_matrix;
};
// BEGIN f5
static void plf_check(plf_ctx* ctx, plf_status st, const char* what) {
  if (st != PLF_OK) throw std::runtime_error(std::string(what) + ": " + plf_last_error(ctx));
}

// MapHandler construction, where dbow_voc_p / dbow_voc_l are loaded (kind 0 = points, 1 = lines)
static void bow_load_vocabulary(plf_ctx* ctx, int kind, const char* path) {
  plf_vocab v;
  plf_check(nullptr, plf_vocab_read_yml(path, &v), "plf_vocab_read_yml");
  const plf_status st = plf_bow_set_vocabulary(ctx, kind, &v);
  plf_vocab_free(&v);
  plf_check(ctx, st, "plf_bow_set_vocabulary");
}

// initialize (:82-98, the transform) and insertKFBowVectorP / L / PL (:3007-3128, the transform and the score rows):
// one call.  score_p / score_l come back with kf->kf_idx + 1 entries, NaN where map_keyframes[i] is absent or erased.
static void bow_insert(BowMap& m, KeyFrame* kf, std::vector<double>& score_p, std::vector<double>& score_l) {
  const StVO::StereoFrame* sf = kf->stereo_frame;
  plf_frame_view v = {};                                   // the rows of pdesc_l / ldesc_l
  v.n_pt = sf->pdesc_l.rows; v.pdesc = const_cast<uint8_t*>(sf->pdesc_l.ptr<uint8_t>());
  v.n_ls = sf->ldesc_l.rows; v.ldesc = const_cast<uint8_t*>(sf->ldesc_l.ptr<uint8_t>());
  score_p.assign(kf->kf_idx + 1, 0.0);
  score_l.assign(kf->kf_idx + 1, 0.0);
  plf_check(m.ctx, plf_bow_insert(m.ctx, kf->kf_idx, &v, m.has_points ? score_p.data() : nullptr,
                                  m.has_lines ? score_l.data() : nullptr), "plf_bow_insert");
}

// insertKFBowVectorP (:3018-3029); insertKFBowVectorL is the same on score_l.  insertKFBowVectorPL keeps its loop
// (:3070-3127, it reads stvo-pl's vector_stdv) with score_p[i] / score_l[i] in place of the two score() calls.
static void bow_fill_conf_matrix_p(BowMap& m, const KeyFrame* kf, const std::vector<double>& score_p) {
  const int idx = kf->kf_idx;
  for (int i = 0; i < idx; i++) {
    if (m.map_keyframes[i] != NULL) {
      m.conf_matrix[idx][i] = score_p[i];
      m.conf_matrix[i][idx] = score_p[i];
    }
  }
  m.conf_matrix[idx][idx] = score_p[idx];
}

// removeRedundantKFs (:2931-2932), next to `delete map_keyframes[kf_idx]; map_keyframes[kf_idx] = nullptr;`
static void bow_erase(BowMap& m, int kf_idx) { plf_check(m.ctx, plf_bow_erase(m.ctx, kf_idx), "plf_bow_erase"); }
// END f5

static void print_doubles(const char* name, int k, const std::vector<double>& v) {
  std::printf("bow %s %d", name, k);
  for (double x : v) std::printf(" %.17g", x);
  std::printf("\n");
}

// `vo_demo frames.bin ... --bow-selftest voc_p.yml voc_l.yml`: every frame becomes keyframe kf_idx = frame index through
// the f5 functions above; keyframe 1 is erased after keyframe 2 is inserted.  Prints each keyframe's two score rows, its
// conf_matrix row, and its two stored BowVectors, which the Python binding must reproduce.
static void bow_selftest_frame(BowMap& m, StVO::StereoFrame* cur, int frame_counter) {
  KeyFrame* kf = new KeyFrame{frame_counter, cur};
  m.map_keyframes.push_back(kf);
  for (auto& row : m.conf_matrix) row.resize(m.map_keyframes.size(), 0.f);
  m.conf_matrix.emplace_back(m.map_keyframes.size(), 0.f);
  std::vector<double> sp, sl;
  bow_insert(m, kf, sp, sl);
  bow_fill_conf_matrix_p(m, kf, sp);
  print_doubles("score_p", kf->kf_idx, sp);
  print_doubles("score_l", kf->kf_idx, sl);
  std::vector<double> conf(m.conf_matrix[kf->kf_idx].begin(), m.conf_matrix[kf->kf_idx].end());
  print_doubles("conf", kf->kf_idx, conf);
  for (int kind = 0; kind < 2; ++kind) {
    int n = 0;
    plf_check(m.ctx, plf_bow_get(m.ctx, kf->kf_idx, kind, 0, nullptr, nullptr, &n), "plf_bow_get");
    std::vector<uint32_t> w(n);
    std::vector<double> x(n);
    plf_check(m.ctx, plf_bow_get(m.ctx, kf->kf_idx, kind, n, w.data(), x.data(), &n), "plf_bow_get");
    std::printf("bow words%d %d", kind, kf->kf_idx);
    for (uint32_t v : w) std::printf(" %u", v);
    std::printf("\n");
    print_doubles(kind ? "vals1" : "vals0", kf->kf_idx, x);
  }
  kf->stereo_frame = nullptr;   // the frame is the handler's; only the index stays
  if (frame_counter == 2) {
    bow_erase(m, 1);
    delete m.map_keyframes[1];
    m.map_keyframes[1] = nullptr;
  }
}

// ---- INTEGRATION.md §4 f8: loop-candidate detection (the text between the two markers is the snippet shown there) ----
// What it reads beyond f5's BowMap: full_graph (include/mapHandler.h:145) and the SlamConfig values lookForLoopCandidates
// reads; the keyframe's stereo_pt[i]->pl and stereo_ls[i]->spl / epl (the rows of pdesc_l / ldesc_l).
struct LcMap {
  BowMap bow;
  std::vector<std::vector<unsigned int>> full_graph;
  int lc_kf_dist, lc_kf_max_dist, lc_nkf_closest, min_lm_cov_graph, min_kf_local_map;   // SlamConfig::lcKFDist() ...
};
// BEGIN f8
// insertKFBowVectorP / L / PL (:3007-3128) and lookForLoopCandidates (:3130-3190) in one call.  Call it where the
// reference calls lookForLoopCandidates, once full_graph holds the keyframe's covisibility: loopClosureThread() right
// after the insert (:1144-1154), loopClosure() at :2950 with the insert of addKeyFrame (:196-202) removed (nothing in
// between reads conf_matrix or descDBoW_*, while the local BA may still lower full_graph).  Returns kf_prev_idx or -1.
static int lc_detect(LcMap& m, KeyFrame* kf) {
  const StVO::StereoFrame* sf = kf->stereo_frame;
  const int idx = kf->kf_idx;
  std::vector<double> pt_pl, ls_spl, ls_epl;                 // row i of pdesc_l <-> stereo_pt[i], of ldesc_l <-> stereo_ls[i]
  for (const StVO::PointFeature* pt : sf->stereo_pt) { pt_pl.push_back(pt->pl(0)); pt_pl.push_back(pt->pl(1)); }
  for (const StVO::LineFeature* ls : sf->stereo_ls) {
    ls_spl.push_back(ls->spl(0)); ls_spl.push_back(ls->spl(1));
    ls_epl.push_back(ls->epl(0)); ls_epl.push_back(ls->epl(1));
  }
  plf_frame_view v = {};
  v.n_pt = sf->pdesc_l.rows; v.pdesc = const_cast<uint8_t*>(sf->pdesc_l.ptr<uint8_t>()); v.pt_pl = pt_pl.data();
  v.n_ls = sf->ldesc_l.rows; v.ldesc = const_cast<uint8_t*>(sf->ldesc_l.ptr<uint8_t>());
  v.ls_spl = ls_spl.data(); v.ls_epl = ls_epl.data();
  std::vector<uint32_t> covis(m.full_graph[idx].begin(), m.full_graph[idx].begin() + idx);   // full_graph[idx][i], i < idx
  std::vector<float> conf(idx + 1);
  plf_lc_detect_opts o = {m.lc_kf_dist, m.lc_kf_max_dist, m.lc_nkf_closest, m.min_lm_cov_graph, m.min_kf_local_map};
  plf_lc_detect_problem pr = {};
  pr.kf_idx = idx; pr.kf = &v; pr.covis = covis.data(); pr.conf = conf.data();
  plf_check(m.bow.ctx, plf_bow_detect(m.bow.ctx, &o, &pr), "plf_bow_detect");
  // conf_matrix as insertKFBowVector* leaves it (only lookForLoopCandidates reads it; keep it for other readers)
  for (int i = 0; i < idx; i++) {
    if (m.bow.map_keyframes[i] != NULL) {
      m.bow.conf_matrix[idx][i] = conf[i];
      m.bow.conf_matrix[i][idx] = conf[i];
    }
  }
  m.bow.conf_matrix[idx][idx] = conf[idx];
  return pr.result.candidate;
}
// END f8

// `vo_demo frames.bin ... --lc-detect-selftest voc_p.yml voc_l.yml`: every frame becomes keyframe kf_idx = frame index
// through lc_detect, with full_graph[i][j] = (i j + i + j) mod 40 and options 1, 2, 1, 20, 0 (lcKFDist, lcKFMaxDist,
// lcNKFClosest, minLMCovGraph, minKFLocalMap) so that short streams reach every step; keyframe 1 is erased after
// keyframe 2.  Prints each keyframe's conf_matrix row and result, which the Python binding must reproduce.
static void lc_selftest_frame(LcMap& m, StVO::StereoFrame* cur, int frame_counter) {
  KeyFrame* kf = new KeyFrame{frame_counter, cur};
  m.bow.map_keyframes.push_back(kf);
  const size_t n = m.bow.map_keyframes.size();
  for (auto& row : m.bow.conf_matrix) row.resize(n, 0.f);        // expandGraphs (:823-835)
  m.bow.conf_matrix.emplace_back(n, 0.f);
  for (auto& row : m.full_graph) row.resize(n, 0u);
  m.full_graph.emplace_back(n, 0u);
  for (size_t i = 0; i < n; ++i)
    m.full_graph[n - 1][i] = m.full_graph[i][n - 1] = (unsigned)((i * (n - 1) + i + (n - 1)) % 40);
  const int cand = lc_detect(m, kf);
  std::printf("lc conf %d", kf->kf_idx);
  for (float x : m.bow.conf_matrix[kf->kf_idx]) std::printf(" %.9g", x);
  std::printf("\nlc cand %d %d\n", kf->kf_idx, cand);
  kf->stereo_frame = nullptr;
  if (frame_counter == 2) {
    bow_erase(m.bow, 1);
    delete m.bow.map_keyframes[1];
    m.bow.map_keyframes[1] = nullptr;
  }
}

// ---- INTEGRATION.md §4 f6: global bundle adjustment (the text between the two markers is the snippet shown there) ----
// What MapHandler's GBA reads and writes: the map_keyframes / map_points / map_lines lists (NULL where deleted),
// MapPoint::idx / point3D / obs_list / kf_obs_list and MapLine::idx / line3D / obs_list / kf_obs_list
// (include/mapFeatures.h), and the SlamConfig values levMarquardtOptimizationGBA reuses.  The pose graph (f7 below) also
// moves med_obs_dir and dir_list.
struct MapPoint {
  int idx;
  StVO::Vector3d point3D;
  std::vector<StVO::Vector2d> obs_list;
  std::vector<int> kf_obs_list;
  StVO::Vector3d med_obs_dir;
  std::vector<StVO::Vector3d> dir_list;
};
struct MapLine {
  int idx;
  StVO::Vector6d line3D;
  std::vector<StVO::Vector3d> obs_list;
  std::vector<int> kf_obs_list;
  StVO::Vector3d med_obs_dir;
  std::vector<StVO::Vector3d> dir_list;
};
struct GbaMap {
  plf_ctx* ctx;
  double lambda_lba_lm, lambda_lba_k, homog_th;   // SlamConfig::lambdaLbaLM / lambdaLbaK / homogTh
  int max_iters_lba;                              // SlamConfig::maxItersLba
  std::vector<KeyFrame*> map_keyframes;
  std::vector<MapPoint*> map_points;
  std::vector<MapLine*> map_lines;
};
// BEGIN f6
// MapHandler::globalBundleAdjustment (:1995-2099): the lists, plf_global_ba, the write-back (:2673-2697)
static plf_lba_result global_bundle_adjustment(GbaMap& m) {
  std::vector<double> X;                                    // [x_kf_w of every live KF but 0 | point3D | line3D]
  std::unordered_map<int, int> kf_loc;                      // kf_idx -> local index (:2001-2014)
  std::vector<int> kf_list, pt_list, ls_list, pt_lm, pt_kf, ls_lm, ls_kf;
  std::vector<double> pt_xy, ls_le, fixed_T;                // fixed_T: row-major T_kf_w of keyframe 0
  for (KeyFrame* kf : m.map_keyframes)
    if (kf && kf->kf_idx != 0) {
      kf_loc[kf->kf_idx] = (int)kf_list.size();
      kf_list.push_back(kf->kf_idx);
      for (int i = 0; i < 6; ++i) X.push_back(kf->x_kf_w(i));
    }
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) fixed_T.push_back(m.map_keyframes[0]->T_kf_w(r, c));
  auto kf_index = [&](int kf_idx) { auto it = kf_loc.find(kf_idx); return it == kf_loc.end() ? -1 : it->second; };
  // :2017-2052 / :2054-2090.  The reference skips observations made by erased keyframes (:2131, :2239): they are left
  // out, and so is a landmark left without observations (plf_global_ba refuses one: it would be a zero pivot).
  for (MapPoint* pt : m.map_points) {
    if (!pt) continue;
    int n = 0;
    for (size_t i = 0; i < pt->obs_list.size(); ++i) {
      const int k = pt->kf_obs_list[i];
      if (!m.map_keyframes[k]) continue;
      pt_lm.push_back((int)pt_list.size());
      pt_kf.push_back(kf_index(k));                         // -1: keyframe 0 = fixed_T[0]
      for (int c = 0; c < 2; ++c) pt_xy.push_back(pt->obs_list[i](c));
      ++n;
    }
    if (!n) continue;
    pt_list.push_back(pt->idx);
    for (int c = 0; c < 3; ++c) X.push_back(pt->point3D(c));
  }
  for (MapLine* ls : m.map_lines) {
    if (!ls) continue;
    int n = 0;
    for (size_t i = 0; i < ls->obs_list.size(); ++i) {
      const int k = ls->kf_obs_list[i];
      if (!m.map_keyframes[k]) continue;
      ls_lm.push_back((int)ls_list.size());
      ls_kf.push_back(kf_index(k));
      for (int c = 0; c < 3; ++c) ls_le.push_back(ls->obs_list[i](c));
      ++n;
    }
    if (!n) continue;
    ls_list.push_back(ls->idx);
    for (int c = 0; c < 6; ++c) X.push_back(ls->line3D(c));
  }
  plf_lba_problem p = {};
  p.n_kf = (int)kf_list.size(); p.n_pt = (int)pt_list.size(); p.n_ls = (int)ls_list.size(); p.n_fixed = 1;
  p.kf_pose = X.data(); p.pt = X.data() + 6 * p.n_kf; p.ls = p.pt + 3 * p.n_pt; p.fixed_T = fixed_T.data();
  p.n_pt_obs = (int)pt_lm.size(); p.pt_obs_lm = pt_lm.data(); p.pt_obs_kf = pt_kf.data(); p.pt_obs_xy = pt_xy.data();
  p.n_ls_obs = (int)ls_lm.size(); p.ls_obs_lm = ls_lm.data(); p.ls_obs_kf = ls_kf.data(); p.ls_obs_le = ls_le.data();
  plf_lba_opts o = {m.lambda_lba_lm, m.lambda_lba_k, m.max_iters_lba, m.homog_th,
                    DBL_EPSILON, DBL_EPSILON, /*ref_quirks=*/1};  // :2116, :2391, :2637, :2667
  plf_lba_result res;
  plf_check(m.ctx, plf_global_ba(m.ctx, &o, &p, &res), "plf_global_ba");
  for (size_t i = 0; i < kf_list.size(); ++i) {             // :2673-2697
    StVO::Vector6d x;
    for (int c = 0; c < 6; ++c) x(c) = p.kf_pose[6 * i + c];
    m.map_keyframes[kf_list[i]]->T_kf_w = StVO::expmap_se3(x);
  }
  for (size_t i = 0; i < pt_list.size(); ++i)
    for (int c = 0; c < 3; ++c) m.map_points[pt_list[i]]->point3D(c) = p.pt[3 * i + c];
  for (size_t i = 0; i < ls_list.size(); ++i)
    for (int c = 0; c < 6; ++c) m.map_lines[ls_list[i]]->line3D(c) = p.ls[6 * i + c];
  return res;
}
// END f6

// `vo_demo --gba-selftest problem.bin`: reads a map (little-endian: int32 width, height; f64 fx, fy, cx, cy, b, lambda,
// lambda_k, homog_th; int32 max_iters; then keyframe, point and line slots, each an int32 `present` flag followed by
// the object: keyframe x_kf_w[6], T_kf_w[16] row-major; point point3D[3], int32 n_obs, n_obs x (int32 kf_idx, f64[2]);
// line line3D[6], int32 n_obs, n_obs x (int32 kf_idx, f64[3])), runs the f6 function above on it and prints the result,
// every live keyframe's T_kf_w and every live landmark, which the Python binding must reproduce.
static int gba_selftest(const char* path) {
  FILE* f = std::fopen(path, "rb");
  if (!f) { std::perror("open"); return 1; }
  bool ok = true;
  auto i32 = [&]() { int32_t v = 0; ok = ok && std::fread(&v, 4, 1, f) == 1; return (int)v; };
  auto f64 = [&]() { double v = 0; ok = ok && std::fread(&v, 8, 1, f) == 1; return v; };
  plf_camera cam;
  cam.width = i32(); cam.height = i32();
  cam.fx = f64(); cam.fy = f64(); cam.cx = f64(); cam.cy = f64(); cam.b = f64();
  GbaMap m = {};
  m.lambda_lba_lm = f64(); m.lambda_lba_k = f64(); m.homog_th = f64(); m.max_iters_lba = i32();
  for (int i = 0, n = i32(); ok && i < n; ++i) {
    KeyFrame* kf = nullptr;
    if (i32()) {
      kf = new KeyFrame{i, nullptr, {}, {}};
      for (int c = 0; c < 6; ++c) kf->x_kf_w(c) = f64();
      for (int c = 0; c < 16; ++c) kf->T_kf_w.v[c] = f64();
    }
    m.map_keyframes.push_back(kf);
  }
  for (int i = 0, n = i32(); ok && i < n; ++i) {
    MapPoint* pt = nullptr;
    if (i32()) {
      pt = new MapPoint{i, {}, {}, {}};
      for (int c = 0; c < 3; ++c) pt->point3D(c) = f64();
      for (int k = 0, no = i32(); ok && k < no; ++k) {
        pt->kf_obs_list.push_back(i32());
        StVO::Vector2d z;
        for (int c = 0; c < 2; ++c) z(c) = f64();
        pt->obs_list.push_back(z);
      }
    }
    m.map_points.push_back(pt);
  }
  for (int i = 0, n = i32(); ok && i < n; ++i) {
    MapLine* ls = nullptr;
    if (i32()) {
      ls = new MapLine{i, {}, {}, {}};
      for (int c = 0; c < 6; ++c) ls->line3D(c) = f64();
      for (int k = 0, no = i32(); ok && k < no; ++k) {
        ls->kf_obs_list.push_back(i32());
        StVO::Vector3d z;
        for (int c = 0; c < 3; ++c) z(c) = f64();
        ls->obs_list.push_back(z);
      }
    }
    m.map_lines.push_back(ls);
  }
  std::fclose(f);
  int rc = 0;
  if (!ok) { std::fprintf(stderr, "short read\n"); rc = 1; }
  plf_params prm;
  plf_default_params(&prm);
  plf_limits lim;
  plf_default_limits(&lim);
  lim.max_batch = 1;
  if (!rc && plf_create(&prm, &cam, &lim, 0, &m.ctx) != PLF_OK) {
    std::fprintf(stderr, "plf_create: %s\n", plf_last_error(nullptr));
    rc = 2;
  }
  if (!rc) {
    try {
      const plf_lba_result res = global_bundle_adjustment(m);
      std::printf("gba result %d %.17g %.17g\n", res.iters, res.err, res.lambda);
      for (KeyFrame* kf : m.map_keyframes) {
        if (!kf || kf->kf_idx == 0) continue;
        std::printf("gba kf %d", kf->kf_idx);
        for (int c = 0; c < 16; ++c) std::printf(" %.17g", kf->T_kf_w.v[c]);
        std::printf("\n");
      }
      for (MapPoint* pt : m.map_points) {
        if (!pt) continue;
        std::printf("gba pt %d", pt->idx);
        for (int c = 0; c < 3; ++c) std::printf(" %.17g", pt->point3D(c));
        std::printf("\n");
      }
      for (MapLine* ls : m.map_lines) {
        if (!ls) continue;
        std::printf("gba ls %d", ls->idx);
        for (int c = 0; c < 6; ++c) std::printf(" %.17g", ls->line3D(c));
        std::printf("\n");
      }
    } catch (const std::exception& e) {
      std::fprintf(stderr, "error: %s\n", e.what());
      rc = 2;
    }
    plf_destroy(m.ctx);
  }
  for (KeyFrame* kf : m.map_keyframes) delete kf;
  for (MapPoint* pt : m.map_points) delete pt;
  for (MapLine* ls : m.map_lines) delete ls;
  return rc;
}

// ---- INTEGRATION.md §4 f7: loop-closure pose graph (the text between the two markers is the snippet shown there) ----
// What loopClosureOptimizationCovGraphG2O reads and writes (include/mapHandler.h): map_keyframes (T_kf_w, x_kf_w),
// full_graph, lc_idx_list (Vector3i: the two keyframes and the "not yet optimised" flag), lc_pose_list, map_points /
// map_lines with the landmarks anchored at each keyframe (map_points_kf_idx / map_lines_kf_idx), and
// SlamConfig::minLMEssGraph / minLMCovGraph / maxItersPGO.
struct PgoMap {
  plf_ctx* ctx;
  int min_lm_ess_graph, min_lm_cov_graph, max_iters_pgo;
  std::vector<KeyFrame*> map_keyframes;
  std::vector<std::vector<unsigned int>> full_graph;
  std::vector<std::array<int, 3>> lc_idx_list;
  std::vector<StVO::Vector6d> lc_pose_list;
  std::vector<MapPoint*> map_points;
  std::vector<MapLine*> map_lines;
  std::vector<std::vector<int>> map_points_kf_idx, map_lines_kf_idx;
};
// BEGIN f7
// Tkfw_corr.block(0,0,3,3) * v + Tkfw_corr.block(0,3,3,1): directions are moved like points, as the reference writes it
static StVO::Vector3d pgo_xf(const StVO::Matrix4d& C, const StVO::Vector3d& v) {
  StVO::Vector3d o;
  for (int r = 0; r < 3; ++r) o(r) = C(r, 0) * v(0) + C(r, 1) * v(1) + C(r, 2) * v(2) + C(r, 3);
  return o;
}
// MapHandler::loopClosureOptimizationCovGraphG2O (:4185-4410): the graph (:4198-4290), plf_pose_graph in place of g2o's
// computeInitialGuess + optimize (:4290-4294), the write-back (:4298-4398).  loopClosureFuseLandmarks() follows.
static plf_pgo_result loop_closure_optimization_cov_graph(PgoMap& m) {
  int kf_curr_idx = -1;                                     // :4198-4208; kf_prev_idx is forced to 0
  for (const auto& lc : m.lc_idx_list) kf_curr_idx = std::max(kf_curr_idx, lc[1]);
  const int kf_prev_idx = 0;
  std::vector<int> kf_list, pos(kf_curr_idx + 1, -1);      // vertex of each keyframe (the problem's vertices in id order)
  std::vector<double> T, Z;                                 // row-major copies: never .data() of an Eigen::Matrix4d
  std::vector<uint8_t> fixed;
  std::vector<int> from, to;
  auto push_rm = [](std::vector<double>& dst, const StVO::Matrix4d& M) {
    double t[16];
    row_major(M, t);
    dst.insert(dst.end(), t, t + 16);
  };
  for (int i = kf_prev_idx; i <= kf_curr_idx; i++)          // :4211-4247
    if (m.map_keyframes[i] != NULL) {
      pos[i] = (int)kf_list.size();
      kf_list.push_back(i);
      push_rm(T, m.map_keyframes[i]->T_kf_w);
      fixed.push_back(i == 0);
    }
  for (int i = kf_prev_idx; i <= kf_curr_idx; i++)          // :4250-4273, in (i asc, j asc) order
    for (int j = i + 1; j <= kf_curr_idx; j++)
      if (m.map_keyframes[i] != NULL && m.map_keyframes[j] != NULL &&
          (m.full_graph[i][j] >= (unsigned)m.min_lm_ess_graph || m.full_graph[i][j] >= (unsigned)m.min_lm_cov_graph ||
           std::abs(i - j) == 1)) {
        from.push_back(pos[i]); to.push_back(pos[j]);
        push_rm(Z, StVO::inverse_se3(m.map_keyframes[i]->T_kf_w) * m.map_keyframes[j]->T_kf_w);
      }
  for (size_t k = 0; k < m.lc_idx_list.size(); k++) {      // :4276-4288
    from.push_back(pos[m.lc_idx_list[k][0]]); to.push_back(pos[m.lc_idx_list[k][1]]);
    push_rm(Z, StVO::expmap_se3(m.lc_pose_list[k]));
  }
  plf_pgo_problem p = {};
  p.n_v = (int)kf_list.size(); p.n_e = (int)from.size();
  p.T = T.data(); p.fixed = fixed.data(); p.from = from.data(); p.to = to.data(); p.Z = Z.data();
  plf_pgo_opts o = {m.max_iters_pgo, 1e-10};               // setUserLambdaInit(1e-10), optimize(maxItersPGO)
  plf_pgo_result res = {};
  plf_check(m.ctx, plf_pose_graph(m.ctx, &o, &p, &res), "plf_pose_graph");
  auto move_landmarks = [&](int kf, const StVO::Matrix4d& C) {
    for (int i : m.map_points_kf_idx.at(kf)) {
      MapPoint* pt = m.map_points[i];
      if (pt == NULL) continue;
      pt->point3D = pgo_xf(C, pt->point3D);
      pt->med_obs_dir = pgo_xf(C, pt->med_obs_dir);
      for (auto& d : pt->dir_list) d = pgo_xf(C, d);
    }
    for (int i : m.map_lines_kf_idx.at(kf)) {
      MapLine* ls = m.map_lines[i];
      if (ls == NULL) continue;
      StVO::Vector3d sP(ls->line3D(0), ls->line3D(1), ls->line3D(2)), eP(ls->line3D(3), ls->line3D(4), ls->line3D(5));
      sP = pgo_xf(C, sP);
      eP = pgo_xf(C, eP);
      for (int c = 0; c < 3; ++c) { ls->line3D(c) = sP(c); ls->line3D(3 + c) = eP(c); }
      ls->med_obs_dir = pgo_xf(C, ls->med_obs_dir);
      for (auto& d : ls->dir_list) d = pgo_xf(C, d);
    }
  };
  StVO::Matrix4d Tkfw_corr;                                 // :4298-4348
  for (size_t n = 0; n < kf_list.size(); n++) {
    KeyFrame* kf = m.map_keyframes[kf_list[n]];
    StVO::Matrix4d Tkfw;
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) Tkfw(r, c) = p.T[16 * n + 4 * r + c];
    const StVO::Matrix4d Tkfw_prev = kf->T_kf_w;
    kf->T_kf_w = Tkfw;
    kf->x_kf_w = StVO::logmap_se3(Tkfw);
    Tkfw_corr = Tkfw * StVO::inverse_se3(Tkfw_prev);
    move_landmarks(kf_list[n], Tkfw_corr);
  }
  for (size_t i = kf_curr_idx + 1; i < m.map_keyframes.size(); i++) {   // :4351-4393, no NULL check (:4357)
    m.map_keyframes[i]->T_kf_w = Tkfw_corr * m.map_keyframes[i]->T_kf_w;
    m.map_keyframes[i]->x_kf_w = StVO::logmap_se3(m.map_keyframes[i]->T_kf_w);
    move_landmarks((int)i, Tkfw_corr);
  }
  for (auto& lc : m.lc_idx_list) lc[2] = 0;                 // :4396-4397
  return res;
}
// END f7

// `vo_demo --pgo-selftest map.bin`: reads a map (little-endian: int32 minLMEssGraph, minLMCovGraph, maxItersPGO, n_kf;
// n_kf keyframe slots, each an int32 `present` flag followed by T_kf_w[16] row-major; full_graph as n_kf x n_kf int32;
// int32 n_lc, n_lc x (int32 kf0, kf1, f64 lc_pose[6]); int32 n_pt and the point slots: int32 present, point3D[3],
// med_obs_dir[3], int32 n_dir, n_dir x f64[3]; the same for lines with line3D[6]; then per keyframe the anchored points
// (int32 n, n x int32) and per keyframe the anchored lines), runs the f7 function above on it and prints the result,
// every keyframe's T_kf_w and every landmark, which oracle/pgo.py's lists + the Python binding + its write-back must give.
static int pgo_selftest(const char* path) {
  FILE* f = std::fopen(path, "rb");
  if (!f) { std::perror("open"); return 1; }
  bool ok = true;
  auto i32 = [&]() { int32_t v = 0; ok = ok && std::fread(&v, 4, 1, f) == 1; return (int)v; };
  auto f64 = [&]() { double v = 0; ok = ok && std::fread(&v, 8, 1, f) == 1; return v; };
  auto v3 = [&]() { StVO::Vector3d v; for (int c = 0; c < 3; ++c) v(c) = f64(); return v; };
  PgoMap m = {};
  m.min_lm_ess_graph = i32(); m.min_lm_cov_graph = i32(); m.max_iters_pgo = i32();
  const int n_kf = i32();
  for (int i = 0; ok && i < n_kf; ++i) {
    KeyFrame* kf = nullptr;
    if (i32()) {
      kf = new KeyFrame{i, nullptr, {}, {}};
      for (int c = 0; c < 16; ++c) kf->T_kf_w.v[c] = f64();
      kf->x_kf_w = StVO::logmap_se3(kf->T_kf_w);
    }
    m.map_keyframes.push_back(kf);
  }
  m.full_graph.assign(std::max(n_kf, 0), std::vector<unsigned int>(std::max(n_kf, 0), 0));
  for (int i = 0; ok && i < n_kf; ++i)
    for (int j = 0; ok && j < n_kf; ++j) m.full_graph[i][j] = (unsigned)i32();
  for (int k = 0, n = i32(); ok && k < n; ++k) {
    const int a = i32(), b = i32();
    m.lc_idx_list.push_back({a, b, 1});
    StVO::Vector6d x;
    for (int c = 0; c < 6; ++c) x(c) = f64();
    m.lc_pose_list.push_back(x);
  }
  for (int i = 0, n = i32(); ok && i < n; ++i) {
    MapPoint* pt = nullptr;
    if (i32()) {
      pt = new MapPoint{i, {}, {}, {}, {}, {}};
      pt->point3D = v3();
      pt->med_obs_dir = v3();
      for (int k = 0, nd = i32(); ok && k < nd; ++k) pt->dir_list.push_back(v3());
    }
    m.map_points.push_back(pt);
  }
  for (int i = 0, n = i32(); ok && i < n; ++i) {
    MapLine* ls = nullptr;
    if (i32()) {
      ls = new MapLine{i, {}, {}, {}, {}, {}};
      for (int c = 0; c < 6; ++c) ls->line3D(c) = f64();
      ls->med_obs_dir = v3();
      for (int k = 0, nd = i32(); ok && k < nd; ++k) ls->dir_list.push_back(v3());
    }
    m.map_lines.push_back(ls);
  }
  for (auto* lists : {&m.map_points_kf_idx, &m.map_lines_kf_idx})
    for (int i = 0; ok && i < n_kf; ++i) {
      std::vector<int> l;
      for (int k = 0, n = i32(); ok && k < n; ++k) l.push_back(i32());
      lists->push_back(l);
    }
  std::fclose(f);
  int rc = 0;
  if (!ok) { std::fprintf(stderr, "short read\n"); rc = 1; }
  plf_params prm;
  plf_default_params(&prm);
  plf_limits lim;
  plf_default_limits(&lim);
  lim.max_batch = 1;
  plf_camera cam = {1242, 375, 718.856, 718.856, 607.1928, 185.2157, 0.537165719};
  if (!rc && plf_create(&prm, &cam, &lim, 0, &m.ctx) != PLF_OK) {
    std::fprintf(stderr, "plf_create: %s\n", plf_last_error(nullptr));
    rc = 2;
  }
  auto print3 = [](const StVO::Vector3d& v) { for (int c = 0; c < 3; ++c) std::printf(" %.17g", v(c)); };
  if (!rc) {
    try {
      const plf_pgo_result res = loop_closure_optimization_cov_graph(m);
      std::printf("pgo result %d %d %d %.17g %.17g %.17g\n", res.iters, res.stop, res.trials, res.chi2_init, res.chi2,
                  res.lambda);
      for (KeyFrame* kf : m.map_keyframes) {
        if (!kf) continue;
        std::printf("pgo kf %d", kf->kf_idx);
        for (int c = 0; c < 16; ++c) std::printf(" %.17g", kf->T_kf_w.v[c]);
        std::printf("\n");
      }
      for (MapPoint* pt : m.map_points) {
        if (!pt) continue;
        std::printf("pgo pt %d", pt->idx);
        print3(pt->point3D);
        print3(pt->med_obs_dir);
        for (const auto& d : pt->dir_list) print3(d);
        std::printf("\n");
      }
      for (MapLine* ls : m.map_lines) {
        if (!ls) continue;
        std::printf("pgo ls %d", ls->idx);
        for (int c = 0; c < 6; ++c) std::printf(" %.17g", ls->line3D(c));
        print3(ls->med_obs_dir);
        for (const auto& d : ls->dir_list) print3(d);
        std::printf("\n");
      }
      for (const auto& lc : m.lc_idx_list) std::printf("pgo lc %d %d %d\n", lc[0], lc[1], lc[2]);
    } catch (const std::exception& e) {
      std::fprintf(stderr, "error: %s\n", e.what());
      rc = 2;
    }
    plf_destroy(m.ctx);
  }
  for (KeyFrame* kf : m.map_keyframes) delete kf;
  for (MapPoint* pt : m.map_points) delete pt;
  for (MapLine* ls : m.map_lines) delete ls;
  return rc;
}

int main(int argc, char** argv) {
  bool grid_test = false, kf_test = false;
  if (argc == 3 && std::string(argv[1]) == "--gba-selftest") return gba_selftest(argv[2]);
  if (argc == 3 && std::string(argv[1]) == "--pgo-selftest") return pgo_selftest(argv[2]);
  const char* bow_voc[2] = {nullptr, nullptr};
  bool lc_test = false;
  if (argc >= 4 && (std::string(argv[argc - 3]) == "--bow-selftest" || std::string(argv[argc - 3]) == "--lc-detect-selftest")) {
    lc_test = std::string(argv[argc - 3]) == "--lc-detect-selftest";
    bow_voc[0] = argv[argc - 2];
    bow_voc[1] = argv[argc - 1];
    argc -= 3;
  }
  // --color C (last): frames.bin holds colour images, C = 3 (BGR) or 4 (BGRA) interleaved bytes per pixel, which the shim
  // uploads as they are and the device converts to grey
  int channels = 1;
  if (argc >= 3 && std::string(argv[argc - 2]) == "--color") {
    channels = std::atoi(argv[argc - 1]);
    argc -= 2;
  }
  // --motion-model (last): stvo-pl's use_motion_model; prints "motion k valid T[16]", the prediction frame k started from,
  // after each frame's line
  bool motion_on = false;
  if (argc >= 2 && std::string(argv[argc - 1]) == "--motion-model") { motion_on = true; --argc; }
  // --adaptive-fast min max inc feat err: stvo-pl's adaptative_fast (fast_min_th .. fast_err_th); prints "fast_th k th",
  // the threshold frame k was detected with, after each frame's line
  plf_adaptive_fast afast;
  bool afast_on = false;
  if (argc >= 7 && std::string(argv[argc - 6]) == "--adaptive-fast") {
    afast = {std::atoi(argv[argc - 5]), std::atoi(argv[argc - 4]), std::atoi(argv[argc - 3]), std::atoi(argv[argc - 2]),
             std::atof(argv[argc - 1])};
    afast_on = true;
    argc -= 6;
  }
  if (argc >= 2 && std::string(argv[argc - 1]) == "--grid-selftest") { grid_test = true; --argc; }
  if (argc >= 2 && std::string(argv[argc - 1]) == "--kf-match-selftest") { kf_test = true; --argc; }
  if (argc < 2) {
    std::fprintf(stderr, "usage: %s frames.bin [orb_nfeatures lsd_nfeatures] [--color 3|4]\n", argv[0]);
    return 1;
  }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) { std::perror("open"); return 1; }
  int32_t hdr[3];
  double cam[5];
  if (std::fread(hdr, 4, 3, f) != 3 || std::fread(cam, 8, 5, f) != 5) { std::fprintf(stderr, "bad header\n"); return 1; }
  const int n = hdr[0], w = hdr[1], h = hdr[2];
  std::vector<uint8_t> buf((size_t)2 * w * h * channels);
  try {
    StVO::PinholeStereoCamera cam_pin(w, h, cam[0], cam[1], cam[2], cam[3], cam[4]);
    plf_params prm;
    plf_default_params(&prm);
    if (argc >= 4) { prm.orb_nfeatures = std::atoi(argv[2]); prm.lsd_nfeatures = std::atoi(argv[3]); }
    StVO::StereoFrameHandler* StVO_ = new StVO::StereoFrameHandler(&cam_pin, &prm, 0, afast_on ? &afast : nullptr, motion_on);   // app:109
    KfArrays* first_kf = nullptr;   // --kf-match-selftest: frame 0 against the last frame
    BowMap bow = {StVO_->ctx(), prm.has_points != 0, prm.has_lines != 0, {}, {}};
    LcMap lc = {bow, {}, 1, 2, 1, 20, 0};
    if (bow_voc[0]) {
      bow_load_vocabulary(bow.ctx, 0, bow_voc[0]);
      bow_load_vocabulary(bow.ctx, 1, bow_voc[1]);
    }
    int rc = 0;
    for (int frame_counter = 0; frame_counter < n; ++frame_counter) {                   // app:111
      if (std::fread(buf.data(), 1, buf.size(), f) != buf.size()) { std::fprintf(stderr, "short read\n"); return 1; }
      plf::Image img_l{buf.data(), w, h, w * channels, channels}, img_r{buf.data() + (size_t)w * h * channels, w, h, w * channels, channels};
      bool new_kf = false;
      StVO::StereoFrame* cur;
      const int fast_th = StVO_->orbFastTh();
      double T_pred[16];
      const bool pred_valid = StVO_->motionPrior(T_pred);
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
      if (afast_on) std::printf("fast_th %d %d\n", frame_counter, fast_th);
      if (motion_on) {
        std::printf("motion %d %d", frame_counter, pred_valid ? 1 : 0);
        for (int i = 0; i < 16; ++i) std::printf(" %.17g", T_pred[i]);
        std::printf("\n");
      }
      if (bow_voc[0] && !lc_test) bow_selftest_frame(bow, cur, frame_counter);
      if (lc_test) lc_selftest_frame(lc, cur, frame_counter);
      if (kf_test && frame_counter == 0) first_kf = new KfArrays(cur);
      if (kf_test && frame_counter == n - 1 && first_kf) {
        KfArrays last_kf(cur);
        rc = kf_match_selftest(StVO_->ctx(), *first_kf, last_kf);
      }
      if (frame_counter > 0) StVO_->updateFrame();                                      // app:159
    }
    delete first_kf;
    for (KeyFrame* kf : bow.map_keyframes) delete kf;
    for (KeyFrame* kf : lc.bow.map_keyframes) delete kf;
    delete StVO_;
    if (rc) return rc;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "error: %s\n", e.what());
    return 2;
  }
  std::fclose(f);
  return 0;
}
