"""ctypes binding of libplslam_b200.so (the C ABI in include/plslam_b200.h).

Thin by design: numpy arrays in, numpy arrays out, every call goes straight through the C ABI to the
CUDA kernels.  There is NO CPU fallback: if the shared library is missing or no CUDA device is
present, construction raises.  Used by tests/, bench.py and __graft_entry__.py.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

_PKG_DIR = Path(__file__).resolve().parent.parent  # pl-slam_b200/
REPO_ROOT = _PKG_DIR.parent
LIB_PATH = _PKG_DIR / "lib" / "libplslam_b200.so"

DESC_BYTES = 32
PLF_ERR_CAPACITY = -4   # plf_status of a call or batch problem that exceeded a capacity


class PlfError(RuntimeError):
    pass


class plf_params(C.Structure):
    _fields_ = [
        ("has_points", C.c_int), ("has_lines", C.c_int), ("best_lr_matches", C.c_int),
        ("max_dist_epip", C.c_float), ("min_disp", C.c_float), ("min_ratio_12_p", C.c_float),
        ("line_sim_th", C.c_float), ("stereo_overlap_th", C.c_float), ("f2f_overlap_th", C.c_float),
        ("min_line_length", C.c_float), ("line_horiz_th", C.c_float), ("min_ratio_12_l", C.c_float),
        ("ls_min_disp_ratio", C.c_float),
        ("homog_th", C.c_double),
        ("min_features", C.c_int), ("max_iters", C.c_int), ("max_iters_ref", C.c_int),
        ("min_error", C.c_double), ("min_error_change", C.c_double), ("inlier_k", C.c_double),
        ("orb_nfeatures", C.c_int), ("orb_scale_factor", C.c_float),
        ("orb_nlevels", C.c_int), ("orb_edge_th", C.c_int), ("orb_wta_k", C.c_int),
        ("orb_score", C.c_int), ("orb_patch_size", C.c_int), ("orb_fast_th", C.c_int),
        ("lsd_nfeatures", C.c_int), ("lsd_refine", C.c_int),
        ("lsd_scale", C.c_double), ("lsd_sigma_scale", C.c_double), ("lsd_quant", C.c_double),
        ("lsd_ang_th", C.c_double), ("lsd_log_eps", C.c_double), ("lsd_density_th", C.c_double),
        ("lsd_n_bins", C.c_int),
        ("matching_strategy", C.c_int), ("matching_s_ws", C.c_int), ("matching_f2f_ws", C.c_int),
        ("min_pt_matches", C.c_int), ("min_ls_matches", C.c_int),
    ]


class plf_camera(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("b", C.c_double)]


class plf_limits(C.Structure):
    _fields_ = [("max_batch", C.c_int), ("max_keypoints", C.c_int), ("max_segments", C.c_int),
                ("max_lines", C.c_int)]


class plf_adaptive_fast(C.Structure):
    _fields_ = [("min_th", C.c_int), ("max_th", C.c_int), ("inc_th", C.c_int), ("feat_th", C.c_int), ("err_th", C.c_double)]


# stvo-pl's fast_*_th block as every reference config sets it (config_euroc.yaml:36-41; fast_min_th 0 in config_kitti.yaml)
ADAPTIVE_FAST_DEFAULTS = dict(min_th=5, max_th=50, inc_th=5, feat_th=50, err_th=0.5)


class plf_lba_opts(C.Structure):
    _fields_ = [("lambda_", C.c_double), ("lambda_k", C.c_double), ("max_iters", C.c_int), ("homog_th", C.c_double),
                ("min_error", C.c_double), ("min_error_change", C.c_double), ("ref_quirks", C.c_int)]


class plf_lba_problem(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int), ("n_fixed", C.c_int),
                ("kf_pose", C.c_void_p), ("pt", C.c_void_p), ("ls", C.c_void_p), ("fixed_T", C.c_void_p),
                ("n_pt_obs", C.c_int), ("pt_obs_lm", C.c_void_p), ("pt_obs_kf", C.c_void_p), ("pt_obs_xy", C.c_void_p),
                ("n_ls_obs", C.c_int), ("ls_obs_lm", C.c_void_p), ("ls_obs_kf", C.c_void_p), ("ls_obs_le", C.c_void_p),
                ("pt_moved", C.c_void_p), ("ls_moved", C.c_void_p)]


class plf_lba_result(C.Structure):
    _fields_ = [("iters", C.c_int), ("err", C.c_double), ("lambda_", C.c_double)]


class plf_pgo_opts(C.Structure):
    _fields_ = [("max_iters", C.c_int), ("lambda_init", C.c_double)]


class plf_pgo_problem(C.Structure):
    _fields_ = [("n_v", C.c_int), ("n_e", C.c_int), ("T", C.c_void_p), ("fixed", C.c_void_p), ("from_", C.c_void_p),
                ("to", C.c_void_p), ("Z", C.c_void_p)]


class plf_pgo_trial(C.Structure):
    _fields_ = [("iter", C.c_int), ("accepted", C.c_int), ("lambda_", C.c_double), ("chi", C.c_double),
                ("chi_t", C.c_double), ("rho", C.c_double)]


class plf_pgo_result(C.Structure):
    _fields_ = [("iters", C.c_int), ("stop", C.c_int), ("trials", C.c_int), ("chi2_init", C.c_double),
                ("chi2", C.c_double), ("lambda_", C.c_double), ("trace", C.c_void_p), ("trace_cap", C.c_int),
                ("n_trace", C.c_int), ("scratch_bytes", C.c_size_t)]


PGO_STOP = {0: "max_iters", 1: "trials", 2: "rho_zero", 3: "lambda"}   # plf_pgo_result.stop
PGO_TRACE_DTYPE = np.dtype([("iter", np.int32), ("accepted", np.int32), ("lambda_", np.float64), ("chi", np.float64),
                            ("chi_t", np.float64), ("rho", np.float64)], align=True)
assert PGO_TRACE_DTYPE.itemsize == C.sizeof(plf_pgo_trial)


class plf_grid_window(C.Structure):
    _fields_ = [("width_lo", C.c_int), ("width_hi", C.c_int), ("height_lo", C.c_int), ("height_hi", C.c_int)]


class plf_gn_opts(C.Structure):
    _fields_ = [("homog_th", C.c_double), ("max_iters", C.c_int), ("max_iters_ref", C.c_int),
                ("eps_err", C.c_double), ("eps_change", C.c_double), ("eps_step", C.c_double)]


class plf_pose_result(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("cov", C.c_double * 36), ("x", C.c_double * 6),
                ("err", C.c_double), ("iters1", C.c_int), ("iters2", C.c_int),
                ("n_inliers_pt", C.c_int), ("n_inliers_ls", C.c_int)]


class plf_frame_result(C.Structure):
    _fields_ = [("DT", C.c_double * 16), ("DT_cov", C.c_double * 36), ("err", C.c_double), ("status", C.c_int),
                ("n_kp_l", C.c_int), ("n_kp_r", C.c_int), ("n_lines_l", C.c_int), ("n_lines_r", C.c_int),
                ("n_stereo_pt", C.c_int), ("n_stereo_ls", C.c_int), ("n_matched_pt", C.c_int),
                ("n_matched_ls", C.c_int), ("n_inliers_pt", C.c_int), ("n_inliers_ls", C.c_int),
                ("iters1", C.c_int), ("iters2", C.c_int)]


class plf_frame_view(C.Structure):
    _fields_ = [("cap_pt", C.c_int), ("cap_ls", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int),
                ("pt_pl", C.c_void_p), ("pt_disp", C.c_void_p), ("pt_P", C.c_void_p), ("pt_octave", C.c_void_p),
                ("pdesc", C.c_void_p), ("ls_spl", C.c_void_p), ("ls_epl", C.c_void_p), ("ls_sdisp", C.c_void_p),
                ("ls_edisp", C.c_void_p), ("ls_sP", C.c_void_p), ("ls_eP", C.c_void_p), ("ls_le", C.c_void_p),
                ("ls_angle", C.c_void_p), ("ldesc", C.c_void_p)]


class plf_match_view(C.Structure):
    _fields_ = [("cap_pt", C.c_int), ("cap_ls", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int),
                ("P", C.c_void_p), ("pl_obs", C.c_void_p), ("inlier_pt", C.c_void_p), ("sP", C.c_void_p),
                ("eP", C.c_void_p), ("le_obs", C.c_void_p), ("inlier_ls", C.c_void_p)]


class plf_lc_params(C.Structure):
    _fields_ = [("lc_res", C.c_double), ("lc_unc", C.c_double), ("lc_inl", C.c_double), ("lc_trs", C.c_double),
                ("lc_rot", C.c_double), ("lc_inlier_ratio", C.c_double)]


class plf_lc_keyframe(C.Structure):
    _fields_ = [("n_pt", C.c_int), ("n_ls", C.c_int), ("pdesc", C.c_void_p), ("P", C.c_void_p), ("pl", C.c_void_p),
                ("ldesc", C.c_void_p), ("sP", C.c_void_p), ("eP", C.c_void_p), ("le", C.c_void_p)]


class plf_lc_result(C.Structure):
    _fields_ = [("accepted", C.c_int), ("estimated", C.c_int), ("common_pt", C.c_int), ("common_ls", C.c_int),
                ("n_pt", C.c_int), ("n_ls", C.c_int), ("inl_ratio_pt", C.c_double), ("inl_ratio_ls", C.c_double),
                ("err", C.c_double), ("max_cov_eig", C.c_double), ("ratio_inliers", C.c_double), ("t", C.c_double),
                ("r", C.c_double), ("x_inc", C.c_double * 6), ("pose_inc", C.c_double * 6)]


class plf_gn_problem(C.Structure):
    _fields_ = [("P", C.c_void_p), ("pl_obs", C.c_void_p), ("inlier_pt", C.c_void_p), ("np", C.c_int),
                ("sP", C.c_void_p), ("eP", C.c_void_p), ("le_obs", C.c_void_p), ("inlier_ls", C.c_void_p), ("nl", C.c_int),
                ("T_init", C.c_void_p), ("out", plf_pose_result)]


class plf_lc_problem(C.Structure):
    _fields_ = [("kf0", C.POINTER(plf_lc_keyframe)), ("kf1", C.POINTER(plf_lc_keyframe)), ("pt_pairs", C.c_void_p),
                ("cap_pt", C.c_int), ("ls_pairs", C.c_void_p), ("cap_ls", C.c_int), ("out", plf_lc_result),
                ("status", C.c_int)]


class plf_kf_match_opts(C.Structure):
    _fields_ = [("fast_matching", C.c_int), ("max_kf_epip_p", C.c_double), ("max_kf_epip_l", C.c_double)]


class plf_local_map(C.Structure):
    _fields_ = [("n_pt", C.c_int), ("pt_X", C.c_void_p), ("pt_desc", C.c_void_p), ("pt_use", C.c_void_p),
                ("n_ls", C.c_int), ("ls_X", C.c_void_p), ("ls_desc", C.c_void_p), ("ls_use", C.c_void_p)]


class plf_kf2kf_problem(C.Structure):
    _fields_ = [("prev", C.POINTER(plf_frame_view)), ("curr", C.POINTER(plf_frame_view)), ("DT", C.c_double * 16),
                ("m_pt", C.c_void_p), ("m_ls", C.c_void_p), ("n_pt", C.c_int), ("n_ls", C.c_int)]


class plf_map2kf_problem(C.Structure):
    _fields_ = [("map", C.POINTER(plf_local_map)), ("kf", C.POINTER(plf_frame_view)), ("Twf", C.c_double * 16),
                ("kf_pt_lm", C.c_void_p), ("kf_ls_lm", C.c_void_p), ("lm_pt", C.c_void_p), ("lm_ls", C.c_void_p),
                ("n_pt", C.c_int), ("n_ls", C.c_int)]


class plf_bow_problem(C.Structure):
    _fields_ = [("kf_idx", C.c_int), ("kf", C.POINTER(plf_frame_view)), ("score_p", C.c_void_p), ("score_l", C.c_void_p)]


class plf_lc_detect_opts(C.Structure):
    _fields_ = [("lc_kf_dist", C.c_int), ("lc_kf_max_dist", C.c_int), ("lc_nkf_closest", C.c_int),
                ("min_lm_cov_graph", C.c_int), ("min_kf_local_map", C.c_int)]


class plf_lc_detect_result(C.Structure):
    _fields_ = [("candidate", C.c_int), ("best", C.c_int), ("n_listed", C.c_int), ("n_closest", C.c_int),
                ("min_score", C.c_double)]


class plf_lc_detect_problem(C.Structure):
    _fields_ = [("kf_idx", C.c_int), ("kf", C.POINTER(plf_frame_view)), ("covis", C.c_void_p), ("conf", C.c_void_p),
                ("score_p", C.c_void_p), ("score_l", C.c_void_p), ("result", plf_lc_detect_result)]


# SlamConfig's loop-closure detection defaults (src/slamConfig.cpp:61-62, :80-82)
LC_DETECT_DEFAULTS = dict(lc_kf_dist=50, lc_kf_max_dist=50, lc_nkf_closest=4, min_lm_cov_graph=75, min_kf_local_map=3)
LC_RESULT_FIELDS = ("candidate", "best", "n_listed", "n_closest", "min_score")
# SlamConfig's loop-closure pose check defaults (src/slamConfig.cpp:73-77, :83)
LC_POSE_DEFAULTS = dict(lc_res=1.0, lc_unc=0.01, lc_inl=0.3, lc_trs=1.5, lc_rot=35.0, lc_inlier_ratio=30.0)


def _lc_opts(opts):
    o = dict(LC_DETECT_DEFAULTS, **(opts or {}))
    return plf_lc_detect_opts(*[int(o[f]) for f, _ in plf_lc_detect_opts._fields_])


def _lc_params(lc):
    return plf_lc_params(**dict(LC_POSE_DEFAULTS, **(lc or {})))


class plf_vocab(C.Structure):
    _fields_ = [("k", C.c_int), ("L", C.c_int), ("scoring", C.c_int), ("weighting", C.c_int), ("n_nodes", C.c_int),
                ("node_id", C.c_void_p), ("parent_id", C.c_void_p), ("weight", C.c_void_p), ("desc", C.c_void_p),
                ("n_words", C.c_int), ("word_id", C.c_void_p), ("word_node", C.c_void_p)]


# plf_vocab arrays: (name, dtype, columns, count field)
_VOCAB_ARRAYS = (("node_id", np.int32, 0, "n_nodes"), ("parent_id", np.int32, 0, "n_nodes"),
                 ("weight", np.float64, 0, "n_nodes"), ("desc", np.uint8, 32, "n_nodes"),
                 ("word_id", np.int32, 0, "n_words"), ("word_node", np.int32, 0, "n_words"))


def read_vocab_yml(path) -> dict:
    """plf_vocab_read_yml: a DBoW2 vocabulary YAML file as a dict of k, L, scoring, weighting and the arrays in file order
    (node_id, parent_id, weight, desc [n][32], word_id, word_node).  Host only; raises PlfError on a malformed file."""
    lib = load_library()
    v = plf_vocab()
    st = lib.plf_vocab_read_yml(str(path).encode(), C.byref(v))
    if st != 0:
        raise PlfError(f"plf_vocab_read_yml failed ({st}): {lib.plf_last_error(None).decode()}")
    try:
        out = dict(k=v.k, L=v.L, scoring=v.scoring, weighting=v.weighting)
        for name, dt, cols, count in _VOCAB_ARRAYS:
            n = getattr(v, count) * max(cols, 1)
            a = np.ctypeslib.as_array(C.cast(getattr(v, name), C.POINTER(np.ctypeslib.as_ctypes_type(dt))), (n,)).copy()
            out[name] = a.reshape(-1, cols) if cols else a
    finally:
        lib.plf_vocab_free(C.byref(v))
    return out


def _vocab_struct(voc: dict, keep: list) -> plf_vocab:
    v = plf_vocab(int(voc["k"]), int(voc.get("L", 0)), int(voc.get("scoring", 0)), int(voc.get("weighting", 0)))
    for name, dt, cols, count in _VOCAB_ARRAYS:
        a = np.ascontiguousarray(voc[name], dt)
        keep.append(a)
        setattr(v, name, a.ctypes.data if a.size else None)
        setattr(v, count, len(a))
    return v


# the plf_frame_view fields the keyframe matchers read: (name, dtype, columns)
_KF_VIEW_FIELDS = (("pt_pl", np.float64, 2), ("pt_P", np.float64, 3), ("pdesc", np.uint8, 32), ("ls_spl", np.float64, 2),
                   ("ls_epl", np.float64, 2), ("ls_sP", np.float64, 3), ("ls_eP", np.float64, 3), ("ls_le", np.float64, 3),
                   ("ldesc", np.uint8, 32))


def _frame_view(frame, keep):
    """A plf_frame_view over the arrays of a get_frame dict (missing arrays stay NULL; `keep` holds the copies alive)."""
    v = plf_frame_view()
    v.n_pt, v.n_ls = len(frame.get("pdesc", ())), len(frame.get("ldesc", ()))
    for name, dt, cols in _KF_VIEW_FIELDS:
        if name in frame:
            a = np.ascontiguousarray(frame[name], dt).reshape(-1, cols)
            keep.append(a)
            setattr(v, name, a.ctypes.data if a.size else None)
    return v


def _local_map(local_map, kf_view, kf_pt_lm, kf_ls_lm, keep, who):
    """(plf_local_map, kf_pt_lm, kf_ls_lm) over a match_map2kf local-map dict and the keyframe's landmark indices (arrays
    or None), checked against the keyframe's feature counts; `keep` holds the copies alive."""
    m = plf_local_map()

    def arr(a, dt, cols):
        a = np.ascontiguousarray(a, dt).reshape(-1, cols) if cols else np.ascontiguousarray(a, dt).ravel()
        keep.append(a)
        return a
    for key, cols in (("pt", 3), ("ls", 6)):
        X = arr(local_map.get(key + "_X", np.zeros((0, cols))), np.float64, cols)
        d = arr(local_map.get(key + "_desc", np.zeros((0, 32))), np.uint8, 32)
        u = local_map.get(key + "_use")
        setattr(m, "n_" + key, len(X))
        setattr(m, key + "_X", X.ctypes.data if X.size else None)
        setattr(m, key + "_desc", d.ctypes.data if d.size else None)
        if u is not None:
            u = arr(np.asarray(u).astype(np.uint8), np.uint8, 0)
            setattr(m, key + "_use", u.ctypes.data if u.size else None)
    lms = [None if v is None else arr(v, np.int32, 0) for v in (kf_pt_lm, kf_ls_lm)]
    for a, n, name in ((lms[0], kf_view.n_pt, "kf_pt_lm"), (lms[1], kf_view.n_ls, "kf_ls_lm")):
        if a is not None and len(a) != n:
            raise PlfError(f"{who}: {name} has {len(a)} entries for {n} keyframe features")
    return m, lms[0], lms[1]


def _kf_match_opts(fast_matching, max_kf_epip_p, max_kf_epip_l):
    return plf_kf_match_opts(int(bool(fast_matching)), float(max_kf_epip_p), float(max_kf_epip_l))


def _kf2kf_problem(prev, curr, DT, keep):
    """(plf_kf2kf_problem, m_pt, m_ls) over match_kf2kf's arguments: the struct and its output arrays, cut to the previous
    keyframe's feature counts; `keep` holds the copies alive."""
    p, c = _frame_view(prev, keep), _frame_view(curr, keep)
    m_pt, m_ls = np.full(max(p.n_pt, 1), -1, np.int32), np.full(max(p.n_ls, 1), -1, np.int32)
    keep += [p, c]
    T = (C.c_double * 16)(*np.ascontiguousarray(DT, np.float64).reshape(16))
    prob = plf_kf2kf_problem(C.pointer(p), C.pointer(c), T, m_pt.ctypes.data, m_ls.ctypes.data, 0, 0)
    return prob, m_pt[:p.n_pt], m_ls[:p.n_ls]


def _map2kf_problem(local_map, Twf, kf, kf_pt_lm, kf_ls_lm, keep, who):
    """(plf_map2kf_problem, lm_pt, lm_ls) over match_map2kf's arguments: the struct and its output arrays, cut to the
    local map's landmark counts; `keep` holds the copies alive."""
    kv = _frame_view(kf, keep)
    m, pt_lm, ls_lm = _local_map(local_map, kv, kf_pt_lm, kf_ls_lm, keep, who)
    lm_pt, lm_ls = np.full(max(m.n_pt, 1), -1, np.int32), np.full(max(m.n_ls, 1), -1, np.int32)
    keep += [kv, m]
    ad = lambda a: None if a is None or not a.size else a.ctypes.data
    T = (C.c_double * 16)(*np.ascontiguousarray(Twf, np.float64).reshape(16))
    prob = plf_map2kf_problem(C.pointer(m), C.pointer(kv), T, ad(pt_lm), ad(ls_lm), lm_pt.ctypes.data, lm_ls.ctypes.data,
                              0, 0)
    return prob, lm_pt[:m.n_pt], lm_ls[:m.n_ls]


RESULT_DTYPE =np.dtype([("DT", np.float64, (4, 4)), ("DT_cov", np.float64, (6, 6)), ("err", np.float64),
                         ("status", np.int32), ("n_kp_l", np.int32), ("n_kp_r", np.int32), ("n_lines_l", np.int32),
                         ("n_lines_r", np.int32), ("n_stereo_pt", np.int32), ("n_stereo_ls", np.int32),
                         ("n_matched_pt", np.int32), ("n_matched_ls", np.int32), ("n_inliers_pt", np.int32),
                         ("n_inliers_ls", np.int32), ("iters1", np.int32), ("iters2", np.int32)], align=True)
assert RESULT_DTYPE.itemsize == C.sizeof(plf_frame_result)

class plf_image_geometry(C.Structure):
    _fields_ = [("pitch", C.c_int), ("orb_nlevels", C.c_int), ("orb_w", C.c_int * 8), ("orb_h", C.c_int * 8),
                ("lsd_w", C.c_int), ("lsd_h", C.c_int), ("grid_iw", C.c_double), ("grid_ih", C.c_double)]


def image_geometry(width, height, params=None):
    """What the front-end derives from a width x height image, as the library computes it (host only, no device):
    dict of pitch, orb_levels [(w, h) per ORB level], lsd_size (w, h) and grid_scale (64 / w, 48 / h).  params: a
    plf_params (None: the defaults).  Raises PlfError for a size the pipeline refuses.  plf_get_image_geometry."""
    lib = load_library()
    g = plf_image_geometry()
    st = lib.plf_get_image_geometry(None if params is None else C.byref(params), int(width), int(height), C.byref(g))
    if st != 0:
        raise PlfError(f"plf_get_image_geometry failed ({st}): {lib.plf_last_error(None).decode()}")
    return dict(pitch=g.pitch, orb_levels=[(g.orb_w[l], g.orb_h[l]) for l in range(g.orb_nlevels)],
                lsd_size=(g.lsd_w, g.lsd_h), grid_scale=(g.grid_iw, g.grid_ih))


RESULT_FIELDS = ["status", "n_kp_l", "n_kp_r", "n_lines_l", "n_lines_r", "n_stereo_pt", "n_stereo_ls", "n_matched_pt",
                 "n_matched_ls", "n_inliers_pt", "n_inliers_ls", "iters1", "iters2"]

KEYLINE_DTYPE = np.dtype([
    ("angle", np.float32), ("class_id", np.int32), ("octave", np.int32),
    ("ptx", np.float32), ("pty", np.float32), ("response", np.float32), ("size", np.float32),
    ("startPointX", np.float32), ("startPointY", np.float32), ("endPointX", np.float32),
    ("endPointY", np.float32), ("sPointInOctaveX", np.float32), ("sPointInOctaveY", np.float32),
    ("ePointInOctaveX", np.float32), ("ePointInOctaveY", np.float32), ("lineLength", np.float32),
    ("numOfPixels", np.int32)])  # == plf_keyline == cv::line_descriptor::KeyLine

KEYPOINT_DTYPE = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                           ("response", np.float32), ("octave", np.int32), ("class_id", np.int32)])  # cv::KeyPoint

_lib = None


def load_library() -> C.CDLL:
    """Loads libplslam_b200.so; raises PlfError (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise PlfError(f"{LIB_PATH} not built: run `make` (or __graft_entry__.build()) first; "
                       "there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    lib.plf_last_error.restype = C.c_char_p
    lib.plf_last_error.argtypes = [C.c_void_p]
    lib.plf_sequence_param_fields.restype = C.c_int
    lib.plf_sequence_param_fields.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int]
    lib.plf_launch_count.restype = C.c_longlong
    lib.plf_launch_count.argtypes = [C.c_void_p]
    lib.plf_stream.restype = C.c_void_p
    lib.plf_stream.argtypes = [C.c_void_p]
    _pi, _pu8 = C.POINTER(C.c_int), C.POINTER(C.c_uint8)
    lib.plf_match_grid_points.argtypes = [C.c_void_p, _pi, _pu8, C.c_int, _pi, _pi, _pu8, C.c_int, C.c_int, C.c_int,
                                          plf_grid_window, C.c_float, C.c_int, C.POINTER(C.c_int32), _pi]
    lib.plf_match_grid_lines.argtypes = [C.c_void_p, _pi, _pu8, C.c_int, _pi, _pi, C.POINTER(C.c_double), _pu8, C.c_int,
                                         C.c_int, C.c_int, plf_grid_window, C.c_float, C.c_double, C.c_int,
                                         C.POINTER(C.c_int32), _pi]
    lib.plf_debug_match_grid_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _pi, _pi, C.POINTER(C.c_double),
                                               _pu8, _pu8, _pi, _pi, _pi, C.c_int, C.c_int, plf_grid_window, C.c_int,
                                               C.c_int, C.c_float, C.c_double, C.c_int, C.POINTER(C.c_int32), _pi]
    lib.plf_destroy.restype = None
    lib.plf_destroy.argtypes = [C.c_void_p]
    lib.plf_batch_device_images.restype = C.c_void_p
    lib.plf_batch_device_images.argtypes = [C.c_void_p]
    lib.plf_default_params.restype = None
    lib.plf_default_limits.restype = None
    _lib = lib
    return lib


def default_params() -> plf_params:
    p = plf_params()
    load_library().plf_default_params(C.byref(p))
    return p


def default_limits() -> plf_limits:
    l = plf_limits()
    load_library().plf_default_limits(C.byref(l))
    return l


KITTI_CAMERA = dict(width=1242, height=375, fx=718.856, fy=718.856, cx=607.1928, cy=185.2157,
                    b=0.537165719)  # config/dataset_params/kitti00-02.yaml:2-10
EUROC_CAMERA = dict(width=752, height=480, fx=458.654, fy=457.296, cx=367.215, cy=248.375,
                    b=0.110077842)  # config/dataset_params/euroc_params.yaml:2,8 (pre-rectified)
DBL_EPSILON = float(np.finfo(np.float64).eps)   # numeric_limits<double>::epsilon(), the GBA stop thresholds


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def _i32_or_null(a):
    """int32* over a, or NULL for None (the seq arrays of the batch calls)."""
    return None if a is None else _ptr(a, C.c_int32)


def _lba_opts(lambda_, lambda_k, max_iters, homog_th, min_error, min_error_change, ref_quirks):
    return plf_lba_opts(lambda_, lambda_k, max_iters, homog_th, min_error, min_error_change, int(ref_quirks))


PARAM_CLASSES = {1: "sequence", 2: "context", 3: "ignored"}   # PLF_PARAM_SEQUENCE, _CONTEXT, _IGNORED


def sequence_param_fields():
    """{plf_params field: "sequence" | "context" | "ignored"}: how Frontend.set_sequence_params treats each field, as the
    library classifies them (plf_sequence_param_fields).  "sequence" fields may differ per sequence, "context" fields
    must equal the context's, "ignored" fields have no effect."""
    lib = load_library()
    n = lib.plf_sequence_param_fields(None, None, 0)
    names, classes = (C.c_char_p * n)(), (C.c_int * n)()
    lib.plf_sequence_param_fields(names, classes, n)
    return {names[i].decode(): PARAM_CLASSES[classes[i]] for i in range(n)}


class Frontend:
    """One plf_ctx (one device, one stream).  Mirrors the role of `StereoFrameHandler`
    (app/plslam_dataset.cpp:109) plus the free operators the reference calls on the path."""

    def __init__(self, params: plf_params | None = None, camera: dict | plf_camera | None = None,
                 limits: plf_limits | None = None, device: int = 0, max_sequences: int = 1,
                 adaptive_fast: dict | None = None, motion_model: bool = False, image_sizes=None, **overrides):
        """max_sequences: the number of sequences batch_run / process_batch can track at once (plf_set_max_sequences).
        image_sizes: None, or the (width, height) image sizes the batched pipeline accepts besides the camera's
        (set_image_sizes).
        adaptive_fast: None, or the per-sequence FAST threshold adaptation as set_adaptive_fast takes it.
        motion_model: stvo-pl's use_motion_model (set_motion_model)."""
        self.lib = load_library()
        self.params = params if params is not None else default_params()
        for k, v in overrides.items():
            if hasattr(self.params, k):
                setattr(self.params, k, v)
            else:
                raise PlfError(f"unknown parameter {k}")
        if camera is None:
            camera = KITTI_CAMERA
        self.camera = camera if isinstance(camera, plf_camera) else plf_camera(**camera)
        self.limits = limits if limits is not None else default_limits()
        self._ctx = C.c_void_p()
        self.image_sizes = []
        st = self.lib.plf_create(C.byref(self.params), C.byref(self.camera), C.byref(self.limits),
                                 int(device), C.byref(self._ctx))
        if st != 0:
            raise PlfError(f"plf_create failed ({st}): {self.lib.plf_last_error(None).decode()}")
        try:
            self._check(self.lib.plf_set_max_sequences(self._ctx, int(max_sequences)), "plf_set_max_sequences")
            if image_sizes:
                self.set_image_sizes(image_sizes)
            if adaptive_fast is not None:
                self.set_adaptive_fast(adaptive_fast)
            if motion_model:
                self.set_motion_model(True)
        except PlfError:
            self.close()
            raise
        self.max_sequences = int(max_sequences)

    # -- plumbing --------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.plf_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, st: int, what: str):
        if st != 0:
            raise PlfError(f"{what} failed ({st}): {self.lib.plf_last_error(self._ctx).decode()}")

    @property
    def launches(self) -> int:
        return int(self.lib.plf_launch_count(self._ctx))

    @property
    def stream(self) -> int:
        return int(self.lib.plf_stream(self._ctx) or 0)

    def sync(self):
        self._check(self.lib.plf_sync(self._ctx), "plf_sync")

    # -- matching --------------------------------------------------------------------------------
    def hamming_knn2(self, d1, d2):
        """cv::BFMatcher(NORM_HAMMING).knnMatch(d1, d2, k=2): returns idx1, dist1, idx2, dist2."""
        d1 = _u8(d1).reshape(-1, DESC_BYTES)
        d2 = _u8(d2).reshape(-1, DESC_BYTES)
        n1, n2 = len(d1), len(d2)
        out = [np.full(n1, -1, np.int32) for _ in range(4)]
        st = self.lib.plf_hamming_knn2(self._ctx, _ptr(d1, C.c_uint8), n1, _ptr(d2, C.c_uint8), n2,
                                       *[_ptr(o, C.c_int32) for o in out])
        self._check(st, "plf_hamming_knn2")
        return tuple(out)

    def match(self, d1, d2, nnr: float, best_lr: bool = True):
        """stvo-pl match(): returns (matches_12 int32[n1], n_matches)."""
        d1 = _u8(d1).reshape(-1, DESC_BYTES)
        d2 = _u8(d2).reshape(-1, DESC_BYTES)
        n1, n2 = len(d1), len(d2)
        m = np.full(n1, -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match(self._ctx, _ptr(d1, C.c_uint8), n1, _ptr(d2, C.c_uint8), n2,
                                C.c_float(nnr), int(bool(best_lr)), _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match")
        return m, cnt.value

    def match_grid_points(self, q_cell, d1, cell_start, cell_items, d2, cols, rows, w, nnr, best_lr=True):
        """stvo-pl matchGrid (points): q_cell int32 [n1,2]; the GridStructure as (cell_start, cell_items), cell (x, y) at
        x*rows + y; w = (width.first, width.second, height.first, height.second)."""
        q = np.ascontiguousarray(q_cell, np.int32).reshape(-1, 2)
        cs = np.ascontiguousarray(cell_start, np.int32); ci = np.ascontiguousarray(cell_items, np.int32)
        d1 = _u8(d1).reshape(-1, DESC_BYTES); d2 = _u8(d2).reshape(-1, DESC_BYTES)
        m = np.full(len(q), -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match_grid_points(self._ctx, _ptr(q, C.c_int), _ptr(d1, C.c_uint8), len(q), _ptr(cs, C.c_int),
                                            _ptr(ci, C.c_int), _ptr(d2, C.c_uint8), len(d2), int(cols), int(rows),
                                            plf_grid_window(*[int(v) for v in w]), C.c_float(nnr), int(bool(best_lr)),
                                            _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match_grid_points")
        return m, cnt.value

    def match_grid_lines(self, q_line, d1, cell_start, cell_items, t_dir, d2, cols, rows, w, nnr, line_sim_th, best_lr=True):
        """stvo-pl matchGrid (lines): q_line int32 [n1,4] end-point cells, grid as above, directions2 f64 [n2,2]."""
        q = np.ascontiguousarray(q_line, np.int32).reshape(-1, 4)
        cs = np.ascontiguousarray(cell_start, np.int32); ci = np.ascontiguousarray(cell_items, np.int32)
        td = np.ascontiguousarray(t_dir, np.float64).reshape(-1, 2)
        d1 = _u8(d1).reshape(-1, DESC_BYTES); d2 = _u8(d2).reshape(-1, DESC_BYTES)
        m = np.full(len(q), -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match_grid_lines(self._ctx, _ptr(q, C.c_int), _ptr(d1, C.c_uint8), len(q), _ptr(cs, C.c_int),
                                           _ptr(ci, C.c_int), _ptr(td, C.c_double), _ptr(d2, C.c_uint8), len(d2), int(cols),
                                           int(rows), plf_grid_window(*[int(v) for v in w]), C.c_float(nnr),
                                           C.c_double(line_sim_th), int(bool(best_lr)), _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match_grid_lines")
        return m, cnt.value

    def debug_match_grid_batch(self, q_geo, t_geo, d1, d2, n1, n2, cols, rows, w, nnr, t_dir=None, line_sim_th=0.0,
                               best_lr=True, clip=False, q_slot=None):
        """The batched windowed matcher on P problems at uniform capacities: q_geo int32 [P,K,2] query cells (points)
        or [P,K,4] end points (lines, then t_dir f64 [P,Kt,2] is required), t_geo [P,Kt,2|4], d1 [P,K,32],
        d2 [P,Kt,32], counts n1 / n2 [P] (clamped to K / Kt), q_slot [P] or None.  Returns (matches_12 int32 [P,K],
        n_matches int32 [P]).  plf_debug_match_grid_batch."""
        q = np.ascontiguousarray(q_geo, np.int32)
        t = np.ascontiguousarray(t_geo, np.int32)
        P, K, g = q.shape
        Kt = t.shape[1]
        lines = g == 4
        if t.shape != (P, Kt, g) or g not in (2, 4) or (lines and t_dir is None):
            raise PlfError(f"debug_match_grid_batch: q_geo {q.shape} and t_geo {t.shape} must be [P,K,2|4] and [P,Kt,2|4]"
                           " (t_dir with lines)")
        d1 = _u8(d1).reshape(P, K, DESC_BYTES); d2 = _u8(d2).reshape(P, Kt, DESC_BYTES)
        td = np.ascontiguousarray(t_dir if lines else np.zeros((P, Kt, 2)), np.float64).reshape(P, Kt, 2)
        n1 = np.ascontiguousarray(n1, np.int32).reshape(P); n2 = np.ascontiguousarray(n2, np.int32).reshape(P)
        qs = None if q_slot is None else np.ascontiguousarray(q_slot, np.int32).reshape(P)
        m = np.full((P, K), -1, np.int32)
        cnt = np.zeros(P, np.int32)
        st = self.lib.plf_debug_match_grid_batch(self._ctx, P, K, Kt, _ptr(q, C.c_int), _ptr(t, C.c_int),
                                                 _ptr(td, C.c_double), _ptr(d1, C.c_uint8), _ptr(d2, C.c_uint8),
                                                 _ptr(n1, C.c_int), _ptr(n2, C.c_int), None if qs is None else _ptr(qs, C.c_int),
                                                 int(cols), int(rows), plf_grid_window(*[int(v) for v in w]), int(lines),
                                                 int(bool(clip)), C.c_float(nnr), C.c_double(line_sim_th),
                                                 int(bool(best_lr)), _ptr(m, C.c_int32), _ptr(cnt, C.c_int))
        self._check(st, "plf_debug_match_grid_batch")
        return m, cnt

    def median_descriptors(self, desc, offsets, dirs=None):
        """MapPoint/MapLine::updateAverageDescDir over many landmarks: (med_idx int32[L], med_dir f64[L,3] or None)."""
        desc = _u8(desc).reshape(-1, DESC_BYTES)
        offsets = np.ascontiguousarray(offsets, np.int32)
        L = len(offsets) - 1
        idx = np.full(max(L, 0), -1, np.int32)
        md = None
        dp = None
        if dirs is not None:
            dirs = np.ascontiguousarray(dirs, np.float64).reshape(-1, 3)
            md = np.zeros((max(L, 0), 3), np.float64)
            dp = _ptr(dirs, C.c_double)
        st = self.lib.plf_median_descriptors(self._ctx, _ptr(desc, C.c_uint8), _ptr(offsets, C.c_int), dp, L,
                                             _ptr(idx, C.c_int), _ptr(md, C.c_double) if md is not None else None)
        self._check(st, "plf_median_descriptors")
        return idx, md

    # -- line descriptor -------------------------------------------------------------------------
    def lbd_gradients(self, img):
        """BinaryDescriptor::computeSobel: returns (dx, dy) int16 of the 5x5-blurred image."""
        img = _u8(img)
        h, w = img.shape
        out = np.empty((h, w, 2), np.int16)
        st = self.lib.plf_lbd_gradients(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                        _ptr(out, C.c_int16))
        self._check(st, "plf_lbd_gradients")
        return out[..., 0].copy(), out[..., 1].copy()

    def lbd(self, img, keylines, want_float=False):
        """BinaryDescriptor::compute(img, keylines, desc): returns uint8[n,32] (and float32[n,72])."""
        img = _u8(img)
        h, w = img.shape
        kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
        n = len(kl)
        desc = np.zeros((n, 32), np.uint8)
        fl = np.zeros((n, 72), np.float32) if want_float else None
        st = self.lib.plf_lbd(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                              kl.ctypes.data_as(C.c_void_p), n, _ptr(desc, C.c_uint8),
                              _ptr(fl, C.c_float) if want_float else None)
        self._check(st, "plf_lbd")
        return (desc, fl) if want_float else desc

    # -- pose refinement -------------------------------------------------------------------------
    def gn_pose(self, P, pl_obs, sP, eP, le_obs, inlier_pt=None, inlier_ls=None, T_init=None, opts=None):
        """StereoFrameHandler::optimizePose.  Returns dict(T, cov, x, err, iters, inlier_pt, inlier_ls)."""
        keep = []
        p, ip, il = self._gn_problem(dict(P=P, pl_obs=pl_obs, sP=sP, eP=eP, le_obs=le_obs, inlier_pt=inlier_pt,
                                          inlier_ls=inlier_ls, T_init=T_init), keep)
        vp = C.c_void_p
        st = self.lib.plf_gn_pose(self._ctx, C.byref(opts) if opts is not None else None, vp(p.P), vp(p.pl_obs),
                                  vp(p.inlier_pt), p.np, vp(p.sP), vp(p.eP), vp(p.le_obs), vp(p.inlier_ls), p.nl,
                                  vp(p.T_init), C.byref(p.out))
        self._check(st, "plf_gn_pose")
        return self._gn_result(p.out, ip, il)

    @staticmethod
    def _gn_problem(pr, keep):
        """(plf_gn_problem, inlier_pt, inlier_ls) over a gn_pose_batch problem dict's arrays, converted where needed and
        kept alive in keep; the inlier flags are copies, which the call updates."""
        f64 = lambda a, k: np.ascontiguousarray(a, np.float64).reshape(-1, k)
        P, O, sP, eP, le = f64(pr["P"], 3), f64(pr["pl_obs"], 2), f64(pr["sP"], 3), f64(pr["eP"], 3), f64(pr["le_obs"], 3)
        ip = pr.get("inlier_pt"); il = pr.get("inlier_ls")
        ip = np.ones(len(P), np.uint8) if ip is None else np.ascontiguousarray(ip, np.uint8).copy()
        il = np.ones(len(sP), np.uint8) if il is None else np.ascontiguousarray(il, np.uint8).copy()
        T0 = pr.get("T_init")
        T0 = None if T0 is None else np.ascontiguousarray(T0, np.float64).reshape(16)
        keep += [P, O, sP, eP, le, T0]
        ad = lambda a: a.ctypes.data if a is not None and a.size else None
        return plf_gn_problem(ad(P), ad(O), ad(ip), len(P), ad(sP), ad(eP), ad(le), ad(il), len(sP), ad(T0)), ip, il

    @staticmethod
    def _gn_result(out, ip, il):
        return dict(T=np.array(out.T).reshape(4, 4), cov=np.array(out.cov).reshape(6, 6), x=np.array(out.x),
                    err=out.err, iters=(out.iters1, out.iters2), inlier_pt=ip, inlier_ls=il,
                    n_inliers=(out.n_inliers_pt, out.n_inliers_ls))

    def gn_pose_batch(self, problems, seq=None, opts=None):
        """Many gn_pose in one device call (plf_gn_pose_batch), with one opts.  problems: dicts P, pl_obs, sP, eP, le_obs and
        optionally inlier_pt, inlier_ls, T_init, as gn_pose takes them; seq: per problem, -1 for the context's camera or a
        sequence whose camera (sequence_camera) to project with (None = all -1).  Returns one gn_pose dict per problem plus
        `status` (0)."""
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        keep, flags = [], []
        arr = (plf_gn_problem * max(P, 1))()
        for k, pr in enumerate(problems):
            arr[k], ip, il = self._gn_problem(pr, keep)
            flags.append((ip, il))
        self._check(self.lib.plf_gn_pose_batch(self._ctx, C.byref(opts) if opts is not None else None, P, arr,
                                               _i32_or_null(seq_a)), "plf_gn_pose_batch")
        return [dict(self._gn_result(arr[k].out, ip, il), status=0) for k, (ip, il) in enumerate(flags)]

    def loop_closure_pose(self, kf0, kf1, lc=None):
        """MapHandler::isLoopClosure + computeRelativePoseRobustGN (src/mapHandler.cpp:3192-3300, :3566-3957).
        kf0 / kf1: dicts with pdesc, P, pl, ldesc, sP, eP, le (numpy); lc: dict of the lc_* thresholds."""
        lcp = _lc_params(lc)
        keep = []
        k0, k1 = self._lc_keyframe(kf0, keep), self._lc_keyframe(kf1, keep)
        cap_p, cap_l = max(k0.n_pt, 1), max(k0.n_ls, 1)
        pp = np.full((cap_p, 2), -1, np.int32); lp = np.full((cap_l, 2), -1, np.int32)
        out = plf_lc_result()
        st = self.lib.plf_loop_closure_pose(self._ctx, C.byref(lcp), C.byref(k0), C.byref(k1), C.byref(out),
                                            _ptr(pp, C.c_int32), cap_p, _ptr(lp, C.c_int32), cap_l)
        self._check(st, "plf_loop_closure_pose")
        return self._lc_pose_result(out, pp, lp)

    @staticmethod
    def _lc_pose_result(out, pp, lp):
        """loop_closure_pose's dict from a plf_lc_result and its pair arrays (cut to the capacities the call had)."""
        r = {f: getattr(out, f) for f, _ in plf_lc_result._fields_ if f not in ("x_inc", "pose_inc")}
        r.update(accepted=bool(out.accepted), estimated=bool(out.estimated), x_inc=np.array(out.x_inc),
                 pose_inc=np.array(out.pose_inc), pt_pairs=pp[:out.n_pt].copy(), ls_pairs=lp[:out.n_ls].copy())
        return r

    @staticmethod
    def _lc_keyframe(k, keep):
        """plf_lc_keyframe over copies of a keyframe dict's arrays (kept alive in keep)."""
        f = plf_lc_keyframe()
        pd = _u8(k["pdesc"]).reshape(-1, 32); ld = _u8(k["ldesc"]).reshape(-1, 32)
        arrs = dict(pdesc=pd, ldesc=ld)
        for name, cols in (("P", 3), ("pl", 2), ("sP", 3), ("eP", 3), ("le", 3)):
            arrs[name] = np.ascontiguousarray(k[name], np.float64).reshape(-1, cols)
        f.n_pt, f.n_ls = len(pd), len(ld)
        for name, a in arrs.items():
            keep.append(a)
            setattr(f, name, a.ctypes.data if a.size else None)
        keep.append(f)
        return f

    def loop_closure_pose_batch(self, pairs, seq=None, lc=None):
        """Many loop_closure_pose in one device call (plf_loop_closure_pose_batch), with one set of lc thresholds.  pairs:
        (kf0, kf1) tuples of loop_closure_pose's keyframe dicts, or dicts kf0, kf1 and optionally cap_pt / cap_ls (pair
        capacities; default: kf0's feature counts, which always suffice); seq: as gn_pose_batch.  Returns one
        loop_closure_pose dict per pair plus `status` (0, or PLF_ERR_CAPACITY = -4 when that pair's correspondences
        exceed its capacity: its dict then holds what the single call leaves, pairs cut at the capacity).  Raises
        PlfError for the refusals before any work."""
        pairs = list(pairs)
        P = len(pairs)
        seq_a = self._problem_sequences(P, seq)
        lcp = _lc_params(lc)
        keep, outs = [], []
        arr = (plf_lc_problem * max(P, 1))()
        for k, pr in enumerate(pairs):
            if not isinstance(pr, dict):
                pr = dict(kf0=pr[0], kf1=pr[1])
            k0, k1 = self._lc_keyframe(pr["kf0"], keep), self._lc_keyframe(pr["kf1"], keep)
            cap_p, cap_l = int(pr.get("cap_pt", k0.n_pt)), int(pr.get("cap_ls", k0.n_ls))
            pp = np.full((max(cap_p, 1), 2), -1, np.int32); lp = np.full((max(cap_l, 1), 2), -1, np.int32)
            outs.append((pp[:cap_p], lp[:cap_l]))
            arr[k] = plf_lc_problem(C.pointer(k0), C.pointer(k1), pp.ctypes.data, cap_p, lp.ctypes.data, cap_l,
                                    plf_lc_result(), 1)   # 1 is no plf_status: marks entries the call did not write
        rc = self.lib.plf_loop_closure_pose_batch(self._ctx, C.byref(lcp), P, arr, _i32_or_null(seq_a))
        if rc != 0 and (rc != PLF_ERR_CAPACITY or P == 0 or any(arr[k].status == 1 for k in range(P))):
            self._check(rc, "plf_loop_closure_pose_batch")
        return [dict(self._lc_pose_result(arr[k].out, pp, lp), status=int(arr[k].status))
                for k, (pp, lp) in enumerate(outs)]

    def local_ba(self, prob, lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=1e-7,
                 min_error_change=1e-7, ref_quirks=1):
        """MapHandler::levMarquardtOptimizationLBA on the device (plf_local_ba; src/mapHandler.cpp:1332-1989).
        prob: dict as produced by synth.lba_problem (kf_pose, pt, ls, fixed_T, pt_obs_*, ls_obs_*)."""
        return self._bundle_adjust("plf_local_ba", prob, lambda_, lambda_k, max_iters, homog_th, min_error,
                                   min_error_change, ref_quirks)

    def global_ba(self, prob, lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=DBL_EPSILON,
                  min_error_change=DBL_EPSILON, ref_quirks=1):
        """MapHandler::levMarquardtOptimizationGBA on the device (plf_global_ba; src/mapHandler.cpp:2101-2699): every
        keyframe but keyframe 0 and every landmark.  prob: dict as produced by synth.gba_problem (plf_local_ba's layout;
        fixed_T holds keyframe 0).  The stop thresholds default to the reference's DBL_EPSILON literals (:2637, :2667)."""
        return self._bundle_adjust("plf_global_ba", prob, lambda_, lambda_k, max_iters, homog_th, min_error,
                                   min_error_change, ref_quirks)

    def local_ba_batch(self, problems, seq=None, lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=1e-7,
                       min_error_change=1e-7, ref_quirks=1):
        """Many local BAs in one device call (plf_local_ba_batch), with local_ba's options for all of them.  problems:
        dicts as local_ba takes; seq: per problem, -1 for the context's camera or a sequence whose camera
        (sequence_camera) to project with (None = all -1).  Returns one dict per problem in local_ba's shape plus
        `status` (0, or PLF_ERR_INVALID = -1 when the device refused that problem: a landmark whose first-pass block has a
        zero diagonal entry; its dict then holds its unchanged inputs and iters / err / lambda_ None).  Raises PlfError
        for the refusals before any work."""
        return self._bundle_adjust_batch("plf_local_ba_batch", problems, seq, lambda_, lambda_k, max_iters, homog_th,
                                         min_error, min_error_change, ref_quirks)

    def global_ba_batch(self, problems, seq=None, lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7,
                        min_error=DBL_EPSILON, min_error_change=DBL_EPSILON, ref_quirks=1):
        """Many global BAs in one device call (plf_global_ba_batch), with global_ba's options (and its DBL_EPSILON stop
        thresholds) for all of them.  problems: dicts as global_ba takes; seq and the result as local_ba_batch: one dict
        per problem in global_ba's shape plus `status` (0, or PLF_ERR_INVALID = -1 when the device refused that problem;
        its dict then holds its unchanged inputs and iters / err / lambda_ None).  Raises PlfError for the refusals before
        any work."""
        return self._bundle_adjust_batch("plf_global_ba_batch", problems, seq, lambda_, lambda_k, max_iters, homog_th,
                                         min_error, min_error_change, ref_quirks)

    def _bundle_adjust_batch(self, fn, problems, seq, *opts):
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        args = [self._lba_args(p) for p in problems]
        arr = (plf_lba_problem * max(P, 1))(*[a[0] for a in args])
        res = (plf_lba_result * max(P, 1))()
        st = np.full(max(P, 1), 1, np.int32)   # 1 is no plf_status: marks entries the call did not write
        rc = getattr(self.lib, fn)(self._ctx, C.byref(_lba_opts(*opts)), P, arr, _i32_or_null(seq_a), res,
                                   _ptr(st, C.c_int32))
        if rc != 0 and (P == 0 or np.any(st[:P] == 1)):
            self._check(rc, fn)
        out = []
        for k in range(P):
            d = self._lba_result(args[k][1], res[k] if st[k] == 0 else None)
            d["status"] = int(st[k])
            out.append(d)
        return out

    @staticmethod
    def _problem_sequences(P, seq):
        """seq of the batch calls (local_ba_batch, match_*_batch, batch_run): None, or an integer array of P entries
        (checked before any library call)."""
        if seq is None:
            return None
        a = np.asarray(seq)
        if a.shape != (P,) or a.dtype.kind not in "iu":
            raise PlfError(f"seq must be a 1-D integer array of {P} entries (got {a.dtype}{list(a.shape)})")
        s = np.ascontiguousarray(a, np.int32)
        if not np.array_equal(s, a):
            raise PlfError("seq: values do not fit int32")
        return s

    @staticmethod
    def _lba_args(prob):
        """(plf_lba_problem, arrays): copies of a problem dict's arrays, which the call updates in place, and the struct
        that points at them."""
        f64 = lambda a, c: np.ascontiguousarray(a, np.float64).reshape(-1, c).copy()
        i32 = lambda a: np.ascontiguousarray(a, np.int32).ravel().copy()
        kf, pt, ls = f64(prob["kf_pose"], 6), f64(prob["pt"], 3), f64(prob["ls"], 6)
        fT = np.ascontiguousarray(prob.get("fixed_T", np.zeros((0, 4, 4))), np.float64).reshape(-1, 16).copy()
        po_lm, po_kf, po_xy = i32(prob["pt_obs_lm"]), i32(prob["pt_obs_kf"]), f64(prob["pt_obs_xy"], 2)
        lo_lm, lo_kf, lo_le = i32(prob["ls_obs_lm"]), i32(prob["ls_obs_kf"]), f64(prob["ls_obs_le"], 3)
        pm, lm = np.zeros(max(len(pt), 1), np.uint8), np.zeros(max(len(ls), 1), np.uint8)
        ad = lambda a: a.ctypes.data if a.size else None
        p = plf_lba_problem(len(kf), len(pt), len(ls), len(fT), ad(kf), ad(pt), ad(ls), ad(fT), len(po_lm), ad(po_lm), ad(po_kf),
                            ad(po_xy), len(lo_lm), ad(lo_lm), ad(lo_kf), ad(lo_le), ad(pm), ad(lm))
        arrays = dict(kf_pose=kf, pt=pt, ls=ls, fT=fT, po=(po_lm, po_kf, po_xy), lo=(lo_lm, lo_kf, lo_le), pm=pm, lm=lm)
        return p, arrays

    @staticmethod
    def _lba_result(a, res):
        """local_ba's result dict from _lba_args' arrays and a plf_lba_result (None: no result, the inputs unchanged)."""
        n_pt, n_ls = len(a["pt"]), len(a["ls"])
        return dict(kf_pose=a["kf_pose"], pt=a["pt"], ls=a["ls"], pt_moved=a["pm"][:n_pt].astype(bool),
                    ls_moved=a["lm"][:n_ls].astype(bool), iters=None if res is None else res.iters,
                    err=None if res is None else res.err, lambda_=None if res is None else res.lambda_)

    def _bundle_adjust(self, fn, prob, *opts):
        p, a = self._lba_args(prob)
        res = plf_lba_result()
        self._check(getattr(self.lib, fn)(self._ctx, C.byref(_lba_opts(*opts)), C.byref(p), C.byref(res)), fn)
        return self._lba_result(a, res)

    def pose_graph(self, prob, max_iters=100, lambda_init=1e-10, trace=True):
        """The g2o optimisation of MapHandler::loopClosureOptimizationCovGraphG2O on the device (plf_pose_graph;
        src/mapHandler.cpp:4185-4410).  prob: dict T [n_v, 4, 4], fixed [n_v], from / to [n_e], Z [n_e, 4, 4], as
        synth.pose_graph_problem or oracle.pgo.cov_graph_lists give it.  Returns dict(T, iters, stop (PGO_STOP's names),
        trials, chi2_init, chi2, lambda_, scratch_bytes, trace: a PGO_TRACE_DTYPE array with one row per trial when
        `trace`)."""
        p, res, a = self._pgo_args(prob, max_iters, trace)
        o = plf_pgo_opts(int(max_iters), float(lambda_init))
        self._check(self.lib.plf_pose_graph(self._ctx, C.byref(o), C.byref(p), C.byref(res)), "plf_pose_graph")
        return self._pgo_result(a, res, trace)

    def pose_graph_batch(self, problems, max_iters=100, lambda_init=1e-10, trace=True):
        """Many pose graphs in one device call (plf_pose_graph_batch), with one max_iters / lambda_init for all of them.
        problems: dicts as pose_graph takes.  Returns one dict per problem in pose_graph's shape, each bit-identical to
        what pose_graph returns for that problem alone.  Raises PlfError for the refusals (nothing is computed then)."""
        problems = list(problems)
        P = len(problems)
        args = [self._pgo_args(p, max_iters, trace) for p in problems]
        arr = (plf_pgo_problem * max(P, 1))(*[p for p, _, _ in args])
        res = (plf_pgo_result * max(P, 1))(*[r for _, r, _ in args])
        o = plf_pgo_opts(int(max_iters), float(lambda_init))
        self._check(self.lib.plf_pose_graph_batch(self._ctx, C.byref(o), P, arr, res), "plf_pose_graph_batch")
        return [self._pgo_result(a, res[k], trace) for k, (_, _, a) in enumerate(args)]

    @staticmethod
    def _pgo_args(prob, max_iters, trace):
        """(plf_pgo_problem, plf_pgo_result, arrays): a copy of the problem's poses, which the call updates in place, its
        other arrays and a trace of 10 max_iters rows (none without `trace`), the problem struct that points at them and
        a result struct that points at the trace."""
        T = np.ascontiguousarray(prob["T"], np.float64).reshape(-1, 16).copy()
        fixed = np.ascontiguousarray(prob["fixed"], np.uint8).ravel()
        frm = np.ascontiguousarray(prob["from"], np.int32).ravel()
        to = np.ascontiguousarray(prob["to"], np.int32).ravel()
        Z = np.ascontiguousarray(prob["Z"], np.float64).reshape(-1, 16)
        ad = lambda a: a.ctypes.data if a.size else None
        p = plf_pgo_problem(len(T), len(frm), ad(T), ad(fixed), ad(frm), ad(to), ad(Z))
        tr = np.zeros(max(10 * int(max_iters), 1) if trace else 0, PGO_TRACE_DTYPE)
        res = plf_pgo_result(trace=ad(tr), trace_cap=len(tr))
        return p, res, dict(T=T, fixed=fixed, frm=frm, to=to, Z=Z, trace=tr)

    @staticmethod
    def _pgo_result(a, res, trace):
        out = dict(T=a["T"].reshape(-1, 4, 4), iters=res.iters, stop=PGO_STOP[res.stop], trials=res.trials,
                   chi2_init=res.chi2_init, chi2=res.chi2, lambda_=res.lambda_, scratch_bytes=res.scratch_bytes)
        if trace:
            out["trace"] = a["trace"][:res.n_trace].copy()
        return out

    def match_kf2kf(self, prev, curr, DT, fast_matching=True, max_kf_epip_p=1.0, max_kf_epip_l=1.0):
        """MapHandler::matchKF2KFPoints / matchKF2KFLines, matching part (plf_match_kf2kf).  prev / curr: get_frame dicts;
        DT: 4x4.  Returns dict(m_pt, n_pt, m_ls, n_ls): per previous-keyframe feature the current one or -1."""
        keep = []
        p, m_pt, m_ls = _kf2kf_problem(prev, curr, DT, keep)
        o = _kf_match_opts(fast_matching, max_kf_epip_p, max_kf_epip_l)
        n_pt, n_ls = C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_match_kf2kf(self._ctx, C.byref(o), p.prev, p.curr, p.DT, C.c_void_p(p.m_pt),
                                             C.c_void_p(p.m_ls), C.byref(n_pt), C.byref(n_ls)), "plf_match_kf2kf")
        return dict(m_pt=m_pt.copy(), n_pt=n_pt.value, m_ls=m_ls.copy(), n_ls=n_ls.value)

    def match_map2kf(self, local_map, Twf, kf, kf_pt_lm=None, kf_ls_lm=None, fast_matching=True, max_kf_epip_p=1.0,
                     max_kf_epip_l=1.0):
        """MapHandler::matchMap2KFPoints / matchMap2KFLines (plf_match_map2kf).  local_map: dict pt_X [n,3], pt_desc,
        optional pt_use, ls_X [n,6], ls_desc, optional ls_use; kf: get_frame dict; kf_*_lm: landmark index per keyframe
        feature (-1 = unmatched) or None.  Returns dict(lm_pt, n_pt, lm_ls, n_ls)."""
        keep = []
        p, lm_pt, lm_ls = _map2kf_problem(local_map, Twf, kf, kf_pt_lm, kf_ls_lm, keep, "match_map2kf")
        o = _kf_match_opts(fast_matching, max_kf_epip_p, max_kf_epip_l)
        n_pt, n_ls = C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_match_map2kf(self._ctx, C.byref(o), p.map, p.Twf, p.kf, C.c_void_p(p.kf_pt_lm),
                                              C.c_void_p(p.kf_ls_lm), C.c_void_p(p.lm_pt), C.c_void_p(p.lm_ls),
                                              C.byref(n_pt), C.byref(n_ls)), "plf_match_map2kf")
        return dict(lm_pt=lm_pt.copy(), n_pt=n_pt.value, lm_ls=lm_ls.copy(), n_ls=n_ls.value)

    def match_kf2kf_batch(self, problems, seq=None, fast_matching=True, max_kf_epip_p=1.0, max_kf_epip_l=1.0):
        """Many match_kf2kf in one device call (plf_match_kf2kf_batch), with one set of options.  problems: dicts
        prev, curr (get_frame dicts) and DT (4x4); seq: per problem, -1 for the context's camera or a sequence whose
        camera (sequence_camera) to project with (None = all -1).  Returns one match_kf2kf dict per problem."""
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        keep, outs = [], []
        arr = (plf_kf2kf_problem * max(P, 1))()
        for k, pr in enumerate(problems):
            arr[k], m_pt, m_ls = _kf2kf_problem(pr["prev"], pr["curr"], pr["DT"], keep)
            outs.append((m_pt, m_ls))
        o = _kf_match_opts(fast_matching, max_kf_epip_p, max_kf_epip_l)
        self._check(self.lib.plf_match_kf2kf_batch(self._ctx, C.byref(o), P, arr, _i32_or_null(seq_a)),
                    "plf_match_kf2kf_batch")
        return [dict(m_pt=m_pt.copy(), n_pt=arr[k].n_pt, m_ls=m_ls.copy(), n_ls=arr[k].n_ls) for k, (m_pt, m_ls) in enumerate(outs)]

    def match_map2kf_batch(self, problems, seq=None, fast_matching=True, max_kf_epip_p=1.0, max_kf_epip_l=1.0):
        """Many match_map2kf in one device call (plf_match_map2kf_batch), with one set of options.  problems: dicts
        local_map, Twf, kf and optionally kf_pt_lm / kf_ls_lm, as match_map2kf takes them; seq: as match_kf2kf_batch.
        Returns one match_map2kf dict per problem."""
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        keep, outs = [], []
        arr = (plf_map2kf_problem * max(P, 1))()
        for k, pr in enumerate(problems):
            arr[k], lm_pt, lm_ls = _map2kf_problem(pr["local_map"], pr["Twf"], pr["kf"], pr.get("kf_pt_lm"),
                                                   pr.get("kf_ls_lm"), keep, f"match_map2kf_batch: problem {k}")
            outs.append((lm_pt, lm_ls))
        o = _kf_match_opts(fast_matching, max_kf_epip_p, max_kf_epip_l)
        self._check(self.lib.plf_match_map2kf_batch(self._ctx, C.byref(o), P, arr, _i32_or_null(seq_a)),
                    "plf_match_map2kf_batch")
        return [dict(lm_pt=lm_pt.copy(), n_pt=arr[k].n_pt, lm_ls=lm_ls.copy(), n_ls=arr[k].n_ls)
                for k, (lm_pt, lm_ls) in enumerate(outs)]

    # -- place recognition (DBoW2) -----------------------------------------------------------------
    def bow_set_vocabulary(self, kind, voc):
        """plf_bow_set_vocabulary: kind 0 (points) / 1 (lines); voc: a YAML path or a dict as read_vocab_yml returns.
        Empties that kind's keyframe database."""
        if not isinstance(voc, dict):
            voc = read_vocab_yml(voc)
        keep = []
        v = _vocab_struct(voc, keep)
        self._check(self.lib.plf_bow_set_vocabulary(self._ctx, int(kind), C.byref(v)), "plf_bow_set_vocabulary")

    def bow_insert(self, kf_idx, pdesc=None, ldesc=None, rows=(True, True)):
        """plf_bow_insert: stores the BoW vectors of the keyframe's descriptors under kf_idx and returns (score_p, score_l),
        float64 [kf_idx + 1] each (NaN: absent keyframe), None for a row not requested (rows) or of a disabled kind."""
        keep = []
        v = _frame_view({key: d for key, d in (("pdesc", pdesc), ("ldesc", ldesc)) if d is not None}, keep)
        out = self._score_rows(kf_idx, rows)
        ptr = [C.c_void_p(o.ctypes.data) if o is not None else C.c_void_p() for o in out]
        self._check(self.lib.plf_bow_insert(self._ctx, int(kf_idx), C.byref(v), ptr[0], ptr[1]), "plf_bow_insert")
        return out[0], out[1]

    def _score_rows(self, kf_idx, rows):
        """The (score_p, score_l) rows a keyframe insert fills: NaN float64 [kf_idx + 1] for each kind requested in
        `rows` and enabled in the context's parameters, else None."""
        enabled = (self.params.has_points, self.params.has_lines)
        return [np.full(kf_idx + 1, np.nan) if (rows[c] and enabled[c] and kf_idx >= 0) else None for c in range(2)]

    def bow_insert_batch(self, problems, seq=None, rows=(True, True)):
        """Many bow_insert in one device call (plf_bow_insert_batch).  problems: dicts kf_idx, pdesc, ldesc (either
        descriptor array may be missing: no features of that kind); seq: per problem the database, -1 for the context's
        (the one bow_insert uses) or a sequence in [0, max_sequences) (None = all -1).  Returns one (score_p, score_l) per
        problem, as bow_insert does.  Raises PlfError for the refusals before any work."""
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        keep, outs = [], []
        arr = (plf_bow_problem * max(P, 1))()
        for k, pr in enumerate(problems):
            v = _frame_view({key: pr[key] for key in ("pdesc", "ldesc") if pr.get(key) is not None}, keep)
            keep.append(v)
            kf = int(pr["kf_idx"])
            out = self._score_rows(kf, rows)
            outs.append(tuple(out))
            arr[k] = plf_bow_problem(kf, C.pointer(v), *[o.ctypes.data if o is not None else None for o in out])
        self._check(self.lib.plf_bow_insert_batch(self._ctx, P, arr, _i32_or_null(seq_a)), "plf_bow_insert_batch")
        return outs

    def _lc_problem(self, pr, rows, conf, keep, who):
        """(plf_lc_detect_problem, (score_p, score_l), conf) over one bow_detect_batch problem dict."""
        n = {d: 0 if pr.get(d) is None else len(pr[d]) for d in ("pdesc", "ldesc")}
        for key, desc in (("pt_pl", "pdesc"), ("ls_spl", "ldesc"), ("ls_epl", "ldesc")):
            if pr.get(key) is not None and np.asarray(pr[key]).size != 2 * n[desc]:
                raise PlfError(f"{who}: {key} has {np.asarray(pr[key]).size} values for {n[desc]} rows of {desc} "
                               f"(2 per row)")
        v = _frame_view({key: pr[key] for key in ("pdesc", "ldesc", "pt_pl", "ls_spl", "ls_epl")
                         if pr.get(key) is not None}, keep)
        keep.append(v)
        kf = int(pr["kf_idx"])
        out = self._score_rows(kf, rows)
        cf = np.full(max(kf + 1, 1), np.nan, np.float32) if conf else None
        cov = pr.get("covis")
        if cov is not None:
            cov = np.ascontiguousarray(cov, np.uint32)
            if len(cov) != max(kf, 0):
                raise PlfError(f"{who}: covis has {len(cov)} entries for kf_idx {kf}")
        keep += [out, cf, cov]
        ad = lambda a: None if a is None or not a.size else a.ctypes.data
        return (plf_lc_detect_problem(kf, C.pointer(v), ad(cov), ad(cf), ad(out[0]), ad(out[1])), out,
                None if cf is None else cf[:kf + 1])

    @staticmethod
    def _lc_result(st, out, cf):
        r = {f: getattr(st.result, f) for f in LC_RESULT_FIELDS}
        r.update(conf=cf, score_p=out[0], score_l=out[1])
        return r

    def bow_detect_batch(self, problems, opts=None, seq=None, rows=(False, False), conf=True):
        """Many keyframe inserts with loop-candidate detection in one device call (plf_bow_detect_batch).  problems: dicts
        kf_idx, pdesc, ldesc, pt_pl [n_pt][2], ls_spl / ls_epl [n_ls][2] (the coordinates are read when both kinds are
        enabled) and optionally covis [kf_idx] (full_graph[kf_idx][i]; missing = all zero); opts: a dict over
        LC_DETECT_DEFAULTS; seq: as bow_insert_batch.  Returns one dict per problem: the result fields (candidate, best,
        n_listed, n_closest, min_score), conf float32 [kf_idx + 1] (None unless conf) and score_p / score_l as
        bow_insert_batch returns them for `rows`."""
        problems = list(problems)
        P = len(problems)
        seq_a = self._problem_sequences(P, seq)
        keep, outs = [], []
        arr = (plf_lc_detect_problem * max(P, 1))()
        for k, pr in enumerate(problems):
            arr[k], out, cf = self._lc_problem(pr, rows, conf, keep, f"bow_detect_batch: problem {k}")
            outs.append((out, cf))
        o = _lc_opts(opts)
        self._check(self.lib.plf_bow_detect_batch(self._ctx, C.byref(o), P, arr, _i32_or_null(seq_a)),
                    "plf_bow_detect_batch")
        return [self._lc_result(arr[k], out, cf) for k, (out, cf) in enumerate(outs)]

    def bow_detect(self, problem, opts=None, rows=(False, False), conf=True):
        """plf_bow_detect: one bow_detect_batch problem on the context's database (the one bow_insert uses)."""
        keep = []
        pr, out, cf = self._lc_problem(problem, rows, conf, keep, "bow_detect")
        o = _lc_opts(opts)
        self._check(self.lib.plf_bow_detect(self._ctx, C.byref(o), C.byref(pr)), "plf_bow_detect")
        return self._lc_result(pr, out, cf)

    def debug_loop_candidates(self, columns, opts=None):
        """plf_debug_loop_candidates: lookForLoopCandidates on the device over caller columns.  columns: dicts kf_idx,
        conf float32 [kf_idx + 1], live bool [kf_idx + 1] and optionally covis uint32 [kf_idx].  Returns one result dict
        per column."""
        columns = list(columns)
        n = len(columns)
        keep = []
        kf = np.array([int(c["kf_idx"]) for c in columns] or [0], np.int32)
        pc, pl, pv = (C.c_void_p * max(n, 1))(), (C.c_void_p * max(n, 1))(), (C.c_void_p * max(n, 1))()
        for k, c in enumerate(columns):
            m = int(c["kf_idx"]) + 1
            cf = np.ascontiguousarray(c["conf"], np.float32)
            lv = np.ascontiguousarray(c["live"], np.uint8)
            if len(cf) != m or len(lv) != m:
                raise PlfError(f"debug_loop_candidates: column {k}: conf / live need kf_idx + 1 = {m} entries")
            keep += [cf, lv]
            pc[k], pl[k] = cf.ctypes.data, lv.ctypes.data
            if c.get("covis") is not None:
                cv = np.ascontiguousarray(c["covis"], np.uint32)
                if len(cv) != m - 1:
                    raise PlfError(f"debug_loop_candidates: column {k}: covis needs kf_idx = {m - 1} entries")
                keep.append(cv)
                pv[k] = cv.ctypes.data if cv.size else None
        out = (plf_lc_detect_result * max(n, 1))()
        o = _lc_opts(opts)
        self._check(self.lib.plf_debug_loop_candidates(self._ctx, C.byref(o), n, _ptr(kf, C.c_int), pc, pl, pv, out),
                    "plf_debug_loop_candidates")
        return [{f: getattr(out[k], f) for f in LC_RESULT_FIELDS} for k in range(n)]

    def bow_erase(self, kf_idx, seq=None):
        """plf_bow_erase, or plf_bow_erase_seq on sequence seq's database (-1: the context's)."""
        if seq is None:
            self._check(self.lib.plf_bow_erase(self._ctx, int(kf_idx)), "plf_bow_erase")
        else:
            self._check(self.lib.plf_bow_erase_seq(self._ctx, int(seq), int(kf_idx)), "plf_bow_erase_seq")

    def bow_vector(self, kf_idx, kind, seq=None):
        """plf_bow_get: the stored BowVector of keyframe kf_idx, kind 0 / 1, as (words uint32, values float64); with seq,
        plf_bow_get_seq on that sequence's database (-1: the context's)."""
        if seq is None:
            fn, get = "plf_bow_get", lambda *a: self.lib.plf_bow_get(self._ctx, *a)
        else:
            fn, get = "plf_bow_get_seq", lambda *a: self.lib.plf_bow_get_seq(self._ctx, int(seq), *a)
        n = C.c_int(0)
        self._check(get(int(kf_idx), int(kind), 0, None, None, C.byref(n)), fn)
        w, x = np.zeros(max(n.value, 1), np.uint32), np.zeros(max(n.value, 1), np.float64)
        self._check(get(int(kf_idx), int(kind), n.value, C.c_void_p(w.ctypes.data), C.c_void_p(x.ctypes.data),
                        C.byref(n)), fn)
        return w[:n.value].copy(), x[:n.value].copy()

    def bow_clear_sequence(self, s):
        """plf_bow_clear_sequence: empties sequence s's bag-of-words database and frees its device memory."""
        self._check(self.lib.plf_bow_clear_sequence(self._ctx, int(s)), "plf_bow_clear_sequence")

    def expmap_se3(self, x):
        x = np.ascontiguousarray(x, np.float64).reshape(6)
        T = np.zeros(16)
        self._check(self.lib.plf_se3(self._ctx, 0, x.ctypes.data_as(C.POINTER(C.c_double)),
                                     T.ctypes.data_as(C.POINTER(C.c_double))), "plf_se3")
        return T.reshape(4, 4)

    def logmap_se3(self, T):
        T = np.ascontiguousarray(T, np.float64).reshape(16)
        x = np.zeros(6)
        self._check(self.lib.plf_se3(self._ctx, 1, T.ctypes.data_as(C.POINTER(C.c_double)),
                                     x.ctypes.data_as(C.POINTER(C.c_double))), "plf_se3")
        return x

    # -- point features --------------------------------------------------------------------------
    def orb(self, img, cap=8192, mask=None):
        """cv::ORB::detectAndCompute with the ctx parameters: returns (keypoints[KEYPOINT_DTYPE], desc u8[n,32])
        in canonical (octave, y, x) order.  mask: u8 [H, W] of the image's shape (non-zero = allowed), as
        detectAndCompute's mask argument (plf_orb_masked); None detects everywhere (plf_orb)."""
        img = _u8(img)
        h, w = img.shape
        kps = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        if mask is None:
            st = self.lib.plf_orb(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                  kps.ctypes.data_as(C.c_void_p), _ptr(desc, C.c_uint8), cap, C.byref(n))
            self._check(st, "plf_orb")
        else:
            m = self._mask(mask, h, w, "orb")
            st = self.lib.plf_orb_masked(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0], _ptr(m, C.c_uint8),
                                         m.strides[0], kps.ctypes.data_as(C.c_void_p), _ptr(desc, C.c_uint8), cap,
                                         C.byref(n))
            self._check(st, "plf_orb_masked")
        return kps[:n.value].copy(), desc[:n.value].copy()

    # -- line features ---------------------------------------------------------------------------
    def lsd(self, img, cap=16384):
        """cv::LineSegmentDetector::detect with the ctx LSD parameters: float32[n,4] in OpenCV's order."""
        img = _u8(img)
        h, w = img.shape
        segs = np.zeros((cap, 4), np.float32)
        n = C.c_int(0)
        st = self.lib.plf_lsd(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0], _ptr(segs, C.c_float), cap,
                              C.byref(n))
        self._check(st, "plf_lsd")
        return segs[:n.value].copy()

    def detect_lines(self, img, cap=4096, mask=None):
        """stvo-pl detectLineFeatures: (keylines[KEYLINE_DTYPE], LBD desc u8[n,32]).  mask: u8 [H, W] of the image's
        shape, as LSDDetectorC::detect's mask argument (plf_detect_lines_masked): a line is dropped when both its end
        points fall on 0; None detects everywhere (plf_detect_lines)."""
        img = _u8(img)
        h, w = img.shape
        kl = np.zeros(cap, KEYLINE_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        if mask is None:
            st = self.lib.plf_detect_lines(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                           kl.ctypes.data_as(C.c_void_p), _ptr(desc, C.c_uint8), cap, C.byref(n))
            self._check(st, "plf_detect_lines")
        else:
            m = self._mask(mask, h, w, "detect_lines")
            st = self.lib.plf_detect_lines_masked(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                                  _ptr(m, C.c_uint8), m.strides[0], kl.ctypes.data_as(C.c_void_p),
                                                  _ptr(desc, C.c_uint8), cap, C.byref(n))
            self._check(st, "plf_detect_lines_masked")
        return kl[:n.value].copy(), desc[:n.value].copy()

    def debug_sincosf(self, x):
        x = np.ascontiguousarray(x, np.float32)
        s = np.empty_like(x); c = np.empty_like(x)
        st = self.lib.plf_debug_sincosf(self._ctx, _ptr(x, C.c_float), _ptr(s, C.c_float), _ptr(c, C.c_float), len(x))
        self._check(st, "plf_debug_sincosf")
        return s, c

    def _debug_lsd_pre(self, n, w, h, pitch, img_stride, bufs=(None,) * 5):
        """plf_debug_lsd_pre on bufs = (images, pix, seedlist, segcnt, maxmag2); all None: the launch only."""
        f = self.lib.plf_debug_lsd_pre
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p,
                      C.c_void_p, C.c_void_p, C.c_void_p]
        sizes = np.zeros(6, np.int32)
        ptrs = [None if a is None else a.ctypes.data for a in bufs]
        self._check(f(self._ctx, ptrs[0], n, w, h, pitch, img_stride, sizes.ctypes.data, *ptrs[1:]), "plf_debug_lsd_pre")
        return dict(zip(("ws", "hs", "nxb", "ks", "th", "np"), (int(v) for v in sizes)))

    def debug_lsd_pre_geometry(self, w, h):
        """The launch LSD's pre-grow kernel takes for w x h images at this context's parameters: dict(ws, hs, nxb, ks, th,
        np) - the scaled size, the 512-column segments per row, the pre-blur's taps (1: none), the scaled rows per CTA
        and the column pieces per segment."""
        pitch = (w + 15) // 16 * 16
        return self._debug_lsd_pre(1, w, h, pitch, pitch * h)

    def debug_lsd_pre(self, imgs, pitch=None, img_stride=None, pad_byte=0xA5):
        """LSD's gradient stage on the (n, h, w) uint8 images, by the pre-blur + resample + gradient kernel.  The images
        are laid out with row pitch `pitch` and image stride `img_stride` bytes (multiples of 16; default: the
        pipeline's) and the padding filled with pad_byte.  Returns dict(pix=(n, hs*ws) uint64 records,
        seedlist=(n, hs*ws) uint32, segcnt=(n, hs, nxb) int32, maxmag2=(n,) int32) and the launch
        (debug_lsd_pre_geometry's keys)."""
        imgs = np.ascontiguousarray(imgs, np.uint8)
        n, h, w = imgs.shape
        pitch = pitch or (w + 15) // 16 * 16
        img_stride = img_stride or pitch * h
        geo = self.debug_lsd_pre_geometry(w, h)
        ws, hs, nxb = geo["ws"], geo["hs"], geo["nxb"]
        buf = np.full(n * img_stride, pad_byte, np.uint8)
        for i in range(n):
            v = buf[i * img_stride:i * img_stride + pitch * h].reshape(h, pitch)
            v[:, :w] = imgs[i]
        pix = np.empty((n, hs * ws), np.uint64)
        seed = np.empty((n, hs * ws), np.uint32)
        seg = np.empty((n, hs, nxb), np.int32)
        mm = np.empty(n, np.int32)
        self._debug_lsd_pre(n, w, h, pitch, img_stride, (buf, pix, seed, seg, mm))
        return dict(geo, pix=pix, seedlist=seed, segcnt=seg, maxmag2=mm)

    def debug_ldlt(self, S, g, path=0, overwrite_s=False):
        """LDL^T without pivoting of the symmetric S (6 n6 x 6 n6, lower triangle read) and the solution of S x = g, by
        the tiled factorisation of global_ba / pose_graph beyond 64 keyframes, on one system (path 0), or the one-CTA
        one of local_ba, without the zeroing that follows it there (path 1).  Returns
        (LD, x, nz): LD holds L strictly below its diagonal and D on it (upper triangle unspecified); nz (path 0, else
        None) is the n_t x n_t zero flag of each L tile (i > k), n_t = ceil(n / 64).  overwrite_s: factor S's own buffer
        (a C-contiguous float64 array) instead of a copy.  plf_debug_ldlt."""
        g, x, nz = self._ldlt_buffers(S, g, "debug_ldlt")
        if overwrite_s:
            if S.dtype != np.float64 or not S.flags.c_contiguous or not S.flags.writeable:
                raise PlfError("debug_ldlt: overwrite_s needs a writeable C-contiguous float64 S")
            LD = S
        else:
            LD = np.array(S, np.float64, order="C")
        nz = nz if path == 0 else None
        st = self.lib.plf_debug_ldlt(self._ctx, int(path), len(x) // 6, _ptr(LD, C.c_double), _ptr(g, C.c_double),
                                     _ptr(x, C.c_double), None if nz is None else _ptr(nz, C.c_uint8))
        self._check(st, "plf_debug_ldlt")
        return LD, x, nz

    @staticmethod
    def _ldlt_buffers(S, g, who):
        """(g, x, nz) of one debug_ldlt system, once S is checked 6 n6 square and g 6 n6 long: g as float64, the
        solution and the tile zero flags to fill."""
        n = S.shape[0]
        if S.shape != (n, n) or n % 6 or len(g) != n:
            raise PlfError(f"{who}: S {S.shape} and g {len(g)} must be 6 n6 square and 6 n6 long")
        nt = (n + 63) // 64
        return np.ascontiguousarray(g, np.float64), np.empty(n, np.float64), np.zeros((nt, nt), np.uint8)

    def debug_ldlt_batch(self, mats):
        """debug_ldlt(S, g, path=0) on every (S, g) of `mats`, factored in one launch chain by the batched tiled LDL^T
        of global_ba_batch.  Returns one (LD, x, nz) per matrix, as debug_ldlt.  plf_debug_ldlt_batch."""
        mats = list(mats)
        n6, LDs, gs, xs, nzs = [], [], [], [], []
        for S, g in mats:
            g, x, nz = self._ldlt_buffers(S, g, "debug_ldlt_batch")
            n6.append(len(x) // 6)
            LDs.append(np.array(S, np.float64, order="C"))
            gs.append(g); xs.append(x); nzs.append(nz)
        k = max(len(mats), 1)
        ptrs = lambda arrs: (C.c_void_p * k)(*[a.ctypes.data for a in arrs])
        n6a = np.array(n6 or [0], np.int32)
        st = self.lib.plf_debug_ldlt_batch(self._ctx, len(mats), _ptr(n6a, C.c_int32), ptrs(LDs), ptrs(gs), ptrs(xs),
                                           ptrs(nzs))
        self._check(st, "plf_debug_ldlt_batch")
        return list(zip(LDs, xs, nzs))

    def debug_timeline(self):
        """Device-clock start/end (ms) of the E, G, M phases of the two most recent batches: array [2, 3, 2]."""
        out = np.zeros(12, np.float32)
        self._check(self.lib.plf_debug_timeline(self._ctx, _ptr(out, C.c_float)), "plf_debug_timeline")
        return out.reshape(2, 3, 2)

    # -- batched front-end -----------------------------------------------------------------------
    def reset_sequence(self):
        self._check(self.lib.plf_reset_sequence(self._ctx), "plf_reset_sequence")

    def set_image_sizes(self, sizes=()):
        """The image sizes the batched pipeline accepts besides the camera's: (width, height) pairs, at most 8; an
        empty list restores the single-size context.  A batch is of one size; a sequence takes its size from its camera
        (set_sequence_camera).  Valid only before the first batch call.  plf_set_image_sizes."""
        wh = np.ascontiguousarray(np.asarray(list(sizes), np.int32).reshape(-1, 2))
        self._check(self.lib.plf_set_image_sizes(self._ctx, len(wh), _ptr(wh, C.c_int32) if len(wh) else None),
                    "plf_set_image_sizes")
        own = (self.camera.width, self.camera.height)
        self.image_sizes = list(dict.fromkeys(tuple(int(v) for v in x) for x in wh if tuple(x) != own))

    def _sizes_hw(self):
        """Every accepted image size as (height, width), the camera's first."""
        return [(self.camera.height, self.camera.width)] + [(h, w) for w, h in self.image_sizes]

    def set_sequence_camera(self, s, camera=None):
        """Gives sequence s its own calibration: a camera dict as Frontend(camera=...) takes, or a plf_camera, of the
        context's width and height or one of image_sizes.  None returns s to the context's camera.  Either restarts s: its next pair in a run is
        a first frame.  Batches already run keep their cameras.  plf_set_sequence_camera."""
        cam = None if camera is None else (camera if isinstance(camera, plf_camera) else plf_camera(**camera))
        self._check(self.lib.plf_set_sequence_camera(self._ctx, int(s), None if cam is None else C.byref(cam)),
                    "plf_set_sequence_camera")

    def set_sequence_params(self, s, params=None, **fields):
        """Gives sequence s its own front-end settings: params (a plf_params, default the context's) with the named fields
        replaced, e.g. set_sequence_params(1, lsd_nfeatures=300, matching_strategy=3).  No params and no fields returns s
        to the context's settings.  sequence_param_fields() tells which fields may differ.  Either restarts s: its next
        pair in a run is a first frame.  Batches already run keep their settings.  plf_set_sequence_params."""
        if params is None and not fields:
            self._check(self.lib.plf_set_sequence_params(self._ctx, int(s), None), "plf_set_sequence_params")
            return
        p = plf_params()
        C.pointer(p)[0] = params if params is not None else self.params
        names = {name for name, _ in plf_params._fields_}
        for k, v in fields.items():
            if k not in names:
                raise PlfError(f"unknown parameter {k}")
            setattr(p, k, v)
        self._check(self.lib.plf_set_sequence_params(self._ctx, int(s), C.byref(p)), "plf_set_sequence_params")

    def get_sequence_params(self, s):
        """The settings the next batch uses for sequence s, its own or the context's, as a plf_params.
        plf_get_sequence_params."""
        out = plf_params()
        self._check(self.lib.plf_get_sequence_params(self._ctx, int(s), C.byref(out)), "plf_get_sequence_params")
        return out

    def sequence_camera(self, s):
        """The calibration the next batch uses for sequence s, as a camera dict.  plf_get_sequence_camera."""
        out = plf_camera()
        self._check(self.lib.plf_get_sequence_camera(self._ctx, int(s), C.byref(out)), "plf_get_sequence_camera")
        return {name: getattr(out, name) for name, _ in plf_camera._fields_}

    def set_sequence_rectification(self, s, left=None, right=None):
        """Rectifies sequence s's raw pairs on the device before extraction, byte for byte cv::remap(img, map1, map2,
        INTER_LINEAR) with a constant 0 border.  left / right: (map1, map2) of that image, as cv2.initUndistortRectifyMap
        (..., cv2.CV_16SC2, ...) returns them: map1 int16 [H, W, 2], map2 uint16 [H, W], for the sequence camera's H x W.  Both None
        clears the rectification.  Either restarts s; batches already run keep their maps.  The camera of the rectified
        images is set with set_sequence_camera.  plf_set_sequence_rectification."""
        if left is None and right is None:
            self._check(self.lib.plf_set_sequence_rectification(self._ctx, int(s), None, None, None, None),
                        "plf_set_sequence_rectification")
            return
        if left is None or right is None:
            raise PlfError("set_sequence_rectification: give the maps of both images, or neither to clear")
        cam = self.sequence_camera(s)
        H, W = cam["height"], cam["width"]
        maps = []
        for side, pair in (("left", left), ("right", right)):
            m1, m2 = pair
            for name, a, dt, shape in (("map1", m1, np.int16, (H, W, 2)), ("map2", m2, np.uint16, (H, W))):
                a = np.asarray(a)
                if a.dtype != dt or a.shape != shape:
                    raise PlfError(f"set_sequence_rectification: {side} {name} must be {np.dtype(dt)}{list(shape)} "
                                   f"(got {a.dtype}{list(a.shape)})")
                maps.append(np.ascontiguousarray(a))
        m1l, m2l, m1r, m2r = maps
        self._check(self.lib.plf_set_sequence_rectification(self._ctx, int(s), _ptr(m1l, C.c_int16), _ptr(m2l, C.c_uint16),
                                                            _ptr(m1r, C.c_int16), _ptr(m2r, C.c_uint16)),
                    "plf_set_sequence_rectification")

    @staticmethod
    def _mask(mask, h, w, who, B=None):
        """mask as a uint8 [h, w] array (B given: [B, h, w], mask k h rows after mask k-1) with unit column stride (rows
        may be strided)."""
        m = np.asarray(mask)
        shape = (h, w) if B is None else (B, h, w)
        if m.dtype != np.uint8 or m.shape != shape:
            raise PlfError(f"{who}: mask must be uint8{list(shape)} (got {m.dtype}{list(m.shape)})")
        rows = m.strides[-2]
        ok = m.strides[-1] == 1 and rows >= w and (B is None or m.strides[0] == rows * h)
        return m if ok else np.ascontiguousarray(m)

    def set_sequence_mask(self, s, left=None, right=None):
        """Restricts sequence s's ORB and line detection in the batched pipeline to masks: uint8 [H, W] of the sequence
        camera's shape, in the geometry the detectors see (after rectification, one channel), non-zero = allowed.  None
        for an image leaves it unmasked; both None clears them.  Batches already run keep their masks; s is not
        restarted.  plf_set_sequence_mask."""
        cam = self.sequence_camera(s)
        H, W = cam["height"], cam["width"]
        ml = None if left is None else np.ascontiguousarray(self._mask(left, H, W, "set_sequence_mask"))
        mr = None if right is None else np.ascontiguousarray(self._mask(right, H, W, "set_sequence_mask"))
        self._check(self.lib.plf_set_sequence_mask(self._ctx, int(s), None if ml is None else _ptr(ml, C.c_uint8),
                                                   None if mr is None else _ptr(mr, C.c_uint8), W),
                    "plf_set_sequence_mask")

    def batch_upload_masks(self, left=None, right=None):
        """Restricts detection on the pairs of the most recent upload to masks of their own: uint8 [B, H, W] host arrays
        of that upload's size (device_layout), dense or row-strided, in the geometry the detectors see (after
        rectification, one channel), non-zero = allowed.  None leaves a side to its sequences' masks; with a sequence mask
        an image is restricted to the AND of the two.  The run that consumes the upload uses them, and only it.
        plf_batch_upload_masks."""
        if left is None and right is None:
            raise PlfError("batch_upload_masks: give the masks of at least one side")
        W, H, _ = self.device_layout
        B = (left if left is not None else right).shape[0]
        ml = None if left is None else self._mask(left, H, W, "batch_upload_masks", B)
        mr = None if right is None else self._mask(right, H, W, "batch_upload_masks", B)
        strides = {m.strides[1] for m in (ml, mr) if m is not None}
        if len(strides) > 1:   # one stride for both sides
            ml, mr = (None if m is None else np.ascontiguousarray(m) for m in (ml, mr))
        stride = (ml if ml is not None else mr).strides[1]
        self._check(self.lib.plf_batch_upload_masks(self._ctx, int(B), None if ml is None else _ptr(ml, C.c_uint8),
                                                    None if mr is None else _ptr(mr, C.c_uint8), int(stride)),
                    "plf_batch_upload_masks")

    def batch_upload_masks_raw(self, B, left_ptr, right_ptr, stride=None):
        """batch_upload_masks from raw addresses (0 / None: that side has no pair masks): B masks per side of H rows of
        `stride` bytes (None: W), mask k at offset k * stride * H.  Host memory, pageable or pinned, or device memory of
        the context's device: a torch CUDA uint8 tensor's data_ptr(), its producer's stream synchronised first.  Keep
        them unchanged until that batch's download.  plf_batch_upload_masks."""
        W, _, _ = self.device_layout
        stride = W if stride is None else int(stride)
        self._check(self.lib.plf_batch_upload_masks(self._ctx, int(B), C.c_void_p(left_ptr or None), C.c_void_p(right_ptr or None),
                                                    stride), "plf_batch_upload_masks")

    def sequence_mask_set(self, s):
        """(left, right): whether sequence s has a mask on each image.  plf_get_sequence_mask_set."""
        left, right = C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_get_sequence_mask_set(self._ctx, int(s), C.byref(left), C.byref(right)),
                    "plf_get_sequence_mask_set")
        return bool(left.value), bool(right.value)

    def set_adaptive_fast(self, cfg=None):
        """stvo-pl's adaptative_fast for the batched pipeline: a dict of min_th, max_th, inc_th, feat_th and err_th (the
        config keys fast_*_th; missing keys take ADAPTIVE_FAST_DEFAULTS), or None to turn it off.  With it on, a batch
        holds at most one pair of each sequence.  Every sequence's threshold starts again at orb_fast_th.
        plf_set_adaptive_fast."""
        a = None
        if cfg is not None:
            unknown = set(cfg) - set(ADAPTIVE_FAST_DEFAULTS)
            if unknown:
                raise PlfError(f"unknown adaptive_fast keys {sorted(unknown)}")
            a = plf_adaptive_fast(**dict(ADAPTIVE_FAST_DEFAULTS, **cfg))
        self._check(self.lib.plf_set_adaptive_fast(self._ctx, None if a is None else C.byref(a)), "plf_set_adaptive_fast")

    def sequence_fast_th(self, s):
        """The FAST threshold the next pair of sequence s will be detected with.  plf_get_sequence_fast_th."""
        th = C.c_int(0)
        self._check(self.lib.plf_get_sequence_fast_th(self._ctx, int(s), C.byref(th)), "plf_get_sequence_fast_th")
        return th.value

    def set_motion_model(self, on=True):
        """stvo-pl's use_motion_model for the batched pipeline: each sequence's next pair starts from the prediction its
        last pair gave (its windowed frame-to-frame matching projects through it, and the pose solver is seeded with it).
        With it on, a batch holds at most one pair of each sequence.  Turning it on sets every prediction back to the
        identity.  plf_set_motion_model."""
        self._check(self.lib.plf_set_motion_model(self._ctx, 1 if on else 0), "plf_set_motion_model")

    def sequence_motion(self, s):
        """(T, valid): the prediction (4x4 float64) the next pair of sequence s will start from, and whether it came from
        a good solution (the identity and False otherwise).  plf_get_sequence_motion."""
        T = np.zeros(16, np.float64)
        valid = C.c_int(0)
        self._check(self.lib.plf_get_sequence_motion(self._ctx, int(s), _ptr(T, C.c_double), C.byref(valid)),
                    "plf_get_sequence_motion")
        return T.reshape(4, 4), bool(valid.value)

    def debug_motion_prior(self, DT, DT_cov, err, status):
        """plf_debug_motion_prior: the device's prediction rule on n results (DT [n,4,4], DT_cov [n,6,6], err [n],
        status [n]); returns (T [n,4,4], valid [n] bool)."""
        DT = np.ascontiguousarray(DT, np.float64).reshape(-1, 16)
        n = len(DT)
        cov = np.ascontiguousarray(DT_cov, np.float64).reshape(n, 36)
        err = np.ascontiguousarray(err, np.float64).reshape(n)
        status = np.ascontiguousarray(status, np.int32).reshape(n)
        T = np.zeros((n, 16), np.float64)
        valid = np.zeros(n, np.int32)
        self._check(self.lib.plf_debug_motion_prior(self._ctx, n, _ptr(DT, C.c_double), _ptr(cov, C.c_double),
                                                    _ptr(err, C.c_double), _ptr(status, C.c_int32), _ptr(T, C.c_double),
                                                    _ptr(valid, C.c_int32)), "plf_debug_motion_prior")
        return T.reshape(n, 4, 4), valid.astype(bool)

    @staticmethod
    def _result_dicts(res, B):
        out = []
        for k in range(B):
            r = res[k]
            d = {f: getattr(r, f) for f in RESULT_FIELDS}
            d["DT"] = np.array(r.DT).reshape(4, 4)
            d["DT_cov"] = np.array(r.DT_cov).reshape(6, 6)
            d["err"] = r.err
            out.append(d)
        return out

    def _stack(self, left, right):
        """(left, right, channels): grey uint8 [B,H,W] (or [H,W]) with channels 1, or colour uint8 [B,H,W,C] (or
        [H,W,C]), C = 3 (BGR) or 4 (BGRA), with channels C.  H x W is the camera's size or one of image_sizes; any
        other shape is refused here, before the library is called."""
        left = np.ascontiguousarray(left, np.uint8); right = np.ascontiguousarray(right, np.uint8)
        sizes = self._sizes_hw()
        if left.ndim == 3 and left.shape[:2] in sizes and left.shape[2] in (3, 4) and left.shape[1:] not in sizes:
            left, right = left[None], right[None]   # one colour pair
        if left.ndim == 4:
            if not (left.shape == right.shape and left.shape[1:3] in sizes and left.shape[3] in (3, 4)):
                hw = sizes[0] if len(sizes) == 1 else ("H", "W")
                raise PlfError(f"colour images must be uint8 [B, {hw[0]}, {hw[1]}, 3 | 4] (BGR or BGRA), left and right "
                               f"alike{self._sizes_text()} (got {list(left.shape)} and {list(right.shape)})")
            return left, right, left.shape[3]
        if left.ndim == 2:
            left, right = left[None], right[None]
        if not (left.ndim == 3 and left.shape == right.shape and left.shape[1:] in sizes):
            raise PlfError(f"grey images must be uint8 [B, H, W], left and right alike{self._sizes_text()} "
                           f"(got {list(left.shape)} and {list(right.shape)})")
        return left, right, 1

    def _sizes_text(self):
        return ", H x W one of " + ", ".join(f"{h} x {w}" for h, w in self._sizes_hw())

    def process_batch(self, left, right, seq=None, restart=None, masks=None):
        """B x (insertStereoPair + optimizePose): left/right uint8 [B,H,W] grey or [B,H,W,3|4] BGR / BGRA host arrays,
        H x W the camera's size or one of image_sizes -> list of result dicts.  seq / restart: as batch_run.  masks:
        (left, right) pair masks of the batch, as batch_upload_masks takes them."""
        left, right, ch = self._stack(left, right)
        B = left.shape[0]
        if (seq is None and restart is None and masks is None and ch == 1
                and left.shape[1:3] == (self.camera.height, self.camera.width)):
            res = (plf_frame_result * B)()
            st = self.lib.plf_process_batch(self._ctx, B, _ptr(left, C.c_uint8), _ptr(right, C.c_uint8),
                                            self.camera.width, res)
            self._check(st, "plf_process_batch")
            return self._result_dicts(res, B)
        seq_a, restart_a = self._sequence_table(B, seq, restart)   # checked before anything is uploaded
        self.batch_upload(left, right)
        if masks is not None:
            self.batch_upload_masks(*masks)
        self._run_sequences(B, seq_a, restart_a)
        return self.batch_download(B)

    def batch_upload(self, left, right):
        """Uploads grey uint8 [B,H,W] pairs (plf_batch_upload) or BGR / BGRA uint8 [B,H,W,3|4] pairs, which the run
        converts to grey on the device (plf_batch_upload_color).  Pairs of one of image_sizes go through
        plf_batch_upload_sized.  Returns B."""
        left, right, ch = self._stack(left, right)
        H, W = left.shape[1:3]
        if (H, W) != (self.camera.height, self.camera.width):
            self._check(self.lib.plf_batch_upload_sized(self._ctx, left.shape[0], int(W), int(H), _ptr(left, C.c_uint8),
                                                        _ptr(right, C.c_uint8), ch * int(W), ch), "plf_batch_upload_sized")
        elif ch == 1:
            self._check(self.lib.plf_batch_upload(self._ctx, left.shape[0], _ptr(left, C.c_uint8), _ptr(right, C.c_uint8),
                                                  self.camera.width), "plf_batch_upload")
        else:
            self._check(self.lib.plf_batch_upload_color(self._ctx, left.shape[0], _ptr(left, C.c_uint8),
                                                        _ptr(right, C.c_uint8), ch * self.camera.width, ch),
                        "plf_batch_upload_color")
        return left.shape[0]

    def batch_upload_raw(self, B, left_ptr, right_ptr, channels=1, stride=None, size=None):
        """Upload from raw host addresses (e.g. pinned memory): B images per side of H rows of `stride` bytes (None:
        channels * W), grey (channels 1) or BGR / BGRA (3 / 4, plf_batch_upload_color).  size: (W, H) of the images,
        the camera's (None) or one of image_sizes (plf_batch_upload_sized)."""
        W, H = (self.camera.width, self.camera.height) if size is None else (int(size[0]), int(size[1]))
        stride = channels * W if stride is None else int(stride)
        if (W, H) != (self.camera.width, self.camera.height):
            self._check(self.lib.plf_batch_upload_sized(self._ctx, int(B), W, H, C.c_void_p(left_ptr), C.c_void_p(right_ptr),
                                                        stride, int(channels)), "plf_batch_upload_sized")
        elif channels == 1:
            self._check(self.lib.plf_batch_upload(self._ctx, int(B), C.c_void_p(left_ptr), C.c_void_p(right_ptr), stride),
                        "plf_batch_upload")
        else:
            self._check(self.lib.plf_batch_upload_color(self._ctx, int(B), C.c_void_p(left_ptr), C.c_void_p(right_ptr),
                                                        stride, int(channels)), "plf_batch_upload_color")

    @staticmethod
    def _sequence_table(B, seq, restart):
        """seq: integer [B] (sequence of each pair, None = all 0); restart: bool / integer [B] (None = none)."""
        s = Frontend._problem_sequences(B, seq)
        if restart is None:
            return s, None
        r = np.asarray(restart)
        if r.shape != (B,) or r.dtype.kind not in "biu":
            raise PlfError(f"restart must be a 1-D bool or integer array of {B} entries (got {r.dtype}{list(r.shape)})")
        return s, np.ascontiguousarray(r != 0, np.uint8)

    def _run_sequences(self, B, seq, restart):
        self._check(self.lib.plf_batch_run_sequences(self._ctx, int(B), _i32_or_null(seq),
                                                     None if restart is None else _ptr(restart, C.c_uint8)),
                    "plf_batch_run_sequences")

    def batch_run(self, B, seq=None, restart=None):
        """Runs the most recent upload.  seq: the sequence of each pair (integer [B] in [0, max_sequences), None = all 0);
        restart: per pair, nonzero makes it a first frame (None = none).  plf_batch_run_sequences."""
        self._run_sequences(B, *self._sequence_table(B, seq, restart))

    def batch_download(self, B):
        res = (plf_frame_result * B)()
        self._check(self.lib.plf_batch_download(self._ctx, int(B), res), "plf_batch_download")
        return self._result_dicts(res, B)

    def batch_download_array(self, B):
        """Same as batch_download but returns one numpy structured array (RESULT_DTYPE) — no per-frame Python objects."""
        out = np.zeros(B, RESULT_DTYPE)
        self._check(self.lib.plf_batch_download(self._ctx, int(B), out.ctypes.data_as(C.c_void_p)), "plf_batch_download")
        return out

    def batch_device_poses(self, B, dst_device_ptr, stream=0):
        """DT [B,16] f64 of the oldest batch in flight -> caller's device buffer, on the caller's CUDA stream."""
        self._check(self.lib.plf_batch_device_poses(self._ctx, int(B), C.c_void_p(int(dst_device_ptr)), C.c_void_p(int(stream))),
                    "plf_batch_device_poses")

    @property
    def device_images(self) -> int:
        return int(self.lib.plf_batch_device_images(self._ctx) or 0)

    @property
    def device_layout(self):
        """(width, height, pitch) of device_images' slot: the most recent upload's size.  plf_batch_device_layout."""
        w, h, p = C.c_int(0), C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_batch_device_layout(self._ctx, C.byref(w), C.byref(h), C.byref(p)), "plf_batch_device_layout")
        return w.value, h.value, p.value

    def get_frame(self, k):
        """Stereo-valid features of frame k of the last batch (dict of numpy arrays)."""
        K, Ln = self.limits.max_keypoints, self.limits.max_lines
        a = dict(pt_pl=np.zeros((K, 2)), pt_disp=np.zeros(K), pt_P=np.zeros((K, 3)), pt_octave=np.zeros(K, np.int32),
                 pdesc=np.zeros((K, 32), np.uint8), ls_spl=np.zeros((Ln, 2)), ls_epl=np.zeros((Ln, 2)),
                 ls_sdisp=np.zeros(Ln), ls_edisp=np.zeros(Ln), ls_sP=np.zeros((Ln, 3)), ls_eP=np.zeros((Ln, 3)),
                 ls_le=np.zeros((Ln, 3)), ls_angle=np.zeros(Ln, np.float32), ldesc=np.zeros((Ln, 32), np.uint8))
        v = plf_frame_view(cap_pt=K, cap_ls=Ln)
        for name, arr in a.items():
            setattr(v, name, arr.ctypes.data)
        self._check(self.lib.plf_get_frame(self._ctx, int(k), C.byref(v)), "plf_get_frame")
        out = {}
        for name, arr in a.items():
            n = v.n_pt if name.startswith("pt_") or name == "pdesc" else v.n_ls
            out[name] = arr[:n].copy()
        return out

    def get_matches(self, k):
        """Frame-to-frame correspondences of pair k of the last batch (matched_pt / matched_ls after optimizePose), in the
        previous frame's row order: dict with P, pl_obs, inlier_pt (bool) and sP, eP, le_obs, inlier_ls (bool)."""
        K, Ln = self.limits.max_keypoints, self.limits.max_lines
        a = dict(P=np.zeros((K, 3)), pl_obs=np.zeros((K, 2)), inlier_pt=np.zeros(K, np.uint8), sP=np.zeros((Ln, 3)),
                 eP=np.zeros((Ln, 3)), le_obs=np.zeros((Ln, 3)), inlier_ls=np.zeros(Ln, np.uint8))
        v = plf_match_view(cap_pt=K, cap_ls=Ln)
        for name, arr in a.items():
            setattr(v, name, arr.ctypes.data)
        self._check(self.lib.plf_get_matches(self._ctx, int(k), C.byref(v)), "plf_get_matches")
        out = {}
        for name, arr in a.items():
            n = v.n_pt if name in ("P", "pl_obs", "inlier_pt") else v.n_ls
            out[name] = arr[:n].astype(bool) if name.startswith("inlier") else arr[:n].copy()
        return out

    # -- profiling -------------------------------------------------------------------------------
    def profile_enable(self, on=True):
        self._check(self.lib.plf_profile_enable(self._ctx, int(on)), "plf_profile_enable")  # 2: keep the pipeline on

    def profile_read(self):
        """Returns [(stage name, ms)] of the batch_run calls since profiling was enabled / last read."""
        buf = C.create_string_buffer(16384)
        ms = (C.c_float * 1024)()
        n = C.c_int(0)
        self._check(self.lib.plf_profile_read(self._ctx, buf, 16384, ms, 1024, C.byref(n)), "plf_profile_read")
        names = buf.value.decode().split(";")[:n.value]
        return list(zip(names, [ms[i] for i in range(min(n.value, 1024))]))
