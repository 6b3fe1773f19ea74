"""Oracle compositions of the per-image / per-pair front-end stages (numpy + the C restatements).
TEST / BENCH INFRASTRUCTURE ONLY.

detect_lines   stvo-pl StereoFrame::detectLineFeatures, LSD branch (SURVEY.md Appendix A.2, [UPSTREAM-RECALL],
               unpinned): LSDDetectorC::detect (LSDDetector_custom.cpp:218-324) -> if more than lsd_nfeatures lines
               (and lsd_nfeatures != 0): sort by response descending (std::sort ties are implementation-defined in
               the reference; canonical here: detection order), keep lsd_nfeatures, class_id = rank ->
               BinaryDescriptor::compute (binary_descriptor_custom.cpp:524).
"""
import numpy as np

from oracle import clib


def detect_lines(img, lsd_nfeatures=300, min_line_length=0.025, lsd_kwargs=None, segs=None):
    h, w = img.shape
    if segs is None:
        segs = clib.lsd(img, **(lsd_kwargs or {}))
    kl = clib.keylines_from_segments(segs, w, h, float(np.float32(min_line_length)) * min(w, h))
    if lsd_nfeatures != 0 and len(kl) > lsd_nfeatures:
        order = np.lexsort((np.arange(len(kl)), -kl["response"].astype(np.float64)))
        kl = kl[order[:lsd_nfeatures]].copy()
        kl["class_id"] = np.arange(lsd_nfeatures, dtype=np.int32)
    desc = clib.lbd_compute(img, kl) if len(kl) else np.zeros((0, 32), np.uint8)
    return kl, desc


# =====================================================================================================
# Stereo association, frame-to-frame tracking and the full per-frame front-end (SURVEY.md §8 a6, a7).
# stvo-pl is not vendored: everything below is a restatement of SURVEY.md Appendix A.2 / A.3
# ([UPSTREAM-RECALL]) => "parity unpinned"; the field patterns match the in-tree analogue
# MapHandler::matchKF2KFPoints / matchKF2KFLines (src/mapHandler.py:234-363, :365-530).
# =====================================================================================================
from dataclasses import dataclass, field

from oracle import matching as om

DEFAULTS = dict(  # config/config/config_euroc.yaml:9-77; every field of plf_default_params() (pl-slam_b200/csrc/plf_ctx.cu)
    has_points=True, has_lines=True,
    best_lr_matches=True, max_dist_epip=1.0, min_disp=1.0, min_ratio_12_p=0.9, line_sim_th=0.75,
    stereo_overlap_th=0.75, f2f_overlap_th=0.75, min_line_length=0.025, line_horiz_th=0.1, min_ratio_12_l=0.9,
    ls_min_disp_ratio=0.7, homog_th=1e-7, min_features=10, max_iters=5, max_iters_ref=10, min_error=1e-7,
    min_error_change=1e-7, inlier_k=4.0,
    orb_nfeatures=800, orb_scale_factor=1.2, orb_nlevels=4, orb_edge_th=19, orb_wta_k=2, orb_score=1, orb_patch_size=31,
    orb_fast_th=20,
    lsd_nfeatures=300, lsd_refine=0, lsd_scale=1.2, lsd_sigma_scale=0.6, lsd_quant=2.0, lsd_ang_th=22.5, lsd_log_eps=1.0,
    lsd_density_th=0.6, lsd_n_bins=1024,
    # matching strategy (config_euroc.yaml:55-57; 0 = descriptor only, the default of this library; the reference
    # configs select 3 = windowed) and the fall-back thresholds of the in-tree analogue (src/slamConfig.cpp:85-86)
    matching_strategy=0, matching_s_ws=10, matching_f2f_ws=3, min_pt_matches=10, min_ls_matches=6)

GRID_ROWS, GRID_COLS = 48, 64   # stvo-pl gridStructure.h (SURVEY Appendix A.2)


def f32(x):
    return float(np.float32(x))


def back_projection(cam, u, v, disp):
    """PinholeStereoCamera::backProjection (SURVEY A.4): Z = fx b / d, X = Z (u - cx) / fx, Y = Z (v - cy) / fy."""
    Z = cam["fx"] * cam["b"] / disp
    return np.array([Z * (u - cam["cx"]) / cam["fx"], Z * (v - cam["cy"]) / cam["fy"], Z])


def line_overlap_stereo(spl_obs, epl_obs, spl_proj, epl_proj, line_horiz_th):
    """stvo-pl StereoFrame::lineSegmentOverlapStereo on the endpoints' rows."""
    overlap = 1.0
    if abs(epl_obs - spl_obs) > line_horiz_th:
        sln, eln = min(spl_obs, epl_obs), max(spl_obs, epl_obs)
        spn, epn = min(spl_proj, epl_proj), max(spl_proj, epl_proj)
        length = eln - spn
        if epn < sln or spn > eln:
            overlap = 0.0
        elif epn > eln and spn < sln:
            overlap = eln - sln
        else:
            overlap = min(eln, epn) - max(sln, spn)
        overlap = overlap / length if length > f32(0.01) else 0.0
        if overlap > 1.0:
            overlap = 1.0
    return overlap


@dataclass
class Frame:
    """The stereo-valid content of a StVO::StereoFrame (Appendix A.1): row i of pdesc/ldesc <-> stereo_pt/ls[i]."""
    pt_pl: np.ndarray = field(default_factory=lambda: np.zeros((0, 2)))
    pt_disp: np.ndarray = field(default_factory=lambda: np.zeros(0))
    pt_P: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    pt_octave: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    pdesc: np.ndarray = field(default_factory=lambda: np.zeros((0, 32), np.uint8))
    ls_spl: np.ndarray = field(default_factory=lambda: np.zeros((0, 2)))
    ls_epl: np.ndarray = field(default_factory=lambda: np.zeros((0, 2)))
    ls_sdisp: np.ndarray = field(default_factory=lambda: np.zeros(0))
    ls_edisp: np.ndarray = field(default_factory=lambda: np.zeros(0))
    ls_sP: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    ls_eP: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    ls_le: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    ls_angle: np.ndarray = field(default_factory=lambda: np.zeros(0, np.float32))
    ldesc: np.ndarray = field(default_factory=lambda: np.zeros((0, 32), np.uint8))


def grid_scales(cam):
    """StereoFrame::inv_width / inv_height = GRID_COLS / width, GRID_ROWS / height (f64)."""
    return GRID_COLS / float(cam["width"]), GRID_ROWS / float(cam["height"])


def _cell(v):
    """double -> int conversion of a scaled coordinate (C++ truncation toward zero)."""
    return np.trunc(np.asarray(v, np.float64)).astype(np.int64)


def grid_match_points(cam, q_xy, d1, t_xy, d2, w, nnr, best_lr):
    """matchGrid (points): queries / train features at pixel positions q_xy / t_xy (f64 [n,2])."""
    from oracle import matchgrid as mg
    iw, ih = grid_scales(cam)
    q_xy = np.asarray(q_xy, np.float64).reshape(-1, 2)
    t_xy = np.asarray(t_xy, np.float64).reshape(-1, 2)
    q_cell = np.stack([_cell(q_xy[:, 0] * iw), _cell(q_xy[:, 1] * ih)], 1)
    t_cell = np.stack([_cell(t_xy[:, 0] * iw), _cell(t_xy[:, 1] * ih)], 1)
    return mg.match_grid_points(q_cell, d1, mg.grid_from_points(t_cell, GRID_ROWS, GRID_COLS), d2, w, nnr, best_lr)


def grid_match_lines(cam, q_se, d1, t_se, d2, w, nnr, line_sim_th, best_lr):
    """matchGrid (lines): q_se / t_se = [n,4] pixel end points (sx, sy, ex, ey), f64.  Train directions are the
    normalised scaled deltas ((ex - sx) inv_width, (ey - sy) inv_height) (src/mapHandler.cpp:402-404)."""
    from oracle import matchgrid as mg
    iw, ih = grid_scales(cam)
    sc = np.array([iw, ih, iw, ih])
    q_se = np.asarray(q_se, np.float64).reshape(-1, 4)
    t_se = np.asarray(t_se, np.float64).reshape(-1, 4)
    q_line, t_line = _cell(q_se * sc), _cell(t_se * sc)
    vx, vy = (t_se[:, 2] - t_se[:, 0]) * iw, (t_se[:, 3] - t_se[:, 1]) * ih
    with np.errstate(invalid="ignore", divide="ignore"):
        nrm = np.sqrt(vx * vx + vy * vy)
        t_dir = np.stack([vx / nrm, vy / nrm], 1)
    return mg.match_grid_lines(q_line, d1, mg.grid_from_lines(t_line, GRID_ROWS, GRID_COLS), t_dir, d2, w, nnr,
                               float(np.float32(line_sim_th)), best_lr)


def stereo_points(cam, kp_l, desc_l, kp_r, desc_r, prm, match_fn=None):
    if prm.get("matching_strategy", 0) and match_fn is None:
        # stvo-pl matchStereoPoints: window (matching_s_ws, 0) x (0, 0) left of / on the query's cell (A.2)
        q = np.stack([kp_l["x"].astype(np.float64), kp_l["y"].astype(np.float64)], 1)
        t = np.stack([kp_r["x"].astype(np.float64), kp_r["y"].astype(np.float64)], 1)
        m12, _ = grid_match_points(cam, q, desc_l, t, desc_r, (int(prm["matching_s_ws"]), 0, 0, 0), prm["min_ratio_12_p"],
                                   prm["best_lr_matches"])
    else:
        m12, _ = (match_fn or om.match)(desc_l, desc_r, prm["min_ratio_12_p"], prm["best_lr_matches"])
    pl, disp, P, octv, rows = [], [], [], [], []
    for i, j in enumerate(m12):
        if j < 0:
            continue
        xl, yl, xr, yr = kp_l["x"][i], kp_l["y"][i], kp_r["x"][j], kp_r["y"][j]   # float32 pixels
        if abs(np.float32(yl - yr)) <= f32(prm["max_dist_epip"]):
            d = float(np.float32(xl - xr))
            if d >= f32(prm["min_disp"]):
                pl.append((float(xl), float(yl))); disp.append(d)
                P.append(back_projection(cam, float(xl), float(yl), d)); octv.append(int(kp_l["octave"][i])); rows.append(i)
    n = len(rows)
    return (np.array(pl, np.float64).reshape(n, 2), np.array(disp, np.float64), np.array(P, np.float64).reshape(n, 3),
            np.array(octv, np.int32), desc_l[rows].reshape(n, 32))


def _kl_se(kl):
    return np.stack([kl["startPointX"], kl["startPointY"], kl["endPointX"], kl["endPointY"]], 1).astype(np.float64)


def stereo_lines(cam, kl_l, desc_l, kl_r, desc_r, prm, match_fn=None):
    if prm.get("matching_strategy", 0) and match_fn is None:
        m12, _ = grid_match_lines(cam, _kl_se(kl_l), desc_l, _kl_se(kl_r), desc_r, (int(prm["matching_s_ws"]), 0, 0, 0),
                                  prm["min_ratio_12_l"], prm["line_sim_th"], prm["best_lr_matches"])
    else:
        m12, _ = (match_fn or om.match)(desc_l, desc_r, prm["min_ratio_12_l"], prm["best_lr_matches"])
    out = dict(spl=[], epl=[], sdisp=[], edisp=[], sP=[], eP=[], le=[], angle=[], rows=[])
    for i, j in enumerate(m12):
        if j < 0:
            continue
        sp_l = np.array([float(kl_l["startPointX"][i]), float(kl_l["startPointY"][i]), 1.0])
        ep_l = np.array([float(kl_l["endPointX"][i]), float(kl_l["endPointY"][i]), 1.0])
        le_l = np.cross(sp_l, ep_l)
        le_l = le_l / np.sqrt(le_l[0] * le_l[0] + le_l[1] * le_l[1])
        sp_r = np.array([float(kl_r["startPointX"][j]), float(kl_r["startPointY"][j]), 1.0])
        ep_r = np.array([float(kl_r["endPointX"][j]), float(kl_r["endPointY"][j]), 1.0])
        le_r = np.cross(sp_r, ep_r)
        overlap = line_overlap_stereo(sp_l[1], ep_l[1], sp_r[1], ep_r[1], f32(prm["line_horiz_th"]))
        with np.errstate(divide="ignore", invalid="ignore"):
            sxr = -(le_r[2] + le_r[1] * sp_l[1]) / le_r[0]
            exr = -(le_r[2] + le_r[1] * ep_l[1]) / le_r[0]
        disp_s, disp_e = sp_l[0] - sxr, ep_l[0] - exr
        # filterLineSegmentDisparity
        with np.errstate(divide="ignore", invalid="ignore"):
            if not (min(disp_s, disp_e) / max(disp_s, disp_e) >= f32(prm["ls_min_disp_ratio"])):
                disp_s = disp_e = -1.0
        if (disp_s >= f32(prm["min_disp"]) and disp_e >= f32(prm["min_disp"]) and
                abs(np.float32(le_r[0])) > f32(prm["line_horiz_th"]) and overlap > f32(prm["stereo_overlap_th"])):
            out["spl"].append(sp_l[:2]); out["epl"].append(ep_l[:2]); out["sdisp"].append(disp_s); out["edisp"].append(disp_e)
            out["sP"].append(back_projection(cam, sp_l[0], sp_l[1], disp_s))
            out["eP"].append(back_projection(cam, ep_l[0], ep_l[1], disp_e))
            out["le"].append(le_l); out["angle"].append(kl_l["angle"][i]); out["rows"].append(i)
    n = len(out["rows"])
    a = lambda k, c: np.array(out[k], np.float64).reshape(n, c) if c > 1 else np.array(out[k], np.float64)
    return (a("spl", 2), a("epl", 2), a("sdisp", 1), a("edisp", 1), a("sP", 3), a("eP", 3), a("le", 3),
            np.array(out["angle"], np.float32), desc_l[out["rows"]].reshape(n, 32))


def extract_stereo(cam, left, right, prm, orb_fn=None, lines_fn=None, match_fn=None, pool=None):
    """StereoFrame::extractStereoFeatures.  orb_fn / lines_fn default to the C restatements (bit-identical to cv2)."""
    if orb_fn is None:
        orb_fn = lambda im: _orb_c(im, prm)
    if lines_fn is None:
        lines_fn = lambda im: detect_lines(im, prm["lsd_nfeatures"], prm["min_line_length"], lsd_kwargs(prm))
    # has_points / has_lines = false: stvo-pl neither detects nor matches the disabled kind
    has_p, has_l = prm.get("has_points", True), prm.get("has_lines", True)
    none = lambda im: (None, None)
    orb_fn, lines_fn = (orb_fn if has_p else none), (lines_fn if has_l else none)
    if pool is not None:   # lr_in_parallel / pl_in_parallel (config_euroc.yaml:14-15): 4 concurrent tasks
        fa, fb, fc, fd = (pool.submit(orb_fn, left), pool.submit(orb_fn, right), pool.submit(lines_fn, left),
                          pool.submit(lines_fn, right))
        (kp_l, d_l), (kp_r, d_r), (kl_l, ld_l), (kl_r, ld_r) = fa.result(), fb.result(), fc.result(), fd.result()
    else:
        kp_l, d_l = orb_fn(left); kp_r, d_r = orb_fn(right)
        kl_l, ld_l = lines_fn(left); kl_r, ld_r = lines_fn(right)
    f = Frame()
    if has_p:
        f.pt_pl, f.pt_disp, f.pt_P, f.pt_octave, f.pdesc = stereo_points(cam, kp_l, d_l, kp_r, d_r, prm, match_fn)
    if has_l:
        (f.ls_spl, f.ls_epl, f.ls_sdisp, f.ls_edisp, f.ls_sP, f.ls_eP, f.ls_le, f.ls_angle, f.ldesc) = \
            stereo_lines(cam, kl_l, ld_l, kl_r, ld_r, prm, match_fn)
    return f


def _orb_c(img, prm):
    """cv::ORB::create(orb_nfeatures, orb_scale_factor, orb_nlevels, orb_edge_th, 0, orb_wta_k, orb_score,
    orb_patch_size, orb_fast_th) as restated by oracle/orb.c: WTA_K 2 and the FAST score only."""
    if prm.get("orb_wta_k", 2) != 2 or prm.get("orb_score", 1) != 1:
        raise ValueError("the ORB oracle restates WTA_K = 2 with the FAST score only")
    return clib.orb(img, prm["orb_nfeatures"], prm.get("orb_scale_factor", 1.2), prm["orb_nlevels"],
                    prm.get("orb_edge_th", 19), prm.get("orb_patch_size", 31), prm["orb_fast_th"])


def lsd_kwargs(prm):
    """The cv::createLineSegmentDetector options of prm for clib.lsd.  lsd_log_eps / lsd_density_th only act when
    lines are refined, which the oracle (like the library) does not support."""
    if prm.get("lsd_refine", 0) != 0:
        raise ValueError("the LSD oracle restates lsd_refine = 0 only")
    return dict(scale=prm.get("lsd_scale", 1.2), sigma_scale=prm.get("lsd_sigma_scale", 0.6), quant=prm.get("lsd_quant", 2.0),
                ang_th=prm.get("lsd_ang_th", 22.5), n_bins=prm.get("lsd_n_bins", 1024))


def projection(cam, P):
    """PinholeStereoCamera::projection (A.4)."""
    P = np.asarray(P, np.float64).reshape(-1, 3)
    return np.stack([cam["cx"] + cam["fx"] * P[:, 0] / P[:, 2], cam["cy"] + cam["fy"] * P[:, 1] / P[:, 2]], 1)


def track_matches(cam, prev: Frame, curr: Frame, prm, match_fn=None):
    """The two matches_12 vectors of f2fTracking.  matching_strategy 0: match() on the stereo-valid descriptors (A.2).
    Otherwise the control flow of the in-tree analogue (src/mapHandler.cpp:247-278, :379-425) with DT = identity
    (use_motion_model false): the previous frame's 3-D features are projected, matched in a +-matching_f2f_ws window of
    the current frame's grid, and match() takes over when fewer than min_pt_matches / min_ls_matches survive (both
    frames holding more features than that).  Projected lines are scaled to grid units like the points (the analogue
    leaves them in pixels, :395, which empties the window; not reproduced)."""
    mfn = match_fn or om.match
    if not prm.get("matching_strategy", 0) or match_fn is not None:
        mp, _ = mfn(prev.pdesc, curr.pdesc, prm["min_ratio_12_p"], prm["best_lr_matches"])
        ml, _ = mfn(prev.ldesc, curr.ldesc, prm["min_ratio_12_l"], prm["best_lr_matches"])
        return mp, ml
    ws = int(prm["matching_f2f_ws"])
    w = (ws, ws, ws, ws)
    mp, ml = np.full(len(prev.pdesc), -1, np.int32), np.full(len(prev.ldesc), -1, np.int32)
    if len(prev.pdesc) and len(curr.pdesc):
        mp, n = grid_match_points(cam, projection(cam, prev.pt_P), prev.pdesc, curr.pt_pl, curr.pdesc, w,
                                  prm["min_ratio_12_p"], prm["best_lr_matches"])
        k = int(prm["min_pt_matches"])
        if len(curr.pdesc) > k and len(prev.pdesc) > k and n < k:
            mp, _ = om.match(prev.pdesc, curr.pdesc, prm["min_ratio_12_p"], prm["best_lr_matches"])
    if len(prev.ldesc) and len(curr.ldesc):
        q = np.concatenate([projection(cam, prev.ls_sP), projection(cam, prev.ls_eP)], 1)
        t = np.concatenate([curr.ls_spl, curr.ls_epl], 1)
        ml, n = grid_match_lines(cam, q, prev.ldesc, t, curr.ldesc, w, prm["min_ratio_12_l"], prm["line_sim_th"],
                                 prm["best_lr_matches"])
        k = int(prm["min_ls_matches"])
        if len(curr.ldesc) > k and len(prev.ldesc) > k and n < k:
            ml, _ = om.match(prev.ldesc, curr.ldesc, prm["min_ratio_12_l"], prm["best_lr_matches"])
    return mp, ml


def track(prev: Frame, curr: Frame, prm, match_fn=None, cam=None):
    """f2fTracking: the two matches_12 vectors (track_matches), then the GN rows."""
    mp, ml = track_matches(cam, prev, curr, prm, match_fn)
    ip = np.nonzero(mp >= 0)[0]
    P, obs = prev.pt_P[ip], curr.pt_pl[mp[ip]]
    il = np.nonzero(ml >= 0)[0]
    sP, eP, le = prev.ls_sP[il], prev.ls_eP[il], curr.ls_le[ml[il]]
    return dict(P=P, obs=obs, sP=sP, eP=eP, le=le, mp=mp, ml=ml)


def optimize_pose(cam, tr, prm):
    """optimizePose: two-stage GN from identity; fewer than min_features rows -> identity.  Returns curr.DT
    (= inverse of the optimised increment), the raw result (with the solver's stop-decision trace, its options, camera
    and rows, so that a result of another solver can be compared with it: clib.gn_decidable) and a status flag."""
    n = len(tr["P"]) + len(tr["sP"])
    if n < prm["min_features"]:
        return np.eye(4), None, 1
    o = clib.gn_opts(prm["homog_th"], prm["max_iters"], prm["max_iters_ref"], prm["min_error"], prm["min_error_change"])
    r = clib.gn_pose(cam, tr["P"], tr["obs"], tr["sP"], tr["eP"], tr["le"], opts=o, trace=True)
    r.update(opts=o, cam=cam, rows={k: tr[k] for k in ("P", "obs", "sP", "eP", "le")})
    return clib.inverse_se3(r["T"]), r, 0


def run_sequence(cam, pairs, prm=None, orb_fn=None, lines_fn=None, match_fn=None, pool=None, frames=None):
    """The hot loop of app/plslam_dataset.cpp:111-163 without keyframe hand-off: returns per-frame DT (4x4), Tfw."""
    prm = dict(DEFAULTS, **(prm or {}))
    prev, Tfw, out = None, np.eye(4), []
    for idx, (L, R) in enumerate(pairs):
        cur = frames[idx] if frames is not None else extract_stereo(cam, L, R, prm, orb_fn, lines_fn, match_fn, pool)
        if prev is None:
            DT, status, res = np.eye(4), 2, None      # initialize(): first frame
        else:
            tr = track(prev, cur, prm, match_fn, cam=cam)
            DT, res, status = optimize_pose(cam, tr, prm)
        Tfw = Tfw @ DT
        out.append(dict(DT=DT, Tfw=Tfw.copy(), status=status, n_pt=len(cur.pt_pl), n_ls=len(cur.ls_spl), res=res, frame=cur))
        prev = cur
    return out
