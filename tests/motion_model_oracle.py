"""stvo-pl's use_motion_model restated for the tests (plf_set_motion_model; DESIGN.md §8).  stvo-pl is not vendored: the
rule is [UPSTREAM-RECALL].  StereoFrameHandler::optimizePose starts from prev_frame->DT when isGoodSolution accepts it:

    isGoodSolution(DT, DT_cov, err):  reject when  eig_min(DT_cov) < 0 || eig_max(DT_cov) > 1 || err < 0 || err > 1
                                                   || DT has a non-finite entry

Every test is a rejection, so a NaN eigenvalue or err passes.  Here, after pair k of a sequence with result r, the
prediction of its next pair is T = inverse_se3(r.DT) (the optimiser's own transform, previous frame into current) when
status is 0 and r passes, else the identity.  The recalled line is `DT = prev_frame->DT`, the published increment, whose
inverse is the optimiser's variable; the library uses the optimiser's transform.  A covariance with a non-finite entry
has NaN eigenvalues.  The next pair projects the previous frame's 3-D features through T before the windowed
frame-to-frame matching (matching_strategy != 0) and seeds the pose solver with it.  With the model off, everything is
oracle/frontend.py as it stands."""
import numpy as np

from oracle import clib
from oracle import frontend as ofe
from oracle import matching as om
from oracle.kfmatching import rigid


def eig_range(cov):
    """(smallest, largest) eigenvalue of the symmetric part of a 6x6 covariance; NaN for a non-finite entry."""
    cov = np.asarray(cov, np.float64).reshape(6, 6)
    if not np.all(np.isfinite(cov)):
        return np.nan, np.nan
    e = np.linalg.eigvalsh(0.5 * (cov + cov.T))
    return float(e[0]), float(e[-1])


def is_good(status, DT, DT_cov, err):
    """stvo-pl's isGoodSolution as recalled, on a tracked pair (status 0)."""
    if int(status) != 0 or not np.all(np.isfinite(np.asarray(DT, np.float64))):
        return False
    lo, hi = eig_range(DT_cov)
    return not (lo < 0.0 or hi > 1.0 or err < 0.0 or err > 1.0)


def prior(status, DT, DT_cov, err):
    """(T, valid): the prediction a pair's result gives its sequence's next pair."""
    if is_good(status, DT, DT_cov, err):
        return clib.inverse_se3(np.asarray(DT, np.float64).reshape(4, 4)), True
    return np.eye(4), False


def result_prior(r):
    """prior on a plf_frame_result (dict or RESULT_DTYPE row)."""
    return prior(int(np.asarray(r["status"])), np.asarray(r["DT"]).reshape(4, 4), np.asarray(r["DT_cov"]).reshape(6, 6),
                 float(np.asarray(r["err"])))


def track_matches(cam, prev, curr, prm, T_pred, stats=None):
    """oracle/frontend.py track_matches with the previous frame's points and line end points moved by T_pred before the
    projection (src/mapHandler.cpp:254-256, :384-389 project through DT).  stats (a dict, matching_strategy != 0) gets
    the windowed point / line match counts (pt_window, ls_window) and whether match() took over (pt_fallback,
    ls_fallback)."""
    if not prm.get("matching_strategy", 0):
        return ofe.track_matches(cam, prev, curr, prm)
    proj = lambda X: ofe.projection(cam, rigid(T_pred, X))
    ws = int(prm["matching_f2f_ws"])
    w = (ws, ws, ws, ws)
    mp, ml = np.full(len(prev.pdesc), -1, np.int32), np.full(len(prev.ldesc), -1, np.int32)
    if len(prev.pdesc) and len(curr.pdesc):
        mp, n = ofe.grid_match_points(cam, proj(prev.pt_P), prev.pdesc, curr.pt_pl, curr.pdesc, w, prm["min_ratio_12_p"],
                                      prm["best_lr_matches"])
        k = int(prm["min_pt_matches"])
        fall = len(curr.pdesc) > k and len(prev.pdesc) > k and n < k
        if fall:
            mp, _ = om.match(prev.pdesc, curr.pdesc, prm["min_ratio_12_p"], prm["best_lr_matches"])
        if stats is not None:
            stats.update(pt_window=int(n), pt_fallback=bool(fall))
    if len(prev.ldesc) and len(curr.ldesc):
        q = np.concatenate([proj(prev.ls_sP), proj(prev.ls_eP)], 1)
        t = np.concatenate([curr.ls_spl, curr.ls_epl], 1)
        ml, n = ofe.grid_match_lines(cam, q, prev.ldesc, t, curr.ldesc, w, prm["min_ratio_12_l"], prm["line_sim_th"],
                                     prm["best_lr_matches"])
        k = int(prm["min_ls_matches"])
        fall = len(curr.ldesc) > k and len(prev.ldesc) > k and n < k
        if fall:
            ml, _ = om.match(prev.ldesc, curr.ldesc, prm["min_ratio_12_l"], prm["best_lr_matches"])
        if stats is not None:
            stats.update(ls_window=int(n), ls_fallback=bool(fall))
    return mp, ml


def track(cam, prev, curr, prm, T_pred):
    """oracle/frontend.py track with track_matches above; its stats under "stats"."""
    stats = {}
    mp, ml = track_matches(cam, prev, curr, prm, T_pred, stats)
    ip, il = np.nonzero(mp >= 0)[0], np.nonzero(ml >= 0)[0]
    return dict(P=prev.pt_P[ip], obs=curr.pt_pl[mp[ip]], sP=prev.ls_sP[il], eP=prev.ls_eP[il], le=curr.ls_le[ml[il]],
                mp=mp, ml=ml, stats=stats)


def optimize_pose(cam, tr, prm, T_pred):
    """oracle/frontend.py optimize_pose with the solver seeded with T_pred (clib.gn_pose T_init)."""
    if len(tr["P"]) + len(tr["sP"]) < prm["min_features"]:
        return np.eye(4), None, 1
    o = clib.gn_opts(prm["homog_th"], prm["max_iters"], prm["max_iters_ref"], prm["min_error"], prm["min_error_change"])
    r = clib.gn_pose(cam, tr["P"], tr["obs"], tr["sP"], tr["eP"], tr["le"], T_init=T_pred, opts=o, trace=True)
    r.update(opts=o, cam=cam, rows={k: tr[k] for k in ("P", "obs", "sP", "eP", "le")})
    return clib.inverse_se3(r["T"]), r, 0


def run_sequence(cam, pairs, prm=None, motion_model=True, preds=None, restarts=(), frames=None, fast_th=None):
    """oracle/frontend.py run_sequence with the motion model.  Pair i starts from preds[i] when given (the predictions
    another run used, so that a rounding difference at an edge of the rule cannot make two runs diverge), else from the
    prediction carried from pair i - 1; `restarts` are pair indices that are first frames; fast_th[i]: the FAST
    threshold pair i is detected at (adaptive FAST).  Each entry also holds T_pred (used), T_next / valid_next (the
    rule on this run's own result) and, with the model on, the windowed matching's stats (track_matches).  With
    motion_model False every pair goes through oracle/frontend.py's own track and optimize_pose, as its run_sequence
    does."""
    prm = dict(ofe.DEFAULTS, **(prm or {}))
    prev, Tfw, T, out = None, np.eye(4), np.eye(4), []
    for i, (L, R) in enumerate(pairs):
        if i in restarts:
            prev = None
        if prev is None:
            T = np.eye(4)
        if preds is not None:
            T = np.asarray(preds[i], np.float64).reshape(4, 4)
        p = prm if fast_th is None else dict(prm, orb_fast_th=int(fast_th[i]))
        cur = frames[i] if frames is not None else ofe.extract_stereo(cam, L, R, p)
        stats = {}
        if prev is None:
            DT, status, res = np.eye(4), 2, None
        elif motion_model:
            tr = track(cam, prev, cur, prm, T)
            stats = tr["stats"]
            DT, res, status = optimize_pose(cam, tr, prm, T)
        else:
            DT, res, status = ofe.optimize_pose(cam, ofe.track(prev, cur, prm, cam=cam), prm)
        Tfw = Tfw @ DT
        cov = res["cov"] if status == 0 else np.zeros((6, 6))
        err = res["err"] if status == 0 else -1.0
        T_next, valid = prior(status, DT, cov, err)
        out.append(dict(DT=DT, Tfw=Tfw.copy(), status=status, n_pt=len(cur.pt_pl), n_ls=len(cur.ls_spl), res=res, frame=cur,
                        T_pred=T, T_next=T_next, valid_next=valid, stats=stats))
        prev, T = cur, (T_next if motion_model else np.eye(4))
    return out
