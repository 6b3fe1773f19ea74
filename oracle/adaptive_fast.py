"""stvo-pl's adaptative_fast restated (plf_set_adaptive_fast; DESIGN.md §8, SURVEY.md Appendix A.2).  TEST / BENCH
INFRASTRUCTURE ONLY.  stvo-pl is not vendored: the rule is [UPSTREAM-RECALL].  StereoFrameHandler::updateFrame moves
orb_fast_th after each tracked frame; here it runs after pair k of a sequence, th being the threshold pair k was detected
with and r its result:

    first frame (status 2)                  no update (stvo-pl's initialize() runs no updateFrame)
    DT == I exactly, or err > err_th        th = max(min_th, th - 2 inc_th)      (status 1 lands here: DT = I)
    else n_inliers_pt <  feat_th            th = max(min_th, th - 2 inc_th)
    else n_inliers_pt <  2 feat_th          th = max(min_th, th - inc_th)
    else n_inliers_pt >  3 feat_th          th = min(max_th, th + inc_th)
    else n_inliers_pt >  4 feat_th          th = min(max_th, th + 2 inc_th)      unreachable as stvo-pl orders the tests

err is curr_frame->err_norm, -1 when no optimisation ran.  Every first frame of a sequence is detected at orb_fast_th
(stvo-pl sets the threshold once, in the handler's constructor; this library restarts it with the sequence).
oracle/frontend.py run_sequence(adaptive_fast=...) applies it along a stream."""
import numpy as np

BRANCHES = ("first", "bad_pose", "few", "some", "many", "very_many", "keep")


def fast_th_next(th, status, DT, err, n_inliers_pt, cfg, trace=False):
    """The threshold after a pair detected at th with the given result fields; trace=True also returns the branch."""
    lo, hi, inc, f = cfg["min_th"], cfg["max_th"], cfg["inc_th"], cfg["feat_th"]
    if status == 2:
        b, t = "first", th
    elif np.array_equal(np.asarray(DT, np.float64).reshape(4, 4), np.eye(4)) or err > cfg["err_th"]:
        b, t = "bad_pose", max(lo, th - 2 * inc)
    elif n_inliers_pt < f:
        b, t = "few", max(lo, th - 2 * inc)
    elif n_inliers_pt < 2 * f:
        b, t = "some", max(lo, th - inc)
    elif n_inliers_pt > 3 * f:
        b, t = "many", min(hi, th + inc)
    elif n_inliers_pt > 4 * f:
        b, t = "very_many", min(hi, th + 2 * inc)
    else:
        b, t = "keep", th
    return (t, b) if trace else t


def fast_th0(prm):
    """orb_fast_th as the detector applies it (clamped to [0, 255])."""
    return min(max(int(prm["orb_fast_th"]), 0), 255)


def result_next(th, r, cfg, trace=False):
    """fast_th_next on a plf_frame_result (dict or RESULT_DTYPE row)."""
    return fast_th_next(th, int(r["status"]), r["DT"], float(r["err"]), int(r["n_inliers_pt"]), cfg, trace)
