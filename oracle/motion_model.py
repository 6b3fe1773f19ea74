"""stvo-pl's use_motion_model restated (plf_set_motion_model; DESIGN.md §8).  TEST / BENCH INFRASTRUCTURE ONLY.  stvo-pl
is not vendored: the rule is [UPSTREAM-RECALL].  StereoFrameHandler::optimizePose starts from prev_frame->DT when
isGoodSolution accepts it:

    isGoodSolution(DT, DT_cov, err):  reject when  eig_min(DT_cov) < 0 || eig_max(DT_cov) > 1 || err < 0 || err > 1
                                                   || DT has a non-finite entry

Every test is a rejection, so a NaN eigenvalue or err passes.  Here, after pair k of a sequence with result r, the
prediction of its next pair is T = inverse_se3(r.DT) (the optimiser's own transform, previous frame into current) when
status is 0 and r passes, else the identity.  The recalled line is `DT = prev_frame->DT`, the published increment, whose
inverse is the optimiser's variable; the library uses the optimiser's transform.  A covariance with a non-finite entry
has NaN eigenvalues.  The next pair projects the previous frame's 3-D features through T before the windowed
frame-to-frame matching (matching_strategy != 0) and seeds the pose solver with it: oracle/frontend.py
run_sequence(motion_model=True)."""
import numpy as np

from oracle import clib


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
