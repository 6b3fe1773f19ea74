"""Loop-closure candidate detection restated in Python: the conf_matrix column of MapHandler::insertKFBowVectorP / L / PL
(src/mapHandler.cpp:3007-3128) and lookForLoopCandidates (:3130-3190).  TEST INFRASTRUCTURE ONLY.

Scalars are Python floats (IEEE double, no contraction), conf_matrix entries numpy float32, as the reference stores them.
The BoW scores themselves come from oracle/dbow.py."""
import math

import numpy as np

DEFAULTS = dict(lc_kf_dist=50, lc_kf_max_dist=50, lc_nkf_closest=4, min_lm_cov_graph=75, min_kf_local_map=3)


def _div(a, b):
    """a / b in IEEE double: 0 / 0 and x / 0 give NaN / inf as in C, not an exception."""
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def vector_stdv(xs):
    """stvo-pl's vector_stdv, recalled (stvo-pl is not in the reference tree): the mean a sequential sum in index order
    over n, then sqrt(sum of (x - mean) * (x - mean), sequentially, / (n - 1)); an empty vector gives 0, one element NaN."""
    xs = [float(x) for x in xs]
    n = len(xs)
    if n == 0:
        return 0.0
    s = 0.0
    for x in xs:
        s += x
    mean = _div(s, n)
    acc = 0.0
    for x in xs:
        d = x - mean
        acc += d * d
    q = _div(acc, n - 1)
    return math.sqrt(q) if q == q and q >= 0 else float("nan")


def dispersions(pt_pl, ls_spl, ls_epl):
    """(std_pt, std_ls) of insertKFBowVectorPL (:3070-3101): over the stereo points' pl and the lines' midpoints."""
    pt = np.asarray(pt_pl, np.float64).reshape(-1, 2)
    s, e = np.asarray(ls_spl, np.float64).reshape(-1, 2), np.asarray(ls_epl, np.float64).reshape(-1, 2)
    mx = [(float(a) + float(b)) * 0.5 for a, b in zip(s[:, 0], e[:, 0])]
    my = [(float(a) + float(b)) * 0.5 for a, b in zip(s[:, 1], e[:, 1])]
    return vector_stdv(pt[:, 0]) + vector_stdv(pt[:, 1]), vector_stdv(mx) + vector_stdv(my)


def conf_row(kinds, live, score_p=None, score_l=None, n_pt=0, n_ls=0, std_pt=0.0, std_ls=0.0):
    """conf_matrix[kf_idx][i] for i <= kf_idx as float32 (NaN where not live).  kinds = (has_points, has_lines): P only
    (float)score_p, L only (float)score_l, both the PL combination of :3109-3127 in double, rounded to float."""
    live = np.asarray(live, bool)
    out = np.full(len(live), np.nan, np.float32)
    std_pl = std_ls + std_pt
    n_pl = n_pt + n_ls
    for i in np.nonzero(live)[0]:
        if kinds[0] and kinds[1]:
            sp, sl = float(score_p[i]), float(score_l[i])
            score = 0.0
            score += _div(sp * n_pt + sl * n_ls, n_pl)
            score += _div(sp * std_pt + sl * std_ls, std_pl)
        else:
            score = float(score_p[i] if kinds[0] else score_l[i])
        out[i] = np.float32(score)
    return out


def look_for_loop_candidates(conf, live, covis, kf_idx, opts=None):
    """lookForLoopCandidates(kf_idx) over conf = conf_matrix[i][kf_idx] (float32 [kf_idx + 1]), live =
    map_keyframes[i] != NULL, covis = full_graph[i][kf_idx] ([kf_idx] or None = all zero).  Returns the result fields
    of plf_lc_detect_result.  C++'s conversions are kept: full_graph is unsigned, size() > lcKFMaxDist() compares as
    size_t.  Equal maxima: the lowest index first (a stable sort); NaN ranks below every number.  Listed indices stop at
    kf_idx (the map holds no keyframe after it)."""
    o = dict(DEFAULTS, **(opts or {}))
    conf = np.asarray(conf, np.float32)
    live = np.asarray(live, bool)
    cov = np.zeros(kf_idx, np.uint32) if covis is None else np.asarray(covis, np.uint32)
    res = dict(candidate=-1, best=-1, n_listed=0, n_closest=0, min_score=float("nan"))
    score = lambda i: float(conf[i]) if live[i] else 0.0   # absent: never written, zero-filled (expandGraphs)
    max_confmat = [(i, float(conf[i])) for i in range(min(kf_idx - o["lc_kf_dist"], kf_idx + 1)) if live[i]]
    res["n_listed"] = len(max_confmat)
    if not len(max_confmat) > o["lc_kf_max_dist"] % (1 << 64):
        return res
    max_confmat.sort(key=lambda e: (0, 0.0) if math.isnan(e[1]) else (1, e[1]), reverse=True)
    lc_min_score = 1.0
    for i in range(kf_idx):
        if int(cov[i]) >= o["min_lm_cov_graph"] % (1 << 32) or kf_idx - i <= o["min_kf_local_map"] + 3:
            s = score(i)
            if s < lc_min_score and s > 0.001:
                lc_min_score = s
    res["min_score"] = lc_min_score
    idx_max = max_confmat[0][0]
    res["best"] = idx_max
    if max_confmat[0][1] >= lc_min_score:
        n = 0
        for idx, s in max_confmat[1:]:
            if abs(idx - idx_max) <= o["lc_kf_max_dist"] and s >= lc_min_score * 0.8:
                n += 1
        res["n_closest"] = n
        if n >= o["lc_nkf_closest"]:
            res["candidate"] = idx_max
    return res
