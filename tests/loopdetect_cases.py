"""Hand-built columns for lookForLoopCandidates (src/mapHandler.cpp:3130-3190), one per branch and threshold, with the
result each must give.  Shared by the oracle's CPU tests and the device's (plf_debug_loop_candidates).

The base column: kf_idx 30 and opts O.  Listed: live i < 25.  The local window (kf_idx - i <= min_kf_local_map + 3 = 4)
is i = 26..29 with scores 0.30, 0.40, 0.35, 0.50, so lc_min_score is float(0.3f) and the 0.8 threshold about 0.24.
Listed filler sits at 0.05 + 0.001 i, the best match at i = 10 (0.60) and its two close supporters at i = 8 and 12
(0.25).  Every case changes a few entries; `exact` lists the indices a case puts on a threshold on purpose, and every
other score stays well away from each threshold (test_loop_detect.py checks it)."""
import numpy as np

O = dict(lc_kf_dist=5, lc_kf_max_dist=4, lc_nkf_closest=2, min_lm_cov_graph=10, min_kf_local_map=1)
F = np.float32
MIN = float(F(0.30))
NAN = float("nan")


def below(x):
    return F(np.nextafter(F(x), F(-1)))


def above(x):
    return F(np.nextafter(F(x), F(2)))


def column(kf=30, vals=None, dead=(), covis=None, filler=True):
    conf = np.full(kf + 1, np.nan, np.float32)
    if filler:
        for i in range(kf + 1):
            conf[i] = F(0.05 + 0.001 * i)
        for i, v in zip(range(kf - 4, kf), (0.30, 0.40, 0.35, 0.50)):
            if i >= 0:
                conf[i] = F(v)
        if kf == 30:
            conf[10], conf[8], conf[12] = F(0.60), F(0.25), F(0.25)
        conf[kf] = F(0.95)   # the self-score: never listed while lc_kf_dist >= 0
    for i, v in (vals or {}).items():
        conf[i] = v
    live = np.ones(kf + 1, bool)
    live[list(dead)] = False
    cv = None
    if covis is not None:
        cv = np.zeros(kf, np.uint32)
        for i, v in covis.items():
            cv[i] = v
    return dict(kf_idx=kf, conf=conf, live=live, covis=cv)


def R(candidate, best, n_listed, n_closest, min_score):
    return dict(candidate=candidate, best=best, n_listed=n_listed, n_closest=n_closest, min_score=min_score)


def case(name, col, want, opts=None, exact=()):
    return dict(name=name, col=col, opts=dict(O, **(opts or {})), want=want, exact=set(exact))


def cases():
    c = []
    c.append(case("base", column(), R(10, 10, 25, 2, MIN)))
    # the list size around lc_kf_max_dist (4): 3, 4 (not sorted) and 5 listed keyframes
    c.append(case("listed_3", column(kf=8), R(-1, -1, 3, 0, NAN)))
    c.append(case("listed_4", column(kf=9), R(-1, -1, 4, 0, NAN)))
    c.append(case("listed_5", column(kf=10, vals={0: F(0.9), 1: F(0.8), 2: F(0.7)}), R(0, 0, 5, 2, float(F(0.30)))))
    # kf_idx <= lc_kf_dist: nothing listed
    c.append(case("kf_at_dist", column(kf=5), R(-1, -1, 0, 0, NAN)))
    c.append(case("kf_below_dist", column(kf=2), R(-1, -1, 0, 0, NAN)))
    c.append(case("kf_0", column(kf=0), R(-1, -1, 0, 0, NAN)))
    # the minimum score chosen by covisibility: covis 10 (= min_lm_cov_graph) qualifies, 9 does not
    c.append(case("min_by_covis", column(vals={15: F(0.20), 16: F(0.10)}, covis={15: 10, 16: 9}),
                  R(10, 10, 25, 2, float(F(0.20)))))
    # chosen by distance: kf_idx - i = 4 (= min_kf_local_map + 3) qualifies, 5 does not
    c.append(case("min_by_distance", column(vals={26: F(0.28), 25: F(0.02)}), R(10, 10, 25, 2, float(F(0.28)))))
    # 0.001: the float just above it is taken, the float just below is not
    c.append(case("min_0001_above", column(vals={27: F(0.001)}), R(10, 10, 25, 8, float(F(0.001))), exact=(27,)))
    c.append(case("min_0001_below", column(vals={27: below(0.001)}), R(10, 10, 25, 2, MIN), exact=(27,)))
    # no qualifying score in (0.001, 1): lc_min_score stays 1.0
    c.append(case("min_stays_one", column(vals={26: F(1.0), 27: F(0.0), 28: F(-0.2), 29: F(1.5)}), R(-1, 10, 25, 0, 1.0),
                  exact=(26,)))
    # the best score just below, equal to and above lc_min_score
    c.append(case("max_below_min", column(vals={10: below(0.30), 8: F(0.01), 12: F(0.01)}), R(-1, 10, 25, 0, MIN),
                  exact=(10,)))
    c.append(case("max_equal_min", column(vals={10: F(0.30), 8: F(0.25), 12: F(0.25)}), R(10, 10, 25, 2, MIN),
                  exact=(10,)))
    c.append(case("max_above_min", column(vals={10: above(0.30), 8: F(0.25), 12: F(0.25)}), R(10, 10, 25, 2, MIN),
                  exact=(10,)))
    # Nkf_closest at lc_nkf_closest - 1 and at lc_nkf_closest; a supporter 5 away from the best does not count
    c.append(case("closest_one_short", column(vals={12: F(0.06)}), R(-1, 10, 25, 1, MIN)))
    c.append(case("closest_far", column(vals={12: F(0.06), 15: F(0.5)}), R(-1, 10, 25, 1, MIN)))
    c.append(case("closest_at_4", column(vals={12: F(0.06), 14: F(0.5)}), R(10, 10, 25, 2, MIN)))
    # the 0.8 product at equality: 0.625 * 0.8 is 0.5 in double, and 0.5f counts while the float below it does not
    c.append(case("product_equal", column(vals={26: F(0.625), 27: F(0.7), 28: F(0.7), 29: F(0.7), 10: F(0.9),
                                               8: F(0.5), 12: F(0.5)}), R(10, 10, 25, 2, 0.625), exact=(8, 12, 26)))
    c.append(case("product_below", column(vals={26: F(0.625), 27: F(0.7), 28: F(0.7), 29: F(0.7), 10: F(0.9),
                                               8: F(0.5), 12: below(0.5)}), R(-1, 10, 25, 1, 0.625),
                  exact=(8, 12, 26)))
    # ties at the maximum: the lowest index is best (20 is its tie, 22 supports only 20)
    c.append(case("tie_two", column(vals={20: F(0.60), 22: F(0.5)}), R(10, 10, 25, 2, MIN), exact=(10, 20)))
    c.append(case("tie_low_first", column(vals={14: F(0.60), 8: F(0.06), 12: F(0.06), 18: F(0.5)}),
                  R(-1, 10, 25, 1, MIN), exact=(10, 14)))
    c.append(case("tie_zero_signs", column(filler=False, kf=30, vals={i: F(-0.0) if i % 2 else F(0.0) for i in range(31)}),
                  R(-1, 0, 25, 0, 1.0), exact=tuple(range(31))))
    # negative options keep C++'s conversions
    c.append(case("neg_max_dist", column(), R(-1, -1, 25, 0, NAN), opts=dict(lc_kf_max_dist=-1)))
    c.append(case("neg_cov_graph", column(vals={15: F(0.20), 16: F(0.10)}, covis={15: 0xFFFFFFFF, 16: 0x7FFFFFFF}),
                  R(10, 10, 25, 2, float(F(0.20))), opts=dict(min_lm_cov_graph=-1)))
    c.append(case("zero_cov_graph", column(), R(10, 10, 25, 8, float(F(0.05))), opts=dict(min_lm_cov_graph=0)))
    c.append(case("neg_kf_dist", column(), R(30, 30, 31, 4, MIN), opts=dict(lc_kf_dist=-3)))
    c.append(case("neg_local_map", column(), R(-1, 10, 25, 0, 1.0), opts=dict(min_kf_local_map=-4)))
    c.append(case("neg_nkf_closest", column(vals={8: F(0.06), 12: F(0.06)}), R(10, 10, 25, 0, MIN),
                  opts=dict(lc_nkf_closest=-1)))
    # erased keyframes: a dead best is not listed, a dead local entry counts as 0
    c.append(case("erased_best", column(vals={10: F(0.99)}, dead=(10, 26)), R(-1, 8, 24, 0, float(F(0.35))), exact=(8, 12)))
    c.append(case("erased_support", column(dead=(8,)), R(-1, 10, 24, 1, MIN)))
    # a NaN column (PL with one feature, no feature or zero dispersion): no candidate, lc_min_score 1.0, best index 0
    c.append(case("nan_column", column(filler=False), R(-1, 0, 25, 0, 1.0)))
    # NaN among numbers (only reachable here): NaN ranks below every number and never supports
    c.append(case("nan_mixed", column(vals={3: F(NAN), 11: F(NAN), 27: F(NAN)}), R(10, 10, 25, 2, MIN)))
    # the reference's defaults on a 200-keyframe column
    col = column(kf=200, filler=False)
    col["conf"][:] = np.float32(0.05) + np.arange(201, dtype=np.float32) * np.float32(1e-4)
    col["conf"][194:200] = F(0.30)
    col["conf"][40], col["conf"][[20, 60, 70, 89]] = F(0.8), F(0.3)
    col["conf"][91] = F(0.3)
    c.append(case("defaults", col, R(40, 40, 150, 4, MIN), opts=dict(DEFAULTS_OPTS), exact=(20, 60, 70, 89, 91)))
    return c


DEFAULTS_OPTS = dict(lc_kf_dist=50, lc_kf_max_dist=50, lc_nkf_closest=4, min_lm_cov_graph=75, min_kf_local_map=3)
