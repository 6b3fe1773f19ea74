"""CPU checks of the global-bundle-adjustment restatement (oracle/gba.py; MapHandler::levMarquardtOptimizationGBA,
src/mapHandler.cpp:2101-2699) and of the map generator synth.gba_problem."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, gba
from plslam_b200 import synth

CAM = plf.KITTI_CAMERA


def _rel(a, b, p):
    out = 0.0
    for k in ("kf_pose", "pt", "ls"):
        if a[k].size:
            out = max(out, np.abs(a[k] - b[k]).max() / max(np.abs(b[k] - p[k]).max(), 1e-300))
    return out


@pytest.mark.parametrize("seed,kw", [(1, {}), (2, dict(n_kf=8, n_fixed=3, n_pt=400, n_ls=120)), (3, dict(n_ls=0)),
                                     (4, dict(n_pt=0, n_ls=60)), (6, dict(n_fixed=0, n_kf=6))])
def test_first_step_equals_the_local_ba_oracle(seed, kw):
    """With the intent of every quirk and one step, GBA and LBA are the same algebra: oracle/gba.py (sparse, splu) equals
    oracle/lba.c (dense LDL^T) to 1e-9 of the step."""
    p = synth.lba_problem(CAM, seed=seed, **kw)
    a = clib.local_ba(CAM, p, clib.lba_opts(ref_quirks=0, max_iters=1))
    b = gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=1))
    assert _rel(b, a, p) <= 1e-9
    assert a["iters"] == b["iters"] == 1
    assert abs(a["lambda_"] - b["lambda_"]) <= 1e-12 * a["lambda_"] and abs(a["err"] - b["err"]) <= 1e-12 * a["err"]


def test_sparse_lower_triangle_solve_equals_a_dense_solve():
    p = synth.gba_problem(CAM, n_kf=6, pts_per_kf=8, ls_per_kf=3, seed=3)
    X = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    for first, quirks in ((True, True), (True, False), (False, True), (False, False)):
        Hl, g, _ = gba.normal_equations(CAM, p, X, T0inv, first, quirks, 1e-7)
        assert (abs(Hl - gba.sp.tril(Hl))).sum() == 0        # only the lower triangle is assembled
        Hd = np.tril(Hl.toarray())
        Hd = Hd + np.tril(Hd, -1).T
        Hd += np.diag(0.1 * np.diag(Hd))
        Hs = gba.sp.csc_matrix(np.tril(Hd))
        want, got = np.linalg.solve(Hd, g), gba.solve_lower(Hs, g)
        assert np.abs(Hd @ got - g).max() <= 1e-10 * np.abs(g).max()
        if not quirks:   # (g4) makes the line blocks of the iterations near-singular: compare residuals only
            assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()


def test_g1_first_error_divides_by_zero_counters():
    p = synth.gba_problem(CAM, n_kf=5, pts_per_kf=10, ls_per_kf=3, seed=4)
    a = gba.global_ba(CAM, p, gba.opts(ref_quirks=1, max_iters=1))
    b = gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=1))
    assert a["err"] == np.inf and np.isfinite(b["err"]) and b["err"] > 0


def test_g2_int_maximum():
    # the scan as written: truncation, below 1 -> 0, >= 2^31 -> INT_MIN replaced by the next entry
    assert gba.hmax_int([0.3, 0.7]) == 0.0
    assert gba.hmax_int([3.7, 3.2, 0.5]) == 3.0
    assert gba.hmax_int([5.5, 3e9, 2.2, 1.9]) == 2.0
    assert gba.hmax_int([5.5, 3e9]) == float(gba.INT_MIN)
    assert gba.hmax_int([3e9, 7.9, 4e9, 1.5]) == 1.0
    nan = float("nan")
    assert gba.hmax_int([3e9, nan, nan]) == float(gba.INT_MIN)   # a NaN entry never replaces the int (comparisons false)
    assert gba.hmax_int([2.5, nan, 3e9, nan, 1.5]) == 1.0
    assert gba.hmax_int([nan, 0.5]) == 0.0
    assert gba.cvttsd2si(2147483647.9) == 2147483647 and gba.cvttsd2si(2147483648.0) == gba.INT_MIN
    # end to end, maximum below 1: lambda = 0, an undamped first step
    p = g2_small_problem()
    a = gba.global_ba(CAM, p, gba.opts(ref_quirks=1, max_iters=1))
    b = gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=1))
    assert a["lambda_"] == 0.0 and 0.0 < b["lambda_"] < 1e-5
    # end to end, beyond 2^31: the last diagonal entry decides (INT_MIN), a negative lambda
    q = g2_big_problem()
    a = gba.global_ba(g2_big_cam(), q, gba.opts(ref_quirks=1, max_iters=1))
    b = gba.global_ba(g2_big_cam(), q, gba.opts(ref_quirks=0, max_iters=1))
    assert a["lambda_"] == 1e-5 * gba.INT_MIN and b["lambda_"] > 1e-5 * 2.0 ** 31


def g2_small_problem():
    """observations 1e4 px off: Cauchy weights ~1e-8 put every diagonal entry below 1"""
    return synth.lba_problem(CAM, seed=5, n_kf=3, n_fixed=1, n_pt=40, n_ls=0, px_noise=1e4)


def g2_big_cam():
    return dict(CAM, fx=1e6, fy=1e6)


def g2_big_problem():
    """one fixed keyframe at the origin, two points observed 1e-3 px off: the last diagonal entry (the second point's
    z) is about 5e9 > 2^31"""
    cam = g2_big_cam()
    pt = np.array([[0.2, 0.1, 8.0], [8.0, 4.0, 10.0]])
    xy = np.stack([cam["cx"] + cam["fx"] * pt[:, 0] / pt[:, 2] + 1e-3, cam["cy"] + cam["fy"] * pt[:, 1] / pt[:, 2] + 2e-3], 1)
    return dict(kf_pose=np.zeros((0, 6)), pt=pt, ls=np.zeros((0, 6)), fixed_T=np.eye(4)[None],
                pt_obs_lm=np.array([0, 1], np.int32), pt_obs_kf=np.array([-1, -1], np.int32), pt_obs_xy=xy,
                ls_obs_lm=np.zeros(0, np.int32), ls_obs_kf=np.zeros(0, np.int32), ls_obs_le=np.zeros((0, 3)))


def test_g3_iterations_never_stop_on_the_error():
    p = synth.gba_problem(CAM, n_kf=6, pts_per_kf=12, ls_per_kf=0, seed=6, pose_noise=1e-4, lm_noise=1e-4, px_noise=0.05)
    # a min_error no error is below: the intent stops at the first test, the as-written err (+inf) never does
    a = gba.global_ba(CAM, p, gba.opts(ref_quirks=1, max_iters=6, min_error=1e10))
    b = gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=6, min_error=1e10))
    first = gba.global_ba(CAM, p, gba.opts(ref_quirks=1, max_iters=1))
    assert a["err"] == np.inf and np.isfinite(b["err"])
    assert a["iters"] == 6 and b["iters"] == 1
    # every step applied with lambda *= lambda_k
    assert a["lambda_"] == pytest.approx(first["lambda_"] * 10.0 ** 5, rel=1e-12)


def _line_map(seed=7):
    return synth.gba_problem(CAM, n_kf=4, pts_per_kf=0, ls_per_kf=6, seed=seed)


def test_g4_line_rows_read_one_block_at_stride_3():
    p = _line_map()
    nkf, nls = len(p["kf_pose"]), len(p["ls"])
    X = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Hq, gq, eq = gba.normal_equations(CAM, p, X, T0inv, False, True, 1e-7)
    # as written == the intent on a map whose line l has both end points at X[base + 3 l]
    Xs = X.copy()
    base = 6 * nkf
    for l in range(nls):
        Xs[base + 6 * l:base + 6 * l + 3] = Xs[base + 6 * l + 3:base + 6 * l + 6] = X[base + 3 * l:base + 3 * l + 3]
    Hi, gi, ei = gba.normal_equations(CAM, p, Xs, T0inv, False, False, 1e-7)
    assert abs(Hq - Hi).max() == 0 and np.array_equal(gq, gi) and eq == ei
    Hn, _, _ = gba.normal_equations(CAM, p, X, T0inv, False, False, 1e-7)
    assert abs(Hq - Hn).max() > 0


def test_g5_line_rows_take_the_map_pose():
    p = _line_map(8)
    X = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Xm = X.copy()
    Xm[:6 * len(p["kf_pose"])] += 0.01          # the optimised poses moved away from the map
    Hq, gq, _ = gba.normal_equations(CAM, p, Xm, T0inv, False, True, 1e-7)
    Hq0, gq0, _ = gba.normal_equations(CAM, p, X, T0inv, False, True, 1e-7)
    assert abs(Hq - Hq0).max() == 0 and np.array_equal(gq, gq0)     # as written: X's poses are not read
    Hi, _, _ = gba.normal_equations(CAM, p, Xm, T0inv, False, False, 1e-7)
    Hi0, _, _ = gba.normal_equations(CAM, p, X, T0inv, False, False, 1e-7)
    assert abs(Hi - Hi0).max() > 0


def test_g6_first_pass_line_coupling_is_transposed():
    p = synth.lba_problem(CAM, seed=9, n_kf=1, n_fixed=0, n_pt=0, n_ls=1)   # one keyframe, one line, one observation
    assert len(p["ls_obs_lm"]) == 1 and p["ls_obs_kf"][0] == 0
    X = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Hq, gq, _ = gba.normal_equations(CAM, p, X, T0inv, True, True, 1e-7)
    Hi, gi, _ = gba.normal_equations(CAM, p, X, T0inv, True, False, 1e-7)
    Hq, Hi = Hq.toarray(), Hi.toarray()
    assert np.array_equal(Hq[:6, :6], Hi[:6, :6]) and np.array_equal(Hq[6:, 6:], Hi[6:, 6:]) and np.array_equal(gq, gi)
    assert np.allclose(Hq[6:, :6], Hi[6:, :6].T, rtol=1e-14, atol=0) and not np.allclose(Hq[6:, :6], Hi[6:, :6])
    # the LM iterations write the coupling correctly (at X = the map, their rows are the first pass's)
    assert np.array_equal(gba.normal_equations(CAM, p, X, T0inv, False, False, 1e-7)[0].toarray(), Hi)
    a = gba.global_ba(CAM, p, gba.opts(ref_quirks=1, max_iters=1))
    b = gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=1))
    assert not np.allclose(a["kf_pose"], b["kf_pose"], rtol=1e-9, atol=0)


def test_generator():
    a = synth.gba_problem(CAM, n_kf=300, pts_per_kf=20, ls_per_kf=4, seed=11)
    b = synth.gba_problem(CAM, n_kf=300, pts_per_kf=20, ls_per_kf=4, seed=11)
    for k in a:
        if k != "truth":
            assert np.array_equal(a[k], b[k]), k
    n_tot = 301
    for kind, n in (("pt", len(a["pt"])), ("ls", len(a["ls"]))):
        lm, kf = a[kind + "_obs_lm"], a[kind + "_obs_kf"]
        assert np.all(np.diff(lm) >= 0)                          # grouped, ascending
        assert np.array_equal(np.unique(lm), np.arange(n))       # every landmark observed
        assert kf.min() >= -1 and kf.max() < 300
        creator = np.arange(n) // (20 if kind == "pt" else 4)
        late = kf >= 300 - 3
        assert np.any(late & (creator[lm] < 3)), kind            # the loop closure: late keyframes, early landmarks
    assert len(a["fixed_T"]) == 1 and len(a["kf_pose"]) == n_tot - 1
