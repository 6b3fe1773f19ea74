"""CPU tests: the C restatement of the Gauss-Newton pose refinement (src/mapHandler.cpp:3566-3957) —
se(3) identities, QR solve, convergence to a planted pose."""
import numpy as np
import pytest

from oracle import clib, synth

CAM = dict(width=1242, height=375, fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, b=0.537165719)


def test_se3_roundtrip_and_inverse():
    rng = np.random.default_rng(0)
    for _ in range(50):
        x = np.concatenate([rng.normal(0, 2, 3), rng.normal(0, 0.8, 3)])
        T = clib.expmap_se3(x)
        assert np.allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3), atol=1e-12)
        assert np.allclose(clib.logmap_se3(T), x, atol=1e-9)
        assert np.allclose(clib.inverse_se3(T) @ T, np.eye(4), atol=1e-12)
    assert np.allclose(clib.expmap_se3(np.zeros(6)), np.eye(4))
    assert np.allclose(clib.logmap_se3(np.eye(4)), 0)
    # small-angle branch (theta < 1e-6): R = I, t passes through
    T = clib.expmap_se3([1, 2, 3, 1e-8, 0, 0])
    assert np.allclose(T[:3, 3], [1, 2, 3]) and np.allclose(T[:3, :3], np.eye(3))


def test_colpiv_qr_matches_numpy():
    rng = np.random.default_rng(1)
    for _ in range(20):
        J = rng.normal(size=(40, 6)); H = J.T @ J; g = rng.normal(size=6)
        assert np.allclose(clib.colpiv_qr_solve6(H, g), np.linalg.solve(H, g), rtol=1e-9, atol=1e-10)
    # rank-deficient: solution lives in the well-determined subspace, zeros elsewhere (Eigen semantics)
    H = np.diag([4.0, 3.0, 2.0, 0, 0, 0]); g = np.array([4.0, 6.0, 2.0, 0, 0, 0])
    assert np.allclose(clib.colpiv_qr_solve6(H, g), [1, 2, 1, 0, 0, 0])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_converges_to_planted_pose(seed):
    pr = synth.gn_problem(CAM, seed=seed, px_noise=0.0, outlier_frac=0.0)
    r = clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"],
                     opts=clib.gn_opts(max_iters=20, max_iters_ref=20, eps_err=1e-16, eps_change=1e-16))
    assert np.allclose(r["T"], pr["T_true"], atol=5e-6)
    assert r["n_inliers"] == (300, 80)


def test_outliers_are_gated():
    pr = synth.gn_problem(CAM, seed=5, px_noise=0.3, outlier_frac=0.1)
    r = clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"], opts=clib.gn_opts(max_iters=10, max_iters_ref=20))
    assert np.linalg.norm(r["x"] - pr["x_true"]) < 2e-2
    assert r["inlier_pt"][:30].sum() <= 3 and r["inlier_pt"][30:].mean() > 0.95   # planted outliers removed


def test_degenerate_inputs():
    r = clib.gn_pose(CAM, np.zeros((0, 3)), np.zeros((0, 2)), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
    assert np.allclose(r["T"], np.eye(4)) and r["n_inliers"] == (0, 0)


@pytest.mark.parametrize("cfg", [dict(max_iters=5, max_iters_ref=10), dict(max_iters=100, max_iters_ref=100),
                                 dict(max_iters=100, max_iters_ref=100, eps_change=1e-2),
                                 dict(max_iters=20, max_iters_ref=20, eps_step=1e-3),
                                 dict(max_iters=0, max_iters_ref=1), dict(max_iters=1, max_iters_ref=0)])
@pytest.mark.parametrize("exact", [False, True])
def test_stop_trace_consistent_with_result(cfg, exact):
    """orc_gn_pose_trace: one record per accumulation, in stage order; a stage's iteration count is its records
    minus the one the error test stopped without a step; the stage's exit reason is its last record's (max_iters when
    it ran none); the change test compares each error with the last one that took a step; the last error is err; and
    the trace does not change the result."""
    pr = synth.gn_problem(CAM, seed=9, **(dict(px_noise=0.0, outlier_frac=0.0) if exact else {}))
    o = clib.gn_opts(**cfg)
    r = clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"], opts=o, trace=True)
    plain = clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"], opts=o)
    for k in ("T", "cov", "x", "inlier_pt", "inlier_ls"):
        assert np.array_equal(r[k], plain[k], equal_nan=True), k
    assert r["iters"] == plain["iters"] and r["n_inliers"] == plain["n_inliers"]
    rec, exits = r["trace"]["rec"], r["trace"]["exit"]
    assert np.all(np.diff(rec["stage"]) >= 0)
    e_prev = clib.GN_ERR_PREV0
    for s in (0, 1):
        st = rec[rec["stage"] == s]
        assert len(st) <= (o.max_iters, o.max_iters_ref)[s]
        assert r["iters"][s] == len(st) - (exits[s] == clib.GN_EXIT_ERROR)
        assert exits[s] == (st["exit"][-1] if len(st) else clib.GN_EXIT_MAXIT)
        assert np.all(st["exit"][:-1] == clib.GN_CONTINUE)
        for t in st:
            assert t["e_prev"] == e_prev
            took_step = t["exit"] != clib.GN_EXIT_ERROR
            assert (t["step"] >= 0) == took_step
            if t["exit"] == clib.GN_EXIT_ERROR:
                assert abs(t["e"] - t["e_prev"]) < o.eps_change or t["e"] < o.eps_err
            if t["exit"] == clib.GN_EXIT_STEP:
                assert t["step"] < o.eps_step
            if t["exit"] in (clib.GN_CONTINUE, clib.GN_EXIT_MAXIT):
                e_prev = t["e"]
    if len(rec):
        assert rec["e"][-1] == r["err"]
