"""CPU checks of oracle/pgo.py, the restatement of g2o's pose-graph optimisation as MapHandler::
loopClosureOptimizationCovGraphG2O (src/mapHandler.cpp:4185-4410) uses it: the MQT maps, the Jacobians against central
differences, the initial guess's breadth-first search, the Levenberg-Marquardt schedule on scripted chi2 sequences, the
graph lists and write-back of the reference, and the optimisation itself on synthetic loops."""
import math

import numpy as np
import pytest

from oracle import pgo
from plslam_b200 import synth


def _rand_iso(rng, n):
    return synth._iso(synth._rodrigues(rng.uniform(-1.0, 1.0, (n, 3)) * 1.2), rng.standard_normal((n, 3)))


def test_mqt_round_trip_and_sign():
    rng = np.random.default_rng(0)
    T = _rand_iso(rng, 200)
    m = pgo.mqt(T)
    assert np.abs(pgo.inc(m) - T).max() < 1e-14
    assert np.all(pgo.quat(T)[:, 0] >= 0.0)
    # a rotation by more than pi about z: Eigen's quaternion has w < 0 there, MQT flips the sign
    Rz = synth._rodrigues([[0.0, 0.0, 0.9 * math.pi]])[0]
    q = pgo.quat(synth._iso(Rz[None], np.zeros((1, 3))))[0]
    assert q[0] >= 0.0 and q[3] == pytest.approx(math.sin(0.45 * math.pi))
    # every branch of the trace test: trace > 0 and each largest diagonal entry
    for w in ([0.1, 0.2, 0.3], [3.0, 0.1, 0.0], [0.0, 3.0, 0.1], [0.1, 0.0, 3.0]):
        T1 = synth._iso(synth._rodrigues([w]), np.zeros((1, 3)))
        assert np.abs(pgo.inc(pgo.mqt(T1)) - T1).max() < 1e-14


def test_increment_beyond_the_unit_ball_is_the_identity_rotation():
    d = np.array([0.5, -1.0, 2.0, 0.8, 0.5, 0.4])   # |d_q|^2 = 1.05
    T = pgo.inc(d)
    assert np.array_equal(T[:3, :3], np.eye(3)) and np.array_equal(T[:3, 3], d[:3])
    X = _rand_iso(np.random.default_rng(1), 1)[0]
    assert np.array_equal(pgo.oplus(X, d), pgo.iso_mul(X, T))


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(2)
    Xi, Xj = _rand_iso(rng, 50), _rand_iso(rng, 50)
    Z = pgo.iso_mul(pgo.iso_mul(pgo.iso_inv(Xi), Xj), synth._iso(
        synth._rodrigues(0.3 * rng.standard_normal((50, 3))), 0.3 * rng.standard_normal((50, 3))))
    w = pgo.quat(pgo.iso_mul(pgo.iso_inv(Z), pgo.iso_mul(pgo.iso_inv(Xi), Xj)))[:, 0]
    keep = w > 0.2   # away from w = 0, where the sign normalisation makes the error discontinuous
    Xi, Xj, Z = Xi[keep], Xj[keep], Z[keep]
    e, Ji, Jj = pgo.jacobians(Xi, Xj, Z)
    assert np.abs(e - pgo.error(Xi, Xj, Z)).max() == 0.0
    h = 1e-6
    for k in range(6):
        d = np.zeros(6); d[k] = h
        ni = (pgo.error(pgo.oplus(Xi, d), Xj, Z) - pgo.error(pgo.oplus(Xi, -d), Xj, Z)) / (2 * h)
        nj = (pgo.error(Xi, pgo.oplus(Xj, d), Z) - pgo.error(Xi, pgo.oplus(Xj, -d), Z)) / (2 * h)
        assert np.abs(ni - Ji[:, :, k]).max() < 1e-7, k
        assert np.abs(nj - Jj[:, :, k]).max() < 1e-7, k


def _prob(T, fixed, edges, Z):
    return (np.asarray(T, np.float64), np.asarray(fixed, bool), np.array([a for a, _ in edges]),
            np.array([b for _, b in edges]), np.asarray(Z, np.float64))


def test_initial_guess_on_a_tree():
    rng = np.random.default_rng(3)
    T, Z = _rand_iso(rng, 5), _rand_iso(rng, 4)
    # 0 (fixed) -> 1, 2 -> 1 (reached backwards, through Z^-1), 1 -> 3, 4 isolated
    X = pgo.initial_guess(*_prob(T, [1, 0, 0, 0, 0], [(0, 1), (2, 1), (1, 3)], Z[:3]))
    assert np.array_equal(X[0], T[0]) and np.array_equal(X[4], T[4])
    assert np.array_equal(X[1], pgo.iso_mul(T[0], Z[0]))
    assert np.array_equal(X[2], pgo.iso_mul(X[1], pgo.iso_inv(Z[1])))
    assert np.array_equal(X[3], pgo.iso_mul(X[1], Z[2]))


def test_initial_guess_tie_goes_to_the_edge_order():
    """a cycle 0 - 1 - 2 - 0: vertex 2 is one hop from 0 directly, so the direct edge sets it whatever its position;
    vertex 3, two hops away through 1 or through 2, takes the parent whose edge comes first in the order given"""
    rng = np.random.default_rng(4)
    T, Z = _rand_iso(rng, 4), _rand_iso(rng, 5)
    edges = [(0, 1), (1, 2), (2, 0), (1, 3), (2, 3)]
    X = pgo.initial_guess(*_prob(T, [1, 0, 0, 0], edges, Z))
    assert np.array_equal(X[2], pgo.iso_mul(T[0], pgo.iso_inv(Z[2])))
    assert np.array_equal(X[3], pgo.iso_mul(X[1], Z[3]))
    e2 = [edges[i] for i in (0, 1, 2, 4, 3)]
    X2 = pgo.initial_guess(*_prob(T, [1, 0, 0, 0], e2, Z[[0, 1, 2, 4, 3]]))
    assert np.array_equal(X2[3], pgo.iso_mul(X2[1], Z[3]))      # 1 is still popped before 2: its edge (1, 3) wins
    e3 = [(0, 2), (0, 1), (1, 2), (2, 3), (1, 3)]                 # now 2 is discovered and popped first
    X3 = pgo.initial_guess(*_prob(T, [1, 0, 0, 0], e3, Z))
    assert np.array_equal(X3[3], pgo.iso_mul(X3[2], Z[3]))


def test_initial_guess_leaves_fixed_and_unreachable_vertices():
    rng = np.random.default_rng(5)
    T, Z = _rand_iso(rng, 5), _rand_iso(rng, 4)
    # 0 and 2 fixed; 3 - 4 unreachable from both
    X = pgo.initial_guess(*_prob(T, [1, 0, 1, 0, 0], [(0, 1), (1, 2), (3, 4), (2, 0)], Z))
    assert np.array_equal(X[[0, 2, 3, 4]], T[[0, 2, 3, 4]])
    assert np.array_equal(X[1], pgo.iso_mul(T[0], Z[0]))


def _scripted(seq):
    """a trial function returning the scripted (chi_t, scale, ok) in turn"""
    it = iter(seq)
    return lambda lam: (*next(it), None)


def test_lambda_schedule_accept_clipped_and_unclipped():
    # rho = 1: alpha = 1 - 1 = 0 -> clipped to 1/3
    chi, lam, ni, trials, rho, _ = pgo.lm_trials(10.0, 1.0, 8, _scripted([(10.0 - (1.0 + 1e-3), 1.0, True)]))
    assert (trials, ni, chi) == (1, 2, 10.0 - 1.001) and rho == pytest.approx(1.0) and lam == pytest.approx(1.0 / 3.0)
    # rho = 0.5: alpha = 1 -> clipped to 2/3
    chi, lam, *_ = pgo.lm_trials(10.0, 1.0, 2, _scripted([(10.0 - 0.5 * 1.001, 1.0, True)]))
    assert lam == pytest.approx(2.0 / 3.0)
    # rho = 0.75: alpha = 1 - 0.125 = 0.875 -> 2/3;  rho = 0.9: alpha = 1 - 0.512 = 0.488, unclipped
    chi, lam, *_ = pgo.lm_trials(10.0, 1.0, 2, _scripted([(10.0 - 0.9 * 1.001, 1.0, True)]))
    assert lam == pytest.approx(1.0 - (2 * 0.9 - 1) ** 3)


def test_lambda_schedule_rejections():
    trace = []
    # two rejections (ni doubling), then an acceptance
    seq = [(11.0, 1.0, True), (12.0, 1.0, True), (9.0, 1.0, True)]
    chi, lam, ni, trials, rho, _ = pgo.lm_trials(10.0, 1.0, 2, _scripted(seq), 0, trace)
    assert trials == 3 and [t["lambda_"] for t in trace] == [1.0, 2.0, 8.0] and ni == 2 and chi == 9.0
    assert [t["accepted"] for t in trace] == [0, 0, 1]
    # ten rejections
    chi, lam, ni, trials, rho, _ = pgo.lm_trials(10.0, 1.0, 2, _scripted([(11.0, 1.0, True)] * 10))
    assert trials == 10 and lam == 2.0 ** sum(range(1, 11)) and pgo.stop_reason(trials, rho, lam) == "trials"
    # rho == 0: rejected, lambda doubled, the iteration ends and so does the optimisation
    chi, lam, ni, trials, rho, _ = pgo.lm_trials(0.0, 1e-10, 2, _scripted([(0.0, 0.0, True)]))
    assert (trials, rho, lam, ni) == (1, 0.0, 2e-10, 4) and pgo.stop_reason(trials, rho, lam) == "rho_zero"
    # a NaN chi2: rejected, and rho < 0 is false, so the trials end and the next iteration follows
    chi, lam, ni, trials, rho, st = pgo.lm_trials(10.0, 1.0, 2, _scripted([(float("nan"), 1.0, True)]))
    assert trials == 1 and math.isnan(rho) and lam == 2.0 and st is None and pgo.stop_reason(trials, rho, lam) is None
    # a failed solve counts as chi_t = DBL_MAX
    trace = []
    pgo.lm_trials(10.0, 1.0, 2, _scripted([(5.0, 1.0, False), (5.0, 1.0, True)]), 0, trace)
    assert trace[0]["chi_t"] == pgo.DBL_MAX and trace[0]["accepted"] == 0 and trace[1]["accepted"] == 1
    # lambda overflowing ends the optimisation
    assert pgo.stop_reason(3, 0.5, float("inf")) == "lambda"


def test_cov_graph_lists():
    rng = np.random.default_rng(6)
    n = 10
    live = np.ones(n, bool)
    live[[3, 6]] = False                               # erased keyframes
    T = _rand_iso(rng, n)
    fg = np.zeros((n, n), int)
    fg[0, 5] = 75                                      # >= minLMCovGraph: an edge
    fg[1, 7] = 74                                      # below both: none
    fg[2, 4] = 200                                     # >= minLMEssGraph
    fg[4, 9] = 500                                     # beyond kf_curr_idx = 8: none
    lc_idx = [(1, 8, 1), (0, 7, 1)]
    lc_pose = [rng.standard_normal(6) * 0.1 for _ in lc_idx]
    g = pgo.cov_graph_lists(fg, live, T, lc_idx, lc_pose)
    assert g["kf_list"] == [0, 1, 2, 4, 5, 7, 8]
    kf = g["kf_list"]
    pairs = [(kf[a], kf[b]) for a, b in zip(g["from"], g["to"])]
    # |i - j| == 1 on raw indices only: (2, 4) and (5, 7) are not neighbours, (2, 4) comes from the full graph
    assert pairs == [(0, 1), (0, 5), (1, 2), (2, 4), (4, 5), (7, 8), (1, 8), (0, 7)]
    assert np.array_equal(g["fixed"], [1, 0, 0, 0, 0, 0, 0]) and np.array_equal(g["T"], T[kf])
    assert np.allclose(g["Z"][0], np.linalg.inv(T[0]) @ T[1], atol=1e-12)
    from oracle import clib
    assert np.array_equal(g["Z"][-1], clib.expmap_se3(lc_pose[1]))


def test_cov_graph_write_back():
    rng = np.random.default_rng(7)
    n = 6
    T = _rand_iso(rng, n)
    live = np.ones(n, bool)
    kf_list = [0, 1, 3]
    live[2] = False
    T_opt = _rand_iso(rng, 3)
    mk = lambda: dict(point3D=rng.standard_normal(3), med_obs_dir=rng.standard_normal(3), dir_list=rng.standard_normal((2, 3)))
    points = [mk(), None, mk(), mk()]
    lines = [dict(line3D=rng.standard_normal(6), med_obs_dir=rng.standard_normal(3), dir_list=rng.standard_normal((1, 3)))]
    pkf = [[0], [1], [], [2], [], [3]]
    lkf = [[], [], [], [], [0], []]
    T2, P2, L2 = pgo.cov_graph_write_back(T, live, kf_list, T_opt, points, lines, pkf, lkf)
    assert np.array_equal(T2[kf_list], T_opt) and P2[1] is None
    C0 = T_opt[0] @ np.linalg.inv(T[0])
    assert np.allclose(P2[0]["point3D"], C0[:3, :3] @ points[0]["point3D"] + C0[:3, 3])
    assert np.allclose(P2[0]["dir_list"][1], C0[:3, :3] @ points[0]["dir_list"][1] + C0[:3, 3])   # translated too
    C = T_opt[2] @ pgo.iso_inv(T[3])                   # the last correction moves keyframes 4, 5 and their landmarks
    assert np.allclose(T2[4], C @ T[4]) and np.allclose(T2[5], C @ T[5])
    assert np.allclose(P2[3]["med_obs_dir"], C[:3, :3] @ points[3]["med_obs_dir"] + C[:3, 3])
    assert np.allclose(L2[0]["line3D"][3:], C[:3, :3] @ lines[0]["line3D"][3:] + C[:3, 3])
    live[5] = False
    with pytest.raises(ValueError):
        pgo.cov_graph_write_back(T, live, kf_list, T_opt, points, lines, pkf, lkf)


def test_optimize_dense_and_sparse_agree_and_close_the_loop():
    p = synth.pose_graph_problem(25, 5, 3, drift=0.02, seed=8)
    d = pgo.optimize(p, solver="dense")
    s = pgo.optimize(p, solver="sparse")
    sc = np.abs(d["T"]).max()
    assert np.abs(d["T"] - s["T"]).max() <= 1e-9 * sc and d["chi2"] == pytest.approx(s["chi2"], rel=1e-6)
    err = lambda T: np.linalg.norm(T[:, :3, 3] - p["T_true"][:, :3, 3], axis=1).max()
    assert err(d["T"]) < 0.5 * err(p["T"])
    assert d["chi2"] < 0.1 * d["chi2_init"]


@pytest.mark.parametrize("n_kf,window,n_lc", [(12, 5, 1), (101, 5, 1), (684, 5, 4)])
def test_spread_under_a_permutation_of_the_edges(n_kf, window, n_lc):
    """the oracle's own spread: the same start, the edges in another order (the sums of H, b and chi2 reorder).  The
    GPU tests compare final poses at 100 times 1e-8 (tests/test_pgo_gpu.py: TOL = 1e-6)"""
    p = synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=n_kf)
    T0, fixed, frm, to, Z = pgo._arrays(p)
    X0 = pgo.initial_guess(T0, fixed, frm, to, Z)
    a = pgo.optimize(dict(p, T=X0), guess=False)
    perm = np.random.default_rng(1).permutation(len(frm))
    b = pgo.optimize({"T": X0, "fixed": fixed, "from": frm[perm], "to": to[perm], "Z": Z[perm]}, guess=False)
    spread = np.abs(a["T"] - b["T"]).max() / np.abs(a["T"]).max()
    print(f"oracle spread under an edge permutation, {n_kf} keyframes: {spread:.2e}")
    assert spread <= 1e-8


@pytest.mark.parametrize("n_kf,window,n_lc", [(684, 5, 4), (684, 1, 1)])
def test_spread_under_another_elimination_order(n_kf, window, n_lc):
    """the oracle's own spread when only splu's column ordering changes: the chains make H ill-conditioned, so the
    first steps' chi2_t and the final poses move beyond the summation-order spread above (at 2 049 keyframes, measured
    once: 5.8e-9 of the largest pose entry, 1e-8 of chi2 on a trial's chi2_t).  The GPU tests allow 100 times that
    (tests/test_pgo_gpu.py: TOL, TRIAL_TOL = 1e-6)"""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    p = synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=n_kf + window + n_lc)
    a = pgo.optimize(p)
    orig = pgo.solve

    def colamd(H, lam, b, solver="auto"):
        x = spla.splu((H + lam * sp.identity(H.shape[0], format="csc")).tocsc(), permc_spec="COLAMD").solve(b)
        return x, bool(np.all(np.isfinite(x)))
    try:
        pgo.solve = colamd
        b = pgo.optimize(p)
    finally:
        pgo.solve = orig
    spread = np.abs(a["T"] - b["T"]).max() / np.abs(a["T"]).max()
    trial = max(abs(x["chi_t"] - y["chi_t"]) / x["chi"] for x, y in zip(a["trace"][:3], b["trace"][:3]))
    print(f"oracle spread under another elimination order, {n_kf} keyframes: poses {spread:.2e}, chi2_t {trial:.2e}")
    assert spread <= 1e-8 and trial <= 1e-8
