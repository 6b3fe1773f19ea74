"""GPU parity of the loop-closure pose-graph optimisation (plf_pose_graph, csrc/pgo.cu) with the CPU restatement of
g2o's computeInitialGuess() + Levenberg-Marquardt in MapHandler::loopClosureOptimizationCovGraphG2O (oracle/pgo.py).

The tolerances are 100 times the oracle's own spread when only the order of its sums or of its sparse elimination
changes (tests/test_pgo_oracle.py): the long chains make H ill-conditioned, so the first Gauss-Newton steps from a poor
initial guess move chi2_t by up to 1e-8 of chi2, and the final poses by up to 5.8e-9 of the largest pose entry (2 049
keyframes).  The trace is compared trial by trial (decisions; chi2_t to TRIAL_TOL chi2) up to the first trial whose
|chi - chi_t| is within ROUNDING chi, whose decision is then left to rounding; the final poses are compared to TOL."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import pgo
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
TOL = 1e-6         # final poses, relative to the largest pose entry; final chi2, relative
TRIAL_TOL = 1e-6   # a trial's chi2_t, relative to its chi2
# |chi - chi_t| <= ROUNDING chi: the trial's decision is left to rounding.  1e-5 is ten times TRIAL_TOL and far above the
# measured chi2_t spread (1e-8 of chi2 in the oracle under another elimination order, 2e-7 at most between the device and
# the oracle), so every decision compared before that point is one both sides must take the same way.
ROUNDING = 1e-5
PLF_ERR_INVALID = -1
PLF_ERR_CAPACITY = -4

# (n_kf, window, loop edges): n_kf - 1 free vertices; 684 keyframes = n = 4098, not a multiple of the 64-wide tiles
CASES = [(3, 1, 0), (3, 5, 1), (12, 5, 1), (12, 1, 4), (65, 1, 4), (65, 5, 0), (101, 5, 1), (101, 1, 4), (684, 5, 4),
         (684, 1, 1), (1001, 1, 1), (1001, 5, 4), (2049, 5, 4)]


def _compare(got, ref):
    """trial-by-trial agreement up to the first rounding-decided trial; returns whether one was met"""
    tg, tr = got["trace"], ref["trace"]
    prev = None   # chi of the trial before: a trial's chi is an earlier chi_t
    for k in range(min(len(tg), len(tr))):
        a, b = tg[k], tr[k]
        # lambda follows rho = (chi - chi_t) / ...: a TRIAL_TOL difference in chi_t moves it by up to 0.1 ROUNDING chi / gap
        assert a["iter"] == b["iter"] and a["lambda_"] == pytest.approx(b["lambda_"], rel=1e-3), k
        assert a["chi"] == pytest.approx(b["chi"], rel=1e-9, abs=TRIAL_TOL * prev if prev else 1e-20), k
        if abs(b["chi"] - b["chi_t"]) <= ROUNDING * abs(b["chi"]) or abs(a["chi"] - a["chi_t"]) <= ROUNDING * abs(a["chi"]):
            return True
        assert bool(a["accepted"]) == bool(b["accepted"]), k
        assert a["chi_t"] == pytest.approx(b["chi_t"], rel=1e-9, abs=TRIAL_TOL * b["chi"]), k
        prev = b["chi"]
    assert len(tg) == len(tr)
    assert (got["iters"], got["stop"], got["trials"]) == (ref["iters"], ref["stop"], ref["trials"])
    assert got["lambda_"] == pytest.approx(ref["lambda_"], rel=1e-3)
    return False


def _final(p, got, ref):
    sc = max(1.0, np.abs(ref["T"]).max())
    assert np.abs(got["T"] - ref["T"]).max() <= TOL * sc
    assert got["chi2"] == pytest.approx(ref["chi2"], rel=TOL, abs=1e-20)
    assert got["chi2_init"] == pytest.approx(ref["chi2_init"], rel=1e-9, abs=1e-20)
    free = np.asarray(p["fixed"]) == 0
    assert np.array_equal(got["T"][~free], np.asarray(p["T"])[~free])   # fixed vertices are never written


@pytest.mark.parametrize("n_kf,window,n_lc", CASES)
def test_pose_graph_matches_the_oracle(fe, n_kf, window, n_lc):
    p = synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=n_kf + window + n_lc)
    ref = pgo.optimize(p)
    got = fe.pose_graph(p)
    rounding = _compare(got, ref)
    print(f"pgo parity n_kf={n_kf} window={window} n_lc={n_lc}: iters {got['iters']} / {ref['iters']}, trials "
          f"{got['trials']} / {ref['trials']}, ends in a rounding-decided trial: {rounding}")
    _final(p, got, ref)
    if n_lc and n_kf > 2 * window + 2:   # with loop edges the drifted trajectory is pulled back towards the truth
        err = lambda T: np.abs(T[:, :3, 3] - p["T_true"][:, :3, 3]).max()
        assert err(got["T"]) < err(p["T"])


@pytest.mark.parametrize("n_kf,window,n_lc", [(12, 5, 1), (684, 5, 4), (2049, 1, 4)])
def test_max_iters_0_gives_the_initial_guess(fe, n_kf, window, n_lc):
    p = synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=3)
    ref = pgo.optimize(p, max_iters=0)
    got = fe.pose_graph(p, max_iters=0)
    assert got["iters"] == 0 and got["trials"] == 0 and len(got["trace"]) == 0
    assert np.abs(got["T"] - ref["T"]).max() <= 1e-12 * max(1.0, np.abs(ref["T"]).max())
    assert got["chi2_init"] == got["chi2"] == pytest.approx(ref["chi2_init"], rel=1e-9, abs=1e-20)


def test_identity_graph_stops_on_rho_zero(fe):
    """e = 0 exactly: x = 0, chi_t = chi = 0, rho = 0: one iteration, one rejected trial, lambda doubled"""
    n = 6
    I = np.tile(np.eye(4), (n, 1, 1))
    frm = np.array([0, 1, 2, 3, 4, 0], np.int32)
    to = np.array([1, 2, 3, 4, 5, 5], np.int32)
    p = {"T": I, "fixed": np.eye(1, n, dtype=np.uint8)[0], "from": frm, "to": to, "Z": np.tile(np.eye(4), (len(frm), 1, 1))}
    got = fe.pose_graph(p)
    assert (got["iters"], got["stop"], got["trials"], got["chi2_init"], got["chi2"]) == (1, "rho_zero", 1, 0.0, 0.0)
    assert got["lambda_"] == 2e-10
    assert np.array_equal(got["T"], I)


def test_two_runs_are_bit_identical(fe):
    p = synth.pose_graph_problem(700, 5, 4, drift=0.01, seed=9)
    a, b = fe.pose_graph(p), fe.pose_graph(p)
    assert np.array_equal(a["T"], b["T"]) and np.array_equal(a["trace"], b["trace"])
    assert (a["chi2"], a["lambda_"], a["iters"], a["trials"]) == (b["chi2"], b["lambda_"], b["iters"], b["trials"])


def test_isolated_vertex_and_fixed_pair(fe):
    """a vertex without edges keeps its pose bit for bit; an edge between two fixed vertices adds to chi2 only"""
    p = synth.pose_graph_problem(30, 3, 1, drift=0.02, seed=4)
    rng = np.random.default_rng(0)
    lone = synth._iso(synth._rodrigues(rng.standard_normal((2, 3))), rng.standard_normal((2, 3)))
    T = np.concatenate([p["T"], lone])                         # vertex 30: no edges; vertex 31: fixed
    fixed = np.concatenate([p["fixed"], [0, 1]]).astype(np.uint8)
    Zf = synth._iso(synth._rodrigues([[0.1, 0.0, 0.0]]), [[0.0, 0.5, 0.0]])[0]   # inconsistent with T_0^-1 T_31
    q = {"T": T, "fixed": fixed, "from": np.append(p["from"], 0).astype(np.int32),
         "to": np.append(p["to"], 31).astype(np.int32), "Z": np.concatenate([p["Z"], Zf[None]])}
    ref = pgo.optimize(q)
    got = fe.pose_graph(q)
    _compare(got, ref)
    _final(q, got, ref)
    assert np.array_equal(got["T"][30], T[30]) and np.array_equal(got["T"][31], T[31])
    e = pgo.error(T[0], T[31], Zf)
    assert got["chi2"] >= float(e @ e)


def _raw(fe, p, null=None, max_iters=5):
    """plf_pose_graph through ctypes with explicit counts and pointers (NULL where named by `null`)"""
    keep = []

    def arr(k, dt, cols):
        a = np.ascontiguousarray(p[k], dt).reshape(-1, cols) if cols else np.ascontiguousarray(p[k], dt).ravel()
        keep.append(a)
        return None if k == null or not a.size else a.ctypes.data
    T = np.ascontiguousarray(p["T"], np.float64).reshape(-1, 16).copy()
    keep.append(T)
    prob = plf.plf_pgo_problem(len(T), len(np.ravel(p["from"])), None if null == "T" else T.ctypes.data,
                               arr("fixed", np.uint8, 0), arr("from", np.int32, 0), arr("to", np.int32, 0),
                               arr("Z", np.float64, 16))
    res = plf.plf_pgo_result()
    return fe.lib.plf_pose_graph(fe._ctx, C.byref(plf.plf_pgo_opts(max_iters, 1e-10)), C.byref(prob), C.byref(res))


def test_pose_graph_rejects_bad_input_and_stays_usable(fe):
    p = synth.pose_graph_problem(40, 3, 2, drift=0.01, seed=5)
    want = pgo.optimize(p)

    def valid():
        got = fe.pose_graph(p)
        _compare(got, want)
        _final(p, got, want)

    big = synth.pose_graph_problem(4098, 1, 0, drift=0.0, seed=1)   # 4097 free vertices: refused before allocating
    assert _raw(fe, big) == PLF_ERR_CAPACITY
    valid()
    for field in ("T", "fixed", "from", "to", "Z"):
        assert _raw(fe, p, null=field) == PLF_ERR_INVALID, field
        valid()
    bad = []
    f = p["from"].copy(); f[3] = len(p["T"])
    bad.append(("edge out of range", dict(p, **{"from": f})))
    f = p["from"].copy(); f[3] = -1
    bad.append(("negative vertex", dict(p, **{"from": f})))
    t = p["to"].copy(); t[5] = p["from"][5]
    bad.append(("self edge", dict(p, to=t)))
    T = p["T"].copy(); T[7, 1, 2] = np.nan
    bad.append(("NaN pose", dict(p, T=T)))
    Z = p["Z"].copy(); Z[2, 0, 3] = np.inf
    bad.append(("infinite measurement", dict(p, Z=Z)))
    T = np.concatenate([p["T"], p["T"][:2]])                         # two free vertices joined only to each other
    bad.append(("component without a fixed vertex", {
        "T": T, "fixed": np.concatenate([p["fixed"], [0, 0]]), "from": np.append(p["from"], 40).astype(np.int32),
        "to": np.append(p["to"], 41).astype(np.int32), "Z": np.concatenate([p["Z"], p["Z"][:1]])}))
    for name, q in bad:
        with pytest.raises(plf.PlfError):
            fe.pose_graph(q)
        valid()


# the first iterations from a poor initial guess: large chi2 decreases, no decision left to rounding, so the iteration
# and trial counts and the stop reason (max_iters) are compared exactly
@pytest.mark.parametrize("n_kf,window,n_lc,max_iters", [(101, 5, 1, 2), (684, 5, 4, 3), (1001, 1, 1, 3), (2049, 5, 4, 4)])
def test_first_iterations_match_exactly(fe, n_kf, window, n_lc, max_iters):
    p = synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=n_kf + window + n_lc)
    ref = pgo.optimize(p, max_iters=max_iters)
    got = fe.pose_graph(p, max_iters=max_iters)
    assert not _compare(got, ref)      # compares len(trace), iters, stop and trials exactly
    assert got["stop"] == "max_iters" and got["iters"] == max_iters
    _final(p, got, ref)


def test_failed_factorisation_counts_as_dbl_max_and_lambda_overflow_stops(fe):
    """an edge whose translation is 1e160 gives J_i entries of 2e160 and an infinite H (the inputs are finite): every
    pivot check fails, chi2_t is DBL_MAX and rho NaN, so each iteration is one rejected trial; lambda doubles more each
    time until it overflows at iteration 46 and the run stops on lambda.  The dense oracle (n = 6) takes the same path."""
    Z = np.eye(4)[None].copy()
    Z[0, 0, 3] = -1e160
    p = {"T": np.tile(np.eye(4), (2, 1, 1)), "fixed": np.array([1, 0], np.uint8), "from": np.array([1], np.int32),
         "to": np.array([0], np.int32), "Z": Z}
    ref = pgo.optimize(p)
    got = fe.pose_graph(p)
    assert (got["iters"], got["stop"], got["trials"]) == (ref["iters"], ref["stop"], ref["trials"]) == (46, "lambda", 46)
    assert got["lambda_"] == ref["lambda_"] == float("inf") and got["chi2"] == ref["chi2"] == 0.0
    tr = got["trace"]
    assert np.all(tr["chi_t"] == pgo.DBL_MAX) and not tr["accepted"].any() and np.all(np.isnan(tr["rho"]))
    assert np.array_equal(tr["lambda_"], [t["lambda_"] for t in ref["trace"]])
    assert np.array_equal(got["T"], ref["T"])   # never stepped: the initial guess


def test_lambda_init_must_be_positive_and_finite(fe):
    p = synth.pose_graph_problem(20, 3, 1, drift=0.01, seed=2)
    want = fe.pose_graph(p)
    for lam in (0.0, -1e-10, float("nan"), float("inf")):
        with pytest.raises(plf.PlfError, match="lambda_init"):
            fe.pose_graph(p, lambda_init=lam)
        again = fe.pose_graph(p)
        assert np.array_equal(again["T"], want["T"])


def test_scratch_bytes_reported(fe):
    p = synth.pose_graph_problem(300, 5, 2, drift=0.01, seed=3)
    r = fe.pose_graph(p, max_iters=1)
    nf, ne = 299, len(p["from"])
    assert 288 * nf * nf + 760 * ne <= r["scratch_bytes"] <= 288 * nf * nf + 900 * ne + 500 * 300 + 64 * 256 * 8 * 8


def _write_pgo_map(path, rng, n_tot=48, erased=(5, 17), lc=((2, 41), (8, 38))):
    """the map vo_demo --pgo-selftest reads (format in vo_demo.cpp); returns what cov_graph_lists / write-back take"""
    import struct
    from oracle import clib
    g = synth.pose_graph_problem(n_tot, 3, 0, drift=0.01, seed=int(rng.integers(1 << 30)))
    T, T_true = g["T"], g["T_true"]
    live = np.ones(n_tot, bool)
    live[list(erased)] = False
    fg = np.zeros((n_tot, n_tot), np.int32)
    for i in range(n_tot):
        for j in range(i + 1, min(i + 4, n_tot)):
            fg[i, j] = fg[j, i] = rng.integers(0, 200)
    fg[3, 20] = fg[20, 3] = 90                                   # a long covisibility edge
    lc_pose = [clib.logmap_se3(np.linalg.inv(T_true[a]) @ T_true[b]) for a, b in lc]
    mk = lambda dim: None if rng.random() < 0.1 else dict(
        X=rng.standard_normal(dim) * 5, med_obs_dir=rng.standard_normal(3), dir_list=rng.standard_normal((rng.integers(0, 4), 3)))
    pts, lns = [mk(3) for _ in range(60)], [mk(6) for _ in range(25)]
    live_ids = np.nonzero(live)[0]
    pkf, lkf = [[] for _ in range(n_tot)], [[] for _ in range(n_tot)]
    for lists, n in ((pkf, len(pts)), (lkf, len(lns))):
        for i in range(n):
            lists[int(rng.choice(live_ids))].append(i)
    b = [struct.pack("<4i", 150, 75, 100, n_tot)]
    for i in range(n_tot):
        b.append(struct.pack("<i16d", 1, *T[i].ravel()) if live[i] else struct.pack("<i", 0))
    b.append(fg.astype("<i4").tobytes())
    b.append(struct.pack("<i", len(lc)))
    for (a, c), x in zip(lc, lc_pose):
        b.append(struct.pack("<2i6d", a, c, *x))
    for slots in (pts, lns):
        b.append(struct.pack("<i", len(slots)))
        for sl in slots:
            if sl is None:
                b.append(struct.pack("<i", 0))
                continue
            b.append(struct.pack(f"<i{len(sl['X'])}d3di", 1, *sl["X"], *sl["med_obs_dir"], len(sl["dir_list"])))
            b.append(np.asarray(sl["dir_list"], "<f8").tobytes())
    for lists in (pkf, lkf):
        for l in lists:
            b.append(struct.pack(f"<i{len(l)}i", len(l), *l))
    with open(path, "wb") as f:
        f.write(b"".join(b))
    as_map = lambda slots, key: [None if s is None else dict({key: s["X"]}, med_obs_dir=s["med_obs_dir"],
                                                              dir_list=s["dir_list"]) for s in slots]
    return dict(T=T, live=live, fg=fg, lc=lc, lc_pose=lc_pose, pts=as_map(pts, "point3D"), lns=as_map(lns, "line3D"),
                pkf=pkf, lkf=lkf)


def test_vo_demo_pgo_selftest(built, tmp_path):
    """`vo_demo --pgo-selftest`: the INTEGRATION.md §4 f7 function, compiled against the shim, builds the graph from a
    map with erased keyframes, deleted landmarks and keyframes after the loop, calls plf_pose_graph and writes the poses
    and landmarks back; the result must be oracle/pgo.py's cov_graph_lists + the Python binding + cov_graph_write_back"""
    import subprocess
    from pathlib import Path
    demo = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "lib" / "vo_demo"
    m = _write_pgo_map(tmp_path / "map.bin", np.random.default_rng(11))
    out = subprocess.run([str(demo), "--pgo-selftest", str(tmp_path / "map.bin")], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr
    rows = [l.split() for l in out.stdout.splitlines() if l.startswith("pgo ")]
    g = pgo.cov_graph_lists(m["fg"], m["live"], m["T"], m["lc"], m["lc_pose"])
    with plf.Frontend() as f2:
        r = f2.pose_graph(g)
    T2, P2, L2 = pgo.cov_graph_write_back(m["T"], m["live"], g["kf_list"], r["T"], m["pts"], m["lns"], m["pkf"], m["lkf"])
    res = [x for x in rows if x[1] == "result"][0]
    assert float(res[5]) == pytest.approx(r["chi2_init"], rel=1e-9, abs=1e-20)
    assert float(res[6]) == pytest.approx(r["chi2"], rel=TOL, abs=1e-20)
    kfs = [x for x in rows if x[1] == "kf"]
    assert [int(x[2]) for x in kfs] == list(np.nonzero(m["live"])[0])
    T = np.array([[float(v) for v in x[3:]] for x in kfs]).reshape(-1, 4, 4)
    sc = np.abs(T2).max()
    assert np.abs(T - T2[m["live"]]).max() <= TOL * sc
    assert not np.allclose(T2[m["live"]], m["T"][m["live"]])      # the loop moved the trajectory
    for kind, key, dim, want in (("pt", "point3D", 3, P2), ("ls", "line3D", 6, L2)):
        got = {int(x[2]): np.array([float(v) for v in x[3:]]) for x in rows if x[1] == kind}
        assert sorted(got) == [i for i, w in enumerate(want) if w is not None], kind
        for i, v in got.items():
            w = want[i]
            ref = np.concatenate([w[key], w["med_obs_dir"], np.asarray(w["dir_list"]).ravel()])
            assert v.shape == ref.shape and np.abs(v - ref).max() <= TOL * max(sc, np.abs(ref).max()), (kind, i)
    assert [tuple(int(v) for v in x[2:]) for x in rows if x[1] == "lc"] == [(2, 41, 0), (8, 38, 0)]
