"""The pose solver (k_gn_pose, csrc/gn.cu, through plf_gn_pose) against the oracle (oracle/gn.c) on every field - T, x,
cov, err, iteration counts, inlier masks and counts - at the edges where a batched fp64 reduction and a rank-revealing
6x6 solve go wrong: row counts around the CTA's 128-thread stride and its 4-warp reduction, fewer rows than unknowns
and other rank-deficient geometry, the homog_th clamps, rows gated out, zero iteration limits and non-identity starts.

Rules (DESIGN.md section 3):
  - masks and counts exactly; x within 1e-6 relative; err within 1e-9 relative; NaN / inf in the same places;
  - cov within 1e-12 kappa(H) ||cov|| (kappa: condition number) of the oracle's;
  - iteration counts exactly on decidable runs (clib.gn_decidable: no stop test the oracle evaluated sat within
    summation-order rounding of its threshold); the others are counted, and their share must stay small;
  - where the run's last stop was the error test (then the last accumulation was made at the final pose with the final
    masks), err and cov against an exactly rounded restatement of that accumulation (accumulate_fsum) at the device's
    own T and masks: err within 1e-11, cov within 1e-12 kappa(H) ||cov|| of inv(H).  This checks the kernel's
    reduction against sums that do not share its rounding, nor the oracle's.
"""
import math

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth

CAM = plf.KITTI_CAMERA
EPS = np.finfo(np.float64).eps
X_REL_TOL = 1e-6        # pose (se(3) log), as tests/test_gn_gpu.py; north-star bar 1e-4
ERR_REL_TOL = 1e-9
FSUM_ERR_REL_TOL = 1e-11
COV_KAPPA_TOL = 1e-12
BAND_SHARE_MAX = 0.2    # share of runs whose iteration counts are not decidable, per test
SPREAD_FACTOR = 100     # tolerances widen to this multiple of the oracle's own spread under reordered sums (check)

EUROC = dict(max_iters=5, max_iters_ref=10)                       # config_euroc.yaml
KITTI = dict(max_iters=100, max_iters_ref=100)                    # config_kitti.yaml
ONE_STEP = dict(max_iters=1, max_iters_ref=0)
TWIN = dict(max_iters=5, max_iters_ref=10, eps_err=EPS, eps_change=EPS)   # the in-tree twin's stop thresholds
ROW_COUNTS = (1, 2, 5, 6, 7, 31, 32, 33, 127, 128, 129, 255, 256, 257, 2049)


# ---- exactly rounded restatement of one accumulation pass (oracle/gn.c gn_accumulate) ---------------------------
def _transform(T, X):
    return [T[i, 0] * X[:, 0] + T[i, 1] * X[:, 1] + T[i, 2] * X[:, 2] + T[i, 3] for i in range(3)]


def _project(cam, Q):
    return cam["cx"] + cam["fx"] * Q[0] / Q[2], cam["cy"] + cam["fy"] * Q[1] / Q[2]


def _jac6(fgz2, gx, gy, gz, ax, ay):
    return np.stack([fgz2 * ax * gz, fgz2 * ay * gz, -fgz2 * (gx * ax + gy * ay),
                     -fgz2 * (gx * gy * ax + gy * gy * ay + gz * gz * ay),
                     fgz2 * (gx * gx * ax + gz * gz * ax + gx * gy * ay),
                     fgz2 * (gx * gz * ay - gy * gz * ax)], 1)


def accumulate_fsum(cam, homog_th, T, pr, inlier_pt, inlier_ls):
    """H (6x6), g, e and the row count of one accumulation at pose T: every point and line row computed as gn.c computes
    it (same operations, same order, elementwise), the sums over rows exactly rounded (math.fsum)."""
    T = np.asarray(T, np.float64)
    mp, ml = np.asarray(inlier_pt, bool), np.asarray(inlier_ls, bool)
    P, obs = np.asarray(pr["P"], np.float64)[mp], np.asarray(pr["obs"], np.float64)[mp]
    Pc = _transform(T, P)
    u, v = _project(cam, Pc)
    e0, e1 = u - obs[:, 0], v - obs[:, 1]
    r_p = np.sqrt(e0 * e0 + e1 * e1)
    J_p = _jac6(cam["fx"] / np.maximum(homog_th, Pc[2] * Pc[2]), Pc[0], Pc[1], Pc[2], e0, e1)
    J_p = J_p / np.maximum(homog_th, r_p)[:, None]
    le = np.asarray(pr["le"], np.float64)[ml]
    S, E = _transform(T, np.asarray(pr["sP"], np.float64)[ml]), _transform(T, np.asarray(pr["eP"], np.float64)[ml])
    (su, sv), (eu, ev) = _project(cam, S), _project(cam, E)
    e0 = le[:, 0] * su + le[:, 1] * sv + le[:, 2]
    e1 = le[:, 0] * eu + le[:, 1] * ev + le[:, 2]
    r_l = np.sqrt(e0 * e0 + e1 * e1)
    Js = _jac6(cam["fx"] / np.maximum(homog_th, S[2] * S[2]), S[0], S[1], S[2], le[:, 0], le[:, 1])
    Je = _jac6(cam["fx"] / np.maximum(homog_th, E[2] * E[2]), E[0], E[1], E[2], le[:, 0], le[:, 1])
    J_l = (Js * e0[:, None] + Je * e1[:, None]) / np.maximum(homog_th, r_l)[:, None]
    J, r = np.concatenate([J_p, J_l]), np.concatenate([r_p, r_l])
    w = 1.0 / (1.0 + r * r)
    H = np.array([[math.fsum(J[:, a] * J[:, b] * w) for b in range(6)] for a in range(6)])
    g = np.array([math.fsum(J[:, a] * r * w) for a in range(6)])
    n = len(r)
    return H, g, (math.fsum(r * r * w) / n if n else math.nan), n


# ---- comparison rules -------------------------------------------------------------------------------------------
def rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12)


def same_nonfinite(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
            and np.array_equal(np.isneginf(a), np.isneginf(b)))


def err_close(err, ref, tol=ERR_REL_TOL):
    """err within tol relative of ref; NaN where ref is NaN (no row left)."""
    if not np.isfinite(ref):
        return same_nonfinite(err, ref)
    return abs(err - ref) <= tol * abs(ref)


def cov_dist(cov, ref):
    """||cov - ref|| / (kappa ||ref||), kappa the condition number of ref (= that of H).  0 when both are equally
    non-finite (the inverse of a zero H: NaN / inf in the same places, equal elsewhere), and 0 when H is singular to
    working precision on both sides (kappa >= 1 / eps, or not finite): its inverse is then rounding, on either side.
    Otherwise inf when only one side is finite or singular."""
    cov, ref = np.asarray(cov, np.float64), np.asarray(ref, np.float64)
    singular = lambda c: not np.isfinite(c).all() or np.linalg.cond(c) >= 1 / EPS
    if not (np.isfinite(ref).all() and np.isfinite(cov).all()):
        fin = np.isfinite(ref)
        if same_nonfinite(cov, ref) and np.array_equal(cov[fin], ref[fin]):
            return 0.0
    if singular(ref) or singular(cov):
        return 0.0 if singular(ref) and singular(cov) else math.inf
    return np.linalg.norm(cov - ref) / (np.linalg.cond(ref) * np.linalg.norm(ref))


def cov_close(cov, ref, tol=COV_KAPPA_TOL):
    return cov_dist(cov, ref) <= tol


class Tally:
    """Runs compared: decidable or in the band (iteration counts), and how many were order-sensitive."""

    def __init__(self):
        self.decided, self.band, self.fsum, self.sensitive = 0, [], 0, []

    @property
    def runs(self):
        return self.decided + len(self.band)

    def report(self, what):
        print(f"{what}: {self.runs} runs, {self.decided} decidable, {len(self.band)} in the band, "
              f"{len(self.sensitive)} order-sensitive, {self.fsum} checked against the exactly rounded sums")

    def assert_band_small(self, what):
        self.report(what)
        assert self.runs and len(self.band) <= BAND_SHARE_MAX * self.runs, (what, self.band)


def oracle_spread(pr, o, r_o, inlier_pt=None, inlier_ls=None, T_init=None, cam=CAM):
    """How far the oracle's result r_o moves when its rows are summed in other orders (reversed, and one fixed
    shuffle): what rounding alone can move it by.  A run that amplifies rounding shows it in at least one of them."""
    sp = dict(x=0.0, T=0.0, err=0.0, cov=0.0, iters=False, masks=False)
    n_p, n_l = len(pr["P"]), len(pr["sP"])
    rng = np.random.default_rng(n_p * 7919 + n_l)
    for perm_p, perm_l in ((np.arange(n_p)[::-1], np.arange(n_l)[::-1]), (rng.permutation(n_p), rng.permutation(n_l))):
        take = lambda a, perm: None if a is None else np.ascontiguousarray(np.asarray(a)[perm])
        r = clib.gn_pose(cam, take(pr["P"], perm_p), take(pr["obs"], perm_p), take(pr["sP"], perm_l),
                         take(pr["eP"], perm_l), take(pr["le"], perm_l), inlier_pt=take(inlier_pt, perm_p),
                         inlier_ls=take(inlier_ls, perm_l), T_init=T_init, opts=o)
        ip, il = np.empty_like(r["inlier_pt"]), np.empty_like(r["inlier_ls"])
        ip[perm_p], il[perm_l] = r["inlier_pt"], r["inlier_ls"]
        sp["x"] = max(sp["x"], rel(r["x"], r_o["x"]))
        sp["T"] = max(sp["T"], np.abs(r["T"] - r_o["T"]).max())
        if not err_close(r["err"], r_o["err"], 0.0):
            sp["err"] = max(sp["err"], abs(r["err"] - r_o["err"]) / abs(r_o["err"]))
        sp["cov"] = max(sp["cov"], cov_dist(r["cov"], r_o["cov"]))
        sp["iters"] |= r["iters"] != r_o["iters"]
        sp["masks"] |= not (np.array_equal(ip, r_o["inlier_pt"]) and np.array_equal(il, r_o["inlier_ls"]))
    return sp


def run_both(fe, pr, opts, inlier_pt=None, inlier_ls=None, T_init=None):
    """The device and the oracle on one problem; res["spread"] of the oracle's is its oracle_spread."""
    o = clib.gn_opts(**opts)
    po = plf.plf_gn_opts(o.homog_th, o.max_iters, o.max_iters_ref, o.eps_err, o.eps_change, o.eps_step)
    args = (pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"])
    r_o = clib.gn_pose(CAM, *args, inlier_pt=inlier_pt, inlier_ls=inlier_ls, T_init=T_init, opts=o, trace=True)
    r_o["spread"] = oracle_spread(pr, o, r_o, inlier_pt, inlier_ls, T_init)
    r_g = fe.gn_pose(*args, inlier_pt=inlier_pt, inlier_ls=inlier_ls, T_init=T_init, opts=po)
    return r_o, r_g, o


def check(r_g, r_o, o, pr, tally, what):
    """Every field of the device result r_g against the oracle's r_o (from run_both, under options o).

    Each tolerance is widened to SPREAD_FACTOR times the oracle's own spread under a change of summation order where
    that is larger: an undamped Gauss-Newton run that does not converge (100 iterations on a few dozen rows with
    outliers), or that walks along the null space of a singular H, amplifies rounding, and there the reference itself
    does not determine its result to the fixed tolerances.  Such runs are counted as order-sensitive."""
    sp = r_o["spread"]
    tol = lambda t, s: max(t, SPREAD_FACTOR * s)
    if max(sp["x"] / X_REL_TOL, sp["err"] / ERR_REL_TOL, sp["cov"] / COV_KAPPA_TOL) > 1 / SPREAD_FACTOR or sp["iters"]:
        tally.sensitive.append(what)
    same_masks = np.array_equal(r_g["inlier_pt"], r_o["inlier_pt"]) and np.array_equal(r_g["inlier_ls"], r_o["inlier_ls"])
    if sp["masks"] or (not same_masks and sp["x"] > X_REL_TOL):
        # the chi2 gate went another way under reordered sums, or the stage-1 pose it is applied at is not determined
        # to the pose tolerance: the stage-2 problems may differ, nothing further is comparable
        tally.sensitive.append(what)
        return
    assert same_masks, what
    assert r_g["n_inliers"] == r_o["n_inliers"], what
    assert rel(r_g["x"], r_o["x"]) <= tol(X_REL_TOL, sp["x"]), (what, r_g["x"], r_o["x"], sp)
    assert np.abs(r_g["T"] - r_o["T"]).max() <= tol(1e-8, sp["T"]), (what, sp)
    assert err_close(r_g["err"], r_o["err"], tol(ERR_REL_TOL, sp["err"])), (what, r_g["err"], r_o["err"], sp)
    assert cov_close(r_g["cov"], r_o["cov"], tol(COV_KAPPA_TOL, sp["cov"])), (what, r_g["cov"], r_o["cov"], sp)
    if sp["iters"] or not clib.gn_decidable(r_o["trace"], o):
        tally.band.append(what)
        return
    tally.decided += 1
    assert r_g["iters"] == r_o["iters"], (what, r_g["iters"], r_o["iters"])
    if r_o["trace"]["exit"][1] == clib.GN_EXIT_ERROR and sum(r_o["n_inliers"]) > 0:
        # the last accumulation was at the final pose, with the final masks: restate it exactly rounded
        H, _, e, _ = accumulate_fsum(CAM, o.homog_th, r_g["T"], pr, r_g["inlier_pt"], r_g["inlier_ls"])
        assert err_close(r_g["err"], e, FSUM_ERR_REL_TOL), (what, r_g["err"], e)
        if np.linalg.cond(H) < 1 / EPS:
            assert cov_close(r_g["cov"], np.linalg.inv(H)), (what, "fsum", r_g["cov"], np.linalg.inv(H))
        tally.fsum += 1


def problem(n_pts, n_lines, seed, **kw):
    return synth.gn_problem(CAM, n_pts=n_pts, n_lines=n_lines, seed=seed, **kw)


# ---- CPU: the exactly rounded restatement against gn.c itself ---------------------------------------------------
@pytest.mark.parametrize("n_pts,n_lines", [(300, 80), (0, 40), (25, 0), (4, 4)])
def test_fsum_reference_matches_oracle(n_pts, n_lines):
    """accumulate_fsum at the oracle's final pose and masks gives the oracle's own err and cov (when its last stop was
    the error test), and would see a single row gone missing."""
    pr = problem(n_pts, n_lines, seed=n_pts + n_lines)
    o = clib.gn_opts(**dict(KITTI, eps_change=1e-2))     # stops on the change test once the error settles
    r = clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"], opts=o, trace=True)
    assert r["trace"]["exit"][1] == clib.GN_EXIT_ERROR
    H, g, e, n = accumulate_fsum(CAM, o.homog_th, r["T"], pr, r["inlier_pt"], r["inlier_ls"])
    assert n == sum(r["n_inliers"])
    assert err_close(r["err"], e, FSUM_ERR_REL_TOL) and cov_close(r["cov"], np.linalg.inv(H))
    ip = r["inlier_pt"].copy() if n_pts else r["inlier_pt"]
    il = r["inlier_ls"].copy()
    (ip if n_pts else il)[np.flatnonzero(ip if n_pts else il)[-1]] = 0
    H1, _, e1, _ = accumulate_fsum(CAM, o.homog_th, r["T"], pr, ip, il)
    assert not err_close(r["err"], e1, FSUM_ERR_REL_TOL) or not cov_close(r["cov"], np.linalg.inv(H1))


# ---- GPU ---------------------------------------------------------------------------------------------------------
def layouts(n):
    """Points only, lines only, and two mixes (one line with the rest points; half and half)."""
    out = [(n, 0), (0, n)]
    if n > 1:
        out += [(n - 1, 1), (n // 2, n - n // 2)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["euroc", "kitti", "kitti-exact", "twin"])
def test_row_counts(fe, cfg):
    """Rows around the CTA stride (128) and the warp boundaries of its reduction (32, 64, 96), from 6 rows up, as points
    only, lines only and mixed (1, 2 and 5 rows, fewer than the unknowns, are in test_rank_deficient).  The twin's
    thresholds (DBL_EPSILON) would put a converging run's change test inside the band; these runs do not converge
    (the solver settles into a two-state cycle, DESIGN.md section 8), so their stop decisions stay decidable too."""
    opts = dict(euroc=EUROC, kitti=KITTI, twin=TWIN)[cfg.split("-")[0]]
    clean = dict(px_noise=0.0, outlier_frac=0.0) if cfg.endswith("exact") else {}   # e -> 0: runs end on the error test
    tally = Tally()
    for n in (n for n in ROW_COUNTS if n >= 6):
        for n_pts, n_lines in layouts(n):
            pr = problem(n_pts, n_lines, seed=1000 * n + n_lines, **clean)
            r_o, r_g, o = run_both(fe, pr, opts)
            check(r_g, r_o, o, pr, tally, (cfg, n_pts, n_lines))
    tally.assert_band_small(f"row counts, {cfg}")


def observe_lines(T, sP, eP, rng, px_noise):
    """Normalised image lines (sp x ep) of segments sP-eP seen under T, with pixel noise on the end points."""
    sp = synth.project(CAM, sP @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, px_noise, (len(sP), 2))
    ep = synth.project(CAM, eP @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, px_noise, (len(eP), 2))
    le = np.cross(np.c_[sp, np.ones(len(sp))], np.c_[ep, np.ones(len(ep))])
    return le / np.sqrt(le[:, :1] ** 2 + le[:, 1:2] ** 2)


def one_location(n, seed):
    """n observations of a single 3-D point: every row's Jacobian lies in one 2-D subspace (rank 2)."""
    pr, rng = problem(1, 0, seed, outlier_frac=0.0), np.random.default_rng(seed)
    T = pr["T_true"]
    pr["P"] = np.repeat(pr["P"], n, 0)
    pr["obs"] = synth.project(CAM, pr["P"] @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, 1.0, (n, 2))
    return pr


def parallel_coplanar(n, seed):
    """n segments in the plane y = 1.5, all along x: no row sees a translation along x."""
    pr, rng = problem(0, 0, seed), np.random.default_rng(seed)
    sP = np.stack([rng.uniform(-8, 8, n), np.full(n, 1.5), rng.uniform(5, 30, n)], 1)
    eP = sP + np.array([2.0, 0.0, 0.0])
    pr.update(sP=sP, eP=eP, le=observe_lines(pr["T_true"], sP, eP, rng, 0.3))
    return pr


@pytest.mark.gpu
def test_rank_deficient(fe):
    """H singular by construction: fewer rows than unknowns, all points at one 3-D location, all lines parallel and
    coplanar.  The column-pivoting QR's rank cut (|R_kk| > 6 eps max|R_kk|) decides which directions the step moves."""
    tally = Tally()
    cases = [(f"{n_pts}+{n_lines} rows", problem(n_pts, n_lines, seed=70 + 10 * n_pts + n_lines))
             for n in (1, 2, 3, 4, 5) for n_pts, n_lines in layouts(n)]
    cases += [(f"one location x{n}", one_location(n, seed=n)) for n in (2, 7, 40, 300)]
    cases += [(f"parallel coplanar x{n}", parallel_coplanar(n, seed=n)) for n in (3, 12, 60, 257)]
    for what, pr in cases:
        for cfg in (ONE_STEP, EUROC):
            r_o, r_g, o = run_both(fe, pr, cfg)
            check(r_g, r_o, o, pr, tally, (what, cfg["max_iters"]))
    tally.assert_band_small("rank deficient")


@pytest.mark.gpu
def test_clamps(fe):
    """The homog_th clamps: depth^2 below homog_th at T_init (fx / max(homog_th, z^2)), points and line end points
    behind the camera, exact observations (residual norm below homog_th: J / max(homog_th, r)), and homog_th = 1 with
    depths from 0.3 m, where both clamps act on many rows."""
    tally = Tally()
    near = problem(200, 40, seed=5)
    near["P"][:4] = [[0.5, 0.3, 1e-4], [-0.5, 0.3, 2e-4], [0.5, -0.3, -1.5e-4], [1.0, 1.0, 3e-4]]
    near["sP"][:2, 2] = [2e-4, -1e-4]
    behind = problem(200, 40, seed=6)
    behind["P"][:6, 2] *= -1
    behind["sP"][:3, 2] *= -1
    exact = problem(150, 30, seed=7, px_noise=0.0, outlier_frac=0.0)
    half = problem(150, 30, seed=8)
    exact_half = problem(150, 30, seed=8, px_noise=0.0, outlier_frac=0.0)
    half["obs"][:75], half["le"][:15] = exact_half["obs"][:75], exact_half["le"][:15]
    shallow = problem(200, 40, seed=9, z_range=(0.3, 3.0), x_true=[0.01, -0.005, 0.08, 0.004, -0.006, 0.002])
    runs = [("near", near, EUROC, None), ("near, one step", near, dict(max_iters=1, max_iters_ref=0), None),
            ("behind", behind, EUROC, None), ("behind", behind, KITTI, None),
            ("exact", exact, EUROC, exact["T_true"]), ("exact", exact, EUROC, None),
            ("half exact", half, EUROC, half["T_true"]), ("half exact", half, KITTI, half["T_true"]),
            ("homog_th 1", shallow, dict(EUROC, homog_th=1.0), None), ("homog_th 1", shallow, dict(KITTI, homog_th=1.0), None),
            ("homog_th 1, one step", shallow, dict(max_iters=1, max_iters_ref=0, homog_th=1.0), None)]
    for what, pr, cfg, T0 in runs:
        r_o, r_g, o = run_both(fe, pr, cfg, T_init=T0)
        check(r_g, r_o, o, pr, tally, what)
    tally.assert_band_small("clamps")


def all_outliers(n_pts, n_lines, cfg):
    """Observations unrelated to the 3-D features, at the first seed where the oracle gates every row after stage 1."""
    for seed in range(200):
        pr, rng = problem(n_pts, n_lines, seed, outlier_frac=0.0), np.random.default_rng(seed)
        a = rng.uniform(0, 2 * np.pi, n_pts)
        pr["obs"] += rng.uniform(20, 60, n_pts)[:, None] * np.stack([np.cos(a), np.sin(a)], 1)
        pr["le"] = observe_lines(pr["T_true"], pr["sP"], pr["eP"], rng, 30.0)
        if clib.gn_pose(CAM, pr["P"], pr["obs"], pr["sP"], pr["eP"], pr["le"], opts=clib.gn_opts(**cfg))["n_inliers"] == (0, 0):
            return pr
    raise AssertionError("no seed gates every row")


@pytest.mark.gpu
def test_gating(fe):
    """Every row gated out after stage 1 (stage 2 accumulates nothing: e = 0/0 and cov = inverse of a zero H, NaN / inf
    in the same places on both sides), inlier masks preset to all-zero, and preset mixes."""
    tally = Tally()
    ONE_FIRST = dict(max_iters=1, max_iters_ref=10)
    rng = np.random.default_rng(3)
    pr = problem(300, 60, seed=12)
    runs = [("all gated", all_outliers(40, 10, EUROC), EUROC, None, None), ("all gated, pts", all_outliers(30, 0, ONE_FIRST), ONE_FIRST, None, None),
            ("preset zero", pr, EUROC, np.zeros(300, np.uint8), np.zeros(60, np.uint8)),
            ("preset zero pts", pr, EUROC, np.zeros(300, np.uint8), None),
            ("preset zero lines", pr, KITTI, None, np.zeros(60, np.uint8)),
            ("preset mix", pr, EUROC, rng.integers(0, 2, 300).astype(np.uint8), rng.integers(0, 2, 60).astype(np.uint8)),
            ("preset one row", pr, EUROC, np.eye(1, 300, 150, dtype=np.uint8)[0], np.zeros(60, np.uint8))]
    for what, p, cfg, ip, il in runs:
        r_o, r_g, o = run_both(fe, p, cfg, inlier_pt=ip, inlier_ls=il)
        check(r_g, r_o, o, p, tally, what)
        if what.startswith("all gated") or what == "preset zero":
            assert r_g["n_inliers"] == (0, 0) and np.isnan(r_g["err"]) and not np.isfinite(r_g["cov"]).all(), what
    tally.assert_band_small("gating")


@pytest.mark.gpu
def test_iteration_limits_and_start(fe):
    """max_iters in {0, 1} x max_iters_ref in {0, 1, 10}, from the identity and from two other poses."""
    tally = Tally()
    pr = problem(300, 60, seed=13)
    starts = [None, synth.expmap_se3(pr["x_true"] + [0.01, -0.01, 0.02, 0.002, 0.001, -0.002]),
              synth.expmap_se3([0.3, 0.1, -0.2, 0.05, 0.1, -0.05])]
    for mi in (0, 1):
        for mir in (0, 1, 10):
            for k, T0 in enumerate(starts):
                r_o, r_g, o = run_both(fe, pr, dict(max_iters=mi, max_iters_ref=mir), T_init=T0)
                check(r_g, r_o, o, pr, tally, (mi, mir, k))
    for k, T0 in enumerate(starts[1:]):
        r_o, r_g, o = run_both(fe, pr, KITTI, T_init=T0)
        check(r_g, r_o, o, pr, tally, ("kitti", k))
    tally.assert_band_small("iteration limits")
