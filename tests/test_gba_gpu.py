"""GPU parity of the global bundle adjustment (plf_global_ba, csrc/lba.cu) against the CPU restatement of
MapHandler::levMarquardtOptimizationGBA (oracle/gba.py; src/mapHandler.cpp:2101-2699).  The oracle solves the reference's
sparse system (lower triangle, scipy splu); the device solves the same normal equations through the Schur complement on
the landmarks, factoring the reduced system in one CTA up to 64 keyframes and with the tiled LDL^T beyond, so agreement
is to rounding: 1e-6 relative on the update of every block, as for the local BA."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, gba
from oracle import synth as osynth
from plslam_b200 import synth

pytestmark = pytest.mark.gpu
CAM = plf.KITTI_CAMERA
TOL = 1e-6
PLF_ERR_INVALID = -1
PLF_ERR_CAPACITY = -4


def _check(p, got, ref):
    assert got["iters"] == ref["iters"]
    for k in ("kf_pose", "pt", "ls"):
        if ref[k].size:
            step = np.abs(ref[k] - p[k]).max()
            assert np.abs(got[k] - ref[k]).max() <= TOL * max(step, 1e-3), k
    assert np.array_equal(got["pt_moved"], ref["pt_moved"]) and np.array_equal(got["ls_moved"], ref["ls_moved"])
    assert abs(got["lambda_"] - ref["lambda_"]) <= 1e-9 * abs(ref["lambda_"])
    if np.isfinite(ref["err"]):
        assert abs(got["err"] - ref["err"]) <= 1e-9 * abs(ref["err"])
    else:
        assert np.array_equal(np.isnan(got["err"]), np.isnan(ref["err"])) and not np.isfinite(got["err"])


CASES = [  # (n_kf, pts_per_kf, ls_per_kf, n_fixed): 64 keyframes = n 384 (one CTA), 65 = the smallest tiled solve
    (1, 30, 8, 1), (8, 20, 6, 3), (64, 12, 4, 1), (65, 12, 0, 1), (65, 0, 5, 2), (200, 8, 3, 4), (600, 6, 2, 1)]


# With the intent, the error is finite and the DBL_EPSILON stop tests of the reference compare errors that differ in the
# last bits between two summation orders, so those runs use LBA's 1e-7 thresholds; as written, err is +inf and the run
# ends at max_iters (or |DX| < DBL_EPSILON).
@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("n_kf,ppk,lpk,n_fixed", CASES)
def test_global_ba_matches_the_oracle(fe, n_kf, ppk, lpk, n_fixed, quirks):
    p = synth.gba_problem(CAM, n_kf=n_kf, pts_per_kf=ppk, ls_per_kf=lpk, n_fixed=n_fixed, seed=n_kf + 17 * n_fixed)
    kw = {} if quirks else dict(min_error=1e-7, min_error_change=1e-7)
    ref = gba.global_ba(CAM, p, gba.opts(ref_quirks=quirks, **kw))
    got = fe.global_ba(p, ref_quirks=quirks, **kw)
    _check(p, got, ref)


def test_g2_int_maximum_on_the_device(fe):
    """(g2) below 1: lambda = 0; beyond 2^31 on the last diagonal entry: lambda = lambda_0 INT_MIN"""
    import test_gba_oracle as t
    p = t.g2_small_problem()
    _check(p, fe.global_ba(p, max_iters=1, ref_quirks=0), gba.global_ba(CAM, p, gba.opts(ref_quirks=0, max_iters=1)))
    # as written the first step is undamped (lambda = 0) on a near-singular system: only lambda is compared
    assert fe.global_ba(p, max_iters=1, ref_quirks=1)["lambda_"] == 0.0 == gba.global_ba(CAM, p, gba.opts(max_iters=1))["lambda_"]
    cam = t.g2_big_cam()
    q = t.g2_big_problem()
    with plf.Frontend(camera=cam) as f2:
        got = f2.global_ba(q, max_iters=1, ref_quirks=1)
    assert got["lambda_"] == 1e-5 * gba.INT_MIN
    _check(q, got, gba.global_ba(cam, q, gba.opts(ref_quirks=1, max_iters=1)))


@pytest.mark.parametrize("quirks", [0, 1])
def test_2048_keyframes_one_step_solves_the_damped_system(fe, quirks):
    """max_iters = 1 on a 2048-keyframe map (the tiled solve over 192 tile columns): the step recovered from the output
    solves the damped first-pass system, assembled by scipy.sparse from the oracle's rows (the reference's lower triangle,
    (g6) included as written, lambda by (g2)), to a relative residual of 1e-8"""
    import scipy.sparse as sp
    p = synth.gba_problem(CAM, n_kf=2048, pts_per_kf=40, ls_per_kf=6, seed=5)
    got = fe.global_ba(p, max_iters=1, ref_quirks=quirks)
    nkf = len(p["kf_pose"])
    X0 = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Hl, g, _ = gba.normal_equations(CAM, p, X0, T0inv, True, bool(quirks), 1e-7)
    dg = Hl.diagonal()
    lam = 1e-5 * (gba.hmax_int(dg) if quirks else np.abs(dg).max())
    assert got["lambda_"] == pytest.approx(lam, rel=1e-9)
    Hl = Hl + sp.diags(lam * dg)
    H = (Hl + Hl.T - sp.diags(Hl.diagonal())).tocsr()
    # T_out = T_in inverse(exp(dx)): dx = log(T_out^-1 T_in); landmarks: X_out - X_in
    dk = np.stack([clib.logmap_se3(clib.inverse_se3(clib.expmap_se3(a)) @ clib.expmap_se3(b))
                   for a, b in zip(got["kf_pose"], p["kf_pose"])])
    DX = np.concatenate([dk.ravel(), np.concatenate([got["pt"].ravel(), got["ls"].ravel()]) - X0[6 * nkf:]])
    assert np.linalg.norm(H @ DX - g) <= 1e-8 * np.linalg.norm(g)


def _raw_args(p, keep, null=None):
    """plf_lba_problem fields for a problem dict; `null` names an array passed as NULL.  `keep` holds the arrays alive."""
    args = dict(n_kf=len(p["kf_pose"]), n_pt=len(p["pt"]), n_ls=len(p["ls"]), n_fixed=len(p["fixed_T"]),
                n_pt_obs=len(p["pt_obs_lm"]), n_ls_obs=len(p["ls_obs_lm"]))
    for k, dt in (("kf_pose", np.float64), ("pt", np.float64), ("ls", np.float64), ("fixed_T", np.float64),
                  ("pt_obs_lm", np.int32), ("pt_obs_kf", np.int32), ("pt_obs_xy", np.float64), ("ls_obs_lm", np.int32),
                  ("ls_obs_kf", np.int32), ("ls_obs_le", np.float64)):
        a = np.ascontiguousarray(p[k], dt).copy()
        keep.append(a)
        args[k] = None if k == null or not a.size else a.ctypes.data
    return args


def _raw_call(fe, prob_kw, quirks=1):
    """plf_global_ba through ctypes with explicit counts and pointers (NULL where None)"""
    p = plf.plf_lba_problem(**prob_kw)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, gba.DBL_EPSILON, gba.DBL_EPSILON, quirks)
    res = plf.plf_lba_result()
    return fe.lib.plf_global_ba(fe._ctx, C.byref(o), C.byref(p), C.byref(res))


def test_global_ba_rejects_bad_input_and_stays_usable(fe):
    p = synth.gba_problem(CAM, n_kf=6, pts_per_kf=10, ls_per_kf=3, seed=2)
    want = gba.global_ba(CAM, p, gba.opts())

    def valid():
        _check(p, fe.global_ba(p), want)

    bad = []
    big = synth.gba_problem(CAM, n_kf=4097, pts_per_kf=1, ls_per_kf=0, seed=1, loop=False)
    keep = []
    assert _raw_call(fe, _raw_args(big, keep)) == PLF_ERR_CAPACITY
    valid()
    orphan = dict(p, pt=np.concatenate([p["pt"], p["pt"][:1]]))        # a point without observations
    bad.append(("orphan point", orphan, plf.PlfError))
    orphan_l = dict(p, ls=np.concatenate([p["ls"], p["ls"][:1]]))
    bad.append(("orphan line", orphan_l, plf.PlfError))
    bad.append(("ungrouped", dict(p, pt_obs_lm=p["pt_obs_lm"][::-1].copy()), plf.PlfError))
    lm = p["pt_obs_lm"].copy(); lm[-1] = len(p["pt"])
    bad.append(("landmark out of range", dict(p, pt_obs_lm=lm), plf.PlfError))
    kf = p["ls_obs_kf"].copy(); kf[0] = len(p["kf_pose"])
    bad.append(("keyframe out of range", dict(p, ls_obs_kf=kf), plf.PlfError))
    kf = p["pt_obs_kf"].copy(); kf[0] = -2                               # only one fixed keyframe
    bad.append(("fixed keyframe out of range", dict(p, pt_obs_kf=kf), plf.PlfError))
    empty = dict(p, pt_obs_lm=np.zeros(0, np.int32), pt_obs_kf=np.zeros(0, np.int32), pt_obs_xy=np.zeros((0, 2)),
                 ls_obs_lm=np.zeros(0, np.int32), ls_obs_kf=np.zeros(0, np.int32), ls_obs_le=np.zeros((0, 3)))
    bad.append(("empty", empty, plf.PlfError))
    for name, q, exc in bad:
        with pytest.raises(exc):
            fe.global_ba(q)
        valid()
    # NULL arrays with non-zero counts
    for field in ("kf_pose", "pt", "ls", "fixed_T", "pt_obs_lm", "ls_obs_le"):
        keep = []
        assert _raw_call(fe, _raw_args(p, keep, null=field)) == PLF_ERR_INVALID, field
        valid()


def test_global_ba_between_batches_leaves_the_pipeline_unchanged(built):
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = osynth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    frames = list(osynth.stream(cam, 8, world=world, seed=5, step=0.1))
    L = np.stack([f[0] for f in frames]); R = np.stack([f[1] for f in frames])
    lim = plf.default_limits(); lim.max_batch = 2
    p = synth.gba_problem(cam, n_kf=80, pts_per_kf=10, ls_per_kf=3, seed=4)

    def run(with_gba):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=500, lsd_nfeatures=100) as fe:
            out, ba = [], None
            for b in range(0, 8, 2):
                fe.batch_upload(L[b:b + 2], R[b:b + 2])
                fe.batch_run(2)
                if with_gba and b == 4:   # two batches, global_ba with the third in flight, two batches
                    ba = fe.global_ba(p)
                res = fe.batch_download_array(2)
                out += [np.ascontiguousarray(res[f]) for f in res.dtype.names]
                out += [np.ascontiguousarray(a) for a in fe.get_frame(1).values() if isinstance(a, np.ndarray)]
            return out, ba

    (a, _), (b, ba) = run(False), run(True)
    assert len(a) == len(b) and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    with plf.Frontend(camera=cam) as fe:
        fresh = fe.global_ba(p)
    _check(p, ba, fresh)   # float atomics: equal to rounding, not bit for bit


def _write_map(path, cam, p, erased_kf, prm):
    """the map vo_demo --gba-selftest reads (format in vo_demo.cpp): p's keyframes in kf_idx order with the slots in
    `erased_kf` empty (NULL), a deleted point and line slot, a point and a line seen only by erased keyframes, and one
    observation by an erased keyframe appended to every fifth landmark.  Returns the map index of p's landmarks."""
    import struct
    n_tot = 1 + len(p["kf_pose"]) + len(erased_kf)
    live = [i for i in range(n_tot) if i not in erased_kf]          # live[0] = 0: keyframe 0
    b = [struct.pack("<2i5d3di", cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["b"],
                     prm["lambda_"], prm["lambda_k"], prm["homog_th"], prm["max_iters"])]
    slot = {}
    for j, i in enumerate(live):
        slot[i] = (clib.logmap_se3(p["fixed_T"][0]), p["fixed_T"][0]) if j == 0 else \
            (p["kf_pose"][j - 1], clib.expmap_se3(p["kf_pose"][j - 1]))
    b.append(struct.pack("<i", n_tot))
    for i in range(n_tot):
        if i in slot:
            b.append(struct.pack("<i6d16d", 1, *slot[i][0], *np.asarray(slot[i][1]).ravel()))
        else:
            b.append(struct.pack("<i", 0))
    kf_idx = lambda k: live[0] if k < 0 else live[k + 1]
    index = {}
    for kind, dim, odim, X, Z in (("pt", 3, 2, p["pt"], p["pt_obs_xy"]), ("ls", 6, 3, p["ls"], p["ls_obs_le"])):
        lm, kf = p[kind + "_obs_lm"], p[kind + "_obs_kf"]
        start = np.searchsorted(lm, np.arange(len(X) + 1))
        slots = []
        for l in range(len(X)):
            obs = [(kf_idx(kf[o]), Z[o]) for o in range(start[l], start[l + 1])]
            if l % 5 == 0:
                obs.append((erased_kf[0], np.full(odim, 7.0)))
            slots.append((X[l], obs))
            if l == 2:
                slots.append(None)                                             # a deleted landmark
            if l == 4:
                slots.append((X[l] + 1.0, [(e, np.full(odim, 3.0)) for e in erased_kf]))   # seen only by erased keyframes
        b.append(struct.pack("<i", len(slots)))
        idx = []
        for m, sl in enumerate(slots):
            if sl is None:
                b.append(struct.pack("<i", 0))
                continue
            x, obs = sl
            b.append(struct.pack(f"<i{dim}di", 1, *x, len(obs)))
            for k, z in obs:
                b.append(struct.pack(f"<i{odim}d", k, *z))
            if all(k in erased_kf for k, _ in obs):
                continue
            idx.append(m)
        index[kind] = idx
    with open(path, "wb") as f:
        f.write(b"".join(b))
    return live, index


def test_vo_demo_gba_selftest(built, tmp_path):
    """`vo_demo --gba-selftest`: the INTEGRATION.md §4 f6 function, compiled against the shim, assembles the lists from a
    map with erased keyframes and deleted landmarks and gives the result, poses and landmarks the Python binding gives
    on the same problem"""
    import subprocess
    from pathlib import Path
    demo = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "lib" / "vo_demo"
    p = synth.gba_problem(CAM, n_kf=70, pts_per_kf=8, ls_per_kf=3, seed=12)
    prm = dict(lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7)
    live, index = _write_map(tmp_path / "map.bin", CAM, p, [3, 20], prm)
    out = subprocess.run([str(demo), "--gba-selftest", str(tmp_path / "map.bin")], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr
    rows = [l.split() for l in out.stdout.splitlines() if l.startswith("gba ")]
    with plf.Frontend(camera=CAM) as fe:
        want = fe.global_ba(p, **prm)
    res = [r for r in rows if r[1] == "result"][0]
    assert int(res[2]) == want["iters"] and float(res[4]) == pytest.approx(want["lambda_"], rel=1e-12)
    assert not np.isfinite(float(res[3])) and not np.isfinite(want["err"])
    kfs = [r for r in rows if r[1] == "kf"]
    assert [int(r[2]) for r in kfs] == live[1:]
    T = np.array([[float(v) for v in r[3:]] for r in kfs]).reshape(-1, 4, 4)
    T_want = np.stack([clib.expmap_se3(x) for x in want["kf_pose"]])
    assert np.abs(T - T_want).max() <= 1e-9 * max(1.0, np.abs(T_want).max())
    for kind, dim in (("pt", 3), ("ls", 6)):
        got = [r for r in rows if r[1] == kind]
        X = np.array([[float(v) for v in r[3:]] for r in got]).reshape(-1, dim)
        # every map slot prints; the live ones the call optimised carry the binding's values, the rest are unchanged
        pos = {int(r[2]): n for n, r in enumerate(got)}
        opt = np.stack([X[pos[m]] for m in index[kind]])
        assert np.abs(opt - want[kind]).max() <= 1e-9 * max(1.0, np.abs(want[kind]).max()), kind
        assert len(got) == len(index[kind]) + 1                              # + the landmark seen only by erased keyframes
