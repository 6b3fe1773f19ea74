"""GPU tests of plf_loop_closure_pose_batch and plf_gn_pose_batch: many loop-closure checks / pose refinements in one call,
each with its sequence's camera.  Every problem's result is bit-identical to the single call (plf_loop_closure_pose /
plf_gn_pose) on a context created with its camera, and the loop-closure results match oracle/loopclosure.py with that
camera at the tolerances of test_loopclosure_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import loopclosure as olc
from plslam_b200 import synth
from test_loopclosure_gpu import rel
from test_loopclosure_oracle import PRM
from test_sequence_cameras_gpu import CAM as BASE, CAMS   # BASE: the context's camera

pytestmark = pytest.mark.gpu

GN_PRM = dict(max_iters=PRM["max_iters"], max_iters_ref=PRM["max_iters_ref"])
EMPTY = dict(pdesc=np.zeros((0, 32), np.uint8), P=np.zeros((0, 3)), pl=np.zeros((0, 2)), ldesc=np.zeros((0, 32), np.uint8),
             sP=np.zeros((0, 3)), eP=np.zeros((0, 3)), le=np.zeros((0, 3)))
LCS = [None, dict(lc_unc=1e-12), dict(lc_res=1e-9), dict(lc_rot=0.01), dict(lc_trs=1e-3), dict(lc_inlier_ratio=101.0)]


def keyframes(cam, **kw):
    return synth.loop_closure_keyframes(cam, **kw)[:3]


def mixed_pairs(cam, seed):
    """Candidate pairs of every kind the single call treats differently, rendered with `cam`."""
    out = []
    for k, frac in enumerate((0.0, 0.05, 0.1, 0.15)):               # true revisits, 0 to 15 % outliers
        kf0, kf1, _ = keyframes(cam, seed=seed + k, outlier_frac=frac, x_true=np.array([0.08, -0.03, 0.4, 0.01, -0.04, 0.006]))
        out.append((kf0, kf1))
    kf0, kf1, _ = keyframes(cam, seed=seed + 5, x_true=np.array([0.5, 0.2, 1.9, 0.02, 0.05, 0.0]))   # |t| > lc_trs
    out.append((kf0, kf1))
    kf0, kf1, _ = keyframes(cam, seed=seed + 6)
    rng = np.random.default_rng(seed)
    out.append((kf0, dict(kf1, pdesc=rng.integers(0, 256, kf1["pdesc"].shape, dtype=np.uint8))))   # unrelated descriptors
    out.append((kf0, EMPTY))                                                                        # an empty keyframe
    out.append((EMPTY, kf1))                                                                        # 0 / 0 ratios
    return out


def same(a, b):
    """Bit equality of two result dicts (NaN-safe); `status` is the batch's own field."""
    assert set(a) - {"status"} == set(b) - {"status"}
    for k in set(a) - {"status"}:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k


def check_oracle(cam, kf0, kf1, prm, lc, g):
    r = olc.is_loop_closure(cam, kf0, kf1, prm, lc)
    assert g["estimated"] == r["estimated"] and g["accepted"] == r["accepted"]
    assert (g["common_pt"], g["common_ls"]) == (r["common_pt"], r["common_ls"])
    for k in ("inl_ratio_pt", "inl_ratio_ls"):
        assert g[k] == r[k] or (np.isnan(g[k]) and np.isnan(r[k]))
    if r["estimated"]:
        assert rel(g["x_inc"], r["x_inc"]) < 1e-6 and abs(g["err"] - r["err"]) <= 1e-6 * max(r["err"], 1e-12)
        assert abs(g["max_cov_eig"] - r["max_cov_eig"]) <= 1e-5 * r["max_cov_eig"]
        assert abs(g["t"] - r["t"]) < 1e-9 and abs(g["r"] - r["r"]) < 1e-7 and g["ratio_inliers"] == r["ratio_inliers"]
    if r["accepted"]:
        assert np.array_equal(g["pt_pairs"], r["pt_pairs"]) and np.array_equal(g["ls_pairs"], r["ls_pairs"])
        assert rel(g["pose_inc"], r["pose_inc"]) < 1e-6
    return r


def seq_context(**kw):
    fs = plf.Frontend(camera=BASE, max_sequences=4, **GN_PRM, **kw)
    for c in range(4):
        fs.set_sequence_camera(c, CAMS[c])
    return fs


def test_mixed_batch_equals_single_calls_per_camera(built):
    pairs, seq = [], []
    for c in range(4):
        for pr in mixed_pairs(CAMS[c], seed=10 * c):
            pairs.append(pr); seq.append(c)
    seq = np.array(seq, np.int32)
    singles = [plf.Frontend(camera=CAMS[c], **GN_PRM) for c in range(4)]
    seen = set()
    try:
        with seq_context() as fs:
            for lc in LCS:
                got = fs.loop_closure_pose_batch(pairs, seq=seq, lc=lc)
                for p, ((kf0, kf1), g) in enumerate(zip(pairs, got)):
                    assert g["status"] == 0
                    same(g, singles[seq[p]].loop_closure_pose(kf0, kf1, lc))
                    seen.add((g["estimated"], g["accepted"]))
                    if lc is None:
                        check_oracle(CAMS[seq[p]], kf0, kf1, PRM, lc, g)
                    if p % 8 == 7:
                        assert np.isnan(g["inl_ratio_pt"]) and np.isnan(g["inl_ratio_ls"]) and not g["estimated"]
    finally:
        for f in singles:
            f.close()
    assert seen == {(False, False), (True, False), (True, True)}


@pytest.mark.parametrize("kind", ["has_lines", "has_points"])
def test_points_only_and_lines_only(built, kind):
    prm = dict(PRM, **{kind: False})
    pairs = [pr for c in range(4) for pr in mixed_pairs(CAMS[c], seed=50 + c)[:5:2]]
    seq = np.repeat(np.arange(4, dtype=np.int32), 3)
    with seq_context(**{kind: 0}) as fs:
        got = fs.loop_closure_pose_batch(pairs, seq=seq)
        for c in range(4):
            with plf.Frontend(camera=CAMS[c], **GN_PRM, **{kind: 0}) as fe:
                for p in np.flatnonzero(seq == c):
                    same(got[p], fe.loop_closure_pose(*pairs[p]))
                    check_oracle(CAMS[c], *pairs[p], prm, None, got[p])
    assert any(g["accepted"] for g in got)
    assert all(len(g["ls_pairs" if kind == "has_lines" else "pt_pairs"]) == 0 for g in got)


def test_camera_selection_and_changes(built):
    pairs = mixed_pairs(BASE, seed=70)[:5]
    P = len(pairs)
    with plf.Frontend(camera=BASE, max_sequences=4, **GN_PRM) as fs, plf.Frontend(camera=BASE, **GN_PRM) as fe:
        ref = [fe.loop_closure_pose(*pr) for pr in pairs]
        a = fs.loop_closure_pose_batch(pairs)
        b = fs.loop_closure_pose_batch(pairs, seq=np.full(P, -1, np.int32))
        for s in range(4):
            fs.set_sequence_camera(s, BASE)
        seq = np.arange(P, dtype=np.int32) % 4
        c = fs.loop_closure_pose_batch(pairs, seq=seq)
        for x, y, z, r in zip(a, b, c, ref):
            same(x, r); same(y, r); same(z, r)
        fs.set_sequence_camera(1, CAMS[1])                        # the next call projects sequence 1 with CAMS[1]
        d = fs.loop_closure_pose_batch(pairs, seq=seq)
        with plf.Frontend(camera=CAMS[1], **GN_PRM) as f1:
            for p in range(P):
                same(d[p], f1.loop_closure_pose(*pairs[p]) if seq[p] == 1 else ref[p])
        assert any(d[p]["x_inc"].tobytes() != ref[p]["x_inc"].tobytes() for p in range(P) if seq[p] == 1)


def test_order_duplicates_and_single_problem_batches(built):
    pairs = [pr for c in range(4) for pr in mixed_pairs(CAMS[c], seed=90 + c)[::3]]
    seq = np.repeat(np.arange(4, dtype=np.int32), 3)
    with seq_context() as fs:
        base = fs.loop_closure_pose_batch(pairs, seq=seq)
        perm = np.random.default_rng(3).permutation(len(pairs))
        got = fs.loop_closure_pose_batch([pairs[i] for i in perm], seq=seq[perm])
        for j, i in enumerate(perm):
            same(got[j], base[i])
        dup = fs.loop_closure_pose_batch([pairs[0], pairs[4], pairs[0]], seq=seq[[0, 4, 0]])
        same(dup[0], base[0]); same(dup[1], base[4]); same(dup[2], base[0])
        for i in (0, 4, 11):
            same(fs.loop_closure_pose_batch([pairs[i]], seq=seq[[i]])[0], base[i])


def test_capacity_is_per_problem(built):
    pairs = [pr for c in range(2) for pr in mixed_pairs(CAMS[c], seed=110 + c)[:2]]
    seq = np.array([0, 0, 1, 1], np.int32)
    with seq_context() as fs:
        full = fs.loop_closure_pose_batch(pairs, seq=seq)
        assert full[2]["accepted"] and full[2]["n_pt"] > 5
        capped = [dict(kf0=p[0], kf1=p[1]) for p in pairs]
        capped[2]["cap_pt"] = 5
        got = fs.loop_closure_pose_batch(capped, seq=seq)
        msg = fs.lib.plf_last_error(fs._ctx).decode()
        assert "plf_loop_closure_pose_batch: problem 2:" in msg and "exceed the caller's capacity" in msg
        for p in (0, 1, 3):
            same(got[p], full[p])
            assert got[p]["status"] == 0
        g, f = got[2], full[2]
        assert g["status"] == plf.PLF_ERR_CAPACITY and g["estimated"] and not g["accepted"]
        assert (g["n_pt"], g["n_ls"]) == (f["n_pt"], f["n_ls"]) and np.array_equal(g["pt_pairs"], f["pt_pairs"][:5])
        assert np.array_equal(g["ls_pairs"], f["ls_pairs"]) and not g["pose_inc"].any()
        for k in ("err", "max_cov_eig", "t", "r", "ratio_inliers", "x_inc", "common_pt", "inl_ratio_pt"):
            assert np.asarray(g[k]).tobytes() == np.asarray(f[k]).tobytes()
        # the context stays usable
        same(fs.loop_closure_pose_batch(pairs, seq=seq)[2], full[2])


def lc_array(fs, pairs, keep):
    arr = (plf.plf_lc_problem * len(pairs))()
    for k, (kf0, kf1) in enumerate(pairs):
        k0, k1 = fs._lc_keyframe(kf0, keep), fs._lc_keyframe(kf1, keep)
        pp = np.full((4, 2), -7, np.int32); lp = np.full((4, 2), -7, np.int32)
        keep += [pp, lp]
        arr[k] = plf.plf_lc_problem(C.pointer(k0), C.pointer(k1), pp.ctypes.data, 4, lp.ctypes.data, 4, plf.plf_lc_result(), 12345)
        arr[k].out.accepted = 777
    return arr


def untouched(arr, keep):
    assert all(arr[k].status == 12345 and arr[k].out.accepted == 777 and arr[k].out.common_pt == 0 for k in range(len(arr)))
    assert all((a == -7).all() for a in keep if isinstance(a, np.ndarray) and a.dtype == np.int32)


def test_refusals_before_any_work(built):
    pairs = mixed_pairs(CAMS[0], seed=130)[:3]
    lcp = plf.plf_lc_params(1.0, 0.01, 0.3, 1.5, 35.0, 30.0)
    with seq_context() as fs:
        lib = fs.lib
        err = lambda: lib.plf_last_error(fs._ctx).decode()
        i32 = lambda v: (C.c_int32 * len(v))(*v)
        cases = [(-1, None, lambda a: None, "n_problems = -1"),
                 (3, i32([0, 4, 0]), lambda a: None, "problem 1: seq[1] = 4 outside [-1, 4)"),
                 (3, i32([0, -2, 0]), lambda a: None, "problem 1: seq[1] = -2"),
                 (3, None, lambda a: setattr(a[2], "kf0", None), "problem 2: bad arguments"),
                 (3, None, lambda a: setattr(a[1].kf1.contents, "pdesc", None), "problem 1: point arrays missing"),
                 (3, None, lambda a: setattr(a[1].kf0.contents, "eP", None), "problem 1: line arrays missing"),
                 (3, None, lambda a: setattr(a[0].kf0.contents, "n_pt", 70000), "problem 0: 70000 / 360 points"),
                 (3, None, lambda a: setattr(a[2].kf1.contents, "n_ls", -1), "problem 2: bad arguments")]
        for n, seq, spoil, msg in cases:
            keep = []
            arr = lc_array(fs, pairs, keep)
            spoil(arr)
            n0 = fs.launches
            assert lib.plf_loop_closure_pose_batch(fs._ctx, C.byref(lcp), n, arr, seq) == -1, msg
            assert msg in err() and fs.launches == n0
            untouched(arr, keep)
        keep = []
        arr = lc_array(fs, pairs, keep)
        assert lib.plf_loop_closure_pose_batch(fs._ctx, C.byref(lcp), 65536, arr, None) == plf.PLF_ERR_CAPACITY
        assert "65536 exceeds 65535" in err()
        untouched(arr, keep)
        n0 = fs.launches
        assert lib.plf_loop_closure_pose_batch(fs._ctx, C.byref(lcp), 0, None, None) == 0 and fs.launches == n0
        assert fs.loop_closure_pose_batch([]) == [] and fs.gn_pose_batch([]) == [] and fs.launches == n0
        # GN refusals
        g = synth.gn_problem(CAMS[0], seed=1)
        garr = (plf.plf_gn_problem * 2)()
        for k in range(2):
            garr[k] = plf.plf_gn_problem(g["P"].ctypes.data, g["obs"].ctypes.data, None, len(g["P"]))
            garr[k].out.iters1 = 555
        assert lib.plf_gn_pose_batch(fs._ctx, None, 2, garr, None) == -1 and "problem 0: np = 300, nl = 0" in err()
        assert lib.plf_gn_pose_batch(fs._ctx, None, -3, garr, None) == -1 and "n_problems = -3" in err()
        garr[0].np = 0; garr[1].np = 0
        assert lib.plf_gn_pose_batch(fs._ctx, None, 2, garr, i32([0, 9])) == -1 and "problem 1: seq[1] = 9" in err()
        assert garr[0].out.iters1 == 555 and garr[1].out.iters1 == 555 and fs.launches == n0
        # still usable
        same(fs.loop_closure_pose_batch(pairs[:1], seq=[0])[0], fs.loop_closure_pose_batch(pairs[:1], seq=np.zeros(1, np.int32))[0])


def test_launch_count_does_not_depend_on_the_batch(built):
    pairs = mixed_pairs(CAMS[0], seed=150)[:2]
    with seq_context() as fs:
        counts = []
        for P in (1, 64):
            batch = [pairs[p % 2] for p in range(P)]
            n0 = fs.launches
            fs.loop_closure_pose_batch(batch, seq=np.arange(P, dtype=np.int32) % 4)
            counts.append(fs.launches - n0)
        assert counts[0] == counts[1] == 9          # per kind: 2-NN both ways + NNR; rows, solver, decision
        g = synth.gn_problem(CAMS[0], seed=2)
        gp = dict(P=g["P"], pl_obs=g["obs"], sP=g["sP"], eP=g["eP"], le_obs=g["le"])
        for P in (1, 64):
            n0 = fs.launches
            fs.gn_pose_batch([gp] * P)
            assert fs.launches - n0 == 1


def gn_problems(c, seed):
    """Refinement problems rendered with CAMS[c]: plain, with given inlier flags and T_init, points only, zero rows."""
    out = []
    for k in range(3):
        g = synth.gn_problem(CAMS[c], n_pts=200 + 50 * k, n_lines=40 + 20 * k, seed=seed + k, outlier_frac=0.05 * k)
        d = dict(P=g["P"], pl_obs=g["obs"], sP=g["sP"], eP=g["eP"], le_obs=g["le"])
        if k == 1:
            rng = np.random.default_rng(seed)
            d["inlier_pt"] = (rng.random(len(g["P"])) > 0.2).astype(np.uint8)
            d["inlier_ls"] = (rng.random(len(g["sP"])) > 0.2).astype(np.uint8)
            d["T_init"] = synth.expmap_se3(np.array([0.01, 0.0, 0.5, 0.0, 0.01, 0.0]))
        if k == 2:
            d.update(sP=np.zeros((0, 3)), eP=np.zeros((0, 3)), le_obs=np.zeros((0, 3)))
        out.append(d)
    z = np.zeros((0, 3))
    out.append(dict(P=z, pl_obs=np.zeros((0, 2)), sP=z, eP=z, le_obs=z))   # zero rows: what the single call gives
    return out


def single_gn(fe, d, opts=None):
    return fe.gn_pose(d["P"], d["pl_obs"], d["sP"], d["eP"], d["le_obs"], d.get("inlier_pt"), d.get("inlier_ls"),
                      d.get("T_init"), opts=opts)


def test_gn_pose_batch_equals_single_calls(built):
    probs, seq = [], []
    for c in range(4):
        for d in gn_problems(c, seed=20 * c):
            probs.append(d); seq.append(c)
    seq = np.array(seq, np.int32)
    o = plf.plf_gn_opts(1e-7, 5, 10, 1e-7, 1e-7, plf.DBL_EPSILON)
    with seq_context() as fs:
        for opts in (None, o):
            got = fs.gn_pose_batch(probs, seq=seq, opts=opts)
            for c in range(4):
                with plf.Frontend(camera=CAMS[c], **GN_PRM) as fe:
                    for p in np.flatnonzero(seq == c):
                        assert got[p]["status"] == 0
                        same(got[p], single_gn(fe, probs[p], opts))
        # seq semantics: NULL, -1 and sequences set to the context's camera agree; permuted order and duplicates too
        with plf.Frontend(camera=BASE, **GN_PRM) as fe:
            ref = [single_gn(fe, d) for d in probs]
        for s in range(4):
            fs.set_sequence_camera(s, None)
        a = fs.gn_pose_batch(probs)
        b = fs.gn_pose_batch(probs, seq=np.full(len(probs), -1, np.int32))
        c_ = fs.gn_pose_batch(probs, seq=seq)
        for x, y, z, r in zip(a, b, c_, ref):
            same(x, r); same(y, r); same(z, r)
        perm = np.random.default_rng(5).permutation(len(probs))
        got = fs.gn_pose_batch([probs[i] for i in list(perm) + [0]])
        for j, i in enumerate(list(perm) + [0]):
            same(got[j], ref[i])
        same(fs.gn_pose_batch([probs[3]])[0], ref[3])
        assert np.isnan(ref[3]["err"])                    # zero rows: 0 / 0, as plf_gn_pose gives it
