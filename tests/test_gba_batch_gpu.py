"""GPU parity of the batched global bundle adjustment (plf_global_ba_batch, csrc/lba.cu) with oracle/gba.py and with
plf_global_ba, each problem with its camera: mixed sizes on both factorisations, per-sequence cameras, independence from
the neighbours in the batch, both (g2) edges, the per-problem refusal found on the device, the refusals before any work,
a launch count that does not grow with the batch, the batched tiled LDL^T against the single one, 2048-keyframe maps
and the pipeline around a call.  The batches come from tests/test_gba_batch.py, which checks them on the CPU."""
import ctypes as C

import numpy as np
import pytest

import ldlt_cases as lc
import plslam_b200 as plf
import test_gba_oracle as g2
from oracle import clib, gba
from oracle import synth as osynth
from plslam_b200 import synth
from test_gba_batch import GBA_CAMS, camera_batch, mixed_batch, opts_kw, oracle_run, seq_camera
from test_gba_gpu import _check, _raw_args
from test_lba_edges import orphan_map, zero_block_map

pytestmark = pytest.mark.gpu
CAM = plf.KITTI_CAMERA
PLF_ERR_INVALID = -1
PLF_ERR_CAPACITY = -4
PLF_ERR_CUDA = -3


@pytest.fixture(scope="module")
def fe4(built):
    """a four-sequence context, each sequence with its GBA_CAMS calibration"""
    f = plf.Frontend(device=0, max_sequences=4)
    for s, cam in enumerate(GBA_CAMS):
        f.set_sequence_camera(s, cam)
    yield f
    f.close()


@pytest.mark.parametrize("quirks", [1, 0])
def test_mixed_sizes_match_the_oracle(fe, quirks):
    probs = mixed_batch()
    got = fe.global_ba_batch(probs, **opts_kw(quirks))
    for i, (p, g) in enumerate(zip(probs, got)):
        ref, _, _ = oracle_run("mixed", i, quirks)
        assert g["status"] == 0
        _check(p, g, ref)


@pytest.mark.parametrize("quirks", [1, 0])
def test_sequence_cameras(fe4, quirks):
    probs, seq = camera_batch()
    got = fe4.global_ba_batch(probs, seq=np.array(seq), **opts_kw(quirks))
    for i, (p, g) in enumerate(zip(probs, got)):
        assert g["status"] == 0
        _check(p, g, oracle_run("camera", i, quirks)[0])
    # each problem agrees with plf_global_ba on a context created with its camera
    for s in sorted(set(seq)):
        with plf.Frontend(device=0, camera=seq_camera(s)) as one:
            for i in [i for i, t in enumerate(seq) if t == s]:
                _check(probs[i], got[i], one.global_ba(probs[i], **opts_kw(quirks)))


def test_neighbours_do_not_matter(fe):
    probs = [mixed_batch()[i] for i in (0, 1, 3, 5)]
    fwd = fe.global_ba_batch(probs)
    rev = fe.global_ba_batch(probs[::-1])[::-1]
    for p, a, b in zip(probs, fwd, rev):
        _check(p, a, b)
    for p, a in zip(probs, fwd):
        (alone,) = fe.global_ba_batch([p])
        _check(p, a, alone)
        _check(p, alone, fe.global_ba(p))


def test_g2_edges_in_one_batch(built):
    """(g2) below 1: lambda = 0; beyond 2^31 on the last diagonal entry, through sequence 0's camera: lambda_0 INT_MIN"""
    small, big = g2.g2_small_problem(), g2.g2_big_problem()
    with plf.Frontend(device=0, max_sequences=1) as f:
        f.set_sequence_camera(0, g2.g2_big_cam())
        a, b = f.global_ba_batch([small, big], seq=[-1, 0], max_iters=1, ref_quirks=1)
        assert a["status"] == b["status"] == 0
        assert a["lambda_"] == 0.0 == gba.global_ba(CAM, small, gba.opts(max_iters=1))["lambda_"]
        assert b["lambda_"] == 1e-5 * gba.INT_MIN
        _check(big, b, gba.global_ba(g2.g2_big_cam(), big, gba.opts(ref_quirks=1, max_iters=1)))
        (c,) = f.global_ba_batch([small], max_iters=1, ref_quirks=0)
        _check(small, c, gba.global_ba(CAM, small, gba.opts(ref_quirks=0, max_iters=1)))


@pytest.mark.parametrize("kind", ["pt", "ls"])
def test_zero_block_refuses_its_problem_only(fe, kind):
    q, lm = zero_block_map(kind)
    probs = [mixed_batch()[i] for i in (1, 3)]
    probs.insert(1, q)
    keep = []
    args = [plf.plf_lba_problem(**_raw_args(p, keep)) for p in probs]
    before = [a.copy() for a in keep]
    arr = (plf.plf_lba_problem * 3)(*args)
    out = (plf.plf_lba_result * 3)()
    st = np.full(3, 7, np.int32)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, gba.DBL_EPSILON, gba.DBL_EPSILON, 1)
    rc = fe.lib.plf_global_ba_batch(fe._ctx, C.byref(o), 3, arr, None, out, st.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == PLF_ERR_INVALID
    assert st.tolist() == [0, PLF_ERR_INVALID, 0]
    msg = fe.lib.plf_last_error(fe._ctx).decode()
    n_pt = len(q["pt"])
    name = f"point landmark {lm}" if kind == "pt" else f"line landmark {lm - n_pt}"
    assert "plf_global_ba_batch: problem 1" in msg and name in msg and "zero diagonal" in msg, msg
    assert out[1].iters == 0 and out[1].err == 0.0 and out[1].lambda_ == 0.0
    n_arrays = len(keep) // 3
    for a, b in zip(keep[n_arrays:2 * n_arrays], before[n_arrays:2 * n_arrays]):
        assert np.array_equal(a, b)
    got = fe.global_ba_batch(probs)
    assert [g["status"] for g in got] == [0, PLF_ERR_INVALID, 0]
    assert np.array_equal(got[1]["pt"], q["pt"]) and got[1]["iters"] is None
    for i in (0, 2):
        _check(probs[i], got[i], gba.global_ba(CAM, probs[i], gba.opts()))


def _raw_batch(f, probs, seq=None, n=None):
    """plf_global_ba_batch through ctypes: (return code, whether any input array, out or status changed)"""
    keep = []
    args = [plf.plf_lba_problem(**_raw_args(p, keep)) for p in probs]
    before = [a.copy() for a in keep]
    m = len(probs)
    arr = (plf.plf_lba_problem * max(m, 1))(*args)
    out = (plf.plf_lba_result * max(m, 1))()
    st = np.full(max(m, 1), 7, np.int32)
    s = None if seq is None else np.asarray(seq, np.int32)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, gba.DBL_EPSILON, gba.DBL_EPSILON, 1)
    rc = f.lib.plf_global_ba_batch(f._ctx, C.byref(o), m if n is None else n, arr,
                                   None if s is None else s.ctypes.data_as(C.POINTER(C.c_int32)), out,
                                   st.ctypes.data_as(C.POINTER(C.c_int32)))
    changed = (any(not np.array_equal(a, b) for a, b in zip(keep, before)) or np.any(st != 7)
               or any(r.iters or r.err or r.lambda_ for r in out))
    return rc, changed


def test_refusals_before_any_work(fe4):
    base = [mixed_batch()[i] for i in (0, 1, 3)]
    big = synth.gba_problem(CAM, n_kf=4097, pts_per_kf=1, ls_per_kf=0, seed=1, loop=False)
    empty = dict(base[0], pt_obs_lm=np.zeros(0, np.int32), pt_obs_kf=np.zeros(0, np.int32), pt_obs_xy=np.zeros((0, 2)),
                 ls_obs_lm=np.zeros(0, np.int32), ls_obs_kf=np.zeros(0, np.int32), ls_obs_le=np.zeros((0, 3)))
    lm = base[1]["pt_obs_lm"].copy(); lm[-1] = len(base[1]["pt"])
    cases = [(base[:1] + [orphan_map("pt")[0]] + base[1:], None, PLF_ERR_INVALID, "problem 1: point landmark"),
             (base[:2] + [orphan_map("ls")[0]], None, PLF_ERR_INVALID, "problem 2: line landmark"),
             (base + [dict(base[1], pt_obs_lm=base[1]["pt_obs_lm"][::-1].copy())], None, PLF_ERR_INVALID, "problem 3: observations must be grouped"),
             ([dict(base[1], pt_obs_lm=lm)] + base, None, PLF_ERR_INVALID, "problem 0: observation"),
             (base + [empty], None, PLF_ERR_INVALID, "problem 3: empty problem"),
             (base + [big], None, PLF_ERR_CAPACITY, "problem 3: 4097 keyframes (limit 4096)"),
             (base, [0, 4, 1], PLF_ERR_INVALID, "seq[1] = 4"),
             (base, [0, -2, 1], PLF_ERR_INVALID, "seq[1] = -2")]

    def usable():
        for p, g in zip(base, fe4.global_ba_batch(base)):
            _check(p, g, gba.global_ba(CAM, p, gba.opts()))

    for probs, seq, code, msg in cases:
        rc, changed = _raw_batch(fe4, probs, seq)
        assert rc == code and not changed, (msg, rc)
        assert msg in fe4.lib.plf_last_error(fe4._ctx).decode(), fe4.lib.plf_last_error(fe4._ctx).decode()
        usable()
    keep = []   # a NULL array with a non-zero count
    args = _raw_args(base[1], keep, null="pt_obs_xy")
    arr = (plf.plf_lba_problem * 2)(plf.plf_lba_problem(**_raw_args(base[0], keep)), plf.plf_lba_problem(**args))
    st = np.full(2, 7, np.int32)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, gba.DBL_EPSILON, gba.DBL_EPSILON, 1)
    rc = fe4.lib.plf_global_ba_batch(fe4._ctx, C.byref(o), 2, arr, None, None, st.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == PLF_ERR_INVALID and st.tolist() == [7, 7] and "problem 1: null array" in fe4.lib.plf_last_error(fe4._ctx).decode()
    assert _raw_batch(fe4, base, n=-1) == (PLF_ERR_INVALID, False)
    assert _raw_batch(fe4, base, n=65536)[0] == PLF_ERR_CAPACITY
    assert _raw_batch(fe4, []) == (0, False)
    usable()
    assert fe4.global_ba_batch([]) == []


def test_scratch_that_does_not_fit_fails_and_the_context_stays_usable(fe):
    """twenty 4096-keyframe maps need 20 x 4.8 GB of dense reduced systems, more than the card holds"""
    big = synth.gba_problem(CAM, n_kf=4096, pts_per_kf=1, ls_per_kf=0, seed=1, loop=False)
    rc, changed = _raw_batch(fe, [big] * 20)
    assert rc == PLF_ERR_CUDA and not changed and "scratch" in fe.lib.plf_last_error(fe._ctx).decode()
    probs = [mixed_batch()[i] for i in (0, 3)]
    for p, g in zip(probs, fe.global_ba_batch(probs)):
        _check(p, g, gba.global_ba(CAM, p, gba.opts()))


def test_launch_count_does_not_grow_with_the_batch(fe):
    """at fixed max_iters and largest tile count (a 100-keyframe map in both), 2 or 16 problems cost the same launches"""
    probs = [synth.gba_problem(CAM, n_kf=100, pts_per_kf=4, ls_per_kf=1, seed=9)]
    probs += [synth.gba_problem(CAM, n_kf=3 + i % 40 + 30 * (i % 3), pts_per_kf=4, ls_per_kf=1, seed=300 + i) for i in range(15)]
    counts = []
    for n in (2, 16):
        n0 = fe.launches
        got = fe.global_ba_batch(probs[:n], max_iters=4)
        counts.append(fe.launches - n0)
        assert all(g["status"] == 0 for g in got)
    assert counts[0] == counts[1], counts


def test_batched_ldlt_is_the_single_one_bit_for_bit(fe):
    """plf_debug_ldlt_batch on mixed sizes and patterns equals plf_debug_ldlt path 0 on each matrix, in L, D, x and nz"""
    sizes = (11, 65, 96, 200, 266, 1)
    mats = []
    for i, n6 in enumerate(sizes):
        pat = lc.PATTERNS[(3 * i) % len(lc.PATTERNS)]
        S, g, _ = lc.make(lc.Case(pat, lc.VALUES[i % len(lc.VALUES)], n6, seed=i))
        mats.append((S, g))
    for order in (mats, mats[::-1]):
        got = fe.debug_ldlt_batch(order)
        for (S, g), (LD, x, nz) in zip(order, got):
            LD1, x1, nz1 = fe.debug_ldlt(S, g, 0)
            low = np.tril_indices(len(S))
            assert np.array_equal(LD[low].view(np.uint64), LD1[low].view(np.uint64))
            assert np.array_equal(x.view(np.uint64), x1.view(np.uint64))
            assert np.array_equal(nz, nz1)
    assert fe.debug_ldlt_batch([]) == []


def _first_step_residual(p, got, quirks):
    """|H DX - g| / |g| of the step recovered from the output, on the damped first-pass system assembled by scipy.sparse
    from the oracle's rows, as tests/test_gba_gpu.py's 2048-keyframe test computes it"""
    import scipy.sparse as sp
    nkf = len(p["kf_pose"])
    X0 = np.concatenate([p["kf_pose"].ravel(), p["pt"].ravel(), p["ls"].ravel()])
    T0inv = np.stack([gba._pose_inv(x) for x in p["kf_pose"]])
    Hl, g, _ = gba.normal_equations(CAM, p, X0, T0inv, True, bool(quirks), 1e-7)
    dg = Hl.diagonal()
    lam = 1e-5 * (gba.hmax_int(dg) if quirks else np.abs(dg).max())
    assert got["lambda_"] == pytest.approx(lam, rel=1e-9)
    Hl = Hl + sp.diags(lam * dg)
    H = (Hl + Hl.T - sp.diags(Hl.diagonal())).tocsr()
    dk = np.stack([clib.logmap_se3(clib.inverse_se3(clib.expmap_se3(a)) @ clib.expmap_se3(b))
                   for a, b in zip(got["kf_pose"], p["kf_pose"])])
    DX = np.concatenate([dk.ravel(), np.concatenate([got["pt"].ravel(), got["ls"].ravel()]) - X0[6 * nkf:]])
    return np.linalg.norm(H @ DX - g) / np.linalg.norm(g)


@pytest.mark.parametrize("quirks", [0, 1])
def test_two_2048_keyframe_maps_one_step_each(fe, quirks):
    """max_iters = 1 on tests/test_gba_gpu.py's 2048-keyframe map (192 tile columns), twice, around a small map: each
    large step solves its damped system to 1e-8, and the small one is the oracle's first step"""
    big = synth.gba_problem(CAM, n_kf=2048, pts_per_kf=40, ls_per_kf=6, seed=5)
    small = synth.gba_problem(CAM, n_kf=30, pts_per_kf=10, ls_per_kf=3, seed=7)
    got = fe.global_ba_batch([big, small, big], max_iters=1, ref_quirks=quirks)
    assert [g["status"] for g in got] == [0, 0, 0] and [g["iters"] for g in got] == [1, 1, 1]
    for g in (got[0], got[2]):
        assert _first_step_residual(big, g, quirks) <= 1e-8
    _check(small, got[1], gba.global_ba(CAM, small, gba.opts(ref_quirks=quirks, max_iters=1)))


def test_global_ba_batch_between_batches_leaves_the_pipeline_unchanged(built):
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = osynth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    frames = list(osynth.stream(cam, 8, world=world, seed=5, step=0.1))
    L = np.stack([f[0] for f in frames]); R = np.stack([f[1] for f in frames])
    lim = plf.default_limits(); lim.max_batch = 2
    probs = [synth.gba_problem(cam, n_kf=80, pts_per_kf=10, ls_per_kf=3, seed=4),
             synth.gba_problem(cam, n_kf=20, pts_per_kf=10, ls_per_kf=3, seed=5)]

    def run(with_gba):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=500, lsd_nfeatures=100) as f:
            out, ba = [], None
            for b in range(0, 8, 2):
                f.batch_upload(L[b:b + 2], R[b:b + 2])
                f.batch_run(2)
                if with_gba and b == 4:   # two batches, global_ba_batch with the third in flight, two batches
                    ba = f.global_ba_batch(probs)
                res = f.batch_download_array(2)
                out += [np.ascontiguousarray(res[k]) for k in res.dtype.names]
                out += [np.ascontiguousarray(a) for a in f.get_frame(1).values() if isinstance(a, np.ndarray)]
            return out, ba

    (a, _), (b, ba) = run(False), run(True)
    assert len(a) == len(b) and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    with plf.Frontend(camera=cam) as f:
        for p, got in zip(probs, ba):
            _check(p, got, f.global_ba(p))
