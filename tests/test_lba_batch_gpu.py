"""GPU parity of the batched local bundle adjustment (plf_local_ba_batch, csrc/lba.cu) with oracle/lba.c, each problem with
its camera: mixed batches that stop at different iterations and by different exits, every host-loop branch, per-sequence
cameras, independence from the neighbours in the batch, the per-problem refusal found on the device, the refusals before
any work, and a launch count that does not grow with the batch.  The batches come from tests/test_lba_batch.py, which
checks them on the CPU."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib
from plslam_b200 import synth
from test_gba_gpu import _raw_args
from test_lba_batch import (MIXED_MAX_ITERS, SEQ_CAMS, camera_batch, mixed_batch, oracle_run, seq_camera)
from test_lba_edges import BRANCH_MAP, BRANCHES, branch_case, decidable, orphan_map, took, zero_block_map

pytestmark = pytest.mark.gpu
CAM = plf.KITTI_CAMERA
TOL = 1e-6
PLF_ERR_INVALID = -1
PLF_ERR_CAPACITY = -4
BRANCH_EXTRA = [dict(n_kf=7, seed=3), dict(seed=12), dict(seed=14)]   # beside BRANCH_MAP: maps that take every branch too


def _check(p, got, ref):
    """as tests/test_lba_gpu.py: exact iters and moved flags, 1e-6 of the step on every block, lambda and err to 1e-9"""
    assert got["iters"] == ref["iters"]
    for k in ("kf_pose", "pt", "ls"):
        if ref[k].size:
            step = np.abs(ref[k] - p[k]).max()
            assert np.abs(got[k] - ref[k]).max() <= TOL * max(step, 1e-3), k
    assert np.array_equal(got["pt_moved"], ref["pt_moved"]) and np.array_equal(got["ls_moved"], ref["ls_moved"])
    assert abs(got["lambda_"] - ref["lambda_"]) <= 1e-9 * abs(ref["lambda_"])
    if np.isfinite(ref["err"]):
        assert abs(got["err"] - ref["err"]) <= 1e-9 * abs(ref["err"])


@pytest.fixture(scope="module")
def fe4(built):
    """a four-sequence context: sequences 0-2 with SEQ_CAMS, sequence 3 on the context's camera"""
    f = plf.Frontend(device=0, max_sequences=4)
    for s, cam in enumerate(SEQ_CAMS):
        f.set_sequence_camera(s, cam)
    yield f
    f.close()


@pytest.mark.parametrize("quirks", [1, 0])
def test_mixed_batch_matches_the_oracle(fe, quirks):
    probs = mixed_batch()
    got = fe.local_ba_batch(probs, max_iters=MIXED_MAX_ITERS, ref_quirks=quirks)
    iters = set()
    for i, (p, g) in enumerate(zip(probs, got)):
        ref, o = oracle_run("mixed", i, quirks, MIXED_MAX_ITERS)
        assert ref["rc"] == 0 and decidable(ref["trace"], o)
        assert g["status"] == 0
        _check(p, g, ref)
        iters.add(g["iters"])
    if quirks:
        assert len(iters) > 2   # the problems stopped at different iterations


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("name", [b[0] for b in BRANCHES])
def test_every_exit_in_a_batch(fe, name, quirks):
    """3-4 maps under the branch's opts, each taking the branch on the oracle"""
    p0, okw = branch_case(name, quirks)
    _, mkw, _, what = [b for b in BRANCHES if b[0] == name][0]
    probs = [p0] + [synth.local_map_problem(CAM, **dict(BRANCH_MAP, **kw, **mkw)) for kw in BRANCH_EXTRA]
    o = clib.lba_opts(**okw)
    refs = [clib.local_ba(CAM, p, o) for p in probs]
    for r in refs:
        assert r["rc"] == 0 and decidable(r["trace"], o) and took(r["trace"], what), r["trace"]
    got = fe.local_ba_batch(probs, **okw)
    for p, g, r in zip(probs, got, refs):
        assert g["status"] == 0
        _check(p, g, r)


@pytest.mark.parametrize("quirks", [1, 0])
def test_sequence_cameras(fe4, quirks):
    probs, seq = camera_batch()
    got = fe4.local_ba_batch(probs, seq=np.array(seq), ref_quirks=quirks)
    for i, (p, g) in enumerate(zip(probs, got)):
        ref, _ = oracle_run("camera", i, quirks)
        assert g["status"] == 0
        _check(p, g, ref)
    # seq = None: the context's camera
    ctx_probs = [p for p, s in zip(probs, seq) if seq_camera(s) is CAM]
    ctx_idx = [i for i, s in enumerate(seq) if seq_camera(s) is CAM]
    for i, p, g in zip(ctx_idx, ctx_probs, fe4.local_ba_batch(ctx_probs, ref_quirks=quirks)):
        _check(p, g, oracle_run("camera", i, quirks)[0])
    # a problem routed to sequence s agrees with the same problem on a context created with s's camera
    for s, cam in enumerate(SEQ_CAMS):
        with plf.Frontend(device=0, camera=cam) as one:
            for i in [i for i, t in enumerate(seq) if t == s]:
                _check(probs[i], got[i], one.local_ba(probs[i], ref_quirks=quirks))


def test_neighbours_do_not_matter(fe):
    probs = mixed_batch()[:6] + mixed_batch()[11:16]
    fwd = fe.local_ba_batch(probs)
    rev = fe.local_ba_batch(probs[::-1])[::-1]
    for p, a, b in zip(probs, fwd, rev):
        _check(p, a, b)
    for p, a in zip(probs, fwd):
        (alone,) = fe.local_ba_batch([p])
        _check(p, a, alone)
        _check(p, alone, fe.local_ba(p))


@pytest.mark.parametrize("kind", ["pt", "ls"])
def test_zero_block_refuses_its_problem_only(fe, kind):
    q, lm = zero_block_map(kind)
    probs = list(mixed_batch()[11:15])
    probs.insert(2, q)
    keep = []
    args = [plf.plf_lba_problem(**_raw_args(p, keep)) for p in probs]
    before = [a.copy() for a in keep]
    arr = (plf.plf_lba_problem * len(probs))(*args)
    out = (plf.plf_lba_result * len(probs))()
    st = np.full(len(probs), 7, np.int32)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, 1e-7, 1e-7, 1)
    rc = fe.lib.plf_local_ba_batch(fe._ctx, C.byref(o), len(probs), arr, None, out, st.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == PLF_ERR_INVALID
    assert st.tolist() == [0, 0, PLF_ERR_INVALID, 0, 0]
    msg = fe.lib.plf_last_error(fe._ctx).decode()
    n_pt = len(q["pt"])
    name = f"point landmark {lm}" if kind == "pt" else f"line landmark {lm - n_pt}"
    assert "problem 2" in msg and name in msg and "zero diagonal" in msg, msg
    assert out[2].iters == 0 and out[2].err == 0.0 and out[2].lambda_ == 0.0
    n_arrays = len(keep) // len(probs)
    for a, b in zip(keep[2 * n_arrays:3 * n_arrays], before[2 * n_arrays:3 * n_arrays]):
        assert np.array_equal(a, b)
    # the others are solved; through the binding, the refused problem's dict holds its inputs
    got = fe.local_ba_batch(probs)
    assert [g["status"] for g in got] == [0, 0, PLF_ERR_INVALID, 0, 0]
    assert np.array_equal(got[2]["pt"], q["pt"]) and got[2]["iters"] is None
    for i, (p, g) in enumerate(zip(probs, got)):
        if i != 2:
            _check(p, g, clib.local_ba(CAM, p, clib.lba_opts()))
    _next_batch_is_correct(fe)


def _next_batch_is_correct(fe):
    probs = mixed_batch()[16:19]
    for p, g in zip(probs, fe.local_ba_batch(probs)):
        _check(p, g, clib.local_ba(CAM, p, clib.lba_opts()))


def _raw_batch(f, probs, seq=None):
    """plf_local_ba_batch through ctypes: (return code, whether any input array, out or status changed)"""
    keep = []
    args = [plf.plf_lba_problem(**_raw_args(p, keep)) for p in probs]
    before = [a.copy() for a in keep]
    n = len(probs)
    arr = (plf.plf_lba_problem * max(n, 1))(*args)
    out = (plf.plf_lba_result * max(n, 1))()
    st = np.full(max(n, 1), 7, np.int32)
    s = None if seq is None else np.asarray(seq, np.int32)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, 1e-7, 1e-7, 1)
    rc = f.lib.plf_local_ba_batch(f._ctx, C.byref(o), n, arr, None if s is None else s.ctypes.data_as(C.POINTER(C.c_int32)),
                                  out, st.ctypes.data_as(C.POINTER(C.c_int32)))
    changed = (any(not np.array_equal(a, b) for a, b in zip(keep, before)) or np.any(st != 7)
               or any(r.iters or r.err or r.lambda_ for r in out))
    return rc, changed


def test_refusals_before_any_work(fe4):
    base = list(mixed_batch()[16:19])
    big = synth.local_map_problem(CAM, n_kf=65, n_fixed=1, pts_per_kf=1, ls_per_kf=0, seed=1)
    cases = [(base[:1] + [orphan_map("pt")[0]] + base[1:], None, PLF_ERR_INVALID, "problem 1: point landmark"),
             (base[:2] + [orphan_map("ls")[0]], None, PLF_ERR_INVALID, "problem 2: line landmark"),
             (base + [big], None, PLF_ERR_CAPACITY, "problem 3: 65 keyframes"),
             (base, [0, 4, 1], PLF_ERR_INVALID, "seq[1] = 4"),
             (base, [0, -2, 1], PLF_ERR_INVALID, "seq[1] = -2")]
    for probs, seq, code, msg in cases:
        rc, changed = _raw_batch(fe4, probs, seq)
        assert rc == code and not changed, (msg, rc)
        assert msg in fe4.lib.plf_last_error(fe4._ctx).decode()
        for p, g in zip(base, fe4.local_ba_batch(base)):
            _check(p, g, clib.local_ba(CAM, p, clib.lba_opts()))
    assert _raw_batch(fe4, []) == (0, False)
    assert fe4.local_ba_batch([]) == []
    with pytest.raises(plf.PlfError, match="seq"):
        fe4.local_ba_batch(base, seq=[0, 1])
    with pytest.raises(plf.PlfError, match="orphan|no observation"):
        fe4.local_ba_batch([orphan_map("pt")[0]])


def test_launch_count_does_not_grow_with_the_batch(fe):
    probs = [synth.local_map_problem(CAM, n_kf=5 + i % 6, n_fixed=2, seed=300 + i) for i in range(64)]
    counts = []
    for n in (2, 64):
        n0 = fe.launches
        got = fe.local_ba_batch(probs[:n], max_iters=6)
        counts.append(fe.launches - n0)
        assert all(g["status"] == 0 for g in got)
    assert counts[0] == counts[1], counts
