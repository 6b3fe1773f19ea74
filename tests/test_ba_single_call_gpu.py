"""GPU tests of plf_local_ba and plf_global_ba as the one-problem case of the batched driver (csrc/lba.cu): a single
call enqueues the launches of a batch of one, on bench_local_ba_batch.py's local maps and on a global map over 64
keyframes (the tiled factorisation), and its refusals, on the host and on the device, are worded for the single call:
"plf_local_ba: <rule>" / "plf_global_ba: <rule>", with no problem index."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import gba
from plslam_b200 import synth
from test_gba_gpu import _raw_args
from test_lba_edges import orphan_map, zero_block_map

pytestmark = pytest.mark.gpu
CAM = plf.KITTI_CAMERA
PLF_ERR_INVALID = -1
GLOBAL = "plf_global_ba"
LOCAL = "plf_local_ba"


def _launches(fe, run):
    n0 = fe.launches
    run()
    return fe.launches - n0


@pytest.mark.parametrize("quirks", [1, 0])
def test_local_ba_launches_what_a_batch_of_one_launches(fe, quirks):
    """bench_local_ba_batch.py's maps (5 + p % 6 local keyframes, 2 fixed, 100 points and 20 lines per keyframe)"""
    for i in (0, 5):
        p = synth.local_map_problem(CAM, n_kf=5 + i, n_fixed=2, pts_per_kf=100, ls_per_kf=20, seed=1000 + i)
        one = _launches(fe, lambda: fe.local_ba(p, ref_quirks=quirks))
        batch = _launches(fe, lambda: fe.local_ba_batch([p], ref_quirks=quirks))
        assert one == batch, (i, one, batch)


@pytest.mark.parametrize("quirks", [1, 0])
def test_global_ba_over_64_keyframes_launches_what_a_batch_of_one_launches(fe, quirks):
    p = synth.gba_problem(CAM, n_kf=100, pts_per_kf=4, ls_per_kf=1, seed=9)
    one = _launches(fe, lambda: fe.global_ba(p, ref_quirks=quirks))
    batch = _launches(fe, lambda: fe.global_ba_batch([p], ref_quirks=quirks))
    assert one == batch, (one, batch)


def _raw_single(fe, fn, p):
    """plf_local_ba / plf_global_ba through ctypes: (return code, last error, whether any input array or out changed)"""
    keep = []
    prob = plf.plf_lba_problem(**_raw_args(p, keep))
    before = [a.copy() for a in keep]
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, gba.DBL_EPSILON, gba.DBL_EPSILON, 1)
    res = plf.plf_lba_result()
    rc = getattr(fe.lib, fn)(fe._ctx, C.byref(o), C.byref(prob), C.byref(res))
    changed = any(not np.array_equal(a, b) for a, b in zip(keep, before)) or bool(res.iters or res.err or res.lambda_)
    return rc, fe.lib.plf_last_error(fe._ctx).decode(), changed


def _landmark(q, kind, lm):
    return f"point landmark {lm}" if kind == "pt" else f"line landmark {lm - len(q['pt'])}"


@pytest.mark.parametrize("fn", [LOCAL, GLOBAL])
@pytest.mark.parametrize("kind", ["pt", "ls"])
def test_refusals_name_the_single_call(fe, fn, kind):
    """a landmark without observations (refused on the host) and one whose first-pass block has a zero diagonal entry
    (refused on the device): the message is the single call's, and nothing is written"""
    q, lm = orphan_map(kind)
    rc, msg, changed = _raw_single(fe, fn, q)
    assert rc == PLF_ERR_INVALID and not changed
    assert msg == f"{fn}: {_landmark(q, kind, lm)} has no observation", msg
    q, lm = zero_block_map(kind)
    rc, msg, changed = _raw_single(fe, fn, q)
    assert rc == PLF_ERR_INVALID and not changed
    assert msg == (f"{fn}: {_landmark(q, kind, lm)} has a zero diagonal entry in its first-pass block "
                   "(no row constrains it)"), msg


@pytest.mark.parametrize("fn", [LOCAL, GLOBAL])
def test_bad_arguments_name_the_single_call(fe, fn):
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, 1e-7, 1e-7, 1)
    assert getattr(fe.lib, fn)(fe._ctx, C.byref(o), None, None) == PLF_ERR_INVALID
    assert fe.lib.plf_last_error(fe._ctx).decode() == f"{fn}: bad arguments"
