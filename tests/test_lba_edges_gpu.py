"""GPU parity of the local bundle adjustment (plf_local_ba, csrc/lba.cu) with oracle/lba.c on maps shaped like the
reference's local maps (synth.local_map_problem: a sliding window, 20-40 % of the landmarks seen once, fixed keyframes
that are earlier keyframes), at the keyframe counts where lba_solve's strided loops change (one pass up to 42, a
second from 43) up to its limit of 64, at every exit and branch of the LM control, with rows on the clamps and signs of
lba_rows, and the refusals, after each of which the context stays usable.  Maps come from tests/test_lba_edges.py,
which checks them on the CPU."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, gba
from plslam_b200 import synth
from test_gba_gpu import _raw_args
from test_lba_edges import (BACKWARD_MAPS, BRANCHES, branch_case, decidable, edge_map, first_step_residual, orphan_map,
                            took, zero_block_map)

pytestmark = pytest.mark.gpu
CAM = plf.KITTI_CAMERA
TOL = 1e-6
PLF_ERR_INVALID = -1
PLF_ERR_CAPACITY = -4


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


def _run(fe, p, **kw):
    """the oracle (its run asserted decidable: no stop decision within rounding of its threshold) and the device"""
    o = clib.lba_opts(**kw)
    ref = clib.local_ba(CAM, p, o)
    assert ref["rc"] == 0 and decidable(ref["trace"], o), ref["trace"]
    _check(p, fe.local_ba(p, **kw), ref)
    return ref


# (n_kf, n_fixed, points / lines per keyframe, t0): N = 6 n_kf + 3 n_pt + 6 n_ls stays below 1 500 for the dense oracle
PARITY = [(1, 2, 6, 2, 0), (1, 3, 6, 0, 4), (9, 3, 6, 2, 2), (9, 0, 6, 2, 0), (42, 4, 3, 1, 0), (43, 2, 3, 1, 5),
          (43, 3, 4, 0, 0), (43, 0, 3, 1, 0), (64, 4, 3, 1, 0), (64, 2, 4, 0, 3), (64, 0, 3, 1, 0)]


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("n_kf,n_fixed,ppk,lpk,t0", PARITY)
def test_local_map_matches_the_oracle(fe, n_kf, n_fixed, ppk, lpk, t0, quirks):
    p = synth.local_map_problem(CAM, n_kf=n_kf, n_fixed=n_fixed, pts_per_kf=ppk, ls_per_kf=lpk, t0=t0,
                                seed=n_kf + 7 * n_fixed + t0)
    _run(fe, p, ref_quirks=quirks)


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("n_kf", [43, 64])
def test_one_step_solves_the_damped_system(fe, n_kf, quirks):
    """max_iters = 1: the step recovered from the output solves the damped first pass, assembled by scipy.sparse from
    oracle/gba.py's rows (LBA's first pass in both modes), to 1e-8 - with a third of the landmarks seen once"""
    p = synth.local_map_problem(CAM, **BACKWARD_MAPS[n_kf])
    got = fe.local_ba(p, max_iters=1, ref_quirks=quirks)
    res, lam = first_step_residual(p, got)
    assert got["iters"] == 1 and got["lambda_"] == pytest.approx(lam, rel=1e-9)
    assert res <= 1e-8, res


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("name", [b[0] for b in BRANCHES])
def test_every_host_loop_branch_matches_the_oracle(fe, name, quirks):
    p, okw = branch_case(name, quirks)
    ref = _run(fe, p, **okw)
    assert took(ref["trace"], [b for b in BRANCHES if b[0] == name][0][3]), ref["trace"]


@pytest.mark.parametrize("quirks", [1, 0])
@pytest.mark.parametrize("homog_th", [1e-7, 1e-3])
def test_clamp_and_sign_edges_match_the_oracle(fe, homog_th, quirks):
    _run(fe, edge_map(homog_th), ref_quirks=quirks, homog_th=homog_th)


def _raw_local(fe, prob_kw):
    p = plf.plf_lba_problem(**prob_kw)
    o = plf.plf_lba_opts(1e-5, 10.0, 15, 1e-7, 1e-7, 1e-7, 1)
    res = plf.plf_lba_result()
    return fe.lib.plf_local_ba(fe._ctx, C.byref(o), C.byref(p), C.byref(res))


def test_local_ba_rejects_bad_input_and_stays_usable(fe):
    p = synth.local_map_problem(CAM, n_kf=6, n_fixed=2, seed=2)
    want = clib.local_ba(CAM, p, clib.lba_opts())

    def valid():
        _check(p, fe.local_ba(p), want)

    keep = []
    big = synth.local_map_problem(CAM, n_kf=65, n_fixed=1, pts_per_kf=1, ls_per_kf=0, seed=1)
    assert _raw_local(fe, _raw_args(big, keep)) == PLF_ERR_CAPACITY
    valid()
    for field in ("kf_pose", "pt", "ls", "fixed_T", "pt_obs_lm", "pt_obs_kf", "pt_obs_xy", "ls_obs_lm", "ls_obs_kf",
                  "ls_obs_le"):
        keep = []
        assert _raw_local(fe, _raw_args(p, keep, null=field)) == PLF_ERR_INVALID, field
        valid()
    bad = []
    lm = p["pt_obs_lm"].copy(); lm[-1] = len(p["pt"])
    bad.append(dict(p, pt_obs_lm=lm))
    lm = p["ls_obs_lm"].copy(); lm[-1] = len(p["ls"])
    bad.append(dict(p, ls_obs_lm=lm))
    kf = p["pt_obs_kf"].copy(); kf[0] = len(p["kf_pose"])
    bad.append(dict(p, pt_obs_kf=kf))
    kf = p["ls_obs_kf"].copy(); kf[0] = -3                                # kf < -n_fixed
    bad.append(dict(p, ls_obs_kf=kf))
    bad += [orphan_map("pt")[0], orphan_map("ls")[0]]
    for q in bad:
        with pytest.raises(plf.PlfError):
            fe.local_ba(q)
        valid()


@pytest.mark.parametrize("kind", ["pt", "ls"])
def test_zero_information_landmark_is_refused_before_any_step(fe, kind):
    """a landmark seen once at its exact projection: both routines refuse it by name, the inputs are unchanged, and
    the context stays usable.  Without the refusal the landmark, then every keyframe it is seen from, turns NaN."""
    q, lm = zero_block_map(kind)
    for quirks in (1, 0):
        assert clib.local_ba(CAM, q, clib.lba_opts(ref_quirks=quirks))["rc"] == clib.LBA_ZERO_BLOCK
    keep = []
    args = _raw_args(q, keep)
    before = [a.copy() for a in keep]
    assert _raw_local(fe, args) == PLF_ERR_INVALID
    msg = fe.lib.plf_last_error(fe._ctx).decode()
    n_pt = len(q["pt"])
    name = f"point landmark {lm}" if kind == "pt" else f"line landmark {lm - n_pt}"
    assert name in msg and "zero diagonal" in msg, msg
    assert all(np.array_equal(a, b) for a, b in zip(keep, before))
    with pytest.raises(plf.PlfError, match="zero diagonal"):
        fe.global_ba(q)
    p = synth.local_map_problem(CAM, n_kf=3, n_fixed=2, seed=1)
    _check(p, fe.local_ba(p), clib.local_ba(CAM, p, clib.lba_opts()))
    _check(p, fe.global_ba(p), gba.global_ba(CAM, p, gba.opts()))
