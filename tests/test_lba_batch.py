"""CPU checks behind tests/test_lba_batch_gpu.py (plf_local_ba_batch): the batches the GPU file runs, each problem with
its camera, are decidable on oracle/lba.c (no stop decision within rounding of its threshold) and stop by the exits the
GPU file relies on; the binding refuses a malformed `seq` before any library call.  The helpers here build the batches."""
import functools

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib
from plslam_b200 import synth
from test_lba_edges import BRANCH_MAP, decidable
from test_lba_edges_gpu import PARITY

CAM = plf.KITTI_CAMERA
# three calibrations for sequences 0-2 of a four-sequence context (sequence 3 keeps the context's camera), perturbed from
# the KITTI camera as bench_sequence_cameras.py perturbs it
SEQ_CAMS = [dict(CAM, fx=CAM["fx"] * f, fy=CAM["fy"] * g, cx=CAM["cx"] + dx, cy=CAM["cy"] + dy, b=CAM["b"] * s)
            for f, g, dx, dy, s in ((0.97, 0.975, -6.5, 3.25, 0.96), (1.03, 1.025, 4.0, -2.5, 1.04),
                                    (0.985, 0.99, 9.0, 5.0, 1.02))]
MIXED_MAX_ITERS = 8   # under ref_quirks = 1 some maps stop by the change test before it, others reach it


def seq_camera(s):
    """the camera problem routed to sequence s (-1 or 3: the context's) projects with"""
    return SEQ_CAMS[s] if 0 <= s < len(SEQ_CAMS) else CAM


@functools.lru_cache(maxsize=None)
def mixed_batch():
    """24 problems with the context's camera: every PARITY shape of test_lba_edges_gpu.py (1 to 64 local keyframes, with
    and without fixed keyframes), a points-only, a lines-only and a structure-only map (n_kf = 0), the map whose error
    grows, and local maps of 5 to 10 keyframes at growing pixel noise."""
    probs = [synth.local_map_problem(CAM, n_kf=n_kf, n_fixed=n_fixed, pts_per_kf=ppk, ls_per_kf=lpk, t0=t0,
                                     seed=n_kf + 7 * n_fixed + t0) for n_kf, n_fixed, ppk, lpk, t0 in PARITY]
    probs += [synth.lba_problem(CAM, seed=3, n_ls=0), synth.lba_problem(CAM, seed=4, n_pt=0, n_ls=60),
              synth.lba_problem(CAM, seed=8, n_kf=0, n_fixed=5),
              synth.local_map_problem(CAM, **dict(BRANCH_MAP, px_noise=3.0))]
    probs += [synth.local_map_problem(CAM, n_kf=5 + i % 6, n_fixed=2 + i % 2, seed=100 + i, px_noise=0.3 + 0.5 * (i % 6))
              for i in range(9)]
    return tuple(probs)


@functools.lru_cache(maxsize=None)
def camera_batch():
    """(problems, seq): two problems per sequence 0-3 and two with seq = -1, each map generated with the camera of its
    sequence, in an interleaved order"""
    seq = [0, 1, 2, 3, -1, 2, 1, 0, -1, 3]
    probs = [synth.local_map_problem(seq_camera(s), n_kf=5 + i % 6, n_fixed=2, ls_per_kf=2 if i % 3 else 0, seed=200 + i)
             for i, s in enumerate(seq)]
    return tuple(probs), tuple(seq)


@functools.lru_cache(maxsize=None)
def oracle_run(kind, i, quirks, max_iters=15):
    """oracle/lba.c on problem i of mixed_batch() ('mixed') or camera_batch() ('camera'), with that problem's camera"""
    if kind == "mixed":
        p, cam = mixed_batch()[i], CAM
    else:
        probs, seq = camera_batch()
        p, cam = probs[i], seq_camera(seq[i])
    o = clib.lba_opts(ref_quirks=quirks, max_iters=max_iters)
    return clib.local_ba(cam, p, o), o


def exits(trace):
    """(the stop of the last pass, whether an iteration's error grew)"""
    return int(trace["stop"][-1]), bool(np.any((trace["applied"][1:] == 0) & (trace["step"][1:] >= 0)))


@pytest.mark.parametrize("quirks", [1, 0])
def test_mixed_batch_is_decidable_and_takes_several_exits(quirks):
    stops, grew = set(), False
    for i in range(len(mixed_batch())):
        ref, o = oracle_run("mixed", i, quirks, MIXED_MAX_ITERS)
        assert ref["rc"] == 0 and decidable(ref["trace"], o), (i, ref["trace"])
        s, g = exits(ref["trace"])
        stops.add(s)
        grew |= g
    assert clib.LBA_STOP_CHANGE in stops and grew
    if quirks:   # the evident intent's maps all grow once, then stop by the change test at iteration 2
        assert clib.LBA_STOP_MAXIT in stops


@pytest.mark.parametrize("quirks", [1, 0])
def test_camera_batch_is_decidable_with_each_camera(quirks):
    probs, seq = camera_batch()
    assert set(seq) == {-1, 0, 1, 2, 3}
    for i in range(len(probs)):
        ref, o = oracle_run("camera", i, quirks)
        assert ref["rc"] == 0 and decidable(ref["trace"], o), (i, ref["trace"])


def test_each_camera_changes_the_result():
    """the cameras differ enough that a problem projected with the wrong one gets another answer"""
    probs, seq = camera_batch()
    i = seq.index(0)
    right = clib.local_ba(SEQ_CAMS[0], probs[i], clib.lba_opts())
    wrong = clib.local_ba(CAM, probs[i], clib.lba_opts())
    assert np.abs(right["kf_pose"] - wrong["kf_pose"]).max() > 1e-4


@pytest.mark.parametrize("seq,msg", [([0, 1], "3 entries"), (np.zeros((3, 1), np.int32), "3 entries"),
                                     (np.zeros(3, np.float64), "integer"), ([0, 1, 2 ** 40], "int32")])
def test_binding_refuses_a_malformed_seq(seq, msg):
    with pytest.raises(plf.PlfError, match=msg):
        plf.Frontend._problem_sequences(3, seq)
    assert plf.Frontend._problem_sequences(3, None) is None
    assert plf.Frontend._problem_sequences(3, [-1, 0, 2]).dtype == np.int32
