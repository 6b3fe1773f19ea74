"""CPU checks behind tests/test_gba_batch_gpu.py (plf_global_ba_batch): the batches the GPU file runs, each problem with
its camera, are decidable on oracle/gba.py (no stop decision and no iteration count within rounding of its threshold),
and with the evident intent they stop by more than one exit; each camera of the camera batch changes the oracle's
answer.  The helpers here build the batches and trace the oracle's decisions."""
import contextlib
import functools

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import gba
from plslam_b200 import synth
from test_lba_batch import SEQ_CAMS
from test_lba_edges import decidable

CAM = plf.KITTI_CAMERA
# sequences 0-3 of a four-sequence context, each with its own calibration
GBA_CAMS = SEQ_CAMS + [dict(CAM, fx=CAM["fx"] * 1.015, fy=CAM["fy"] * 1.01, cx=CAM["cx"] - 8.0, cy=CAM["cy"] + 4.5)]
# (n_kf, pts_per_kf, ls_per_kf, n_fixed): one CTA up to 64 keyframes, the tiled LDL^T from 65, tile counts 7, 19 and 57
MIXED = [(1, 30, 8, 1), (8, 20, 6, 3), (64, 12, 4, 1), (65, 12, 0, 1), (65, 0, 5, 2), (200, 8, 3, 4), (600, 6, 2, 1)]
CAMERA_SEQ = (0, 1, 2, 3, -1, 2, 0)
# the evident intent's runs: finite errors, so LBA's thresholds, and a max_iters that some maps reach and others do not
INTENT = dict(min_error=1e-7, min_error_change=1e-7, max_iters=5)


def seq_camera(s):
    return GBA_CAMS[s] if s >= 0 else CAM


def opts_kw(quirks):
    """global_ba's options at a quirk setting: the DBL_EPSILON literals as written, 1e-7 with the intent"""
    return dict(ref_quirks=quirks) if quirks else dict(ref_quirks=0, **INTENT)


@functools.lru_cache(maxsize=None)
def mixed_batch():
    """the maps of tests/test_gba_gpu.py's parity cases, every size from 1 to 600 keyframes"""
    return tuple(synth.gba_problem(CAM, n_kf=n, pts_per_kf=ppk, ls_per_kf=lpk, n_fixed=nf, seed=n + 17 * nf)
                 for n, ppk, lpk, nf in MIXED)


@functools.lru_cache(maxsize=None)
def camera_batch():
    """(problems, seq): maps generated with the camera of their sequence, one of them tiled (70 keyframes)"""
    probs = tuple(synth.gba_problem(seq_camera(s), n_kf=(6, 12, 70, 9, 5, 20, 3)[i], pts_per_kf=10, ls_per_kf=3,
                                    n_fixed=1 + i % 2, seed=400 + i) for i, s in enumerate(CAMERA_SEQ))
    return probs, CAMERA_SEQ


@contextlib.contextmanager
def _recording():
    """records, while active, the error sum of every pass and |DX| of every solve of oracle/gba.global_ba"""
    ne, sl = gba.normal_equations, gba.solve_lower
    rec = dict(sums=[], steps=[], solves=[])

    def normal_equations(*a, **k):
        H, g, s = ne(*a, **k)
        rec["sums"].append(s)
        rec["solves"].append(len(rec["steps"]))
        return H, g, s

    def solve_lower(*a, **k):
        dx = sl(*a, **k)
        rec["steps"].append(float(np.sqrt(dx @ dx)))
        return dx

    gba.normal_equations, gba.solve_lower = normal_equations, solve_lower
    try:
        yield rec
    finally:
        gba.normal_equations, gba.solve_lower = ne, sl


def traced(cam, p, quirks, **kw):
    """(oracle result, trace, opts): trace["err"][i] is pass i's normalised error, trace["step"][i] its |DX| (-1 when the
    pass stopped before solving), in the layout test_lba_edges.decidable reads"""
    o = gba.opts(**dict(opts_kw(quirks), **kw))
    with _recording() as rec:
        ref = gba.global_ba(cam, p, o)
    nobs = len(p["pt_obs_lm"]) + len(p["ls_obs_lm"])
    with np.errstate(divide="ignore", invalid="ignore"):
        err = np.array([np.float64(s) / np.float64(0 if quirks else nobs) for s in rec["sums"]])
    n = len(err)
    step = np.full(n, -1.0)
    for i in range(n):
        nxt = rec["solves"][i + 1] if i + 1 < n else len(rec["steps"])
        if nxt > rec["solves"][i]:
            step[i] = rec["steps"][rec["solves"][i]]
    return ref, dict(err=err, step=step), o


def gba_decidable(trace, o):
    """decidable() of the local BA; as written the errors are +inf, so only the |DX| test decides"""
    if np.all(np.isfinite(trace["err"])):
        return decidable(trace, o)
    s, mec = trace["step"][1:], o["min_error_change"]
    return not np.isfinite(trace["err"]).any() and bool(np.all(np.abs(s - mec) > 1e-6 * mec))


def exit_of(trace, o):
    """how the oracle's run ended: 'error' (the change or min-error test), 'step' (|DX|) or 'max_iters'"""
    if trace["step"][-1] < 0:
        return "error"
    if len(trace["step"]) > 1 and trace["step"][-1] < o["min_error_change"]:
        return "step"
    return "max_iters"


@functools.lru_cache(maxsize=None)
def oracle_run(kind, i, quirks):
    """(result, trace, opts) of problem i of mixed_batch() ('mixed') or camera_batch() ('camera'), with its camera"""
    if kind == "mixed":
        return traced(CAM, mixed_batch()[i], quirks)
    probs, seq = camera_batch()
    return traced(seq_camera(seq[i]), probs[i], quirks)


@pytest.mark.parametrize("quirks", [1, 0])
def test_mixed_batch_is_decidable(quirks):
    exits = set()
    for i in range(len(MIXED)):
        ref, tr, o = oracle_run("mixed", i, quirks)
        assert ref["rc"] == 0 and gba_decidable(tr, o), (i, tr)
        exits.add(exit_of(tr, o))
    if quirks:   # (g3): only max_iters or |DX| ends a run
        assert exits <= {"max_iters", "step"}
    else:
        assert len(exits) > 1, exits


@pytest.mark.parametrize("quirks", [1, 0])
def test_camera_batch_is_decidable(quirks):
    probs, seq = camera_batch()
    assert set(seq) == {-1, 0, 1, 2, 3} and max(len(p["kf_pose"]) for p in probs) > 64
    exits = set()
    for i in range(len(probs)):
        ref, tr, o = oracle_run("camera", i, quirks)
        assert ref["rc"] == 0 and gba_decidable(tr, o), (i, tr)
        exits.add(exit_of(tr, o))
    if not quirks:
        assert len(exits) > 1, exits


def test_each_camera_changes_the_result():
    """a problem projected with another sequence's camera, or the context's, gets another answer"""
    probs, seq = camera_batch()
    for i, s in enumerate(seq):
        if s < 0:
            continue
        right = oracle_run("camera", i, 1)[0]
        for other in [c for c in GBA_CAMS + [CAM] if c is not GBA_CAMS[s]]:
            wrong = gba.global_ba(other, probs[i], gba.opts())
            assert np.abs(right["kf_pose"] - wrong["kf_pose"]).max() > 1e-4, (i, s)
