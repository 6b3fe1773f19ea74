"""GPU tests of the batched pipeline's stereo association and frame-to-frame matching at their gate thresholds
(pipeline.cu k_stereo_points, k_stereo_lines, the mutual check, k_mg_geom_*, k_mg_select, k_f2f_build): every case of
tests/stereo_cases.py and every pinned setting, at matching_strategy 0 and 3, through plf_process_batch against the oracle
pipeline - every field of every frame (test_pipeline_gpu.compare).  tests/test_stereo_gates.py shows on the CPU that each
case and setting reaches what it is built for."""
import numpy as np
import pytest

import plslam_b200 as plf
import stereo_cases as sc
from oracle import frontend as ofe
from test_pipeline_gpu import compare, run_both

pytestmark = pytest.mark.gpu

_PINS = {}


def pins():
    if not _PINS:
        _PINS["gates"] = {st: sc.pins(st) for st in sc.PIN_LABELS}
        _PINS["fallback"] = sc.fallback_pins()[0]
    return _PINS


def run_case(name, strategy, frames=None, **over):
    c = sc.build(name)
    frames = c["frames"] if frames is None else frames
    ref, got, feats = run_both(c["cam"], frames, len(frames), limits=c["limits"], **dict(c["prm"], matching_strategy=strategy, **over))
    compare(ref, got, feats)
    return ref, got


@pytest.mark.parametrize("strategy", [0, 3])
@pytest.mark.parametrize("name", [n for n in sc.NAMES if n != "same"])
def test_case_matches_oracle(built, name, strategy):
    ref, got = run_case(name, strategy)
    assert got[0]["status"] == 2 and all(g["status"] == r["status"] for g, r in zip(got, ref))


@pytest.mark.parametrize("label,strategy", [(lb, st) for st, labels in sc.PIN_LABELS.items() for lb in labels])
def test_pinned_gate(built, label, strategy):
    """Both settings of a gate pinned at this matching strategy (stereo_cases.pins): the candidate's decision flips and
    the device follows it."""
    (_, name, param, acc, rej, _), = [p for p in pins()["gates"][strategy] if p[0] == label]
    for v in (acc, rej):
        run_case(name, strategy, **{param: v})


@pytest.mark.parametrize("label", ["pt_n", "pt_n+1", "pt_n_curr", "ls_n", "ls_n+1", "ls_n_curr"])
def test_pinned_fallback(built, label):
    (_, frames, over), = [p for p in pins()["fallback"] if p[0] == label]
    run_case("shear", 3, frames=frames, **over)


@pytest.mark.parametrize("strategy", [0, 3])
def test_zero_disparity_rows_at_infinity(built, strategy):
    """L == R with min_disp = 0: every stereo point has Z = inf.  The windowed path projects the previous frame to NaN,
    whose cell is 0 on both sides (plf_qcell / ofe._cell); the pose solver meets rows at infinity.  Every result field
    equals the oracle's, NaN for NaN."""
    c = sc.build("same")
    over = dict(min_disp=0.0, matching_strategy=strategy, matching_f2f_ws=10, min_pt_matches=0, min_ls_matches=0)
    prm = dict(ofe.DEFAULTS, **c["prm"], **over)
    ref = ofe.run_sequence(c["cam"], [(a, b) for a, b, _ in c["frames"]], prm)
    lim = plf.default_limits(); lim.max_batch = len(c["frames"])
    kw = {k: prm[k] for k, _ in plf.plf_params._fields_}
    with plf.Frontend(camera=c["cam"], limits=lim, **kw) as fe:
        got = fe.process_batch(np.stack([f[0] for f in c["frames"]]), np.stack([f[1] for f in c["frames"]]))
        feats = [fe.get_frame(k) for k in range(len(c["frames"]))]
    for k, (r, g) in enumerate(zip(ref, got)):
        for name, v in vars(r["frame"]).items():      # X or Y is NaN on the centre column or row: NaN for NaN
            assert np.array_equal(feats[k][name], v, equal_nan=v.dtype.kind == "f"), (k, name)
        assert g["status"] == r["status"] and (g["n_stereo_pt"], g["n_stereo_ls"]) == (r["n_pt"], r["n_ls"]), k
        assert r["n_pt"] > 500 and r["n_ls"] == 0
        if k == 0:
            continue
        res = r["res"]
        print(f"strategy {strategy} frame {k}: status {r['status']}, {len(res['inlier_pt'])} rows, inliers {res['n_inliers']}, "
              f"err {res['err']}, iters {res['iters']}; device err {g['err']}, iters {(g['iters1'], g['iters2'])}")
        assert g["n_matched_pt"] == len(res["inlier_pt"]) > 0 and g["n_matched_ls"] == 0
        assert (g["n_inliers_pt"], g["n_inliers_ls"]) == res["n_inliers"]
        assert (g["iters1"], g["iters2"]) == res["iters"]
        assert np.array_equal(g["DT"], r["DT"], equal_nan=True)
        assert np.array_equal(np.isnan(g["DT_cov"]), np.isnan(res["cov"])), k
        assert np.array_equal(g["DT_cov"][~np.isnan(g["DT_cov"])], res["cov"][~np.isnan(res["cov"])])
        assert (np.isnan(g["err"]) and np.isnan(res["err"])) or g["err"] == res["err"]
        # what DESIGN.md §8 states for rows at infinity, on the device itself: tracked, identity pose, every point row an
        # inlier, NaN error and covariance, one iteration per stage
        n = g["n_matched_pt"]
        assert g["status"] == 0 and np.array_equal(g["DT"], np.eye(4)), k
        assert (g["n_inliers_pt"], g["n_inliers_ls"]) == (n, 0), k
        assert np.isnan(g["err"]) and np.isnan(g["DT_cov"]).all() and (g["iters1"], g["iters2"]) == (1, 1), k


def test_mixed_cases_with_own_cameras(built):
    """Five cases as five sequences of one batched context, each with its own camera (plf_set_sequence_camera), their
    pairs interleaved in every batch: each sequence equals the oracle run with its camera, so no pair's gates or camera
    leak into a neighbouring block."""
    names = ["shift", "shear", "band", "mirror", "lattice"]
    cams = [dict(sc.CAM, fx=500.0 + 7 * s, fy=498.0 + 5 * s, cx=318.0 + s, cy=181.0 - s, b=0.5 + 0.02 * s)
            for s in range(len(names))]
    seqs = [sc.build(n)["frames"] for n in names]
    prm = dict(ofe.DEFAULTS, matching_strategy=3)
    refs = [ofe.run_sequence(cams[s], [(a, b) for a, b, _ in seqs[s]], prm) for s in range(len(names))]
    lim = plf.default_limits(); lim.max_batch = len(names)
    kw = {k: prm[k] for k, _ in plf.plf_params._fields_}
    got = {}
    with plf.Frontend(camera=sc.CAM, limits=lim, max_sequences=len(names), **kw) as fe:
        for s, cam in enumerate(cams):
            fe.set_sequence_camera(s, cam)
        for i in range(len(seqs[0])):
            order = [(s + i) % len(names) for s in range(len(names))]   # a different block per sequence in each batch
            res = fe.process_batch(np.stack([seqs[s][i][0] for s in order]), np.stack([seqs[s][i][1] for s in order]),
                                   seq=np.array(order, np.int32))
            for k, s in enumerate(order):
                got[(s, i)] = (res[k], fe.get_frame(k))
    for s in range(len(names)):
        g = [got[(s, i)][0] for i in range(len(seqs[s]))]
        f = [got[(s, i)][1] for i in range(len(seqs[s]))]
        compare(refs[s], g, f)
