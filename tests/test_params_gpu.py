"""GPU tests of the front-end away from its defaults, driven by tests/param_cases.py.

Standalone: ORB and LSD / detect_lines bit-equal to the C restatements (themselves pinned to cv2 4.13 by
tests/test_orb_oracle.py / tests/test_lsd_oracle.py) for every ORB / LSD case, on a KITTI-size and an odd-size image;
read-but-ignored parameters leave the output unchanged; unsupported values raise PlfError, every time they are used.
Pipeline: the reference configs and the one-at-a-time sweeps through compare() (features and matches bit-equal, pose
within 1e-4), each shown to change the run it is measured against; has_points / has_lines; plf_get_matches."""
import numpy as np
import pytest

import param_cases as pc
import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe
from test_pipeline_gpu import POSE_REL_TOL, compare, corridor_world, rel, run_both

pytestmark = pytest.mark.gpu

FIELDS = ["x", "y", "size", "angle", "response", "octave"]
IMAGES = {"kitti_1242x375": (1242, 375, 1), "odd_641x359": (641, 359, 7)}


def cam(w, h):
    return dict(plf.KITTI_CAMERA, width=w, height=h, cx=w / 2.0, cy=h / 2.0)


def image(name):
    w, h, seed = IMAGES[name]
    return w, h, synth.scene_pair(w=w, h=h, seed=seed)[0]


# ---- standalone detectors ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("img", sorted(IMAGES))
@pytest.mark.parametrize("case", sorted(pc.ORB_CASES))
def test_orb_param_cases(built, case, img):
    w, h, L = image(img)
    prm = dict(ofe.DEFAULTS, **pc.ORB_CASES[case])
    with plf.Frontend(camera=cam(w, h), **pc.ORB_CASES[case]) as fe:
        kp, desc = fe.orb(L)
    rk, rd = ofe._orb_c(L, prm)
    assert len(rk) > 100 and len(kp) == len(rk)
    for f in FIELDS:
        assert np.array_equal(kp[f], rk[f]), f
    assert np.array_equal(desc, rd)
    assert kp["octave"].max() == prm["orb_nlevels"] - 1 or len(kp) < prm["orb_nfeatures"]


@pytest.mark.parametrize("img", sorted(IMAGES))
@pytest.mark.parametrize("case", sorted(pc.LSD_CASES))
def test_lsd_param_cases(built, case, img):
    w, h, L = image(img)
    prm = dict(ofe.DEFAULTS, **pc.LSD_CASES[case])
    lim = plf.default_limits(); lim.max_segments = 32768
    with plf.Frontend(camera=cam(w, h), limits=lim, **pc.LSD_CASES[case]) as fe:
        segs = fe.lsd(L, cap=32768)
        kl, desc = fe.detect_lines(L) if img.startswith("odd") else (None, None)
    ref = clib.lsd(L, **ofe.lsd_kwargs(prm))
    assert len(ref) > 50 and segs.shape == ref.shape and np.array_equal(segs, ref)
    if kl is not None:   # KeyLine stage + top-K + LBD on the same segments
        okl, odesc = ofe.detect_lines(L, prm["lsd_nfeatures"], prm["min_line_length"], ofe.lsd_kwargs(prm))
        assert len(kl) == len(okl) and kl.tobytes() == okl.tobytes() and np.array_equal(desc, odesc)


def test_ignored_lsd_parameters_leave_segments_unchanged(built):
    w, h, L = image("odd_641x359")
    with plf.Frontend(camera=cam(w, h)) as fe:
        base = fe.lsd(L)
    assert np.array_equal(base, clib.lsd(L))
    for k in ("lsd_log_eps", "lsd_density_th"):
        with plf.Frontend(camera=cam(w, h), **{k: pc.INVARIANT[k]}) as fe:
            assert np.array_equal(fe.lsd(L), base), k


@pytest.mark.parametrize("field,value", [(f, v) for f, (_, bad) in pc.REJECTED.items() for v in bad] +
                         [(f, v) for f, bad in pc.OUT_OF_RANGE.items() for v in bad])
def test_unsupported_values_raise(built, field, value):
    """The error repeats on a second call (a failed set-up leaves no half-built state behind) and the pipeline reports
    it too."""
    w, h, L = image("odd_641x359")
    op = "orb" if field.startswith("orb") else "lsd"
    lim = plf.default_limits(); lim.max_batch = 1
    with plf.Frontend(camera=cam(w, h), limits=lim, **{field: value}) as fe:
        for _ in range(2):
            with pytest.raises(plf.PlfError, match="ORB" if op == "orb" else "LSD"):
                getattr(fe, op)(L)
        with pytest.raises(plf.PlfError):
            fe.process_batch(L, L)


def test_orb_level_smaller_than_edge_raises_and_recovers(built):
    """8 levels at 1.2 shrink a 200x120 image to 56x33 on the top level, below 2 edge + 8 = 46 rows: PlfError.  The same
    context then still runs a size it supports, bit-equal to the oracle."""
    big_w, big_h, big = image("odd_641x359")
    small = synth.scene_pair(w=200, h=120, seed=2)[0]
    with plf.Frontend(camera=cam(big_w, big_h), orb_nlevels=8) as fe:
        kp0, d0 = fe.orb(big)
        with pytest.raises(plf.PlfError, match="too small"):
            fe.orb(small)
        with pytest.raises(plf.PlfError, match="too small"):
            fe.orb(small)
        kp1, d1 = fe.orb(big)
    rk, rd = ofe._orb_c(big, dict(ofe.DEFAULTS, orb_nlevels=8))
    assert kp0.tobytes() == kp1.tobytes() and np.array_equal(d0, d1)
    assert np.array_equal(kp1["x"], rk["x"]) and np.array_equal(kp1["octave"], rk["octave"]) and np.array_equal(d1, rd)


def test_both_kinds_disabled_is_rejected_at_create(built):
    with pytest.raises(plf.PlfError, match="has_points and has_lines"):
        plf.Frontend(has_points=0, has_lines=0)


# ---- pipeline --------------------------------------------------------------------------------------------------------
SMALL_CAM = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)


def small_stream(n=5):
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    return list(synth.stream(SMALL_CAM, n, world=world, seed=11, step=0.15))


def gpu_only(cam_, frames, B, prm):
    lim = plf.default_limits(); lim.max_batch = B
    out = []
    with plf.Frontend(camera=cam_, limits=lim, **prm) as fe:
        for s0 in range(0, len(frames), B):
            chunk = frames[s0:s0 + B]
            out += fe.process_batch(np.stack([c[0] for c in chunk]), np.stack([c[1] for c in chunk]))
    return out


def stereo_counts(res):
    return [(g["n_stereo_pt"], g["n_stereo_ls"]) for g in res]


@pytest.mark.parametrize("name", sorted(pc.REFERENCE_CONFIGS))
def test_reference_config_stream(built, name):
    """Each reference config over 5 KITTI-shape frames in batches of 2 (a partial batch last); config_kitti.yaml selects
    FLD lines (use_fld_lines), which this library does not implement - that case runs with LSD."""
    cam_ = plf.KITTI_CAMERA
    frames = list(synth.stream(cam_, 5))
    ref, got, feats = run_both(cam_, frames, 2, **pc.REFERENCE_CONFIGS[name])
    compare(ref, got, feats)
    assert sum(r["status"] == 0 for r in ref) == 4
    assert stereo_counts(got) != stereo_counts(gpu_only(cam_, frames, 2, {}))   # the config changes the association


@pytest.mark.parametrize("name", sorted(pc.PIPELINE_SWEEPS))
def test_pipeline_sweep(built, name):
    case = pc.PIPELINE_SWEEPS[name]
    frames = small_stream()
    ref, got, feats = run_both(SMALL_CAM, frames, 2, **case["base"], **case["change"])
    compare(ref, got, feats)
    base = gpu_only(SMALL_CAM, frames, 2, case["base"])
    if case["moves"] == "stereo":
        assert stereo_counts(got) != stereo_counts(base)
    else:
        assert any((g["iters1"], g["iters2"]) != (b["iters1"], b["iters2"]) or
                   rel(clib.logmap_se3(g["DT"]), clib.logmap_se3(b["DT"])) > POSE_REL_TOL for g, b in zip(got[1:], base[1:]))


def test_ignored_parameters_leave_the_pipeline_unchanged(built):
    """f2f_overlap_th, inlier_k, lsd_log_eps and lsd_density_th together: every result field and pose bit-identical."""
    frames = small_stream(4)
    base, changed = gpu_only(SMALL_CAM, frames, 2, {}), gpu_only(SMALL_CAM, frames, 2, pc.INVARIANT)
    for a, b in zip(base, changed):
        assert all(a[f] == b[f] for f in plf.RESULT_FIELDS) and np.array_equal(a["DT"], b["DT"])


def lines_only_stream():
    return plf.KITTI_CAMERA, list(synth.stream(plf.KITTI_CAMERA, 4, world=corridor_world(), seed=17, noise=2))


@pytest.mark.parametrize("name", sorted(pc.SWITCH_CASES))
def test_single_feature_kind(built, name):
    """has_lines = 0 (points only) on the textured stream, has_points = 0 (lines only) on the lines-dominant corridor: the
    disabled kind is not detected, associated, matched or used in the pose; the enabled kind is what it is with both."""
    sw = pc.SWITCH_CASES[name]
    if name == "lines_only":
        cam_, frames = lines_only_stream()
        over = dict(orb_nfeatures=150, lsd_nfeatures=0)
    else:
        cam_, frames, over = SMALL_CAM, small_stream(4), dict(orb_nfeatures=700, lsd_nfeatures=150)
    ref, got, feats = run_both(cam_, frames, 2, **over, **sw)
    compare(ref, got, feats)
    both = gpu_only(cam_, frames, 2, over)
    off = "pt" if name == "lines_only" else "ls"
    on = "ls" if off == "pt" else "pt"
    for g, b in zip(got, both):
        if off == "pt":
            assert g["n_kp_l"] == g["n_kp_r"] == 0 and g["n_lines_l"] == b["n_lines_l"] > 0
        else:
            assert g["n_lines_l"] == g["n_lines_r"] == 0 and g["n_kp_l"] == b["n_kp_l"] > 0
        assert g[f"n_stereo_{off}"] == g[f"n_matched_{off}"] == g[f"n_inliers_{off}"] == 0
        assert g[f"n_stereo_{on}"] == b[f"n_stereo_{on}"] > 0
    assert sum(r["status"] == 0 for r in ref) == 3


@pytest.mark.parametrize("name", sorted(pc.SWITCH_CASES))
def test_single_feature_kind_too_few_features(built, name):
    """min_features between what the enabled kind alone and both kinds together match on frame 1: with one kind that
    frame has status 1 (identity pose), as in the oracle."""
    sw = pc.SWITCH_CASES[name]
    if name == "lines_only":
        cam_, frames = lines_only_stream()
        over = dict(orb_nfeatures=150, lsd_nfeatures=0)
    else:
        cam_, frames, over = SMALL_CAM, small_stream(4), dict(orb_nfeatures=700, lsd_nfeatures=150)
    full = ofe.run_sequence(cam_, [(a, b) for a, b, _ in frames], dict(ofe.DEFAULTS, **over))
    n_pt, n_ls = len(full[1]["res"]["inlier_pt"]), len(full[1]["res"]["inlier_ls"])
    alone = n_ls if name == "lines_only" else n_pt
    assert 0 < alone < n_pt + n_ls
    ref, got, feats = run_both(cam_, frames, 2, **over, **sw, min_features=alone + 1)
    compare(ref, got, feats)
    assert ref[1]["status"] == got[1]["status"] == 1 and np.array_equal(got[1]["DT"], np.eye(4))


@pytest.mark.parametrize("scene", ["default", "windowed", "lines_only"])
def test_get_matches_equal_oracle_rows(built, scene):
    """plf_get_matches: P / pl_obs and sP / eP / le_obs of every tracked frame equal the oracle's track() rows (previous
    frame's row order), and the inlier flags equal the oracle GN's."""
    B = 2
    if scene == "lines_only":
        cam_, frames = lines_only_stream()
        prm = dict(ofe.DEFAULTS, orb_nfeatures=150, lsd_nfeatures=0, has_points=0)
    else:
        cam_, frames = SMALL_CAM, small_stream(5)
        prm = dict(ofe.DEFAULTS, orb_nfeatures=700, lsd_nfeatures=150, matching_strategy=3 if scene == "windowed" else 0)
    ref = ofe.run_sequence(cam_, [(a, b) for a, b, _ in frames], prm)
    lim = plf.default_limits(); lim.max_batch = B
    got, rows = [], []
    with plf.Frontend(camera=cam_, limits=lim, **{k: prm[k] for k, _ in plf.plf_params._fields_}) as fe:
        for s0 in range(0, len(frames), B):
            chunk = frames[s0:s0 + B]
            got += fe.process_batch(np.stack([c[0] for c in chunk]), np.stack([c[1] for c in chunk]))
            rows += [fe.get_matches(k) for k in range(len(chunk))]
    assert len(rows[0]["P"]) == len(rows[0]["sP"]) == 0          # first frame: nothing tracked
    tracked = 0
    for i in range(1, len(frames)):
        tr = ofe.track(ref[i - 1]["frame"], ref[i]["frame"], prm, cam=cam_)
        m = rows[i]
        for k, o in (("P", "P"), ("pl_obs", "obs"), ("sP", "sP"), ("eP", "eP"), ("le_obs", "le")):
            assert np.array_equal(m[k], tr[o]), (i, k)
        assert got[i]["n_matched_pt"] == len(m["P"]) and got[i]["n_matched_ls"] == len(m["sP"])
        if ref[i]["status"] == 0:
            tracked += 1
            assert np.array_equal(m["inlier_pt"], ref[i]["res"]["inlier_pt"].astype(bool)), i
            assert np.array_equal(m["inlier_ls"], ref[i]["res"]["inlier_ls"].astype(bool)), i
            assert got[i]["n_inliers_pt"] == int(m["inlier_pt"].sum()) and got[i]["n_inliers_ls"] == int(m["inlier_ls"].sum())
    assert tracked == len(frames) - 1
    assert any(len(r["sP"]) > 0 for r in rows) and (scene == "lines_only" or any(len(r["P"]) > 0 for r in rows))
