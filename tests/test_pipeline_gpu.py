"""GPU parity tests for the batched front-end (stereo association, f2f tracking, pose) through the C ABI, against
the oracle pipeline (oracle/frontend.py: C restatements of ORB / LSD / LBD / GN + numpy matcher)."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe

pytestmark = pytest.mark.gpu
POSE_REL_TOL = 1e-4   # north_star: pose within 1e-4 relative on the se(3) log


def rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-9)


def check_frame(fg, fo: ofe.Frame):
    assert len(fg["pt_pl"]) == len(fo.pt_pl) and len(fg["ls_spl"]) == len(fo.ls_spl)
    assert np.array_equal(fg["pt_pl"], fo.pt_pl) and np.array_equal(fg["pt_disp"], fo.pt_disp)
    assert np.array_equal(fg["pt_P"], fo.pt_P) and np.array_equal(fg["pt_octave"], fo.pt_octave)
    assert np.array_equal(fg["pdesc"], fo.pdesc)
    for k, v in (("ls_spl", fo.ls_spl), ("ls_epl", fo.ls_epl), ("ls_sdisp", fo.ls_sdisp), ("ls_edisp", fo.ls_edisp),
                 ("ls_sP", fo.ls_sP), ("ls_eP", fo.ls_eP), ("ls_le", fo.ls_le), ("ls_angle", fo.ls_angle), ("ldesc", fo.ldesc)):
        assert np.array_equal(fg[k], v), k


def run_both(cam, frames, B, **prm_over):
    prm = dict(ofe.DEFAULTS, **prm_over)
    ref = ofe.run_sequence(cam, [(a, b) for a, b, _ in frames], prm)
    lim = plf.default_limits(); lim.max_batch = B
    kw = {k: prm[k] for k, _ in plf.plf_params._fields_}   # the oracle's parameters, every one of them, on the device too
    got, feats = [], []
    with plf.Frontend(camera=cam, limits=lim, **kw) as fe:
        for s0 in range(0, len(frames), B):
            chunk = frames[s0:s0 + B]
            res = fe.process_batch(np.stack([c[0] for c in chunk]), np.stack([c[1] for c in chunk]))
            got += res
            feats += [fe.get_frame(k) for k in range(len(chunk))]
    return ref, got, feats


def compare(ref, got, feats):
    for k, (r, g) in enumerate(zip(ref, got)):
        assert g["status"] == r["status"], k
        assert (g["n_stereo_pt"], g["n_stereo_ls"]) == (r["n_pt"], r["n_ls"]), k
        check_frame(feats[k], r["frame"])
        if r["status"] == 0:
            assert g["n_matched_pt"] == len(r["res"]["inlier_pt"]) and g["n_matched_ls"] == len(r["res"]["inlier_ls"])
            assert (g["n_inliers_pt"], g["n_inliers_ls"]) == r["res"]["n_inliers"]
            assert rel(clib.logmap_se3(g["DT"]), clib.logmap_se3(r["DT"])) < POSE_REL_TOL
        else:
            assert np.array_equal(g["DT"], np.eye(4))


def test_pipeline_kitti_shape_stream(built):
    """BASELINE config 2 shape: 1242x375, ~1500 ORB + 200 lines, tracking a planted trajectory; batches of 3."""
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, 6))
    ref, got, feats = run_both(cam, frames, 3, orb_nfeatures=1500, lsd_nfeatures=200)
    compare(ref, got, feats)
    # the planted motion is recovered (ATE-style check on the chained trajectory)
    T = np.eye(4)
    for g in got:
        T = T @ g["DT"]
    T_true = np.linalg.inv(frames[0][2]) @ frames[-1][2]
    assert np.linalg.norm(T[:3, 3] - T_true[:3, 3]) < 0.05 * np.linalg.norm(T_true[:3, 3])


def test_pipeline_euroc_shape_stream(built):
    """BASELINE config 3 shape: 752x480 full front-end + pose refine (max_iters 5 / 10); one frame per call."""
    cam = plf.EUROC_CAMERA
    world = synth.World(seed=8, length=40.0, n_quads=220, n_segs=120, half_width=5.0, half_height=3.0)
    frames = list(synth.stream(cam, 4, world=world, seed=43, step=0.08, yaw_deg=0.8))
    ref, got, feats = run_both(cam, frames, 1, orb_nfeatures=1200, lsd_nfeatures=300)
    compare(ref, got, feats)


@pytest.mark.parametrize("shape", ["kitti", "euroc", "lowtex"])
def test_pipeline_windowed_matching_strategy(built, shape):
    """plf_params.matching_strategy = 3 (the reference configs, config_euroc.yaml:55-57): stereo association through
    matchGrid() with the (matching_s_ws, 0) x (0, 0) window, frame-to-frame tracking through matchGrid() in a
    +-matching_f2f_ws window with the match() fall-back of src/mapHandler.cpp:274-278 - features, matches and poses
    equal to the oracle's (oracle/frontend.py track_matches / grid_match_*), all on the device."""
    if shape == "kitti":
        cam, frames, over, B = plf.KITTI_CAMERA, list(synth.stream(plf.KITTI_CAMERA, 5)), dict(orb_nfeatures=1500, lsd_nfeatures=200), 3
    elif shape == "euroc":
        cam = plf.EUROC_CAMERA
        world = synth.World(seed=8, length=40.0, n_quads=220, n_segs=120, half_width=5.0, half_height=3.0)
        frames, over, B = list(synth.stream(cam, 4, world=world, seed=43, step=0.08, yaw_deg=0.8)), dict(orb_nfeatures=1200, lsd_nfeatures=300), 2
    else:
        cam = plf.KITTI_CAMERA
        frames, over, B = list(synth.stream(cam, 3, world=synth.corridor_world(), seed=17, noise=2)), dict(orb_nfeatures=150, lsd_nfeatures=0), 3
    ref, got, feats = run_both(cam, frames, B, matching_strategy=3, **over)
    compare(ref, got, feats)
    ref0 = ofe.run_sequence(cam, [(a, b) for a, b, _ in frames[:2]], dict(ofe.DEFAULTS, **over))
    assert (ref[1]["n_pt"], ref[1]["n_ls"]) != (ref0[1]["n_pt"], ref0[1]["n_ls"])   # the strategy does change the association


def test_pipeline_windowed_matching_fallback(built):
    """A window of 0 cells with a large min_pt_matches forces the match() fall-back for points while lines keep the
    window result (min_ls_matches = 0)."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 4, world=world, seed=9, step=0.9))     # large motion: the 0-cell window loses most points
    ref, got, feats = run_both(cam, frames, 2, orb_nfeatures=800, lsd_nfeatures=150, matching_strategy=3, matching_f2f_ws=0,
                               min_pt_matches=500, min_ls_matches=0)
    compare(ref, got, feats)


corridor_world = synth.corridor_world   # lines-dominant scene (now part of the input generator: bench.py --config lowtex)


def test_pipeline_low_texture_stream(built):
    """BASELINE config 5 shape: lines-dominant frames (< 200 ORB keypoints kept, > 400 LSD lines with
    lsd_nfeatures = 0 = keep all) - stresses LBD and the line rows of the pose Jacobian."""
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, 3, world=corridor_world(), seed=17, noise=2))
    ref, got, feats = run_both(cam, frames, 3, orb_nfeatures=150, lsd_nfeatures=0)
    assert all(g["n_kp_l"] < 200 for g in got) and all(g["n_lines_l"] > 400 for g in got)
    assert got[1]["status"] == 0 and got[1]["n_inliers_ls"] > got[1]["n_inliers_pt"]
    compare(ref, got, feats)


def test_pipeline_reset_and_too_few_features(built):
    cam = dict(plf.KITTI_CAMERA, width=320, height=200, cx=160.0, cy=100.0)
    lim = plf.default_limits(); lim.max_batch = 2
    flat = np.full((2, 200, 320), 100, np.uint8)
    with plf.Frontend(camera=cam, limits=lim, orb_nlevels=2) as fe:
        r = fe.process_batch(flat, flat)
        assert r[0]["status"] == 2 and r[1]["status"] == 1          # first frame; then nothing to track
        assert np.array_equal(r[1]["DT"], np.eye(4)) and r[1]["n_stereo_pt"] == 0
        fe.reset_sequence()
        r = fe.process_batch(flat[:1], flat[:1])
        assert r[0]["status"] == 2


def test_batches_in_flight_match_sequential(built):
    """run, run, (run,) download, ... (software-pipelined use, up to three batches in flight) gives exactly the results
    of run/download pairs."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = [(L, R) for L, R, _ in synth.stream(cam, 12, world=world, seed=11, step=0.15)]
    Ls = np.stack([f[0] for f in frames]); Rs = np.stack([f[1] for f in frames])
    lim = plf.default_limits(); lim.max_batch = 2
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        seq = []
        for s0 in range(0, 12, 2):
            seq += fe.process_batch(Ls[s0:s0 + 2], Rs[s0:s0 + 2])
    for depth in (2, 3):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
            piped = []
            inflight = 0
            for s0 in range(0, 12, 2):
                fe.batch_upload(Ls[s0:s0 + 2], Rs[s0:s0 + 2]); fe.batch_run(2)
                inflight += 1
                if inflight == depth:
                    piped += list(fe.batch_download_array(2))
                    inflight -= 1
            while inflight:
                piped += list(fe.batch_download_array(2))
                inflight -= 1
            with pytest.raises(plf.PlfError, match="no batch in flight"):
                fe.batch_download(2)
            fe.batch_upload(Ls[0:2], Rs[0:2]); fe.batch_run(2); fe.batch_run(2); fe.batch_run(2)
            with pytest.raises(plf.PlfError, match="three batches already in flight"):
                fe.batch_run(2)
            fe.batch_download(2); fe.batch_download(2); fe.batch_download(2)
        assert len(piped) == len(seq) == 12
        for a, b in zip(seq, piped):
            assert a["status"] == b["status"] and a["n_stereo_pt"] == b["n_stereo_pt"] and a["n_inliers_pt"] == b["n_inliers_pt"]
            assert a["n_stereo_ls"] == b["n_stereo_ls"] and a["n_inliers_ls"] == b["n_inliers_ls"]
            assert np.array_equal(a["DT"], b["DT"])          # same kernels, same inputs: bit-identical poses


def test_standalone_operators_between_batches(built):
    """fe.orb / fe.lsd / fe.detect_lines / fe.lbd on an image of another size, called between batches on the same
    context, rebuild the ORB and LSD state and use their own tensor maps: the batches after them give exactly the results
    and frames of an uninterrupted run, and the operators return what they return on a fresh context."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 8, world=world, seed=21, step=0.12))
    Ls, Rs = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    other = next(iter(synth.stream(dict(cam, width=480, height=300, cx=240.0, cy=150.0), 1, world=world, seed=5)))[0]
    lim = plf.default_limits(); lim.max_batch = 2
    prm = dict(orb_nfeatures=700, lsd_nfeatures=150)

    def batch(fe, s0):
        res = fe.process_batch(Ls[s0:s0 + 2], Rs[s0:s0 + 2])
        return res, [fe.get_frame(k) for k in range(2)]

    def operators(fe):
        kps, desc = fe.orb(other)
        segs = fe.lsd(other)
        kls, ldesc = fe.detect_lines(other)
        return kps, desc, segs, kls, ldesc, fe.lbd(other, kls)

    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        base = [batch(fe, s0) for s0 in (0, 2, 4, 6)]
    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        got = [batch(fe, 0), batch(fe, 2)]
        ops = operators(fe)
        got += [batch(fe, 4), batch(fe, 6)]
    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        fresh = operators(fe)
    assert len(ops[0]) > 0 and len(ops[3]) > 0
    for a, b in zip(ops, fresh):
        assert np.array_equal(a, b)
    for (res_a, fr_a), (res_b, fr_b) in zip(base, got):
        for a, b in zip(res_a, res_b):
            for f in plf.RESULT_FIELDS:
                assert a[f] == b[f], f
            assert np.array_equal(a["DT"], b["DT"])
        for a, b in zip(fr_a, fr_b):
            for k in a:
                assert np.array_equal(a[k], b[k]), k


def test_trajectory_ate_vs_oracle_and_ground_truth(built):
    """north_star: trajectory ATE within 1 % of the reference (CPU oracle) on the same synthetic sequence."""
    cam = dict(plf.KITTI_CAMERA, width=800, height=300, cx=400.0, cy=150.0, fx=520.0, fy=520.0)
    world = synth.World(seed=5, length=70.0, n_quads=240, n_segs=120, half_width=10.0, half_height=3.5)
    frames = list(synth.stream(cam, 20, world=world, seed=21, step=0.3))
    prm = dict(orb_nfeatures=1000, lsd_nfeatures=150)
    ref = ofe.run_sequence(cam, [(a, b) for a, b, _ in frames], dict(ofe.DEFAULTS, **prm))
    lim = plf.default_limits(); lim.max_batch = 5
    got = []
    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        for s0 in range(0, 20, 5):
            got += fe.process_batch(np.stack([f[0] for f in frames[s0:s0 + 5]]), np.stack([f[1] for f in frames[s0:s0 + 5]]))

    def chain(dts):
        T, out = np.eye(4), []
        for d in dts:
            T = T @ d
            out.append(T[:3, 3].copy())
        return np.array(out)
    p_gpu, p_ref = chain([g["DT"] for g in got]), chain([r["DT"] for r in ref])
    T0inv = np.linalg.inv(frames[0][2])
    p_gt = np.array([(T0inv @ f[2])[:3, 3] for f in frames])
    ate = lambda p: float(np.sqrt(np.mean(np.sum((p - p_gt) ** 2, axis=1))))
    ate_gpu, ate_ref = ate(p_gpu), ate(p_ref)
    assert abs(ate_gpu - ate_ref) <= 0.01 * max(ate_ref, 1e-9)          # within 1 % of the reference's ATE
    assert np.max(np.linalg.norm(p_gpu - p_ref, axis=1)) < 1e-6          # in fact the trajectories coincide
    assert ate_gpu < 0.02 * np.linalg.norm(p_gt[-1])                     # and both follow the planted trajectory


def test_lsd_maps_per_batch_parity(built, monkeypatch):
    """PLF_LSD_PARITIES=2: the LSD hand-off maps exist per batch parity and the pre-grow chain runs on its own stream
    (pre-grow of batch i+1 under the growing of batch i).  Same results as the default single-copy pipeline, sequentially
    and with three batches in flight."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 8, world=world, seed=21, step=0.12))
    Ls, Rs = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])

    def run(in_flight):
        lim = plf.default_limits(); lim.max_batch = 2
        out = []
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
            pend = 0
            for s0 in range(0, 8, 2):
                fe.batch_upload(Ls[s0:s0 + 2], Rs[s0:s0 + 2]); fe.batch_run(2); pend += 1
                if pend == in_flight:
                    out += list(fe.batch_download_array(2)); pend -= 1
            while pend:
                out += list(fe.batch_download_array(2)); pend -= 1
        return out
    monkeypatch.delenv("PLF_LSD_PARITIES", raising=False)
    base = run(1)
    monkeypatch.setenv("PLF_LSD_PARITIES", "2")
    for depth in (1, 3):
        got = run(depth)
        for a, b in zip(base, got):
            for f in plf.RESULT_FIELDS:
                assert a[f] == b[f], f
            assert np.array_equal(a["DT"], b["DT"])
