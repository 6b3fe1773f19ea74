"""GPU parity of plf_match_kf2kf / plf_match_map2kf (keyframe and local-map matching on the device) against
oracle/kfmatching.py, on keyframes taken from the batched front-end on the synthetic KITTI-shape stream."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import frontend as ofe
from oracle import kfmatching as kfm
from oracle import synth

pytestmark = pytest.mark.gpu
PRM = dict(orb_nfeatures=1500, lsd_nfeatures=200)
N_FRAMES = 7


@pytest.fixture(scope="module")
def stream(built):
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, N_FRAMES))
    lim = plf.default_limits(); lim.max_batch = N_FRAMES
    with plf.Frontend(camera=cam, limits=lim, **PRM) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        feats = [fe.get_frame(k) for k in range(N_FRAMES)]
    assert all(len(f["pdesc"]) > 100 and len(f["ldesc"]) > 20 for f in feats)
    return cam, [f[2] for f in frames], feats


def DT_between(T_wc, a, b):
    """MapHandler::DT from keyframe a to keyframe b: points of a's camera frame in b's."""
    return np.linalg.inv(T_wc[b]) @ T_wc[a]


def prm_of(fe):
    return dict(ofe.DEFAULTS, **{k: getattr(fe.params, k) for k, _ in plf.plf_params._fields_})


def check_kf2kf(fe, cam, prev, curr, DT, fast):
    got = fe.match_kf2kf(prev, curr, DT, fast_matching=fast)
    m_pt, n_pt, m_ls, n_ls = kfm.match_kf2kf(cam, prm_of(fe), prev, curr, DT, fast_matching=fast)
    assert np.array_equal(got["m_pt"], m_pt) and got["n_pt"] == n_pt
    assert np.array_equal(got["m_ls"], m_ls) and got["n_ls"] == n_ls
    return got


@pytest.mark.parametrize("kmin", ["zero", "default", "high"])
@pytest.mark.parametrize("ws", [3, 10])
@pytest.mark.parametrize("fast", [0, 1])
@pytest.mark.parametrize("delta", [1, 5])
def test_kf2kf_vs_oracle(stream, delta, fast, ws, kmin):
    cam, T_wc, feats = stream
    prev, curr = feats[0], feats[delta]
    if kmin == "zero":
        over = dict(min_pt_matches=0, min_ls_matches=0)          # the windowed result always stands
    elif kmin == "high":                                       # windowed almost surely short of it: match() takes over
        over = dict(min_pt_matches=min(len(prev["pdesc"]), len(curr["pdesc"])) - 1,
                    min_ls_matches=min(len(prev["ldesc"]), len(curr["ldesc"])) - 1)
    else:
        over = {}
    with plf.Frontend(camera=cam, matching_f2f_ws=ws, **PRM, **over) as fe:
        got = check_kf2kf(fe, cam, prev, curr, DT_between(T_wc, 0, delta), fast)
    if fast or kmin == "high":
        assert got["n_pt"] > 0


def local_map(T_wc, feats, kfs, rng, n_dup=40, p_unused=0.1):
    """Landmarks from the features of keyframes `kfs` moved into world coordinates, plus duplicated descriptors (order
    decides their ties) and some unused entries."""
    pt_X, pt_d, ls_X, ls_d = [], [], [], []
    for k in kfs:
        f, T = feats[k], T_wc[k]
        w = lambda P: (T[:3, :3] @ P.T).T + T[:3, 3]
        pt_X.append(w(f["pt_P"])); pt_d.append(f["pdesc"])
        ls_X.append(np.concatenate([w(f["ls_sP"]), w(f["ls_eP"])], 1)); ls_d.append(f["ldesc"])
    pt_X, pt_d, ls_X, ls_d = np.concatenate(pt_X), np.concatenate(pt_d), np.concatenate(ls_X), np.concatenate(ls_d)
    i = rng.integers(0, len(pt_X), n_dup); j = rng.integers(0, len(ls_X), n_dup // 4)
    pt_X = np.concatenate([pt_X, pt_X[i] + 0.01]); pt_d = np.concatenate([pt_d, pt_d[i]])
    ls_X = np.concatenate([ls_X, ls_X[j] + 0.01]); ls_d = np.concatenate([ls_d, ls_d[j]])
    return dict(pt_X=pt_X, pt_desc=pt_d, pt_use=(rng.random(len(pt_X)) > p_unused).astype(np.uint8),
                ls_X=ls_X, ls_desc=ls_d, ls_use=(rng.random(len(ls_X)) > p_unused).astype(np.uint8))


def check_map2kf(fe, cam, lmap, Twf, kf, pt_lm, ls_lm, fast, epip=(1.0, 1.0)):
    got = fe.match_map2kf(lmap, Twf, kf, pt_lm, ls_lm, fast_matching=fast, max_kf_epip_p=epip[0], max_kf_epip_l=epip[1])
    lm_pt, n_pt, lm_ls, n_ls = kfm.match_map2kf(cam, prm_of(fe), lmap, Twf, kf, pt_lm, ls_lm, fast_matching=fast,
                                                max_kf_epip_p=epip[0], max_kf_epip_l=epip[1])
    assert np.array_equal(got["lm_pt"], lm_pt) and got["n_pt"] == n_pt
    assert np.array_equal(got["lm_ls"], lm_ls) and got["n_ls"] == n_ls
    return got


@pytest.mark.parametrize("epip", [(1.0, 1.0), (3.0, 0.02)])
@pytest.mark.parametrize("ws", [3, 10])
@pytest.mark.parametrize("fast", [0, 1])
def test_map2kf_vs_oracle(stream, fast, ws, epip):
    cam, T_wc, feats = stream
    rng = np.random.default_rng(ws + 10 * fast)
    lmap = local_map(T_wc, feats, [0, 1, 2, 3], rng)
    kf = feats[5]
    pt_lm = np.where(rng.random(len(kf["pdesc"])) < 0.2, 3, -1).astype(np.int32)   # some features matched already
    ls_lm = np.where(rng.random(len(kf["ldesc"])) < 0.2, 1, -1).astype(np.int32)
    with plf.Frontend(camera=cam, matching_f2f_ws=ws, **PRM) as fe:
        got = check_map2kf(fe, cam, lmap, np.linalg.inv(T_wc[5]), kf, pt_lm, ls_lm, fast, epip)
        assert got["n_pt"] > 0
    # a window of 0 cells with high min_*_matches: the fallback decision taken on other counts
    with plf.Frontend(camera=cam, matching_f2f_ws=0, min_pt_matches=2000, min_ls_matches=300, **PRM) as fe:
        check_map2kf(fe, cam, lmap, np.linalg.inv(T_wc[5]), kf, pt_lm, ls_lm, fast, epip)


def test_edge_cases(stream):
    cam, T_wc, feats = stream
    rng = np.random.default_rng(3)
    lmap = local_map(T_wc, feats, [0, 1], rng)
    kf, Twf = feats[3], np.linalg.inv(T_wc[3])
    empty = dict(pt_X=np.zeros((0, 3)), pt_desc=np.zeros((0, 32), np.uint8), ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32), np.uint8))
    with plf.Frontend(camera=cam, **PRM) as fe:
        r = check_map2kf(fe, cam, empty, Twf, kf, None, None, 1)
        assert r["n_pt"] == r["n_ls"] == 0
        r = check_map2kf(fe, cam, lmap, np.diag([1.0, 1.0, -1.0, 1.0]) @ Twf, kf, None, None, 1)   # nothing visible
        assert r["n_pt"] == r["n_ls"] == 0 and (r["lm_pt"] == -1).all()
        r = check_map2kf(fe, cam, lmap, Twf, kf, np.zeros(len(kf["pdesc"]), np.int32), np.zeros(len(kf["ldesc"]), np.int32), 1)
        assert r["n_pt"] == r["n_ls"] == 0
        no_lines = dict(kf, ls_spl=np.zeros((0, 2)), ls_epl=np.zeros((0, 2)), ls_le=np.zeros((0, 3)), ldesc=np.zeros((0, 32), np.uint8))
        r = check_map2kf(fe, cam, lmap, Twf, no_lines, None, None, 1)
        assert r["n_ls"] == 0 and r["n_pt"] > 0
    for sw in ("has_points", "has_lines"):
        with plf.Frontend(camera=cam, **PRM, **{sw: 0}) as fe:
            r = check_kf2kf(fe, cam, feats[0], feats[1], DT_between(T_wc, 0, 1), 1)
            assert (r["n_pt"] == 0) == (sw == "has_points") and (r["n_ls"] == 0) == (sw == "has_lines")
            r = check_map2kf(fe, cam, lmap, Twf, kf, None, None, 1)
            assert (r["n_pt"] == 0) == (sw == "has_points")


def test_size_limits(stream):
    """65535 landmarks and 8192 keyframe features per kind are accepted, one more is PLF_ERR_INVALID, and the context
    keeps working."""
    cam, T_wc, feats = stream
    rng = np.random.default_rng(4)
    kf, Twf = feats[3], np.linalg.inv(T_wc[3])
    small = local_map(T_wc, feats, [1, 2], rng)
    n = 65535
    idx = rng.integers(0, len(small["pt_X"]), n)
    big = dict(small, pt_X=small["pt_X"][idx], pt_desc=small["pt_desc"][idx],
               pt_use=(rng.random(n) < 0.01).astype(np.uint8))                 # ~650 used: the oracle stays cheap
    with plf.Frontend(camera=cam, **PRM) as fe:
        r = check_map2kf(fe, cam, big, Twf, kf, None, None, 1)
        assert len(r["lm_pt"]) == n and r["n_pt"] > 0
        over = dict(big, pt_X=np.concatenate([big["pt_X"], big["pt_X"][:1]]), pt_desc=np.concatenate([big["pt_desc"], big["pt_desc"][:1]]),
                    pt_use=np.concatenate([big["pt_use"], [1]]).astype(np.uint8))
        with pytest.raises(plf.PlfError, match="65535"):
            fe.match_map2kf(over, Twf, kf)
        check_map2kf(fe, cam, small, Twf, kf, None, None, 1)
        m = 8192
        j = rng.integers(0, len(kf["pdesc"]), m)
        big_kf = dict(kf, pt_pl=kf["pt_pl"][j], pdesc=kf["pdesc"][j], pt_P=kf["pt_P"][j])
        lm = np.where(rng.random(m) < 0.9, 0, -1).astype(np.int32)
        check_map2kf(fe, cam, small, Twf, big_kf, lm, None, 1)
        check_kf2kf(fe, cam, big_kf, feats[4], DT_between(T_wc, 3, 4), 1)
        big_kf1 = dict(big_kf, pt_pl=np.concatenate([big_kf["pt_pl"], kf["pt_pl"][:1]]), pdesc=np.concatenate([big_kf["pdesc"], kf["pdesc"][:1]]),
                       pt_P=np.concatenate([big_kf["pt_P"], kf["pt_P"][:1]]))
        with pytest.raises(plf.PlfError, match="8192"):
            fe.match_map2kf(small, Twf, big_kf1)
        with pytest.raises(plf.PlfError, match="8192"):
            fe.match_kf2kf(big_kf1, feats[4], np.eye(4))
        # a NULL array with a count > 0
        v = plf.plf_frame_view(); v.n_pt = 5
        m_pt = np.zeros(5, np.int32); o = plf.plf_kf_match_opts(1, 1.0, 1.0)
        st = fe.lib.plf_match_kf2kf(fe._ctx, C.byref(o), C.byref(v), C.byref(v), np.eye(4).ctypes.data_as(C.c_void_p),
                                    m_pt.ctypes.data_as(C.c_void_p), None, None, None)
        assert st == -1 and b"NULL" in fe.lib.plf_last_error(fe._ctx)
        check_kf2kf(fe, cam, feats[0], feats[1], DT_between(T_wc, 0, 1), 1)


def test_kf2kf_points_at_identity_are_the_pipeline_tracking(built):
    """On a matching_strategy != 0 context, plf_match_kf2kf points with DT = I between frames k and k+1 give the rows
    get_matches(k+1) reports."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 4, world=world, seed=11, step=0.15))
    lim = plf.default_limits(); lim.max_batch = 4
    with plf.Frontend(camera=cam, limits=lim, matching_strategy=3, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        fr = [fe.get_frame(k) for k in range(4)]
        for k in range(3):
            mt = fe.get_matches(k + 1)
            r = fe.match_kf2kf(fr[k], fr[k + 1], np.eye(4), fast_matching=True)
            rows = np.nonzero(r["m_pt"] >= 0)[0]
            assert len(rows) > 20
            assert np.array_equal(mt["P"], fr[k]["pt_P"][rows]) and np.array_equal(mt["pl_obs"], fr[k + 1]["pt_pl"][r["m_pt"][rows]])


def test_operators_while_batches_in_flight(stream):
    """Both operators called with two batches in flight (run, run, operators, download, download, ...): the pipeline's
    results and get_frame rows equal an uninterrupted run, and the operators return what they return on a fresh context."""
    cam_k, T_wc, feats = stream
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 8, world=world, seed=21, step=0.12))
    Ls, Rs = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    lim = plf.default_limits(); lim.max_batch = 2
    lmap = local_map(T_wc, feats, [0, 1, 2], np.random.default_rng(5))
    # the operators match the KITTI-shape keyframes with this context's camera: what matters here is that they are the
    # same with and without batches in flight
    ops_in = (feats[0], feats[2], DT_between(T_wc, 0, 2), lmap, np.linalg.inv(T_wc[4]), feats[4])

    def operators(fe):
        a = fe.match_kf2kf(*ops_in[:3])
        b = fe.match_map2kf(*ops_in[3:])
        return a, b

    def run(fe, with_ops):
        res, rows, ops = [], [], None
        for s0 in (0, 4):
            fe.batch_upload(Ls[s0:s0 + 2], Rs[s0:s0 + 2]); fe.batch_run(2)
            fe.batch_upload(Ls[s0 + 2:s0 + 4], Rs[s0 + 2:s0 + 4]); fe.batch_run(2)
            if with_ops:
                ops = operators(fe)
            res += list(fe.batch_download_array(2)) + list(fe.batch_download_array(2))
            rows += [fe.get_frame(k) for k in range(2)]
        return res, rows, ops

    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        base, base_rows, _ = run(fe, False)
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        got, got_rows, ops = run(fe, True)
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        fresh = operators(fe)
    for a, b in zip(base, got):
        for f in plf.RESULT_FIELDS:
            assert a[f] == b[f], f
        assert np.array_equal(a["DT"], b["DT"])
    for a, b in zip(base_rows, got_rows):
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    for x, y in zip(ops, fresh):
        for k in x:
            assert np.array_equal(x[k], y[k]), k


def test_pixel_unit_lines_entering_the_grid(built):
    """KF-to-KF query lines stay in pixels, so a projected line can start hundreds of cells outside the grid: the mask
    walk then starts at the first step whose window reaches the grid (closed-form state of the walk) and stops after the
    last.  Hand-built lines: one from far left, one steep from far above, one leaving to the right, one never near the
    grid; each previous line shares its descriptor with the current line drawn (in grid units) where it crosses the grid."""
    cam = dict(width=640, height=480, fx=512.0, fy=512.0, cx=320.0, cy=240.0, b=0.5)
    back = lambda u, v, Z=2.0: np.array([(u - cam["cx"]) * Z / cam["fx"], (v - cam["cy"]) * Z / cam["fy"], Z])
    d = np.random.default_rng(12).integers(0, 256, (4, 32), dtype=np.uint8)
    prev_px = np.array([(-500, 20, 40, 30), (20, -400, 30, 40), (60, 40, 1000, 10), (-900, -900, -500, -880)], np.float64)
    curr_px = np.array([(0, 290, 400, 300), (290, 0, 300, 400), (600, 400, 630, 399), (500, 100, 600, 110)], np.float64)
    prev = dict(pdesc=np.zeros((0, 32), np.uint8), ls_sP=np.array([back(*p[:2]) for p in prev_px]),
                ls_eP=np.array([back(*p[2:]) for p in prev_px]), ldesc=d)
    curr = dict(pdesc=np.zeros((0, 32), np.uint8), ls_spl=curr_px[:, :2], ls_epl=curr_px[:, 2:], ldesc=d)
    for ws in (0, 3):
        with plf.Frontend(camera=cam, matching_f2f_ws=ws, min_ls_matches=0) as fe:
            got = check_kf2kf(fe, cam, prev, curr, np.eye(4), 1)
        assert list(got["m_ls"]) == [0, 1, 2, -1] and got["n_ls"] == 3


def test_line_size_limits(stream):
    """Lines at the limits: 65535 landmark lines (the largest query mask) and 8192 keyframe lines, against the oracle;
    one more is PLF_ERR_INVALID."""
    cam, T_wc, feats = stream
    rng = np.random.default_rng(8)
    kf, Twf = feats[3], np.linalg.inv(T_wc[3])
    small = local_map(T_wc, feats, [1, 2], rng)
    n = 65535
    idx = rng.integers(0, len(small["ls_X"]), n)
    big = dict(small, ls_X=small["ls_X"][idx], ls_desc=small["ls_desc"][idx], ls_use=(rng.random(n) < 0.01).astype(np.uint8))
    m = 8192
    j = rng.integers(0, len(kf["ldesc"]), m)
    big_kf = dict(kf, ls_spl=kf["ls_spl"][j], ls_epl=kf["ls_epl"][j], ls_le=kf["ls_le"][j], ls_sP=kf["ls_sP"][j],
                  ls_eP=kf["ls_eP"][j], ldesc=kf["ldesc"][j])
    with plf.Frontend(camera=cam, **PRM) as fe:
        for fast in (0, 1):
            r = check_map2kf(fe, cam, big, Twf, kf, None, None, fast)
            assert len(r["lm_ls"]) == n
            check_map2kf(fe, cam, small, Twf, big_kf, None, np.where(rng.random(m) < 0.9, 0, -1).astype(np.int32), fast)
            check_kf2kf(fe, cam, big_kf, feats[4], DT_between(T_wc, 3, 4), fast)
        over = dict(big, ls_X=np.concatenate([big["ls_X"], big["ls_X"][:1]]), ls_desc=np.concatenate([big["ls_desc"], big["ls_desc"][:1]]),
                    ls_use=np.concatenate([big["ls_use"], [1]]).astype(np.uint8))
        with pytest.raises(plf.PlfError, match="65535"):
            fe.match_map2kf(over, Twf, kf)
        big_kf1 = {k: (np.concatenate([v, v[:1]]) if k.startswith("ls_") or k == "ldesc" else v) for k, v in big_kf.items()}
        with pytest.raises(plf.PlfError, match="8192"):
            fe.match_kf2kf(big_kf1, feats[4], np.eye(4))
        check_map2kf(fe, cam, small, Twf, kf, None, None, 1)


def test_vo_demo_kf_match_selftest(built, tmp_path):
    """`vo_demo --kf-match-selftest`: both calls written against the shim (row-major copies of DT and Twf, the local map
    built from the previous keyframe after the KF-to-KF step) give what the Python binding gives on the same frames."""
    import struct
    import subprocess
    from pathlib import Path
    demo = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "lib" / "vo_demo"
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = [(L, R) for L, R, _ in synth.stream(cam, 5, world=world, seed=11, step=0.15)]
    p = tmp_path / "frames.bin"
    with open(p, "wb") as f:
        f.write(struct.pack("<3i", len(frames), cam["width"], cam["height"]))
        f.write(struct.pack("<5d", cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["b"]))
        for L, R in frames:
            f.write(np.ascontiguousarray(L, np.uint8).tobytes() + np.ascontiguousarray(R, np.uint8).tobytes())
    r = subprocess.run([str(demo), str(p), "700", "150", "--kf-match-selftest"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rows = [ln.split() for ln in r.stdout.strip().splitlines()]
    kfm_rows = {ln[1]: ln[2:] for ln in rows if ln[0] == "kfm"}
    frame_rows = [ln for ln in rows if ln[0] != "kfm"]
    assert len(frame_rows) == 5
    ints = lambda k: np.array([int(v) for v in kfm_rows[k]], np.int32)
    Tfw0 = np.array([float(v) for v in frame_rows[0][6:22]]).reshape(4, 4)
    DT = np.array([float(v) for v in kfm_rows["DT"]]).reshape(4, 4)
    Twf = np.array([float(v) for v in kfm_rows["Twf"]]).reshape(4, 4)
    Tfw4 = np.array([float(v) for v in frame_rows[4][6:22]]).reshape(4, 4)
    assert np.allclose(Twf @ Tfw4, np.eye(4), atol=1e-12) and np.allclose(DT, Twf @ Tfw0, atol=1e-12)
    lim = plf.default_limits(); lim.max_batch = 1
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        feats = []
        for L, R in frames:
            fe.process_batch(L, R)
            feats.append(fe.get_frame(0))
        f0, f4 = feats[0], feats[4]
        a = fe.match_kf2kf(f0, f4, DT, fast_matching=True)
        assert np.array_equal(a["m_pt"], ints("m_pt")) and np.array_equal(a["m_ls"], ints("m_ls"))
        assert [a["n_pt"], a["n_ls"]] == [int(v) for v in kfm_rows["kf2kf"]] and a["n_pt"] > 0
        pt_lm = np.full(len(f4["pdesc"]), -1, np.int32); ls_lm = np.full(len(f4["ldesc"]), -1, np.int32)
        pt_lm[a["m_pt"][a["m_pt"] >= 0]] = np.nonzero(a["m_pt"] >= 0)[0]
        ls_lm[a["m_ls"][a["m_ls"] >= 0]] = np.nonzero(a["m_ls"] >= 0)[0]
        lmap = dict(pt_X=kfm.rigid(Tfw0, f0["pt_P"]), pt_desc=f0["pdesc"], pt_use=(a["m_pt"] < 0).astype(np.uint8),
                    ls_X=np.concatenate([kfm.rigid(Tfw0, f0["ls_sP"]), kfm.rigid(Tfw0, f0["ls_eP"])], 1), ls_desc=f0["ldesc"],
                    ls_use=(a["m_ls"] < 0).astype(np.uint8))
        b = fe.match_map2kf(lmap, Twf, f4, pt_lm, ls_lm, fast_matching=True)
        assert np.array_equal(b["lm_pt"], ints("lm_pt")) and np.array_equal(b["lm_ls"], ints("lm_ls"))
        assert [b["n_pt"], b["n_ls"]] == [int(v) for v in kfm_rows["map2kf"]]
        assert check_map2kf(fe, cam, lmap, Twf, f4, pt_lm, ls_lm, 1)["n_pt"] == b["n_pt"]
