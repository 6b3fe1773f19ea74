"""GPU tests of plf_match_kf2kf_batch / plf_match_map2kf_batch: many keyframe matchings in one device call, each with its
sequence's camera.

Keyframes come from four sequences rendered with distinct calibrations (one image size, distinct fx, fy, cx, cy and b,
as test_sequence_cameras_gpu.py renders them), each taken from a context created with that sequence's camera.  Every
problem of a batch is held, exactly, to oracle/kfmatching.py with its sequence's camera and to the single call on a
context created with that camera."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import kfmatching as kfm
from oracle import synth
from test_kfmatching_gpu import DT_between, local_map, prm_of
from test_sequence_cameras_gpu import CAM, CAMS

pytestmark = pytest.mark.gpu
PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
N_FRAMES = 7
PLF_ERR_INVALID, PLF_ERR_CAPACITY = -1, -4


@pytest.fixture(scope="module")
def seqs(built):
    """Per sequence s: (T_wc of its frames, get_frame dicts) from a context created with CAMS[s]."""
    out = []
    lim = plf.default_limits(); lim.max_batch = N_FRAMES
    for s, cam in enumerate(CAMS):
        world = synth.World(seed=40 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
        frames = list(synth.stream(cam, N_FRAMES, world=world, seed=50 + s, step=0.15))
        with plf.Frontend(camera=cam, limits=lim, **PRM) as fe:
            fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
            feats = [fe.get_frame(k) for k in range(N_FRAMES)]
        counts = [(len(f["pdesc"]), len(f["ldesc"])) for f in feats]
        assert all(n_pt > 100 and n_ls > 12 for n_pt, n_ls in counts), (s, counts)
        out.append(([f[2] for f in frames], feats))
    return out


def cam_of(s):
    return CAMS[s] if s >= 0 else CAM


def thin(f, n_pt, n_ls):
    """The first n_pt points and n_ls lines of a keyframe."""
    return {k: (v[:n_ls] if k.startswith("ls_") or k == "ldesc" else v[:n_pt]) for k, v in f.items()}


def batch_context(cams=CAMS, **over):
    """A context of camera CAM whose sequences 0-3 have cams[s] (None: the context's camera, never set)."""
    fe = plf.Frontend(camera=CAM, max_sequences=4, **PRM, **over)
    for s, c in enumerate(cams):
        if c is not None:
            fe.set_sequence_camera(s, c)
    return fe


def same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def check_kf2kf_batch(fe, problems, seq, fast, over):
    """The batch on fe against the oracle and the single call on a context created with each problem's camera."""
    got = fe.match_kf2kf_batch(problems, seq=seq, fast_matching=fast)
    singles = {}
    try:
        for pr, s, g in zip(problems, seq, got):
            if s not in singles:
                singles[s] = plf.Frontend(camera=cam_of(s), **PRM, **over)
            one = singles[s].match_kf2kf(pr["prev"], pr["curr"], pr["DT"], fast_matching=fast)
            same(g, one)
            m_pt, n_pt, m_ls, n_ls = kfm.match_kf2kf(cam_of(s), prm_of(fe), pr["prev"], pr["curr"], pr["DT"], fast_matching=fast)
            assert np.array_equal(g["m_pt"], m_pt) and g["n_pt"] == n_pt
            assert np.array_equal(g["m_ls"], m_ls) and g["n_ls"] == n_ls
    finally:
        for f in singles.values():
            f.close()
    return got


def kf2kf_problems(seqs):
    """(problems, seq): per sequence a pair 1 frame apart, one 5 apart and one against a thinned keyframe (too few
    features for the fallback), plus two with the context's camera; interleaved."""
    probs, seq = [], []
    for a, b, th in ((0, 1, False), (0, 5, False), (2, 3, True)):
        for s in (0, 2, 1, 3):
            T_wc, feats = seqs[s]
            curr = thin(feats[b], 40, 6) if th else feats[b]
            probs.append(dict(prev=feats[a], curr=curr, DT=DT_between(T_wc, a, b)))
            seq.append(s)
    for s, (a, b) in ((1, (1, 3)), (3, (4, 6))):
        T_wc, feats = seqs[s]
        probs.append(dict(prev=feats[a], curr=feats[b], DT=DT_between(T_wc, a, b)))
        seq.append(-1)
    return probs, seq


@pytest.mark.parametrize("ws", [3, 10])
@pytest.mark.parametrize("fast", [0, 1])
def test_kf2kf_mixed_batch(seqs, fast, ws):
    probs, seq = kf2kf_problems(seqs)
    # min_*_matches at the median of the windowed counts, and above the thinned keyframe's features: within the batch,
    # problems with more windowed matches keep them, the full ones with fewer fall back to match(), and the thinned ones
    # cannot.  (KF-to-KF query lines stay in pixels, so the windowed line counts are mostly 0.)
    with batch_context(matching_f2f_ws=ws, min_pt_matches=0, min_ls_matches=0) as fe:
        win = fe.match_kf2kf_batch(probs, seq=seq, fast_matching=1)
    over = dict(matching_f2f_ws=ws)
    for kind, n_thin in (("pt", 40), ("ls", 6)):
        over["min_%s_matches" % kind] = max(int(np.median([w["n_" + kind] for w in win])), n_thin + 2)
    with batch_context(**over) as fe:
        got = check_kf2kf_batch(fe, probs, seq, fast, over)
    for kind, key in (("pt", "pdesc"), ("ls", "ldesc")):
        kmin = over["min_%s_matches" % kind]
        fell = [len(p["prev"][key]) > kmin and len(p["curr"][key]) > kmin and (w["n_" + kind] if fast else 0) < kmin
                for p, w in zip(probs, win)]
        assert any(fell) and not all(fell), (kind, kmin, fell)
    assert sum(g["n_pt"] > 0 for g in got) >= len(got) // 2


def map2kf_problems(seqs, rng):
    """(problems, seq): maps of different sizes in one batch, the edge cases among them."""
    probs, seq = [], []
    empty = dict(pt_X=np.zeros((0, 3)), pt_desc=np.zeros((0, 32), np.uint8), ls_X=np.zeros((0, 6)), ls_desc=np.zeros((0, 32), np.uint8))
    for s in range(4):
        T_wc, feats = seqs[s]
        kf, Twf = feats[5], np.linalg.inv(T_wc[5])
        big = local_map(T_wc, feats, [0, 1, 2, 3, 4], rng)
        small = local_map(T_wc, feats, [3], rng, n_dup=8)
        pt_lm = np.where(rng.random(len(kf["pdesc"])) < 0.2, 3, -1).astype(np.int32)
        ls_lm = np.where(rng.random(len(kf["ldesc"])) < 0.2, 1, -1).astype(np.int32)
        probs += [dict(local_map=big, Twf=Twf, kf=kf, kf_pt_lm=pt_lm, kf_ls_lm=ls_lm),
                  dict(local_map=small, Twf=Twf, kf=kf)]
        seq += [s, s]
    T_wc, feats = seqs[1]
    kf, Twf = feats[4], np.linalg.inv(T_wc[4])
    lmap = local_map(T_wc, feats, [0, 1, 2], rng)
    no_lines = dict(kf, ls_spl=np.zeros((0, 2)), ls_epl=np.zeros((0, 2)), ls_le=np.zeros((0, 3)), ldesc=np.zeros((0, 32), np.uint8))
    unused = dict(lmap, pt_use=np.zeros(len(lmap["pt_X"]), np.uint8), ls_use=np.zeros(len(lmap["ls_X"]), np.uint8))
    probs += [dict(local_map=empty, Twf=Twf, kf=kf),
              dict(local_map=lmap, Twf=np.diag([1.0, 1.0, -1.0, 1.0]) @ Twf, kf=kf),    # nothing visible
              dict(local_map=unused, Twf=Twf, kf=kf),
              dict(local_map=lmap, Twf=Twf, kf=no_lines, kf_pt_lm=np.full(len(kf["pdesc"]), -1, np.int32)),
              dict(local_map=lmap, Twf=Twf, kf=kf, kf_pt_lm=np.zeros(len(kf["pdesc"]), np.int32)),   # every feature matched
              dict(local_map=lmap, Twf=Twf, kf=kf)]
    seq += [1, 1, 1, 1, 1, -1]
    return probs, seq


def check_map2kf_batch(fe, problems, seq, fast, epip, over):
    got = fe.match_map2kf_batch(problems, seq=seq, fast_matching=fast, max_kf_epip_p=epip[0], max_kf_epip_l=epip[1])
    singles = {}
    try:
        for pr, s, g in zip(problems, seq, got):
            if s not in singles:
                singles[s] = plf.Frontend(camera=cam_of(s), **PRM, **over)
            args = (pr["local_map"], pr["Twf"], pr["kf"], pr.get("kf_pt_lm"), pr.get("kf_ls_lm"))
            one = singles[s].match_map2kf(*args, fast_matching=fast, max_kf_epip_p=epip[0], max_kf_epip_l=epip[1])
            same(g, one)
            lm_pt, n_pt, lm_ls, n_ls = kfm.match_map2kf(cam_of(s), prm_of(fe), *args, fast_matching=fast,
                                                        max_kf_epip_p=epip[0], max_kf_epip_l=epip[1])
            assert np.array_equal(g["lm_pt"], lm_pt) and g["n_pt"] == n_pt
            assert np.array_equal(g["lm_ls"], lm_ls) and g["n_ls"] == n_ls
    finally:
        for f in singles.values():
            f.close()
    return got


@pytest.mark.parametrize("epip", [(1.0, 1.0), (3.0, 0.02)])
@pytest.mark.parametrize("fast", [0, 1])
def test_map2kf_mixed_batch(seqs, fast, epip):
    probs, seq = map2kf_problems(seqs, np.random.default_rng(7 + fast))
    with batch_context() as fe:
        got = check_map2kf_batch(fe, probs, seq, fast, epip, {})
    assert got[0]["n_pt"] > 0 and got[2]["n_pt"] > 0
    assert all(g["n_pt"] == g["n_ls"] == 0 for g in got[8:11])   # empty, nothing visible, all unused
    assert got[11]["n_ls"] == 0 and got[11]["n_pt"] > 0 and got[12]["n_pt"] == 0


def test_map2kf_batch_without_points(seqs):
    probs, seq = map2kf_problems(seqs, np.random.default_rng(9))
    with batch_context(has_points=0) as fe:
        got = check_map2kf_batch(fe, probs, seq, 1, (1.0, 1.0), dict(has_points=0))
    assert all(g["n_pt"] == 0 and (g["lm_pt"] == -1).all() for g in got) and got[0]["n_ls"] > 0


def test_context_camera_three_ways(seqs):
    """seq = None, all -1, and every sequence explicitly set to the context's camera give identical results."""
    kp, _ = kf2kf_problems(seqs)
    mp, _ = map2kf_problems(seqs, np.random.default_rng(11))
    runs = []
    for cams, seq in (([None] * 4, None), ([None] * 4, lambda n: [-1] * n), ([CAM] * 4, lambda n: [i % 4 for i in range(n)])):
        with batch_context(cams) as fe:
            runs.append((fe.match_kf2kf_batch(kp, seq=seq and seq(len(kp))), fe.match_map2kf_batch(mp, seq=seq and seq(len(mp)))))
    for other in runs[1:]:
        for a, b in zip(runs[0][0] + runs[0][1], other[0] + other[1]):
            same(a, b)
    with plf.Frontend(camera=CAM, **PRM) as one:
        for pr, g in zip(kp, runs[0][0]):
            same(g, one.match_kf2kf(pr["prev"], pr["curr"], pr["DT"]))


def test_order_and_single_problem_batches(seqs):
    """A reversed batch gives the same per-problem results; a one-problem batch equals the single call."""
    kp, ks = kf2kf_problems(seqs)
    mp, ms = map2kf_problems(seqs, np.random.default_rng(13))
    with batch_context() as fe:
        a, b = fe.match_kf2kf_batch(kp, seq=ks), fe.match_map2kf_batch(mp, seq=ms)
        ra, rb = fe.match_kf2kf_batch(kp[::-1], seq=ks[::-1]), fe.match_map2kf_batch(mp[::-1], seq=ms[::-1])
        for x, y in zip(a + b, ra[::-1] + rb[::-1]):
            same(x, y)
        for i in (0, 5, len(kp) - 1):
            same(fe.match_kf2kf_batch([kp[i]], seq=[ks[i]])[0], a[i])
        for i in (0, 3, 9, len(mp) - 1):
            same(fe.match_map2kf_batch([mp[i]], seq=[ms[i]])[0], b[i])
    with plf.Frontend(camera=CAMS[2], **PRM) as one:
        i = ks.index(2)
        same(one.match_kf2kf_batch([kp[i]])[0], one.match_kf2kf(kp[i]["prev"], kp[i]["curr"], kp[i]["DT"]))
        pr = mp[ms.index(2)]
        same(one.match_map2kf_batch([pr])[0],
             one.match_map2kf(pr["local_map"], pr["Twf"], pr["kf"], pr.get("kf_pt_lm"), pr.get("kf_ls_lm")))
        assert one.match_kf2kf_batch([]) == [] and one.match_map2kf_batch([]) == []


def test_windowed_matcher_over_several_chunks(seqs):
    """One map of 65535 landmarks against a keyframe of 8192 points pads every problem of its batch to a 1 GB distance
    matrix, so the matcher runs the four problems in two chunks of at most 2 GB."""
    rng = np.random.default_rng(17)
    T_wc, feats = seqs[2]
    kf, Twf = feats[3], np.linalg.inv(T_wc[3])
    small = local_map(T_wc, feats, [1, 2], rng)
    n, m = 65535, 8192
    idx, j = rng.integers(0, len(small["pt_X"]), n), rng.integers(0, len(kf["pdesc"]), m)
    big = dict(small, pt_X=small["pt_X"][idx], pt_desc=small["pt_desc"][idx], pt_use=(rng.random(n) < 0.01).astype(np.uint8))
    big_kf = dict(kf, pt_pl=kf["pt_pl"][j], pdesc=kf["pdesc"][j], pt_P=kf["pt_P"][j])
    assert 4 * 2 * n * m > 2 ** 31
    probs = [dict(local_map=big, Twf=Twf, kf=big_kf, kf_pt_lm=np.where(rng.random(m) < 0.9, 0, -1).astype(np.int32))]
    seq = [2]
    for s in (0, 1, 3):
        T, f = seqs[s]
        probs.append(dict(local_map=local_map(T, f, [2, 3], rng), Twf=np.linalg.inv(T[4]), kf=f[4]))
        seq.append(s)
    with batch_context() as fe:
        got = check_map2kf_batch(fe, probs, seq, 1, (1.0, 1.0), {})
    assert got[0]["n_pt"] > 0 and all(g["n_pt"] > 0 for g in got[1:])


def _kf2kf_raw(fe, probs, seq=None, n=None, keep=None):
    """plf_match_kf2kf_batch through ctypes on sentinel outputs: (return code, whether any output changed)."""
    keep = [] if keep is None else keep
    arr = (plf.plf_kf2kf_problem * max(len(probs), 1))()
    outs = []
    for k, pr in enumerate(probs):
        p, c = plf._frame_view(pr["prev"], keep), plf._frame_view(pr["curr"], keep)
        keep += [p, c]
        o = [np.full(max(p.n_pt, 1), -7, np.int32), np.full(max(p.n_ls, 1), -7, np.int32)]
        outs += o
        arr[k] = plf.plf_kf2kf_problem(C.pointer(p), C.pointer(c), (C.c_double * 16)(*np.asarray(pr["DT"], np.float64).ravel()),
                                       o[0].ctypes.data, o[1].ctypes.data, 12345, 12345)
        for key, v in pr.get("raw", {}).items():
            setattr(arr[k], key, v)
    s = None if seq is None else np.asarray(seq, np.int32)
    o = plf.plf_kf_match_opts(1, 1.0, 1.0)
    rc = fe.lib.plf_match_kf2kf_batch(fe._ctx, C.byref(o), len(probs) if n is None else n, arr,
                                      None if s is None else s.ctypes.data_as(C.POINTER(C.c_int32)))
    changed = any((a != -7).any() for a in outs) or any(arr[k].n_pt != 12345 or arr[k].n_ls != 12345 for k in range(len(probs)))
    return rc, changed


def _kf2kf_many(fe, pr, n):
    """n copies of one problem, all writing to one sentinel output, through ctypes: as _kf2kf_raw."""
    keep = []
    p, c = plf._frame_view(pr["prev"], keep), plf._frame_view(pr["curr"], keep)
    m_pt, m_ls = np.full(max(p.n_pt, 1), -7, np.int32), np.full(max(p.n_ls, 1), -7, np.int32)
    one = plf.plf_kf2kf_problem(C.pointer(p), C.pointer(c), (C.c_double * 16)(*np.asarray(pr["DT"], np.float64).ravel()),
                                m_pt.ctypes.data, m_ls.ctypes.data, 12345, 12345)
    arr = (plf.plf_kf2kf_problem * n)(*([one] * n))
    o = plf.plf_kf_match_opts(1, 1.0, 1.0)
    rc = fe.lib.plf_match_kf2kf_batch(fe._ctx, C.byref(o), n, arr, None)
    return rc, bool((m_pt != -7).any() or (m_ls != -7).any() or any(a.n_pt != 12345 or a.n_ls != 12345 for a in arr))


def _map2kf_raw(fe, probs, seq=None):
    keep = []
    arr = (plf.plf_map2kf_problem * max(len(probs), 1))()
    outs = []
    for k, pr in enumerate(probs):
        kv = plf._frame_view(pr["kf"], keep)
        m, _, _ = plf._local_map(pr["local_map"], kv, None, None, keep, "raw")
        keep += [kv, m]
        o = [np.full(max(m.n_pt, 1), -7, np.int32), np.full(max(m.n_ls, 1), -7, np.int32)]
        outs += o
        arr[k] = plf.plf_map2kf_problem(C.pointer(m), C.pointer(kv), (C.c_double * 16)(*np.asarray(pr["Twf"], np.float64).ravel()),
                                        None, None, o[0].ctypes.data, o[1].ctypes.data, 12345, 12345)
    s = None if seq is None else np.asarray(seq, np.int32)
    o = plf.plf_kf_match_opts(1, 1.0, 1.0)
    rc = fe.lib.plf_match_map2kf_batch(fe._ctx, C.byref(o), len(probs), arr,
                                       None if s is None else s.ctypes.data_as(C.POINTER(C.c_int32)))
    changed = any((a != -7).any() for a in outs) or any(arr[k].n_pt != 12345 or arr[k].n_ls != 12345 for k in range(len(probs)))
    return rc, changed


def test_refusals_before_any_work(seqs):
    kp, ks = kf2kf_problems(seqs)
    kp, ks = kp[:4], ks[:4]
    mp, ms = map2kf_problems(seqs, np.random.default_rng(19))
    mp, ms = mp[:4], ms[:4]
    f0 = kp[2]["prev"]
    many = dict(f0, pt_pl=np.resize(f0["pt_pl"], (8193, 2)), pt_P=np.resize(f0["pt_P"], (8193, 3)),
                pdesc=np.resize(f0["pdesc"], (8193, 32)))
    lm = mp[2]["local_map"]
    n = 65536
    huge = dict(lm, pt_X=np.resize(lm["pt_X"], (n, 3)), pt_desc=np.resize(lm["pt_desc"], (n, 32)), pt_use=None)
    nan_DT = np.eye(4); nan_DT[1, 3] = np.nan
    with batch_context() as fe:
        ref_k, ref_m = fe.match_kf2kf_batch(kp, seq=ks), fe.match_map2kf_batch(mp, seq=ms)
        cases = [
            (lambda: _kf2kf_raw(fe, kp, ks, n=-1), PLF_ERR_INVALID, "n_problems = -1"),
            (lambda: _kf2kf_raw(fe, kp, [0, 1, 4, 2]), PLF_ERR_INVALID, "problem 2: seq[2] = 4"),
            (lambda: _kf2kf_raw(fe, kp, [0, -2, 1, 2]), PLF_ERR_INVALID, "problem 1: seq[1] = -2"),
            (lambda: _kf2kf_raw(fe, kp[:2] + [dict(kp[2], raw=dict(m_pt=None))] + kp[3:], ks), PLF_ERR_INVALID,
             "problem 2: a feature array is NULL"),
            (lambda: _kf2kf_raw(fe, kp[:3] + [dict(kp[3], DT=nan_DT)], ks), PLF_ERR_INVALID, "problem 3: prev, curr and a finite DT"),
            (lambda: _kf2kf_raw(fe, kp[:1] + [dict(kp[1], prev=many)] + kp[2:], ks), PLF_ERR_INVALID, "problem 1: n_pt=8193"),
            (lambda: _kf2kf_many(fe, kp[0], 65536), PLF_ERR_CAPACITY, "n_problems = 65536 exceeds 65535"),
            (lambda: _map2kf_raw(fe, mp[:2] + [dict(mp[2], local_map=huge)] + mp[3:], ms), PLF_ERR_INVALID,
             "problem 2: map n_pt=65536"),
            (lambda: _map2kf_raw(fe, mp[:3] + [dict(mp[3], Twf=nan_DT)], ms), PLF_ERR_INVALID, "problem 3: map, kf and a finite Twf"),
            (lambda: _map2kf_raw(fe, mp, [0, 0, 9, 0]), PLF_ERR_INVALID, "problem 2: seq[2] = 9"),
        ]
        for run, code, msg in cases:
            rc, changed = run()
            assert rc == code and not changed, (msg, rc)
            assert msg in fe.lib.plf_last_error(fe._ctx).decode(), msg
        assert _kf2kf_raw(fe, []) == (0, False)
        for a, b in zip(ref_k + ref_m, fe.match_kf2kf_batch(kp, seq=ks) + fe.match_map2kf_batch(mp, seq=ms)):
            same(a, b)
        with pytest.raises(plf.PlfError, match="seq"):
            fe.match_kf2kf_batch(kp, seq=[0, 1])


def test_launch_count_does_not_grow_with_the_batch(seqs):
    T_wc, feats = seqs[0]
    kp = dict(prev=feats[0], curr=feats[5], DT=DT_between(T_wc, 0, 5))
    mp = dict(local_map=local_map(T_wc, feats, [0, 1, 2], np.random.default_rng(23)), Twf=np.linalg.inv(T_wc[5]), kf=feats[5])
    counts = []
    with batch_context() as fe:
        for P in (1, 8, 32):
            seq = [p % 4 for p in range(P)]
            n0 = fe.launches
            a = fe.match_kf2kf_batch([kp] * P, seq=seq)
            b = fe.match_map2kf_batch([mp] * P, seq=seq)
            counts.append(fe.launches - n0)
            assert a[0]["n_pt"] > 0 and b[0]["n_pt"] > 0   # (the copies routed to other cameras match less)
    assert counts[0] == counts[1] == counts[2], counts
