"""GPU tests of the adaptive FAST threshold (plf_set_adaptive_fast / plf_get_sequence_fast_th) in the batched pipeline.

Round-robin streams at KITTI shape, each sequence with its own camera, mix rich frames with near-flat ones (the same
synth.World at a low albedo_sigma) and blank ones, so that the thresholds reach min_th and max_th and take every live
branch of the rule.  Every pair is checked against the oracle pipeline run at the threshold the device used
(oracle/frontend.py run_sequence with oracle/adaptive_fast.py), and every threshold the device carries against the rule applied to its own result."""
import subprocess

import cv2
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import synth
from oracle.adaptive_fast import result_next
from oracle.frontend import run_sequence
from test_multi_sequence_gpu import assert_same
from test_pipeline_gpu import compare
from test_shim import DEMO, write_frames

pytestmark = pytest.mark.gpu

K = plf.KITTI_CAMERA
CAMS = [dict(K, fx=K["fx"] * (1 + 0.01 * (c - 1.5)), fy=K["fy"] * (1 + 0.012 * (c - 1.5)), cx=K["cx"] + 1.5 * (c - 2),
             cy=K["cy"] - 0.75 * (c - 2), b=K["b"] * (1 + 0.02 * (c - 1.5))) for c in range(4)]
PRM = dict(orb_nfeatures=1500, lsd_nfeatures=200)
CFG = dict(min_th=0, max_th=50, inc_th=10, feat_th=50, err_th=0.5)   # min 0 as config_kitti.yaml; inc 10 reaches both ends
# albedo_sigma of each pair (0 = a blank pair: no features, status 1); rich 60, near-flat 8 and 20
SCHEDULES = [[60, 60, 60, 60, 8, 8, 8, 60], [60, 20, 20, 20, 60, 60], [60, 60, 0, 0, 60, 60], [8, 8, 60, 60, 60, 60, 60]]

_CACHE = {}


def sequences():
    """Sequence s: SCHEDULES[s] pairs rendered with CAMS[s] along one trajectory through worlds that differ only in albedo
    contrast (one seed: the same quads and segments).  The sequences share the world and the trajectory; their cameras
    and schedules differ."""
    if "seqs" not in _CACHE:
        seqs = []
        for s, sig in enumerate(SCHEDULES):
            rendered = {}
            for a in sorted(set(sig) - {0}):
                world = synth.World(seed=3, albedo_sigma=float(a))
                rendered[a] = list(synth.stream(CAMS[s], len(sig), world=world, seed=4))
            blank = np.full((K["height"], K["width"]), 128, np.uint8)
            seqs.append([(blank, blank) if a == 0 else rendered[a][i][:2] for i, a in enumerate(sig)])
        _CACHE["seqs"] = seqs
    return _CACHE["seqs"]


def round_robin(seqs):
    return [[(s, i) for s in range(len(seqs)) if i < len(seqs[s])] for i in range(max(map(len, seqs)))]


def make(nseq, B, cfg=CFG, cams=CAMS):
    lim = plf.default_limits()
    lim.max_batch = B
    fe = plf.Frontend(camera=K, limits=lim, max_sequences=nseq, adaptive_fast=cfg, **PRM)
    for s in range(nseq):
        fe.set_sequence_camera(s, cams[s])
    return fe


def run_device(seqs, batches, in_flight=1, views=True, cfg=CFG):
    """The batches through one context; returns {(s, i): (result, frame, matches)} (views only with in_flight = 1),
    {(s, i): threshold pair i was detected with} and {(s, i): the sequence's threshold after the batch}."""
    out, th_used, th_after = {}, {}, {}
    with make(len(seqs), max(map(len, batches)), cfg) as fe:
        pending = []
        for j, batch in enumerate(batches):
            if in_flight == 1:
                th_used.update({key: fe.sequence_fast_th(key[0]) for key in batch})
            fe.batch_upload(np.stack([seqs[s][i][0] for s, i in batch]), np.stack([seqs[s][i][1] for s, i in batch]))
            fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
            pending.append(batch)
            if len(pending) == in_flight or j == len(batches) - 1:
                while pending:
                    b = pending.pop(0)
                    res = fe.batch_download_array(len(b))
                    for k, key in enumerate(b):
                        out[key] = (res[k], fe.get_frame(k), fe.get_matches(k)) if views else (res[k],)
                if in_flight == 1:
                    th_after.update({key: fe.sequence_fast_th(key[0]) for key in batch})
        final = [fe.sequence_fast_th(s) for s in range(len(seqs))]
    return out, th_used, th_after, final


def as_dict(r):
    return {f: (np.array(r[f]).reshape(4, 4) if f == "DT" else np.array(r[f]).reshape(6, 6) if f == "DT_cov" else r[f].item())
            for f in r.dtype.names}


def cv2_count(img, th):
    orb = cv2.ORB_create(PRM["orb_nfeatures"], 1.2, 4, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, th)
    return len(orb.detect(img, None))


def test_round_robin_matches_oracle(built):
    seqs = sequences()
    got, th_used, th_after, _ = run_device(seqs, round_robin(seqs))
    branches, ths = set(), set()
    for s in range(len(seqs)):
        n = len(seqs[s])
        ths_s = [th_used[(s, i)] for i in range(n)]
        assert ths_s[0] == 20   # a first frame: orb_fast_th
        ref = run_sequence(CAMS[s], seqs[s], PRM, adaptive_fast=CFG, fast_th=ths_s)
        res = [as_dict(got[(s, i)][0]) for i in range(n)]
        compare(ref, res, [got[(s, i)][1] for i in range(n)])
        for i in range(n):
            r = got[(s, i)][0]
            if ref[i]["status"] == 0:   # the matches, bit for bit (pose rows: P from the previous frame, obs from this one)
                m, tr = got[(s, i)][2], ref[i]["res"]["rows"]
                assert np.array_equal(m["P"], tr["P"]) and np.array_equal(m["pl_obs"], tr["obs"]), (s, i)
                assert np.array_equal(m["sP"], tr["sP"]) and np.array_equal(m["le_obs"], tr["le"]), (s, i)
            nxt, b = result_next(ths_s[i], as_dict(r), CFG, trace=True)
            assert th_after[(s, i)] == nxt, (s, i, ths_s[i], b)   # the device's update is the rule on its own result
            if i + 1 < n:
                assert th_used[(s, i + 1)] == nxt
            L, R = seqs[s][i]
            assert (r["n_kp_l"], r["n_kp_r"]) == (cv2_count(L, ths_s[i]), cv2_count(R, ths_s[i])), (s, i, ths_s[i])
            branches.add(b)
            ths.add(ths_s[i])
    print("branches", sorted(branches), "thresholds", sorted(ths))
    assert {CFG["min_th"], CFG["max_th"]} <= ths
    assert branches == {"first", "bad_pose", "few", "some", "keep", "many"}


def test_in_flight_equals_one_at_a_time(built):
    """Three batches in flight, each E phase waiting for the previous batch's threshold update: bit-identical results
    and final thresholds."""
    seqs = sequences()
    ref, _, _, th_ref = run_device(seqs, round_robin(seqs), views=False)
    got, _, _, th_got = run_device(seqs, round_robin(seqs), in_flight=3, views=False)
    assert th_got == th_ref
    for key in ref:
        for f in ref[key][0].dtype.names:
            assert ref[key][0][f].tobytes() == got[key][0][f].tobytes(), (key, f)


def test_each_sequence_alone_equals_round_robin(built):
    seqs = sequences()
    rr, th_used, _, _ = run_device(seqs, round_robin(seqs))
    alone = {}
    for s in range(len(seqs)):
        lim = plf.default_limits()
        lim.max_batch = 1
        with plf.Frontend(camera=CAMS[s], limits=lim, adaptive_fast=CFG, **PRM) as fe:
            for i, (L, R) in enumerate(seqs[s]):
                assert fe.sequence_fast_th(0) == th_used[(s, i)], (s, i)
                fe.batch_upload(L, R)
                fe.batch_run(1)
                alone[(s, i)] = (fe.batch_download_array(1)[0], fe.get_frame(0), fe.get_matches(0))
    assert_same(alone, rr)


def test_two_pairs_of_one_sequence_are_refused(built):
    seqs = sequences()[:2]
    batches = round_robin(seqs)[:4]
    ref, _, _, th_ref = run_device(seqs, batches, views=False)
    got = {}
    with make(2, 3) as fe:
        for j, batch in enumerate(batches):
            if j == 2:   # two pairs of sequence 0 in one batch: refused, nothing changes
                before = [fe.sequence_fast_th(s) for s in range(2)]
                bad = [(0, 2), (1, 2), (0, 3)]
                fe.batch_upload(np.stack([seqs[s][i][0] for s, i in bad]), np.stack([seqs[s][i][1] for s, i in bad]))
                with pytest.raises(plf.PlfError, match=r"pairs 0 and 2 are both of sequence 0"):
                    fe.batch_run(3, seq=np.array([0, 1, 0], np.int32))
                with pytest.raises(plf.PlfError, match=r"both of sequence 0"):
                    fe.batch_run(2)   # seq NULL: every pair is sequence 0
                assert [fe.sequence_fast_th(s) for s in range(2)] == before
            fe.batch_upload(np.stack([seqs[s][i][0] for s, i in batch]), np.stack([seqs[s][i][1] for s, i in batch]))
            fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
            res = fe.batch_download_array(len(batch))
            for k, key in enumerate(batch):
                got[key] = res[k]
        assert [fe.sequence_fast_th(s) for s in range(2)] == th_ref
    for key in ref:
        for f in ref[key][0].dtype.names:
            assert ref[key][0][f].tobytes() == got[key][f].tobytes(), (key, f)


def test_refused_settings_change_nothing(built):
    seqs = sequences()[:1]
    with make(1, 1) as fe:
        for i in range(3):
            fe.process_batch(*seqs[0][i])
        th = fe.sequence_fast_th(0)
        assert th != 20
        for field, v in (("min_th", -1), ("max_th", 256), ("min_th", 51), ("inc_th", -1), ("feat_th", -1), ("err_th", float("nan"))):
            with pytest.raises(plf.PlfError, match=field):
                fe.set_adaptive_fast(dict(CFG, **{field: v}))
            assert fe.sequence_fast_th(0) == th
        fe.batch_upload(*seqs[0][3])
        fe.batch_run(1)
        with pytest.raises(plf.PlfError, match="in flight"):
            fe.set_adaptive_fast(CFG)
        with pytest.raises(plf.PlfError, match="in flight"):
            fe.set_adaptive_fast(None)
        fe.batch_download(1)
        fe.reset_sequence()
        assert fe.sequence_fast_th(0) == 20
        with pytest.raises(plf.PlfError, match="outside"):
            fe.sequence_fast_th(1)


def _off_run(seqs, setup):
    """Two sequences in batches of B = 4 (two pairs of each: allowed with the adaptation off)."""
    order = [(s, i) for i in range(6) for s in range(2)]
    batches = [order[j:j + 4] for j in range(0, len(order), 4)]
    out = {}
    lim = plf.default_limits()
    lim.max_batch = 4
    with plf.Frontend(camera=K, limits=lim, max_sequences=2, **PRM) as fe:
        for s in range(2):
            fe.set_sequence_camera(s, CAMS[s])
        setup(fe)
        for batch in batches:
            fe.batch_upload(np.stack([seqs[s][i][0] for s, i in batch]), np.stack([seqs[s][i][1] for s, i in batch]))
            fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
            res = fe.batch_download_array(len(batch))
            for k, key in enumerate(batch):
                out[key] = (res[k], fe.get_frame(k), fe.get_matches(k))
        assert all(fe.sequence_fast_th(s) == 20 for s in range(2))
    return out


def test_off_is_bit_identical(built):
    seqs = sequences()[:2]
    never = _off_run(seqs, lambda fe: None)
    assert_same(never, _off_run(seqs, lambda fe: fe.set_adaptive_fast(None)))

    def on_then_off(fe):
        fe.set_adaptive_fast(CFG)
        fe.set_adaptive_fast(None)
    assert_same(never, _off_run(seqs, on_then_off))


def test_turned_on_mid_stream_restarts_thresholds(built):
    """Turning the adaptation on after batches have run starts every sequence at orb_fast_th; its sequences keep their
    carried frames (the next pair tracks)."""
    seqs = sequences()[:2]
    with make(2, 2, cfg=None) as fe:
        fe.batch_upload(np.stack([seqs[s][0][0] for s in range(2)]), np.stack([seqs[s][0][1] for s in range(2)]))
        fe.batch_run(2, seq=np.array([0, 1], np.int32))
        fe.batch_download(2)
        fe.set_adaptive_fast(CFG)
        assert [fe.sequence_fast_th(s) for s in range(2)] == [20, 20]
        fe.batch_upload(np.stack([seqs[s][1][0] for s in range(2)]), np.stack([seqs[s][1][1] for s in range(2)]))
        fe.batch_run(2, seq=np.array([0, 1], np.int32))
        res = fe.batch_download(2)
        assert [r["status"] for r in res] == [0, 0]
        assert [fe.sequence_fast_th(s) for s in range(2)] == [result_next(20, r, CFG) for r in res]


def test_vo_demo_flag_matches_binding(built, tmp_path):
    seqs = sequences()
    frames = seqs[0]
    p = tmp_path / "frames.bin"
    write_frames(p, CAMS[0], frames)
    args = [str(v) for v in (CFG["min_th"], CFG["max_th"], CFG["inc_th"], CFG["feat_th"], CFG["err_th"])]
    r = subprocess.run([str(DEMO), str(p), str(PRM["orb_nfeatures"]), str(PRM["lsd_nfeatures"]), "--adaptive-fast", *args],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().splitlines()]
    rows = [ln for ln in lines if ln[0] != "fast_th"]
    ths = [int(ln[2]) for ln in lines if ln[0] == "fast_th"]
    assert len(rows) == len(ths) == len(frames)
    lim = plf.default_limits()
    lim.max_batch = 1
    T = np.eye(4)
    with plf.Frontend(camera=CAMS[0], limits=lim, adaptive_fast=CFG, **PRM) as fe:
        for k, (L, R) in enumerate(frames):
            assert ths[k] == fe.sequence_fast_th(0), k
            g = fe.process_batch(L, R)[0]
            T = T @ g["DT"]
            row = rows[k]
            assert int(row[0]) == k and int(row[1]) == g["status"]
            assert int(row[2]) == g["n_stereo_pt"] and int(row[3]) == g["n_stereo_ls"]
            assert np.allclose(np.array([float(v) for v in row[6:22]]).reshape(4, 4), T, rtol=0, atol=1e-12)
    assert len(set(ths)) >= 3
