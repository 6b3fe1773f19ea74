"""GPU tests of the motion model (plf_set_motion_model / plf_get_sequence_motion / plf_debug_motion_prior) in the batched
pipeline.

Round-robin streams of several sequences, each with its own camera, at KITTI and EuRoC shape, with matching_strategy 0
and 3 and with adaptive FAST thresholds on.  Every pair is checked against the oracle pipeline run with the predictions
the device used (oracle/frontend.py run_sequence with oracle/motion_model.py), and every prediction the device carries against the rule applied to the
device's own result of the previous pair."""
import subprocess

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import synth
from oracle.frontend import run_sequence
from oracle.motion_model import prior, result_prior
from test_motion_model import EDGES
from test_multi_sequence_gpu import assert_same
from test_pipeline_gpu import compare
from test_shim import DEMO, write_frames

pytestmark = pytest.mark.gpu

KITTI, EUROC = plf.KITTI_CAMERA, plf.EUROC_CAMERA


def cams(base, n):
    return [dict(base, fx=base["fx"] * (1 + 0.01 * (c - 1)), fy=base["fy"] * (1 + 0.012 * (c - 1)), cx=base["cx"] + 1.5 * (c - 1),
                 cy=base["cy"] - 0.75 * (c - 1), b=base["b"] * (1 + 0.02 * (c - 1))) for c in range(n)]


SHAPES = {
    "kitti": dict(cam=KITTI, prm=dict(orb_nfeatures=1500, lsd_nfeatures=200), n=(4, 3, 4), stream={}),
    "euroc": dict(cam=EUROC, prm=dict(orb_nfeatures=1200, lsd_nfeatures=300), n=(3, 4),
                  stream=dict(step=0.08, yaw_deg=0.8),
                  world=dict(seed=8, length=40.0, n_quads=220, n_segs=120, half_width=5.0, half_height=3.0)),
}
AFAST = dict(min_th=5, max_th=50, inc_th=5, feat_th=50, err_th=0.5)   # config_euroc.yaml:36-41

_CACHE = {}


def sequences(shape):
    """Sequence s of a shape: n[s] pairs rendered with its own camera along its own trajectory."""
    if shape not in _CACHE:
        sh = SHAPES[shape]
        cs = cams(sh["cam"], len(sh["n"]))
        seqs = []
        for s, n in enumerate(sh["n"]):
            world = synth.World(**sh["world"]) if "world" in sh else None
            seqs.append([f[:2] for f in synth.stream(cs[s], n, world=world, seed=40 + 7 * s, **sh["stream"])])
        _CACHE[shape] = (cs, seqs)
    return _CACHE[shape]


def round_robin(seqs):
    return [[(s, i) for s in range(len(seqs)) if i < len(seqs[s])] for i in range(max(map(len, seqs)))]


def make(base, cs, B, prm, motion=True, afast=None):
    lim = plf.default_limits()
    lim.max_batch = B
    fe = plf.Frontend(camera=base, limits=lim, max_sequences=len(cs), adaptive_fast=afast, motion_model=motion, **prm)
    for s, c in enumerate(cs):
        fe.set_sequence_camera(s, c)
    return fe


def upload_run(fe, seqs, batch, restart=None):
    fe.batch_upload(np.stack([seqs[s][i][0] for s, i in batch]), np.stack([seqs[s][i][1] for s, i in batch]))
    fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32), restart=restart)


def run_device(shape, prm, afast=None):
    """The round-robin batches through one context, one batch at a time: {(s, i): (result, frame, matches)}, the
    prediction each pair started from, the one its sequence carries after it, and the FAST threshold it was detected at."""
    sh = SHAPES[shape]
    cs, seqs = sequences(shape)
    out, used, after, ths = {}, {}, {}, {}
    batches = round_robin(seqs)
    with make(sh["cam"], cs, max(map(len, batches)), prm, afast=afast) as fe:
        for batch in batches:
            for key in batch:
                used[key] = fe.sequence_motion(key[0])
                ths[key] = fe.sequence_fast_th(key[0])
            upload_run(fe, seqs, batch)
            res = fe.batch_download_array(len(batch))
            for k, key in enumerate(batch):
                out[key] = (res[k], fe.get_frame(k), fe.get_matches(k))
                after[key] = fe.sequence_motion(key[0])
    return out, used, after, ths


def as_dict(r):
    return {f: (np.array(r[f]).reshape(4, 4) if f == "DT" else np.array(r[f]).reshape(6, 6) if f == "DT_cov" else r[f].item())
            for f in r.dtype.names}


@pytest.mark.parametrize("shape, strategy, afast", [("kitti", 0, False), ("kitti", 3, False), ("kitti", 3, True),
                                                    ("euroc", 0, False), ("euroc", 3, False)])
def test_streams_match_oracle(built, shape, strategy, afast):
    sh = SHAPES[shape]
    cs, seqs = sequences(shape)
    prm = dict(sh["prm"], matching_strategy=strategy)
    got, used, after, ths = run_device(shape, prm, AFAST if afast else None)
    valid_used = 0
    for s in range(len(seqs)):
        n = len(seqs[s])
        preds = [used[(s, i)][0] for i in range(n)]
        assert np.array_equal(preds[0], np.eye(4)) and not used[(s, 0)][1]   # a first frame starts from identity
        ref = run_sequence(cs[s], seqs[s], prm, motion_model=True, preds=preds, fast_th=[ths[(s, i)] for i in range(n)] if afast else None)
        res = [as_dict(got[(s, i)][0]) for i in range(n)]
        compare(ref, res, [got[(s, i)][1] for i in range(n)])
        for i in range(n):
            r = got[(s, i)][0]
            if ref[i]["status"] == 0:   # the matches, bit for bit (P from the previous frame, obs from this one)
                m, tr = got[(s, i)][2], ref[i]["res"]["rows"]
                assert np.array_equal(m["P"], tr["P"]) and np.array_equal(m["pl_obs"], tr["obs"]), (s, i)
                assert np.array_equal(m["sP"], tr["sP"]) and np.array_equal(m["le_obs"], tr["le"]), (s, i)
            # the carried prediction is the rule on the device's own result, bit for bit
            T, valid = result_prior(r)
            assert after[(s, i)][1] == valid and np.array_equal(after[(s, i)][0], T), (s, i)
            if i + 1 < n:
                assert np.array_equal(used[(s, i + 1)][0], T) and used[(s, i + 1)][1] == valid
            valid_used += used[(s, i)][1]
    assert valid_used >= sum(len(q) - 2 for q in seqs)   # the streams do carry motion


def test_device_rule_at_each_edge(built):
    """plf_debug_motion_prior gives the oracle's decision and prediction at every edge (diagonal covariances: the
    eigenvalues are exact on both sides)."""
    with plf.Frontend() as fe:
        T, valid = fe.debug_motion_prior([e[2] for e in EDGES], [e[3] for e in EDGES], [e[4] for e in EDGES],
                                         [e[1] for e in EDGES])
    for k, (name, status, DT, cov, err, good) in enumerate(EDGES):
        T_o, v_o = prior(status, DT, cov, err)
        assert valid[k] == v_o == good, name
        assert np.array_equal(T[k], T_o), name


def test_two_pairs_of_one_sequence_are_refused(built):
    cs, seqs = sequences("kitti")
    prm = SHAPES["kitti"]["prm"]
    with make(KITTI, cs[:2], 3, prm) as fe:
        upload_run(fe, seqs, [(0, 0), (1, 0)])
        fe.batch_download(2)
        upload_run(fe, seqs, [(0, 1), (1, 1)])
        fe.batch_download(2)
        before = [fe.sequence_motion(s) for s in range(2)]
        assert all(v for _, v in before)
        bad = [(0, 2), (1, 2), (0, 3)]
        fe.batch_upload(np.stack([seqs[s][i][0] for s, i in bad]), np.stack([seqs[s][i][1] for s, i in bad]))
        with pytest.raises(plf.PlfError, match=r"pairs 0 and 2 are both of sequence 0; with the motion model"):
            fe.batch_run(3, seq=np.array([0, 1, 0], np.int32))
        with pytest.raises(plf.PlfError, match=r"both of sequence 0"):
            fe.batch_run(2)   # seq NULL: every pair is sequence 0
        after = [fe.sequence_motion(s) for s in range(2)]
        for (Ta, va), (Tb, vb) in zip(before, after):
            assert va == vb and np.array_equal(Ta, Tb)
        # the next good batch tracks against the carried frames and predictions as if nothing happened
        upload_run(fe, seqs, [(0, 2), (1, 2)])
        assert [r["status"] for r in fe.batch_download(2)] == [0, 0]
        # enabling (or disabling) with a batch in flight is refused
        upload_run(fe, seqs, [(0, 3), (1, 3)] if len(seqs[1]) > 3 else [(0, 3)])
        with pytest.raises(plf.PlfError, match="in flight"):
            fe.set_motion_model(True)
        with pytest.raises(plf.PlfError, match="in flight"):
            fe.set_motion_model(False)
        fe.batch_download(2 if len(seqs[1]) > 3 else 1)
        with pytest.raises(plf.PlfError, match="outside"):
            fe.sequence_motion(2)


def _identity(fe, s):
    T, valid = fe.sequence_motion(s)
    return np.array_equal(T, np.eye(4)) and not valid


def test_every_reset_gives_an_identity_seed(built):
    cs, seqs = sequences("kitti")
    prm = SHAPES["kitti"]["prm"]
    K = KITTI

    def warm(fe):   # two pairs of sequences 0 and 1: both carry a valid prediction
        for i in range(2):
            upload_run(fe, seqs, [(0, i), (1, i)])
            fe.batch_download(2)
        assert not _identity(fe, 0) and not _identity(fe, 1)

    with make(K, cs[:2], 2, prm) as fe:
        assert _identity(fe, 0) and _identity(fe, 1)            # before any pair: a first frame
        warm(fe)
        upload_run(fe, seqs, [(0, 2), (1, 2)], restart=np.array([1, 0], np.uint8))
        res = fe.batch_download(2)
        assert [r["status"] for r in res] == [2, 0]             # restart[k]: a first frame, no pose to predict from
        assert _identity(fe, 0) and not _identity(fe, 1)
        fe.reset_sequence()
        assert _identity(fe, 0) and _identity(fe, 1)
        warm(fe)
        fe.set_sequence_camera(0, cs[0])
        assert _identity(fe, 0) and not _identity(fe, 1)
        warm(fe)
        w, h = K["width"], K["height"]
        xy = np.stack(np.meshgrid(np.arange(w), np.arange(h)), -1).astype(np.int16)
        fe.set_sequence_rectification(1, left=(xy, np.zeros((h, w), np.uint16)), right=(xy, np.zeros((h, w), np.uint16)))
        assert not _identity(fe, 0) and _identity(fe, 1)
        fe.set_sequence_rectification(1)
        warm(fe)
        fe.set_motion_model(True)                                # every successful enable
        assert _identity(fe, 0) and _identity(fe, 1)
        upload_run(fe, seqs, [(0, 2), (1, 2)])
        assert [r["status"] for r in fe.batch_download(2)] == [0, 0]   # the carried frames stay: the pairs track
        fe.set_motion_model(False)
        assert _identity(fe, 0) and _identity(fe, 1)
    # plf_set_max_sequences (before the pipeline exists): every sequence of the new count starts from identity
    with make(K, cs, 3, prm) as fe:
        fe.lib.plf_set_max_sequences(fe._ctx, 2)
        assert _identity(fe, 0) and _identity(fe, 1)


def _off_run(setup):
    """Two sequences in batches of B = 4 (two pairs of each: allowed with the model off), matching_strategy 3."""
    cs, seqs = sequences("kitti")
    order = [(s, i) for i in range(3) for s in range(2)]
    batches = [order[j:j + 4] for j in range(0, len(order), 4)]
    out = {}
    with make(KITTI, cs[:2], 4, dict(SHAPES["kitti"]["prm"], matching_strategy=3), motion=False) as fe:
        setup(fe)
        for batch in batches:
            upload_run(fe, seqs, batch)
            res = fe.batch_download_array(len(batch))
            for k, key in enumerate(batch):
                out[key] = (res[k], fe.get_frame(k), fe.get_matches(k))
        assert _identity(fe, 0) and _identity(fe, 1)
    return out


def test_off_is_bit_identical(built):
    never = _off_run(lambda fe: None)
    assert_same(never, _off_run(lambda fe: fe.set_motion_model(False)))

    def on_then_off(fe):
        fe.set_motion_model(True)
        fe.set_motion_model(False)
    assert_same(never, _off_run(on_then_off))


def test_vo_demo_flag_matches_binding(built, tmp_path):
    cs, seqs = sequences("kitti")
    frames = seqs[0]
    prm = SHAPES["kitti"]["prm"]
    p = tmp_path / "frames.bin"
    write_frames(p, cs[0], frames)
    r = subprocess.run([str(DEMO), str(p), str(prm["orb_nfeatures"]), str(prm["lsd_nfeatures"]), "--motion-model"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().splitlines()]
    rows = [ln for ln in lines if ln[0] != "motion"]
    mot = [ln for ln in lines if ln[0] == "motion"]
    assert len(rows) == len(mot) == len(frames)
    lim = plf.default_limits()
    lim.max_batch = 1
    T = np.eye(4)
    with plf.Frontend(camera=cs[0], limits=lim, motion_model=True, **prm) as fe:
        for k, (L, R) in enumerate(frames):
            Tp, valid = fe.sequence_motion(0)
            assert int(mot[k][1]) == k and int(mot[k][2]) == int(valid), k
            assert np.array_equal(np.array([float(v) for v in mot[k][3:19]]).reshape(4, 4), Tp), k
            g = fe.process_batch(L, R)[0]
            T = T @ g["DT"]
            row = rows[k]
            assert int(row[0]) == k and int(row[1]) == g["status"]
            assert int(row[2]) == g["n_stereo_pt"] and int(row[3]) == g["n_stereo_ls"]
            assert np.allclose(np.array([float(v) for v in row[6:22]]).reshape(4, 4), T, rtol=0, atol=1e-12)
    assert sum(int(m[2]) for m in mot) >= len(frames) - 2
