"""GPU tests of per-sequence calibrations in one batched context (plf_set_sequence_camera / plf_get_sequence_camera).

The oracle is the library itself: every pair of a mixed batch whose sequences have their own cameras must give, bit for
bit, what a single-sequence context created with that sequence's camera gives for the same frames in the same order -
every plf_frame_result field (DT included), get_frame(k) and get_matches(k).  The single-camera path is pinned to the CPU
oracle by test_pipeline_gpu.py, so this ties the per-sequence path to it too.  Each sequence is rendered with its own
camera: one image size, distinct fx, fy, cx, cy and b."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import synth
from test_multi_sequence_gpu import assert_same, chunks, interleavings

pytestmark = pytest.mark.gpu

W, H = 640, 360
CAM = dict(plf.KITTI_CAMERA, width=W, height=H, cx=320.0, cy=180.0, fx=500.0, fy=500.0)   # the context's camera
CAMS = [   # one per sequence, none equal to CAM; fx * b differs between all of them, so every depth differs
    dict(width=W, height=H, fx=510.0, fy=508.0, cx=322.5, cy=178.0, b=0.537165719),
    dict(width=W, height=H, fx=470.0, fy=472.5, cx=314.5, cy=183.25, b=0.50),
    dict(width=W, height=H, fx=532.0, fy=527.0, cx=326.0, cy=176.5, b=0.57),
    dict(width=W, height=H, fx=455.0, fy=458.0, cx=317.0, cy=186.0, b=0.48),
]
NEW_CAM = dict(width=W, height=H, fx=488.0, fy=490.0, cx=318.0, cy=181.5, b=0.52)
PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
LENGTHS = (8, 12, 10, 9)

_FRAMES = {}


def sequences():
    """Four sequences of LENGTHS (left, right, T_wc), sequence s rendered with CAMS[s] through its own synth.World."""
    if "seqs" not in _FRAMES:
        seqs = []
        for s, n in enumerate(LENGTHS):
            world = synth.World(seed=40 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
            seqs.append(list(synth.stream(CAMS[s], n, world=world, seed=50 + s, step=0.15)))
        _FRAMES["seqs"] = seqs
    return _FRAMES["seqs"]


def limits(B):
    lim = plf.default_limits()
    lim.max_batch = B
    return lim


def collect(fe, keys, res, out, views=True):
    for k, key in enumerate(keys):
        out[key] = (res[k], fe.get_frame(k), fe.get_matches(k)) if views else (res[k],)


def alone(seqs, prm, segments):
    """segments: (s, a, b, camera) - pairs a .. b-1 of sequence s through a single-sequence context created with `camera`,
    reset_sequence() first.  Returns {(s, i): (result, frame, matches)}."""
    out, ctxs = {}, {}
    try:
        for s, a, b, cam in segments:
            key = tuple(sorted(cam.items()))
            if key not in ctxs:
                ctxs[key] = plf.Frontend(camera=cam, limits=limits(max(LENGTHS)), **prm)
            fe = ctxs[key]
            fe.reset_sequence()
            fe.batch_upload(np.stack([f[0] for f in seqs[s][a:b]]), np.stack([f[1] for f in seqs[s][a:b]]))
            fe.batch_run(b - a)
            collect(fe, [(s, i) for i in range(a, b)], fe.batch_download_array(b - a), out)
    finally:
        for fe in ctxs.values():
            fe.close()
    return out


def whole(seqs, cams):
    return [(s, 0, len(seqs[s]), cams[s]) for s in range(len(seqs))]


def batch_args(seqs, batch):
    L = np.stack([seqs[s][i][0] for s, i in batch])
    R = np.stack([seqs[s][i][1] for s, i in batch])
    return L, R, np.array([s for s, _ in batch], np.int32)


def mixed(seqs, batches, prm, cams, nseq=4, ctx_cam=CAM):
    """The batches through one context of camera ctx_cam with max_sequences = nseq; sequence s gets cams[s] (None: keep
    the context's) before the first batch."""
    out = {}
    with plf.Frontend(camera=ctx_cam, limits=limits(max(map(len, batches))), max_sequences=nseq, **prm) as fe:
        for s, c in enumerate(cams):
            if c is not None:
                fe.set_sequence_camera(s, c)
        for batch in batches:
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq)
            collect(fe, batch, fe.batch_download_array(len(batch)), out)
    return out


@pytest.mark.parametrize("strategy", [0, 3])
def test_mixed_calibrations_equal_each_sequence_alone(built, strategy):
    """Four sequences with four calibrations, in the four interleavings of test_multi_sequence_gpu.py: every pair equals
    its sequence run alone through a context created with its camera.  matching_strategy = 3 takes the windowed
    frame-to-frame path, whose query cells are the previous frame projected with the pair's camera."""
    prm = dict(PRM, matching_strategy=strategy)
    seqs = sequences()
    ref = alone(seqs, prm, whole(seqs, CAMS))
    tracked = sum(r["status"] == 0 for r, _, _ in ref.values())
    assert tracked >= 0.75 * (sum(LENGTHS) - len(LENGTHS)), tracked   # the sequences do track
    for name, batches in interleavings(LENGTHS).items():
        got = mixed(seqs, batches, prm, CAMS)
        assert_same(ref, got)
        for s in range(4):
            assert got[(s, 0)][0]["status"] == 2, (name, s)


def test_mixed_calibrations_three_batches_in_flight(built):
    """Up to three batches in flight, each with its own ring entry of pair cameras: results equal each sequence alone, and
    so do the frames and matches of the last batch."""
    prm = dict(PRM, matching_strategy=3)
    seqs = sequences()
    ref = alone(seqs, prm, whole(seqs, CAMS))
    batches = interleavings(LENGTHS)["random"]
    got = {}
    with plf.Frontend(camera=CAM, limits=limits(6), max_sequences=4, **prm) as fe:
        for s, c in enumerate(CAMS):
            fe.set_sequence_camera(s, c)
        pending = []
        for j, batch in enumerate(batches):
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq)
            pending.append(batch)
            if len(pending) == 3 or j == len(batches) - 1:
                while pending:
                    b = pending.pop(0)
                    res = fe.batch_download_array(len(b))
                    for k, key in enumerate(b):
                        got[key] = res[k]
        frames = {key: (fe.get_frame(k), fe.get_matches(k)) for k, key in enumerate(batches[-1])}
    assert got.keys() == ref.keys()
    for key in ref:
        for f in got[key].dtype.names:
            assert got[key][f].tobytes() == ref[key][0][f].tobytes(), (key, f)
    for key, (fr, ma) in frames.items():
        for a, b in ((fr, ref[key][1]), (ma, ref[key][2])):
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), (key, k)


def test_the_pair_camera_is_used(built):
    """The same batches with the calibrations permuted between the sequences: the stereo rows are the same (association
    reads pixels only) but every row's P, sP and eP changes, and so does the DT of every tracked pair.  With its own
    camera, each sequence recovers its planted motion (the tolerance of test_pipeline_gpu.py's planted trajectory)."""
    seqs = sequences()
    batches = interleavings(LENGTHS)["round_robin"]
    own = mixed(seqs, batches, PRM, CAMS)
    perm = mixed(seqs, batches, PRM, [CAMS[(s + 1) % 4] for s in range(4)])
    n_rows = 0
    for key in own:
        (ra, fa, _), (rb, fb, _) = own[key], perm[key]
        assert (ra["n_stereo_pt"], ra["n_stereo_ls"]) == (rb["n_stereo_pt"], rb["n_stereo_ls"]), key
        assert np.array_equal(fa["pt_pl"], fb["pt_pl"]) and np.array_equal(fa["ls_spl"], fb["ls_spl"]), key
        for f in ("pt_P", "ls_sP", "ls_eP"):
            assert np.all(np.any(fa[f] != fb[f], axis=1)), (key, f)
            n_rows += len(fa[f])
        if ra["status"] == 0 and rb["status"] == 0:
            assert not np.array_equal(ra["DT"], rb["DT"]), key
    assert n_rows > 1000, n_rows
    for s in range(4):
        T = np.eye(4)
        for i in range(1, LENGTHS[s]):
            r = own[(s, i)][0]
            assert r["status"] == 0, (s, i)
            T = T @ r["DT"].reshape(4, 4)
        T_true = np.linalg.inv(seqs[s][0][2]) @ seqs[s][-1][2]
        assert np.linalg.norm(T[:3, 3] - T_true[:3, 3]) < 0.05 * np.linalg.norm(T_true[:3, 3]), s


@pytest.mark.parametrize("in_flight", [0, 1, 2])
def test_change_mid_stream(built, in_flight):
    """Round robin (B = 4).  Before batch 3 is run, with `in_flight` batches not yet downloaded, sequence 1 gets NEW_CAM;
    before batch 7, NULL returns it to the context's camera.  Batches already run are unchanged; the pair of sequence 1
    in batch 3 (and in batch 7) is a first frame, and from there on it equals a fresh single context with the new camera
    started at that pair; the other sequences are untouched."""
    prm = PRM
    seqs = sequences()
    batches = interleavings(LENGTHS)["round_robin"]
    j1, j2 = 3, 7
    segs = [seg for seg in whole(seqs, CAMS) if seg[0] != 1]
    segs += [(1, 0, j1, CAMS[1]), (1, j1, j2, NEW_CAM), (1, j2, LENGTHS[1], CAM)]
    ref = alone(seqs, prm, segs)
    base = mixed(seqs, batches, prm, CAMS)
    got = {}
    views = in_flight == 0   # get_frame / get_matches refer to the batch most recently run
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=4, **prm) as fe:
        for s, c in enumerate(CAMS):
            fe.set_sequence_camera(s, c)
        pending = []
        for j, batch in enumerate(batches):
            if j == j1:
                assert len(pending) == in_flight
                fe.set_sequence_camera(1, NEW_CAM)
                assert fe.sequence_camera(1) == NEW_CAM
            if j == j2:
                assert len(pending) == in_flight
                fe.set_sequence_camera(1, None)
                assert fe.sequence_camera(1) == CAM
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq)
            pending.append(batch)
            while len(pending) > in_flight or (pending and j == len(batches) - 1):
                b = pending.pop(0)
                collect(fe, b, fe.batch_download_array(len(b)), got, views)
    if views:
        assert_same(ref, got)
    else:
        assert got.keys() == ref.keys()
        for key in ref:
            for f in ref[key][0].dtype.names:
                assert ref[key][0][f].tobytes() == got[key][0][f].tobytes(), (key, f)
    for key in got:   # batches run before the change, and every other sequence, as without it
        if key[0] != 1 or key[1] < j1:
            for f in base[key][0].dtype.names:
                assert base[key][0][f].tobytes() == got[key][0][f].tobytes(), (key, f)
    assert got[(1, j1)][0]["status"] == 2 and got[(1, j2)][0]["status"] == 2
    assert got[(1, j1 + 1)][0]["status"] == 0 and got[(1, j2 + 1)][0]["status"] == 0


@pytest.mark.parametrize("strategy", [0, 3])
def test_context_camera_set_explicitly_equals_default(built, strategy):
    """Setting every sequence to the context's own camera before the first batch (so every batch carries a camera table)
    gives what a context that never calls plf_set_sequence_camera gives."""
    prm = dict(PRM, matching_strategy=strategy)
    seqs = [list(synth.stream(CAM, n, world=synth.World(seed=60 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0,
                                                        half_height=3.5), seed=70 + s, step=0.15))
            for s, n in enumerate(LENGTHS)]
    batches = interleavings(LENGTHS)["random"]
    base = mixed(seqs, batches, prm, [None] * 4)
    assert sum(r["status"] == 0 for r, _, _ in base.values()) >= 0.75 * (sum(LENGTHS) - len(LENGTHS))
    assert_same(base, mixed(seqs, batches, prm, [CAM] * 4))


def test_errors_change_nothing(built):
    """Every refusal returns PLF_ERR_INVALID with a message naming the field, and changes neither the camera nor the
    sequence state: the next batch tracks on (no restart) and equals the uninterrupted run.  After plf_set_max_sequences
    the getter reports the context's camera."""
    seqs = sequences()
    batches = [[(0, 0), (1, 0), (0, 1), (1, 1)], [(1, 2), (0, 2), (1, 3), (0, 3)]]
    ref = alone(seqs, PRM, [(0, 0, 4, CAMS[0]), (1, 0, 4, CAMS[1])])
    bad = [(dict(CAMS[0], width=W + 16), r"width = 656, the context's is 640"),
           (dict(CAMS[0], height=H - 8), r"height = 352, the context's is 360")]
    for f in ("fx", "fy", "b"):
        for v in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
            bad.append((dict(CAMS[0], **{f: v}), rf"\b{f} = .*need a finite value > 0"))
    for f in ("cx", "cy"):
        for v in (float("nan"), float("inf"), -float("inf")):
            bad.append((dict(CAMS[0], **{f: v}), rf"\b{f} = .*need a finite value$"))
    got = {}
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=2, **PRM) as fe:
        fe.set_sequence_camera(0, CAMS[0])
        fe.set_sequence_camera(1, CAMS[1])
        for j, batch in enumerate(batches):
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            if j == 1:
                for s in (-1, 2):
                    for c in (CAMS[1], None):
                        with pytest.raises(plf.PlfError, match=rf"plf_set_sequence_camera failed \(-1\).*s = {s} outside \[0, 2\)"):
                            fe.set_sequence_camera(s, c)
                    with pytest.raises(plf.PlfError, match=rf"plf_get_sequence_camera failed \(-1\).*s = {s} outside \[0, 2\)"):
                        fe.sequence_camera(s)
                for c, msg in bad:
                    with pytest.raises(plf.PlfError, match=r"plf_set_sequence_camera failed \(-1\).*" + msg):
                        fe.set_sequence_camera(1, c)
                with pytest.raises(plf.PlfError, match=r"plf_get_sequence_camera failed \(-1\).*out is NULL"):
                    fe._check(fe.lib.plf_get_sequence_camera(fe._ctx, 0, None), "plf_get_sequence_camera")
                cam = plf.plf_camera(**CAMS[1])
                assert fe.lib.plf_set_sequence_camera(None, 0, C.byref(cam)) == -1
                assert fe.lib.plf_set_sequence_camera(None, 0, None) == -1
                assert fe.lib.plf_get_sequence_camera(None, 0, C.byref(cam)) == -1
                assert fe.sequence_camera(0) == CAMS[0] and fe.sequence_camera(1) == CAMS[1]
            fe.batch_run(4, seq=seq)
            collect(fe, batch, fe.batch_download_array(4), got)
    assert_same(ref, got)
    assert all(got[key][0]["status"] == 0 for key in batches[1])
    with plf.Frontend(camera=CAM, limits=limits(1), max_sequences=3) as fe:
        assert fe.sequence_camera(2) == CAM
        fe.set_sequence_camera(2, CAMS[2])
        assert fe.sequence_camera(2) == CAMS[2]
        fe.reset_sequence()   # keeps the cameras
        assert fe.sequence_camera(2) == CAMS[2]
        fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 4), "plf_set_max_sequences")
        assert all(fe.sequence_camera(s) == CAM for s in range(4))


def test_live_cameras_at_kitti_shape(built):
    """KITTI shape, 8 live cameras with 8 calibrations: one batch of B = 8 per step holds one pair of every camera, for 3
    steps.  Each camera equals a single context created with its calibration."""
    n, steps = 8, 3
    k = plf.KITTI_CAMERA
    cams = [dict(k, fx=k["fx"] * (1 + 0.01 * (c - 3.5)), fy=k["fy"] * (1 + 0.012 * (c - 3.5)), cx=k["cx"] + 1.5 * (c - 4),
                 cy=k["cy"] - 0.75 * (c - 4), b=k["b"] * (1 + 0.02 * (c - 3.5))) for c in range(n)]
    world = synth.World(seed=7)
    seqs = [list(synth.stream(cams[c], steps, world=world, seed=100 + c)) for c in range(n)]
    prm = dict(orb_nfeatures=1500, lsd_nfeatures=200)
    ref = {}
    for c in range(n):
        with plf.Frontend(camera=cams[c], limits=limits(steps), **prm) as fe:
            fe.batch_upload(np.stack([f[0] for f in seqs[c]]), np.stack([f[1] for f in seqs[c]]))
            fe.batch_run(steps)
            collect(fe, [(c, i) for i in range(steps)], fe.batch_download_array(steps), ref)
    got = mixed(seqs, [[(c, i) for c in range(n)] for i in range(steps)], prm, cams, nseq=n, ctx_cam=k)
    assert_same(ref, got)
    assert sum(got[(c, i)][0]["status"] == 0 for c in range(n) for i in range(1, steps)) >= 0.75 * n * (steps - 1)
