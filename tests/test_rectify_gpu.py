"""GPU tests of per-sequence rectification in the batched pipeline (plf_set_sequence_rectification).

Two rectified streams A and B are rendered with the rectified camera of EuRoC's calibration (scaled to 632 x 360: the
16-byte row pitch is 640, so dense uploads go through the landing buffer) and distorted back into raw pairs.  In one
context, sequences 0 and 1 are rectified on the device and fed A's and B's raw pairs; their twins 2 and 3 are not and
are fed the same raw pairs through cv2.remap on the host.  Every pair of a rectified sequence must equal its twin's bit
for bit: plf_frame_result, plf_get_frame and plf_get_matches."""
import ctypes as C

import numpy as np
import pytest
import torch

import plslam_b200 as plf
from oracle import rectify, synth

cv2 = pytest.importorskip("cv2")

pytestmark = pytest.mark.gpu

W, H = 632, 360
PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
N = 8   # pairs per stream
TWIN = {0: 2, 1: 3}

_DATA = {}


def data():
    """(maps left, maps right, camera, raw[stream][i] = (L, R), host-rectified[stream][i] = (L, R))."""
    if not _DATA:
        left, right, cam = rectify.stereo_maps(size=(W, H))
        raw, rect = [], []
        for s in range(2):
            world = synth.World(seed=70 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
            frames = list(synth.stream(cam, N, world=world, seed=80 + s, step=0.12))
            raw.append([rectify.distort(l, r) for l, r, _ in frames])
            rect.append([(cv2.remap(l, *left, cv2.INTER_LINEAR), cv2.remap(r, *right, cv2.INTER_LINEAR)) for l, r in raw[s]])
        _DATA.update(left=left, right=right, cam=cam, raw=raw, rect=rect)
    return _DATA


def frontend(B, **kw):
    lim = plf.default_limits()
    lim.max_batch = B
    return plf.Frontend(camera=data()["cam"], limits=lim, max_sequences=4, **dict(PRM, **kw))


def pair(s, i):
    """The images sequence s is fed at step i: raw for the rectified sequences 0, 1, host-rectified for 2, 3."""
    d = data()
    return d["raw"][s][i] if s < 2 else d["rect"][s - 2][i]


def upload(fe, L, R, strided):
    if not strided:
        fe.batch_upload(L, R)
        return
    B, stride = len(L), W + 24   # rows of W bytes inside wider host rows
    Ls, Rs = (np.zeros((B, H, stride), np.uint8) for _ in range(2))
    Ls[..., :W], Rs[..., :W] = L, R
    st = fe.lib.plf_batch_upload(fe._ctx, B, Ls.ctypes.data_as(C.POINTER(C.c_uint8)), Rs.ctypes.data_as(C.POINTER(C.c_uint8)),
                                 stride)
    fe._check(st, "plf_batch_upload")


def round_robin(seed=0):
    """One pair of every sequence per batch, in a shuffled order (rectified pairs adjacent or apart)."""
    rng = np.random.default_rng(seed)
    return [[(int(s), i) for s in rng.permutation(4)] for i in range(N)]


def merged(seed=1, B=6):
    """A seeded merge of the four sequences in batches of B (several pairs of a sequence per batch)."""
    rng = np.random.default_rng(seed)
    pos, order = [0] * 4, []
    while len(order) < 4 * N:
        s = int(rng.choice([q for q in range(4) if pos[q] < N]))
        order.append((s, pos[s]))
        pos[s] += 1
    return [order[j:j + B] for j in range(0, len(order), B)]


def run(fe, batches, strided=False, in_flight=1, before=None, restart=None, feed=pair):
    """The batches through fe with up to in_flight batches in flight.  before(j, fe) runs before batch j is uploaded;
    restart: {(s, i)} pairs run with restart[k] = 1; feed(s, i): the images of pair (s, i).  Returns {(s, i): (result
    row, frame, matches)}, frame and matches for the last batch only."""
    out, pending = {}, []

    def drain():
        b = pending.pop(0)
        res = fe.batch_download_array(len(b))
        for k, key in enumerate(b):
            out[key] = (res[k],)

    for j, batch in enumerate(batches):
        if before:
            before(j, fe)
        while len(pending) >= in_flight:
            drain()
        L = np.stack([feed(s, i)[0] for s, i in batch])
        R = np.stack([feed(s, i)[1] for s, i in batch])
        upload(fe, L, R, strided)
        rs = None if restart is None else np.array([key in restart for key in batch])
        fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32), restart=rs)
        pending.append(batch)
    last = pending[-1]
    while pending:
        drain()
    for k, key in enumerate(last):
        out[key] = out[key] + (fe.get_frame(k), fe.get_matches(k))
    return out


def run_sync(fe, batches, strided=False, before=None, restart=None, feed=pair):
    """run() with frames and matches of every pair (one batch at a time)."""
    out = {}
    for j, batch in enumerate(batches):
        if before:
            before(j, fe)
        out.update(run(fe, [batch], strided, restart=restart, feed=feed))
    return out


def set_maps(fe, s, maps=None):
    d = data()
    left, right = maps or (d["left"], d["right"])
    fe.set_sequence_rectification(s, left=left, right=right)


def assert_twins(got):
    """Each pair of sequences 0 and 1 equals its twin's (2 and 3) field for field, bit for bit."""
    n = 0
    for (s, i) in sorted(got):
        if s not in TWIN:
            continue
        a, b = got[(s, i)], got[(TWIN[s], i)]   # frames and matches where both were read (run(): the last batch)
        for f in a[0].dtype.names:
            assert a[0][f].tobytes() == b[0][f].tobytes(), (s, i, f)
        for da, db in zip(a[1:], b[1:]):
            assert da.keys() == db.keys()
            for k in da:
                assert da[k].shape == db[k].shape and da[k].tobytes() == db[k].tobytes(), (s, i, k)
        n += 1
    return n


def assert_tracks(got):
    rows = [v[0] for v in got.values()]
    assert sum(int(r["status"]) == 0 for r in rows) >= len(rows) // 2, [int(r["status"]) for r in rows]
    assert sum(int(r["n_matched_pt"]) + int(r["n_matched_ls"]) for r in rows) > 50 * len(rows)


def device_pairs(fe, B):
    """The batch's images in the slot plf_batch_device_images returns: uint8 [B, 2, H, W]."""
    pitch = (W + 15) // 16 * 16

    class Dev:
        __cuda_array_interface__ = {"shape": (2 * B, H, pitch), "typestr": "|u1", "data": (fe.device_images, False),
                                    "version": 3, "strides": None}

    torch.cuda.synchronize()
    a = torch.as_tensor(Dev(), device="cuda").cpu().numpy()
    return a[..., :W].reshape(B, 2, H, W)


# ---- 1. the rectified images ----

@pytest.mark.parametrize("strided", [False, True], ids=["dense", "strided"])
def test_device_images_are_cv_remap(built, strided):
    """Pairs of rectified sequences are cv2.remap of their raw inputs byte for byte after a run; the others are what
    was uploaded."""
    d = data()
    batch = [(2, 0), (0, 0), (0, 1), (3, 2), (1, 3), (2, 1)]   # rectified pairs at 1, 2 and 4
    with frontend(6) as fe:
        set_maps(fe, 0)
        set_maps(fe, 1, (d["right"], d["left"]))   # sequence 1 reads its own maps: the two swapped
        L = np.stack([d["raw"][s % 2][i][0] for s, i in batch])
        R = np.stack([d["raw"][s % 2][i][1] for s, i in batch])
        upload(fe, L, R, strided)
        fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
        fe.batch_download_array(len(batch))
        got = device_pairs(fe, len(batch))
    for k, (s, _) in enumerate(batch):
        if s == 0:
            want = (cv2.remap(L[k], *d["left"], cv2.INTER_LINEAR), cv2.remap(R[k], *d["right"], cv2.INTER_LINEAR))
        elif s == 1:
            want = (cv2.remap(L[k], *d["right"], cv2.INTER_LINEAR), cv2.remap(R[k], *d["left"], cv2.INTER_LINEAR))
        else:
            want = (L[k], R[k])
        for side in range(2):
            assert np.array_equal(got[k, side], want[side]), (k, s, side)


# ---- 2. raw pairs through a rectified sequence == host-rectified pairs through an unrectified one ----

@pytest.mark.parametrize("strided", [False, True], ids=["dense", "strided"])
@pytest.mark.parametrize("in_flight", [1, 3])
def test_raw_equals_host_rectified(built, strided, in_flight):
    for batches, B in ((round_robin(), 4), (merged(), 6)):
        with frontend(B) as fe:
            set_maps(fe, 0)
            set_maps(fe, 1)
            got = run_sync(fe, batches, strided=strided) if in_flight == 1 else run(fe, batches, strided, in_flight)
        assert assert_twins(got) == 2 * N
        assert_tracks(got)
        for s in range(4):
            assert int(got[(s, 0)][0]["status"]) == 2


def test_raw_equals_host_rectified_adaptive_fast(built):
    """With adaptive FAST thresholds each sequence's threshold follows its own frames; the twins' thresholds and
    results stay equal."""
    with frontend(4, adaptive_fast={}) as fe:
        set_maps(fe, 0)
        set_maps(fe, 1)
        th = {}

        def before(j, f):
            th[j] = [f.sequence_fast_th(s) for s in range(4)]

        got = run(fe, round_robin(2), strided=False, in_flight=3, before=before)
    assert assert_twins(got) == 2 * N
    assert_tracks(got)
    for v in th.values():
        assert v[0] == v[2] and v[1] == v[3], th


# ---- 3. set, clear and restart semantics; refusals; plf_set_max_sequences ----

@pytest.mark.parametrize("in_flight", [1, 3])
def test_change_and_clear_mid_stream(built, in_flight):
    """Before batch 3, sequence 0 gets other maps (left and right swapped); before batch 6 its maps are cleared and it
    is fed its twin's host-rectified pairs.  Each call restarts sequence 0; its twin restarts there too (restart flags)
    and is fed the host remap of the maps in force.  With batches in flight, those already run keep their maps."""
    d = data()
    swapped = (d["right"], d["left"])
    j_swap, j_clear = 3, 6

    def feed(s, i):
        if s != 0 and s != 2:
            return pair(s, i)
        raw = d["raw"][0][i]
        if j_swap <= i < j_clear:   # the swapped maps, host-remapped for the twin
            host = (cv2.remap(raw[0], *swapped[0], cv2.INTER_LINEAR), cv2.remap(raw[1], *swapped[1], cv2.INTER_LINEAR))
        else:
            host = d["rect"][0][i]
        return raw if (s == 0 and i < j_clear) else host

    def before(j, fe):
        if j == j_swap:
            set_maps(fe, 0, swapped)
        if j == j_clear:
            fe.set_sequence_rectification(0)

    with frontend(4) as fe:
        set_maps(fe, 0)
        set_maps(fe, 1)
        restart = {(2, j_swap), (2, j_clear)}
        batches = round_robin(3)
        got = (run_sync(fe, batches, before=before, restart=restart, feed=feed) if in_flight == 1
               else run(fe, batches, False, in_flight, before=before, restart=restart, feed=feed))
    assert assert_twins(got) == 2 * N
    for i in (0, j_swap, j_clear):
        assert int(got[(0, i)][0]["status"]) == 2, i
    assert int(got[(0, j_swap + 1)][0]["status"]) != 2


def test_refusals_change_nothing(built):
    d = data()
    (m1, m2), (r1, r2) = d["left"], d["right"]
    p16 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int16))
    pu16 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint16))
    with frontend(4) as fe:
        set_maps(fe, 0)
        set_maps(fe, 1)
        batches = round_robin(4)
        got = run_sync(fe, batches[:2])

        lib, ctx = fe.lib, fe._ctx
        for s in (-1, 4):
            assert lib.plf_set_sequence_rectification(ctx, s, p16(m1), pu16(m2), p16(r1), pu16(r2)) == -1
            assert "outside" in lib.plf_last_error(ctx).decode()
        for drop in range(4):
            args = [p16(m1), pu16(m2), p16(r1), pu16(r2)]
            args[drop] = None
            assert lib.plf_set_sequence_rectification(ctx, 0, *args) == -1
            assert "all four or none" in lib.plf_last_error(ctx).decode()
        assert lib.plf_set_sequence_rectification(None, 0, None, None, None, None) == -1
        with pytest.raises(plf.PlfError):
            fe.set_sequence_rectification(0, left=(m1, m2))
        with pytest.raises(plf.PlfError):
            fe.set_sequence_rectification(0, left=(m1.astype(np.int32), m2), right=(r1, r2))
        with pytest.raises(plf.PlfError):
            fe.set_sequence_rectification(0, left=(m1[:-1], m2[:-1]), right=(r1, r2))
        # nothing changed: no restart, the maps still apply
        got.update(run_sync(fe, batches[2:]))
    assert assert_twins(got) == 2 * N
    assert int(got[(0, 2)][0]["status"]) == 0 and int(got[(1, 2)][0]["status"]) == 0


def test_max_sequences_drops_and_reset_keeps(built):
    d = data()
    raw = d["raw"][0][0]
    L, R = raw[0][None], raw[1][None]
    want = (cv2.remap(raw[0], *d["left"], cv2.INTER_LINEAR), cv2.remap(raw[1], *d["right"], cv2.INTER_LINEAR))

    def one(fe):
        fe.batch_upload(L, R)
        fe.batch_run(1, seq=np.array([0], np.int32))
        fe.batch_download_array(1)
        return device_pairs(fe, 1)[0]

    with frontend(1) as fe:
        set_maps(fe, 0)   # before the pipeline exists
        fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 4), "plf_set_max_sequences")
        got = one(fe)
        assert np.array_equal(got[0], raw[0]) and np.array_equal(got[1], raw[1])   # dropped
    with frontend(1) as fe:
        set_maps(fe, 0)
        one(fe)
        fe.reset_sequence()
        got = one(fe)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])   # kept


# ---- 4. without maps nothing changes ----

def test_without_maps_nothing_changes(built):
    """A context whose maps were set and cleared, and a context whose rectified sequence is absent from every batch,
    enqueue the same launches and give the same bytes as a context that never saw the call."""
    batches = [[(s, i) for s in (3, 2, 1)] for i in range(N)]   # sequence 0 never runs

    def go(setup):
        with frontend(3) as fe:
            setup(fe)
            n0 = fe.launches
            got = run_sync(fe, batches)
            return got, fe.launches - n0

    ref, n_ref = go(lambda fe: None)
    for setup in (lambda fe: (set_maps(fe, 1), fe.set_sequence_rectification(1)), lambda fe: set_maps(fe, 0)):
        got, n = go(setup)
        assert n == n_ref
        assert got.keys() == ref.keys()
        for key in ref:
            for a, b in zip(got[key][1:], ref[key][1:]):
                for k in a:
                    assert a[k].tobytes() == b[k].tobytes(), (key, k)
            assert got[key][0].tobytes() == ref[key][0].tobytes(), key
