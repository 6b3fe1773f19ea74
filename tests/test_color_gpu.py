"""GPU tests of colour input to the batched pipeline (plf_batch_upload_color).

The device's grey images must be cv2.cvtColor of the uploaded BGR / BGRA pairs byte for byte, and cv2.cvtColor of
cv2.remap of them for rectified sequences.  Everything after the conversion must be the grey pipeline's: a context fed
colour pairs must give, bit for bit, what a twin context fed cv2.cvtColor's grey pairs in the same batches gives
(plf_frame_result, plf_get_frame and plf_get_matches)."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

import plslam_b200 as plf
from test_rectify_gpu import H, N, W, data, frontend, merged, round_robin
from test_shim import DEMO, write_frames

cv2 = pytest.importorskip("cv2")

pytestmark = pytest.mark.gpu


def gray(img):
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY if img.shape[-1] == 3 else cv2.COLOR_BGRA2GRAY)


def remap(img, maps):
    return cv2.remap(img, *maps, cv2.INTER_LINEAR)


def colourise(g, seed, ch=3):
    """A colour image whose channels differ around the grey image g (so every channel weight matters), alpha random."""
    rng = np.random.default_rng(seed)
    out = np.clip(g[..., None].astype(np.int16) + rng.integers(-24, 25, g.shape + (ch,)), 0, 255).astype(np.uint8)
    if ch == 4:
        out[..., 3] = rng.integers(0, 256, g.shape)
    return out


def smooth_colour(rng, B, h, w, ch):
    """Ramps with a little per-channel noise: few features, so no capacity is reached at any shape."""
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * (1 + c) + y * (2 + c) + 40 * c) % 256 for c in range(ch)], axis=-1)
    return np.clip(base[None] + rng.integers(-3, 4, (B, h, w, ch)), 0, 255).astype(np.uint8)


def upload_color(fe, L, R, strided):
    """L, R: uint8 [B, h, w, ch].  strided: rows of ch w bytes inside wider host rows, the stride a multiple of neither
    16 nor ch."""
    if not strided:
        fe.batch_upload(L, R)
        return
    B, h, w, ch = L.shape
    stride = ch * w + 13
    if stride % 16 == 0:
        stride += 1
    assert stride % 16 and stride % ch
    Ls, Rs = (np.zeros((B, h, stride), np.uint8) for _ in range(2))
    Ls[..., :ch * w], Rs[..., :ch * w] = L.reshape(B, h, -1), R.reshape(B, h, -1)
    fe._check(fe.lib.plf_batch_upload_color(fe._ctx, B, Ls.ctypes.data_as(C.POINTER(C.c_uint8)),
                                            Rs.ctypes.data_as(C.POINTER(C.c_uint8)), stride, ch), "plf_batch_upload_color")


def device_pairs(fe, B, h, w):
    """The batch's grey images in the slot plf_batch_device_images returns: uint8 [B, 2, h, w]."""
    pitch = (w + 15) // 16 * 16

    class Dev:
        __cuda_array_interface__ = {"shape": (2 * B, h, pitch), "typestr": "|u1", "data": (fe.device_images, False),
                                    "version": 3, "strides": None}

    torch.cuda.synchronize()
    return torch.as_tensor(Dev(), device="cuda").cpu().numpy()[..., :w].reshape(B, 2, h, w)


def download_allowing_capacity(fe, B):
    try:
        fe.batch_download_array(B)
    except plf.PlfError as e:   # the images are checked, not the features
        assert "overflowed" in str(e), e


# ---- 1. the grey images ----

SHAPES = {"kitti": (plf.KITTI_CAMERA["width"], plf.KITTI_CAMERA["height"]),
          "euroc": (plf.EUROC_CAMERA["width"], plf.EUROC_CAMERA["height"]), "odd": (333, 201)}


@pytest.mark.parametrize("strided", [False, True], ids=["dense", "strided"])
@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_device_images_are_cvtcolor(built, shape, ch, strided):
    w, h = SHAPES[shape]
    cam = dict(plf.KITTI_CAMERA, width=w, height=h, cx=w / 2, cy=h / 2)
    B = 3
    rng = np.random.default_rng(10 * list(SHAPES).index(shape) + ch)
    L, R = smooth_colour(rng, B, h, w, ch), smooth_colour(rng, B, h, w, ch)
    lim = plf.default_limits()
    lim.max_batch = B
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=300, lsd_nfeatures=50) as fe:
        upload_color(fe, L, R, strided)
        fe.batch_run(B)
        download_allowing_capacity(fe, B)
        got = device_pairs(fe, B, h, w)
    for k in range(B):
        assert np.array_equal(got[k, 0], gray(L[k])), k
        assert np.array_equal(got[k, 1], gray(R[k])), k


@pytest.mark.parametrize("strided", [False, True], ids=["dense", "strided"])
@pytest.mark.parametrize("ch", [3, 4])
def test_rectified_colour_is_cvtcolor_of_remap(built, ch, strided):
    """A batch mixing rectified sequences (0: its maps, 1: the two swapped) and unrectified ones (2, 3)."""
    d = data()
    maps = {0: (d["left"], d["right"]), 1: (d["right"], d["left"])}
    batch = [(2, 0), (0, 0), (0, 1), (3, 2), (1, 3), (2, 1)]
    L = np.stack([colourise(d["raw"][s % 2][i][0], 10 * s + i, ch) for s, i in batch])
    R = np.stack([colourise(d["raw"][s % 2][i][1], 10 * s + i + 5, ch) for s, i in batch])
    with frontend(6) as fe:
        for s, (ml, mr) in maps.items():
            fe.set_sequence_rectification(s, left=ml, right=mr)
        upload_color(fe, L, R, strided)
        fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
        fe.batch_download_array(len(batch))
        got = device_pairs(fe, len(batch), H, W)
    for k, (s, _) in enumerate(batch):
        want = ((gray(remap(L[k], maps[s][0])), gray(remap(R[k], maps[s][1]))) if s in maps else (gray(L[k]), gray(R[k])))
        for side in range(2):
            assert np.array_equal(got[k, side], want[side]), (k, s, side)


# ---- 2. colour pairs == cv2.cvtColor's grey pairs, through the whole pipeline ----

def colour_pair(s, i, ch=3, raw=False):
    """Sequence s's colour pair at step i: a rectified pair of stream s % 2 colourised, or with raw the raw (distorted)
    pair it was rectified from."""
    d = data()
    L, R = d["raw" if raw else "rect"][s % 2][i]
    return colourise(L, 100 * s + 2 * i, ch), colourise(R, 100 * s + 2 * i + 1, ch)


def run(fe, batches, feed, in_flight=1, strided=False):
    """The batches through fe with up to in_flight batches in flight; feed(j, s, i) -> (L, R) of pair (s, i) in batch j,
    grey [h, w] or colour [h, w, ch] (one kind per batch).  Returns {(s, i): (result row, frame, matches)}, frame and
    matches for the last batch only."""
    out, pending = {}, []

    def drain():
        b = pending.pop(0)
        res = fe.batch_download_array(len(b))
        for k, key in enumerate(b):
            out[key] = (res[k],)

    for j, batch in enumerate(batches):
        while len(pending) >= in_flight:
            drain()
        pairs = [feed(j, s, i) for s, i in batch]
        L, R = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
        if L.ndim == 4:
            upload_color(fe, L, R, strided)
        else:
            fe.batch_upload(L, R)
        fe.batch_run(len(batch), seq=np.array([s for s, _ in batch], np.int32))
        pending.append(batch)
    last = pending[-1]
    while pending:
        drain()
    for k, key in enumerate(last):
        out[key] = out[key] + (fe.get_frame(k), fe.get_matches(k))
    return out


def assert_identical(got, ref):
    assert got.keys() == ref.keys()
    for key in ref:
        assert got[key][0].tobytes() == ref[key][0].tobytes(), key
        for a, b in zip(got[key][1:], ref[key][1:]):
            assert a.keys() == b.keys()
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), (key, k)
    rows = [v[0] for v in ref.values()]
    assert sum(int(r["status"]) == 0 for r in rows) >= len(rows) // 2, [int(r["status"]) for r in rows]
    assert sum(int(r["n_matched_pt"]) + int(r["n_matched_ls"]) for r in rows) > 50 * len(rows)


def twins(batches, colour_feed, grey_feed, B, in_flight, strided=False, setup=None, **kw):
    out = []
    for feed in (colour_feed, grey_feed):
        with frontend(B, **kw) as fe:
            if setup:
                setup(fe, feed is colour_feed)
            out.append(run(fe, batches, feed, in_flight, strided))
    return out


@pytest.mark.parametrize("in_flight", [1, 3])
@pytest.mark.parametrize("ch,strided", [(3, False), (4, True)], ids=["bgr-dense", "bgra-strided"])
def test_colour_equals_cvtcolor_grey(built, ch, strided, in_flight):
    for batches, B in ((round_robin(), 4), (merged(), 6)):
        got, ref = twins(batches, lambda j, s, i: colour_pair(s, i, ch),
                         lambda j, s, i: tuple(gray(a) for a in colour_pair(s, i, ch)), B, in_flight, strided)
        assert_identical(got, ref)


def test_grey_and_colour_uploads_alternate(built):
    """Even batches are uploaded in colour, odd ones in grey (BGRA and BGR by turns), three in flight."""
    def feed(j, s, i):
        ch = 4 if j % 4 == 0 else 3
        p = colour_pair(s, i, ch)
        return p if j % 2 == 0 else tuple(gray(a) for a in p)

    got, ref = twins(merged(seed=5), feed, lambda j, s, i: tuple(gray(a) for a in colour_pair(s, i, 4 if j % 4 == 0 else 3)),
                     6, 3)
    assert_identical(got, ref)


def test_rectified_colour_round_robin_adaptive_fast_motion_model(built):
    """Sequence 0 is rectified on the device from raw colour pairs; its twin gets cv2.cvtColor(cv2.remap(raw colour)).
    Round-robin, three in flight, adaptive FAST thresholds and the motion model on."""
    d = data()

    def setup(fe, colour):
        if colour:
            fe.set_sequence_rectification(0, left=d["left"], right=d["right"])

    def grey_feed(j, s, i):
        L, R = colour_pair(s, i, raw=s == 0)
        if s == 0:
            L, R = remap(L, d["left"]), remap(R, d["right"])
        return gray(L), gray(R)

    got, ref = twins(round_robin(7), lambda j, s, i: colour_pair(s, i, raw=s == 0), grey_feed, 4, 3, setup=setup, adaptive_fast={},
                     motion_model=True)
    assert_identical(got, ref)


# ---- 3. refusals, memory, launches ----

def test_refused_upload_changes_nothing(built):
    batch = round_robin()[0]
    pairs = [colour_pair(s, i) for s, i in batch]
    L, R = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    p8 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint8))
    seq = np.array([s for s, _ in batch], np.int32)
    out = []
    for refuse in (False, True):
        with frontend(4) as fe:
            fe.batch_upload(L, R)
            if refuse:
                lib, ctx, w = fe.lib, fe._ctx, W
                for args, word in (((4, p8(L), p8(R), 3 * w, 2), "channels = 2"), ((4, p8(L), p8(R), w, 1), "channels = 1"),
                                   ((4, p8(L), p8(R), 5 * w, 5), "channels = 5"), ((0, p8(L), p8(R), 3 * w, 3), "B = 0"),
                                   ((5, p8(L), p8(R), 3 * w, 3), "B = 5"), ((4, None, p8(R), 3 * w, 3), "left and right"),
                                   ((4, p8(L), None, 3 * w, 3), "left and right"), ((4, p8(L), p8(R), 3 * w - 1, 3), "stride"),
                                   ((4, p8(L), p8(R), 4 * w - 1, 4), "stride")):
                    assert lib.plf_batch_upload_color(ctx, *args) == -1, word
                    assert word in lib.plf_last_error(ctx).decode(), (word, lib.plf_last_error(ctx))
                with pytest.raises(plf.PlfError):
                    fe.batch_upload(L[..., :2], R[..., :2])
            fe.batch_run(4, seq=seq)
            res = fe.batch_download_array(4)
            out.append((res, device_pairs(fe, 4, H, W)))
    assert out[0][0].tobytes() == out[1][0].tobytes()
    assert np.array_equal(out[0][1], out[1][1])
    for k in range(4):
        assert np.array_equal(out[1][1][k, 0], gray(L[k])) and np.array_equal(out[1][1][k, 1], gray(R[k]))


def test_staging_and_launches_only_with_colour(built):
    """Grey batches allocate no landing buffer and enqueue the same launches before and after colour batches; the first
    colour upload allocates 2 max_batch h w ch bytes, a later one of as many channels nothing more, and a colour batch
    enqueues one launch more than a grey one (k_color)."""
    B = 64
    batch = [(s % 4, s // 4) for s in range(B)]
    pairs = [colour_pair(s % 4, i % N) for s, i in batch]
    L, R = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    Lg, Rg = np.stack([gray(a) for a in L]), np.stack([gray(a) for a in R])
    landing = 2 * B * H * W * 3

    def one(fe, left, right):
        n0 = fe.launches
        fe.batch_upload(left, right)
        fe.batch_run(B, seq=np.zeros(B, np.int32))
        fe.batch_download_array(B)
        torch.cuda.synchronize()
        return fe.launches - n0, torch.cuda.mem_get_info()[0]

    with frontend(B) as fe:
        one(fe, Lg, Rg)   # the first run also builds the pipeline
        n_grey, _ = one(fe, Lg, Rg)
        n_grey2, free_grey = one(fe, Lg, Rg)
        n_col, free_col = one(fe, L, R)
        n_col2, free_col2 = one(fe, L, R)
        n_grey3, _ = one(fe, Lg, Rg)
    assert n_grey == n_grey2 == n_grey3 and n_col == n_col2 == n_grey + 1
    assert free_grey - free_col >= landing, (free_grey, free_col, landing)
    assert abs(free_col - free_col2) < landing // 4, (free_col, free_col2)


# ---- 4. the shim and vo_demo ----

@pytest.mark.parametrize("ch", [3, 4])
def test_vo_demo_colour_prints_what_grey_prints(built, tmp_path, ch):
    d = data()
    frames = [colour_pair(2, i, ch) for i in range(N)]
    pc, pg = tmp_path / "colour.bin", tmp_path / "grey.bin"
    write_frames(pc, d["cam"], frames)
    write_frames(pg, d["cam"], [tuple(gray(a) for a in f) for f in frames])
    rc = subprocess.run([str(DEMO), str(pc), "700", "150", "--color", str(ch)], capture_output=True, text=True)
    rg = subprocess.run([str(DEMO), str(pg), "700", "150"], capture_output=True, text=True)
    assert rc.returncode == 0 and rg.returncode == 0, (rc.stderr, rg.stderr)
    assert rc.stdout == rg.stdout
    lines = rg.stdout.strip().splitlines()
    assert len(lines) == N and sum(ln.split()[1] == "0" for ln in lines) >= N // 2


def test_vo_demo_refuses_other_channel_counts(built, tmp_path):
    d = data()
    frames = [tuple(np.zeros((H, W, 2), np.uint8) for _ in range(2))]
    p = tmp_path / "two.bin"
    write_frames(p, d["cam"], frames)
    r = subprocess.run([str(DEMO), str(p), "--color", "2"], capture_output=True, text=True)
    assert r.returncode == 2 and "grey, BGR or BGRA" in r.stderr, (r.returncode, r.stderr)
