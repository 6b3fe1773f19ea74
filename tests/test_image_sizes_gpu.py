"""GPU tests of several image sizes in one batched context (plf_set_image_sizes, plf_batch_upload_sized).

The oracle is the library itself: every pair of a batch of a declared size must give, bit for bit, what its sequence run
alone gives on a context created at that size with its camera - every plf_frame_result field (DT included), and with one
batch in flight get_frame(k) and get_matches(k).  The sizes differ from the context's 640 x 360 in everything the tile
kernels treat differently (tests/test_frontend_geometry.py): one larger in each dimension, one smaller, one whose width
rounds to another 16-byte pitch and other FAST, blur and LSD tile counts, and one of EuRoC's aspect ratio.  A short
stream per size is also checked against the oracle pipeline."""
import numpy as np
import pytest

import plslam_b200 as plf
from adversarial_images import dot_lattice
from oracle import clib, rectify, synth
from oracle import frontend as ofe
from test_color_gpu import colourise
from test_pipeline_gpu import POSE_REL_TOL, check_frame, rel

pytestmark = pytest.mark.gpu

CTX = (640, 360)
SIZES = [(704, 392), (512, 288), (577, 341), (480, 306)]   # larger, smaller, other pitch and tiles, EuRoC's aspect
PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
N = 6   # pairs per sequence


def camera(w, h, k=0):
    f = 0.78 * w + 3 * k
    return dict(width=w, height=h, fx=f, fy=f + 1.5, cx=w / 2 + 1.25 * k, cy=h / 2 - 0.75 * k, b=0.5 + 0.02 * k)


# sequence s: its camera (sequence 0 at the context's size, 5 beside sequence 1 at SIZES[0])
CAMS = [camera(*CTX)] + [camera(w, h, 1 + i) for i, (w, h) in enumerate(SIZES)] + [camera(*SIZES[0], 7)]
_DATA = {}


def frames(s):
    """Sequence s: N grey pairs rendered with its camera."""
    if s not in _DATA:
        world = synth.World(seed=90 + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
        _DATA[s] = [(l, r) for l, r, _ in synth.stream(CAMS[s], N, world=world, seed=100 + s, step=0.15)]
    return _DATA[s]


def size_of(s):
    return CAMS[s]["width"], CAMS[s]["height"]


def limits(B):
    lim = plf.default_limits()
    lim.max_batch = B
    return lim


def schedule(seqs, per=2):
    """Batches of one size each, the sizes alternating: each batch takes up to `per` next pairs of every sequence of its
    size, so the sequences of the other sizes sit out."""
    pos = {s: 0 for s in seqs}
    sizes = list(dict.fromkeys(size_of(s) for s in seqs))
    out = []
    while any(pos[s] < N for s in seqs):
        for sz in sizes:
            batch = []
            for s in seqs:
                if size_of(s) == sz:
                    take = min(per, N - pos[s])
                    batch += [(s, pos[s] + i) for i in range(take)]
                    pos[s] += take
            if batch:
                out.append(batch)
    return out


def feed_grey(s, i):
    return frames(s)[i]


def feed_bgr(s, i):
    l, r = frames(s)[i]
    return colourise(l, 1000 * s + 2 * i), colourise(r, 1000 * s + 2 * i + 1)


def run(fe, batches, feed, in_flight=1, restart=(), alone=False):
    """The batches through fe; {(s, i): (result, frame, matches)} (views only with one batch in flight).  alone: fe
    tracks one sequence, as its sequence 0."""
    out, pending = {}, []

    def drain():
        b = pending.pop(0)
        res = fe.batch_download_array(len(b))
        for k, key in enumerate(b):
            out[key] = (res[k],) + ((fe.get_frame(k), fe.get_matches(k)) if in_flight == 1 else ())

    for batch in batches:
        L = np.stack([feed(s, i)[0] for s, i in batch])
        R = np.stack([feed(s, i)[1] for s, i in batch])
        fe.batch_upload(L, R)
        fe.batch_run(len(batch), seq=np.array([0 if alone else s for s, _ in batch], np.int32),
                     restart=np.array([key in restart for key in batch], np.uint8))
        pending.append(batch)
        if len(pending) == in_flight:
            drain()
    while pending:
        drain()
    return out


def packed(seqs, batches, feed=feed_grey, in_flight=1, restart=(), setup=None, **prm):
    B = max(map(len, batches))
    with plf.Frontend(camera=CAMS[0], limits=limits(B), max_sequences=len(CAMS), image_sizes=SIZES, **dict(PRM, **prm)) as fe:
        for s in seqs:
            if s:
                fe.set_sequence_camera(s, CAMS[s])
            if setup:
                setup(fe, s)
        return run(fe, batches, feed, in_flight, restart)


def alone(seqs, feed=feed_grey, restart=(), setup=None, per=1, **prm):
    """Each sequence by itself on a context created at its size with its camera, `per` pairs per batch."""
    out = {}
    for s in seqs:
        with plf.Frontend(camera=CAMS[s], limits=limits(per), **dict(PRM, **prm)) as fe:
            if setup:
                setup(fe, s, alone=True)
            batches = [[(s, i) for i in range(a, min(a + per, N))] for a in range(0, N, per)]
            got = run(fe, batches, feed, 1, restart, alone=True)
            out.update(got)
    return out


def assert_same(ref, got, views=True):
    assert ref.keys() == got.keys()
    for key in ref:
        for f in ref[key][0].dtype.names:
            assert ref[key][0][f].tobytes() == got[key][0][f].tobytes(), (key, f)
        if views and len(got[key]) > 1:
            for a, b in zip(ref[key][1:], got[key][1:]):
                for k in a:
                    assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (key, k)


SEQS = list(range(len(CAMS)))


@pytest.mark.parametrize("in_flight", [1, 3])
@pytest.mark.parametrize("strategy", [0, 3])
def test_packed_sizes_equal_each_sequence_alone(built, in_flight, strategy):
    """Batches of alternating sizes, two pairs of each sequence of the batch's size; sequences sit out the batches of the
    other sizes, and sequence 2 restarts at pair 3."""
    restart = {(2, 3)}
    ref = alone(SEQS, restart=restart, per=2, matching_strategy=strategy)
    tracked = sum(v[0]["status"] == 0 for v in ref.values())
    assert tracked >= 0.7 * len(ref), tracked
    got = packed(SEQS, schedule(SEQS), in_flight=in_flight, restart=restart, matching_strategy=strategy)
    assert_same(ref, got, views=in_flight == 1)


def test_features_on_at_other_sizes(built):
    """Adaptive FAST, the motion model and matching_strategy 3, one pair per sequence per batch; sequence 1 (larger) is
    masked, sequence 3 (other pitch) rectified and fed BGR, sequence 4 (EuRoC's aspect) masked, rectified and fed BGR:
    masks with adaptive FAST, with the motion model and with rectified colour."""
    afast = dict(plf.ADAPTIVE_FAST_DEFAULTS)
    prm = dict(matching_strategy=3, adaptive_fast=afast, motion_model=True)
    maps = {s: rectify.stereo_maps(size=size_of(s))[:2] for s in (3, 4)}

    def mask(s):
        w, h = size_of(s)
        m = np.full((h, w), 255, np.uint8)
        m[:, : w // 5] = 0
        m[h - h // 6:, :] = 0
        return m

    def setup(fe, s, alone=False):
        if s in (1, 4):
            fe.set_sequence_mask(s if not alone else 0, mask(s), mask(s)[::-1].copy())
        if s in maps:
            fe.set_sequence_rectification(s if not alone else 0, left=maps[s][0], right=maps[s][1])

    feed = lambda s, i: feed_bgr(s, i) if s in (3, 4) else feed_grey(s, i)
    ref = alone(SEQS, feed=feed, setup=setup, **prm)
    got = packed(SEQS, schedule(SEQS, per=1), feed=feed, setup=setup, **prm)
    assert_same(ref, got)
    assert sum(v[0]["status"] == 0 for v in got.values()) >= 0.6 * len(got)


def test_device_layout_follows_the_upload(built):
    with plf.Frontend(camera=CAMS[0], limits=limits(2), max_sequences=2, image_sizes=SIZES, **PRM) as fe:
        assert fe.device_layout == (640, 360, 640)
        for w, h in SIZES + [CTX]:
            a = np.zeros((2, h, w), np.uint8)
            fe.batch_upload(a, a)
            assert fe.device_layout == (w, h, (w + 15) // 16 * 16)


def test_oracle_spot_check(built):
    """One short stream per size against the oracle pipeline: features bit-exact, matches and inliers exact, pose to
    1e-4."""
    prm = dict(ofe.DEFAULTS, **PRM)
    kw = {k: prm[k] for k, _ in plf.plf_params._fields_}
    with plf.Frontend(camera=CAMS[0], limits=limits(3), max_sequences=len(CAMS), image_sizes=SIZES, **kw) as fe:
        for s in range(1, 5):
            fe.set_sequence_camera(s, CAMS[s])
        for s in range(5):
            pairs = frames(s)[:3]
            ref = ofe.run_sequence(CAMS[s], pairs, prm)
            res = fe.process_batch(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), seq=[s] * 3)
            for k, (r, g) in enumerate(zip(ref, res)):
                assert g["status"] == r["status"], (s, k)
                assert (g["n_stereo_pt"], g["n_stereo_ls"]) == (r["n_pt"], r["n_ls"]), (s, k)
                check_frame(fe.get_frame(k), r["frame"])
                if r["status"] == 0:
                    assert g["n_matched_pt"] == len(r["res"]["inlier_pt"]) and g["n_matched_ls"] == len(r["res"]["inlier_ls"])
                    assert (g["n_inliers_pt"], g["n_inliers_ls"]) == r["res"]["n_inliers"], (s, k)
                    assert rel(clib.logmap_se3(g["DT"]), clib.logmap_se3(r["DT"])) < POSE_REL_TOL, (s, k)


def test_capacity_refusal_equals_the_twin(built):
    """Isolated dots every 4 px overflow the ORB candidate list of a 1280 x 720 level (w h / 16 corners against the cap
    of 32768; no image reaches w h / 9 + 64 below that): the download is refused as a context created at that size
    refuses it, with the same message, and the batches of the other sizes around it are unaffected."""
    big = camera(1280, 720, 9)
    img = dot_lattice(4, 4, w=1280, h=720)[0]
    msgs = []
    with plf.Frontend(camera=big, limits=limits(1), **PRM) as fe:
        fe.batch_upload(img[None], img[None])
        fe.batch_run(1)
        with pytest.raises(plf.PlfError) as e:
            fe.batch_download(1)
        msgs.append(str(e.value))
    ref = alone([1, 3], per=1)
    with plf.Frontend(camera=CAMS[0], limits=limits(1), max_sequences=len(CAMS), image_sizes=SIZES + [(1280, 720)],
                      **PRM) as fe:
        for s in (1, 3):
            fe.set_sequence_camera(s, CAMS[s])
        fe.set_sequence_camera(2, big)
        got = {}
        for i in range(N):
            for s in (1, 2, 3):
                L, R = frames(s)[i] if s != 2 else (img, img)
                fe.batch_upload(L[None], R[None])
                fe.batch_run(1, seq=[s])
                if s == 2:
                    with pytest.raises(plf.PlfError) as e:
                        fe.batch_download(1)
                    msgs.append(str(e.value))
                else:
                    got[(s, i)] = (fe.batch_download_array(1)[0], fe.get_frame(0), fe.get_matches(0))
    assert "candidate capacity" in msgs[0] and all(m == msgs[0] for m in msgs), msgs
    assert_same(ref, got)


def kf_problems():
    """Keyframes of two sequences of different sizes (frames 0 and 2 of each), from a packed run."""
    out = {}
    with plf.Frontend(camera=CAMS[0], limits=limits(1), max_sequences=len(CAMS), image_sizes=SIZES, **PRM) as fe:
        for s in (1, 2):
            fe.set_sequence_camera(s, CAMS[s])
            for i in (0, 2):
                L, R = frames(s)[i]
                fe.batch_upload(L[None], R[None])
                fe.batch_run(1, seq=[s], restart=[1])
                fe.batch_download(1)
                out[(s, i)] = fe.get_frame(0)
    return out


def test_keyframe_matching_takes_each_problem_size(built):
    """match_kf2kf_batch / match_map2kf_batch over keyframes of sequences of two sizes in one call equal each problem's
    single call on a context created at that size."""
    kfs = kf_problems()
    DT = np.eye(4)
    DT[2, 3] = -0.3
    probs = [dict(prev=kfs[(s, 0)], curr=kfs[(s, 2)], DT=DT) for s in (1, 2)]
    with plf.Frontend(camera=CAMS[0], limits=limits(1), max_sequences=len(CAMS), image_sizes=SIZES, **PRM) as fe:
        for s in (1, 2):
            fe.set_sequence_camera(s, CAMS[s])
        got = fe.match_kf2kf_batch(probs, seq=[1, 2])
    for j, s in enumerate((1, 2)):
        with plf.Frontend(camera=CAMS[s], limits=limits(1), **PRM) as fe:
            one = fe.match_kf2kf(**probs[j])
        assert one.keys() == got[j].keys()
        for k in one:
            assert np.array_equal(np.asarray(one[k]), np.asarray(got[j][k])), (s, k)
        assert one["n_pt"] > 0, s


def test_refusals_change_nothing(built):
    """A mixed-size batch, an undeclared upload size, set_image_sizes after the first batch, an invalid size and a size
    change with maps or masks set: each is refused with nothing changed, and the run goes on as an uninterrupted one."""
    seqs = [0, 1, 2]
    batches = schedule(seqs)
    ref = packed(seqs, batches)
    with plf.Frontend(camera=CAMS[0], limits=limits(2), max_sequences=len(CAMS), image_sizes=SIZES, **PRM) as fe:
        with pytest.raises(plf.PlfError, match=r"size 1 \(40x40\)"):
            fe.set_image_sizes([(704, 392), (40, 40)])
        with pytest.raises(plf.PlfError, match="n = 9"):
            fe.set_image_sizes([(600 + i, 300) for i in range(9)])
        assert fe.image_sizes == SIZES
        with pytest.raises(plf.PlfError, match=r"size 600x300 is not one of the context's image sizes \(640x360, 704x392"):
            fe.set_sequence_camera(1, camera(600, 300))
        for s in (1, 2):
            fe.set_sequence_camera(s, CAMS[s])
        maps = rectify.stereo_maps(size=size_of(1))[:2]
        fe.set_sequence_rectification(1, left=maps[0], right=maps[1])
        with pytest.raises(plf.PlfError, match="sequence 1 has rectification maps of 704x392; clear it"):
            fe.set_sequence_camera(1, CAMS[2])
        fe.set_sequence_rectification(1)
        w, h = size_of(2)
        fe.set_sequence_mask(2, np.full((h, w), 255, np.uint8))
        with pytest.raises(plf.PlfError, match="sequence 2 has masks of 512x288"):
            fe.set_sequence_camera(2, None)
        fe.set_sequence_mask(2)
        for s in (1, 2):   # the cameras again: each restarts its sequence, as in the uninterrupted run
            fe.set_sequence_camera(s, CAMS[s])
        got = {}
        for j, batch in enumerate(batches):
            L = np.stack([frames(s)[i][0] for s, i in batch])
            R = np.stack([frames(s)[i][1] for s, i in batch])
            if j == 1:
                a = np.zeros((1, 300, 600), np.uint8)
                with pytest.raises(plf.PlfError, match="plf_batch_upload_sized.*600x300"):
                    fe.batch_upload_raw(1, a.ctypes.data, a.ctypes.data, size=(600, 300))
                # a batch whose pairs are of another size than its upload
                other = [k for k in range(3) if size_of(k) != size_of(batch[0][0])][0]
                fe.batch_upload(L, R)
                with pytest.raises(plf.PlfError, match=r"pair 0 is of sequence %d" % other):
                    fe.batch_run(1, seq=[other])
            else:
                fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=[s for s, _ in batch])
            res = fe.batch_download_array(len(batch))
            for k, key in enumerate(batch):
                got[key] = (res[k], fe.get_frame(k), fe.get_matches(k))
            if j == 0:
                with pytest.raises(plf.PlfError, match="the pipeline exists"):
                    fe.set_image_sizes([])
    assert_same(ref, got)
