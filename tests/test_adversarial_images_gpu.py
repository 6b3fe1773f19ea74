"""GPU tests on the images of tests/adversarial_images.py: ORB and LSD bit-exact against the C oracle (which
test_adversarial_images.py pins to cv2 on the same images and settings) on content that reaches both arms of FAST's
packed rejection test, floods of equal scores, saturated arithmetic and the extreme gradients; every internal capacity
reached on purpose, each with a defined outcome; and the overflow path of the batched pipeline, which must blame the
batch that held the image, leave every other batch and sequence untouched and leave clean state behind."""
import ctypes as C

import numpy as np
import pytest

import adversarial_images as adv
import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe
from test_orb_gpu import assert_same

pytestmark = pytest.mark.gpu


def cam(w=adv.W, h=adv.H):
    return dict(plf.KITTI_CAMERA, width=w, height=h, cx=w / 2.0, cy=h / 2.0)


# ---- bit-exact on every generator ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("th", [0, 1, 20, 127, 128, 200, 254, 255])
def test_orb_bit_exact_on_every_generator(built, th):
    """orb_fast_th below 128 takes the `low | d` arm of fast_gt4, 128 and above the `low & d` arm; 0, 127, 128, 254 and 255
    are the ends of both.  The packed test only rejects, so an error in it shows as missing corners."""
    total = corners = 0
    with plf.Frontend(camera=cam(), orb_fast_th=th) as fe:
        for name, img, _ in adv.small_cases(th):
            kp, desc = fe.orb(img)
            rk, rd = clib.orb(img, 800, fast_th=th)
            assert_same(kp, desc, rk, rd)
            total += len(rk)
            corners += name.startswith(("dot_lattice", "ramp_lattice", "blobs", "noise")) and len(rk) > 0
    assert (total, corners) == (0, 0) if th == 255 else (total > 4000 and corners >= 8)


def test_orb_equal_scores_at_every_tile_seam_phase(built):
    """One score everywhere, a corner at every column and row phase of the 62 x 30 FAST tile: the strict 3 x 3 maximum
    reads the neighbouring tile's halo at each seam, and the (octave, y, x) order carries the whole comparison."""
    w, h = adv.SEAM_W, adv.SEAM_H
    with plf.Frontend(camera=cam(w, h), orb_nfeatures=20000, orb_nlevels=1) as fe:
        for px, py, phase in ((11, 13, (1, 2)), (13, 7, (0, 0))):
            img, _ = adv.dot_lattice(px, py, phase, w=w, h=h)
            kp, desc = fe.orb(img)
            rk, rd = clib.orb(img, 20000, nlevels=1)
            assert 2000 < len(rk) < adv.ORB_SORT_CAP and len(np.unique(rk["response"])) == 1
            assert_same(kp, desc, rk, rd)


@pytest.mark.parametrize("nfeat", [0, 50])
@pytest.mark.parametrize("scale", [1.0, 1.2])
def test_lsd_bit_exact_on_every_generator(built, scale, nfeat):
    """lsd_scale 1.0 takes gradients of the image itself (0 / 255 content gives the largest table entries), 1.2 goes
    through the saturating Q8.8 blur and the resample; lsd_nfeatures 0 returns every line, 50 ranks them."""
    nseg = ranked = 0
    with plf.Frontend(camera=cam(), lsd_scale=scale, lsd_nfeatures=nfeat) as fe:
        for name, img, _ in adv.small_cases():
            ref = clib.lsd(img, scale=scale)
            segs = fe.lsd(img)
            assert segs.shape == ref.shape and np.array_equal(segs, ref), name
            kl, desc = fe.detect_lines(img)
            okl, odesc = ofe.detect_lines(img, lsd_nfeatures=nfeat, lsd_kwargs=dict(scale=scale))
            assert kl.tobytes() == okl.tobytes() and np.array_equal(desc, odesc), name
            nseg += len(ref)
            ranked += nfeat != 0 and len(okl) == nfeat
    assert nseg > 500 and (nfeat == 0 or ranked >= 5)


# ---- the capacities, each reached on purpose ----------------------------------------------------------------------------
def exact_or_refused(call, check, names, not_names=()):
    """The defined outcomes of an input whose cv2 answer fits plf_limits: that answer bit for bit, or PLF_ERR_CAPACITY with
    a message naming the limit that was hit (and none that was not).  Returns True when refused."""
    try:
        got = call()
    except plf.PlfError as e:
        assert "(-4)" in str(e) and all(n in str(e) for n in names) and not any(n in str(e) for n in not_names), str(e)
        return True
    check(got)
    return False


def ordinary(w, h, seed=3):
    return synth.scene_pair(w=w, h=h, seed=seed, n_rect=60, n_lines=30)[0]


@pytest.mark.parametrize("case", ["ties", "nfeatures", "candidates", "max_keypoints"])
def test_orb_capacities(built, case):
    w, h, img, nf, max_kp, names, not_names = {
        # 6006 corners of one score on level 0: retainBest keeps them all, max_keypoints holds all 6600
        "ties": (400, 300, adv.dot_lattice(4, 4, w=400, h=300)[0], 800, 8192, ["ORB_SORT_CAP"], ["max_keypoints", "candidate"]),
        # orb_nfeatures asks level 0 for 6684
        "nfeatures": (640, 480, adv.noise_dense(640, 480)[0], 20000, 32768, ["ORB_SORT_CAP"], ["max_keypoints", "candidate"]),
        # 53181 corners on level 0 against a candidate list of 32768
        "candidates": (1280, 720, adv.dot_lattice(4, 4, w=1280, h=720)[0], 800, 65536, ["candidate capacity"], ["max_keypoints"]),
        # the declared limit: the only one plf_limits moves
        "max_keypoints": (256, 192, adv.noise_dense()[0], 5000, 1000, ["max_keypoints=1000"], ["ORB_SORT_CAP", "candidate"]),
    }[case]
    lim = plf.default_limits(); lim.max_keypoints = max_kp
    rk, rd = clib.orb(img, nf, cap=70000)
    assert len(rk) < max_kp or case == "max_keypoints"
    with plf.Frontend(camera=cam(w, h), limits=lim, orb_nfeatures=nf) as fe:
        for _ in range(2):   # a refusal clears the flag: the second call is judged on its own
            refused = exact_or_refused(lambda: fe.orb(img, cap=70000), lambda got: assert_same(*got, rk, rd), names, not_names)
            assert refused or case != "max_keypoints"
            good = ordinary(w, h)
            kp, desc = fe.orb(good, cap=70000)
            ok, od = clib.orb(good, nf, cap=70000)
            assert 0 < len(ok) < min(max_kp, adv.ORB_SORT_CAP)
            assert_same(kp, desc, ok, od)


@pytest.mark.parametrize("case", ["sort", "max_segments", "max_lines", "fits"])
def test_line_capacities(built, case):
    """blobs(11, 5) at 512 x 384: 5369 segments, every one a line at min_line_length 0."""
    w, h = 512, 384
    img, _ = adv.blobs(11, 5, w=w, h=h)
    nfeat, max_seg, max_lines, names, not_names = {
        "sort": (100, 8192, 8192, ["KL_SORT_CAP"], ["max_segments", "max_lines"]),     # 5369 lines to rank for the top 100
        "max_segments": (100, 1000, 8192, ["max_segments=1000"], ["max_lines"]),
        "max_lines": (0, 8192, 1024, ["max_lines=1024"], ["max_segments", "KL_SORT_CAP"]),
        "fits": (0, 8192, 8192, [], []),                                               # nothing is ranked at lsd_nfeatures 0
    }[case]
    lim = plf.default_limits(); lim.max_segments = max_seg; lim.max_lines = max_lines
    segs_ref = clib.lsd(img)
    kl_ref, desc_ref = ofe.detect_lines(img, lsd_nfeatures=nfeat, min_line_length=0.0)
    assert len(segs_ref) > adv.KL_SORT_CAP and len(kl_ref) == (nfeat or len(segs_ref))
    good = ordinary(w, h)
    good_segs = clib.lsd(good)
    good_kl, good_desc = ofe.detect_lines(good, lsd_nfeatures=nfeat, min_line_length=0.0)
    assert 20 < len(good_segs) < 1000

    def same_lines(got):
        assert got[0].tobytes() == kl_ref.tobytes() and np.array_equal(got[1], desc_ref)

    with plf.Frontend(camera=cam(w, h), limits=lim, lsd_nfeatures=nfeat, min_line_length=0.0) as fe:
        for _ in range(2):
            refused = exact_or_refused(lambda: fe.detect_lines(img, cap=8192), same_lines, names, not_names)
            assert refused == (case != "fits")
            if case != "max_segments":     # the segments themselves fit: plf_lsd is exact whatever the KeyLine stage meets
                assert np.array_equal(fe.lsd(img), segs_ref)
            else:
                with pytest.raises(plf.PlfError, match=r"\(-4\).*max_segments=1000"):
                    fe.lsd(img)
            # growing ran out of max_segments, or not: the record map is all-undefined again and the flag is clear
            assert np.array_equal(fe.lsd(good), good_segs)
            kl, desc = fe.detect_lines(good, cap=8192)
            assert kl.tobytes() == good_kl.tobytes() and np.array_equal(desc, good_desc)


# ---- the batched pipeline: one overflowing pair in a sequence of its own ----------------------------------------------
PIPE_CAM = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
PIPE_PRM = dict(orb_nfeatures=700, lsd_nfeatures=150)
N_BATCH, BAD_BATCH, BAD_SEQ = 4, 1, 2
SEQ = np.array([0, 1, 2], np.int32)


@pytest.fixture(scope="module")
def pipe_stream():
    """Three sequences of N_BATCH ordinary pairs each (one world, three trajectories): [batch][sequence] -> (L, R)."""
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    seqs = [list(synth.stream(PIPE_CAM, N_BATCH, world=world, seed=21 + 7 * q, step=0.12)) for q in range(3)]
    return [[(seqs[q][b][0], seqs[q][b][1]) for q in range(3)] for b in range(N_BATCH)]


def bad_image(kind):
    w, h = PIPE_CAM["width"], PIPE_CAM["height"]
    # "orb": 12 000 equal corners on level 0 and not one segment; "lsd": 6 000 segments against max_segments 1000 and a few
    # hundred corners
    return adv.dot_lattice(4, 4, w=w, h=h)[0] if kind == "orb" else adv.blobs(11, 5, w=w, h=h)[0]


def run_stream(stream, depth, bad=None):
    """N_BATCH batches of three pairs (sequences 0, 1, 2) with `depth` batches in flight; `bad` replaces both images of
    sequence BAD_SEQ in batch BAD_BATCH.  That sequence restarts in the next batch, which is what a caller does after a
    refusal.  Returns per batch (status, message, out[]) and the get_frame rows of every batch that was the last one run
    when it was downloaded."""
    lim = plf.default_limits(); lim.max_batch = 3; lim.max_segments = 1000
    downloads, frames = [], {}
    with plf.Frontend(camera=PIPE_CAM, limits=lim, max_sequences=3, **PIPE_PRM) as fe:
        def download(b, last_run):
            out = np.zeros(3, plf.RESULT_DTYPE)
            st = fe.lib.plf_batch_download(fe._ctx, 3, out.ctypes.data_as(C.c_void_p))
            downloads.append((st, fe.lib.plf_last_error(fe._ctx).decode() if st else "", out))
            if b == last_run:
                frames[b] = [fe.get_frame(k) for k in range(3)]

        pending = []
        for b in range(N_BATCH):
            pairs = list(stream[b])
            if bad is not None and b == BAD_BATCH:
                pairs[BAD_SEQ] = (bad, bad)
            restart = np.array([0, 0, b == BAD_BATCH + 1], np.uint8)
            fe.batch_upload(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]))
            fe.batch_run(3, seq=SEQ, restart=restart)
            pending.append(b)
            if len(pending) == depth:
                download(pending.pop(0), b)
        while pending:
            download(pending.pop(0), N_BATCH - 1)
    return downloads, frames


_clean, _oracle_frames = {}, {}


def clean_run(stream, depth, parities):
    if (depth, parities) not in _clean:
        _clean[depth, parities] = run_stream(stream, depth)
    return _clean[depth, parities]


def same_rows(a, b, rows):
    for k in rows:
        assert a[k].tobytes() == b[k].tobytes(), k


def same_frames(fa, fb, rows):
    for k in rows:
        for name in fa[k]:
            assert np.array_equal(fa[k][name], fb[k][name]), (k, name)


@pytest.mark.parametrize("parities", ["2", "1"])
@pytest.mark.parametrize("depth", [1, 2, 3])
@pytest.mark.parametrize("kind", ["orb", "lsd"])
def test_pipeline_overflow_blames_its_batch_only(built, monkeypatch, pipe_stream, kind, depth, parities):
    monkeypatch.setenv("PLF_LSD_PARITIES", parities)
    clean, clean_frames = clean_run(pipe_stream, depth, parities)
    got, got_frames = run_stream(pipe_stream, depth, bad_image(kind))
    assert [st for st, _, _ in clean] == [0] * N_BATCH
    assert sum(out["n_kp_l"].sum() + out["n_lines_l"].sum() for _, _, out in clean) > 0
    others = [q for q in range(3) if q != BAD_SEQ]
    for b, ((st, msg, out), (_, _, ref)) in enumerate(zip(got, clean)):
        # exactly the batch that held the image is refused, and the message names the kind and its limit
        assert st == (-4 if b == BAD_BATCH else 0), (b, st, msg)
        if b == BAD_BATCH:
            assert ("ORB keypoints" in msg) == (kind == "orb") and ("LSD segments/lines" in msg) == (kind == "lsd"), msg
            assert ("max_keypoints=4096" if kind == "orb" else "max_segments=1000") in msg, msg
            # out[] is written all the same: the other sequences' rows are exact, the offending row is the result on the
            # truncated feature lists, its counts within the limits
            bad_row = out[BAD_SEQ]
            assert bad_row["n_kp_l"] == 4096 if kind == "orb" else bad_row["n_kp_l"] < 4096
            assert bad_row["n_lines_l"] <= PIPE_PRM["lsd_nfeatures"]
        # the other sequences never see it; the offending sequence is exact again from its restart
        same_rows(out, ref, others + ([BAD_SEQ] if b != BAD_BATCH else []))
    assert got_frames.keys() == clean_frames.keys() and N_BATCH - 1 in got_frames
    for b in got_frames:
        same_frames(got_frames[b], clean_frames[b], others + ([BAD_SEQ] if b > BAD_BATCH else []))
    # the lines of the first ordinary batch downloaded with its frames after the refusal equal the oracle's (depth 1: the
    # very next batch): the LSD record maps were left all-undefined and the flags clear
    b = min(k for k in got_frames if k > BAD_BATCH)
    prm = dict(ofe.DEFAULTS, **PIPE_PRM)
    for q in range(3):
        if (b, q) not in _oracle_frames:
            _oracle_frames[b, q] = ofe.extract_stereo(PIPE_CAM, *pipe_stream[b][q], prm)
        f = _oracle_frames[b, q]
        g = got_frames[b][q]
        assert len(f.ls_spl) > 5 and np.array_equal(g["ls_spl"], f.ls_spl) and np.array_equal(g["ls_epl"], f.ls_epl)
        assert np.array_equal(g["ldesc"], f.ldesc)
