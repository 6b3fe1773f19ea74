"""The LSD seed ordering (one CTA per image: the image's seed-list entries cut into equal ranges per warp, bin counts in
shared memory) against the oracle, on the shapes that partition of the work meets: a batch mixing an image without seeds,
an image where nearly every pixel is a seed and ordinary frames; all seeds in a few rows, so every warp's range starts
and ends inside one row segment; one bin and 1024 bins; scaled widths that are not a multiple of the 512-column
segment.  The region growing consumes the seeds in order, so segments and KeyLines equal to the oracle's pin the order."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe
from test_pipeline_gpu import compare

pytestmark = pytest.mark.gpu


def dense_noise(h, w, seed):
    """High-contrast noise: nearly every pixel's gradient is above LSD's threshold."""
    rng = np.random.default_rng(seed)
    return np.where(rng.random((h, w)) < 0.5, rng.integers(0, 40, (h, w)), rng.integers(215, 256, (h, w))).astype(np.uint8)


def row_band(h, w, y0, rows, seed):
    """Flat image whose only texture is a band of `rows` noisy rows starting at y0."""
    img = np.full((h, w), 90, np.uint8)
    img[y0:y0 + rows] = dense_noise(rows, w, seed)
    return img


def check_lines(fe, img, prm):
    """plf_lsd segments and plf_detect_lines KeyLines + LBD descriptors equal to the oracle's, bit for bit."""
    segs = fe.lsd(img, cap=65536)
    ref = clib.lsd(img, **ofe.lsd_kwargs(prm))
    assert segs.shape == ref.shape and np.array_equal(segs, ref)
    kl, desc = fe.detect_lines(img)
    okl, odesc = ofe.detect_lines(img, prm["lsd_nfeatures"], prm["min_line_length"], ofe.lsd_kwargs(prm))
    assert len(kl) == len(okl) and kl.tobytes() == okl.tobytes() and np.array_equal(desc, odesc)
    return len(ref)


def test_mixed_batch_blank_noise_and_stream(built):
    """One batch of plf_batch_upload / run / download whose images have 0 seeds (flat), nearly every pixel a seed (dense
    noise), a few seed rows, and stream frames: per-image ranges of very different lengths in one launch, cut inside row
    segments.  Every frame's stereo features, matches and pose against the oracle pipeline; then the same images through
    the standalone plf_lsd / plf_detect_lines."""
    cam = plf.KITTI_CAMERA
    h, w = cam["height"], cam["width"]
    frames = list(synth.stream(cam, 2, seed=7))
    flat = np.full((h, w), 90, np.uint8)
    pairs = [(frames[0][0], frames[0][1]), (flat, flat), (dense_noise(h, w, 1), dense_noise(h, w, 2)),
             (row_band(h, w, 200, 3, 3), row_band(h, w, 201, 3, 4)), (frames[1][0], frames[1][1])]
    prm = dict(ofe.DEFAULTS, orb_nfeatures=1500, lsd_nfeatures=200)
    ref = ofe.run_sequence(cam, pairs, prm)
    lim = plf.default_limits(); lim.max_batch = len(pairs); lim.max_segments = 65536
    kw = {k: prm[k] for k, _ in plf.plf_params._fields_}
    with plf.Frontend(camera=cam, limits=lim, **kw) as fe:
        fe.batch_upload(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]))
        fe.batch_run(len(pairs))
        got = fe.batch_download(len(pairs))
        feats = [fe.get_frame(k) for k in range(len(pairs))]
        compare(ref, got, feats)
        assert got[0]["n_stereo_ls"] > 0
        n = [check_lines(fe, img, prm) for p in pairs for img in p]
    assert n[2] == 0 and n[4] > 100 and n[0] > 50


@pytest.mark.parametrize("n_bins", [1, 1024])
def test_seeds_in_one_row_band(built, n_bins):
    """All seeds in 4 rows of a KITTI-size image (each warp's range a piece of one row), and a stream frame, with every
    seed in one bin (the order is then the raster order) and with 1024 bins."""
    cam = plf.KITTI_CAMERA
    h, w = cam["height"], cam["width"]
    prm = dict(ofe.DEFAULTS, lsd_n_bins=n_bins, lsd_nfeatures=200)
    lim = plf.default_limits(); lim.max_segments = 65536
    L = next(iter(synth.stream(cam, 1, seed=11)))[0]
    with plf.Frontend(camera=cam, limits=lim, lsd_n_bins=n_bins, lsd_nfeatures=200) as fe:
        assert check_lines(fe, row_band(h, w, 150, 4, 5), prm) > 0
        assert check_lines(fe, L, prm) > 50


@pytest.mark.parametrize("w,h,scale", [(1242, 375, 1.0), (1242, 375, 1.2), (640, 360, 1.2), (427, 200, 1.0), (1024, 300, 1.0)])
def test_scaled_widths(built, w, h, scale):
    """Scaled widths 1242, 1490, 768 and 427 (last row segment partly filled; one segment per row) and 1024 (whole
    segments), on a scene and on dense noise."""
    prm = dict(ofe.DEFAULTS, lsd_scale=scale, lsd_nfeatures=200)
    lim = plf.default_limits(); lim.max_segments = 65536
    L, _ = synth.scene_pair(w=w, h=h, seed=w + h)
    with plf.Frontend(camera=dict(plf.KITTI_CAMERA, width=w, height=h), limits=lim, lsd_scale=scale, lsd_nfeatures=200) as fe:
        assert check_lines(fe, L, prm) > 20
        assert check_lines(fe, dense_noise(h, w, 6), prm) > 0
