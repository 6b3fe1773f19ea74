"""The LSD hand-off maps with one copy and with one copy per batch parity give the same pipeline results, and the packed
LSD buffers (8-byte record, one u32 seed-list entry holding the column and |grad|^2 or the bin) stay bit-exact against
the oracle at the extremes of their fields: the largest gradient the 2x2 operator produces, and images where almost
every pixel is defined (full seed lists)."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth

pytestmark = pytest.mark.gpu


def gradients(img):
    """LSD's 2x2 gradient (gx, gy) at every pixel but the last row / column (scale 1: no pre-blur, no resample)."""
    a = img.astype(np.int32)
    A, B, C, D = a[:-1, :-1], a[:-1, 1:], a[1:, :-1], a[1:, 1:]
    return (D - A) + (B - C), (D - A) - (B - C)


@pytest.mark.parametrize("depth", [1, 3])
def test_lsd_one_and_two_parities_agree(built, monkeypatch, depth):
    """PLF_LSD_PARITIES=1 (pre-grow and growing on one stream, one map copy) and =2 (maps per batch parity, pre-grow of
    batch i+1 on its own stream under the growing of batch i): identical results, with `depth` batches in flight."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = list(synth.stream(cam, 8, world=world, seed=21, step=0.12))
    Ls, Rs = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])

    def run():
        lim = plf.default_limits(); lim.max_batch = 2
        out = []
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
            pend = 0
            for s0 in range(0, 8, 2):
                fe.batch_upload(Ls[s0:s0 + 2], Rs[s0:s0 + 2]); fe.batch_run(2); pend += 1
                if pend == depth:
                    out += list(fe.batch_download_array(2)); pend -= 1
            while pend:
                out += list(fe.batch_download_array(2)); pend -= 1
        return out
    monkeypatch.setenv("PLF_LSD_PARITIES", "1")
    one = run()
    monkeypatch.setenv("PLF_LSD_PARITIES", "2")
    two = run()
    assert len(one) == len(two) == 8
    assert sum(r["n_lines_l"] for r in one) > 0
    for a, b in zip(one, two):
        for f in plf.RESULT_FIELDS:
            assert a[f] == b[f], f
        assert np.array_equal(a["DT"], b["DT"])


def test_lsd_extreme_gradient_checkerboard(built):
    """A 0/255 checkerboard at scale 1 (no pre-blur): its edges carry |gx| or |gy| = 510, the largest value of the
    gradient tables and of the seed list's |grad|^2 field."""
    h, w = 300, 520
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.where(((yy // 23) + (xx // 37)) % 2 == 0, 0, 255).astype(np.uint8)
    gx, gy = gradients(img)
    assert max(np.abs(gx).max(), np.abs(gy).max()) == 510
    with plf.Frontend(camera=dict(plf.KITTI_CAMERA, width=w, height=h), lsd_scale=1.0) as fe:
        segs = fe.lsd(img)
    ref = clib.lsd(img, scale=1.0)
    assert len(ref) > 50 and segs.shape == ref.shape and np.array_equal(segs, ref)


@pytest.mark.parametrize("scale", [1.0, 1.2])
def test_lsd_dense_noise_full_seed_lists(built, scale):
    """High-contrast noise at KITTI size: nearly every pixel is defined, so the row-segment seed lists (512 columns)
    are full and the seed ordering sorts almost all of the image."""
    h, w = 375, 1242
    rng = np.random.default_rng(5)
    img = np.where(rng.random((h, w)) < 0.5, rng.integers(0, 40, (h, w)), rng.integers(215, 256, (h, w))).astype(np.uint8)
    if scale == 1.0:
        gx, gy = gradients(img)
        assert np.mean(np.sqrt((gx * gx + gy * gy) / 4.0) > 2.0 / np.sin(np.pi * 22.5 / 180)) > 0.7
    lim = plf.default_limits(); lim.max_segments = 65536
    with plf.Frontend(camera=dict(plf.KITTI_CAMERA, width=w, height=h), limits=lim, lsd_scale=scale) as fe:
        segs = fe.lsd(img, cap=65536)
    ref = clib.lsd(img, scale=scale)
    assert len(ref) > 0 and segs.shape == ref.shape and np.array_equal(segs, ref)
