"""LSD region growing with three queue entries per warp round: segments bit-exact (same values, same order) with the C
restatement on images built for the round's corner cases - neighbours shared by two entries of a round and stale
look-ahead records (thin diagonal and zig-zag edges), regions that end with 1, 2 or 3 entries left in a round (short
strokes of every length), regions of thousands of entries and runs of acceptances that fill the staging ring between
angle evaluations (long, perfectly straight edges), more waiting entries than the shared-memory queue window holds (a
wide ramp), ang_th above 60 degrees, the largest gradients (checkerboard 0/255) and nearly every pixel defined
(noise)."""
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib

pytestmark = pytest.mark.gpu


def cam(w, h):
    return dict(plf.KITTI_CAMERA, width=w, height=h)


def lsd_both(img, **kw):
    h, w = img.shape
    lim = plf.default_limits(); lim.max_segments = 32768
    fkw = {"lsd_" + k: v for k, v in kw.items()}
    with plf.Frontend(camera=cam(w, h), limits=lim, **fkw) as fe:
        got = fe.lsd(img, cap=32768)
    return got, clib.lsd(img, **kw)


def thin_lines(w=480, h=320, seed=3):
    """1-2 px wide diagonals at several slopes and zig-zags on a flat background."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w), 60, np.uint8)
    for _ in range(40):
        x0, y0 = rng.uniform(10, w - 10), rng.uniform(10, h - 10)
        ang = rng.uniform(0, np.pi)
        length = rng.uniform(20, 200)
        width = int(rng.integers(1, 3))
        t = np.linspace(0, length, int(4 * length))
        xs = np.clip(np.round(x0 + t * np.cos(ang)).astype(int), 0, w - 1)
        ys = np.clip(np.round(y0 + t * np.sin(ang)).astype(int), 0, h - 1)
        for dw in range(width):
            img[ys, np.clip(xs + dw, 0, w - 1)] = 200
    for k in range(6):                                   # zig-zags: 45-degree strokes alternating every few pixels
        y, x, dy = 20 + 45 * k, 5, 1
        period = 3 + k
        while x < w - 2:
            img[min(max(y, 0), h - 1), x] = 230
            if k % 2:
                img[min(max(y, 0), h - 1), x + 1] = 230
            x += 1
            y += dy
            if x % period == 0:
                dy = -dy
    return img


def short_strokes(w=480, h=320):
    """Horizontal, vertical and diagonal strokes of 1..24 px, 1..3 px wide, well apart: every queue length mod 3."""
    img = np.full((h, w), 128, np.uint8)
    y = 4
    for width in (1, 2, 3):
        for n in range(1, 25):
            x = 6 + 19 * (n - 1)
            if x + n + 3 >= w or y + 30 >= h:
                break
            img[y:y + width, x:x + n] = 10 if n % 2 else 245                       # horizontal
            img[y + 6:y + 6 + min(n, 16), x:x + width] = 245 if n % 2 else 10      # vertical
            for i in range(min(n, 12)):                                              # diagonal
                img[y + 24 + i, x + i:x + i + width] = 220
        y += 40
    return img


def long_edges(w=900, h=300):
    """Step edges of hundreds of pixels with identical gradients: regions of thousands of queue entries with no angle
    evaluation in between."""
    img = np.zeros((h, w), np.uint8)
    img[40:260, 30:870] = 200
    img[120:180, 100:800] = 90
    return img


def test_thin_diagonals_and_zigzags(built):
    img = thin_lines()
    got, ref = lsd_both(img)
    assert len(ref) > 40 and got.shape == ref.shape and np.array_equal(got, ref)


def test_regions_ending_mid_round(built):
    img = short_strokes()
    got, ref = lsd_both(img)
    assert len(ref) > 40 and got.shape == ref.shape and np.array_equal(got, ref)


def test_long_regions_and_full_staging_ring(built):
    img = long_edges()
    got, ref = lsd_both(img)
    assert len(ref) >= 8 and got.shape == ref.shape and np.array_equal(got, ref)
    assert (np.hypot(ref[:, 2] - ref[:, 0], ref[:, 3] - ref[:, 1]) > 500).any()   # a region far longer than 256 entries


def test_wide_region_queue_beyond_shared_window(built):
    """A ramp of 2 gray levels per pixel at quant 0.25 is one region of ~55 000 pixels spanning ~150 columns of the
    scaled image: its breadth-first front holds more than 256 waiting queue entries (307 in a CPU replay of the
    growing), so the next round's entries are read from the global region-point list, not the shared window."""
    img = np.zeros((300, 400), np.uint8)
    img[:] = np.clip((np.arange(400) - 40) * 2, 0, 255).astype(np.uint8)[None, :]
    got, ref = lsd_both(img, quant=0.25)
    assert len(ref) >= 1 and got.shape == ref.shape and np.array_equal(got, ref)


@pytest.mark.parametrize("ang_th", [65.0, 80.0])
def test_wide_angle_tolerance(built, ang_th):
    for img in (thin_lines(seed=5), long_edges(480, 240)):
        got, ref = lsd_both(img, ang_th=ang_th)
        assert len(ref) > 0 and got.shape == ref.shape and np.array_equal(got, ref)


@pytest.mark.parametrize("cell", [5, 8, 16, 40])
def test_checkerboard_extreme_gradients(built, cell):
    yy, xx = np.mgrid[0:240, 0:320]
    img = np.where(((yy // cell) + (xx // cell)) % 2 == 0, 0, 255).astype(np.uint8)
    got, ref = lsd_both(img)
    assert len(ref) > 50 and got.shape == ref.shape and np.array_equal(got, ref)


@pytest.mark.parametrize("seed", [2, 7])
def test_dense_noise(built, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (240, 320), dtype=np.uint8)
    got, ref = lsd_both(img)
    assert len(ref) > 50 and got.shape == ref.shape and np.array_equal(got, ref)
