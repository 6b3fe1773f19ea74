"""CPU tests: oracle/rectify.py, the restatement k_rectify follows, equals cv2.remap(img, map1, map2, INTER_LINEAR) with
CV_16SC2 maps and the default constant-0 border byte for byte: on EuRoC's calibration, identity maps, maps pointing
partly or wholly outside the image, every entry of the weight table, and an odd image size."""
import numpy as np
import pytest

from oracle import rectify

cv2 = pytest.importorskip("cv2")


def cv_remap(img, m1, m2):
    return cv2.remap(img, m1, m2, cv2.INTER_LINEAR)


def image(rng, h, w):
    """Noise over a smooth ramp: every tap weight changes the result."""
    y, x = np.mgrid[0:h, 0:w]
    return ((x * 3 + y * 5) % 256 ^ rng.integers(0, 256, (h, w))).astype(np.uint8)


def assert_same(img, m1, m2):
    got, ref = rectify.remap(img, m1, m2), cv_remap(img, m1, m2)
    assert got.dtype == ref.dtype == np.uint8 and got.shape == ref.shape
    bad = np.argwhere(got != ref)
    assert bad.size == 0, f"{len(bad)} bytes differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} vs {ref[tuple(bad[0])]}"


def test_weight_table_sums_to_one():
    tab = rectify.weight_table()
    assert tab.shape == (1024, 4) and np.all(tab.sum(axis=1) == 1 << 15) and np.all(tab >= 0)
    fy, fx = np.divmod(np.arange(1024), 32)
    # every weight is an exact multiple of 32: the closed form k_rectify uses
    assert np.array_equal(tab, 32 * np.stack([(32 - fx) * (32 - fy), fx * (32 - fy), (32 - fx) * fy, fx * fy], axis=1))


@pytest.mark.parametrize("side", [0, 1])
def test_euroc_stereo_rectify(side):
    left, right, cam = rectify.stereo_maps()
    m1, m2 = (left, right)[side]
    assert m1.shape == (480, 752, 2) and m1.dtype == np.int16 and m2.dtype == np.uint16
    if side == 0:   # the left map reaches above the first row: the border is exercised too
        assert np.any(m1[..., 1] < 0)
    assert_same(image(np.random.default_rng(side), 480, 752), m1, m2)


def test_identity_maps():
    h, w = 480, 752
    y, x = np.mgrid[0:h, 0:w]
    m1 = np.stack([x, y], axis=-1).astype(np.int16)
    m2 = np.zeros((h, w), np.uint16)
    img = image(np.random.default_rng(2), h, w)
    assert np.array_equal(rectify.remap(img, m1, m2), img)
    assert_same(img, m1, m2)


def test_maps_outside_the_image():
    """Taps around every edge (-1, 0, the last row and column and one past), far outside (including int16's extremes),
    and map2 over its whole uint16 range (OpenCV masks it with 1023)."""
    rng = np.random.default_rng(3)
    h, w = 64, 96
    img = image(rng, h, w)
    edge_x = np.array([-2, -1, 0, 1, w - 2, w - 1, w, w + 1], np.int16)
    edge_y = np.array([-2, -1, 0, 1, h - 2, h - 1, h, h + 1], np.int16)
    far = np.array([-32768, -1000, -33, 1000, 32767], np.int16)
    xs = np.concatenate([edge_x, far, rng.integers(-20, w + 20, 200).astype(np.int16)])
    ys = np.concatenate([edge_y, far, rng.integers(-20, h + 20, 200).astype(np.int16)])
    gx, gy = np.meshgrid(xs, ys)
    m1 = np.stack([gx, gy], axis=-1).astype(np.int16)
    m2 = rng.integers(0, 65536, gx.shape).astype(np.uint16)
    assert_same(img, m1, m2)
    # wholly outside: every byte is the border value
    m1o = np.full_like(m1, -5)
    assert not rectify.remap(img, m1o, m2).any()
    assert_same(img, m1o, m2)


def test_every_table_entry():
    """Each of the 1024 weight-table entries at interior taps and at taps straddling each edge."""
    rng = np.random.default_rng(4)
    h, w = 40, 50
    img = image(rng, h, w)
    f = np.arange(1024, dtype=np.uint16)
    for sx, sy in ((10, 12), (-1, 5), (w - 1, 5), (7, -1), (7, h - 1), (-1, -1), (w - 1, h - 1)):
        m1 = np.broadcast_to(np.array([sx, sy], np.int16), (32, 32, 2)).copy()
        assert_same(img, m1, f.reshape(32, 32))
    # all entries with random interior taps, and the same indices with high bits set
    m1 = np.stack([rng.integers(0, w - 1, (32, 32)), rng.integers(0, h - 1, (32, 32))], axis=-1).astype(np.int16)
    assert_same(img, m1, f.reshape(32, 32))
    assert_same(img, m1, (f | 0xFC00).reshape(32, 32))


def test_odd_image_size():
    rng = np.random.default_rng(5)
    h, w = 23, 37
    img = image(rng, h, w)
    m1 = np.stack([rng.integers(-3, w + 3, (h, w)), rng.integers(-3, h + 3, (h, w))], axis=-1).astype(np.int16)
    m2 = rng.integers(0, 1024, (h, w)).astype(np.uint16)
    assert_same(img, m1, m2)
    # and a distortion map built for that size
    left, right, _ = rectify.stereo_maps(size=(w, h))
    for m in (left, right):
        assert_same(img, *m)
