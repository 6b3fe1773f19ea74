"""CPU tests of colour input: oracle/color.py, the restatement k_color follows, equals cv2.cvtColor(COLOR_BGR2GRAY /
COLOR_BGRA2GRAY) on every 8-bit colour, and its colour remap then conversion equals cv2.cvtColor(cv2.remap(...)) on
EuRoC's calibration maps, identity maps, out-of-image maps and an odd image size.  Also the interface: the header and
library declare and export plf_batch_upload_color, and its refusals that need no device."""
import re
from pathlib import Path

import numpy as np
import pytest

from oracle import color, rectify

cv2 = pytest.importorskip("cv2")

ROOT = Path(__file__).resolve().parent.parent


def all_colours():
    """uint8 [4096, 4096, 3]: every (B, G, R) once."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([v & 255, (v >> 8) & 255, v >> 16], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)


def image(rng, h, w, ch=3):
    """Noise over a smooth ramp per channel: every tap weight and every channel changes the result."""
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([((x * (3 + c) + y * (5 + 2 * c)) % 256 ^ rng.integers(0, 256, (h, w))) for c in range(ch)],
                    axis=-1).astype(np.uint8)


def cv_gray(img):
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY if img.shape[-1] == 3 else cv2.COLOR_BGRA2GRAY)


def assert_same(got, ref):
    assert got.dtype == ref.dtype == np.uint8 and got.shape == ref.shape
    bad = np.argwhere(got != ref)
    assert bad.size == 0, f"{len(bad)} bytes differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} vs {ref[tuple(bad[0])]}"


def test_every_colour_three_channels():
    img = all_colours()
    assert_same(color.bgr_to_gray(img), cv2.cvtColor(img, cv2.COLOR_BGR2GRAY))


def test_every_colour_four_channels_alpha_ignored():
    """BGRA with a random alpha per pixel: both COLOR_BGRA2GRAY and COLOR_BGR2GRAY on the 4-channel image give the
    3-channel result."""
    bgr = all_colours()
    alpha = np.random.default_rng(0).integers(0, 256, bgr.shape[:2], dtype=np.uint8)
    bgra = np.concatenate([bgr, alpha[..., None]], axis=-1)
    want = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
    assert_same(color.bgr_to_gray(bgra), want)
    assert_same(cv2.cvtColor(bgra, cv2.COLOR_BGRA2GRAY), want)
    assert_same(cv2.cvtColor(bgra, cv2.COLOR_BGR2GRAY), want)


def test_opencv3_coefficients_differ():
    """The 14-bit rule of OpenCV 3 is a different function: the project pins OpenCV 4's."""
    img = all_colours().reshape(-1, 3).astype(np.int64)
    old = ((1868 * img[:, 0] + 9617 * img[:, 1] + 4899 * img[:, 2] + (1 << 13)) >> 14).astype(np.uint8)
    assert int(np.count_nonzero(old != color.bgr_to_gray(img.astype(np.uint8)))) == 43864


def assert_remap_gray(img, m1, m2):
    assert_same(color.remap_to_gray(img, m1, m2), cv_gray(cv2.remap(img, m1, m2, cv2.INTER_LINEAR)))
    # the colour remap itself is cv2.remap per channel
    assert_same(color.remap(img, m1, m2), cv2.remap(img, m1, m2, cv2.INTER_LINEAR))


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("side", [0, 1])
def test_euroc_stereo_rectify(side, ch):
    m1, m2 = rectify.stereo_maps()[side]
    assert_remap_gray(image(np.random.default_rng(side), 480, 752, ch), m1, m2)


@pytest.mark.parametrize("ch", [3, 4])
def test_identity_maps(ch):
    h, w = 480, 752
    y, x = np.mgrid[0:h, 0:w]
    m1 = np.stack([x, y], axis=-1).astype(np.int16)
    m2 = np.zeros((h, w), np.uint16)
    img = image(np.random.default_rng(2), h, w, ch)
    assert np.array_equal(color.remap_to_gray(img, m1, m2), cv_gray(img))
    assert_remap_gray(img, m1, m2)


@pytest.mark.parametrize("ch", [3, 4])
def test_maps_outside_the_image(ch):
    rng = np.random.default_rng(3)
    h, w = 64, 96
    img = image(rng, h, w, ch)
    xs = np.concatenate([np.array([-2, -1, 0, 1, w - 2, w - 1, w, w + 1, -32768, 32767], np.int16),
                         rng.integers(-20, w + 20, 100).astype(np.int16)])
    ys = np.concatenate([np.array([-2, -1, 0, 1, h - 2, h - 1, h, h + 1, -32768, 32767], np.int16),
                         rng.integers(-20, h + 20, 100).astype(np.int16)])
    gx, gy = np.meshgrid(xs, ys)
    m1 = np.stack([gx, gy], axis=-1).astype(np.int16)
    m2 = rng.integers(0, 65536, gx.shape).astype(np.uint16)
    assert_remap_gray(img, m1, m2)


@pytest.mark.parametrize("ch", [3, 4])
def test_odd_image_size(ch):
    rng = np.random.default_rng(5)
    h, w = 23, 37
    img = image(rng, h, w, ch)
    m1 = np.stack([rng.integers(-3, w + 3, (h, w)), rng.integers(-3, h + 3, (h, w))], axis=-1).astype(np.int16)
    m2 = rng.integers(0, 1024, (h, w)).astype(np.uint16)
    assert_remap_gray(img, m1, m2)
    for m in rectify.stereo_maps(size=(w, h))[:2]:
        assert_remap_gray(img, *m)


def test_remap_and_conversion_do_not_commute():
    """Converting first and remapping the grey image is not what a rectified colour camera gives: the order matters."""
    img = image(np.random.default_rng(6), 480, 752)
    m1, m2 = rectify.stereo_maps()[0]
    right_order = color.remap_to_gray(img, m1, m2)
    wrong_order = rectify.remap(color.bgr_to_gray(img), m1, m2)
    assert np.count_nonzero(right_order != wrong_order) > 1000
    assert_same(right_order, cv_gray(cv2.remap(img, m1, m2, cv2.INTER_LINEAR)))


def test_upload_color_symbols(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"plf_status plf_batch_upload_color\(plf_ctx\* ctx, int B, const uint8_t\* left, const uint8_t\* right, "
                     r"int stride, int channels\);", hdr)
    lib = plf.load_library()
    assert hasattr(lib, "plf_batch_upload_color")
    assert callable(plf.Frontend.batch_upload) and callable(plf.Frontend.batch_upload_raw)
    # NULL context: PLF_ERR_INVALID, named, without a device
    assert lib.plf_batch_upload_color(None, 1, None, None, 0, 3) == -1
    assert b"ctx is NULL" in lib.plf_last_error(None)
