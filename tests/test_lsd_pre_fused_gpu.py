"""The fused LSD pre-blur + resample + gradient kernel writes exactly what the three kernels it replaces write: the record
map, the seed lists of every row segment, their counts and the per-image maximum of gx^2 + gy^2, byte for byte, at the
image sizes around its tile and box edges, at 5 and 7 taps, upsampling by 1.2 and 2.0, and with strided input."""
import numpy as np
import pytest

import plslam_b200 as plf
import param_cases as pc

pytestmark = pytest.mark.gpu


def images(n, h, w, seed):
    """Textured images: smooth ramps and blobs plus noise and a few hard edges, so that many pixels are defined."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = []
    for _ in range(n):
        a = 128 + 60 * np.sin(xx * rng.uniform(0.05, 0.3) + yy * rng.uniform(0.05, 0.3))
        a += rng.normal(0, 25, (h, w))
        a[(xx // max(1, w // 5) + yy // max(1, h // 4)) % 2 == 0] += 50
        out.append(np.clip(a, 0, 255).astype(np.uint8))
    return np.stack(out)


def compare(fe, imgs, **layout):
    a = fe.debug_lsd_pre(imgs, True, **layout)
    b = fe.debug_lsd_pre(imgs, False, **layout)
    assert a["fused_applies"]
    for k in ("pix", "seedlist", "segcnt", "maxmag2"):
        assert a[k].shape == b[k].shape, k
        bad = np.flatnonzero(a[k].reshape(-1) != b[k].reshape(-1))
        assert bad.size == 0, f"{k}: {bad.size} entries differ, first at {bad[:5]} (shape {a[k].shape})"
    return a


# (w, h): the smallest image; scaled widths at, below and above one and two 512-column segments (w 426..428, 852..854:
# ws 511..514, 1022..1025); scaled heights at, below and above multiples of the 16-row CTA (h 13, 14, 26, 27, 39, 40, 41:
# hs 16, 17, 31, 32, 47, 48, 49) and below one CTA; box columns past both edges of narrow images; a KITTI-class frame
SIZES = [(3, 3), (4, 5), (5, 4), (13, 11), (16, 16), (17, 7), (45, 20), (53, 27), (426, 21), (427, 20), (428, 40),
         (470, 33), (852, 19), (853, 14), (854, 47), (100, 13), (300, 26), (530, 39), (900, 41), (1241, 376)]


@pytest.mark.parametrize("w,h", SIZES)
def test_fused_matches_three_kernels(w, h):
    with plf.Frontend(device=0) as fe:
        a = compare(fe, images(2, h, w, seed=w * 1000 + h))
        if w * h > 1000:
            assert (a["segcnt"] > 0).any()


@pytest.mark.parametrize("case", ["sigma0.4_k5", "scale2.0"])
@pytest.mark.parametrize("w,h", [(3, 3), (200, 61), (427, 20), (853, 35)])
def test_fused_other_taps_and_scales(case, w, h):
    with plf.Frontend(device=0, **pc.LSD_CASES[case]) as fe:
        compare(fe, images(2, h, w, seed=7 * w + h))


@pytest.mark.parametrize("w,h", [(3, 3), (61, 17), (427, 40), (1241, 376)])
def test_fused_strided_input(w, h):
    pitch = (w + 15) // 16 * 16 + 48
    with plf.Frontend(device=0) as fe:
        compare(fe, images(3, h, w, seed=w + h), pitch=pitch, img_stride=pitch * h + 32)


@pytest.mark.parametrize("w,h", [(37, 29), (640, 100)])
def test_fused_flat_and_saturated(w, h):
    flat = np.full((1, h, w), 77, np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    checker = (((xx + yy) % 2) * 255).astype(np.uint8)[None]
    stripes = ((xx // 2 % 2) * 255).astype(np.uint8)[None]
    step = ((xx > w // 2) * 255).astype(np.uint8)[None]
    with plf.Frontend(device=0) as fe:
        a = compare(fe, np.concatenate([flat, checker, stripes, step]))
        assert a["maxmag2"][0] == -1 and (a["segcnt"][0] == 0).all()


def test_fused_applies_where_footprints_fit():
    """Downsampling: a CTA's footprint does not fit the box, the state keeps the three kernels.  Scale 1 has no
    pre-blur."""
    z = np.zeros((1, 64, 1241), np.uint8)
    with plf.Frontend(device=0, lsd_scale=0.8) as fe:
        assert not fe.debug_lsd_pre(z, None)["fused_applies"]
    with plf.Frontend(device=0, lsd_scale=1.0) as fe:
        assert not fe.debug_lsd_pre(z, None)["fused_applies"]
    with plf.Frontend(device=0) as fe:
        assert fe.debug_lsd_pre(z, None)["fused_applies"]
