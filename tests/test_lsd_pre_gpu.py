"""The LSD pre-grow kernel (pre-blur, resample and gradient in one tile kernel) writes, byte for byte, what a CPU reference
computes: the record map, the seed lists of every row segment, their counts and the per-image maximum of gx^2 + gy^2.
The scaled image is oracle/lsd.c's (cv2's pre-blur and INTER_LINEAR_EXACT resample), the gradient, the lists and the
maximum numpy's, the angle clib.fast_atan2.  At the image sizes around the kernel's tile and box edges, with strided input,
on flat and saturated images, at the defaults, at every LSD parameter case, at scale 1 and at 13 taps; and the launch
it takes."""
import math

import numpy as np
import pytest

import plslam_b200 as plf
import param_cases as pc
from oracle import clib
from oracle import frontend as ofe

pytestmark = pytest.mark.gpu

# settings this test runs besides LSD_CASES: scale 1, and the one tap count no LSD case has
LSD_PRE_CASES = {"scale1.0": dict(lsd_scale=1.0), "scale0.4_k13": dict(lsd_scale=0.4)}
CASES = {"default": {}, **pc.LSD_CASES, **LSD_PRE_CASES}
SEG, LUT_DIM, NOTDEF_BITS = 512, 1021, int(np.float32(-1024.0).view(np.uint32))


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


def m2_min(prm):
    """The smallest gx^2 + gy^2 of a defined pixel: its gradient norm exceeds rho (the library's double expression)."""
    rho = prm["lsd_quant"] / math.sin(math.pi * prm["lsd_ang_th"] / 180)
    return next(m for m in range(2 * 510 * 510 + 1) if not (math.sqrt(m / 4.0) <= rho))


def reference(img, prm):
    """(pix, seedlist, segcnt, maxmag2) of one image, as plf_debug_lsd_pre returns them."""
    s = clib.lsd_scaled_image(img, prm["lsd_scale"], prm["lsd_sigma_scale"]).astype(np.int64)
    H, W = s.shape
    DA, BC = s[1:, 1:] - s[:-1, :-1], s[:-1, 1:] - s[1:, :-1]   # pixel (x, y): D - A, B - C
    gx, gy = np.zeros((H, W), np.int64), np.zeros((H, W), np.int64)
    gx[:-1, :-1], gy[:-1, :-1] = DA + BC, DA - BC
    m2 = gx * gx + gy * gy
    defined = np.zeros((H, W), bool)
    defined[:-1, :-1] = m2[:-1, :-1] >= m2_min(prm)
    li = (gx + 510) * LUT_DIM + (gy + 510)
    keys, inv = np.unique(li[defined], return_inverse=True)
    ang = np.array([clib.fast_atan2(float(k // LUT_DIM - 510), float(-(k % LUT_DIM - 510))) for k in keys], np.float32)
    pix = np.full((H, W), NOTDEF_BITS, np.uint64)
    pix[defined] = ang.view(np.uint32)[inv].astype(np.uint64) | (li[defined].astype(np.uint64) << np.uint64(32))
    nxb = (W + SEG - 1) // SEG
    seed = np.zeros(H * W, np.uint32)
    segcnt = np.zeros((H, nxb), np.int32)
    for y in range(H):
        for xb in range(nxb):
            xs = np.flatnonzero(defined[y, xb * SEG:(xb + 1) * SEG])
            o = y * W + xb * SEG
            seed[o:o + len(xs)] = xs | (m2[y, xb * SEG + xs] << 9)
            segcnt[y, xb] = len(xs)
    return pix.reshape(-1), seed, segcnt, int(m2[defined].max()) if defined.any() else -1


@pytest.fixture(scope="module", params=list(CASES))
def case_fe(request):
    with plf.Frontend(device=0, **CASES[request.param]) as fe:
        yield dict(ofe.DEFAULTS, **CASES[request.param]), fe


def compare(case_fe, imgs, **layout):
    """The kernel against the reference on imgs; a size whose scaled image is below 3 x 3 is refused."""
    prm, fe = case_fe
    n, h, w = imgs.shape
    if min(round(w * prm["lsd_scale"]), round(h * prm["lsd_scale"])) < 3:
        with pytest.raises(plf.PlfError, match="out of range"):
            fe.debug_lsd_pre(imgs, **layout)
        return None
    got = fe.debug_lsd_pre(imgs, **layout)
    for i in range(n):
        want = dict(zip(("pix", "seedlist", "segcnt", "maxmag2"), reference(imgs[i], prm)))
        for k, v in want.items():
            a = np.asarray(got[k][i]).reshape(-1)
            b = np.asarray(v).reshape(-1)
            assert a.shape == b.shape, (k, a.shape, b.shape)
            bad = np.flatnonzero(a != b)
            assert bad.size == 0, f"image {i} {k}: {bad.size} entries differ, first at {bad[:5]} (geometry {got['ks'], got['th'], got['np']})"
    return got


# (w, h): the smallest image; scaled widths at, below and above one and two 512-column segments (w 426..428, 852..854:
# ws 511..514, 1022..1025 at scale 1.2); scaled heights at, below and above multiples of the 16-row CTA (h 13, 14, 26, 27,
# 39, 40, 41: hs 16, 17, 31, 32, 47, 48, 49) and below one CTA; box columns past both edges of narrow images; two sizes
# with one segment and a partial second; a KITTI-class frame
SIZES = [(3, 3), (4, 5), (5, 4), (13, 11), (16, 16), (17, 7), (45, 20), (53, 27), (426, 21), (427, 20), (428, 40),
         (470, 33), (852, 19), (853, 14), (854, 47), (100, 13), (300, 26), (530, 39), (900, 41), (200, 61), (853, 35),
         (1241, 376)]


@pytest.mark.parametrize("w,h", SIZES)
def test_pre_matches_cpu_reference(case_fe, w, h):
    got = compare(case_fe, images(2, h, w, seed=w * 1000 + h))
    if got is not None and w * h > 1000:
        assert (got["segcnt"] > 0).any()


@pytest.mark.parametrize("w,h", [(3, 3), (61, 17), (427, 40), (1241, 376)])
def test_pre_strided_input(case_fe, w, h):
    pitch = (w + 15) // 16 * 16 + 48
    compare(case_fe, images(3, h, w, seed=w + h), pitch=pitch, img_stride=pitch * h + 32)


@pytest.mark.parametrize("w,h", [(37, 29), (640, 100)])
def test_pre_flat_and_saturated(case_fe, w, h):
    flat = np.full((1, h, w), 77, np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    checker = (((xx + yy) % 2) * 255).astype(np.uint8)[None]
    stripes = ((xx // 2 % 2) * 255).astype(np.uint8)[None]
    step = ((xx > w // 2) * 255).astype(np.uint8)[None]
    got = compare(case_fe, np.concatenate([flat, checker, stripes, step]))
    if got is not None:
        assert got["maxmag2"][0] == -1 and (got["segcnt"][0] == 0).all()


def test_pre_launch_geometry():
    """The defaults keep one piece of 16 scaled rows at 7 taps; downsampling cuts the segment into pieces; scale 1 and a
    256 centre tap take no blur."""
    def geo(w=1241, h=376, **prm):
        with plf.Frontend(device=0, **prm) as fe:
            return fe.debug_lsd_pre_geometry(w, h)
    g = geo()
    assert (g["ks"], g["th"], g["np"]) == (7, 16, 1), g
    for scale in (0.8, 0.5):
        assert geo(lsd_scale=scale)["np"] > 1, scale
    assert geo(lsd_scale=1.0)["ks"] == 1
    for name in ("sigma0.28_k5_c256", "scale0.9_sigma0.25_k5_c256"):
        assert geo(**pc.LSD_CASES[name])["ks"] == 1, name
