"""CPU checks of tests/adversarial_images.py: every generator provokes what its record says (measured with the C
oracle), oracle/orb.c and oracle/lsd.c equal cv2 bit for bit on every generator - at FAST thresholds on both sides of 128
and at both ends of the range, and at lsd_scale 1.0 and 1.2 - and a plain model of the indices the LSD kernels form shows
that no generator drives one out of its table.  The GPU tests (test_adversarial_images_gpu.py) lean on all three."""
import numpy as np
import pytest

import adversarial_images as adv
from oracle import clib
from oracle import frontend as ofe
from oracle.cvref import lsd_cv2, orb_cv2

FAST_THRESHOLDS = [0, 1, 20, 127, 128, 200, 254, 255]
KP_FIELDS = ["x", "y", "size", "angle", "response", "octave"]


def orb_equal(a, b):
    (ka, da), (kb, db) = a, b
    return len(ka) == len(kb) and all(np.array_equal(ka[f], kb[f]) for f in KP_FIELDS) and np.array_equal(da, db)


# ---- the pin the GPU tests lean on ------------------------------------------------------------------------------------
@pytest.mark.parametrize("th", FAST_THRESHOLDS)
def test_orb_oracle_equals_cv2_on_every_generator(built, th):
    pytest.importorskip("cv2")
    total = 0
    for name, img, _ in adv.small_cases(th):
        got, ref = clib.orb(img, 800, fast_th=th), orb_cv2(img, 800, fast_th=th)
        assert orb_equal(got, ref), (name, th, len(got[0]), len(ref[0]))
        total += len(ref[0])
    print(f"orb_fast_th {th}: {total} keypoints over the generators, oracle == cv2")
    assert (total == 0) == (th == 255)   # no difference exceeds 255; every other threshold finds corners


@pytest.mark.parametrize("scale", [1.0, 1.2])
def test_lsd_oracle_equals_cv2_on_every_generator(built, scale):
    pytest.importorskip("cv2")
    total = 0
    for name, img, _ in adv.small_cases():
        got, ref = clib.lsd(img, scale=scale), lsd_cv2(img, scale=scale)
        assert got.shape == ref.shape and np.array_equal(got, ref), (name, scale, len(got), len(ref))
        total += len(ref)
    print(f"lsd_scale {scale}: {total} segments over the generators, oracle == cv2")
    assert total > 500


def test_capacity_images_oracle_equals_cv2(built):
    """The large images of the capacity tests, where cv2's answer is the one the library must return or refuse."""
    pytest.importorskip("cv2")
    for img, prm in ((adv.dot_lattice(4, 4, w=400, h=300)[0], dict(nfeatures=800)),
                     (adv.noise_dense(640, 480)[0], dict(nfeatures=20000)),
                     (adv.dot_lattice(4, 4, w=1280, h=720)[0], dict(nfeatures=800))):
        assert orb_equal(clib.orb(img, cap=70000, **prm), orb_cv2(img, **prm))
    img = adv.blobs(11, 5, w=512, h=384)[0]
    assert np.array_equal(clib.lsd(img), lsd_cv2(img))


# ---- the generators do what they claim --------------------------------------------------------------------------------
def per_level(kps, nlevels=4):
    return np.bincount(kps["octave"], minlength=nlevels)


def test_tie_flood_exceeds_the_sort_capacity_but_not_max_keypoints(built):
    img, _ = adv.dot_lattice(4, 4, w=400, h=300)
    kps, _ = clib.orb(img, 800, cap=70000)
    lv = per_level(kps)
    print(f"tie flood 400x300: survivors per level {lv.tolist()} against ORB_SORT_CAP {adv.ORB_SORT_CAP}, total {len(kps)}")
    assert lv[0] > adv.ORB_SORT_CAP and len(kps) < 8192          # a level overflows while max_keypoints = 8192 holds all
    assert np.all(kps["response"][kps["octave"] == 0] == 254)    # one score: retainBest keeps every one of them


def test_nfeatures_can_ask_one_level_for_more_than_the_sort_capacity(built):
    img, _ = adv.noise_dense(640, 480)
    kps, _ = clib.orb(img, 20000, cap=70000)
    lv = per_level(kps)
    print(f"noise 640x480, orb_nfeatures 20000: survivors per level {lv.tolist()} against ORB_SORT_CAP {adv.ORB_SORT_CAP}")
    assert lv[0] > adv.ORB_SORT_CAP and len(kps) < 32768


def test_lattice_exceeds_the_candidate_capacity(built):
    w, h = 1280, 720
    img, _ = adv.dot_lattice(4, 4, w=w, h=h)
    kps, _ = clib.orb(img, 800, cap=70000)
    n0 = int(per_level(kps)[0])   # all of one score, so retainBest keeps every level-0 candidate
    print(f"lattice {w}x{h}: {n0} level-0 candidates against cand_cap {adv.cand_cap(w, h)}, total {len(kps)}")
    assert adv.cand_cap(w, h) == adv.CAND_CAP_MAX and n0 > adv.CAND_CAP_MAX and len(kps) < 65536
    # the small lattice stays below its level's capacity, and dense noise comes nowhere near it
    small = per_level(clib.orb(adv.dot_lattice(4, 4)[0], 800)[0])[0]
    noise = int((clib.fast_score_map(adv.noise_dense(w, h)[0], 20) > 0).sum())
    print(f"lattice {adv.W}x{adv.H}: {small} against {adv.cand_cap(adv.W, adv.H)}; noise {w}x{h}: {noise} scored pixels")
    assert small < adv.cand_cap(adv.W, adv.H)


def test_blobs_exceed_the_line_capacities(built):
    img, _ = adv.blobs(11, 5, w=512, h=384)
    segs = clib.lsd(img)
    kl, _ = ofe.detect_lines(img, lsd_nfeatures=0, min_line_length=0.0)
    print(f"blobs 512x384: {len(segs)} segments, {len(kl)} lines against KL_SORT_CAP {adv.KL_SORT_CAP}")
    assert len(kl) > adv.KL_SORT_CAP and len(segs) < 8192


def test_lattices_put_a_corner_at_every_tile_seam_phase(built):
    tw, th_ = adv.FAST_TILE
    for px, py, phase in ((7, 7, (3, 5)), (11, 13, (1, 2))):
        assert np.gcd(px, tw) == 1 and np.gcd(py, th_) == 1
        kps, _ = clib.orb(adv.dot_lattice(px, py, phase, w=adv.SEAM_W, h=adv.SEAM_H)[0], 20000, nlevels=1, cap=70000)
        assert len(np.unique(kps["response"])) == 1
        x, y = kps["x"].astype(int), kps["y"].astype(int)
        assert len(np.unique(x % tw)) == tw and len(np.unique(y % th_)) == th_, (px, py)


def test_binary_images_hold_every_extreme_gradient(built):
    seen = set()
    for img, _ in [adv.checker(c) for c in (1, 2, 3)] + [adv.stripes(p, o) for p in (1, 2) for o in "hv"] + [adv.dot_lattice(4, 4)]:
        gx, gy = adv.gradients(img)
        seen |= set(zip(gx.ravel().tolist(), gy.ravel().tolist()))
    print("extreme (gx, gy) pairs present:", sorted(p for p in seen if 510 in map(abs, p)))
    # gx = (D - A) + (B - C), gy = (D - A) - (B - C) with |D - A|, |B - C| <= 255: the reachable gradients are the diamond
    # |gx| + |gy| <= 510, whose four vertices are the mid-edges of the 1021 x 1021 tables (their first and last rows and
    # columns) and whose edge midpoints are (+-255, +-255), the four sides of an isolated pixel; the tables' corners
    # cannot occur
    assert {(510, 0), (-510, 0), (0, 510), (0, -510)} <= seen
    assert {(255, 255), (255, -255), (-255, 255), (-255, -255)} <= seen
    assert max(gx * gx + gy * gy for gx, gy in seen) == 510 * 510


@pytest.mark.parametrize("th", [1, 20, 127, 128, 200, 254])
def test_threshold_images_straddle_the_threshold(built, th):
    img, _ = adv.ramp_lattice(th)
    d = adv.ring_differences(img)
    assert (d == th).any() and (d == th + 1).any() and d.max() <= th + 1 + 6
    kps, _ = clib.orb(img, 100000, fast_th=th, nlevels=1, cap=70000)
    strong = ((d > th).sum(0) == 16).sum()    # pixels th + 1 (or more) above their whole ring
    print(f"th {th}: {len(kps)} corners of score {np.unique(kps['response']).tolist()}, {strong} full-ring pixels")
    assert len(kps) > 50 and kps["response"].min() == th
    assert len(clib.orb(adv.ramp(th)[0], 800, fast_th=max(th, 1))[0]) == 0


# ---- the indices the LSD kernels form -----------------------------------------------------------------------------------
def lsd_working_image(img, scale):
    """The image LSD takes gradients of: the input at scale 1, else Gaussian blur (sigma 0.6 / scale) + linear resize."""
    if scale == 1.0:
        return img
    h, w = img.shape
    sigma = 0.6 / scale if scale < 1 else 0.6
    ksize = 1 + 2 * int(np.ceil(sigma * np.sqrt(6 * np.log(10))))
    blurred = clib.gaussian_blur_u8(img, ksize, sigma)
    return clib.resize_linear_exact(blurred, int(np.ceil(w * scale)), int(np.ceil(h * scale)), scale, scale)


@pytest.mark.parametrize("scale", [1.0, 1.2])
def test_lsd_indices_stay_inside_their_tables(built, scale):
    """li inside the 1021 x 1021 tables, gx^2 + gy^2 inside the 23 bits above the 9-bit column of a seed-list entry
    (19 bits suffice), the magnitude bin below n_bins - for every generator and the large capacity images."""
    cases = [(n, i) for n, i, _ in adv.small_cases()]
    cases += [("blobs_512", adv.blobs(11, 5, w=512, h=384)[0]), ("noise_640", adv.noise_dense(640, 480)[0]),
              ("lattice_1280", adv.dot_lattice(4, 4, w=1280, h=720)[0])]
    worst = dict(li_max=0, m2_max=0, bin_max=0)
    for name, img in cases:
        for n_bins in (1024, 1):
            b = adv.lsd_index_bounds(lsd_working_image(img, scale), n_bins=n_bins)
            assert 0 <= b["li_min"] and b["li_max"] < 1021 * 1021, (name, b)
            assert b["m2_max"] <= 2 * 510 * 510 < 1 << 19 and b["col_max"] < 1 << 9, (name, b)
            assert b["bin_max"] <= n_bins - 1, (name, b)
            if n_bins == 1024:
                worst = {k: max(v, b[k]) for k, v in worst.items()}
    print(f"lsd_scale {scale}: largest li {worst['li_max']} of {1021 * 1021 - 1}, gx^2+gy^2 {worst['m2_max']}, bin {worst['bin_max']}")
    if scale == 1.0:
        assert worst["li_max"] == 1020 * 1021 + 510 and worst["m2_max"] == 510 * 510 and worst["bin_max"] == 1023
