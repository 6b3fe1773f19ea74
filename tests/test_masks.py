"""CPU tests of the detector masks' oracles (plf_set_sequence_mask, plf_orb_masked, plf_detect_lines_masked).

- oracle/masks.py mask_keylines against a literal transcription of LSDDetector_custom.cpp:310-322 (the erase loop),
  on random masks and KeyLines with end points on the clamp, with exactly one end point allowed, and with fractional
  coordinates that truncate onto a masked pixel; and detect_lines' mask position (before the top-K).
- cv2's detectAndCompute(img, mask) keeps exactly the unmasked run's keypoints (no retainBest cut) that sit on a
  non-zero pixel of the mask pyramid the library builds: level 0 the mask with every non-zero value 255, level l the
  INTER_LINEAR_EXACT resize of level l-1 thresholded at 254."""
import numpy as np
import pytest

from oracle import clib, cvref
from oracle import frontend as ofe
from oracle import masks as om

cv2 = pytest.importorskip("cv2")


def transcription(kl, mask):
    """LSDDetector_custom.cpp:310-322 as written: erase while walking, (int) truncation of float end points."""
    keylines = list(kl)
    k = 0
    while k < len(keylines):
        e = keylines[k]
        if (mask[int(float(e["startPointY"])), int(float(e["startPointX"]))] == 0
                and mask[int(float(e["endPointY"])), int(float(e["endPointX"]))] == 0):
            del keylines[k]
            k -= 1
        k += 1
    return np.array(keylines, kl.dtype) if keylines else kl[:0]


def random_keylines(rng, w, h, n):
    segs = rng.uniform(-20, [w + 20, h + 20, w + 20, h + 20], (n, 4)).astype(np.float32)
    segs[: n // 8, 0] = w + 5          # clamped onto x = w - 1
    segs[n // 8: n // 4, 1] = -3.0     # clamped onto y = 0
    segs[n // 4: n // 3, 2] = w - 1 + 0.999   # stays below w: truncates onto w - 1
    return clib.keylines_from_segments(segs, w, h, 5.0)


@pytest.mark.parametrize("seed", range(6))
def test_keyline_rule_matches_transcription(seed):
    rng = np.random.default_rng(seed)
    w, h = 97 + seed, 61 + 2 * seed
    kl = random_keylines(rng, w, h, 400)
    for density in (0.0, 0.3, 0.7, 1.0):
        mask = (rng.random((h, w)) < density).astype(np.uint8) * rng.integers(1, 256, (h, w)).astype(np.uint8)
        got, ref = om.mask_keylines(kl, mask), transcription(kl, mask)
        assert got.tobytes() == ref.tobytes()
        assert np.array_equal(got["class_id"], ref["class_id"])   # the survivors keep their numbering


def test_keyline_rule_edges():
    w, h = 40, 30
    mask = np.zeros((h, w), np.uint8)
    mask[:, 20:] = 1
    segs = np.array([[5.0, 5.0, 30.0, 5.0],      # one end point allowed: kept although it crosses the masked half
                     [5.0, 5.0, 15.0, 20.0],     # both masked: deleted
                     [19.99, 3.0, 19.5, 25.0],   # fractional: both truncate onto column 19 (masked): deleted
                     [20.0, 3.0, 2.0, 25.0],     # start exactly on the first allowed column: kept
                     [60.0, -9.0, 60.0, 40.0]],  # clamped onto x = w - 1 (allowed): kept
                    np.float32)
    kl = clib.keylines_from_segments(segs, w, h, 1.0)
    assert len(kl) == 5
    got = om.mask_keylines(kl, mask)
    assert list(got["class_id"]) == [0, 3, 4]
    assert got.tobytes() == transcription(kl, mask).tobytes()


def test_detect_lines_masks_before_the_top_k():
    """The top-K ranks the survivors: a mask that drops the longest lines lets shorter ones in, numbered by rank."""
    from oracle import synth
    cam = dict(width=320, height=240, fx=300.0, fy=300.0, cx=160.0, cy=120.0, b=0.3)
    img = next(iter(synth.stream(cam, 1, world=synth.World(seed=1, n_quads=60, n_segs=40))))[0]
    full, _ = ofe.detect_lines(img, 0)
    mask = np.full(img.shape, 255, np.uint8)
    mask[:, : img.shape[1] // 2] = 0
    kept = om.mask_keylines(full, mask)
    K = max(1, len(kept) // 2)
    got, _ = om.detect_lines(img, mask, K)
    order = np.lexsort((np.arange(len(kept)), -kept["response"].astype(np.float64)))
    ref = kept[order[:K]].copy()
    ref["class_id"] = np.arange(K)
    assert got.tobytes() == ref.tobytes()
    with pytest.raises(ValueError):
        om.detect_lines(img, mask[:-1], K)


def mask_pyramid(mask, nlevels, scale=1.2):
    """The library's mask pyramid (plf_orb_mask_build): level 0 = 255 where the mask is non-zero, level l =
    threshold(resize(level l-1, INTER_LINEAR_EXACT), 254, TOZERO)."""
    h, w = mask.shape
    out = [np.where(mask != 0, 255, 0).astype(np.uint8)]
    for l in range(1, nlevels):
        s = float(np.float32(scale ** l))
        size = (int(np.round(w / s)), int(np.round(h / s)))
        m = cv2.resize(out[-1], size, interpolation=cv2.INTER_LINEAR_EXACT)
        out.append(cv2.threshold(m, 254, 0, cv2.THRESH_TOZERO)[1])
    return out


def masks_of(h, w, rng):
    yy, xx = np.mgrid[:h, :w]
    return {"half": np.where(xx < w // 2, 0, 255), "checker4": np.where((yy // 4 + xx // 4) % 2 == 0, 255, 0),
            "values_1_254": np.where(xx < w // 2, 1, 254), "column": np.where(xx == w // 3, 255, 0),
            "values_0_127_254": rng.integers(0, 3, (h, w)) * 127}


@pytest.mark.parametrize("shape", [(375, 620), (480, 752)])
@pytest.mark.parametrize("nlevels", [1, 4, 8])
def test_orb_keypoints_are_the_unmasked_ones_on_the_mask_pyramid(shape, nlevels):
    h, w = shape
    rng = np.random.default_rng(7)
    img = cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (0, 0), 1.5)
    N = 200000   # every level's quota above its corner count: retainBest cuts nothing
    full, _ = cvref.orb_cv2(img, N, 1.2, nlevels)
    for kind, mask in masks_of(h, w, rng).items():
        mask = mask.astype(np.uint8)
        got, _ = om.orb(img, mask, N, 1.2, nlevels)
        pyr = mask_pyramid(mask, nlevels)
        on = []
        for k in full:
            sc = np.float32(1.2 ** int(k["octave"]))
            on.append(pyr[k["octave"]][int(np.round(k["y"] / sc)), int(np.round(k["x"] / sc))] != 0)
        ref = full[np.array(on, bool)]
        assert got[["x", "y", "octave"]].tobytes() == ref[["x", "y", "octave"]].tobytes(), kind
        if kind == "values_1_254":   # every value allowed on every level, as 255 would be
            assert len(got) == len(full)
