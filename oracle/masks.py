"""The detectors' mask arguments (plf_orb_masked, plf_detect_lines_masked, plf_set_sequence_mask), restated beside the
unmasked oracles of oracle/cvref.py and oracle/frontend.py.  TEST / BENCH INFRASTRUCTURE ONLY.

orb            cv::ORB::detectAndCompute(img, mask) of cv2 4.13, as oracle/cvref.py orb_cv2 calls it without a mask.
mask_keylines  LSDDetector_custom.cpp:310-322.
detect_lines   oracle/frontend.py detect_lines with mask_keylines where LSDDetectorC::detect applies it: after the end
               point clamp and the min_length filter, before stvo-pl's top-K."""
import numpy as np

from oracle import clib
from oracle.cvref import KP_DTYPE


def orb(img, mask, nfeatures=800, scale_factor=1.2, nlevels=4, edge_th=19, wta_k=2, patch=31, fast_th=20):
    """cv::ORB::create(...)->detectAndCompute(img, mask), in canonical (octave, y, x) order.  mask: u8 [h, w]."""
    import cv2
    o = cv2.ORB_create(int(nfeatures), float(scale_factor), int(nlevels), int(edge_th), 0, int(wta_k),
                       cv2.ORB_FAST_SCORE, int(patch), int(fast_th))
    kps, desc = o.detectAndCompute(img, np.ascontiguousarray(mask, np.uint8))
    out = np.zeros(len(kps), KP_DTYPE)
    for i, k in enumerate(kps):
        out[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, k.class_id)
    if len(kps) == 0:
        return out, np.zeros((0, 32), np.uint8)
    order = np.lexsort((out["x"], out["y"], out["octave"]))
    return out[order], np.ascontiguousarray(desc[order])


def mask_keylines(kl, mask):
    """LSDDetector_custom.cpp:310-322: after the end point clamp and the min_length filter (which numbered class_id), a
    KeyLine is deleted when mask[(int) startPointY][(int) startPointX] == 0 and mask[(int) endPointY][(int) endPointX]
    == 0 ((int): truncation; the clamped end points lie in the image).  The survivors keep their class_id."""
    mask = np.asarray(mask)
    if mask.ndim != 2 or mask.dtype != np.uint8:
        raise ValueError("mask must be a u8 [h, w] array")   # LSDDetectorC::detect throws (:220-221)
    t = lambda v: np.trunc(v.astype(np.float64)).astype(np.int64)
    s = mask[t(kl["startPointY"]), t(kl["startPointX"])]
    e = mask[t(kl["endPointY"]), t(kl["endPointX"])]
    return kl[(s != 0) | (e != 0)].copy()


def detect_lines(img, mask, lsd_nfeatures=300, min_line_length=0.025, lsd_kwargs=None):
    """oracle/frontend.py detect_lines with LSDDetectorC::detect's mask: KeyLines, mask_keylines, then the top-K of the
    survivors (class_id = rank), then LBD."""
    h, w = img.shape
    if np.shape(mask) != (h, w):
        raise ValueError("mask must have the image's size")   # LSDDetectorC::detect throws (:220-221)
    segs = clib.lsd(img, **(lsd_kwargs or {}))
    kl = mask_keylines(clib.keylines_from_segments(segs, w, h, float(np.float32(min_line_length)) * min(w, h)), mask)
    if lsd_nfeatures != 0 and len(kl) > lsd_nfeatures:
        order = np.lexsort((np.arange(len(kl)), -kl["response"].astype(np.float64)))
        kl = kl[order[:lsd_nfeatures]].copy()
        kl["class_id"] = np.arange(lsd_nfeatures, dtype=np.int32)
    desc = clib.lbd_compute(img, kl) if len(kl) else np.zeros((0, 32), np.uint8)
    return kl, desc
