"""The per-pair masks of the pair-mask tests (plf_batch_upload_masks): the moving objects a segmentation network would mask
out frame by frame, a static hood mask to AND them with, and two sparse masks whose AND gives another mask pyramid than
the AND of their pyramids."""
import numpy as np


def moving(h, w, i, side, seed=0):
    """255 except a box and a disc that move across the image with frame i (0 inside them, the dynamic objects); the
    right image's objects sit a few pixels of disparity to the left, and a band of the allowed area holds 1s instead of
    255s (any non-zero value allows)."""
    yy, xx = np.mgrid[:h, :w]
    shift = 0 if side == 0 else max(2, w // 60)
    bx = int(((0.08 + 0.13 * i + 0.05 * seed) % 0.8) * w) - shift
    by = int(0.2 * h)
    box = (xx >= bx) & (xx < bx + w // 6) & (yy >= by) & (yy < by + h // 3)
    cx, cy = int(((0.85 - 0.11 * i - 0.07 * seed) % 1.0) * w) - shift, int(0.62 * h)
    disc = (xx - cx) ** 2 + (yy - cy) ** 2 < (h // 6) ** 2
    out = np.full((h, w), 255, np.uint8)
    out[(yy // 16) % 5 == 4] = 1
    out[box | disc] = 0
    return out


def hood(h, w):
    """A static sequence mask: the bottom fifth (a vehicle's hood) and a burned-in timestamp masked out."""
    m = np.full((h, w), 255, np.uint8)
    m[int(0.8 * h):] = 0
    m[:max(12, h // 20), :w // 4] = 0
    return m


# Two masks of isolated 0s on interleaved grids, with a pixel of the 4-level KITTI-shape pyramid of their AND masked that
# neither of their pyramids masks (a level-3 pixel two of whose four resize taps weigh at most 128 / 65536 each: either
# 0 alone rounds back to 255, both together do not).
def sparse_pair(h, w):
    yy, xx = np.mgrid[:h, :w]
    s = np.where((xx % 5 == 0) & (yy % 5 == 0), 0, 255).astype(np.uint8)
    p = np.where((xx % 5 == 1) & (yy % 5 == 1), 0, 255).astype(np.uint8)
    return s, p


def mask_pyramid(mask, nlevels, scale=1.2):
    """The mask pyramid cv2 4.13's detectAndCompute(img, mask) applies (tests/test_masks.py): level 0 = 255 where the
    mask is non-zero, level l = threshold(resize(level l-1, INTER_LINEAR_EXACT), 254, TOZERO)."""
    import cv2
    h, w = mask.shape
    out = [np.where(mask != 0, 255, 0).astype(np.uint8)]
    for l in range(1, nlevels):
        s = float(np.float32(scale ** l))
        m = cv2.resize(out[-1], (int(np.round(w / s)), int(np.round(h / s))), interpolation=cv2.INTER_LINEAR_EXACT)
        out.append(cv2.threshold(m, 254, 0, cv2.THRESH_TOZERO)[1])
    return out


def streams(cam, nseq, n):
    """nseq rendered stereo streams of n pairs at camera cam, the frames the pair-mask tests run."""
    from oracle import synth
    return [[f[:2] for f in synth.stream(cam, n, world=synth.World(seed=30 + s), seed=40 + s, step=0.1)] for s in range(nseq)]
