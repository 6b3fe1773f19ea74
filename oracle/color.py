"""cv::cvtColor(src, dst, COLOR_BGR2GRAY) (and COLOR_BGRA2GRAY) of an 8-bit image as OpenCV 4 computes it: what
LSDDetectorC::detectImpl, BinaryDescriptor::computeImpl and ORB::detectAndCompute do to a colour image, and what k_color
(csrc/pipeline.cu) restates on the device.

gray = (3735 B + 19235 G + 9798 R + 2^14) >> 15: the coefficients 0.114, 0.587, 0.299 in 15-bit fixed point (they sum to
2^15).  OpenCV 3's (1868, 9617, 4899) >> 14 gives other values for some colours; this project follows OpenCV 4
(DESIGN.md section 8).  A fourth channel (alpha) is ignored.

stvo-pl's dataset reader remaps the image it read, so for a colour camera the remap comes first, per channel, and the
conversion after; the two orders give different images."""
import numpy as np

from oracle import rectify

COEFS = (3735, 19235, 9798)   # B, G, R
SHIFT = 15


def bgr_to_gray(img):
    """img uint8 [..., 3 | 4] (BGR or BGRA) -> uint8 [...]."""
    img = np.asarray(img, np.uint8)
    assert img.shape[-1] in (3, 4), img.shape
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    return ((COEFS[0] * b + COEFS[1] * g + COEFS[2] * r + (1 << (SHIFT - 1))) >> SHIFT).astype(np.uint8)


def remap(img, map1, map2):
    """cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a colour image: rectify.remap on each channel with the same maps."""
    img = np.asarray(img, np.uint8)
    return np.stack([rectify.remap(img[..., c], map1, map2) for c in range(img.shape[-1])], axis=-1)


def remap_to_gray(img, map1, map2):
    """What a rectified colour sequence extracts from: the remapped colour image, converted."""
    return bgr_to_gray(remap(img, map1, map2))
