"""cv::remap(src, dst, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) of an 8-bit image with CV_16SC2 / CV_16UC1 maps:
what stvo-pl's dataset reader does to each raw image before insertStereoPair, and what k_rectify (csrc/pipeline.cu)
restates on the device.

map1[y, x] = (sx, sy) is the integer tap, map2[y, x] & 1023 = 32 fy + fx the index into a 32 x 32 table of fixed-point
bilinear weights.  Each weight is cvRound(w * 32768) of the float product of the 1-D weights (1 - t, t), t = k / 32, with
the rounding excess put back on the largest weight so the four sum to 32768; the output is (sum w_i p_i + 2^14) >> 15.
Taps outside the image read 0 (the constant border)."""
import numpy as np

COEF_BITS = 15
TAB_SIZE = 32


def weight_table():
    """[1024, 4] int32: the weights of the taps (x, y), (x+1, y), (x, y+1), (x+1, y+1) for map2 = 32 fy + fx."""
    t = (np.arange(TAB_SIZE, dtype=np.float32) / np.float32(TAB_SIZE)).astype(np.float32)
    one = np.stack([np.float32(1) - t, t], axis=1).astype(np.float32)          # [32][2] 1-D weights
    tab = np.zeros((TAB_SIZE * TAB_SIZE, 4), np.int32)
    for fy in range(TAB_SIZE):
        for fx in range(TAB_SIZE):
            v = np.array([one[fy, a] * one[fx, b] for a in range(2) for b in range(2)], np.float32)
            w = np.rint(v * np.float32(1 << COEF_BITS)).astype(np.int32)     # cvRound: half to even
            diff = int(w.sum()) - (1 << COEF_BITS)
            if diff:
                w[int(np.argmax(w))] -= diff
            tab[fy * TAB_SIZE + fx] = w
    return tab


_TAB = weight_table()


def remap(img, map1, map2):
    """img uint8 [h, w]; map1 int16 [H, W, 2] (x, y); map2 uint16 [H, W].  Returns uint8 [H, W]."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    sx = map1[..., 0].astype(np.int64)
    sy = map1[..., 1].astype(np.int64)
    wt = _TAB[np.asarray(map2).astype(np.int64) & (TAB_SIZE * TAB_SIZE - 1)]

    def tap(x, y):
        inside = (x >= 0) & (x < w) & (y >= 0) & (y < h)
        return np.where(inside, img[np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)], 0).astype(np.int64)

    acc = (wt[..., 0] * tap(sx, sy) + wt[..., 1] * tap(sx + 1, sy) + wt[..., 2] * tap(sx, sy + 1) +
           wt[..., 3] * tap(sx + 1, sy + 1))
    return ((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS).astype(np.uint8)


# EuRoC's stereo calibration (config/dataset_params/euroc_params.yaml of pl-slam: cam0 Kl, Dl; cam1 Kr, Dr; R, t from
# the left to the right camera), for the maps a caller builds.
EUROC = dict(
    size=(752, 480),
    Kl=(458.654, 457.296, 367.215, 248.375), Dl=(-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05),
    Kr=(457.587, 456.134, 379.999, 255.238), Dr=(-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05),
    R=(9.99997256e-01, 2.31206719e-03, 3.76008102e-04, -2.31713572e-03, 9.99898049e-01, 1.40898358e-02,
       -3.43393121e-04, -1.40906685e-02, 9.99900663e-01),
    t=(-0.11007381, 0.00039912, -0.0008537))


def _stereo_rectify(calib, size):
    import cv2
    w0, h0 = calib["size"]
    w, h = size or (w0, h0)
    sx, sy = w / w0, h / h0

    def K(k):
        return np.array([[k[0] * sx, 0, k[2] * sx], [0, k[1] * sy, k[3] * sy], [0, 0, 1]], np.float64)

    Kl, Kr = K(calib["Kl"]), K(calib["Kr"])
    Dl, Dr = np.array(calib["Dl"], np.float64), np.array(calib["Dr"], np.float64)
    R = np.array(calib["R"], np.float64).reshape(3, 3)
    t = np.array(calib["t"], np.float64)
    R1, R2, P1, P2, _, _, _ = cv2.stereoRectify(Kl, Dl, Kr, Dr, (w, h), R, t, flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)
    return (w, h), ((Kl, Dl, R1, P1), (Kr, Dr, R2, P2))


def stereo_maps(calib=EUROC, size=None):
    """((map1_l, map2_l), (map1_r, map2_r), camera dict) of a calibration through cv2.stereoRectify (CALIB_ZERO_DISPARITY,
    alpha 0) and cv2.initUndistortRectifyMap(..., CV_16SC2), at `size` (w, h; default the calibration's, the intrinsics
    scaled with it).  The camera is P1's fx, fy, cx, cy with the baseline -P2[0, 3] / P2[0, 0]."""
    import cv2
    (w, h), sides = _stereo_rectify(calib, size)
    left, right = (cv2.initUndistortRectifyMap(K, D, Rr, P, (w, h), cv2.CV_16SC2) for K, D, Rr, P in sides)
    P1, P2 = sides[0][3], sides[1][3]
    cam = dict(width=w, height=h, fx=float(P1[0, 0]), fy=float(P1[1, 1]), cx=float(P1[0, 2]), cy=float(P1[1, 2]),
               b=float(-P2[0, 3] / P2[0, 0]))
    return left, right, cam


def distort(rect_l, rect_r, calib=EUROC):
    """Raw (distorted, unrectified) images of a rectified pair rendered with stereo_maps' camera at the images' size:
    each raw pixel samples the rectified image where cv2.undistortPoints puts it.  Test and benchmark input only."""
    import cv2
    h, w = rect_l.shape
    _, sides = _stereo_rectify(calib, (w, h))
    y, x = np.mgrid[0:h, 0:w]
    pts = np.stack([x, y], axis=-1).reshape(-1, 1, 2).astype(np.float64)
    out = []
    for img, (K, D, Rr, P) in zip((rect_l, rect_r), sides):
        u = cv2.undistortPoints(pts, K, D, R=Rr, P=P).reshape(h, w, 2).astype(np.float32)
        out.append(cv2.remap(img, u[..., 0], u[..., 1], cv2.INTER_LINEAR))
    return out[0], out[1]
