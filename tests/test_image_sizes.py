"""CPU tests of several image sizes per batched context (plf_set_image_sizes, plf_batch_upload_sized,
plf_batch_device_layout, plf_get_image_geometry): the header declares the calls and the library exports them, the binding
refuses shapes of no accepted size before it calls the library and routes the others to the right upload, and what the
library derives from each size (ORB level sizes, LSD scaled size, windowed-matcher grid scale) is what cv2 and the
oracle derive."""
import ctypes as C
import re
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import frontend as ofe

ROOT = Path(__file__).resolve().parent.parent

# the reference's KITTI calibrations (kitti00-02, kitti03, kitti04-10), EuRoC, and sizes that move the 16-byte pitch and
# the FAST (64), blur (62 / 64) and LSD segment (512) tile counts against 1242 x 375
SIZES = [(1241, 376), (1242, 375), (1226, 370), (752, 480), (1280, 384), (640, 200), (1025, 377), (513, 300), (1600, 1200)]


def test_symbols(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"plf_status plf_set_image_sizes\(plf_ctx\* ctx, int n, const int32_t\* wh\);", hdr)
    assert re.search(r"plf_status plf_batch_upload_sized\(plf_ctx\* ctx, int B, int w, int h, const uint8_t\* left, "
                     r"const uint8_t\* right, int stride,\s+int channels\);", hdr)
    assert re.search(r"plf_status plf_batch_device_layout\(plf_ctx\* ctx, int\* w, int\* h, int\* pitch\);", hdr)
    assert re.search(r"plf_status plf_get_image_geometry\(const plf_params\* params, int w, int h, plf_image_geometry\* out\);",
                     hdr)
    lib = plf.load_library()
    for name in ("plf_set_image_sizes", "plf_batch_upload_sized", "plf_batch_device_layout", "plf_get_image_geometry"):
        assert hasattr(lib, name), name
    assert callable(plf.Frontend.set_image_sizes) and callable(plf.image_geometry)
    # NULL context: PLF_ERR_INVALID, without a device
    assert lib.plf_set_image_sizes(None, 0, None) == -1
    assert lib.plf_batch_upload_sized(None, 1, 1242, 375, None, None, 1242, 1) == -1
    assert lib.plf_batch_device_layout(None, None, None, None) == -1
    assert lib.plf_get_image_geometry(None, 1242, 375, None) == -1


def orb_levels(w, h, scale_factor=1.2, nlevels=4):
    """cv::ORB's level sizes: Size(cvRound(w * (1 / scale)), cvRound(h * (1 / scale))), scale = float(scaleFactor^l),
    as oracle/orb.c restates them (float arithmetic, round half to even)."""
    out = []
    for l in range(nlevels):
        inv = np.float32(1.0) / np.float32(float(np.float32(scale_factor)) ** l)
        out.append((int(np.rint(np.float32(w) * inv)), int(np.rint(np.float32(h) * inv))))
    return out


@pytest.mark.parametrize("w,h", SIZES)
def test_geometry_matches_cv2_and_oracle(built, w, h):
    import plslam_b200 as plf
    g = plf.image_geometry(w, h)
    assert g["pitch"] == (w + 15) // 16 * 16
    assert g["orb_levels"] == orb_levels(w, h)
    # the LSD resample: cv::resize(img, Size(), scale, scale, INTER_LINEAR_EXACT) inside createLineSegmentDetector
    img = np.zeros((h, w), np.uint8)
    sh, sw = cv2.resize(img, None, fx=1.2, fy=1.2, interpolation=cv2.INTER_LINEAR_EXACT).shape
    assert g["lsd_size"] == (sw, sh)
    assert g["grid_scale"] == ofe.grid_scales({"width": w, "height": h})


def test_geometry_follows_parameters(built):
    import plslam_b200 as plf
    p = plf.default_params()
    p.orb_nlevels, p.orb_scale_factor, p.lsd_scale = 8, 1.3, 1.0
    g = plf.image_geometry(1226, 370, p)
    assert g["orb_levels"] == orb_levels(1226, 370, 1.3, 8)
    assert g["lsd_size"] == (1226, 370)


@pytest.mark.parametrize("w,h", [(70, 200), (0, 375), (1242, -1), (4096, 375)])
def test_geometry_refuses_what_the_pipeline_refuses(built, w, h):
    import plslam_b200 as plf
    with pytest.raises(plf.PlfError, match="plf_get_image_geometry"):
        plf.image_geometry(w, h)


class _Recorder:
    """A stand-in library: every call is recorded and succeeds."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return 0
        return call


def _frontend(sizes):
    import plslam_b200 as plf
    fe = plf.Frontend.__new__(plf.Frontend)
    fe.lib = _Recorder()
    fe._ctx = C.c_void_p()
    fe.camera = plf.plf_camera(**plf.KITTI_CAMERA)
    fe.limits = plf.default_limits()
    fe.image_sizes = list(sizes)
    return fe


@pytest.mark.parametrize("shape", [(2, 370, 1242), (2, 375, 1226), (2, 480, 752, 3), (2, 375, 1242, 2), (375, 1241)])
def test_binding_refuses_other_shapes_before_the_library(built, shape):
    import plslam_b200 as plf
    fe = _frontend([(1226, 370)])
    a = np.zeros(shape, np.uint8)
    for call in (lambda: fe.batch_upload(a, a), lambda: fe.process_batch(a, a, seq=[0] * (a.shape[0] if a.ndim > 2 else 1))):
        with pytest.raises(plf.PlfError):
            call()
    assert fe.lib.calls == []
    b = np.zeros((2, 375, 1242), np.uint8)
    with pytest.raises(plf.PlfError):
        fe.batch_upload(b, b[:1])
    assert fe.lib.calls == []


def test_binding_routes_each_size(built):
    fe = _frontend([(1226, 370), (1241, 376)])
    grey = np.zeros((2, 370, 1226), np.uint8)
    fe.batch_upload(grey, grey)
    name, args = fe.lib.calls[-1]
    assert name == "plf_batch_upload_sized" and args[1:4] == (2, 1226, 370) and args[6:] == (1226, 1)
    bgr = np.zeros((3, 376, 1241, 3), np.uint8)
    fe.batch_upload(bgr, bgr)
    name, args = fe.lib.calls[-1]
    assert name == "plf_batch_upload_sized" and args[1:4] == (3, 1241, 376) and args[6:] == (3 * 1241, 3)
    one = np.zeros((370, 1226, 4), np.uint8)   # one BGRA pair
    fe.batch_upload(one, one)
    assert fe.lib.calls[-1][0] == "plf_batch_upload_sized" and fe.lib.calls[-1][1][-1] == 4
    ctx = np.zeros((1, 375, 1242), np.uint8)
    fe.batch_upload(ctx, ctx)
    assert fe.lib.calls[-1][0] == "plf_batch_upload"
    fe.batch_upload_raw(4, 1, 2, size=(1226, 370))
    name, args = fe.lib.calls[-1]
    assert name == "plf_batch_upload_sized" and args[1:4] == (4, 1226, 370) and args[-2:] == (1226, 1)
    fe.batch_upload_raw(4, 1, 2)
    assert fe.lib.calls[-1][0] == "plf_batch_upload"
    # process_batch at another size goes through the sized upload, the run and the download
    fe.lib.calls.clear()
    try:
        fe.process_batch(grey, grey)
    except Exception:
        pass   # the recorder's download leaves zeroed results; only the calls matter here
    assert [c[0] for c in fe.lib.calls][:2] == ["plf_batch_upload_sized", "plf_batch_run_sequences"]
