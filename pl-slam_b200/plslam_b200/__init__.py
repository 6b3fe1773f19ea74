"""ctypes binding of libplslam_b200.so (the C ABI in include/plslam_b200.h).

Thin by design: numpy arrays in, numpy arrays out, every call goes straight through the C ABI to the
CUDA kernels.  There is NO CPU fallback: if the shared library is missing or no CUDA device is
present, construction raises.  Used by tests/, bench.py and __graft_entry__.py.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

_PKG_DIR = Path(__file__).resolve().parent.parent  # pl-slam_b200/
REPO_ROOT = _PKG_DIR.parent
LIB_PATH = _PKG_DIR / "lib" / "libplslam_b200.so"

DESC_BYTES = 32


class PlfError(RuntimeError):
    pass


class plf_params(C.Structure):
    _fields_ = [
        ("has_points", C.c_int), ("has_lines", C.c_int), ("best_lr_matches", C.c_int),
        ("max_dist_epip", C.c_float), ("min_disp", C.c_float), ("min_ratio_12_p", C.c_float),
        ("line_sim_th", C.c_float), ("stereo_overlap_th", C.c_float), ("f2f_overlap_th", C.c_float),
        ("min_line_length", C.c_float), ("line_horiz_th", C.c_float), ("min_ratio_12_l", C.c_float),
        ("ls_min_disp_ratio", C.c_float),
        ("homog_th", C.c_double),
        ("min_features", C.c_int), ("max_iters", C.c_int), ("max_iters_ref", C.c_int),
        ("min_error", C.c_double), ("min_error_change", C.c_double), ("inlier_k", C.c_double),
        ("orb_nfeatures", C.c_int), ("orb_scale_factor", C.c_float),
        ("orb_nlevels", C.c_int), ("orb_edge_th", C.c_int), ("orb_wta_k", C.c_int),
        ("orb_score", C.c_int), ("orb_patch_size", C.c_int), ("orb_fast_th", C.c_int),
        ("lsd_nfeatures", C.c_int), ("lsd_refine", C.c_int),
        ("lsd_scale", C.c_double), ("lsd_sigma_scale", C.c_double), ("lsd_quant", C.c_double),
        ("lsd_ang_th", C.c_double), ("lsd_log_eps", C.c_double), ("lsd_density_th", C.c_double),
        ("lsd_n_bins", C.c_int),
        ("matching_strategy", C.c_int), ("matching_s_ws", C.c_int), ("matching_f2f_ws", C.c_int),
        ("min_pt_matches", C.c_int), ("min_ls_matches", C.c_int),
    ]


class plf_camera(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("b", C.c_double)]


class plf_limits(C.Structure):
    _fields_ = [("max_batch", C.c_int), ("max_keypoints", C.c_int), ("max_segments", C.c_int),
                ("max_lines", C.c_int)]


class plf_lba_opts(C.Structure):
    _fields_ = [("lambda_", C.c_double), ("lambda_k", C.c_double), ("max_iters", C.c_int), ("homog_th", C.c_double),
                ("min_error", C.c_double), ("min_error_change", C.c_double), ("ref_quirks", C.c_int)]


class plf_lba_problem(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int), ("n_fixed", C.c_int),
                ("kf_pose", C.c_void_p), ("pt", C.c_void_p), ("ls", C.c_void_p), ("fixed_T", C.c_void_p),
                ("n_pt_obs", C.c_int), ("pt_obs_lm", C.c_void_p), ("pt_obs_kf", C.c_void_p), ("pt_obs_xy", C.c_void_p),
                ("n_ls_obs", C.c_int), ("ls_obs_lm", C.c_void_p), ("ls_obs_kf", C.c_void_p), ("ls_obs_le", C.c_void_p),
                ("pt_moved", C.c_void_p), ("ls_moved", C.c_void_p)]


class plf_lba_result(C.Structure):
    _fields_ = [("iters", C.c_int), ("err", C.c_double), ("lambda_", C.c_double)]


class plf_grid_window(C.Structure):
    _fields_ = [("width_lo", C.c_int), ("width_hi", C.c_int), ("height_lo", C.c_int), ("height_hi", C.c_int)]


class plf_gn_opts(C.Structure):
    _fields_ = [("homog_th", C.c_double), ("max_iters", C.c_int), ("max_iters_ref", C.c_int),
                ("eps_err", C.c_double), ("eps_change", C.c_double), ("eps_step", C.c_double)]


class plf_pose_result(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("cov", C.c_double * 36), ("x", C.c_double * 6),
                ("err", C.c_double), ("iters1", C.c_int), ("iters2", C.c_int),
                ("n_inliers_pt", C.c_int), ("n_inliers_ls", C.c_int)]


class plf_frame_result(C.Structure):
    _fields_ = [("DT", C.c_double * 16), ("DT_cov", C.c_double * 36), ("err", C.c_double), ("status", C.c_int),
                ("n_kp_l", C.c_int), ("n_kp_r", C.c_int), ("n_lines_l", C.c_int), ("n_lines_r", C.c_int),
                ("n_stereo_pt", C.c_int), ("n_stereo_ls", C.c_int), ("n_matched_pt", C.c_int),
                ("n_matched_ls", C.c_int), ("n_inliers_pt", C.c_int), ("n_inliers_ls", C.c_int),
                ("iters1", C.c_int), ("iters2", C.c_int)]


class plf_frame_view(C.Structure):
    _fields_ = [("cap_pt", C.c_int), ("cap_ls", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int),
                ("pt_pl", C.c_void_p), ("pt_disp", C.c_void_p), ("pt_P", C.c_void_p), ("pt_octave", C.c_void_p),
                ("pdesc", C.c_void_p), ("ls_spl", C.c_void_p), ("ls_epl", C.c_void_p), ("ls_sdisp", C.c_void_p),
                ("ls_edisp", C.c_void_p), ("ls_sP", C.c_void_p), ("ls_eP", C.c_void_p), ("ls_le", C.c_void_p),
                ("ls_angle", C.c_void_p), ("ldesc", C.c_void_p)]


class plf_match_view(C.Structure):
    _fields_ = [("cap_pt", C.c_int), ("cap_ls", C.c_int), ("n_pt", C.c_int), ("n_ls", C.c_int),
                ("P", C.c_void_p), ("pl_obs", C.c_void_p), ("inlier_pt", C.c_void_p), ("sP", C.c_void_p),
                ("eP", C.c_void_p), ("le_obs", C.c_void_p), ("inlier_ls", C.c_void_p)]


class plf_lc_params(C.Structure):
    _fields_ = [("lc_res", C.c_double), ("lc_unc", C.c_double), ("lc_inl", C.c_double), ("lc_trs", C.c_double),
                ("lc_rot", C.c_double), ("lc_inlier_ratio", C.c_double)]


class plf_lc_keyframe(C.Structure):
    _fields_ = [("n_pt", C.c_int), ("n_ls", C.c_int), ("pdesc", C.c_void_p), ("P", C.c_void_p), ("pl", C.c_void_p),
                ("ldesc", C.c_void_p), ("sP", C.c_void_p), ("eP", C.c_void_p), ("le", C.c_void_p)]


class plf_lc_result(C.Structure):
    _fields_ = [("accepted", C.c_int), ("estimated", C.c_int), ("common_pt", C.c_int), ("common_ls", C.c_int),
                ("n_pt", C.c_int), ("n_ls", C.c_int), ("inl_ratio_pt", C.c_double), ("inl_ratio_ls", C.c_double),
                ("err", C.c_double), ("max_cov_eig", C.c_double), ("ratio_inliers", C.c_double), ("t", C.c_double),
                ("r", C.c_double), ("x_inc", C.c_double * 6), ("pose_inc", C.c_double * 6)]


class plf_kf_match_opts(C.Structure):
    _fields_ = [("fast_matching", C.c_int), ("max_kf_epip_p", C.c_double), ("max_kf_epip_l", C.c_double)]


class plf_local_map(C.Structure):
    _fields_ = [("n_pt", C.c_int), ("pt_X", C.c_void_p), ("pt_desc", C.c_void_p), ("pt_use", C.c_void_p),
                ("n_ls", C.c_int), ("ls_X", C.c_void_p), ("ls_desc", C.c_void_p), ("ls_use", C.c_void_p)]


# the plf_frame_view fields the keyframe matchers read: (name, dtype, columns)
_KF_VIEW_FIELDS = (("pt_pl", np.float64, 2), ("pt_P", np.float64, 3), ("pdesc", np.uint8, 32), ("ls_spl", np.float64, 2),
                   ("ls_epl", np.float64, 2), ("ls_sP", np.float64, 3), ("ls_eP", np.float64, 3), ("ls_le", np.float64, 3),
                   ("ldesc", np.uint8, 32))


def _frame_view(frame, keep):
    """A plf_frame_view over the arrays of a get_frame dict (missing arrays stay NULL; `keep` holds the copies alive)."""
    v = plf_frame_view()
    v.n_pt, v.n_ls = len(frame.get("pdesc", ())), len(frame.get("ldesc", ()))
    for name, dt, cols in _KF_VIEW_FIELDS:
        if name in frame:
            a = np.ascontiguousarray(frame[name], dt).reshape(-1, cols)
            keep.append(a)
            setattr(v, name, a.ctypes.data if a.size else None)
    return v


RESULT_DTYPE = np.dtype([("DT", np.float64, (4, 4)), ("DT_cov", np.float64, (6, 6)), ("err", np.float64),
                         ("status", np.int32), ("n_kp_l", np.int32), ("n_kp_r", np.int32), ("n_lines_l", np.int32),
                         ("n_lines_r", np.int32), ("n_stereo_pt", np.int32), ("n_stereo_ls", np.int32),
                         ("n_matched_pt", np.int32), ("n_matched_ls", np.int32), ("n_inliers_pt", np.int32),
                         ("n_inliers_ls", np.int32), ("iters1", np.int32), ("iters2", np.int32)], align=True)
assert RESULT_DTYPE.itemsize == C.sizeof(plf_frame_result)

RESULT_FIELDS = ["status", "n_kp_l", "n_kp_r", "n_lines_l", "n_lines_r", "n_stereo_pt", "n_stereo_ls", "n_matched_pt",
                 "n_matched_ls", "n_inliers_pt", "n_inliers_ls", "iters1", "iters2"]

KEYLINE_DTYPE = np.dtype([
    ("angle", np.float32), ("class_id", np.int32), ("octave", np.int32),
    ("ptx", np.float32), ("pty", np.float32), ("response", np.float32), ("size", np.float32),
    ("startPointX", np.float32), ("startPointY", np.float32), ("endPointX", np.float32),
    ("endPointY", np.float32), ("sPointInOctaveX", np.float32), ("sPointInOctaveY", np.float32),
    ("ePointInOctaveX", np.float32), ("ePointInOctaveY", np.float32), ("lineLength", np.float32),
    ("numOfPixels", np.int32)])  # == plf_keyline == cv::line_descriptor::KeyLine

KEYPOINT_DTYPE = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                           ("response", np.float32), ("octave", np.int32), ("class_id", np.int32)])  # cv::KeyPoint

_lib = None


def load_library() -> C.CDLL:
    """Loads libplslam_b200.so; raises PlfError (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise PlfError(f"{LIB_PATH} not built: run `make` (or __graft_entry__.build()) first; "
                       "there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    lib.plf_last_error.restype = C.c_char_p
    lib.plf_last_error.argtypes = [C.c_void_p]
    lib.plf_launch_count.restype = C.c_longlong
    lib.plf_launch_count.argtypes = [C.c_void_p]
    lib.plf_stream.restype = C.c_void_p
    lib.plf_stream.argtypes = [C.c_void_p]
    _pi, _pu8 = C.POINTER(C.c_int), C.POINTER(C.c_uint8)
    lib.plf_match_grid_points.argtypes = [C.c_void_p, _pi, _pu8, C.c_int, _pi, _pi, _pu8, C.c_int, C.c_int, C.c_int,
                                          plf_grid_window, C.c_float, C.c_int, C.POINTER(C.c_int32), _pi]
    lib.plf_match_grid_lines.argtypes = [C.c_void_p, _pi, _pu8, C.c_int, _pi, _pi, C.POINTER(C.c_double), _pu8, C.c_int,
                                         C.c_int, C.c_int, plf_grid_window, C.c_float, C.c_double, C.c_int,
                                         C.POINTER(C.c_int32), _pi]
    lib.plf_destroy.restype = None
    lib.plf_destroy.argtypes = [C.c_void_p]
    lib.plf_batch_device_images.restype = C.c_void_p
    lib.plf_batch_device_images.argtypes = [C.c_void_p]
    lib.plf_default_params.restype = None
    lib.plf_default_limits.restype = None
    _lib = lib
    return lib


def default_params() -> plf_params:
    p = plf_params()
    load_library().plf_default_params(C.byref(p))
    return p


def default_limits() -> plf_limits:
    l = plf_limits()
    load_library().plf_default_limits(C.byref(l))
    return l


KITTI_CAMERA = dict(width=1242, height=375, fx=718.856, fy=718.856, cx=607.1928, cy=185.2157,
                    b=0.537165719)  # config/dataset_params/kitti00-02.yaml:2-10
EUROC_CAMERA = dict(width=752, height=480, fx=458.654, fy=457.296, cx=367.215, cy=248.375,
                    b=0.110077842)  # config/dataset_params/euroc_params.yaml:2,8 (pre-rectified)


def _u8(a, shape_tail=None):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


class Frontend:
    """One plf_ctx (one device, one stream).  Mirrors the role of `StereoFrameHandler`
    (app/plslam_dataset.cpp:109) plus the free operators the reference calls on the path."""

    def __init__(self, params: plf_params | None = None, camera: dict | plf_camera | None = None,
                 limits: plf_limits | None = None, device: int = 0, **overrides):
        self.lib = load_library()
        self.params = params if params is not None else default_params()
        for k, v in overrides.items():
            if hasattr(self.params, k):
                setattr(self.params, k, v)
            else:
                raise PlfError(f"unknown parameter {k}")
        if camera is None:
            camera = KITTI_CAMERA
        self.camera = camera if isinstance(camera, plf_camera) else plf_camera(**camera)
        self.limits = limits if limits is not None else default_limits()
        self._ctx = C.c_void_p()
        st = self.lib.plf_create(C.byref(self.params), C.byref(self.camera), C.byref(self.limits),
                                 int(device), C.byref(self._ctx))
        if st != 0:
            raise PlfError(f"plf_create failed ({st}): {self.lib.plf_last_error(None).decode()}")

    # -- plumbing --------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.plf_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, st: int, what: str):
        if st != 0:
            raise PlfError(f"{what} failed ({st}): {self.lib.plf_last_error(self._ctx).decode()}")

    @property
    def launches(self) -> int:
        return int(self.lib.plf_launch_count(self._ctx))

    @property
    def stream(self) -> int:
        return int(self.lib.plf_stream(self._ctx) or 0)

    def sync(self):
        self._check(self.lib.plf_sync(self._ctx), "plf_sync")

    # -- matching --------------------------------------------------------------------------------
    def hamming_knn2(self, d1, d2):
        """cv::BFMatcher(NORM_HAMMING).knnMatch(d1, d2, k=2): returns idx1, dist1, idx2, dist2."""
        d1 = _u8(d1).reshape(-1, DESC_BYTES)
        d2 = _u8(d2).reshape(-1, DESC_BYTES)
        n1, n2 = len(d1), len(d2)
        out = [np.full(n1, -1, np.int32) for _ in range(4)]
        st = self.lib.plf_hamming_knn2(self._ctx, _ptr(d1, C.c_uint8), n1, _ptr(d2, C.c_uint8), n2,
                                       *[_ptr(o, C.c_int32) for o in out])
        self._check(st, "plf_hamming_knn2")
        return tuple(out)

    def match(self, d1, d2, nnr: float, best_lr: bool = True):
        """stvo-pl match(): returns (matches_12 int32[n1], n_matches)."""
        d1 = _u8(d1).reshape(-1, DESC_BYTES)
        d2 = _u8(d2).reshape(-1, DESC_BYTES)
        n1, n2 = len(d1), len(d2)
        m = np.full(n1, -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match(self._ctx, _ptr(d1, C.c_uint8), n1, _ptr(d2, C.c_uint8), n2,
                                C.c_float(nnr), int(bool(best_lr)), _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match")
        return m, cnt.value

    def match_grid_points(self, q_cell, d1, cell_start, cell_items, d2, cols, rows, w, nnr, best_lr=True):
        """stvo-pl matchGrid (points): q_cell int32 [n1,2]; the GridStructure as (cell_start, cell_items), cell (x, y) at
        x*rows + y; w = (width.first, width.second, height.first, height.second)."""
        q = np.ascontiguousarray(q_cell, np.int32).reshape(-1, 2)
        cs = np.ascontiguousarray(cell_start, np.int32); ci = np.ascontiguousarray(cell_items, np.int32)
        d1 = _u8(d1).reshape(-1, DESC_BYTES); d2 = _u8(d2).reshape(-1, DESC_BYTES)
        m = np.full(len(q), -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match_grid_points(self._ctx, _ptr(q, C.c_int), _ptr(d1, C.c_uint8), len(q), _ptr(cs, C.c_int),
                                            _ptr(ci, C.c_int), _ptr(d2, C.c_uint8), len(d2), int(cols), int(rows),
                                            plf_grid_window(*[int(v) for v in w]), C.c_float(nnr), int(bool(best_lr)),
                                            _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match_grid_points")
        return m, cnt.value

    def match_grid_lines(self, q_line, d1, cell_start, cell_items, t_dir, d2, cols, rows, w, nnr, line_sim_th, best_lr=True):
        """stvo-pl matchGrid (lines): q_line int32 [n1,4] end-point cells, grid as above, directions2 f64 [n2,2]."""
        q = np.ascontiguousarray(q_line, np.int32).reshape(-1, 4)
        cs = np.ascontiguousarray(cell_start, np.int32); ci = np.ascontiguousarray(cell_items, np.int32)
        td = np.ascontiguousarray(t_dir, np.float64).reshape(-1, 2)
        d1 = _u8(d1).reshape(-1, DESC_BYTES); d2 = _u8(d2).reshape(-1, DESC_BYTES)
        m = np.full(len(q), -1, np.int32)
        cnt = C.c_int(0)
        st = self.lib.plf_match_grid_lines(self._ctx, _ptr(q, C.c_int), _ptr(d1, C.c_uint8), len(q), _ptr(cs, C.c_int),
                                           _ptr(ci, C.c_int), _ptr(td, C.c_double), _ptr(d2, C.c_uint8), len(d2), int(cols),
                                           int(rows), plf_grid_window(*[int(v) for v in w]), C.c_float(nnr),
                                           C.c_double(line_sim_th), int(bool(best_lr)), _ptr(m, C.c_int32), C.byref(cnt))
        self._check(st, "plf_match_grid_lines")
        return m, cnt.value

    def median_descriptors(self, desc, offsets, dirs=None):
        """MapPoint/MapLine::updateAverageDescDir over many landmarks: (med_idx int32[L], med_dir f64[L,3] or None)."""
        desc = _u8(desc).reshape(-1, DESC_BYTES)
        offsets = np.ascontiguousarray(offsets, np.int32)
        L = len(offsets) - 1
        idx = np.full(max(L, 0), -1, np.int32)
        md = None
        dp = None
        if dirs is not None:
            dirs = np.ascontiguousarray(dirs, np.float64).reshape(-1, 3)
            md = np.zeros((max(L, 0), 3), np.float64)
            dp = _ptr(dirs, C.c_double)
        st = self.lib.plf_median_descriptors(self._ctx, _ptr(desc, C.c_uint8), _ptr(offsets, C.c_int), dp, L,
                                             _ptr(idx, C.c_int), _ptr(md, C.c_double) if md is not None else None)
        self._check(st, "plf_median_descriptors")
        return idx, md

    # -- line descriptor -------------------------------------------------------------------------
    def lbd_gradients(self, img):
        """BinaryDescriptor::computeSobel: returns (dx, dy) int16 of the 5x5-blurred image."""
        img = _u8(img)
        h, w = img.shape
        out = np.empty((h, w, 2), np.int16)
        st = self.lib.plf_lbd_gradients(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                        _ptr(out, C.c_int16))
        self._check(st, "plf_lbd_gradients")
        return out[..., 0].copy(), out[..., 1].copy()

    def lbd(self, img, keylines, want_float=False):
        """BinaryDescriptor::compute(img, keylines, desc): returns uint8[n,32] (and float32[n,72])."""
        img = _u8(img)
        h, w = img.shape
        kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
        n = len(kl)
        desc = np.zeros((n, 32), np.uint8)
        fl = np.zeros((n, 72), np.float32) if want_float else None
        st = self.lib.plf_lbd(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                              kl.ctypes.data_as(C.c_void_p), n, _ptr(desc, C.c_uint8),
                              _ptr(fl, C.c_float) if want_float else None)
        self._check(st, "plf_lbd")
        return (desc, fl) if want_float else desc

    # -- pose refinement -------------------------------------------------------------------------
    def gn_pose(self, P, pl_obs, sP, eP, le_obs, inlier_pt=None, inlier_ls=None, T_init=None, opts=None):
        """StereoFrameHandler::optimizePose.  Returns dict(T, cov, x, err, iters, inlier_pt, inlier_ls)."""
        f64 = lambda a, k: np.ascontiguousarray(a, np.float64).reshape(-1, k)
        P, pl_obs, sP, eP, le_obs = f64(P, 3), f64(pl_obs, 2), f64(sP, 3), f64(eP, 3), f64(le_obs, 3)
        n_p, n_l = len(P), len(sP)
        ip = np.ones(n_p, np.uint8) if inlier_pt is None else np.ascontiguousarray(inlier_pt, np.uint8).copy()
        il = np.ones(n_l, np.uint8) if inlier_ls is None else np.ascontiguousarray(inlier_ls, np.uint8).copy()
        T0 = None if T_init is None else np.ascontiguousarray(T_init, np.float64).reshape(16)
        out = plf_pose_result()
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None and a.size else None
        up = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint8)) if a.size else None
        st = self.lib.plf_gn_pose(self._ctx, C.byref(opts) if opts is not None else None, dp(P), dp(pl_obs),
                                  up(ip), n_p, dp(sP), dp(eP), dp(le_obs), up(il), n_l,
                                  dp(T0) if T0 is not None else None, C.byref(out))
        self._check(st, "plf_gn_pose")
        return dict(T=np.array(out.T).reshape(4, 4), cov=np.array(out.cov).reshape(6, 6), x=np.array(out.x),
                    err=out.err, iters=(out.iters1, out.iters2), inlier_pt=ip, inlier_ls=il,
                    n_inliers=(out.n_inliers_pt, out.n_inliers_ls))

    def loop_closure_pose(self, kf0, kf1, lc=None):
        """MapHandler::isLoopClosure + computeRelativePoseRobustGN (src/mapHandler.cpp:3192-3300, :3566-3957).
        kf0 / kf1: dicts with pdesc, P, pl, ldesc, sP, eP, le (numpy); lc: dict of the lc_* thresholds."""
        d = dict(lc_res=1.0, lc_unc=0.01, lc_inl=0.3, lc_trs=1.5, lc_rot=35.0, lc_inlier_ratio=30.0)
        d.update(lc or {})
        lcp = plf_lc_params(**d)
        keep = []

        def kf(k):
            f = plf_lc_keyframe()
            pd = _u8(k["pdesc"]).reshape(-1, 32); ld = _u8(k["ldesc"]).reshape(-1, 32)
            arrs = dict(pdesc=pd, ldesc=ld)
            for name, cols in (("P", 3), ("pl", 2), ("sP", 3), ("eP", 3), ("le", 3)):
                arrs[name] = np.ascontiguousarray(k[name], np.float64).reshape(-1, cols)
            f.n_pt, f.n_ls = len(pd), len(ld)
            for name, a in arrs.items():
                keep.append(a)
                setattr(f, name, a.ctypes.data if a.size else None)
            return f
        k0, k1 = kf(kf0), kf(kf1)
        cap_p, cap_l = max(k0.n_pt, 1), max(k0.n_ls, 1)
        pp = np.full((cap_p, 2), -1, np.int32); lp = np.full((cap_l, 2), -1, np.int32)
        out = plf_lc_result()
        st = self.lib.plf_loop_closure_pose(self._ctx, C.byref(lcp), C.byref(k0), C.byref(k1), C.byref(out),
                                            _ptr(pp, C.c_int32), cap_p, _ptr(lp, C.c_int32), cap_l)
        self._check(st, "plf_loop_closure_pose")
        r = {f: getattr(out, f) for f, _ in plf_lc_result._fields_ if f not in ("x_inc", "pose_inc")}
        r["accepted"] = bool(out.accepted); r["estimated"] = bool(out.estimated)
        r["x_inc"] = np.array(out.x_inc); r["pose_inc"] = np.array(out.pose_inc)
        r["pt_pairs"] = pp[:out.n_pt].copy(); r["ls_pairs"] = lp[:out.n_ls].copy()
        return r

    def local_ba(self, prob, lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=1e-7,
                 min_error_change=1e-7, ref_quirks=1):
        """MapHandler::levMarquardtOptimizationLBA on the device (plf_local_ba; src/mapHandler.cpp:1332-1989).
        prob: dict as produced by synth.lba_problem (kf_pose, pt, ls, fixed_T, pt_obs_*, ls_obs_*)."""
        f64 = lambda a, c: np.ascontiguousarray(a, np.float64).reshape(-1, c).copy()
        i32 = lambda a: np.ascontiguousarray(a, np.int32).ravel().copy()
        kf, pt, ls = f64(prob["kf_pose"], 6), f64(prob["pt"], 3), f64(prob["ls"], 6)
        fT = np.ascontiguousarray(prob.get("fixed_T", np.zeros((0, 4, 4))), np.float64).reshape(-1, 16).copy()
        po_lm, po_kf, po_xy = i32(prob["pt_obs_lm"]), i32(prob["pt_obs_kf"]), f64(prob["pt_obs_xy"], 2)
        lo_lm, lo_kf, lo_le = i32(prob["ls_obs_lm"]), i32(prob["ls_obs_kf"]), f64(prob["ls_obs_le"], 3)
        pm, lm = np.zeros(max(len(pt), 1), np.uint8), np.zeros(max(len(ls), 1), np.uint8)
        ad = lambda a: a.ctypes.data if a.size else None
        p = plf_lba_problem(len(kf), len(pt), len(ls), len(fT), ad(kf), ad(pt), ad(ls), ad(fT), len(po_lm), ad(po_lm), ad(po_kf),
                            ad(po_xy), len(lo_lm), ad(lo_lm), ad(lo_kf), ad(lo_le), ad(pm), ad(lm))
        o = plf_lba_opts(lambda_, lambda_k, max_iters, homog_th, min_error, min_error_change, int(ref_quirks))
        res = plf_lba_result()
        self._check(self.lib.plf_local_ba(self._ctx, C.byref(o), C.byref(p), C.byref(res)), "plf_local_ba")
        return dict(kf_pose=kf, pt=pt, ls=ls, pt_moved=pm[:len(pt)].astype(bool), ls_moved=lm[:len(ls)].astype(bool),
                    iters=res.iters, err=res.err, lambda_=res.lambda_)

    def match_kf2kf(self, prev, curr, DT, fast_matching=True, max_kf_epip_p=1.0, max_kf_epip_l=1.0):
        """MapHandler::matchKF2KFPoints / matchKF2KFLines, matching part (plf_match_kf2kf).  prev / curr: get_frame dicts;
        DT: 4x4.  Returns dict(m_pt, n_pt, m_ls, n_ls): per previous-keyframe feature the current one or -1."""
        keep = []
        p, c = _frame_view(prev, keep), _frame_view(curr, keep)
        T = np.ascontiguousarray(DT, np.float64).reshape(16)
        o = plf_kf_match_opts(int(bool(fast_matching)), float(max_kf_epip_p), float(max_kf_epip_l))
        m_pt, m_ls = np.full(max(p.n_pt, 1), -1, np.int32), np.full(max(p.n_ls, 1), -1, np.int32)
        n_pt, n_ls = C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_match_kf2kf(self._ctx, C.byref(o), C.byref(p), C.byref(c), T.ctypes.data_as(C.c_void_p),
                                             m_pt.ctypes.data_as(C.c_void_p), m_ls.ctypes.data_as(C.c_void_p), C.byref(n_pt),
                                             C.byref(n_ls)), "plf_match_kf2kf")
        return dict(m_pt=m_pt[:p.n_pt].copy(), n_pt=n_pt.value, m_ls=m_ls[:p.n_ls].copy(), n_ls=n_ls.value)

    def match_map2kf(self, local_map, Twf, kf, kf_pt_lm=None, kf_ls_lm=None, fast_matching=True, max_kf_epip_p=1.0,
                     max_kf_epip_l=1.0):
        """MapHandler::matchMap2KFPoints / matchMap2KFLines (plf_match_map2kf).  local_map: dict pt_X [n,3], pt_desc,
        optional pt_use, ls_X [n,6], ls_desc, optional ls_use; kf: get_frame dict; kf_*_lm: landmark index per keyframe
        feature (-1 = unmatched) or None.  Returns dict(lm_pt, n_pt, lm_ls, n_ls)."""
        keep = []
        kv = _frame_view(kf, keep)
        m = plf_local_map()

        def arr(a, dt, cols):
            a = np.ascontiguousarray(a, dt).reshape(-1, cols) if cols else np.ascontiguousarray(a, dt).ravel()
            keep.append(a)
            return a
        for key, cols in (("pt", 3), ("ls", 6)):
            X = arr(local_map.get(key + "_X", np.zeros((0, cols))), np.float64, cols)
            d = arr(local_map.get(key + "_desc", np.zeros((0, 32))), np.uint8, 32)
            u = local_map.get(key + "_use")
            setattr(m, "n_" + key, len(X))
            setattr(m, key + "_X", X.ctypes.data if X.size else None)
            setattr(m, key + "_desc", d.ctypes.data if d.size else None)
            if u is not None:
                u = arr(np.asarray(u).astype(np.uint8), np.uint8, 0)
                setattr(m, key + "_use", u.ctypes.data if u.size else None)
        lms = [None if v is None else arr(v, np.int32, 0) for v in (kf_pt_lm, kf_ls_lm)]
        for a, n, name in ((lms[0], kv.n_pt, "kf_pt_lm"), (lms[1], kv.n_ls, "kf_ls_lm")):
            if a is not None and len(a) != n:
                raise PlfError(f"match_map2kf: {name} has {len(a)} entries for {n} keyframe features")
        T = np.ascontiguousarray(Twf, np.float64).reshape(16)
        o = plf_kf_match_opts(int(bool(fast_matching)), float(max_kf_epip_p), float(max_kf_epip_l))
        lm_pt, lm_ls = np.full(max(m.n_pt, 1), -1, np.int32), np.full(max(m.n_ls, 1), -1, np.int32)
        n_pt, n_ls = C.c_int(0), C.c_int(0)
        self._check(self.lib.plf_match_map2kf(self._ctx, C.byref(o), C.byref(m), T.ctypes.data_as(C.c_void_p), C.byref(kv),
                                              *[C.c_void_p(a.ctypes.data if a is not None and a.size else None) for a in lms],
                                              lm_pt.ctypes.data_as(C.c_void_p), lm_ls.ctypes.data_as(C.c_void_p),
                                              C.byref(n_pt), C.byref(n_ls)), "plf_match_map2kf")
        return dict(lm_pt=lm_pt[:m.n_pt].copy(), n_pt=n_pt.value, lm_ls=lm_ls[:m.n_ls].copy(), n_ls=n_ls.value)

    def expmap_se3(self, x):
        x = np.ascontiguousarray(x, np.float64).reshape(6)
        T = np.zeros(16)
        self._check(self.lib.plf_se3(self._ctx, 0, x.ctypes.data_as(C.POINTER(C.c_double)),
                                     T.ctypes.data_as(C.POINTER(C.c_double))), "plf_se3")
        return T.reshape(4, 4)

    def logmap_se3(self, T):
        T = np.ascontiguousarray(T, np.float64).reshape(16)
        x = np.zeros(6)
        self._check(self.lib.plf_se3(self._ctx, 1, T.ctypes.data_as(C.POINTER(C.c_double)),
                                     x.ctypes.data_as(C.POINTER(C.c_double))), "plf_se3")
        return x

    # -- point features --------------------------------------------------------------------------
    def orb(self, img, cap=8192):
        """cv::ORB::detectAndCompute with the ctx parameters: returns (keypoints[KEYPOINT_DTYPE], desc u8[n,32])
        in canonical (octave, y, x) order."""
        img = _u8(img)
        h, w = img.shape
        kps = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        st = self.lib.plf_orb(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                              kps.ctypes.data_as(C.c_void_p), _ptr(desc, C.c_uint8), cap, C.byref(n))
        self._check(st, "plf_orb")
        return kps[:n.value].copy(), desc[:n.value].copy()

    # -- line features ---------------------------------------------------------------------------
    def lsd(self, img, cap=16384):
        """cv::LineSegmentDetector::detect with the ctx LSD parameters: float32[n,4] in OpenCV's order."""
        img = _u8(img)
        h, w = img.shape
        segs = np.zeros((cap, 4), np.float32)
        n = C.c_int(0)
        st = self.lib.plf_lsd(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0], _ptr(segs, C.c_float), cap,
                              C.byref(n))
        self._check(st, "plf_lsd")
        return segs[:n.value].copy()

    def detect_lines(self, img, cap=4096):
        """stvo-pl detectLineFeatures: (keylines[KEYLINE_DTYPE], LBD desc u8[n,32])."""
        img = _u8(img)
        h, w = img.shape
        kl = np.zeros(cap, KEYLINE_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        st = self.lib.plf_detect_lines(self._ctx, _ptr(img, C.c_uint8), w, h, img.strides[0],
                                       kl.ctypes.data_as(C.c_void_p), _ptr(desc, C.c_uint8), cap, C.byref(n))
        self._check(st, "plf_detect_lines")
        return kl[:n.value].copy(), desc[:n.value].copy()

    def debug_sincosf(self, x):
        x = np.ascontiguousarray(x, np.float32)
        s = np.empty_like(x); c = np.empty_like(x)
        st = self.lib.plf_debug_sincosf(self._ctx, _ptr(x, C.c_float), _ptr(s, C.c_float), _ptr(c, C.c_float), len(x))
        self._check(st, "plf_debug_sincosf")
        return s, c

    def debug_timeline(self):
        """Device-clock start/end (ms) of the E, G, M phases of the two most recent batches: array [2, 3, 2]."""
        out = np.zeros(12, np.float32)
        self._check(self.lib.plf_debug_timeline(self._ctx, _ptr(out, C.c_float)), "plf_debug_timeline")
        return out.reshape(2, 3, 2)

    # -- batched front-end -----------------------------------------------------------------------
    def reset_sequence(self):
        self._check(self.lib.plf_reset_sequence(self._ctx), "plf_reset_sequence")

    @staticmethod
    def _result_dicts(res, B):
        out = []
        for k in range(B):
            r = res[k]
            d = {f: getattr(r, f) for f in RESULT_FIELDS}
            d["DT"] = np.array(r.DT).reshape(4, 4)
            d["DT_cov"] = np.array(r.DT_cov).reshape(6, 6)
            d["err"] = r.err
            out.append(d)
        return out

    def _stack(self, left, right):
        left = np.ascontiguousarray(left, np.uint8); right = np.ascontiguousarray(right, np.uint8)
        if left.ndim == 2:
            left, right = left[None], right[None]
        assert left.shape == right.shape and left.shape[1:] == (self.camera.height, self.camera.width)
        return left, right

    def process_batch(self, left, right):
        """B x (insertStereoPair + optimizePose): left/right uint8 [B,H,W] host arrays -> list of result dicts."""
        left, right = self._stack(left, right)
        B = left.shape[0]
        res = (plf_frame_result * B)()
        st = self.lib.plf_process_batch(self._ctx, B, _ptr(left, C.c_uint8), _ptr(right, C.c_uint8),
                                        self.camera.width, res)
        self._check(st, "plf_process_batch")
        return self._result_dicts(res, B)

    def batch_upload(self, left, right):
        left, right = self._stack(left, right)
        self._check(self.lib.plf_batch_upload(self._ctx, left.shape[0], _ptr(left, C.c_uint8), _ptr(right, C.c_uint8),
                                              self.camera.width), "plf_batch_upload")
        return left.shape[0]

    def batch_upload_raw(self, B, left_ptr, right_ptr):
        """Upload from raw host addresses (e.g. pinned memory)."""
        self._check(self.lib.plf_batch_upload(self._ctx, int(B), C.c_void_p(left_ptr), C.c_void_p(right_ptr),
                                              self.camera.width), "plf_batch_upload")

    def batch_run(self, B):
        self._check(self.lib.plf_batch_run(self._ctx, int(B)), "plf_batch_run")

    def batch_download(self, B):
        res = (plf_frame_result * B)()
        self._check(self.lib.plf_batch_download(self._ctx, int(B), res), "plf_batch_download")
        return self._result_dicts(res, B)

    def batch_download_array(self, B):
        """Same as batch_download but returns one numpy structured array (RESULT_DTYPE) — no per-frame Python objects."""
        out = np.zeros(B, RESULT_DTYPE)
        self._check(self.lib.plf_batch_download(self._ctx, int(B), out.ctypes.data_as(C.c_void_p)), "plf_batch_download")
        return out

    def batch_device_poses(self, B, dst_device_ptr, stream=0):
        """DT [B,16] f64 of the oldest batch in flight -> caller's device buffer, on the caller's CUDA stream."""
        self._check(self.lib.plf_batch_device_poses(self._ctx, int(B), C.c_void_p(int(dst_device_ptr)), C.c_void_p(int(stream))),
                    "plf_batch_device_poses")

    @property
    def device_images(self) -> int:
        return int(self.lib.plf_batch_device_images(self._ctx) or 0)

    def get_frame(self, k):
        """Stereo-valid features of frame k of the last batch (dict of numpy arrays)."""
        K, Ln = self.limits.max_keypoints, self.limits.max_lines
        a = dict(pt_pl=np.zeros((K, 2)), pt_disp=np.zeros(K), pt_P=np.zeros((K, 3)), pt_octave=np.zeros(K, np.int32),
                 pdesc=np.zeros((K, 32), np.uint8), ls_spl=np.zeros((Ln, 2)), ls_epl=np.zeros((Ln, 2)),
                 ls_sdisp=np.zeros(Ln), ls_edisp=np.zeros(Ln), ls_sP=np.zeros((Ln, 3)), ls_eP=np.zeros((Ln, 3)),
                 ls_le=np.zeros((Ln, 3)), ls_angle=np.zeros(Ln, np.float32), ldesc=np.zeros((Ln, 32), np.uint8))
        v = plf_frame_view(cap_pt=K, cap_ls=Ln)
        for name, arr in a.items():
            setattr(v, name, arr.ctypes.data)
        self._check(self.lib.plf_get_frame(self._ctx, int(k), C.byref(v)), "plf_get_frame")
        out = {}
        for name, arr in a.items():
            n = v.n_pt if name.startswith("pt_") or name == "pdesc" else v.n_ls
            out[name] = arr[:n].copy()
        return out

    def get_matches(self, k):
        """Frame-to-frame correspondences of pair k of the last batch (matched_pt / matched_ls after optimizePose), in the
        previous frame's row order: dict with P, pl_obs, inlier_pt (bool) and sP, eP, le_obs, inlier_ls (bool)."""
        K, Ln = self.limits.max_keypoints, self.limits.max_lines
        a = dict(P=np.zeros((K, 3)), pl_obs=np.zeros((K, 2)), inlier_pt=np.zeros(K, np.uint8), sP=np.zeros((Ln, 3)),
                 eP=np.zeros((Ln, 3)), le_obs=np.zeros((Ln, 3)), inlier_ls=np.zeros(Ln, np.uint8))
        v = plf_match_view(cap_pt=K, cap_ls=Ln)
        for name, arr in a.items():
            setattr(v, name, arr.ctypes.data)
        self._check(self.lib.plf_get_matches(self._ctx, int(k), C.byref(v)), "plf_get_matches")
        out = {}
        for name, arr in a.items():
            n = v.n_pt if name in ("P", "pl_obs", "inlier_pt") else v.n_ls
            out[name] = arr[:n].astype(bool) if name.startswith("inlier") else arr[:n].copy()
        return out

    # -- profiling -------------------------------------------------------------------------------
    def profile_enable(self, on=True):
        self._check(self.lib.plf_profile_enable(self._ctx, int(on)), "plf_profile_enable")  # 2: keep the pipeline on

    def profile_read(self):
        """Returns [(stage name, ms)] of the batch_run calls since profiling was enabled / last read."""
        buf = C.create_string_buffer(16384)
        ms = (C.c_float * 1024)()
        n = C.c_int(0)
        self._check(self.lib.plf_profile_read(self._ctx, buf, 16384, ms, 1024, C.byref(n)), "plf_profile_read")
        names = buf.value.decode().split(";")[:n.value]
        return list(zip(names, [ms[i] for i in range(min(n.value, 1024))]))
