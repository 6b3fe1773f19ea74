"""ctypes wrapper of oracle/_build/liboracle.so (the C restatements).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

_DIR = Path(__file__).resolve().parent
_LIB = _DIR / "_build" / "liboracle.so"

KEYLINE_DTYPE = np.dtype([
    ("angle", np.float32), ("class_id", np.int32), ("octave", np.int32),
    ("ptx", np.float32), ("pty", np.float32), ("response", np.float32), ("size", np.float32),
    ("startPointX", np.float32), ("startPointY", np.float32), ("endPointX", np.float32),
    ("endPointY", np.float32), ("sPointInOctaveX", np.float32), ("sPointInOctaveY", np.float32),
    ("ePointInOctaveX", np.float32), ("ePointInOctaveY", np.float32), ("lineLength", np.float32),
    ("numOfPixels", np.int32)])
assert KEYLINE_DTYPE.itemsize == 68

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not _LIB.exists():
            subprocess.run(["make", "oracle"], cwd=_DIR.parent, check=True, capture_output=True)
        _lib = C.CDLL(str(_LIB))
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def gaussian_kernel_q8(ksize, sigma):
    taps = np.zeros(ksize, np.int32)
    lib().orc_gaussian_kernel_q8(int(ksize), C.c_double(sigma), _p(taps))
    return taps


def gaussian_blur_u8(img, ksize, sigma):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty_like(img)
    lib().orc_gaussian_blur_u8(_p(img), img.shape[1], img.shape[0], int(ksize), C.c_double(sigma), _p(out))
    return out


def sobel3_i16(img):
    img = np.ascontiguousarray(img, np.uint8)
    dx = np.empty(img.shape, np.int16); dy = np.empty(img.shape, np.int16)
    lib().orc_sobel3_i16(_p(img), img.shape[1], img.shape[0], _p(dx), _p(dy))
    return dx, dy


def keylines_from_segments(segs, w, h, min_length):
    segs = np.ascontiguousarray(segs, np.float32).reshape(-1, 4)
    out = np.zeros(len(segs), KEYLINE_DTYPE)
    f = lib().orc_keylines_from_segments
    f.restype = C.c_int
    n = f(_p(segs), len(segs), int(w), int(h), C.c_double(min_length), _p(out))
    return out[:n].copy()


def lbd_compute(img, keylines, want_float=False):
    img = np.ascontiguousarray(img, np.uint8)
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    n = len(kl)
    desc = np.zeros((n, 32), np.uint8)
    fl = np.zeros((n, 72), np.float32) if want_float else None
    lib().orc_lbd_compute(_p(img), img.shape[1], img.shape[0], _p(kl), n, _p(desc),
                          _p(fl) if want_float else None)
    return (desc, fl) if want_float else desc


# ---- Gauss-Newton (oracle/gn.c) --------------------------------------------------------------------
class orc_camera(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("b", C.c_double)]


class orc_gn_opts(C.Structure):
    _fields_ = [("homog_th", C.c_double), ("max_iters", C.c_int), ("max_iters_ref", C.c_int),
                ("eps_err", C.c_double), ("eps_change", C.c_double), ("eps_step", C.c_double)]


class orc_pose_result(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("cov", C.c_double * 36), ("x", C.c_double * 6),
                ("err", C.c_double), ("iters1", C.c_int), ("iters2", C.c_int),
                ("n_inliers_pt", C.c_int), ("n_inliers_ls", C.c_int)]


def gn_opts(homog_th=1e-7, max_iters=5, max_iters_ref=10, eps_err=1e-7, eps_change=1e-7,
            eps_step=2.220446049250313e-16):
    return orc_gn_opts(homog_th, max_iters, max_iters_ref, eps_err, eps_change, eps_step)


def expmap_se3(x):
    x = np.ascontiguousarray(x, np.float64).reshape(6); T = np.zeros(16)
    lib().orc_expmap_se3(_p(x), _p(T)); return T.reshape(4, 4)


def logmap_se3(T):
    T = np.ascontiguousarray(T, np.float64).reshape(16); x = np.zeros(6)
    lib().orc_logmap_se3(_p(T), _p(x)); return x


def inverse_se3(T):
    T = np.ascontiguousarray(T, np.float64).reshape(16); Ti = np.zeros(16)
    lib().orc_inverse_se3(_p(T), _p(Ti)); return Ti.reshape(4, 4)


def colpiv_qr_solve6(H, g):
    H = np.ascontiguousarray(H, np.float64).reshape(36); g = np.ascontiguousarray(g, np.float64).reshape(6)
    x = np.zeros(6); lib().orc_colpiv_qr_solve6(_p(H), _p(g), _p(x)); return x


# stop-decision trace (orc_gn_pose_trace): exit reasons and one record per iteration
GN_CONTINUE, GN_EXIT_ERROR, GN_EXIT_STEP, GN_EXIT_MAXIT = range(4)
GN_TRACE_DTYPE = np.dtype([("stage", np.int32), ("exit", np.int32), ("e", np.float64), ("e_prev", np.float64),
                           ("step", np.float64)])
GN_ERR_PREV0 = 999999999.9   # the error the first change test compares with (gn.c gn_pose)


class orc_gn_trace(C.Structure):
    _fields_ = [("rec", C.c_void_p), ("cap", C.c_int), ("n", C.c_int), ("stage_exit", C.c_int * 2)]


def gn_pose(cam, P, pl_obs, sP, eP, le_obs, inlier_pt=None, inlier_ls=None, T_init=None, opts=None, trace=False):
    """orc_gn_pose.  trace=True adds res["trace"] = dict(rec=GN_TRACE_DTYPE records, one per accumulation of either
    stage, exit=(stage-1 exit reason, stage-2 exit reason)).  An accumulation stopped by the error test takes no step
    and does not count in iters; the others do."""
    f64 = lambda a, k: np.ascontiguousarray(a, np.float64).reshape(-1, k)
    P, pl_obs, sP, eP, le_obs = f64(P, 3), f64(pl_obs, 2), f64(sP, 3), f64(eP, 3), f64(le_obs, 3)
    ip = np.ones(len(P), np.uint8) if inlier_pt is None else np.ascontiguousarray(inlier_pt, np.uint8).copy()
    il = np.ones(len(sP), np.uint8) if inlier_ls is None else np.ascontiguousarray(inlier_ls, np.uint8).copy()
    T0 = np.eye(4).reshape(16) if T_init is None else np.ascontiguousarray(T_init, np.float64).reshape(16)
    c = orc_camera(**cam) if isinstance(cam, dict) else cam
    o = opts if opts is not None else gn_opts()
    out = orc_pose_result()
    args = (C.byref(c), C.byref(o), _p(P), _p(pl_obs), _p(ip), len(P), _p(sP), _p(eP), _p(le_obs), _p(il), len(sP),
            _p(T0), C.byref(out))
    if trace:
        rec = np.zeros(max(o.max_iters, 0) + max(o.max_iters_ref, 0), GN_TRACE_DTYPE)
        tr = orc_gn_trace(rec.ctypes.data, len(rec), 0)
        lib().orc_gn_pose_trace(*args, C.byref(tr))
        assert tr.n <= len(rec)
    else:
        lib().orc_gn_pose(*args)
    res = dict(T=np.array(out.T).reshape(4, 4), cov=np.array(out.cov).reshape(6, 6), x=np.array(out.x),
               err=out.err, iters=(out.iters1, out.iters2), inlier_pt=ip, inlier_ls=il,
               n_inliers=(out.n_inliers_pt, out.n_inliers_ls))
    if trace:
        res["trace"] = dict(rec=rec[:tr.n].copy(), exit=(tr.stage_exit[0], tr.stage_exit[1]))
    return res


def gn_decidable(trace, opts, rel_band=1e-10):
    """True when the iteration counts of a run are well defined under a change of summation order: every stop test the
    oracle evaluated (trace of gn_pose(..., trace=True)) lies outside the band that order can move it by.

    A solver that sums its rows in another order (a tree on the device) sees each error e with a relative difference of
    about 1e-12, so a test within rel_band * max(e, e_prev) of its threshold (the change test | |e - e_prev| -
    eps_change |, then the error test |e - eps_err|, which is only evaluated when the change test fails) may go either
    way, and so may a step test with ||dx|| within [eps_step / 10, 10 eps_step].  The constant first e_prev
    (GN_ERR_PREV0) carries no rounding and does not widen the band.  A NaN error (no row left) fails both tests on
    every solver, and so does not count as near."""
    for r in trace["rec"]:
        e, ep = float(r["e"]), float(r["e_prev"])
        if not np.isnan(e):
            band = rel_band * (e if ep == GN_ERR_PREV0 else max(e, ep))
            change = abs(e - ep)
            if abs(change - opts.eps_change) <= band:
                return False
            if not change < opts.eps_change and abs(e - opts.eps_err) <= band:
                return False
        if r["step"] >= 0 and opts.eps_step / 10 <= r["step"] <= 10 * opts.eps_step:
            return False
    return True


# ---- ORB (oracle/orb.c) ------------------------------------------------------------------------------
KEYPOINT_DTYPE = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                           ("response", np.float32), ("octave", np.int32), ("lx", np.int32), ("ly", np.int32)])


def resize_linear_exact(img, dw, dh, fx=None, fy=None):
    img = np.ascontiguousarray(img, np.uint8)
    sh, sw = img.shape
    out = np.empty((dh, dw), np.uint8)
    lib().orc_resize_linear_exact(_p(img), sw, sh, _p(out), dw, dh, C.c_double(fx if fx else dw / sw),
                                  C.c_double(fy if fy else dh / sh))
    return out


def fast_score_map(img, threshold):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty_like(img)
    lib().orc_fast_score_map(_p(img), img.shape[1], img.shape[0], int(threshold), _p(out))
    return out


def fast_atan2(y, x):
    f = lib().orc_fast_atan2
    f.restype = C.c_float
    f.argtypes = [C.c_float, C.c_float]
    return f(y, x)


def orb(img, nfeatures=800, scale_factor=1.2, nlevels=4, edge_th=19, patch_size=31, fast_th=20, cap=20000):
    img = np.ascontiguousarray(img, np.uint8)
    kps = np.zeros(cap, KEYPOINT_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    f = lib().orc_orb_detect_and_compute
    f.restype = C.c_int
    n = f(_p(img), img.shape[1], img.shape[0], int(nfeatures), C.c_float(scale_factor), int(nlevels), int(edge_th),
          int(patch_size), int(fast_th), _p(kps), _p(desc), cap)
    if n < 0:
        raise RuntimeError("orb oracle: capacity exceeded")
    return kps[:n].copy(), desc[:n].copy()


# ---- LSD (oracle/lsd.c) ------------------------------------------------------------------------------
def lsd(img, scale=1.2, sigma_scale=0.6, quant=2.0, ang_th=22.5, n_bins=1024, order_mode=0, trig_mode=0, cap=65536):
    img = np.ascontiguousarray(img, np.uint8)
    segs = np.zeros((cap, 4), np.float32)
    f = lib().orc_lsd_detect
    f.restype = C.c_int
    n = f(_p(img), img.shape[1], img.shape[0], C.c_double(scale), C.c_double(sigma_scale), C.c_double(quant),
          C.c_double(ang_th), int(n_bins), int(order_mode), int(trig_mode), _p(segs), cap)
    if n < 0:
        raise RuntimeError("lsd oracle: capacity exceeded")
    return segs[:n].copy()


class _LbaOpts(C.Structure):
    _fields_ = [("lambda_", C.c_double), ("lambda_k", C.c_double), ("max_iters", C.c_int), ("homog_th", C.c_double),
                ("min_error", C.c_double), ("min_error_change", C.c_double), ("ref_quirks", C.c_int)]


class _LbaResult(C.Structure):
    _fields_ = [("iters", C.c_int), ("err", C.c_double), ("lambda_", C.c_double), ("zero_lm", C.c_int)]


# orc_local_ba's return codes and its iteration trace (orc_local_ba_trace): record 0 is the first pass, record i the
# i-th LM iteration; `stop` is LBA_CONTINUE or why the run ended after that pass
LBA_EMPTY, LBA_ZERO_BLOCK = -1, -2
LBA_CONTINUE, LBA_STOP_CHANGE, LBA_STOP_MIN_ERROR, LBA_STOP_STEP, LBA_STOP_MAXIT = range(5)
LBA_TRACE_DTYPE = np.dtype([("err", np.float64), ("lambda_", np.float64), ("step", np.float64), ("applied", np.int32),
                            ("stop", np.int32)])


class _LbaTrace(C.Structure):
    _fields_ = [("rec", C.c_void_p), ("cap", C.c_int), ("n", C.c_int)]


def lba_opts(lambda_=1e-5, lambda_k=10.0, max_iters=15, homog_th=1e-7, min_error=1e-7, min_error_change=1e-7, ref_quirks=1):
    """Defaults: src/slamConfig.cpp:64-66 (lambda_lba_lm, lambda_lba_k, max_iters_lba), config_euroc.yaml:45,49-50."""
    return dict(lambda_=lambda_, lambda_k=lambda_k, max_iters=max_iters, homog_th=homog_th, min_error=min_error,
                min_error_change=min_error_change, ref_quirks=ref_quirks)


def local_ba(cam, prob, opts=None):
    """MapHandler::levMarquardtOptimizationLBA (oracle/lba.c).  prob: dict with kf_pose [nkf,6], pt [npt,3], ls [nls,6],
    fixed_T [nf,4,4], pt_obs_lm / pt_obs_kf / pt_obs_xy, ls_obs_lm / ls_obs_kf / ls_obs_le (kf < 0: fixed keyframe -1-k).
    Returns rc (0, LBA_EMPTY or LBA_ZERO_BLOCK, with the refused landmark in zero_lm: points first, then lines), the
    optimised values (the input's when refused), iters, err, lambda_ and trace: LBA_TRACE_DTYPE records, one per pass."""
    o = _LbaOpts(**(opts or lba_opts()))
    c = orc_camera(**{k: cam[k] for k in ("width", "height", "fx", "fy", "cx", "cy", "b")})
    kf = np.ascontiguousarray(prob["kf_pose"], np.float64).reshape(-1, 6)
    pt = np.ascontiguousarray(prob["pt"], np.float64).reshape(-1, 3)
    ls = np.ascontiguousarray(prob["ls"], np.float64).reshape(-1, 6)
    X = np.concatenate([kf.ravel(), pt.ravel(), ls.ravel()]).astype(np.float64)
    fT = np.ascontiguousarray(prob.get("fixed_T", np.zeros((0, 4, 4))), np.float64).reshape(-1, 16)
    i32 = lambda k: np.ascontiguousarray(prob[k], np.int32).ravel()
    f64 = lambda k: np.ascontiguousarray(prob[k], np.float64).ravel()
    po_lm, po_kf, po_xy = i32("pt_obs_lm"), i32("pt_obs_kf"), f64("pt_obs_xy")
    lo_lm, lo_kf, lo_le = i32("ls_obs_lm"), i32("ls_obs_kf"), f64("ls_obs_le")
    pm, lm = np.zeros(max(len(pt), 1), np.uint8), np.zeros(max(len(ls), 1), np.uint8)
    res = _LbaResult()
    rec = np.zeros(max(o.max_iters, 1), LBA_TRACE_DTYPE)
    tr = _LbaTrace(rec.ctypes.data, len(rec), 0)
    f = lib().orc_local_ba_trace
    f.restype = C.c_int
    rc = f(C.byref(c), C.byref(o), len(kf), len(pt), len(ls), _p(X), len(fT), _p(fT), len(po_lm), _p(po_lm), _p(po_kf), _p(po_xy),
           len(lo_lm), _p(lo_lm), _p(lo_kf), _p(lo_le), _p(pm), _p(lm), C.byref(res), C.byref(tr))
    assert tr.n <= len(rec)
    nk, npt = 6 * len(kf), 3 * len(pt)
    return dict(rc=rc, kf_pose=X[:nk].reshape(-1, 6), pt=X[nk:nk + npt].reshape(-1, 3), ls=X[nk + npt:].reshape(-1, 6),
                pt_moved=pm[:len(pt)].astype(bool), ls_moved=lm[:len(ls)].astype(bool), iters=res.iters, err=res.err,
                lambda_=res.lambda_, zero_lm=res.zero_lm, trace=rec[:tr.n].copy())
