"""The front-end detectors at every image geometry their tile kernels and uploads treat differently, and with row-strided
input, bit for bit against the C restatements (GPU).

The shapes come from tests/test_frontend_geometry.py, which derives them from the kernels' tile constants and checks on
the CPU that the kernels' index arithmetic reads inside its boxes for every one of them before they run here:
  - fe.orb / fe.lsd / fe.detect_lines over the sweep, the ORB level-boundary sizes, ORB's minimum size and LSD's tiny
    sizes, at the defaults and at param_cases settings that change a blur radius or the size floor;
  - every entry point with a `stride` argument (plf_orb, plf_lsd, plf_detect_lines, plf_lbd, plf_process_batch,
    plf_batch_upload) called through ctypes on a row-strided view of a larger buffer whose padding is poisoned;
  - the batched pipeline (test_pipeline_gpu.compare) at three odd cameras, with partial batches, and below ORB's minimum
    size with has_points = 0."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe
from param_cases import LSD_CASES, ORB_CASES
from test_frontend_geometry import (LSD_REFUSED, LSD_TINY, ORB_MIN_EDGE, ORB_SHAPES_L4, ORB_SHAPES_L8, T, kitti_class_shapes,
                                    orb_level_sizes, orb_ok, orb_size_edges, scene_image, sweep_shapes)
from test_pipeline_gpu import STANDALONE_WORLD, compare

pytestmark = pytest.mark.gpu
ORB_FIELDS = ["x", "y", "size", "angle", "response", "octave"]
LSD_PARAM_CASES = {"default": {}, "sigma0.4_k5": LSD_CASES["sigma0.4_k5"], "sigma0.9_k9": LSD_CASES["sigma0.9_k9"]}


def pitch16(w):
    return (w + 15) & ~15


def assert_orb_same(kp, desc, ok, od, where):
    assert len(kp) == len(ok), where
    for f in ORB_FIELDS:
        assert np.array_equal(kp[f], ok[f]), (where, f)
    assert np.array_equal(desc, od), where


# ---- standalone detectors over the sweep ---------------------------------------------------------------------------
def orb_cases():
    return {
        "l1_sweep": (dict(orb_nlevels=1), [s for s in sweep_shapes() if orb_ok(*s, nlevels=1)]),
        "l4_levels": (dict(orb_nlevels=4), ORB_SHAPES_L4 + [s for s in sweep_shapes() if orb_ok(*s, nlevels=4)]),
        "l8_levels": (dict(orb_nlevels=8), ORB_SHAPES_L8),
        "edge31": (dict(ORB_CASES["edge31"], orb_nlevels=4), [s for s in ORB_SHAPES_L4 + ORB_SHAPES_L8 if orb_ok(*s, nlevels=4, edge=31)]),
        "kitti_class_l8": (dict(orb_nlevels=8), kitti_class_shapes()),
    }


@pytest.mark.parametrize("case", list(orb_cases()))
def test_orb_over_the_sweep(built, case):
    """fe.orb equals clib.orb (every keypoint field, every descriptor) at every shape of the case."""
    over, shapes = orb_cases()[case]
    nl, edge = over.get("orb_nlevels", 4), over.get("orb_edge_th", ORB_MIN_EDGE)
    nf = 2000 if case.startswith("kitti") else 500
    assert len(shapes) >= 2
    total, octaves = 0, set()
    with plf.Frontend(orb_nfeatures=nf, **over) as fe:
        for i, (w, h) in enumerate(shapes):
            img = scene_image(w, h, 7 + i)
            kp, desc = fe.orb(img)
            ok, od = clib.orb(img, nf, nlevels=nl, edge_th=edge)
            assert_orb_same(kp, desc, ok, od, (case, w, h))
            total += len(kp)
            octaves |= set(kp["octave"].tolist())
    assert total > 10 * len(shapes)
    assert octaves >= set(range(min(nl, 4)))        # keypoints on the pyramid levels, not only on level 0


def test_orb_minimum_size(built):
    """The smallest size ORB accepts for each (nlevels, edge_th) runs and matches the oracle; one pixel less in either
    axis is refused with a clean PlfError, and the context stays usable."""
    for nl, edge, s in orb_size_edges():
        with plf.Frontend(orb_nfeatures=300, orb_nlevels=nl, orb_edge_th=edge) as fe:
            img = scene_image(s, s, nl + edge)
            kp, desc = fe.orb(img)
            ok, od = clib.orb(img, 300, nlevels=nl, edge_th=edge)
            assert_orb_same(kp, desc, ok, od, (nl, edge, s))
            for w, h in ((s - 1, s), (s, s - 1)):
                with pytest.raises(plf.PlfError, match="too small"):
                    fe.orb(scene_image(w, h, 1))
            kp2, desc2 = fe.orb(img)
            assert kp2.tobytes() == kp.tobytes() and np.array_equal(desc2, desc)


def lsd_shapes():
    return sweep_shapes() + LSD_TINY


@pytest.mark.parametrize("case", list(LSD_PARAM_CASES))
def test_lsd_over_the_sweep(built, case):
    """fe.lsd equals clib.lsd, segments in order, at every sweep shape and at the tiny sizes (smaller than the blur
    window and than one tile); 1- and 2-pixel sides are refused with PLF_ERR_INVALID."""
    prm = LSD_PARAM_CASES[case]
    kw = ofe.lsd_kwargs(dict(ofe.DEFAULTS, **prm))
    n = 0
    with plf.Frontend(**prm) as fe:
        for i, (w, h) in enumerate(lsd_shapes()):
            img = scene_image(w, h, i)
            segs, ref = fe.lsd(img), clib.lsd(img, **kw)
            assert segs.shape == ref.shape and np.array_equal(segs, ref), (case, w, h)
            n += len(ref)
        for w, h in LSD_REFUSED:
            with pytest.raises(plf.PlfError, match=r"plf_lsd failed \(-1\)"):
                fe.lsd(np.zeros((h, w), np.uint8))
        assert np.array_equal(fe.lsd(scene_image(64, 32, 0)), clib.lsd(scene_image(64, 32, 0), **kw))
    assert n > 15 * len(lsd_shapes())


@pytest.mark.parametrize("case", list(LSD_PARAM_CASES))
def test_detect_lines_over_the_sweep(built, case):
    """fe.detect_lines (LSD -> KeyLines -> LBD) equals oracle.frontend.detect_lines, KeyLine bytes and descriptors."""
    prm = dict(LSD_PARAM_CASES[case], lsd_nfeatures=60)
    full = dict(ofe.DEFAULTS, **prm)
    n = 0
    with plf.Frontend(**prm) as fe:
        for i, (w, h) in enumerate(lsd_shapes()):
            img = scene_image(w, h, 50 + i)
            kl, desc = fe.detect_lines(img)
            okl, odesc = ofe.detect_lines(img, lsd_nfeatures=60, min_line_length=full["min_line_length"], lsd_kwargs=ofe.lsd_kwargs(full))
            assert len(kl) == len(okl) and kl.tobytes() == okl.tobytes(), (case, w, h)
            assert np.array_equal(desc, odesc), (case, w, h)
            n += len(kl)
        for w, h in LSD_REFUSED:
            with pytest.raises(plf.PlfError, match=r"plf_detect_lines failed \(-1\)"):
                fe.detect_lines(np.zeros((h, w), np.uint8))
    assert n > 5 * len(lsd_shapes())


# ---- strided input on every stride entry point ------------------------------------------------------------------------
def strided(img, stride, poison):
    """A (h, w) view with row stride `stride` into a larger buffer whose padding bytes are `poison` (0xFF or a seed)."""
    h, w = img.shape
    if poison == 0xFF:
        buf = np.full((h, stride), 0xFF, np.uint8)
    else:
        buf = np.random.default_rng(poison).integers(0, 256, (h, stride), dtype=np.uint8)
    buf[:, :w] = img
    view = buf[:, :w]
    assert view.strides[0] == stride and not view.flags.c_contiguous
    return buf, view


def call_standalone(fe, name, buf, w, h, stride, kl=None):
    """plf_orb / plf_lsd / plf_detect_lines / plf_lbd through ctypes on the rows at buf (stride bytes apart); returns
    the outputs as bytes."""
    lib, p = fe.lib, buf.ctypes.data_as(C.POINTER(C.c_uint8))
    n = C.c_int(0)
    if name == "orb":
        kps, desc = np.zeros(4096, plf.KEYPOINT_DTYPE), np.zeros((4096, 32), np.uint8)
        fe._check(lib.plf_orb(fe._ctx, p, w, h, stride, kps.ctypes.data_as(C.c_void_p), desc.ctypes.data_as(C.POINTER(C.c_uint8)),
                              4096, C.byref(n)), "plf_orb")
        return kps[:n.value].tobytes() + desc[:n.value].tobytes(), n.value
    if name == "lsd":
        segs = np.zeros((16384, 4), np.float32)
        fe._check(lib.plf_lsd(fe._ctx, p, w, h, stride, segs.ctypes.data_as(C.POINTER(C.c_float)), 16384, C.byref(n)), "plf_lsd")
        return segs[:n.value].tobytes(), n.value
    if name == "detect_lines":
        kls, desc = np.zeros(4096, plf.KEYLINE_DTYPE), np.zeros((4096, 32), np.uint8)
        fe._check(lib.plf_detect_lines(fe._ctx, p, w, h, stride, kls.ctypes.data_as(C.c_void_p),
                                       desc.ctypes.data_as(C.POINTER(C.c_uint8)), 4096, C.byref(n)), "plf_detect_lines")
        return kls[:n.value].tobytes() + desc[:n.value].tobytes(), n.value
    assert name == "lbd"
    kl = np.ascontiguousarray(kl, plf.KEYLINE_DTYPE)
    desc, fl = np.zeros((len(kl), 32), np.uint8), np.zeros((len(kl), 72), np.float32)
    fe._check(lib.plf_lbd(fe._ctx, p, w, h, stride, kl.ctypes.data_as(C.c_void_p), len(kl), desc.ctypes.data_as(C.POINTER(C.c_uint8)),
                          fl.ctypes.data_as(C.POINTER(C.c_float))), "plf_lbd")
    return desc.tobytes() + fl.tobytes(), len(kl)


@pytest.mark.parametrize("shape", [(179, 130), (160, 97)])
def test_standalone_strided_input(built, shape):
    """Each stride entry point on a row-strided view (stride w + 1, w + 15, pitch16(w) + 16, 2 w; padding 0xFF, then
    random) returns exactly what the contiguous call on the same pixels returns."""
    w, h = shape
    img = scene_image(w, h, 3)
    with plf.Frontend(orb_nfeatures=500) as fe:
        kl, _ = fe.detect_lines(img)
        want = {name: call_standalone(fe, name, np.ascontiguousarray(img), w, h, w, kl) for name in ("orb", "lsd", "detect_lines", "lbd")}
        assert all(n > 10 for _, n in want.values()), {k: n for k, (_, n) in want.items()}
        for stride in (w + 1, w + 15, pitch16(w) + 16, 2 * w):
            for poison in (0xFF, stride):
                buf, _ = strided(img, stride, poison)
                for name in want:
                    got, _ = call_standalone(fe, name, buf, w, h, stride, kl)
                    assert got == want[name][0], (name, stride, poison)
        with pytest.raises(plf.PlfError, match=r"plf_orb failed \(-1\)"):
            fe._check(fe.lib.plf_orb(fe._ctx, img.ctypes.data_as(C.POINTER(C.c_uint8)), w, h, w - 1, None, None, 0,
                                     C.byref(C.c_int())), "plf_orb")


def small_cam(w, h):
    f = 0.8 * w
    return dict(plf.KITTI_CAMERA, width=w, height=h, cx=w / 2, cy=h / 2, fx=f, fy=f)


def frames_for(cam, n, seed):
    return list(synth.stream(cam, n, world=STANDALONE_WORLD, seed=seed, step=0.12))


def batch_strided(fe, L, R, stride, poison, upload_run):
    """One batch from host buffers with image k at offset k * stride * h (padding poisoned): plf_process_batch, or
    plf_batch_upload + plf_batch_run + download.  Returns (RESULT_DTYPE array, frames)."""
    B, h, w = L.shape
    bufs = []
    for side, imgs in enumerate((L, R)):
        buf, _ = strided(imgs.reshape(B * h, w), stride, poison + side if poison != 0xFF else 0xFF)
        bufs.append(buf)
    lp, rp = (b.ctypes.data_as(C.POINTER(C.c_uint8)) for b in bufs)
    if upload_run:
        fe._check(fe.lib.plf_batch_upload(fe._ctx, B, lp, rp, stride), "plf_batch_upload")
        fe.batch_run(B)
        res = fe.batch_download_array(B)
    else:
        res = np.zeros(B, plf.RESULT_DTYPE)
        fe._check(fe.lib.plf_process_batch(fe._ctx, B, lp, rp, stride, res.ctypes.data_as(C.c_void_p)), "plf_process_batch")
    return res, [fe.get_frame(k) for k in range(B)]


def same_frames(a, b):
    assert len(a) == len(b)
    for fa, fb in zip(a, b):
        assert fa.keys() == fb.keys()
        for k in fa:
            assert np.array_equal(fa[k], fb[k]), k


@pytest.mark.parametrize("shape", [(203, 121), (208, 120)])
def test_batch_strided_input(built, shape):
    """plf_process_batch / plf_batch_upload with strided host buffers (w % 16 != 0 and == 0; B = 1, a full batch of 3,
    then a partial batch of 2): every result and every frame equal the contiguous run's, which equals the oracle's
    (compare).  stride < w is refused with PLF_ERR_INVALID and leaves the context usable."""
    w, h = shape
    cam = small_cam(w, h)
    frames = frames_for(cam, 6, seed=w)
    Ls, Rs = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    batches = [(0, 1), (1, 4), (4, 6)]
    prm = dict(orb_nfeatures=400, lsd_nfeatures=80)
    lim = plf.default_limits(); lim.max_batch = 3
    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        base_res, base_fr = [], []
        for a, b in batches:
            base_res.append(fe.process_batch(Ls[a:b], Rs[a:b]))
            base_fr.append([fe.get_frame(k) for k in range(b - a)])
    ref = ofe.run_sequence(cam, [(f[0], f[1]) for f in frames], dict(ofe.DEFAULTS, **prm))
    compare(ref, [r for rs in base_res for r in rs], [f for fr in base_fr for f in fr])
    assert sum(r["status"] == 0 for rs in base_res for r in rs) >= 4
    for stride, poison in ((w + 1, 0xFF), (pitch16(w) + 16, 5), (2 * w, 0xFF)):
        with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
            for i, (a, b) in enumerate(batches):
                res, fr = batch_strided(fe, Ls[a:b], Rs[a:b], stride, poison, upload_run=(i == 1))
                for k, r in enumerate(base_res[i]):
                    for f in plf.RESULT_FIELDS:
                        assert res[k][f] == r[f], (stride, i, k, f)
                    assert res[k]["DT"].tobytes() == r["DT"].tobytes() and res[k]["DT_cov"].tobytes() == r["DT_cov"].tobytes()
                    assert res[k]["err"] == r["err"] or (np.isnan(res[k]["err"]) and np.isnan(r["err"]))
                same_frames(fr, base_fr[i])
    with plf.Frontend(camera=cam, limits=lim, **prm) as fe:
        p = Ls[0].ctypes.data_as(C.POINTER(C.c_uint8))
        assert fe.lib.plf_batch_upload(fe._ctx, 1, p, p, w - 1) == -1
        out = np.zeros(1, plf.RESULT_DTYPE)
        assert fe.lib.plf_process_batch(fe._ctx, 1, p, p, w - 1, out.ctypes.data_as(C.c_void_p)) == -1
        res = fe.process_batch(Ls[0:1], Rs[0:1])
        assert res[0]["status"] == base_res[0][0]["status"] and res[0]["n_stereo_pt"] == base_res[0][0]["n_stereo_pt"]
        same_frames([fe.get_frame(0)], base_fr[0])


# ---- the batched pipeline at odd geometries ---------------------------------------------------------------------------
def level_boundary_width(residue, lo=200, hi=420):
    """The smallest w in [lo, hi) with w = residue (mod 16) whose ORB levels >= 1 put a FAST or ORB-blur boundary."""
    ow, tw = T["FN_OW"], T["OBF_TW"]
    xb = {k * ow + d for k in range(1, 8) for d in (-1, 0, 1)} | {k * tw - 13 + d for k in range(1, 8) for d in (-1, 0, 1)}
    return next(w for w in range(lo, hi) if w % 16 == residue and {a for a, _ in orb_level_sizes(w, w, 4)[1:]} & xb)


def pipeline_cameras():
    return {"w1mod16_h1mod30": (305, 181), "w15mod16_level_boundary": (level_boundary_width(15), 150), "w_mult16": (256, 144)}


@pytest.mark.parametrize("name", list(pipeline_cameras()))
def test_pipeline_odd_geometry(built, name):
    """test_pipeline_gpu.compare at a camera the geometry sweep picks: 7 frames in batches of 3 (the last one partial)."""
    w, h = pipeline_cameras()[name]
    if name == "w1mod16_h1mod30":
        assert w % 16 == 1 and h % 30 == 1
    elif name == "w15mod16_level_boundary":
        assert w % 16 == 15
    else:
        assert w % 16 == 0
    cam = small_cam(w, h)
    frames = frames_for(cam, 7, seed=h)
    prm = dict(ofe.DEFAULTS, orb_nfeatures=500, lsd_nfeatures=100)
    ref = ofe.run_sequence(cam, [(a, b) for a, b, _ in frames], prm)
    lim = plf.default_limits(); lim.max_batch = 3
    got, feats = [], []
    with plf.Frontend(camera=cam, limits=lim, **{k: prm[k] for k, _ in plf.plf_params._fields_}) as fe:
        for s0 in range(0, 7, 3):
            chunk = frames[s0:s0 + 3]
            got += fe.process_batch(np.stack([c[0] for c in chunk]), np.stack([c[1] for c in chunk]))
            feats += [fe.get_frame(k) for k in range(len(chunk))]
    compare(ref, got, feats)
    assert sum(g["status"] == 0 for g in got) >= 4 and all(g["n_kp_l"] > 0 and g["n_lines_l"] > 0 for g in got)


def test_pipeline_lines_only_below_orb_minimum(built):
    """has_points = 0 at a camera below ORB's minimum size: the pipeline still builds its ORB state, so the context
    refuses the size at first use with a clean PlfError ("too small"); nothing is left half-built and a context at a
    size ORB accepts runs the LSD / LBD-only pipeline equal to the oracle."""
    s = orb_size_edges()[1][2]             # 4 levels, edge 19
    cam = small_cam(s - 1, s)
    with plf.Frontend(camera=cam, has_points=0) as fe:
        img = np.stack([scene_image(s - 1, s, 0)])
        with pytest.raises(plf.PlfError, match="too small"):
            fe.process_batch(img, img)
        with pytest.raises(plf.PlfError, match="too small"):
            fe.process_batch(img, img)
    cam = small_cam(s, 100)
    frames = frames_for(cam, 4, seed=2)
    prm = dict(ofe.DEFAULTS, has_points=0, lsd_nfeatures=60)
    ref = ofe.run_sequence(cam, [(a, b) for a, b, _ in frames], prm)
    lim = plf.default_limits(); lim.max_batch = 4
    with plf.Frontend(camera=cam, limits=lim, **{k: prm[k] for k, _ in plf.plf_params._fields_}) as fe:
        got = fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        feats = [fe.get_frame(k) for k in range(4)]
    compare(ref, got, feats)
    assert all(g["n_kp_l"] == 0 for g in got) and any(g["n_lines_l"] > 0 for g in got)
