"""GPU tests of the detector masks (plf_orb_masked, plf_detect_lines_masked, plf_set_sequence_mask).

- The standalone operators against cv2's detectAndCompute(img, mask) and oracle/masks.py detect_lines, byte
  for byte, at KITTI and EuRoC shape and an odd one, 1 / 4 / 8 levels, lsd_nfeatures 0 and 300, on masks that are all
  255, all 0, half, a one-pixel column, a 4 x 4 checkerboard, values 1 and 254, and an edge through a FAST corner.
- The batched pipeline, round robin, some sequences masked (left and right differently) and some not, one and three
  batches in flight, bit-exact to oracle/frontend.py run_sequence with masked detectors.
- The setter: batches in flight keep their masks, no restart, set-then-clear is never-set, plf_set_max_sequences drops
  the masks, and every refusal changes nothing."""
import ctypes as C

import cv2
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import cvref, synth
from oracle import frontend as ofe
from oracle import masks as om
from test_multi_sequence_gpu import assert_same
from test_pipeline_gpu import compare

pytestmark = pytest.mark.gpu

K = plf.KITTI_CAMERA
EUROC = plf.EUROC_CAMERA
SHAPES = {"kitti": (375, 1242), "euroc": (480, 752), "odd": (333, 501)}


def texture(h, w, seed):
    rng = np.random.default_rng(seed)
    return cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (0, 0), 1.5)


def masks(img, nlevels):
    h, w = img.shape
    yy, xx = np.mgrid[:h, :w]
    out = {"all255": np.full((h, w), 255), "all0": np.zeros((h, w)), "half": np.where(xx < w // 2, 255, 0),
           "column": np.where(xx == w // 3, 255, 0), "checker4": np.where((yy // 4 + xx // 4) % 2 == 0, 255, 0),
           "values_1_254": np.where(yy < h // 2, 1, 254)}
    kp, _ = cvref.orb_cv2(img, 5000, 1.2, nlevels)   # an edge through the NMS neighbourhood of a level-0 corner
    k0 = kp[kp["octave"] == 0][len(kp[kp["octave"] == 0]) // 2]
    out["edge_at_corner"] = np.where(xx > int(k0["x"]), 255, 0)
    return {k: v.astype(np.uint8) for k, v in out.items()}


FIELDS = ["x", "y", "size", "angle", "response", "octave"]


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("nlevels", [1, 4, 8])
def test_orb_masked_equals_cv2(built, shape, nlevels):
    h, w = SHAPES[shape]
    img = texture(h, w, nlevels)
    with plf.Frontend(camera=dict(K, width=w, height=h), orb_nfeatures=1500, orb_nlevels=nlevels) as fe:
        base = fe.orb(img)
        for kind, m in masks(img, nlevels).items():
            kp, d = fe.orb(img, mask=m)
            rk, rd = om.orb(img, m, 1500, 1.2, nlevels)
            assert kp[FIELDS].tobytes() == rk[FIELDS].tobytes() and d.tobytes() == rd.tobytes(), (shape, nlevels, kind)
            if kind == "all255":
                assert kp.tobytes() == base[0].tobytes() and d.tobytes() == base[1].tobytes()
            if kind == "all0":
                assert len(kp) == 0
        # strided mask rows
        m = masks(img, nlevels)["half"]
        wide = np.zeros((h, w + 40), np.uint8)
        wide[:, :w] = m
        kp, d = fe.orb(img, mask=wide[:, :w])
        rk, rd = om.orb(img, m, 1500, 1.2, nlevels)
        assert kp[FIELDS].tobytes() == rk[FIELDS].tobytes() and d.tobytes() == rd.tobytes()


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("nfeat", [0, 300])
def test_detect_lines_masked_equals_oracle(built, shape, nfeat):
    h, w = SHAPES[shape]
    cam = dict(K, width=w, height=h, cx=w / 2, cy=h / 2)
    img = next(iter(synth.stream(cam, 1, world=synth.World(seed=5, n_quads=160, n_segs=90))))[0]
    with plf.Frontend(camera=cam, lsd_nfeatures=nfeat) as fe:
        base = fe.detect_lines(img)
        for kind, m in masks(img, 4).items():
            kl, d = fe.detect_lines(img, mask=m)
            rk, rd = om.detect_lines(img, m, nfeat)
            assert kl.tobytes() == rk.tobytes() and d.tobytes() == rd.tobytes(), (shape, nfeat, kind)
            if kind == "all255":
                assert kl.tobytes() == base[0].tobytes() and d.tobytes() == base[1].tobytes()
            if kind == "all0":
                assert len(kl) == 0


# ---- the batched pipeline ---------------------------------------------------------------------------------------
N = 5
PRM = dict(orb_nfeatures=1500, lsd_nfeatures=200)


def streams(cam, nseq):
    return [[f[:2] for f in synth.stream(cam, N, world=synth.World(seed=30 + s), seed=40 + s, step=0.1)] for s in range(nseq)]


def seq_masks(cam):
    """Sequence 0: left and right masked differently; 1: left only; 2: none; 3: right only."""
    h, w = cam["height"], cam["width"]
    yy, xx = np.mgrid[:h, :w]
    left = np.where(xx < int(0.6 * w), 255, 0).astype(np.uint8)
    right = np.where((yy > h // 5) & (xx > w // 8), 255, 0).astype(np.uint8)
    return {0: (left, right), 1: (right, None), 2: (None, None), 3: (None, left)}


def masked_fns(cam, pairs, mk):
    """orb_fn / lines_fn of run_sequence that apply each image's mask (the images identified by object)."""
    by_id = {}
    for L, R in pairs:
        by_id[id(L)], by_id[id(R)] = mk
    prm = dict(ofe.DEFAULTS, **PRM)

    def orb_fn(im):
        m = by_id[id(im)]
        if m is None:
            return ofe._orb_c(im, prm)
        return om.orb(im, m, prm["orb_nfeatures"], 1.2, prm["orb_nlevels"])

    def lines_fn(im):
        m = by_id[id(im)]
        if m is None:
            return ofe.detect_lines(im, prm["lsd_nfeatures"], prm["min_line_length"], ofe.lsd_kwargs(prm))
        return om.detect_lines(im, m, prm["lsd_nfeatures"], prm["min_line_length"], ofe.lsd_kwargs(prm))
    return orb_fn, lines_fn


def run_device(cam, seqs, mks, in_flight, **kw):
    lim = plf.default_limits()
    lim.max_batch = len(seqs)
    out = {}
    with plf.Frontend(camera=cam, limits=lim, max_sequences=len(seqs), **dict(PRM, **kw)) as fe:
        for s, (ml, mr) in mks.items():
            fe.set_sequence_mask(s, ml, mr)
            assert fe.sequence_mask_set(s) == (ml is not None, mr is not None)
        rng = np.random.default_rng(0)
        batches = [[(int(s), i) for s in rng.permutation(len(seqs))] for i in range(N)]
        pending = []
        for j, b in enumerate(batches):
            fe.batch_upload(np.stack([seqs[s][i][0] for s, i in b]), np.stack([seqs[s][i][1] for s, i in b]))
            fe.batch_run(len(b), seq=np.array([s for s, _ in b], np.int32))
            pending.append(b)
            if len(pending) == in_flight or j == len(batches) - 1:
                while pending:
                    bb = pending.pop(0)
                    res = fe.batch_download_array(len(bb))
                    for k, key in enumerate(bb):
                        out[key] = (res[k], fe.get_frame(k), fe.get_matches(k)) if in_flight == 1 else (res[k],)
    return out


def as_dict(r):
    return {f: (np.array(r[f]).reshape(4, 4) if f == "DT" else np.array(r[f]).reshape(6, 6) if f == "DT_cov" else r[f].item())
            for f in r.dtype.names}


@pytest.mark.parametrize("cam", [K, EUROC], ids=["kitti", "euroc"])
def test_pipeline_masked_sequences_match_oracle(built, cam):
    seqs = streams(cam, 4)
    mks = seq_masks(cam)
    got = run_device(cam, seqs, mks, 1)
    for s in range(4):
        orb_fn, lines_fn = masked_fns(cam, seqs[s], mks[s])
        ref = ofe.run_sequence(cam, seqs[s], PRM, orb_fn=orb_fn, lines_fn=lines_fn)
        compare(ref, [as_dict(got[(s, i)][0]) for i in range(N)], [got[(s, i)][1] for i in range(N)])
        for i in range(N):
            if ref[i]["status"] == 0:
                m, tr = got[(s, i)][2], ref[i]["res"]["rows"]
                assert np.array_equal(m["P"], tr["P"]) and np.array_equal(m["sP"], tr["sP"]), (s, i)
    three = run_device(cam, seqs, mks, 3)
    for key, v in three.items():
        assert v[0].tobytes() == got[key][0].tobytes(), key


def test_mask_set_between_batches_in_flight(built):
    cam = K
    seqs = streams(cam, 1)
    mk = seq_masks(cam)[0]
    lim = plf.default_limits()
    lim.max_batch = 1

    def run(set_after):
        res = []
        with plf.Frontend(camera=cam, limits=lim, **PRM) as fe:
            for i in range(3):
                fe.batch_upload(seqs[0][i][0][None], seqs[0][i][1][None])
                fe.batch_run(1)
                if i == set_after:
                    fe.set_sequence_mask(0, *mk)   # batches 0 .. i are in flight
            res = [fe.batch_download_array(1)[0] for _ in range(3)]
        return res

    a = run(set_after=0)
    never = run(set_after=99)
    assert a[0].tobytes() == never[0].tobytes()               # the batch in flight keeps no mask
    assert (a[1]["n_kp_l"], a[1]["n_kp_r"]) != (never[1]["n_kp_l"], never[1]["n_kp_r"])
    assert a[1]["status"] != 2 and a[2]["status"] != 2          # no restart
    orb_fn, lines_fn = masked_fns(cam, seqs[0][:3], mk)
    by_frame = lambda i: ofe.extract_stereo(cam, *seqs[0][i], dict(ofe.DEFAULTS, **PRM), orb_fn, lines_fn)
    assert a[1]["n_stereo_pt"] == len(by_frame(1).pt_pl) and a[2]["n_stereo_ls"] == len(by_frame(2).ls_spl)


def test_set_then_clear_is_never_set_and_refusals(built):
    cam = EUROC
    seqs = streams(cam, 2)
    mk = seq_masks(cam)[0]
    lim = plf.default_limits()
    lim.max_batch = 2

    def run(prepare):
        out = {}
        with plf.Frontend(camera=cam, limits=lim, max_sequences=2, **PRM) as fe:
            prepare(fe)
            for i in range(3):
                fe.batch_upload(np.stack([seqs[s][i][0] for s in range(2)]), np.stack([seqs[s][i][1] for s in range(2)]))
                fe.batch_run(2, seq=np.array([0, 1], np.int32))
                res = fe.batch_download_array(2)
                for k in range(2):
                    out[(k, i)] = (res[k], fe.get_frame(k), fe.get_matches(k))
        return out

    def set_clear(fe):
        fe.set_sequence_mask(1, *mk)
        fe.set_sequence_mask(1)
        assert fe.sequence_mask_set(1) == (False, False)

    assert_same(run(lambda fe: None), run(set_clear))
    with plf.Frontend(camera=cam, limits=lim, max_sequences=2, **PRM) as fe:
        fe.set_sequence_mask(0, mk[0])
        h, w = cam["height"], cam["width"]
        m = np.ascontiguousarray(mk[1])
        for s, stride in ((-1, w), (2, w), (0, w - 1)):
            st = fe.lib.plf_set_sequence_mask(fe._ctx, s, m.ctypes.data_as(C.POINTER(C.c_uint8)), None, stride)
            assert st == -1, (s, stride)
            assert fe.sequence_mask_set(0) == (True, False)
        for s in (-1, 2):
            with pytest.raises(plf.PlfError):
                fe.sequence_mask_set(s)
        fe.set_sequence_mask(0, None, mk[1])
        assert fe.sequence_mask_set(0) == (False, True)
        img = seqs[0][0][0]
        with pytest.raises(plf.PlfError):
            fe.orb(img, mask=m[:-1])
        assert fe.lib.plf_orb_masked(fe._ctx, img.ctypes.data_as(C.POINTER(C.c_uint8)), w, h, w, None, w, None, None, 0,
                                     C.byref(C.c_int())) == -1
        assert fe.lib.plf_detect_lines_masked(fe._ctx, img.ctypes.data_as(C.POINTER(C.c_uint8)), w, h, w,
                                              m.ctypes.data_as(C.POINTER(C.c_uint8)), w - 1, None, None, 0,
                                              C.byref(C.c_int())) == -1
    with plf.Frontend(camera=cam, limits=lim, max_sequences=2, **PRM) as fe:
        fe.set_sequence_mask(1, *mk)
        assert fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 3), "plf_set_max_sequences") is None
        assert fe.sequence_mask_set(1) == (False, False)
