"""GPU tests of the per-pair masks of the batched front-end (plf_batch_upload_masks).

- Moving masks (tests/pair_mask_cases.py) at KITTI and EuRoC shape, 1 / 4 / 8 levels, one and three batches in flight:
  bit-exact to oracle/frontend.py run_sequence with each image's own mask (cv2's detectAndCompute(img, mask) and the line
  rule of oracle/masks.py), the pose within the pipeline tests' tolerance.
- Pair masks equal to a sequence's masks give what plf_set_sequence_mask gives, bit for bit.  A pair mask with a sequence
  mask is their AND: bit-exact to the AND given as a pair mask alone, and to the oracle with the AND, left-only and
  right-only uploads and unmasked sequences in the same batches.
- Slots: three batches in flight, masked and unmasked by turns, equal the batches one at a time; the masks belong to
  their upload only; two image sizes in one context.
- Colour and rectified input equal a grey twin fed cv2.cvtColor(cv2.remap(...)) with the same masks; adaptive FAST and
  the motion model on match the oracle; masks in torch CUDA tensors, dense and row-strided, equal host masks.
- Every refusal changes nothing: the next batch is what it is without the refused call."""
import ctypes as C

import numpy as np
import pytest
import torch

import pair_mask_cases as pm
import plslam_b200 as plf
from oracle import frontend as ofe
from oracle import masks as om
from test_color_gpu import assert_identical, colour_pair, data, gray, remap, upload_color
from test_color_gpu import frontend as rect_frontend
from test_multi_sequence_gpu import assert_same
from test_pipeline_gpu import compare

pytestmark = pytest.mark.gpu

K = plf.KITTI_CAMERA
EUROC = plf.EUROC_CAMERA
PRM = dict(orb_nfeatures=1500, lsd_nfeatures=200)
N = 4


def both(a, b):
    """The pixelwise AND of two masks (None: no mask), as a 0 / 255 mask or None."""
    if a is None or b is None:
        return a if b is None else b
    return np.where((a != 0) & (b != 0), 255, 0).astype(np.uint8)


def round_robin(nseq, n=N, seed=0):
    rng = np.random.default_rng(seed)
    return [[(int(s), i) for s in rng.permutation(nseq)] for i in range(n)]


def lim(B):
    l = plf.default_limits()
    l.max_batch = B
    return l


def drive(fe, seqs, batches, pair_masks, in_flight, before=None, upload_masks=None):
    """The batches through fe, up to in_flight in flight.  pair_masks(j, batch) -> (left, right): [B, h, w] or None per
    side (both None: no pair masks).  Returns {(s, i): (row, frame, matches)} (frame and matches with in_flight 1)."""
    out, pending = {}, []

    def drain():
        b = pending.pop(0)
        res = fe.batch_download_array(len(b))
        for k, key in enumerate(b):
            out[key] = (res[k], fe.get_frame(k), fe.get_matches(k)) if in_flight == 1 else (res[k],)

    for j, b in enumerate(batches):
        while len(pending) >= in_flight:
            drain()
        if before:
            before(fe, j, b)
        fe.batch_upload(np.stack([seqs[s][i][0] for s, i in b]), np.stack([seqs[s][i][1] for s, i in b]))
        ml, mr = pair_masks(j, b)
        if ml is not None or mr is not None:
            (upload_masks or fe.batch_upload_masks)(ml, mr)
        fe.batch_run(len(b), seq=np.array([s for s, _ in b], np.int32))
        pending.append(b)
    while pending:
        drain()
    return out


def oracle_fns(prm, masks_by_id):
    """orb_fn / lines_fn of run_sequence applying each image's mask (by image object; None: unmasked)."""
    p = dict(ofe.DEFAULTS, **prm)

    def orb_fn(im):
        m = masks_by_id.get(id(im))
        return ofe._orb_c(im, p) if m is None else om.orb(im, m, p["orb_nfeatures"], 1.2, p["orb_nlevels"], fast_th=p["orb_fast_th"])

    def lines_fn(im):
        m = masks_by_id.get(id(im))
        if m is None:
            return ofe.detect_lines(im, p["lsd_nfeatures"], p["min_line_length"], ofe.lsd_kwargs(p))
        return om.detect_lines(im, m, p["lsd_nfeatures"], p["min_line_length"], ofe.lsd_kwargs(p))
    return orb_fn, lines_fn


def as_dict(r):
    return {f: (np.array(r[f]).reshape(4, 4) if f == "DT" else np.array(r[f]).reshape(6, 6) if f == "DT_cov" else r[f].item())
            for f in r.dtype.names}


def check_oracle(cam, seqs, got, prm, eff):
    """Each sequence against run_sequence with eff(s, i, side) as its images' masks."""
    for s in range(len(seqs)):
        by_id = {id(seqs[s][i][side]): eff(s, i, side) for i in range(len(seqs[s])) for side in (0, 1)}
        orb_fn, lines_fn = oracle_fns(prm, by_id)
        ref = ofe.run_sequence(cam, seqs[s], prm, orb_fn=orb_fn, lines_fn=lines_fn)
        n = len(seqs[s])
        compare(ref, [as_dict(got[(s, i)][0]) for i in range(n)], [got[(s, i)][1] for i in range(n)])
        for i in range(n):
            if ref[i]["status"] == 0:
                m, tr = got[(s, i)][2], ref[i]["res"]["rows"]
                assert np.array_equal(m["P"], tr["P"]) and np.array_equal(m["sP"], tr["sP"]), (s, i)


def moving_of(cam):
    h, w = cam["height"], cam["width"]
    return lambda s, i, side: pm.moving(h, w, i, side, seed=s)


@pytest.mark.parametrize("nlevels", [1, 4, 8])
@pytest.mark.parametrize("cam", [K, EUROC], ids=["kitti", "euroc"])
def test_moving_masks_match_oracle(built, cam, nlevels):
    seqs = pm.streams(cam, 3, N)
    prm = dict(PRM, orb_nlevels=nlevels)
    mv = moving_of(cam)
    masks = lambda j, b: tuple(np.stack([mv(s, i, side) for s, i in b]) for side in (0, 1))
    batches = round_robin(3)
    got = {}
    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **prm) as fe:
        got = drive(fe, seqs, batches, masks, 1)
    check_oracle(cam, seqs, got, prm, mv)
    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **prm) as fe:
        three = drive(fe, seqs, batches, masks, 3)
    for key, v in three.items():
        assert v[0].tobytes() == got[key][0].tobytes(), key


def seq_masks(cam):
    """Sequence 0: a hood mask on both images; 1: on the left only; 2: none; 3: a sparse mask on the right only."""
    h, w = cam["height"], cam["width"]
    H, (S, _) = pm.hood(h, w), pm.sparse_pair(h, w)
    return {0: (H, H), 1: (H, None), 2: (None, None), 3: (None, S)}


def test_pair_masks_equal_sequence_masks(built):
    cam = EUROC
    seqs = pm.streams(cam, 4, N)
    sm = seq_masks(cam)
    full = np.full((cam["height"], cam["width"]), 255, np.uint8)
    batches = round_robin(4, seed=1)

    def by_sequence(fe):
        for s, (l, r) in sm.items():
            fe.set_sequence_mask(s, l, r)

    with plf.Frontend(camera=cam, limits=lim(4), max_sequences=4, **PRM) as fe:
        by_sequence(fe)
        ref = drive(fe, seqs, batches, lambda j, b: (None, None), 1)
    pairs = lambda j, b: tuple(np.stack([full if sm[s][side] is None else sm[s][side] for s, _ in b]) for side in (0, 1))
    with plf.Frontend(camera=cam, limits=lim(4), max_sequences=4, **PRM) as fe:
        got = drive(fe, seqs, batches, pairs, 1)
    assert_same(ref, got)


def test_and_with_sequence_masks(built):
    """Batch j uploads pair masks on both sides (j % 3 == 0), the left only (1) or the right only (2); sequence 3's right
    pair masks are the sparse mask whose AND with its sequence mask has another pyramid than the AND of the pyramids."""
    cam = K
    h, w = cam["height"], cam["width"]
    seqs = pm.streams(cam, 4, 6)
    sm = seq_masks(cam)
    _, P = pm.sparse_pair(h, w)
    full = np.full((h, w), 255, np.uint8)

    def pair(s, i, side):
        return P if (s, side) == (3, 1) else pm.moving(h, w, i, side, seed=s)

    sides = lambda j: {0: (0, 1), 1: (0,), 2: (1,)}[j % 3]
    batches = round_robin(4, 6, seed=2)

    def eff(s, i, side):
        j = next(j for j, b in enumerate(batches) if (s, i) in b)
        return both(sm[s][side], pair(s, i, side) if side in sides(j) else None)

    def with_sequence_masks(j, b):
        return tuple(np.stack([pair(s, i, side) for s, i in b]) if side in sides(j) else None for side in (0, 1))

    def and_alone(j, b):
        return tuple(np.stack([full if eff(s, i, side) is None else eff(s, i, side) for s, i in b]) for side in (0, 1))

    with plf.Frontend(camera=cam, limits=lim(4), max_sequences=4, **PRM) as fe:
        for s, (l, r) in sm.items():
            fe.set_sequence_mask(s, l, r)
        got = drive(fe, seqs, batches, with_sequence_masks, 1)
    with plf.Frontend(camera=cam, limits=lim(4), max_sequences=4, **PRM) as fe:
        alone = drive(fe, seqs, batches, and_alone, 1)
    assert_same(alone, got)
    check_oracle(cam, seqs, got, PRM, eff)


def test_slots_in_flight_and_ownership(built):
    """Three in flight with other masks in every batch and every second batch unmasked, against one at a time; masks
    belong to their upload: a second upload before the run drops them."""
    cam = EUROC
    h, w = cam["height"], cam["width"]
    seqs = pm.streams(cam, 3, 6)
    batches = round_robin(3, 6, seed=3)
    masks = lambda j, b: ((None, None) if j % 2 else tuple(np.stack([pm.moving(h, w, i + j, side, seed=s) for s, i in b])
                                                           for side in (0, 1)))
    outs = []
    for in_flight in (1, 3):
        with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
            outs.append(drive(fe, seqs, batches, masks, in_flight))
    for key in outs[0]:
        assert outs[0][key][0].tobytes() == outs[1][key][0].tobytes(), key
    assert any(outs[0][(s, 0)][0]["n_kp_l"] != 0 for s in range(3))

    def dropped(fe, j, b):   # an upload with masks that is never run
        fe.batch_upload(np.stack([seqs[s][i][1] for s, i in b]), np.stack([seqs[s][i][0] for s, i in b]))
        fe.batch_upload_masks(np.zeros((len(b), h, w), np.uint8), None)

    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
        a = drive(fe, seqs, batches, lambda j, b: (None, None), 1, before=dropped)
    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
        b = drive(fe, seqs, batches, lambda j, b: (None, None), 1)
    assert_same(a, b)


def test_two_image_sizes(built):
    """Sequences 0, 1 at KITTI's size and 2, 3 at EuRoC's, batches of one size by turns, three in flight with pair masks
    on every second batch of each size, against one at a time and the oracle."""
    cams = [K, K, EUROC, EUROC]
    seqs = pm.streams(K, 2, N) + pm.streams(EUROC, 4, N)[2:]
    batches = [[(s, i) for s in ((0, 1) if j % 2 == 0 else (2, 3))] for i in range(N) for j in range(2)]
    mv = lambda s, i, side: pm.moving(cams[s]["height"], cams[s]["width"], i, side, seed=s) if (i % 2 == 0) else None
    masks = lambda j, b: ((None, None) if mv(*b[0], 0) is None else
                          tuple(np.stack([mv(s, i, side) for s, i in b]) for side in (0, 1)))
    outs = []
    for in_flight in (1, 3):
        with plf.Frontend(camera=K, limits=lim(2), max_sequences=4, image_sizes=[(EUROC["width"], EUROC["height"])], **PRM) as fe:
            for s in (2, 3):
                fe.set_sequence_camera(s, EUROC)
            outs.append(drive(fe, seqs, batches, masks, in_flight))
    for key in outs[0]:
        assert outs[0][key][0].tobytes() == outs[1][key][0].tobytes(), key
    for s in range(4):
        check_oracle(cams[s], [seqs[s]], {(0, i): outs[0][(s, i)] for i in range(N)}, PRM, lambda _, i, side: mv(s, i, side))


def test_colour_and_rectified_equal_grey_twin(built):
    """Sequence 0 rectified from raw colour pairs, 1 with a sequence mask, all with moving pair masks, three in flight;
    the twin is fed cv2.cvtColor(cv2.remap(raw colour)) grey pairs and the same masks."""
    d = data()
    h, w = d["cam"]["height"], d["cam"]["width"]
    batches = round_robin(4, 6, seed=4)
    hood = pm.hood(h, w)

    def grey(s, i):
        L, R = colour_pair(s, i, raw=s == 0)
        if s == 0:
            L, R = remap(L, d["left"]), remap(R, d["right"])
        return gray(L), gray(R)

    out = []
    for colour in (True, False):
        with rect_frontend(4) as fe:
            if colour:
                fe.set_sequence_rectification(0, left=d["left"], right=d["right"])
            fe.set_sequence_mask(1, hood, None)
            res, pending = {}, []
            for j, b in enumerate(batches):
                while len(pending) >= 3:
                    bb = pending.pop(0)
                    for k, r in enumerate(fe.batch_download_array(len(bb))):
                        res[bb[k]] = (r,)
                pairs = [colour_pair(s, i, raw=s == 0) if colour else grey(s, i) for s, i in b]
                L, R = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
                if colour:
                    upload_color(fe, L, R, j % 2 == 1)
                else:
                    fe.batch_upload(L, R)
                fe.batch_upload_masks(*(np.stack([pm.moving(h, w, i, side, seed=s) for s, i in b]) for side in (0, 1)))
                fe.batch_run(len(b), seq=np.array([s for s, _ in b], np.int32))
                pending.append(b)
            last = pending[-1]
            while pending:
                bb = pending.pop(0)
                for k, r in enumerate(fe.batch_download_array(len(bb))):
                    res[bb[k]] = (r,)
            for k, key in enumerate(last):
                res[key] = res[key] + (fe.get_frame(k), fe.get_matches(k))
            out.append(res)
    assert_identical(*out)


def test_adaptive_fast_and_motion_model_match_oracle(built):
    cam = K
    seqs = pm.streams(cam, 3, 5)
    mv = moving_of(cam)
    batches = round_robin(3, 5, seed=5)
    used, ths = {}, {}

    def before(fe, j, b):
        for s, i in b:
            used[(s, i)] = fe.sequence_motion(s)[0]
            ths[(s, i)] = fe.sequence_fast_th(s)

    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
        fe.set_adaptive_fast({})
        fe.set_motion_model(True)
        got = drive(fe, seqs, batches, lambda j, b: tuple(np.stack([mv(s, i, side) for s, i in b]) for side in (0, 1)), 1,
                    before=before)
    assert len({v for v in ths.values()}) > 1   # the thresholds do adapt
    # each pair's oracle detection at the threshold the device used, from the prediction it used
    for s in range(3):
        by_id = {id(seqs[s][i][side]): mv(s, i, side) for i in range(5) for side in (0, 1)}
        ref = ofe.run_sequence(cam, seqs[s], PRM, orb_fn=None, lines_fn=None, motion_model=True,
                               preds=[used[(s, i)] for i in range(5)], fast_th=[ths[(s, i)] for i in range(5)],
                               frames=[ofe.extract_stereo(cam, *seqs[s][i], dict(ofe.DEFAULTS, **PRM, orb_fast_th=ths[(s, i)]),
                                                          *oracle_fns(dict(PRM, orb_fast_th=ths[(s, i)]), by_id))
                                       for i in range(5)])
        compare(ref, [as_dict(got[(s, i)][0]) for i in range(5)], [got[(s, i)][1] for i in range(5)])


@pytest.mark.parametrize("strided", [False, True], ids=["dense", "row-strided"])
def test_device_resident_masks(built, strided):
    cam = K
    h, w = cam["height"], cam["width"]
    seqs = pm.streams(cam, 3, N)
    batches = round_robin(3, seed=6)
    host = lambda j, b: (np.stack([pm.moving(h, w, i, 0, seed=s) for s, i in b]), None if j % 2 else
                         np.stack([pm.moving(h, w, i, 1, seed=s) for s, i in b]))
    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
        ref = drive(fe, seqs, batches, host, 1)
    keep = []

    def device_upload(fe):
        def up(ml, mr):
            ptrs, stride = [], w + (48 if strided else 0)
            for m in (ml, mr):
                if m is None:
                    ptrs.append(0)
                    continue
                t = torch.zeros((m.shape[0], h, stride), dtype=torch.uint8, device="cuda")
                t[:, :, :w] = torch.from_numpy(m).cuda()
                keep.append(t)   # unchanged until the batch is downloaded
                ptrs.append(t.data_ptr())
            torch.cuda.synchronize()
            fe.batch_upload_masks_raw(ml.shape[0], ptrs[0], ptrs[1], stride)
        return up

    with plf.Frontend(camera=cam, limits=lim(3), max_sequences=3, **PRM) as fe:
        got = drive(fe, seqs, batches, host, 1, upload_masks=device_upload(fe))
    assert_same(ref, got)


def test_refusals_change_nothing(built):
    cam = EUROC
    h, w = cam["height"], cam["width"]
    seqs = pm.streams(cam, 2, 3)
    batches = round_robin(2, 3, seed=7)
    masks = lambda j, b: tuple(np.stack([pm.moving(h, w, i, side, seed=s) for s, i in b]) for side in (0, 1))
    m = np.ascontiguousarray(pm.moving(h, w, 0, 0)[None].repeat(2, 0))
    p = m.ctypes.data_as(C.POINTER(C.c_uint8))
    with plf.Frontend(camera=cam, limits=lim(2), max_sequences=2, **PRM) as fe:
        assert fe.lib.plf_batch_upload_masks(fe._ctx, 2, p, p, w) == -5   # no upload yet
        assert "no upload" in fe.lib.plf_last_error(fe._ctx).decode()

    def refused(fe, j, b):
        if j == 0:
            return
        for B, l, r, stride in ((0, p, p, w), (3, p, p, w), (2, None, None, w), (2, p, p, w - 1)):
            assert fe.lib.plf_batch_upload_masks(fe._ctx, B, l, r, stride) == -1, (B, stride)
        if torch.cuda.device_count() > 1:   # device memory of another device
            t = torch.zeros((2, h, w), dtype=torch.uint8, device="cuda:1")
            assert fe.lib.plf_batch_upload_masks(fe._ctx, 2, C.c_void_p(t.data_ptr()), None, w) == -1

    def run_b_mismatch(ml, mr):
        fe_ = run_b_mismatch.fe
        fe_.batch_upload_masks(ml, mr)
        assert fe_.lib.plf_batch_run_sequences(fe_._ctx, 1, None, None) == -1
        assert "masks" in fe_.lib.plf_last_error(fe_._ctx).decode()

    with plf.Frontend(camera=cam, limits=lim(2), max_sequences=2, **PRM) as fe:
        ref = drive(fe, seqs, batches, masks, 1)
    with plf.Frontend(camera=cam, limits=lim(2), max_sequences=2, **PRM) as fe:
        run_b_mismatch.fe = fe
        got = drive(fe, seqs, batches, masks, 1, before=refused, upload_masks=run_b_mismatch)
    assert_same(ref, got)
    with pytest.raises(plf.PlfError):
        with plf.Frontend(camera=cam, limits=lim(2), **PRM) as fe:
            fe.batch_upload(seqs[0][0][0][None], seqs[0][0][1][None])
            fe.batch_upload_masks(None, None)
