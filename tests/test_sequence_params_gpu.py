"""GPU tests of per-sequence front-end settings in one batched context (plf_set_sequence_params / plf_get_sequence_params).

The oracle is the library itself: every pair of a batch whose sequences have their own settings must give, bit for bit,
what a single-sequence context created with those settings gives for the same frames in the same order - every
plf_frame_result field (DT included), get_frame(k) and get_matches(k).  The single-context path at the reference configs
is pinned to the CPU oracle by test_params_gpu.py; test_kitti_sequence_in_euroc_context_against_the_oracle checks one
mixed context against it directly."""
import cv2
import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, synth
from oracle import frontend as ofe
from param_cases import ORB_CASES, PIPELINE_SWEEPS, REFERENCE_CONFIGS
from test_multi_sequence_gpu import assert_same, interleavings
from test_pipeline_gpu import POSE_REL_TOL, check_frame, rel

pytestmark = pytest.mark.gpu

W, H = 640, 360
CAM = dict(plf.KITTI_CAMERA, width=W, height=H, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
LENGTHS = (8, 12, 10, 9)
CLASSES = plf.sequence_param_fields()
# the four sequences of the mixed runs: one per reference config, the last at the defaults (config_euroc.yaml)
NAMES = ("kitti", "config", "full", "defaults")

_FRAMES = {}


def full(name="defaults", **over):
    """Every plf_params field of a reference config (or the defaults), with `over` on top."""
    return {**ofe.DEFAULTS, **(REFERENCE_CONFIGS[name] if name != "defaults" else {}), **over}


def sequences(cam=CAM, lengths=LENGTHS, seed=40):
    key = (tuple(sorted(cam.items())), lengths, seed)
    if key not in _FRAMES:
        seqs = []
        for s, n in enumerate(lengths):
            world = synth.World(seed=seed + s, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
            seqs.append([(L, R) for L, R, _ in synth.stream(cam, n, world=world, seed=seed + 10 + s, step=0.15)])
        _FRAMES[key] = seqs
    return _FRAMES[key]


def limits(B):
    lim = plf.default_limits()
    lim.max_batch = B
    return lim


def collect(fe, keys, res, out, views=True):
    for k, key in enumerate(keys):
        out[key] = (res[k], fe.get_frame(k), fe.get_matches(k)) if views else (res[k],)


def alone(seqs, segments, cam=CAM):
    """segments: (s, a, b, params) - pairs a .. b-1 of sequence s through a single-sequence context created with those
    params, reset first.  Returns {(s, i): (result, frame, matches)}."""
    out = {}
    for s, a, b, prm in segments:
        with plf.Frontend(camera=cam, limits=limits(b - a), **prm) as fe:
            fe.batch_upload(np.stack([f[0] for f in seqs[s][a:b]]), np.stack([f[1] for f in seqs[s][a:b]]))
            fe.batch_run(b - a)
            collect(fe, [(s, i) for i in range(a, b)], fe.batch_download_array(b - a), out)
    return out


def batch_args(seqs, batch):
    L = np.stack([seqs[s][i][0] for s, i in batch])
    R = np.stack([seqs[s][i][1] for s, i in batch])
    return L, R, np.array([s for s, _ in batch], np.int32)


def mixed(seqs, batches, ctx_prm, own, in_flight=0, cam=CAM, changes=None):
    """The batches through one context created with ctx_prm; sequence s gets own[s] (None: the context's) before the
    first batch, and changes[j] = (s, params or None) before batch j.  Up to in_flight batches stay undownloaded (the
    frames and matches are then not collected)."""
    out, pending = {}, []
    with plf.Frontend(camera=cam, limits=limits(max(map(len, batches))), max_sequences=len(seqs), **ctx_prm) as fe:
        for s, p in enumerate(own):
            if p is not None:
                fe.set_sequence_params(s, **p)
        for j, batch in enumerate(batches):
            if changes and j in changes:
                assert len(pending) == in_flight
                s, p = changes[j]
                if p is None:
                    fe.set_sequence_params(s)
                else:
                    fe.set_sequence_params(s, **p)
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq)
            pending.append(batch)
            while len(pending) > in_flight or (pending and j == len(batches) - 1):
                b = pending.pop(0)
                collect(fe, b, fe.batch_download_array(len(b)), out, in_flight == 0)
    return out


def assert_same_results(ref, got, keys=None):
    for key in keys if keys is not None else ref:
        for f in ref[key][0].dtype.names:
            assert ref[key][0][f].tobytes() == got[key][0][f].tobytes(), (key, f)


def configs(strategy):
    """The four sequences' settings in a context at matching_strategy `strategy`: every one at 0 in a strategy-0 context,
    sequences 1 and 3 windowed (3) in a strategy-3 one."""
    return [full(n, matching_strategy=strategy if s % 2 else 0) for s, n in enumerate(NAMES)]


@pytest.mark.parametrize("strategy", [0, 3])
def test_mixed_configs_equal_each_sequence_alone(built, strategy):
    """Four sequences, one per reference config, in the four interleavings of test_multi_sequence_gpu.py: every pair
    equals its sequence alone in a context created with its config.  At strategy 3, windowed and descriptor-only
    sequences share the batches."""
    seqs = sequences()
    own = configs(strategy)
    ref = alone(seqs, [(s, 0, LENGTHS[s], own[s]) for s in range(4)])
    tracked = sum(r["status"] == 0 for r, _, _ in ref.values())
    assert tracked >= 0.75 * (sum(LENGTHS) - len(LENGTHS)), tracked
    for name, batches in interleavings(LENGTHS).items():
        got = mixed(seqs, batches, full(matching_strategy=strategy), own)
        assert_same(ref, got)
        for s in range(4):
            assert got[(s, 0)][0]["status"] == 2, (name, s)


@pytest.mark.parametrize("in_flight", [0, 2])
def test_change_mid_stream(built, in_flight):
    """Round robin (B = 4) in a strategy-3 context.  Before batch 3, with `in_flight` batches not yet downloaded,
    sequence 1 gets the KITTI config (strategy 0); before batch 7, None returns it to the context's settings.  Batches
    already run are unchanged, the restart lands on sequence 1's pair of batch 3 (and of batch 7), and from there it
    equals a fresh context of the new settings; the other sequences are untouched."""
    seqs = sequences()
    ctx = full(matching_strategy=3)
    own = configs(3)
    new = full("kitti")
    batches = interleavings(LENGTHS)["round_robin"]
    j1, j2 = 3, 7
    segs = [(s, 0, LENGTHS[s], own[s]) for s in range(4) if s != 1]
    segs += [(1, 0, j1, own[1]), (1, j1, j2, new), (1, j2, LENGTHS[1], ctx)]
    ref = alone(seqs, segs)
    base = mixed(seqs, batches, ctx, own)
    got = mixed(seqs, batches, ctx, own, in_flight, changes={j1: (1, new), j2: (1, None)})
    if in_flight == 0:
        assert_same(ref, got)
    else:
        assert_same_results(ref, got)
    assert_same_results(base, got, [key for key in got if key[0] != 1 or key[1] < j1])
    assert got[(1, j1)][0]["status"] == 2 and got[(1, j2)][0]["status"] == 2
    assert got[(1, j1 + 1)][0]["status"] == 0 and got[(1, j2 + 1)][0]["status"] == 0


# the context of the windowed matcher's fields: a window of 0 cells keeps few enough frame-to-frame matches that
# min_pt_matches / min_ls_matches can decide the match() fall-back (test_pipeline_gpu.py's fallback case)
WINDOWED_CTX = dict(matching_strategy=3, matching_f2f_ws=0)


def field_changes():
    """(field, values, ctx strategy) for every per-sequence field: the values its sweep (param_cases.PIPELINE_SWEEPS) and
    the reference configs give it away from the defaults, else ORB_CASES', else a few of its own.  The windowed matcher's
    fields are run in a strategy-3 context."""
    vals = {f: [] for f, c in CLASSES.items() if c == "sequence"}
    windowed = {"matching_s_ws", "matching_f2f_ws", "min_pt_matches", "min_ls_matches", "line_sim_th", "matching_strategy"}
    for case in PIPELINE_SWEEPS.values():
        for f, v in case["change"].items():
            vals[f].append(v)
    for cfg in list(REFERENCE_CONFIGS.values()) + list(ORB_CASES.values()):
        for f, v in cfg.items():
            if f in vals and f not in windowed:
                vals[f].append(v)
    # orb_fast_th: the configs' 20 and ORB_CASES' 7 and 40 leave the top orb_nfeatures corners of these scenes as they
    # are; min_error: the sweep moves it together with min_error_change
    own = {"matching_strategy": [0], "matching_f2f_ws": [1, 6], "min_pt_matches": [60, 150, 300, 450, 600, 800],
           "min_ls_matches": [30, 80, 150], "min_features": [60, 200, 1000], "orb_fast_th": [60, 100],
           "min_error": [0.1, 1.0, 10.0]}
    out = []
    for f in sorted(vals):
        st = 3 if f in windowed else 0
        d = full(**WINDOWED_CTX) if st else full()
        v = [x for x in dict.fromkeys(vals[f] + own.get(f, [])) if x != d[f] and (f != "orb_nlevels" or x <= d[f])]
        out.append((f, v, st))
    return out


def test_every_sequence_field_has_an_effect(built):
    """Each per-sequence field set alone on sequences of one context: each changes its sequence's results for at least
    one of its values, and the sequence left at the context's settings equals a context that never set any.  Every
    sequence sees the same frames, round robin."""
    changes = field_changes()
    assert {f for f, _, _ in changes} == {f for f, c in CLASSES.items() if c == "sequence"}
    assert all(v for _, v, _ in changes), [f for f, v, _ in changes if not v]
    n = 5
    frames = sequences(lengths=(n,))[0]
    for strategy in (0, 3):
        own = [None] + [{f: x} for f, v, st in changes if st == strategy for x in v]
        keys = [None] + [(f, x) for f, v, st in changes if st == strategy for x in v]
        seqs = [frames] * len(own)
        ctx = full(**WINDOWED_CTX) if strategy else full()
        got = mixed(seqs, [[(s, i) for s in range(len(seqs))] for i in range(n)], ctx, own)
        plain = alone([frames], [(0, 0, n, ctx)])
        assert_same(plain, {(0, i): got[(0, i)] for i in range(n)})
        moved = {}
        for s in range(1, len(seqs)):
            f, _ = keys[s]
            differs = any(a.tobytes() != b.tobytes()
                          for i in range(n) for x, y in zip(got[(0, i)], got[(s, i)])
                          for a, b in ([(x[k], y[k]) for k in x.dtype.names] if hasattr(x, "dtype")
                                       else [(x[k], y[k]) for k in x]))
            moved[f] = moved.get(f, False) or differs
        assert all(moved.values()), [f for f, m in moved.items() if not m]


def test_one_level_sequence_in_four_level_context(built):
    """A sequence at orb_nlevels 1 (config_fast.yaml's ORB) beside a 4-level one: it equals a 1-level context alone, its
    keypoints are cv2.ORB_create(..., nlevels=1)'s (the count of every image, and every stereo point's position), and no
    batch reports an overflow."""
    seqs = sequences(lengths=(6, 6))
    one = full(orb_nlevels=1, orb_nfeatures=600)
    ref = alone(seqs, [(0, 0, 6, full()), (1, 0, 6, one)])
    got = mixed(seqs, [[(0, i), (1, i)] for i in range(6)], full(), [None, one])
    assert_same(ref, got)
    orb = cv2.ORB_create(600, 1.2, 1, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
    for i in range(6):
        r, fr, _ = got[(1, i)]
        kl = orb.detect(seqs[1][i][0], None)
        kr = orb.detect(seqs[1][i][1], None)
        assert (r["n_kp_l"], r["n_kp_r"]) == (len(kl), len(kr)), i
        pts = {(np.float32(k.pt[0]), np.float32(k.pt[1])) for k in kl}
        assert all((np.float32(x), np.float32(y)) in pts for x, y in fr["pt_pl"]), i
        assert np.all(fr["pt_octave"] == 0), i
        assert np.any(got[(0, i)][1]["pt_octave"] > 0), i


def test_adaptive_fast_and_motion_model(built):
    """Adaptive FAST and the motion model on, round robin: each sequence's first frame is detected at its own
    orb_fast_th (sequence_fast_th before the first batch), and every pair equals its sequence alone in a context of
    its settings with the same two switches."""
    cfg = dict(min_th=5, max_th=50, inc_th=5, feat_th=50, err_th=0.5)
    seqs = sequences()
    own = [dict(c, orb_fast_th=th) for c, th in zip(configs(3), (12, 20, 27, 35))]
    ref = {}
    for s in range(4):
        with plf.Frontend(camera=CAM, limits=limits(1), adaptive_fast=cfg, motion_model=True, **own[s]) as fe:
            for i in range(LENGTHS[s]):
                fe.batch_upload(seqs[s][i][0][None], seqs[s][i][1][None])
                fe.batch_run(1)
                collect(fe, [(s, i)], fe.batch_download_array(1), ref)
    got = {}
    batches = interleavings(LENGTHS)["round_robin"]
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=4, adaptive_fast=cfg, motion_model=True,
                      **full(matching_strategy=3)) as fe:
        for s in range(4):
            fe.set_sequence_params(s, **own[s])
            assert fe.sequence_fast_th(s) == own[s]["orb_fast_th"]
        for batch in batches:
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            fe.batch_run(len(batch), seq=seq)
            collect(fe, batch, fe.batch_download_array(len(batch)), got)
    assert_same(ref, got)


def test_two_image_sizes_two_configs(built):
    """A KITTI-shape sequence with the KITTI config and a EuRoC-shape sequence with the EuRoC config (the defaults) in one
    context, alternating batches: each equals its own context alone."""
    kitti = dict(plf.KITTI_CAMERA)
    euroc = dict(width=752, height=480, fx=435.2, fy=435.2, cx=367.2, cy=252.2, b=0.11)
    n = 4
    seqs = [sequences(kitti, (n,), 80)[0], sequences(euroc, (n,), 90)[0]]
    prm = [full("kitti"), full()]
    ref = {}
    for s, cam in enumerate((kitti, euroc)):
        ref.update({(s, i): v for (_, i), v in alone([seqs[s]], [(0, 0, n, prm[s])], cam=cam).items()})
    got = {}
    with plf.Frontend(camera=kitti, limits=limits(2), max_sequences=2, image_sizes=[(752, 480)], **full()) as fe:
        fe.set_sequence_camera(1, euroc)
        fe.set_sequence_params(0, **prm[0])
        for i in range(0, n, 2):
            for s in (0, 1):   # alternating sizes, two pairs per batch
                batch = [(s, i), (s, i + 1)]
                L, R, seq = batch_args(seqs, batch)
                fe.batch_upload(L, R)
                fe.batch_run(2, seq=seq)
                collect(fe, batch, fe.batch_download_array(2), got)
    assert_same(ref, got)


def test_kitti_sequence_in_euroc_context_against_the_oracle(built):
    """A KITTI-config sequence in a context of the EuRoC config (the defaults), against oracle/frontend.run_sequence with
    the KITTI config: features bit-exact, matches and inliers exact, pose to 1e-4."""
    prm = full("kitti")
    pairs = sequences(lengths=(4,))[0]
    ref = ofe.run_sequence(CAM, pairs, prm)
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=2, **full()) as fe:
        fe.set_sequence_params(1, **prm)
        res = fe.process_batch(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), seq=[1] * 4)
        for k, (r, g) in enumerate(zip(ref, res)):
            assert g["status"] == r["status"], k
            assert (g["n_stereo_pt"], g["n_stereo_ls"]) == (r["n_pt"], r["n_ls"]), k
            check_frame(fe.get_frame(k), r["frame"])
            if r["status"] == 0:
                assert g["n_matched_pt"] == len(r["res"]["inlier_pt"]) and g["n_matched_ls"] == len(r["res"]["inlier_ls"])
                assert (g["n_inliers_pt"], g["n_inliers_ls"]) == r["res"]["n_inliers"], k
                assert rel(clib.logmap_se3(g["DT"]), clib.logmap_se3(r["DT"])) < POSE_REL_TOL, k
    assert sum(r["status"] == 0 for r in ref) >= 2


def params_dict(p):
    return {k: getattr(p, k) for k, _ in plf.plf_params._fields_}


def test_defaults_refusals_and_launch_count(built):
    """plf_get_sequence_params round-trips and NULL restores the context's; every refusal returns PLF_ERR_INVALID naming
    the field and changes nothing (the next batch tracks on, equal to the uninterrupted run); plf_set_max_sequences drops
    the settings and plf_reset_sequence keeps them; a batch with no sequence settings launches what it launches on a
    context that never called plf_set_sequence_params, and so does a batch of the sequence that has them."""
    seqs = sequences()
    ctx = full(matching_strategy=0)
    kit = full("kitti")
    batches = [[(0, 0), (1, 0), (0, 1), (1, 1)], [(1, 2), (0, 2), (1, 3), (0, 3)]]
    ref = alone(seqs, [(0, 0, 4, ctx), (1, 0, 4, kit)])
    bad = [(dict(kit, orb_nlevels=5), r"orb_nlevels = 5, need 1 <= orb_nlevels <= the context's 4"),
           (dict(kit, orb_nlevels=0), r"orb_nlevels = 0"),
           (dict(kit, matching_strategy=3), r"matching_strategy = 3, and the context's is 0")]
    for f, c in CLASSES.items():
        if c == "context":
            v = kit[f]
            bad.append((dict(kit, **{f: v + 1 if isinstance(v, int) else v * 1.5 + 1}), rf"\b{f} = .*the context's is"))
        elif c == "sequence":
            if isinstance(kit[f], int):
                bad.append((dict(kit, **{f: -1}), rf"\b{f} = -1, need {f} >= 0"))
            else:
                for v in (float("nan"), float("inf")):
                    bad.append((dict(kit, **{f: v}), rf"\b{f} = .*need a finite value"))
    got = {}
    with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=2, **ctx) as fe:
        assert params_dict(fe.get_sequence_params(1)) == params_dict(fe.params)
        fe.set_sequence_params(1, **kit)
        assert params_dict(fe.get_sequence_params(1)) == params_dict(plf.plf_params(**kit))
        for j, batch in enumerate(batches):
            L, R, seq = batch_args(seqs, batch)
            fe.batch_upload(L, R)
            if j == 1:
                for p, msg in bad:
                    with pytest.raises(plf.PlfError, match=r"plf_set_sequence_params failed \(-1\).*" + msg):
                        fe.set_sequence_params(1, **p)
                for s in (-1, 2):
                    with pytest.raises(plf.PlfError, match=rf"plf_set_sequence_params failed \(-1\).*s = {s} outside"):
                        fe.set_sequence_params(s, **kit)
                    with pytest.raises(plf.PlfError, match=rf"plf_get_sequence_params failed \(-1\).*s = {s} outside"):
                        fe.get_sequence_params(s)
                assert fe.lib.plf_set_sequence_params(None, 0, None) == -1
                assert fe.lib.plf_get_sequence_params(None, 0, None) == -1
                assert params_dict(fe.get_sequence_params(1)) == params_dict(plf.plf_params(**kit))
            fe.batch_run(4, seq=seq)
            collect(fe, batch, fe.batch_download_array(4), got)
        assert_same(ref, got)
        assert all(got[key][0]["status"] == 0 for key in batches[1])
        fe.set_sequence_params(1)
        assert params_dict(fe.get_sequence_params(1)) == params_dict(fe.params)
        fe.set_sequence_params(0, **kit)
        fe.reset_sequence()
        assert params_dict(fe.get_sequence_params(0)) == params_dict(plf.plf_params(**kit))
    with plf.Frontend(camera=CAM, limits=limits(1), max_sequences=2) as fe:
        fe.set_sequence_params(1, **kit)
        fe._check(fe.lib.plf_set_max_sequences(fe._ctx, 3), "plf_set_max_sequences")
        assert all(params_dict(fe.get_sequence_params(s)) == params_dict(fe.params) for s in range(3))
    # launches: a batch of sequence 0 only, on a context that never set any settings and on one whose sequence 1 has
    # settings, and a batch of sequence 1 only
    counts = []
    for setit, s in ((False, 0), (True, 0), (True, 1)):
        with plf.Frontend(camera=CAM, limits=limits(4), max_sequences=2, **ctx) as fe:
            if setit:
                fe.set_sequence_params(1, **kit)
            L, R, seq = batch_args(seqs, [(s, i) for i in range(4)])
            fe.batch_upload(L, R)
            n0 = fe.lib.plf_launch_count(fe._ctx)
            fe.batch_run(4, seq=seq)
            fe.batch_download_array(4)
            counts.append(fe.lib.plf_launch_count(fe._ctx) - n0)
    assert counts[0] == counts[1] == counts[2], counts
