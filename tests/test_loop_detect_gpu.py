"""GPU tests of loop-closure candidate detection (plf_bow_detect / plf_bow_detect_batch / plf_debug_loop_candidates): the
conf columns bit-equal to oracle/loopdetect.py over oracle/dbow.c's rows in P, L and PL contexts, the detection kernel
on every hand-built column, the fused call's candidates, equality with plf_bow_insert_batch and with one call per
problem, the refusals and the launch count."""
import ctypes as C
import math

import numpy as np
import pytest

import plslam_b200 as plf
from loopdetect_cases import cases
from oracle import dbow, synth
from oracle import loopdetect as old
from test_dbow_gpu import Mirror, bits, same  # noqa: F401

pytestmark = pytest.mark.gpu
OPTS = dict(lc_kf_dist=10, lc_kf_max_dist=5, lc_nkf_closest=2, min_lm_cov_graph=10, min_kf_local_map=1)


def vocabs():
    """Two small synth_vocab vocabularies: points and lines."""
    return (dbow.synth_vocab(3, k=6, L=4, fewer_p=0.2, leaf_p=0.1, dup_p=0.1, zero_p=0.05),
            dbow.synth_vocab(13, k=7, L=4, fewer_p=0.2, leaf_p=0.1, dup_p=0.1, zero_p=0.05))


VOCS = vocabs()
ORCS = None


def oracles():
    global ORCS
    if ORCS is None:
        ORCS = tuple(dbow.Vocab(v) for v in VOCS)
    return ORCS


def f32bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
        np.array_equal(f32bits(a[~np.isnan(a)]), f32bits(b[~np.isnan(b)]))


def same_result(a, b):
    return all(a[k] == b[k] or (isinstance(b[k], float) and math.isnan(a[k]) and math.isnan(b[k]))
               for k in plf.LC_RESULT_FIELDS)


class LcMirror:
    """One database as the oracle sees it, with the conf column and the detection of each insert."""

    def __init__(self, kinds):
        self.m, self.kinds = Mirror(list(oracles())), kinds

    def insert(self, pr, opts):
        k = pr["kf_idx"]
        rows = self.m.insert(k, tuple(pr.get(key) if self.kinds[c] else None for c, key in enumerate(("pdesc", "ldesc"))))
        live = np.ones(k + 1, bool)
        for c in range(2):
            if self.kinds[c]:
                live &= ~np.isnan(rows[c])
        std_pt = std_ls = 0.0
        if self.kinds[0] and self.kinds[1]:
            std_pt, std_ls = old.dispersions(pr["pt_pl"], pr["ls_spl"], pr["ls_epl"])
        conf = old.conf_row(self.kinds, live, rows[0], rows[1], len(pr["pdesc"]), len(pr["ldesc"]), std_pt, std_ls)
        res = old.look_for_loop_candidates(conf, live, pr.get("covis"), k, opts)
        return rows, conf, res

    def erase(self, k):
        self.m.erase(k)


def keyframe(rng, k, n_pt, n_ls, descs=None, covis=True):
    pd, ld = descs if descs is not None else (rng.integers(0, 256, (n_pt, 32), dtype=np.uint8),
                                              rng.integers(0, 256, (n_ls, 32), dtype=np.uint8))
    pr = dict(kf_idx=k, pdesc=pd, ldesc=ld, pt_pl=rng.uniform(0, 1242, (len(pd), 2)),
              ls_spl=rng.uniform(0, 1242, (len(ld), 2)), ls_epl=rng.uniform(0, 375, (len(ld), 2)))
    if covis and k:
        pr["covis"] = rng.integers(0, 20, k).astype(np.uint32)
    return pr


def vocab_ctx(kinds, max_sequences=1):
    p = plf.default_params(); p.has_points, p.has_lines = kinds
    fe = plf.Frontend(params=p, max_sequences=max_sequences)
    for c in range(2):
        if kinds[c]:
            fe.bow_set_vocabulary(c, VOCS[c])
    return fe


def test_debug_hook_matches_the_oracle_on_every_case(built):
    cs = cases()
    with plf.Frontend() as fe:
        for c in cs:   # one column per call: each with its own options
            got = fe.debug_loop_candidates([c["col"]], c["opts"])[0]
            assert same_result(got, c["want"]), (c["name"], got, c["want"])
        same_opts = [c for c in cs if c["opts"] == cs[0]["opts"]]
        got = fe.debug_loop_candidates([c["col"] for c in same_opts], same_opts[0]["opts"])
        for c, g in zip(same_opts, got):
            assert same_result(g, c["want"]), c["name"]
        n0 = fe.launches
        fe.debug_loop_candidates([c["col"] for c in same_opts] * 20, same_opts[0]["opts"])
        assert fe.launches - n0 == 1


def stream_keyframes():
    """The stereo features (descriptors and coordinates) of 8 frames of a small synthetic stream."""
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = [(L, R) for L, R, _ in synth.stream(cam, 8, world=world, seed=11, step=0.15)]
    lim = plf.default_limits(); lim.max_batch = 8
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        out = []
        for k in range(8):
            f = fe.get_frame(k)
            out.append(dict(pdesc=f["pdesc"], ldesc=f["ldesc"], pt_pl=f["pt_pl"], ls_spl=f["ls_spl"], ls_epl=f["ls_epl"]))
    assert all(len(f["pdesc"]) > 20 and len(f["ldesc"]) > 5 for f in out)
    return out


@pytest.mark.parametrize("kinds", [(1, 0), (0, 1), (1, 1)], ids=["P", "L", "PL"])
def test_conf_columns_bit_equal_to_the_oracle(built, kinds):
    """Stream keyframes, random ones, one without lines, one with a single point and one without any feature, with gaps
    and an erasure: every conf column, row and result equals the oracle's."""
    rng = np.random.default_rng(31)
    stream = stream_keyframes()
    mir = LcMirror(kinds)
    with vocab_ctx(kinds) as fe:
        k = 0
        for t in range(40):
            if t < 8:
                pr = dict(stream[t], kf_idx=k)
                if k:
                    pr["covis"] = rng.integers(0, 20, k).astype(np.uint32)
            elif t == 20:
                pr = keyframe(rng, k, 80, 0)                 # no lines
            elif t == 21:
                pr = keyframe(rng, k, 1, 30)                 # a single point: NaN dispersion
            elif t == 22:
                pr = keyframe(rng, k, 0, 0)                  # no feature
            else:
                pr = keyframe(rng, k, int(rng.integers(2, 200)), int(rng.integers(2, 60)))
            got = fe.bow_detect(pr, OPTS, rows=(True, True))
            rows, conf, res = mir.insert(pr, OPTS)
            for c in range(2):
                if kinds[c]:
                    assert same(got[("score_p", "score_l")[c]], rows[c]), (t, c)
            assert same_f32(got["conf"], conf), (t, np.nonzero(f32bits(got["conf"]) != f32bits(conf))[0][:5])
            assert same_result(got, res), (t, got, res)
            if kinds == (1, 1) and t in (21, 22):
                assert np.all(np.isnan(got["conf"])) and got["candidate"] == -1
            if t == 15:
                fe.bow_erase(3)
                mir.erase(3)
            k += 1 + (t % 9 == 4)


def place_sequence(rng, n, revisit_from, back):
    """Keyframe k sees places k, k+1, k+2 (60 point and 20 line descriptors each); from revisit_from on it sees again the
    places of keyframe k - back, so its row peaks there."""
    P = [(rng.integers(0, 256, (60, 32), dtype=np.uint8), rng.integers(0, 256, (20, 32), dtype=np.uint8))
         for _ in range(n + 3)]
    out = []
    for k in range(n):
        j = k - back if k >= revisit_from else k
        pd = np.concatenate([P[j + d][0] for d in range(3)])
        ld = np.concatenate([P[j + d][1] for d in range(3)])
        out.append(keyframe(rng, k, 0, 0, descs=(pd, ld)))
    return out


def test_fused_candidates_equal_the_oracle_over_three_sequences(built):
    """Three sequences revisit earlier places, in batches that hold several keyframes of one sequence: every result
    equals the oracle's, candidates appear, and each batch matches a twin context making one call per problem."""
    rng = np.random.default_rng(32)
    seqs = [place_sequence(rng, 90, 50 + 5 * s, 40 + 3 * s) for s in range(3)]
    mirs = [LcMirror((1, 1)) for _ in range(3)]
    n_cand = 0
    with vocab_ctx((1, 1), 3) as fe, vocab_ctx((1, 1), 3) as twin:
        for b in range(0, 90, 3):
            probs, seq = [], []
            for s in range(3):
                for k in range(b, b + 3):
                    probs.append(seqs[s][k]); seq.append(s)
            order = rng.permutation(3)
            probs = [p for s in order for p in probs[3 * s:3 * s + 3]]
            seq = [int(s) for s in order for _ in range(3)]
            got = fe.bow_detect_batch(probs, OPTS, seq=seq)
            for pr, s, g in zip(probs, seq, got):
                one = twin.bow_detect_batch([pr], OPTS, seq=[s])[0]
                _, conf, res = mirs[s].insert(pr, OPTS)
                assert same_f32(g["conf"], conf) and same_result(g, res), (s, pr["kf_idx"], g, res)
                assert same_f32(g["conf"], one["conf"]) and same_result(g, one)
                n_cand += g["candidate"] >= 0
            if b == 60:
                for s in range(3):
                    fe.bow_erase(20 + s, seq=s); twin.bow_erase(20 + s, seq=s); mirs[s].erase(20 + s)
    assert n_cand >= 10, n_cand


def test_equal_to_the_plain_batch_insert(built):
    """plf_bow_detect_batch leaves the database exactly as plf_bow_insert_batch does: rows, stored vectors and the rows
    of later inserts are bit-identical on a twin context."""
    rng = np.random.default_rng(33)
    with vocab_ctx((1, 1), 2) as fe, vocab_ctx((1, 1), 2) as twin:
        for b in range(6):
            probs = [keyframe(rng, 2 * b + j, int(rng.integers(2, 300)), int(rng.integers(2, 80))) for j in (0, 0, 1, 1)]
            seq = [0, 1, 0, 1]
            got = fe.bow_detect_batch(probs, OPTS, seq=seq, rows=(True, True))
            want = twin.bow_insert_batch(probs, seq=seq)
            for g, w in zip(got, want):
                assert np.array_equal(bits(g["score_p"]), bits(w[0])) and np.array_equal(bits(g["score_l"]), bits(w[1]))
        for s in range(2):
            for k in range(12):
                for c in range(2):
                    a, b2 = fe.bow_vector(k, c, seq=s), twin.bow_vector(k, c, seq=s)
                    assert np.array_equal(a[0], b2[0]) and np.array_equal(bits(a[1]), bits(b2[1]))
        # later plain inserts score identically against what each stored
        pr = keyframe(rng, 12, 100, 30)
        a, b2 = fe.bow_insert_batch([pr, pr], seq=[0, 1]), twin.bow_insert_batch([pr, pr], seq=[0, 1])
        for x, y in zip(a, b2):
            assert all(np.array_equal(bits(x[c]), bits(y[c])) for c in range(2))
        # rows not requested are not written, a column not requested is not returned
        g = fe.bow_detect_batch([keyframe(rng, 13, 50, 10)], OPTS, seq=[0], conf=False)[0]
        assert g["conf"] is None and g["score_p"] is None and g["score_l"] is None


def test_refusals_change_nothing(built):
    rng = np.random.default_rng(34)
    mir = LcMirror((1, 1))
    with vocab_ctx((1, 1), 2) as fe:
        for k in range(3):
            pr = keyframe(rng, k, 60, 20)
            got = fe.bow_detect_batch([pr], OPTS, seq=[0])[0]
            assert same_result(got, mir.insert(pr, OPTS)[2])
        keep = []
        good = keyframe(rng, 5, 30, 8)
        v = plf._frame_view(good, keep)
        arr = (plf.plf_lc_detect_problem * 2)(plf.plf_lc_detect_problem(5, C.pointer(v), None, None, None, None),
                                              plf.plf_lc_detect_problem(6, C.pointer(v), None, None, None, None))
        seq = np.array([0, 0], np.int32)
        sp = seq.ctypes.data_as(C.POINTER(C.c_int32))
        o = plf._lc_opts(OPTS)

        def refused(code, msg, *args):
            assert fe.lib.plf_bow_detect_batch(fe._ctx, *args) == code
            assert msg in fe.lib.plf_last_error(fe._ctx).decode()
        refused(-1, "opts is NULL", None, 2, arr, sp)
        refused(-1, "n_problems = -1", C.byref(o), -1, arr, sp)
        refused(-1, "problems is NULL", C.byref(o), 2, None, sp)
        refused(-4, "65536", C.byref(o), 65536, arr, sp)
        arr[1].kf_idx = 2
        refused(-1, "problem 1: kf_idx 2 does not exceed 5", C.byref(o), 2, arr, sp)
        arr[1].kf_idx = 6
        bad = plf._frame_view({k: v for k, v in good.items() if k != "pt_pl"}, keep)
        arr[1].kf = C.pointer(bad)
        refused(-1, "problem 1: pt_pl is NULL with 30 points", C.byref(o), 2, arr, sp)
        bad2 = plf._frame_view({k: v for k, v in good.items() if k != "ls_epl"}, keep)
        arr[1].kf = C.pointer(bad2)
        refused(-1, "problem 1: ls_spl / ls_epl is NULL with 8 lines", C.byref(o), 2, arr, sp)
        assert fe.lib.plf_bow_detect(fe._ctx, None, None) == -1
        assert fe.lib.plf_debug_loop_candidates(fe._ctx, None, 1, None, None, None, None, None) == -1
        with pytest.raises(plf.PlfError, match="kf_idx -1"):
            fe.debug_loop_candidates([dict(kf_idx=-1, conf=np.zeros(0, np.float32), live=np.zeros(0, bool))])
        # nothing changed: index 3 is still free and the database answers as the oracle's
        for k in (3, 5):
            pr = keyframe(rng, k, 60, 20)
            got = fe.bow_detect_batch([pr], OPTS, seq=[0])[0]
            _, conf, res = mir.insert(pr, OPTS)
            assert same_f32(got["conf"], conf) and same_result(got, res), k


def test_launches_do_not_depend_on_the_batch_size(built):
    rng = np.random.default_rng(35)
    with vocab_ctx((1, 1), 256) as fe:
        counts = []
        for b, P in enumerate((1, 256, 1, 256)):
            n0 = fe.launches
            fe.bow_detect_batch([keyframe(rng, b, 40, 9) for _ in range(P)], OPTS, seq=list(range(P)))
            counts.append(fe.launches - n0)
        assert counts == [5, 5, 5, 5], counts
        n0 = fe.launches
        fe.bow_detect(keyframe(rng, 0, 40, 9), OPTS)
        assert fe.launches - n0 == 5


def test_vo_demo_lc_detect_selftest(built, tmp_path):
    """`vo_demo --lc-detect-selftest`: the INTEGRATION.md §4 f8 function, compiled against the shim, leaves the
    conf_matrix rows and returns the candidates the Python binding gives on the same frames (its full_graph and options
    as the selftest sets them; keyframe 1 erased after keyframe 2)."""
    import struct
    import subprocess
    from pathlib import Path
    demo = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "lib" / "vo_demo"
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = [(L, R) for L, R, _ in synth.stream(cam, 9, world=world, seed=11, step=0.15)]
    p = tmp_path / "frames.bin"
    with open(p, "wb") as f:
        f.write(struct.pack("<3i", len(frames), cam["width"], cam["height"]))
        f.write(struct.pack("<5d", cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["b"]))
        for L, R in frames:
            f.write(np.ascontiguousarray(L, np.uint8).tobytes() + np.ascontiguousarray(R, np.uint8).tobytes())
    voc = [tmp_path / "voc_p.yml", tmp_path / "voc_l.yml"]
    for c in range(2):
        dbow.write_yml(VOCS[c], voc[c])
    r = subprocess.run([str(demo), str(p), "700", "150", "--lc-detect-selftest", str(voc[0]), str(voc[1])],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().splitlines() if ln.startswith("lc ")]
    conf_rows = {int(ln[2]): np.array([float(x) for x in ln[3:]], np.float32) for ln in lines if ln[1] == "conf"}
    cands = {int(ln[2]): int(ln[3]) for ln in lines if ln[1] == "cand"}
    assert sorted(conf_rows) == sorted(cands) == list(range(len(frames)))
    opts = dict(lc_kf_dist=1, lc_kf_max_dist=2, lc_nkf_closest=1, min_lm_cov_graph=20, min_kf_local_map=0)
    lim = plf.default_limits(); lim.max_batch = 1
    n_sorted = 0
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        for c in range(2):
            fe.bow_set_vocabulary(c, voc[c])
        for k, (L, R) in enumerate(frames):
            fe.process_batch(L, R)
            f = fe.get_frame(0)
            pr = {key: f[key] for key in ("pdesc", "ldesc", "pt_pl", "ls_spl", "ls_epl")}
            pr.update(kf_idx=k, covis=np.array([(i * k + i + k) % 40 for i in range(k)], np.uint32))
            got = fe.bow_detect(pr, opts, rows=(True, True))
            live = ~np.isnan(got["score_p"]) & ~np.isnan(got["score_l"])
            want = np.where(live, got["conf"], np.float32(0))      # conf_matrix: never written where absent
            assert same_f32(conf_rows[k], want), k
            assert cands[k] == got["candidate"], (k, cands[k], got)
            n_sorted += got["best"] >= 0
            if k == 2:
                fe.bow_erase(1)
    assert n_sorted >= 3
