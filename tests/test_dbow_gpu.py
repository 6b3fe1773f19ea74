"""GPU parity of the DBoW2 keyframe database (plf_bow_set_vocabulary / plf_bow_insert / plf_bow_erase / plf_bow_get)
against oracle/dbow.c and against DBoW2's stored outputs (tests/golden/dbow_v1.npz): every row and every stored vector
bit-equal."""
from pathlib import Path

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import dbow, synth

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "dbow_v1.npz"
N_STREAM = 64


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def same(a, b):
    """Bit-equal, NaN included (every NaN the device writes is the same quiet NaN; compare positions)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
        np.array_equal(bits(a[~np.isnan(a)]), bits(b[~np.isnan(b)]))


@pytest.fixture(scope="module")
def vocabs(built, tmp_path_factory):
    """Two real-shape (k 9, L 6, ~560 k nodes) synthetic vocabularies, written as YAML and read back through
    plf_vocab_read_yml, with their oracle."""
    out = []
    for seed in (5, 6):
        v = dbow.synth_vocab(seed)
        path = tmp_path_factory.mktemp("voc") / f"voc{seed}.yml"
        dbow.write_yml(v, path)
        r = plf.read_vocab_yml(path)
        assert np.array_equal(r["node_id"], v["node_id"]) and len(r["node_id"]) > 500_000
        out.append((r, dbow.Vocab(r)))
    return out


@pytest.fixture(scope="module")
def stream_descs(built):
    """Stereo descriptors (pdesc_l / ldesc_l rows) of N_STREAM frames of the synthetic KITTI-shape stream."""
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, N_STREAM))
    lim = plf.default_limits(); lim.max_batch = 16
    out = []
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=1500, lsd_nfeatures=200) as fe:
        for b in range(0, N_STREAM, 16):
            fe.process_batch(np.stack([f[0] for f in frames[b:b + 16]]), np.stack([f[1] for f in frames[b:b + 16]]))
            for k in range(16):
                f = fe.get_frame(k)
                out.append((f["pdesc"], f["ldesc"]))
    assert all(len(p) > 100 and len(l) > 20 for p, l in out)
    return out


class Mirror:
    """The database as the oracle sees it: per kind the BowVector of every inserted index, None when erased."""

    def __init__(self, orcs):
        self.orcs = orcs
        self.vec = [{}, {}]

    def insert(self, k, descs):
        rows = []
        for c in range(2):
            if descs[c] is None:
                rows.append(None)
                continue
            self.vec[c][k] = self.orcs[c].transform(descs[c])
            rows.append(self.row(c, k))
        return rows

    def row(self, c, k):
        r = np.full(k + 1, np.nan)
        for i, v in self.vec[c].items():
            if i <= k and v is not None:
                r[i] = dbow.score(self.vec[c][k], v)
        return r

    def erase(self, k):
        for c in range(2):
            if k in self.vec[c]:
                self.vec[c][k] = None


def check_insert(fe, mir, k, pd, ld, check_rows=True):
    sp, sl = fe.bow_insert(k, pd, ld)
    want = mir.insert(k, (pd, ld))
    if check_rows:
        assert same(sp, want[0]), (k, np.nonzero(~(bits(sp) == bits(want[0])))[0][:5])
        assert same(sl, want[1]), k
    for c, d in enumerate((pd, ld)):
        w, x = fe.bow_vector(k, c)
        ow, ox = mir.vec[c][k]
        assert np.array_equal(w, ow) and np.array_equal(bits(x), bits(ox)), (k, c)
    return sp, sl


def test_stream_and_random_keyframes(vocabs, stream_descs):
    """~200 keyframes (stream frames, random descriptor sets, an empty one), with gaps and erasures: every row and every
    stored vector equals oracle/dbow.c bit for bit."""
    rng = np.random.default_rng(7)
    mir = Mirror([o for _, o in vocabs])
    with plf.Frontend() as fe:
        for c, (v, _) in enumerate(vocabs):
            fe.bow_set_vocabulary(c, v)
        k = 0
        for t in range(200):
            if t < N_STREAM:
                pd, ld = stream_descs[t]
            elif t == 100:
                pd, ld = np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8)
            else:
                pd = rng.integers(0, 256, (int(rng.integers(0, 900)), 32), dtype=np.uint8)
                ld = rng.integers(0, 256, (int(rng.integers(0, 300)), 32), dtype=np.uint8)
                if t % 3 == 0 and t > N_STREAM:          # revisit: a stream frame's features again, part of them
                    pd, ld = stream_descs[t % N_STREAM][0][::2], stream_descs[t % N_STREAM][1]
            check_insert(fe, mir, k, pd, ld)
            if t % 17 == 5:                              # erase an earlier keyframe (removeRedundantKFs)
                e = int(rng.integers(0, k + 1))
                fe.bow_erase(e)
                mir.erase(e)
            k += 1 + (t % 11 == 0) * 2                   # gaps: absent indices


def test_golden_dbow2_outputs(built):
    """The golden vocabularies reproduce DBoW2's stored BowVectors and scores (kind 0 / 1 = golden vocabulary 0 / 1)."""
    g = np.load(GOLDEN)
    sets = [g[f"set{s}"] for s in range(int(g["n_sets"]))]
    with plf.Frontend() as fe:
        for c in range(2):
            v = {key: g[f"v{c}_{key}"] for key in ("node_id", "parent_id", "weight", "desc", "word_id", "word_node")}
            v.update(k=int(g[f"v{c}_kL"][0]), L=int(g[f"v{c}_kL"][1]), scoring=0, weighting=0)
            fe.bow_set_vocabulary(c, v)
        for s, d in enumerate(sets):
            sp, sl = fe.bow_insert(s, d, d)
            for c, row in enumerate((sp, sl)):
                assert np.array_equal(bits(row), bits(g[f"v{c}_scores"][s, :s + 1])), (c, s)
                w, x = fe.bow_vector(s, c)
                assert np.array_equal(w, g[f"v{c}_s{s}_words"]) and np.array_equal(bits(x), bits(g[f"v{c}_s{s}_vals"]))
    # the disjoint pair of each vocabulary: -0.0
    for c in range(2):
        p = plf.default_params(); p.has_points, p.has_lines = (1, 0) if c == 0 else (0, 1)
        with plf.Frontend(params=p) as fe:
            v = {key: g[f"v{c}_{key}"] for key in ("node_id", "parent_id", "weight", "desc", "word_id", "word_node")}
            v.update(k=int(g[f"v{c}_kL"][0]), L=int(g[f"v{c}_kL"][1]))
            fe.bow_set_vocabulary(c, v)
            a, b = g[f"v{c}_disjoint_a"], g[f"v{c}_disjoint_b"]
            fe.bow_insert(0, a if c == 0 else None, a if c else None)
            rows = fe.bow_insert(1, b if c == 0 else None, b if c else None)
            assert bits(rows[c])[0] == np.uint64(1 << 63) and bits(rows[c])[0] == bits(g[f"v{c}_scores"][-1:, -2])[0]
            assert rows[1 - c] is None


def small_vocab():
    return dbow.synth_vocab(3, k=6, L=4, fewer_p=0.2, leaf_p=0.1, dup_p=0.1, zero_p=0.05)


def test_erase_and_empty(built):
    v = small_vocab()
    o = dbow.Vocab(v)
    mir = Mirror([o, o])
    rng = np.random.default_rng(1)
    with plf.Frontend() as fe:
        fe.bow_set_vocabulary(0, v)
        fe.bow_set_vocabulary(1, v)
        for k in range(6):
            check_insert(fe, mir, k, rng.integers(0, 256, (40, 32), dtype=np.uint8), rng.integers(0, 256, (9, 32), dtype=np.uint8))
        fe.bow_erase(2)
        fe.bow_erase(2)                                  # erasing an absent index is a no-op
        mir.erase(2)
        sp, sl = check_insert(fe, mir, 6, rng.integers(0, 256, (40, 32), dtype=np.uint8), np.zeros((0, 32), np.uint8))
        assert np.isnan(sp[2]) and np.isnan(sl[2])
        # an empty keyframe: every live entry and its self-score are -0.0
        sp, sl = check_insert(fe, mir, 7, np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8))
        live = ~np.isnan(sp)
        assert live.sum() == 7 and np.all(bits(sp[live]) == np.uint64(1 << 63))
        assert np.all(bits(sl[~np.isnan(sl)]) == np.uint64(1 << 63))
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_vector(2, 0)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_erase(-1)


def test_invalid_calls_leave_the_database_usable(built):
    v = small_vocab()
    o = dbow.Vocab(v)
    mir = Mirror([o, o])
    rng = np.random.default_rng(2)
    d = lambda n: rng.integers(0, 256, (n, 32), dtype=np.uint8)
    with plf.Frontend() as fe:
        with pytest.raises(plf.PlfError, match=r"\(-5\)"):
            fe.bow_insert(0, d(10), d(10))               # no vocabulary: PLF_ERR_STATE
        fe.bow_set_vocabulary(0, v)
        with pytest.raises(plf.PlfError, match=r"\(-5\)"):
            fe.bow_insert(0, d(10), d(10))               # lines enabled, no line vocabulary
        fe.bow_set_vocabulary(1, v)
        check_insert(fe, mir, 3, d(50), d(20))
        for bad in (3, 2, -1):
            with pytest.raises(plf.PlfError, match=r"\(-1\)"):
                fe.bow_insert(bad, d(10), d(10))
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_insert(4, d(8193), d(10))
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_insert(4, d(10), d(8193))
        check_insert(fe, mir, 4, d(8192), d(8192))       # the limit itself
        check_insert(fe, mir, 5, d(30), d(5))
        # a bad vocabulary is rejected and leaves the kind as it was
        bad = dict(v, k=40)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_set_vocabulary(0, bad)
        check_insert(fe, mir, 6, d(30), d(5))
        # setting a vocabulary empties that kind's database only
        fe.bow_set_vocabulary(0, v)
        mir.vec[0] = {}
        check_insert(fe, mir, 7, d(30), d(5))


@pytest.mark.parametrize("kinds", [(1, 0), (0, 1), (1, 1)], ids=["P", "L", "PL"])
def test_kind_combinations(built, kinds):
    v = small_vocab()
    o = dbow.Vocab(v)
    p = plf.default_params(); p.has_points, p.has_lines = kinds
    rng = np.random.default_rng(3)
    d = lambda n: rng.integers(0, 256, (n, 32), dtype=np.uint8)
    with plf.Frontend(params=p) as fe:
        for c in range(2):
            if kinds[c]:
                fe.bow_set_vocabulary(c, v)          # a disabled kind needs no vocabulary
        vecs = [[], []]
        for k in range(5):
            pd, ld = d(60), d(25)
            rows = fe.bow_insert(k, pd, ld)
            for c, dd in enumerate((pd, ld)):
                if not kinds[c]:
                    assert rows[c] is None
                    with pytest.raises(plf.PlfError):
                        fe.bow_vector(k, c)
                    continue
                vecs[c].append(o.transform(dd))
                want = np.array([dbow.score(vecs[c][k], vecs[c][i]) for i in range(k + 1)])
                assert np.array_equal(bits(rows[c]), bits(want))


def test_growth_past_initial_capacity(built):
    """3000 keyframes of 400 features: the entry store (65536 entries) and the index table (1024) both reallocate;
    sampled rows stay exact."""
    v = small_vocab()
    o = dbow.Vocab(v)
    rng = np.random.default_rng(4)
    vecs = []
    p = plf.default_params(); p.has_lines = 0
    with plf.Frontend(params=p) as fe:
        fe.bow_set_vocabulary(0, v)
        for k in range(3000):
            pd = rng.integers(0, 256, (400, 32), dtype=np.uint8)
            sp, _ = fe.bow_insert(k, pd, None)
            vecs.append(o.transform(pd))
            if k % 499 == 0 or k == 2999:
                want = np.array([dbow.score(vecs[k], vecs[i]) for i in range(k + 1)])
                assert np.array_equal(bits(sp), bits(want)), k
        for k in (0, 1500, 2999):
            w, x = fe.bow_vector(k, 0)
            assert np.array_equal(w, vecs[k][0]) and np.array_equal(bits(x), bits(vecs[k][1]))


def test_insert_between_batches_leaves_the_pipeline_unchanged(built):
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = synth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    frames = list(synth.stream(cam, 6, world=world, seed=5, step=0.1))
    L = np.stack([f[0] for f in frames]); R = np.stack([f[1] for f in frames])
    v = small_vocab()
    lim = plf.default_limits(); lim.max_batch = 2

    def run(with_bow):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=500, lsd_nfeatures=100) as fe:
            if with_bow:
                fe.bow_set_vocabulary(0, v)
                fe.bow_set_vocabulary(1, v)
            out = []
            rng = np.random.default_rng(9)
            for b in range(0, 6, 2):
                fe.batch_upload(L[b:b + 2], R[b:b + 2])
                fe.batch_run(2)
                if with_bow:
                    fe.bow_insert(b, rng.integers(0, 256, (300, 32), dtype=np.uint8), rng.integers(0, 256, (50, 32), dtype=np.uint8))
                res = fe.batch_download_array(2)
                out += [np.ascontiguousarray(res[f]) for f in res.dtype.names]    # fields: the struct has tail padding
                out += [np.ascontiguousarray(a) for a in fe.get_frame(1).values() if isinstance(a, np.ndarray)]
            return out

    a, b = run(False), run(True)
    assert len(a) == len(b) and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))


def test_vo_demo_bow_selftest(built, tmp_path):
    """`vo_demo --bow-selftest`: the INTEGRATION.md §4 f5 functions, compiled against the shim, give the score rows,
    conf_matrix rows and stored vectors the Python binding gives on the same frames (keyframe 1 erased after keyframe 2)."""
    import struct
    import subprocess
    demo = Path(__file__).resolve().parent.parent / "pl-slam_b200" / "lib" / "vo_demo"
    cam = dict(plf.KITTI_CAMERA, width=640, height=360, cx=320.0, cy=180.0, fx=500.0, fy=500.0)
    world = synth.World(seed=4, length=50.0, n_quads=160, n_segs=80, half_width=8.0, half_height=3.5)
    frames = [(L, R) for L, R, _ in synth.stream(cam, 5, world=world, seed=11, step=0.15)]
    p = tmp_path / "frames.bin"
    with open(p, "wb") as f:
        f.write(struct.pack("<3i", len(frames), cam["width"], cam["height"]))
        f.write(struct.pack("<5d", cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["b"]))
        for L, R in frames:
            f.write(np.ascontiguousarray(L, np.uint8).tobytes() + np.ascontiguousarray(R, np.uint8).tobytes())
    voc = [tmp_path / "voc_p.yml", tmp_path / "voc_l.yml"]
    dbow.write_yml(small_vocab(), voc[0])
    dbow.write_yml(dbow.synth_vocab(13, k=7, L=4, fewer_p=0.2, leaf_p=0.1, dup_p=0.1, zero_p=0.05), voc[1])
    r = subprocess.run([str(demo), str(p), "700", "150", "--bow-selftest", str(voc[0]), str(voc[1])], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    got = {(ln[1], int(ln[2])): ln[3:] for ln in (x.split() for x in r.stdout.strip().splitlines()) if ln[0] == "bow"}
    dbl = lambda key, k: np.array([float(v) for v in got[(key, k)]])
    lim = plf.default_limits(); lim.max_batch = 1
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=700, lsd_nfeatures=150) as fe:
        fe.bow_set_vocabulary(0, voc[0])
        fe.bow_set_vocabulary(1, voc[1])
        for k, (L, R) in enumerate(frames):
            fe.process_batch(L, R)
            f = fe.get_frame(0)
            sp, sl = fe.bow_insert(k, f["pdesc"], f["ldesc"])
            assert same(dbl("score_p", k), sp) and same(dbl("score_l", k), sl), k
            conf = np.where(np.isnan(sp), 0, sp).astype(np.float32).astype(np.float64)
            assert np.array_equal(bits(dbl("conf", k)), bits(conf)), k
            for c in range(2):
                w, x = fe.bow_vector(k, c)
                assert len(w) > 0
                assert np.array_equal(w, np.array([int(v) for v in got[(f"words{c}", k)]], np.uint32))
                assert np.array_equal(bits(x), bits(dbl(f"vals{c}", k)))
            if k == 2:
                fe.bow_erase(1)
        assert np.isnan(sp[1]) and not np.isnan(sp[0])


@pytest.mark.parametrize("kinds", [(1, 0), (0, 1)], ids=["P", "L"])
def test_disabled_kind_row_left_as_it_is(built, kinds):
    """Through the C ABI: a row passed for a kind disabled by has_points / has_lines is not written."""
    import ctypes as C
    v = small_vocab()
    on = kinds.index(1)
    p = plf.default_params(); p.has_points, p.has_lines = kinds
    o = dbow.Vocab(v)
    rng = np.random.default_rng(5)
    keep, vecs = [], []
    with plf.Frontend(params=p) as fe:
        fe.bow_set_vocabulary(on, v)
        for k in range(3):
            d = dict(pdesc=rng.integers(0, 256, (40, 32), dtype=np.uint8), ldesc=rng.integers(0, 256, (30, 32), dtype=np.uint8))
            vecs.append(o.transform(d["pdesc" if on == 0 else "ldesc"]))
            view = plf._frame_view(d, keep)
            rows = [np.full(k + 1, 7.0), np.full(k + 1, 7.0)]
            st = fe.lib.plf_bow_insert(fe._ctx, k, C.byref(view), C.c_void_p(rows[0].ctypes.data),
                                       C.c_void_p(rows[1].ctypes.data))
            assert st == 0
            assert np.all(rows[1 - on] == 7.0)
            want = np.array([dbow.score(vecs[k], vecs[i]) for i in range(k + 1)])
            assert np.array_equal(bits(rows[on]), bits(want))
