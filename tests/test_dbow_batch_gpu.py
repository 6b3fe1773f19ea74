"""GPU tests of the per-sequence bag-of-words databases (plf_bow_insert_batch / plf_bow_erase_seq / plf_bow_get_seq /
plf_bow_clear_sequence): every row and stored vector bit-equal to oracle/dbow.c and to plf_bow_insert on a separate
context per database, isolation between sequences, the kind switches, growth, every refusal and the lifecycle rules."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import dbow, synth
from test_dbow_gpu import Mirror, bits, same, small_vocab, stream_descs, vocabs  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def rand_desc(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


class Checker:
    """A context with max_sequences databases, the oracle's view of each database (Mirror) and, optionally, one separate
    context per database that makes the same inserts one by one with plf_bow_insert."""

    def __init__(self, fe, vocs, n_seq, kinds=(1, 1), singles=False):
        self.fe, self.kinds = fe, kinds
        orcs = [dbow.Vocab(v) if v is not None else None for v in vocs]
        self.mir = {s: Mirror(orcs) for s in range(-1, n_seq)}
        self.single = {}
        for c in range(2):
            if kinds[c]:
                fe.bow_set_vocabulary(c, vocs[c])
        if singles:
            p = plf.default_params(); p.has_points, p.has_lines = kinds
            for s in range(-1, n_seq):
                self.single[s] = plf.Frontend(params=p)
                for c in range(2):
                    if kinds[c]:
                        self.single[s].bow_set_vocabulary(c, vocs[c])

    def close(self):
        for f in self.single.values():
            f.close()

    def batch(self, probs, seq, check_vectors=True):
        """probs: (kf_idx, pdesc, ldesc); seq: a list (None = all -1).  Checks every row and stored vector."""
        got = self.fe.bow_insert_batch([dict(kf_idx=k, pdesc=pd, ldesc=ld) for k, pd, ld in probs], seq=seq)
        ss = [-1] * len(probs) if seq is None else list(seq)
        for (k, pd, ld), s, rows in zip(probs, ss, got):
            want = self.mir[s].insert(k, tuple(d if self.kinds[c] else None for c, d in enumerate((pd, ld))))
            for c in range(2):
                if not self.kinds[c]:
                    assert rows[c] is None
                    continue
                assert same(rows[c], want[c]), (s, k, c, np.nonzero(bits(rows[c]) != bits(want[c]))[0][:5])
            if s in self.single:
                one = self.single[s].bow_insert(k, pd, ld)
                for c in range(2):
                    if self.kinds[c]:
                        assert np.array_equal(bits(one[c]), bits(rows[c])), (s, k, c)
            if check_vectors:
                self.vectors(s, [k])
        return got

    def vectors(self, s, ks):
        for k in ks:
            for c in range(2):
                if not self.kinds[c]:
                    continue
                v = self.mir[s].vec[c].get(k)
                if v is None:
                    with pytest.raises(plf.PlfError, match=r"\(-1\)"):
                        self.fe.bow_vector(k, c, seq=s)
                    continue
                w, x = self.fe.bow_vector(k, c, seq=s)
                assert np.array_equal(w, v[0]) and np.array_equal(bits(x), bits(v[1])), (s, k, c)

    def all_vectors(self):
        for s, m in self.mir.items():
            self.vectors(s, sorted(set(m.vec[0]) | set(m.vec[1])))

    def erase(self, s, k):
        self.fe.bow_erase(k, seq=s)
        self.mir[s].erase(k)
        if s in self.single:
            self.single[s].bow_erase(k)


def test_interleaved_schedule_of_eight_sequences(built):
    """60 batches over 8 sequences: each batch takes a random subset of sequences (others sit it out), 1 to 3 keyframes
    each with gaps between indices, interleaved in problem order; empty keyframes and erasures.  Rows and vectors equal
    the oracle's and those of a separate context per sequence."""
    rng = np.random.default_rng(11)
    v = small_vocab()
    with plf.Frontend(max_sequences=8) as fe:
        ck = Checker(fe, (v, v), 8, singles=True)
        try:
            nxt = [0] * 8
            for b in range(60):
                todo = []
                for s in rng.permutation(8)[:int(rng.integers(1, 9))]:
                    for _ in range(int(rng.integers(1, 4))):
                        k = nxt[s] + int(rng.integers(0, 3))            # gaps: absent indices
                        nxt[s] = k + 1
                        empty = rng.random() < 0.08
                        pd = rand_desc(rng, 0 if empty else int(rng.integers(0, 300)))
                        ld = rand_desc(rng, 0 if empty else int(rng.integers(0, 80)))
                        todo.append((int(s), k, pd, ld))
                # interleave the sequences, keeping each one's order
                slots = [t[0] for t in todo]
                rng.shuffle(slots)
                it = {s: iter([t for t in todo if t[0] == s]) for s in set(slots)}
                probs, seq = [], []
                for s in slots:
                    _, k, pd, ld = next(it[s])
                    probs.append((k, pd, ld)); seq.append(s)
                ck.batch(probs, seq, check_vectors=b % 5 == 0)
                if b % 7 == 3:
                    s = int(rng.integers(0, 8))
                    if nxt[s]:
                        ck.erase(s, int(rng.integers(0, nxt[s])))
            ck.all_vectors()
        finally:
            ck.close()


def test_several_problems_of_one_sequence_in_one_batch(built):
    rng = np.random.default_rng(12)
    v = small_vocab()
    with plf.Frontend(max_sequences=3) as fe:
        ck = Checker(fe, (v, v), 3, singles=True)
        try:
            ck.batch([(k, rand_desc(rng, 60), rand_desc(rng, 20)) for k in range(5)], [1] * 5)
            got = ck.batch([(5, rand_desc(rng, 60), rand_desc(rng, 20)), (0, rand_desc(rng, 40), rand_desc(rng, 9)),
                            (8, rand_desc(rng, 70), rand_desc(rng, 0)), (1, rand_desc(rng, 40), rand_desc(rng, 9)),
                            (9, rand_desc(rng, 60), rand_desc(rng, 20))], [1, 2, 1, 2, 1])
            # the later problem's row holds the earlier one of the same batch, the earlier one's row stops at its index
            assert not np.isnan(got[4][0][5]) and not np.isnan(got[4][0][8]) and np.isnan(got[4][0][6])
            assert len(got[0][0]) == 6
            ck.all_vectors()
        finally:
            ck.close()


def test_context_database_through_the_batch_and_the_single_call(built):
    """seq = NULL and -1 mixed with sequences insert into the context's database; plain plf_bow_insert continues it,
    and plf_bow_erase_seq / plf_bow_get_seq with -1 are plf_bow_erase / plf_bow_get."""
    rng = np.random.default_rng(13)
    v = small_vocab()
    with plf.Frontend(max_sequences=2) as fe:
        ck = Checker(fe, (v, v), 2, singles=True)
        try:
            ck.batch([(0, rand_desc(rng, 50), rand_desc(rng, 10)), (1, rand_desc(rng, 50), rand_desc(rng, 10))], None)
            ck.batch([(2, rand_desc(rng, 50), rand_desc(rng, 10)), (0, rand_desc(rng, 50), rand_desc(rng, 10)),
                      (3, rand_desc(rng, 50), rand_desc(rng, 10)), (0, rand_desc(rng, 50), rand_desc(rng, 10))], [-1, 0, -1, 1])
            for k in (4, 6):
                pd, ld = rand_desc(rng, 50), rand_desc(rng, 10)
                rows = fe.bow_insert(k, pd, ld)
                want = ck.mir[-1].insert(k, (pd, ld))
                one = ck.single[-1].bow_insert(k, pd, ld)
                for c in range(2):
                    assert same(rows[c], want[c]) and np.array_equal(bits(rows[c]), bits(one[c])), (k, c)
            fe.bow_erase(1, seq=-1); ck.mir[-1].erase(1); ck.single[-1].bow_erase(1)
            fe.bow_erase(2); ck.mir[-1].erase(2); ck.single[-1].bow_erase(2)
            ck.batch([(7, rand_desc(rng, 50), rand_desc(rng, 10))], [-1])
            for k in (0, 3, 4, 6, 7):
                for c in range(2):
                    a, b = fe.bow_vector(k, c), fe.bow_vector(k, c, seq=-1)
                    assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
            ck.all_vectors()
        finally:
            ck.close()


def test_isolation_between_sequences(built):
    """The same kf_idx in two sequences: two different vectors; an index only another sequence holds is NaN."""
    rng = np.random.default_rng(14)
    v = small_vocab()
    with plf.Frontend(max_sequences=2) as fe:
        ck = Checker(fe, (v, v), 2)
        shared = rand_desc(rng, 80), rand_desc(rng, 30)
        ck.batch([(0, *shared), (0, *shared), (3, rand_desc(rng, 80), rand_desc(rng, 30))], [0, 1, 1])
        got = ck.batch([(4, *shared), (5, rand_desc(rng, 80), rand_desc(rng, 30))], [0, 1])
        for c in range(2):
            assert np.all(np.isnan(got[0][c][1:4])) and not np.isnan(got[0][c][0])   # seq 1's index 3 is absent in 0
            assert np.all(np.isnan(got[1][c][[1, 2, 4]])) and not np.isnan(got[1][c][3])
        fe.bow_erase(0, seq=1); ck.mir[1].erase(0)
        got = ck.batch([(5, *shared), (6, *shared)], [0, 1])
        assert not np.isnan(got[0][0][0]) and np.isnan(got[1][0][0])      # the erasure stayed in sequence 1
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_vector(3, 0, seq=0)
        ck.all_vectors()


@pytest.mark.parametrize("kinds", [(1, 0), (0, 1), (1, 1)], ids=["P", "L", "PL"])
def test_kind_combinations(built, kinds):
    """A disabled kind needs no vocabulary, gets no row (a row passed through the C ABI is left as it is) and stores
    nothing."""
    rng = np.random.default_rng(15)
    v = small_vocab()
    p = plf.default_params(); p.has_points, p.has_lines = kinds
    with plf.Frontend(params=p, max_sequences=3) as fe:
        ck = Checker(fe, tuple(v if kinds[c] else None for c in range(2)), 3, kinds=kinds, singles=True)
        try:
            for b in range(4):
                ck.batch([(b, rand_desc(rng, 60), rand_desc(rng, 25)) for _ in range(3)] + [(b + 1, rand_desc(rng, 30), rand_desc(rng, 5))],
                         [0, 1, 2, -1])
            ck.all_vectors()
            # through the C ABI: rows of both kinds passed, the disabled kind's is not written
            keep = []
            views = [plf._frame_view(dict(pdesc=rand_desc(rng, 40), ldesc=rand_desc(rng, 30)), keep) for _ in range(2)]
            rows = [[np.full(9, 7.0), np.full(9, 7.0)] for _ in range(2)]
            arr = (plf.plf_bow_problem * 2)(*[plf.plf_bow_problem(8, C.pointer(views[i]), rows[i][0].ctypes.data,
                                                                  rows[i][1].ctypes.data) for i in range(2)])
            seq = np.array([0, 2], np.int32)
            assert fe.lib.plf_bow_insert_batch(fe._ctx, 2, arr, seq.ctypes.data_as(C.POINTER(C.c_int32))) == 0
            for i in range(2):
                for c in range(2):
                    assert np.all(rows[i][c] == 7.0) != bool(kinds[c]), (i, c)
        finally:
            ck.close()


def test_growth_of_several_databases_in_one_batch(built):
    """Several databases pass their first allocation (1024 entries, 64 indices) in one batch, from empty and from
    non-empty, with several problems each; the context's database grows alongside."""
    rng = np.random.default_rng(16)
    v = small_vocab()
    with plf.Frontend(max_sequences=4) as fe:
        ck = Checker(fe, (v, v), 4, singles=True)
        try:
            ck.batch([(0, rand_desc(rng, 100), rand_desc(rng, 20)) for _ in range(2)], [0, 1])
            probs, seq = [], []
            for s in (0, 1, 2, 3, -1):
                for j, k in enumerate((40, 90, 300)):
                    probs.append((k, rand_desc(rng, 1500), rand_desc(rng, 700))); seq.append(s)
            ck.batch(probs, seq)
            ck.batch([(301 + 200 * s if s >= 0 else 1000, rand_desc(rng, 3000), rand_desc(rng, 1200)) for s in (0, 1, 2, 3, -1)],
                     [0, 1, 2, 3, -1])
            ck.all_vectors()
        finally:
            ck.close()


def test_512_problems_on_512_sequences(built):
    rng = np.random.default_rng(17)
    v = small_vocab()
    with plf.Frontend(max_sequences=512) as fe:
        ck = Checker(fe, (v, v), 512)
        for b in range(2):
            ck.batch([(b + (s % 3), rand_desc(rng, int(rng.integers(0, 120))), rand_desc(rng, int(rng.integers(0, 30))))
                      for s in range(512)], list(range(512)), check_vectors=False)
        for s in (0, 1, 255, 511):
            ck.vectors(s, sorted(ck.mir[s].vec[0]))


def test_real_shape_vocabularies_and_stream_keyframes(vocabs, stream_descs):
    """The real-shape synthetic vocabularies and stream descriptors: four sequences walking the stream at different
    offsets and strides, against the oracle and a separate context per sequence."""
    with plf.Frontend(max_sequences=4) as fe:
        ck = Checker(fe, [r for r, _ in vocabs], 4, singles=True)
        try:
            n = len(stream_descs)
            for b in range(12):
                probs = [(b, *stream_descs[(7 * s + b * (s + 1)) % n]) for s in range(4)]
                ck.batch(probs, [0, 1, 2, 3], check_vectors=b % 4 == 0)
            ck.all_vectors()
        finally:
            ck.close()


def raw_batch(fe, probs, seq=None, n=None):
    """plf_bow_insert_batch through the C ABI: probs are (kf_idx, plf_frame_view or None); returns the status."""
    arr = (plf.plf_bow_problem * max(len(probs), 1))(
        *[plf.plf_bow_problem(k, C.pointer(v) if v is not None else None, None, None) for k, v in probs])
    s = None if seq is None else np.ascontiguousarray(seq, np.int32)
    return fe.lib.plf_bow_insert_batch(fe._ctx, len(probs) if n is None else n, arr,
                                       None if s is None else s.ctypes.data_as(C.POINTER(C.c_int32)))


def test_refusals_change_nothing(built):
    rng = np.random.default_rng(18)
    v = small_vocab()
    keep = []
    view = lambda npt, nls: plf._frame_view(dict(pdesc=rand_desc(rng, npt), ldesc=rand_desc(rng, nls)), keep)
    with plf.Frontend(max_sequences=4) as fe:
        with pytest.raises(plf.PlfError, match=r"\(-5\).*problem 0: no point vocabulary"):   # PLF_ERR_STATE
            fe.bow_insert_batch([dict(kf_idx=0), dict(kf_idx=0, pdesc=rand_desc(rng, 3))], seq=[0, 1])
        ck = Checker(fe, (v, v), 4)
        ck.batch([(k, rand_desc(rng, 50), rand_desc(rng, 10)) for k in (0, 1, 2, 3)], [0, 1, 1, -1])
        good = view(30, 8)

        def refused(code, probs, seq=None, n=None, msg=None):
            assert raw_batch(fe, probs, seq, n) == code
            if msg:
                err = fe.lib.plf_last_error(fe._ctx).decode()
                assert msg in err, err
        refused(-1, [(5, good)], n=-1, msg="n_problems = -1")
        refused(-1, [(5, good), (5, good)], [0, 4], msg="problem 1: seq[1] = 4 outside [-1, 4)")
        refused(-1, [(5, good)], [-2])
        refused(-1, [(5, good), (6, None)], [0, 0], msg="problem 1: kf is NULL")
        refused(-1, [(5, good), (-1, good)], [0, 2], msg="problem 1: kf_idx -1")
        refused(-1, [(1 << 24, good)], [2])
        refused(-1, [(5, good), (2, good)], [0, 1], msg="problem 1: kf_idx 2 does not exceed 2")
        refused(-1, [(5, good), (5, good)], [0, 0], msg="problem 1: kf_idx 5 does not exceed 5")
        refused(-1, [(7, good), (6, good)], [2, 2])
        refused(-1, [(5, good), (3, good)], [2, -1], msg="problem 1: kf_idx 3 does not exceed 3")
        refused(-1, [(5, good), (6, view(8193, 1))], [0, 2], msg="problem 1: 8193 point features")
        refused(-1, [(5, good), (6, view(1, 8193))], [0, 2], msg="8193 line features")
        neg = view(1, 1); neg.n_pt = -1
        refused(-1, [(6, neg)], [3])
        nul = view(0, 0); nul.n_ls = 5
        refused(-1, [(5, good), (6, nul)], [0, 3], msg="problem 1: line descriptors are NULL")
        empty = view(0, 0)
        refused(-4, [(k, empty) for k in range(65536)], [3] * 65536, msg="65536")
        assert raw_batch(fe, [], n=0) == 0
        # nothing changed: the refused problems' indices are still free, every row and vector as before
        ck.all_vectors()
        ck.batch([(5, rand_desc(rng, 50), rand_desc(rng, 10)), (5, rand_desc(rng, 50), rand_desc(rng, 10)),
                  (0, rand_desc(rng, 50), rand_desc(rng, 10)), (4, rand_desc(rng, 50), rand_desc(rng, 10))], [0, 2, 3, -1])
        ck.all_vectors()
        # the other calls' refusals
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_erase(0, seq=4)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_erase(-1, seq=0)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_vector(0, 0, seq=-2)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_clear_sequence(-1)
        with pytest.raises(plf.PlfError, match=r"\(-1\)"):
            fe.bow_clear_sequence(4)
        fe.bow_erase(3, seq=2)                 # absent in 2: a no-op
        fe.bow_clear_sequence(3)
        ck.mir[3] = Mirror(ck.mir[0].orcs)
        ck.all_vectors()


def test_lifecycle(built):
    rng = np.random.default_rng(19)
    v = small_vocab()
    d = lambda: (rand_desc(rng, 50), rand_desc(rng, 12))
    with plf.Frontend(max_sequences=3) as fe:
        ck = Checker(fe, (v, v), 3)
        ck.batch([(0, *d()), (0, *d()), (1, *d()), (0, *d())], [0, 1, 1, -1])
        # reset_sequence and set_sequence_camera leave the databases as they are
        fe.reset_sequence()
        fe.set_sequence_camera(1, dict(plf.KITTI_CAMERA, fx=700.0))
        ck.all_vectors()
        ck.batch([(2, *d()), (3, *d())], [1, 0])
        # clear_sequence empties both kinds of one sequence and lets it start at 0 again
        fe.bow_clear_sequence(1)
        for c in range(2):
            with pytest.raises(plf.PlfError, match=r"\(-1\)"):
                fe.bow_vector(0, c, seq=1)
        ck.mir[1] = Mirror(ck.mir[0].orcs)
        got = ck.batch([(0, *d()), (4, *d())], [1, 0])
        assert len(got[0][0]) == 1
        fe.bow_clear_sequence(2)               # never inserted into: a no-op
        # set_vocabulary(kind) empties that kind in every database, the other kind stays
        fe.bow_set_vocabulary(0, v)
        for s in (-1, 0, 1):
            ck.mir[s].vec[0] = {}
        ck.all_vectors()
        got = ck.batch([(5, *d()), (1, *d()), (1, *d())], [0, 1, -1])
        assert np.isnan(got[0][0][0]) and not np.isnan(got[0][1][0])
        # set_max_sequences drops every sequence's databases and keeps the context's
        assert fe.lib.plf_set_max_sequences(fe._ctx, 3) == 0
        for s in (0, 1):
            ck.mir[s] = Mirror(ck.mir[-1].orcs)
        ck.all_vectors()
        for s in (0, 1):
            with pytest.raises(plf.PlfError, match=r"\(-1\)"):
                fe.bow_vector(0, 1, seq=s)
        ck.batch([(0, *d()), (0, *d()), (2, *d())], [0, 1, -1])
        ck.all_vectors()


def test_launches_do_not_depend_on_the_batch_size(built):
    rng = np.random.default_rng(20)
    v = small_vocab()
    with plf.Frontend(max_sequences=256) as fe:
        fe.bow_set_vocabulary(0, v)
        fe.bow_set_vocabulary(1, v)
        counts = []
        for b, P in enumerate((1, 256, 1, 256)):
            n0 = fe.launches
            fe.bow_insert_batch([dict(kf_idx=b, pdesc=rand_desc(rng, 40), ldesc=rand_desc(rng, 9)) for _ in range(P)],
                                seq=list(range(P)))
            counts.append(fe.launches - n0)
        assert counts == [3, 3, 3, 3], counts
        n0 = fe.launches
        fe.bow_insert(0, rand_desc(rng, 40), rand_desc(rng, 9))
        assert fe.launches - n0 == 3


def test_batch_insert_between_batches_leaves_the_pipeline_unchanged(built):
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = synth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    frames = list(synth.stream(cam, 6, world=world, seed=5, step=0.1))
    L = np.stack([f[0] for f in frames]); R = np.stack([f[1] for f in frames])
    v = small_vocab()
    lim = plf.default_limits(); lim.max_batch = 2

    def run(with_bow):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=500, lsd_nfeatures=100, max_sequences=3) as fe:
            if with_bow:
                fe.bow_set_vocabulary(0, v)
                fe.bow_set_vocabulary(1, v)
            out = []
            rng = np.random.default_rng(9)
            for b in range(0, 6, 2):
                fe.batch_upload(L[b:b + 2], R[b:b + 2])
                fe.batch_run(2)
                if with_bow:
                    fe.bow_insert_batch([dict(kf_idx=b, pdesc=rand_desc(rng, 300), ldesc=rand_desc(rng, 50)) for _ in range(4)],
                                        seq=[0, 1, 2, -1])
                res = fe.batch_download_array(2)
                out += [np.ascontiguousarray(res[f]) for f in res.dtype.names]
                out += [np.ascontiguousarray(a) for a in fe.get_frame(1).values() if isinstance(a, np.ndarray)]
            return out

    a, b = run(False), run(True)
    assert len(a) == len(b) and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
