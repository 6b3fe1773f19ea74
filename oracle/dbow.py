"""ctypes wrapper of oracle/dbow.c (DBoW2 transform / L1 score restated).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
from pathlib import Path

import numpy as np

from .clib import lib, _p


class Vocab:
    """A TemplatedVocabulary<FORB> built from the arrays of a vocabulary file in file order (keys of plf_vocab:
    node_id, parent_id, weight, desc, word_id, word_node)."""

    def __init__(self, v):
        self._arr = dict(node_id=np.ascontiguousarray(v["node_id"], np.int32),
                         parent_id=np.ascontiguousarray(v["parent_id"], np.int32),
                         weight=np.ascontiguousarray(v["weight"], np.float64),
                         desc=np.ascontiguousarray(v["desc"], np.uint8).reshape(-1, 32),
                         word_id=np.ascontiguousarray(v["word_id"], np.int32),
                         word_node=np.ascontiguousarray(v["word_node"], np.int32))
        a = self._arr
        f = lib().orc_dbow_new
        f.restype = C.c_void_p
        self._h = C.c_void_p(f(len(a["node_id"]), _p(a["node_id"]), _p(a["parent_id"]), _p(a["weight"]), _p(a["desc"]),
                               len(a["word_id"]), _p(a["word_id"]), _p(a["word_node"])))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_dbow_free(self._h)
            self._h = None

    def transform_one(self, d):
        d = np.ascontiguousarray(d, np.uint8).reshape(32)
        w, x = C.c_int(0), C.c_double(0)
        lib().orc_dbow_transform_one(self._h, _p(d), C.byref(w), C.byref(x))
        return w.value, x.value

    def transform(self, desc):
        """BowVector of the descriptor rows: (words uint32 ascending, values float64)."""
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = len(desc)
        words, vals = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.float64)
        f = lib().orc_dbow_transform
        f.restype = C.c_int
        m = f(self._h, _p(desc), n, _p(words), _p(vals))
        return words[:m].copy(), vals[:m].copy()

    def score(self, a, b):
        return score(a, b)


def score(a, b):
    """L1Scoring::score(a, b); a, b: (words, values)."""
    w1, v1 = np.ascontiguousarray(a[0], np.uint32), np.ascontiguousarray(a[1], np.float64)
    w2, v2 = np.ascontiguousarray(b[0], np.uint32), np.ascontiguousarray(b[1], np.float64)
    f = lib().orc_dbow_score
    f.restype = C.c_double
    return f(_p(w1), _p(v1), len(w1), _p(w2), _p(v2), len(w2))


_REF_SO = Path(__file__).resolve().parent / "_ref" / "libdbow_ref.so"
_ref = None


def ref_available():
    """True when oracle/_ref/libdbow_ref.so (DBoW2 compiled from a pl-slam checkout, oracle/ref_build/dbow.mk) exists."""
    return _REF_SO.exists()


class RefVocab(Vocab):
    """The same vocabulary in DBoW2 itself (TemplatedVocabulary<FORB>::transform and ::score)."""

    def __init__(self, v):
        global _ref
        if _ref is None:
            _ref = C.CDLL(str(_REF_SO))
            _ref.ref_dbow_new.restype = C.c_void_p
            _ref.ref_dbow_transform.restype = C.c_int
            _ref.ref_dbow_score.restype = C.c_double
        Vocab.__init__(self, v)
        a = self._arr
        self._r = C.c_void_p(_ref.ref_dbow_new(int(v["k"]), int(v.get("L", 0)), len(a["node_id"]), _p(a["node_id"]),
                                               _p(a["parent_id"]), _p(a["weight"]), _p(a["desc"]), len(a["word_id"]),
                                               _p(a["word_id"]), _p(a["word_node"])))

    def __del__(self):
        if getattr(self, "_r", None):
            _ref.ref_dbow_free(self._r)
            self._r = None
        Vocab.__del__(self)

    def transform(self, desc):
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = len(desc)
        words, vals = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.float64)
        m = _ref.ref_dbow_transform(self._r, _p(desc), n, _p(words), _p(vals))
        return words[:m].copy(), vals[:m].copy()

    def score(self, a, b):
        w1, v1 = np.ascontiguousarray(a[0], np.uint32), np.ascontiguousarray(a[1], np.float64)
        w2, v2 = np.ascontiguousarray(b[0], np.uint32), np.ascontiguousarray(b[1], np.float64)
        return _ref.ref_dbow_score(self._r, _p(w1), _p(v1), len(w1), _p(w2), _p(v2), len(w2))


def score_row(vecs, live, k):
    """The row plf_bow_insert returns for keyframe k: vecs[i] for i <= k (live[i] False / None -> NaN)."""
    row = np.full(k + 1, np.nan)
    for i in range(k + 1):
        if live[i] and vecs[i] is not None:
            row[i] = score(vecs[k], vecs[i])
    return row


def synth_vocab(seed, k=9, L=6, fewer_p=0.02, leaf_p=0.01, dup_p=0.02, zero_p=0.03):
    """A TemplatedVocabulary-shaped tree for tests: every inner node has k children, or 2..k-1 with probability fewer_p;
    below depth 1 a node is a leaf early with probability leaf_p (shallow leaves); a child repeats its previous sibling's
    descriptor with probability dup_p (ties in the descent); a leaf weighs 0 with probability zero_p (stopped words).
    Children descriptors are their parent's with each bit flipped with probability 1/4.  The file lists the nodes in a
    random order under a random permutation of the ids, and the words in word id order over a random leaf order."""
    rng = np.random.default_rng(seed)
    parent, descs, leaf = [np.array([-1])], [rng.integers(0, 256, (1, 32), dtype=np.uint8)], [np.array([False])]
    cur = np.array([0])
    nxt = 1
    for d in range(1, L + 1):
        nc = np.where(rng.random(len(cur)) < fewer_p, rng.integers(2, max(k, 3), len(cur)), k)
        par = np.repeat(cur, nc)
        pd = np.concatenate(descs)[par]
        flip = rng.integers(0, 256, pd.shape, dtype=np.uint8) & rng.integers(0, 256, pd.shape, dtype=np.uint8)
        dd = pd ^ flip
        first = np.ones(len(par), bool)
        first[1:] = par[1:] != par[:-1]
        dup = (~first) & (rng.random(len(par)) < dup_p)
        for i in np.nonzero(dup)[0]:
            dd[i] = dd[i - 1]
        lf = np.ones(len(par), bool) if d == L else ((rng.random(len(par)) < leaf_p) & (d > 1))
        ids = np.arange(nxt, nxt + len(par))
        nxt += len(par)
        parent.append(par); descs.append(dd); leaf.append(lf)
        cur = ids[~lf]
    parent, desc, leaf = np.concatenate(parent), np.concatenate(descs), np.concatenate(leaf)
    n = len(parent) - 1
    perm = np.concatenate([[0], rng.permutation(n) + 1])      # internal index -> node id
    order = rng.permutation(n) + 1                             # file order of internal indices
    leaves = np.nonzero(leaf)[0]
    weight = np.zeros(n + 1)
    weight[leaves] = rng.uniform(0.5, 10.0, len(leaves))
    weight[leaves[rng.random(len(leaves)) < zero_p]] = 0.0
    wl = rng.permutation(leaves)                               # word id -> internal index
    return dict(k=k, L=L, scoring=0, weighting=0, node_id=perm[order].astype(np.int32),
                parent_id=perm[parent[order]].astype(np.int32), weight=weight[order], desc=desc[order],
                word_id=np.arange(len(wl), dtype=np.int32), word_node=perm[wl].astype(np.int32))


def write_yml(voc, path, header=None, node_lines=None):
    """The vocabulary in the YAML form TemplatedVocabulary::save writes through cv::FileStorage (weights as %.16e, 0 as
    "0.").  header / node_lines: optional overrides of the header lines / node entries, for malformed-file tests."""
    def wfmt(x):
        return "0." if x == 0 else "%.16e" % x
    hdr = header if header is not None else [f"k: {voc['k']}", f"L: {voc['L']}", f"scoringType: {voc['scoring']}",
                                             f"weightingType: {voc['weighting']}"]
    out = ["%YAML:1.0", "---", "vocabulary:"] + ["   " + h for h in hdr] + ["   nodes:"]
    if node_lines is None:
        node_lines = ["      - { nodeId:%d, parentId:%d, weight:%s,\n          descriptor:\"%s \" }"
                      % (i, p, wfmt(w), " ".join(map(str, d)))
                      for i, p, w, d in zip(voc["node_id"].tolist(), voc["parent_id"].tolist(), voc["weight"].tolist(),
                                            np.asarray(voc["desc"]).tolist())]
    out += node_lines
    out.append("   words:")
    out += ["      - { wordId:%d, nodeId:%d }" % (w, nd) for w, nd in zip(voc["word_id"].tolist(), voc["word_node"].tolist())]
    Path(path).write_text("\n".join(out) + "\n")
