"""CPU checks of the DBoW2 restatement (oracle/dbow.c) and of plf_vocab_read_yml: the oracle against DBoW2's stored outputs
(tests/golden/dbow_v1.npz) bit for bit; where a pl-slam checkout is readable, the reader on the reference's two vocabulary
files and the oracle against DBoW2 itself on descriptors of the synthetic stream; one malformed file per rejection rule."""
import re
import tarfile
from pathlib import Path

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import clib, dbow, synth
from oracle.refbin import reference_dir

GOLDEN = Path(__file__).resolve().parent / "golden" / "dbow_v1.npz"
KEYS = ("node_id", "parent_id", "weight", "desc", "word_id", "word_node")


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def golden_vocab(g, c):
    v = {key: g[f"v{c}_{key}"] for key in KEYS}
    v.update(k=int(g[f"v{c}_kL"][0]), L=int(g[f"v{c}_kL"][1]), scoring=0, weighting=0)
    return v


@pytest.mark.parametrize("c", [0, 1])
def test_oracle_equals_dbow2_golden(built, c):
    g = np.load(GOLDEN)
    o = dbow.Vocab(golden_vocab(g, c))
    sets = [g[f"set{s}"] for s in range(int(g["n_sets"]))] + [g[f"v{c}_disjoint_a"], g[f"v{c}_disjoint_b"]]
    vecs = [o.transform(d) for d in sets]
    for s, (w, x) in enumerate(vecs):
        assert np.array_equal(w, g[f"v{c}_s{s}_words"]) and np.array_equal(bits(x), bits(g[f"v{c}_s{s}_vals"])), s
    got = np.array([[dbow.score(p, q) for q in vecs] for p in vecs])
    assert np.array_equal(bits(got), bits(g[f"v{c}_scores"]))
    assert bits(got[-2, -1]) == np.uint64(1 << 63)                      # no common word: -0.0
    assert len(vecs[0][0]) == 0 and np.all(bits(got[0]) == np.uint64(1 << 63))   # empty set


def test_golden_vocabularies_are_irregular():
    """The fixture exercises what the device path must get right: ties, stopped words, shallow leaves, file order."""
    g = np.load(GOLDEN)
    for c in range(2):
        v = golden_vocab(g, c)
        leaf = np.isin(v["node_id"], v["word_node"])
        assert np.any(v["weight"][leaf] == 0)
        assert not np.array_equal(v["node_id"], np.sort(v["node_id"]))
        _, cnt = np.unique(np.c_[v["parent_id"], v["desc"]], axis=0, return_counts=True)
        assert cnt.max() > 1                                             # duplicate sibling descriptors
        depth = {0: 0}
        par = dict(zip(v["node_id"].tolist(), v["parent_id"].tolist()))

        def dep(n):
            if n not in depth:
                depth[n] = dep(par[n]) + 1
            return depth[n]
        leaf_depths = {dep(n) for n in v["word_node"].tolist()}
        assert min(leaf_depths) < v["L"]                                 # leaves above the last level


def test_read_yml_roundtrip(built, tmp_path):
    v = dbow.synth_vocab(8, k=5, L=4, fewer_p=0.3, leaf_p=0.2, dup_p=0.1, zero_p=0.1)
    dbow.write_yml(v, tmp_path / "v.yml")
    r = plf.read_vocab_yml(tmp_path / "v.yml")
    assert (r["k"], r["L"], r["scoring"], r["weighting"]) == (5, 4, 0, 0)
    for key in KEYS:
        assert np.array_equal(bits(r[key]) if key == "weight" else r[key], bits(v[key]) if key == "weight" else v[key]), key


# ---- one malformed file per rejection rule -------------------------------------------------------------------------
def _base():
    return dbow.synth_vocab(9, k=4, L=3, fewer_p=0.5, leaf_p=0.2, dup_p=0.1, zero_p=0.1)


def _children(v):
    out = {}
    for n, p in zip(v["node_id"].tolist(), v["parent_id"].tolist()):
        out.setdefault(p, []).append(n)
    return out


def _mut_cycle(v):
    ch = _children(v)
    # an inner node with fewer than k children whose parent has another child: make it its own parent
    for i, n in enumerate(v["node_id"].tolist()):
        p = int(v["parent_id"][i])
        if n in ch and len(ch[n]) < v["k"] and len(ch[p]) > 1:
            v["parent_id"][i] = n
            return v
    raise AssertionError("no candidate")


def _mut_inner_word(v):
    ch = _children(v)
    inner = next(n for n in v["node_id"].tolist() if n in ch)
    v["word_node"][0] = inner
    return v


def _mut_leaf_without_word(v):
    keep = v["word_id"] != v["word_id"].max()
    v["word_id"], v["word_node"] = v["word_id"][keep], v["word_node"][keep]
    return v


def _drop_last_int(s):
    i = s.index('descriptor:"')
    j = s.index('"', i + len('descriptor:"'))
    ints = s[i + len('descriptor:"'):j].split()
    return s[:i] + 'descriptor:"' + " ".join(ints[:-1]) + ' ' + s[j:]


# rule: (mutation of the arrays, mutation of the text, part of the reason the reader gives)
MALFORMED = {
    "scoring": (lambda v: dict(v, scoring=1), None, "scoring 1 / weighting 0"),
    "weighting": (lambda v: dict(v, weighting=2), None, "scoring 0 / weighting 2"),
    "k_over_32": (lambda v: dict(v, k=33), None, r"k = 33 \(must be in 1\.\.32\)"),
    "duplicate_node_id": (lambda v: (v["node_id"].__setitem__(1, v["node_id"][0]), v)[1], None, "duplicate node id"),
    "node_id_out_of_range": (lambda v: (v["node_id"].__setitem__(0, len(v["node_id"]) + 1), v)[1], None,
                             r"node id \d+ out of range"),
    "missing_parent": (lambda v: (v["parent_id"].__setitem__(0, len(v["node_id"]) + 7), v)[1], None,
                       r"parent \d+ does not exist"),
    "cycle": (_mut_cycle, None, "does not reach the root"),
    "more_than_k_children": (lambda v: dict(v, k=max(len(c) for c in _children(v).values()) - 1), None,
                             "has more than k"),
    "leaf_without_word": (_mut_leaf_without_word, None, r"leaf \d+ has no word"),
    "word_on_inner_node": (_mut_inner_word, None, "lies on inner node"),
    "duplicate_word_id": (lambda v: (v["word_id"].__setitem__(1, v["word_id"][0]), v)[1], None, "duplicate word id"),
    "descriptor_31_ints": (None, _drop_last_int, "descriptor is not 32 integers"),
    "descriptor_256": (None, lambda s: re.sub(r'descriptor:"\d+', 'descriptor:"256', s, count=1),
                       "descriptor is not 32 integers"),
    "descriptor_not_integer": (None, lambda s: re.sub(r'descriptor:"\d+', 'descriptor:"1.5', s, count=1),
                               "descriptor is not 32 integers"),
}


@pytest.mark.parametrize("rule", list(MALFORMED))
def test_malformed_file_rejected(built, tmp_path, rule):
    mut_v, mut_text, reason = MALFORMED[rule]
    v = _base()
    if mut_v:
        v = mut_v(v)
    path = tmp_path / "bad.yml"
    dbow.write_yml(v, path)
    if mut_text:
        path.write_text(mut_text(path.read_text()))
    with pytest.raises(plf.PlfError, match=r"\(-1\).*" + reason):
        plf.read_vocab_yml(path)


def test_base_file_accepted(built, tmp_path):
    dbow.write_yml(_base(), tmp_path / "ok.yml")
    plf.read_vocab_yml(tmp_path / "ok.yml")


# ---- the reference's vocabularies ------------------------------------------------------------------------------------
def _parse_text(path):
    """An independent line parse of the file: (k, L, scoring, weighting), nodes and words in file order."""
    txt = Path(path).read_text()
    hdr = [int(re.search(rf"^\s*{k}:\s*(-?\d+)", txt, re.M).group(1)) for k in ("k", "L", "scoringType", "weightingType")]
    nodes = re.findall(r'nodeId:(\d+), parentId:(\d+), weight:([^,]+),\s*descriptor:"([^"]*)"', txt)
    words = re.findall(r"wordId:(\d+), nodeId:(\d+)", txt)
    return hdr, nodes, words


@pytest.fixture(scope="module")
def mapir(tmp_path_factory):
    ref = reference_dir()
    if ref is None or not (Path(ref) / "vocabulary" / "voc.tar.gz").exists():
        pytest.skip("no readable pl-slam checkout with vocabulary/voc.tar.gz")
    d = tmp_path_factory.mktemp("mapir")
    with tarfile.open(Path(ref) / "vocabulary" / "voc.tar.gz") as t:
        for name in ("mapir_orb.yml", "mapir_lsd.yml"):
            t.extract(name, d, filter="data")
    return d


@pytest.mark.parametrize("name,nodes,words", [("mapir_orb.yml", 589640, 523467), ("mapir_lsd.yml", 557311, 492291)])
def test_reader_on_reference_vocabularies(built, mapir, name, nodes, words):
    r = plf.read_vocab_yml(mapir / name)
    assert (r["k"], r["L"], r["scoring"], r["weighting"]) == (9, 6, 0, 0)
    assert len(r["node_id"]) == nodes and len(r["word_id"]) == words
    hdr, tn, tw = _parse_text(mapir / name)
    assert hdr == [9, 6, 0, 0] and len(tn) == nodes and len(tw) == words
    assert np.array_equal(r["node_id"], np.array([int(x[0]) for x in tn]))
    assert np.array_equal(r["parent_id"], np.array([int(x[1]) for x in tn]))
    assert np.array_equal(bits(r["weight"]), bits(np.array([float(x[2]) for x in tn])))
    assert np.array_equal(r["desc"][::997], np.array([[int(t) for t in tn[i][3].split()] for i in range(0, nodes, 997)]))
    assert np.array_equal(r["word_id"], np.array([int(x[0]) for x in tw]))
    assert np.array_equal(r["word_node"], np.array([int(x[1]) for x in tw]))


def _stream_descriptors():
    """ORB and LBD descriptors of two frames of the synthetic stream, by the CPU restatements."""
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = synth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    out = []
    for left, _, _ in synth.stream(cam, 2, world=world, seed=5, step=0.1):
        _, pd = clib.orb(left, nfeatures=800)
        kl = clib.keylines_from_segments(clib.lsd(left), left.shape[1], left.shape[0], 0.025 * min(left.shape))
        out.append((pd, clib.lbd_compute(left, kl)))
    return out


@pytest.mark.parametrize("name,kind", [("mapir_orb.yml", 0), ("mapir_lsd.yml", 1)])
def test_oracle_equals_dbow2_on_reference_vocabularies(built, mapir, name, kind):
    if not dbow.ref_available():
        pytest.skip("oracle/_ref/libdbow_ref.so not built")
    r = plf.read_vocab_yml(mapir / name)
    o, ref = dbow.Vocab(r), dbow.RefVocab(r)
    vecs = []
    for descs in _stream_descriptors():
        d = descs[kind]
        assert len(d) > 20
        a, b = o.transform(d), ref.transform(d)
        assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
        vecs.append(a)
    for p in vecs:
        for q in vecs:
            assert bits(dbow.score(p, q)) == bits(ref.score(p, q))
