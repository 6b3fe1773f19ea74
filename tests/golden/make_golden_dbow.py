"""Generates tests/golden/dbow_v1.npz: DBoW2's own outputs (TemplatedVocabulary<FORB>::transform, BowVector, L1Scoring,
compiled unmodified from a pl-slam checkout into oracle/_ref/libdbow_ref.so by oracle/ref_build/dbow.mk) on two small
synthetic vocabularies with ties in the descent (duplicate sibling descriptors), stopped words (weight 0), shallow leaves
and a file order unlike the id order.  Stored per vocabulary: its arrays in file order, the BowVector of every descriptor
set (an empty set included), the score of every ordered pair of sets (self-scores included) and one pair of sets with no
common word.  Run: python tests/golden/make_golden_dbow.py (after __graft_entry__.build())."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import dbow  # noqa: E402

VOCABS = [dict(seed=11, k=5, L=4, fewer_p=0.3, leaf_p=0.15, dup_p=0.15, zero_p=0.1),
          dict(seed=12, k=3, L=5, fewer_p=0.2, leaf_p=0.1, dup_p=0.25, zero_p=0.15)]
SET_SIZES = [0, 1, 3, 17, 64, 200, 333]


def main(out=ROOT / "tests" / "golden" / "dbow_v1.npz"):
    if not dbow.ref_available():
        raise SystemExit("oracle/_ref/libdbow_ref.so is missing: run __graft_entry__.build() with a pl-slam checkout")
    rng = np.random.default_rng(2024)
    sets = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in SET_SIZES]
    sets[4][10:20] = sets[4][0]                      # repeated features: addWeight sums into one entry
    g = {"n_sets": len(sets)}
    for s, d in enumerate(sets):
        g[f"set{s}"] = d
    for vi, kw in enumerate(VOCABS):
        v = dbow.synth_vocab(**kw)
        ref = dbow.RefVocab(v)
        for key in ("node_id", "parent_id", "weight", "desc", "word_id", "word_node"):
            g[f"v{vi}_{key}"] = v[key]
        g[f"v{vi}_kL"] = np.array([v["k"], v["L"]], np.int32)
        # a pair of single-feature sets on two different words: no common word, score -0.0
        words = {}
        while len(words) < 2:
            d = rng.integers(0, 256, (1, 32), dtype=np.uint8)
            w, x = ref.transform_one(d)
            if x > 0:
                words.setdefault(w, d)
        a, b = list(words.values())
        all_sets = sets + [a, b]
        g[f"v{vi}_disjoint_a"], g[f"v{vi}_disjoint_b"] = a, b
        vecs = [ref.transform(d) for d in all_sets]
        for s, (w, x) in enumerate(vecs):
            g[f"v{vi}_s{s}_words"], g[f"v{vi}_s{s}_vals"] = w, x
        g[f"v{vi}_scores"] = np.array([[ref.score(p, q) for q in vecs] for p in vecs])
        assert np.float64(g[f"v{vi}_scores"][-2, -1]).view(np.uint64) == np.uint64(1 << 63)   # -0.0
    np.savez_compressed(out, **g)
    print("wrote", out, Path(out).stat().st_size, "bytes")


if __name__ == "__main__":
    main()
