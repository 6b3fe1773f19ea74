"""CPU checks behind tests/test_pgo_batch_gpu.py (plf_pose_graph_batch): on oracle/pgo.py, the GPU file's batches hold
problems that finish in different rounds (a smaller one outlasting the largest), sizes on both sides of the 64-row
tiles up to n = 4098, every stop reason, a problem without free vertices and one without edges.  The builders here make
those batches and count the batch's launches from its outputs, as plslam_b200.h documents them."""
import functools
import math

import numpy as np
import pytest

from oracle import pgo
from plslam_b200 import synth

# (n_kf, window, loop edges) of tests/test_pgo_gpu.py's CASES: n_kf - 1 free vertices; 3 keyframes fill one tile, 684
# give n = 4098, two rows past a tile edge
MIXED = [(3, 1, 0), (12, 5, 1), (65, 5, 0), (101, 1, 4), (684, 5, 4), (12, 1, 4), (101, 5, 1)]
FIRST_ITERS = 3   # a max_iters that the large problems reach (tests/test_pgo_gpu.py's test_first_iterations_match_exactly)


@functools.lru_cache(maxsize=None)
def graph(n_kf, window, n_lc, seed=None):
    return synth.pose_graph_problem(n_kf, window, n_lc, drift=0.01, seed=n_kf + window + n_lc if seed is None else seed)


def identity_graph():
    """e = 0 exactly: one iteration, one trial, rho = 0 (tests/test_pgo_gpu.py's test_identity_graph_stops_on_rho_zero)"""
    n = 6
    frm = np.array([0, 1, 2, 3, 4, 0], np.int32)
    return {"T": np.tile(np.eye(4), (n, 1, 1)), "fixed": np.eye(1, n, dtype=np.uint8)[0], "from": frm,
            "to": np.array([1, 2, 3, 4, 5, 5], np.int32), "Z": np.tile(np.eye(4), (len(frm), 1, 1))}


def overflow_graph():
    """an edge of translation 1e160: every solve fails until lambda overflows at iteration 46 (stop `lambda`)"""
    Z = np.eye(4)[None].copy()
    Z[0, 0, 3] = -1e160
    return {"T": np.tile(np.eye(4), (2, 1, 1)), "fixed": np.array([1, 0], np.uint8), "from": np.array([1], np.int32),
            "to": np.array([0], np.int32), "Z": Z}


def isolated_graph():
    """tests/test_pgo_gpu.py's test_isolated_vertex_and_fixed_pair: a vertex without edges and an edge between two fixed
    vertices"""
    p = synth.pose_graph_problem(30, 3, 1, drift=0.02, seed=4)
    rng = np.random.default_rng(0)
    lone = synth._iso(synth._rodrigues(rng.standard_normal((2, 3))), rng.standard_normal((2, 3)))
    Zf = synth._iso(synth._rodrigues([[0.1, 0.0, 0.0]]), [[0.0, 0.5, 0.0]])[0]
    return {"T": np.concatenate([p["T"], lone]), "fixed": np.concatenate([p["fixed"], [0, 1]]).astype(np.uint8),
            "from": np.append(p["from"], 0).astype(np.int32), "to": np.append(p["to"], 31).astype(np.int32),
            "Z": np.concatenate([p["Z"], Zf[None]])}


def all_fixed_graph():
    """edges but no free vertex: chi2 only, no iteration"""
    p = graph(12, 5, 1)
    return dict(p, fixed=np.ones(len(p["T"]), np.uint8))


def edgeless_graph():
    """n_e = 0: chi2 = 0, no iteration, the poses returned as given"""
    p = graph(12, 5, 1)
    return {"T": p["T"], "fixed": p["fixed"], "from": np.zeros(0, np.int32), "to": np.zeros(0, np.int32),
            "Z": np.zeros((0, 4, 4))}


SPECIAL = {"identity": identity_graph, "overflow": overflow_graph, "isolated": isolated_graph,
           "all_fixed": all_fixed_graph, "edgeless": edgeless_graph}


def mixed_batch():
    """MIXED's graphs and the special ones, interleaved"""
    g = [graph(*c) for c in MIXED]
    s = [f() for f in SPECIAL.values()]
    return [g[0], s[0], g[1], g[2], s[1], g[3], s[2], g[4], s[3], g[5], s[4], g[6]]


def n_free(p):
    return int((pgo.free_index(np.asarray(p["fixed"]).astype(bool), np.asarray(p["from"]), np.asarray(p["to"])) >= 0).sum())


def documented_launches(probs, results):
    """plf_pose_graph_batch's launches (plslam_b200.h) from its outputs: round 0, then one round per trial of the longest
    problem; a round linearises when one of its problems starts an iteration (a new `iter` in its trace) and factors at
    the tile count of the largest problem still running"""
    nf = [n_free(p) for p in probs]
    count = 2 if any(len(np.ravel(p["from"])) for p in probs) else 1
    for r in range(max([res["trials"] for res in results], default=0)):
        run = [k for k, res in enumerate(results) if res["trials"] > r]
        lin = any(r == 0 or results[k]["trace"]["iter"][r] != results[k]["trace"]["iter"][r - 1] for k in run)
        nt = math.ceil(6 * max(nf[k] for k in run) / 64)
        count += 5 * nt + 4 + int(lin)
    return count


@functools.lru_cache(maxsize=None)
def oracle_runs(max_iters=100):
    return tuple(pgo.optimize(p, max_iters=max_iters) for p in mixed_batch())


def test_problems_finish_in_different_rounds():
    trials = [r["trials"] for r in oracle_runs()]
    assert len({t for t in trials if t}) >= 5
    big = max(range(len(trials)), key=lambda k: len(mixed_batch()[k]["T"]))
    assert any(t > trials[big] for t in trials)   # a smaller problem runs more trials than the largest


def test_sizes_straddle_the_tile_edges():
    tiles = {math.ceil(6 * n_free(p) / 64) for p in mixed_batch() if n_free(p)}
    assert 1 in tiles and len(tiles) >= 4
    assert 6 * 683 == 4098 and any(n_free(p) == 683 for p in mixed_batch())


def test_every_stop_reason_and_the_empty_systems():
    stops = {r["stop"] for r in oracle_runs() if r["trials"]}
    stops |= {r["stop"] for r in oracle_runs(FIRST_ITERS) if r["trials"]}
    assert stops == {"max_iters", "trials", "rho_zero", "lambda"}
    runs = dict(zip(range(len(mixed_batch())), oracle_runs()))
    kinds = {k: f() for k, f in SPECIAL.items()}
    assert (runs[1]["stop"], runs[1]["trials"]) == ("rho_zero", 1)                       # identity
    assert (runs[4]["stop"], runs[4]["trials"]) == ("lambda", 46)                        # overflow
    assert n_free(kinds["all_fixed"]) == 0 and len(kinds["edgeless"]["from"]) == 0
    assert runs[8]["trials"] == runs[10]["trials"] == 0


def test_documented_launches_of_a_made_up_run():
    """the counting rule on a hand-made pair: 2 + (5 + 4 + 1) + (5 + 4) for one 1-tile problem with 2 trials in 1
    iteration beside one that ran none"""
    p = graph(3, 1, 0)
    tr = np.zeros(2, [("iter", np.int32)])
    res = [dict(trials=2, trace=tr), dict(trials=0, trace=tr[:0])]
    assert documented_launches([p, edgeless_graph()], res) == 2 + 10 + 9
