"""CPU tests of tests/matchgrid_cases.py: the vectorised reference equals oracle/matchgrid.py on the reduced instance of
every generator, its closed-form Bresenham walk equals the oracle's, and each generator reaches the edge it is built for."""
import numpy as np
import pytest

import matchgrid_cases as mc
from oracle import matchgrid as mg

SMALL = {name: gen(small=True) for name, gen in mc.GENERATORS.items()}


def _by_name(name):
    return next(c for cs in SMALL.values() for c in cs if c.name == name)


@pytest.mark.parametrize("gen", list(mc.GENERATORS))
def test_reference_equals_the_oracle(gen):
    for c in SMALL[gen]:
        for p in range(c.P):
            r = mc.reference(c, p)
            n1, n2 = c.counts(p)
            s = c.slot(p)
            g = mc.oracle_grid(c, p)
            if c.lines:
                m, n = mg.match_grid_lines(c.q[p, :n1], c.d1[s, :n1], g, c.tdir[p, :n2], c.d2[p, :n2], c.w, c.nnr, c.th,
                                           c.best_lr)
            else:
                m, n = mg.match_grid_points(c.q[p, :n1], c.d1[s, :n1], g, c.d2[p, :n2], c.w, c.nnr, c.best_lr)
            assert np.array_equal(m, r["m12"]) and n == r["count"], (c.name, p)


def test_closed_form_walk_equals_bresenham():
    """Every step, and the steps whose window reaches the grid: those cells of the full walk, in order."""
    rng = np.random.default_rng(5)
    for _ in range(3000):
        x1, y1, x2, y2 = (int(v) for v in rng.integers(-300, 400, 4))
        full = mg.bresenham(x1, y1, x2, y2)
        assert list(zip(*(a.tolist() for a in mc.walk(x1, y1, x2, y2)))) == full
        w = tuple(int(v) for v in rng.integers(0, 4, 4))
        reach = lambda c: c[0] + w[1] >= 0 and c[0] - w[0] < mc.COLS and c[1] + w[3] >= 0 and c[1] - w[2] < mc.ROWS  # noqa: E731
        part = list(zip(*(a.tolist() for a in mc.walk(x1, y1, x2, y2, reach=(w, mc.COLS, mc.ROWS)))))
        assert [c for c in full if reach(c)] == [c for c in part if reach(c)]
        assert set(part) <= set(full)


def test_closed_form_walk_at_the_end_point_clamp():
    """At +-2^28 the closed form stays on the line: each cell is within half a cell of the exact segment."""
    R = mc.QCELL
    for x1, y1, x2, y2 in ((-R, 10, R, 12), (20, -R, 22, R), (-R, -R, R, R - 3), (R, 7, -R, -5)):
        x, y = mc.walk(x1, y1, x2, y2, reach=((3, 3, 3, 3), mc.COLS, mc.ROWS))
        assert len(x) > 0
        if abs(x2 - x1) >= abs(y2 - y1):
            exact = y1 + (x - x1) * (y2 - y1) / (x2 - x1)
            assert np.all(np.abs(y - exact) <= 0.5 + 1e-9)
        else:
            exact = x1 + (y - y1) * (x2 - x1) / (y2 - y1)
            assert np.all(np.abs(x - exact) <= 0.5 + 1e-9)


def test_sizes_reach_every_count():
    cases = mc.sizes()
    n1 = {int(c.n1[0]) for c in cases if not c.lines}
    n2 = {int(c.n2[0]) for c in cases if not c.lines}
    assert set(mc.N1) <= n1 and set(mc.N2) <= n2
    assert {0, 3, 4, 5, 127, 128, 129} <= {int(c.n1[0]) for c in cases if c.lines}


@pytest.mark.parametrize("best_lr", [True, False])
def test_a_column_minimum_ties_across_the_query_blocks_and_the_earlier_query_keeps_it(best_lr):
    c = _by_name(f"ties-lr{int(best_lr)}")
    r = mc.reference(c, 0)
    d = mc.hamming(c.d1[0], c.d2[0])
    for (a, b), j in zip(mc.TIE_PAIRS, (3, 7)):
        assert d[a, j] == d[b, j] == 0 and np.array_equal(c.q[0, a], c.q[0, b])
        if best_lr:
            assert r["m21"][j] == a and r["m12"][a] == j and r["m12"][b] != j
        else:
            assert r["m12"][a] == r["m12"][b] == -1 or r["m12"][a] == j
    assert r["best_d"][10] == r["best_d2"][10] and r["m12"][10] == -1     # equal best and second best
    assert r["best_d"][1] == 256 and r["best_d2"][1] == mc.INT_MAX and r["m12"][1] == 64
    far = np.flatnonzero((c.q[0, :, 0] == 60))
    assert len(far) > 50 and np.all(r["best_d"][far] == mc.INT_MAX)        # non-candidates interleaved


def test_ratio_pins_tie_in_f32():
    """At each base ratio the pairs put best_d == f32(best_d2 * nnr) (0.8: never the exact product), which the strict
    '<' rejects; one ulp above 0.9 some pairs still tie in f32 while the exact product exceeds best_d, so exact
    arithmetic would accept them; one ulp above the base some pairs are accepted."""
    up9 = np.nextafter(np.float32(0.9), np.float32(2))
    assert any(mc.f32_ties(b, b2, up9) and b2 * float(up9) > b for b, b2 in mc.ratio_pairs(np.float32(0.9)))
    for nnr0 in (0.9, 0.75, 0.8):
        pairs = mc.ratio_pairs(np.float32(nnr0))
        assert len(pairs) > 20 and all(mc.f32_ties(b, b2, nnr0) for b, b2 in pairs)
        r = mc.reference(_by_name(f"ratio-{nnr0:g}-at"), 0)
        q = range(min(len(pairs), 40))   # the small instances keep the first 40 pairs
        assert all(r["m12"][i] == -1 for i in q)
        ra = mc.reference(_by_name(f"ratio-{nnr0:g}-above"), 0)
        assert any(ra["m12"][i] >= 0 for i in q)
    r1 = mc.reference(_by_name("ratio-1-above"), 0)
    c1 = _by_name("ratio-1-above")
    assert c1.nnr > 1 and np.all(r1["best_d"] < mc.INT_MAX)            # every query has a candidate
    tied = np.flatnonzero((r1["best_d"] == r1["best_d2"]) & (r1["best_d"] > 0))   # 0 < 0 * nnr never holds
    assert len(tied) > 10 and np.all(r1["m12"][tied] >= 0)
    assert np.all(r1["m12"][tied] == r1["best_idx"][tied])             # the earlier train point of the two
    assert np.all(mc.reference(_by_name("ratio-1-at"), 0)["m12"][tied] == -1)
    assert {c.nnr for c in mc.ratio_pins() if c.name.startswith("ratio-config")} == set(mc.RATIOS)


def test_the_gate_sits_exactly_on_line_sim_th():
    c = _by_name("lines-gate-exact")
    vx, vy = mc.line_dirs(c.q[0])
    cosv = np.abs(vx * c.tdir[0, :, 0] + vy * c.tdir[0, :, 1])
    assert cosv[0] == cosv[1] == c.th and cosv[2] == cosv[3] == np.nextafter(c.th, 0.0) and np.isnan(cosv[4])
    r = mc.reference(c, 0)
    assert list(r["m12"]) == [0, 1, -1, -1, 4, 5, -1]
    at, above = mc.reference(_by_name("lines-gate-slanted-at"), 0), mc.reference(_by_name("lines-gate-slanted-above"), 0)
    assert list(at["m12"]) == [0] and list(above["m12"]) == [-1]


def test_grids_sit_at_the_query_mask_and_the_huge_case_spans_chunks():
    assert {(c.cols, c.rows) for c in mc.grids() if c.fits_batch()} == set(mc.GRIDS_BOTH)
    assert all(c * r == mc.MASK_CELLS for c, r in mc.GRIDS_BOTH[1:])
    assert all(c * r > mc.MASK_CELLS for c, r in mc.GRIDS_REFUSED)
    (h,) = mc.huge()
    assert (h.K, h.Kt) == (mc.K_MAX, mc.KT_MAX) and h.counts(0) == (mc.K_MAX, mc.KT_MAX) and mc.chunks(h) == h.P == 3


def test_batches_clamp_share_slots_and_permute():
    cs = {c.name: c for c in mc.batches()}
    for kind in ("points", "lines"):
        over = cs[f"batch-{kind}-over"]
        assert (over.n1 > over.K).any() and (over.n2 > over.Kt).any()
        slots = cs[f"batch-{kind}-slots"].q_slot
        assert len(set(slots.tolist())) < len(slots)
        assert sorted(cs[f"batch-{kind}-permuted"].n1.tolist()) == sorted(cs[f"batch-{kind}-mixed"].n1.tolist())


def test_far_lines_reach_the_clamp_and_windows_reach_in_from_outside():
    far = [c for c in mc.pixel_lines() if c.far]
    assert far and all(np.abs(c.q).max() == mc.QCELL for c in far)
    c = next(c for c in mc.windows() if c.name == "window-points-w3")
    q = c.q[0, :c.n1[0]]
    outside = (q[:, 0] < 0) | (q[:, 0] >= mc.COLS) | (q[:, 1] < 0) | (q[:, 1] >= mc.ROWS)
    r = mc.reference(c, 0)
    assert (r["best_d"][outside] < mc.INT_MAX).any()
