"""CPU tests of tests/ldlt_cases.py: the long-double LDL^T reference against 50-digit mpmath and scipy's Cholesky, the
tile pattern each generator claims and the fill the elimination produces from it, the sizes the sweep covers, and
gba_update's decode of its block index into tile pairs.  No GPU."""
import functools

import numpy as np
import pytest
import scipy.linalg

import ldlt_cases as lc

EPS_LD = float(np.finfo(np.longdouble).eps) / 2   # unit roundoff of np.longdouble


@functools.lru_cache(maxsize=None)
def _ref(case):
    S, g, rec = lc.make(case)
    L, D = lc.ldlt(S)
    return S, g, rec, L, D


def _rel_rows(A, B, Lref):
    """max |A - B| of each row over that row's largest |L| (the unit diagonal included)"""
    scale = np.abs(np.asarray(Lref, np.float64)).max(axis=1)
    return (np.abs(np.asarray(A - B, np.float64)).max(axis=1) / scale).max()


def _mpf(v):
    """a long double as an mpf, exactly (its 64-bit significand is the sum of two doubles)"""
    import mpmath
    hi = np.float64(v)
    return mpmath.mpf(float(hi)) + mpmath.mpf(float(np.float64(v - np.longdouble(hi))))


SMALL_MP = [lc.Case(p, v, n6) for n6 in (1, 10, 11) for p in ("dense", "band1", "randmask", "single") for v in lc.VALUES]


@pytest.mark.parametrize("case", SMALL_MP, ids=lambda c: c.id)
def test_long_double_reference_agrees_with_mpmath(case):
    """n <= 66: the long-double factors and solution within 64 n of its own unit roundoff of the 50-digit ones"""
    import mpmath
    S, g, _, L, D = _ref(case)
    n = len(D)
    Lm, Dm = lc.ldlt_mp(S)
    tol = 64 * n * EPS_LD
    with mpmath.workdps(50):
        for i in range(n):
            row = max(abs(v) for v in Lm[i])
            for j in range(i):
                assert abs(_mpf(L[i, j]) - Lm[i][j]) <= tol * row, (i, j)
        for j in range(n):
            assert abs(_mpf(D[j]) - Dm[j]) <= tol * abs(Dm[j]), (j, D[j], Dm[j])
        x = lc.solve(L, D, g)
        xm = mpmath.lu_solve(mpmath.matrix([[float(S[max(i, j), min(i, j)]) for j in range(n)] for i in range(n)]),
                             mpmath.matrix([float(v) for v in g]))
        err = max(abs(_mpf(x[i]) - xm[i]) for i in range(n))
        big = max(abs(v) for v in xm)
    # the systems are well conditioned (kappa < 1e13 for 'scaled'): the long-double solve keeps far more than double
    assert float(err) <= 1e-12 * float(big), (float(err), float(big))


CHOL = [lc.Case(p, v, n6) for n6 in (11, 32, 65, 96) for p in ("dense", "band5", "rarrow", "blockdiag") for v in ("dominant", "scaled")]


@pytest.mark.parametrize("case", CHOL, ids=lambda c: c.id)
def test_long_double_reference_agrees_with_cholesky(case):
    """SPD cases: L = L_c / diag(L_c), D = diag(L_c)^2 from scipy.linalg.cholesky (double, LAPACK) within 64 n u"""
    S, _, _, L, D = _ref(case)
    n = len(D)
    Lc = scipy.linalg.cholesky(S, lower=True)
    dc = np.diag(Lc)
    Lchol, Dchol = Lc / dc, dc * dc
    tol = 64 * n * lc.U
    assert _rel_rows(np.asarray(L, np.float64), Lchol, L) <= tol
    assert np.all(np.abs(np.asarray(D, np.float64) - Dchol) <= tol * np.abs(Dchol))


@pytest.mark.parametrize("case", lc.finite_cases(), ids=lambda c: c.id)
def test_generator_builds_its_pattern_and_the_elimination_fills_as_claimed(case):
    S, _, rec, L, D = _ref(case)
    n = len(S)
    nt = lc.n_tiles(n)
    assert S.shape == (n, n) and n == 6 * case.n6 and np.array_equal(S, S.T) and np.all(np.isfinite(S))
    tiles = lc.lower_tiles(S)
    assert np.array_equal(tiles, rec["tiles"])
    I, K = np.meshgrid(np.arange(nt), np.arange(nt), indexing="ij")
    low = I > K
    p = case.pattern
    if p == "dense":
        assert np.array_equal(tiles, low)
    elif p in ("band1", "band5"):            # narrower than one tile: only the first sub-diagonal of tiles
        assert np.array_equal(tiles, low & (I == K + 1))
    elif p == "band15":                      # 90 wide: the second sub-diagonal too
        assert np.array_equal(tiles, low & (I <= K + 2))
    elif p == "arrow":
        assert np.array_equal(tiles, low & (I == nt - 1))
    elif p == "rarrow":
        assert np.array_equal(tiles, low & (K == 0))
    elif p == "blockdiag":
        assert np.array_equal(tiles, low & (I // 3 == K // 3))
    elif p == "single":
        for ti, tk in zip(*np.nonzero(tiles)):
            blk = S[64 * ti:64 * ti + 64, 64 * tk:64 * tk + 64]
            r, c = np.nonzero(blk)
            assert len(r) == 1 and c[0] == 63 and (r[0] == 63 or 64 * ti + r[0] == n - 1)
        if nt >= 2:
            assert S[n - 1, :64 * (nt - 1)].any()   # the last valid row of the last tile holds it
    elif p == "negative":
        assert tiles.sum() == (nt >= 2)
        for ti, tk in rec["negative_tiles"]:
            blk = S[64 * ti:64 * ti + 64, 64 * tk:64 * tk + 64]
            assert np.all(blk[:min(64, n - 64 * ti)] < 0)
    elif p == "randmask" and nt >= 4:
        assert 0 < tiles.sum() < low.sum()
    # the values: dominance, scale, signs of D
    off = np.abs(S).sum(axis=1) - np.abs(np.diag(S))
    if case.values != "scaled":
        assert np.all(np.abs(np.diag(S)) > off)
    if case.values == "dominant":
        assert np.all(D > 0)
    elif case.values == "quasi" and n > 1:
        assert (D < 0).any() and (D > 0).any()
        assert np.array_equal(np.sign(np.asarray(D, np.float64)), np.sign(np.diag(S)))
    elif case.values == "scaled" and n >= 60:
        dg = np.abs(np.diag(S))
        assert dg.min() < 1e-3 and dg.max() > 1e3
    # the fill: the reference's zero tiles of L are what the tile-level elimination predicts
    fill = lc.tile_fill(tiles)
    assert np.array_equal(lc.lower_tiles(np.asarray(L, np.float64)), fill)
    if p == "rarrow" and nt >= 3:
        assert np.array_equal(fill, low) and fill.sum() > tiles.sum()   # tiles that start at zero are filled


def test_the_sweep_covers_every_even_residue_and_the_tile_counts():
    n = [6 * n6 for n6 in lc.SIZES_RESIDUE]
    assert {v % 64 for v in n} == set(range(0, 64, 2)) and min(lc.n_tiles(v) for v in n) >= 7
    nt = {n6: lc.n_tiles(6 * n6) for n6 in lc.SIZES_SMALL}
    assert nt[1] == nt[10] == 1 and nt[11] == 2 and 6 * 11 - 64 == 2 and nt[64] == 6 and nt[65] == 7
    assert lc.n_tiles(6 * lc.MAX_N6) == 384 and 383 * 384 // 2 == 73536
    cases = lc.finite_cases()
    for n6 in lc.SIZES_SMALL:
        assert {c.pattern for c in cases if c.n6 == n6} == set(lc.PATTERNS)
    assert {c.n6 for c in cases} >= set(lc.SIZES_SMALL) | set(lc.SIZES_RESIDUE) | set(lc.SIZES_LARGE)


def test_band_plus_loops_fill_matches_the_reference_and_stays_clear_of_underflow():
    """The 4096-keyframe case's shape at 400 keyframes, with loops as long as there: its tile fill by the tile-level
    elimination equals the zero tiles of the reference's L, so the GPU test can take its expected zero flags from
    tile_fill alone, and the smallest non-zero |L| stays far above double's underflow, so that no fill turns into an
    exact zero on the device.  Loops of 2 000 keyframes would not: the fill decays along the band."""
    S, _ = lc.band_plus_loops(400, 4, seed=1)
    assert S.shape == (2400, 2400) and lc.n_tiles(2400) == 38
    Sd = S.toarray()
    L, D = lc.ldlt(Sd)
    assert np.all(D > 0)
    La = np.abs(L[np.tril_indices(len(D), -1)])
    assert La[La > 0].min() > 1e-200
    tiles = lc.sparse_tiles(S)
    assert np.array_equal(tiles, lc.lower_tiles(Sd))
    fill = lc.tile_fill(tiles)
    assert fill.sum() > tiles.sum()
    assert np.array_equal(lc.lower_tiles(np.asarray(L, np.float64)), fill)
    # one loop of 550 .. 1 100 keyframes: factored in double, whole fill tiles underflow to exact zeros
    S, _ = lc.band_plus_loops(1200, 1, seed=1, max_span=1100)
    L, _ = lc.ldlt(S.toarray(), dtype=np.float64)
    fill, got = lc.tile_fill(lc.sparse_tiles(S)), lc.lower_tiles(L)
    assert not np.any(got & ~fill) and got.sum() < fill.sum()


def test_update_decode_enumerates_every_tile_pair_once():
    """k_gbb_update launches m (m + 1) / 2 CTAs per system at tile column k (m = n_t - k - 1 trailing tiles, up to 383)
    and gba_update decodes blockIdx.x into (a, b), 0 <= b <= a < m: for every m each pair is produced exactly once, in
    row order"""
    tmax = 383 * 384 // 2
    a, b = lc.update_pair(np.arange(tmax))
    assert np.all((0 <= b) & (b <= a))
    # row by row: t = a (a + 1) / 2 + b, so the first m (m + 1) / 2 indices are exactly the pairs of rows < m
    assert np.array_equal(a * (a + 1) // 2 + b, np.arange(tmax))
    for m in range(1, 384):
        cnt = m * (m + 1) // 2
        am, bm = a[:cnt], b[:cnt]
        assert am.max() == m - 1
        keys = am * 384 + bm
        assert len(np.unique(keys)) == cnt
    # the square root alone is already exact here; the correction loops never run
    a0 = ((np.sqrt(8.0 * np.arange(tmax) + 1.0) - 1.0) * 0.5).astype(np.int64)
    assert np.array_equal(a0, a)
