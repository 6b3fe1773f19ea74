"""GPU tests of the two dense LDL^T factorisations on their own (fe.debug_ldlt): the tiled one of plf_global_ba /
plf_pose_graph (path 0) at every size of tests/ldlt_cases.py, the one-CTA one of plf_local_ba (path 1) wherever
n6 <= 64.  Each is checked against the long-double reference: the backward error of every lower entry and of the
solution, the forward error on the well-conditioned cases, the zero-tile flags exactly, bit-identical repeats, an
upper triangle that is never read, tile offsets through a block-diagonal matrix, NaN / Inf and zero pivots, and the
plf_global_ba capacity (n6 = 4096)."""
import ctypes as C
import functools
import time

import numpy as np
import pytest

import ldlt_cases as lc

pytestmark = pytest.mark.gpu

_WORST = {}   # path -> (largest backward-error ratio, case id)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for path, (r, name) in sorted(_WORST.items()):
        print(f"\nldlt path {path}: largest backward-error ratio {r:.3g} of the 3 n u bound ({name})")


@functools.lru_cache(maxsize=None)
def _ref(case):
    S, g, rec = lc.make(case)
    L, D = lc.ldlt(S)
    return S, g, rec, L, D


_DEV = {}


def _dev(fe, case, path):
    if (case, path) not in _DEV:
        S, g, _, _, _ = _ref(case)
        _DEV[case, path] = fe.debug_ldlt(S, g, path)
    return _DEV[case, path]


def _paths(n6):
    return [p for p in (0, 1) if n6 <= lc.PATH_MAX_N6[p]]


FINITE = [(c, p) for c in lc.finite_cases() for p in _paths(c.n6)]
FINITE_IDS = [f"{c.id}-path{p}" for c, p in FINITE]


def _lower_bits(A):
    return np.tril(A).view(np.uint64)


@pytest.mark.parametrize("case,path", FINITE, ids=FINITE_IDS)
def test_backward_error_of_every_lower_entry_and_of_the_solution(fe, case, path):
    """|S - L D L^T|_ij <= 3 n u (|L| |D| |L^T|)_ij for every i >= j, and ||S x - g|| <= 3 n u || |L||D||L^T| || ||x||
    (infinity norms), in long double on the device's L, D and x"""
    S, g, _, _, _ = _ref(case)
    LD, x, _ = _dev(fe, case, path)
    n = len(g)
    L, D = lc.split(LD)
    assert np.all(np.isfinite(L)) and np.all(np.isfinite(D)) and np.all(np.isfinite(x))
    P, Q = lc.product(L, D)
    Sl = np.tril(S).astype(np.longdouble)
    err = np.abs(Sl - P)
    bound = 3 * n * lc.U * Q
    assert np.all(err[bound == 0] == 0)
    ratio = float((err[bound > 0] / bound[bound > 0]).max()) if (bound > 0).any() else 0.0
    Sf = S.astype(np.longdouble)
    res = np.abs(Sf @ x.astype(np.longdouble) - g).max()
    La = np.abs(L).astype(np.longdouble)
    qnorm = (La @ (np.abs(D) * (La.T @ np.ones(n, np.longdouble)))).max()
    rres = float(res / (3 * n * lc.U * qnorm * np.abs(x).max()))
    worst = max(ratio, rres)
    if worst > _WORST.get(path, (-1.0, ""))[0]:
        _WORST[path] = (worst, case.id)
    print(f"{case.id} path {path}: backward {ratio:.3g}, residual {rres:.3g}")
    assert ratio <= 1.0 and rres <= 1.0


@pytest.mark.parametrize("case,path", [cp for cp in FINITE if lc.well_conditioned(cp[0])],
                         ids=[i for cp, i in zip(FINITE, FINITE_IDS) if lc.well_conditioned(cp[0])])
def test_forward_error_on_the_well_conditioned_cases(fe, case, path):
    """L within 64 n u of each row's largest |L|, D within 64 n u |D_j|, x within 8 n u kappa_inf(S) ||x||"""
    S, g, _, Lr, Dr = _ref(case)
    LD, x, _ = _dev(fe, case, path)
    n = len(g)
    L, D = lc.split(LD)
    Lr64 = np.asarray(Lr, np.float64)
    tol = 64 * n * lc.U
    row = np.abs(Lr64).max(axis=1)
    assert np.all(np.abs(np.asarray(L - Lr, np.float64)).max(axis=1) <= tol * row)
    assert np.all(np.abs(np.asarray(D - Dr, np.float64)) <= tol * np.abs(np.asarray(Dr, np.float64)))
    xr = lc.solve(Lr, Dr, g)
    kappa = np.abs(S).sum(axis=1).max() * np.abs(np.linalg.inv(S)).sum(axis=1).max()
    assert np.abs(np.asarray(x - xr, np.float64)).max() <= 8 * n * lc.U * kappa * float(np.abs(xr).max())


@pytest.mark.parametrize("case", [c for c in lc.finite_cases()], ids=lambda c: c.id)
def test_zero_flags_are_the_eliminations_and_zero_tiles_stay_plus_zero(fe, case):
    """path 0: nz is 1 exactly on the tiles (i > k) of L the elimination makes non-zero, 0 everywhere else, and every
    lower tile flagged zero holds +0.0 in the output (bit pattern 0)"""
    _, _, rec, Lr, _ = _ref(case)
    LD, _, nz = _dev(fe, case, 0)
    exp = lc.lower_tiles(np.asarray(Lr, np.float64))
    assert np.array_equal(exp, lc.tile_fill(rec["tiles"]))
    assert np.array_equal(nz.astype(bool), exp), np.argwhere(nz.astype(bool) != exp)[:8]
    n = len(LD)
    nt = lc.n_tiles(n)
    for i, k in zip(*np.nonzero(np.tril(~exp, -1))):
        blk = LD[64 * i:min(n, 64 * i + 64), 64 * k:64 * k + 64]
        assert not blk.view(np.uint64).any(), (i, k)
    assert nt == len(nz)


REPEAT = [(c, p) for c, p in FINITE if c.n6 in lc.SIZES_SMALL or c.n6 in (96, 200)]


@pytest.mark.parametrize("case,path", REPEAT, ids=[f"{c.id}-path{p}" for c, p in REPEAT])
def test_repeats_are_bit_identical_and_the_upper_triangle_is_never_read(fe, case, path):
    """Two calls give the same bits (no atomics), and NaN in every strict-upper entry changes neither the lower
    triangle nor x by a single bit"""
    S, g, _, _, _ = _ref(case)
    LD, x, nz = _dev(fe, case, path)
    LD2, x2, nz2 = fe.debug_ldlt(S, g, path)
    assert np.array_equal(_lower_bits(LD), _lower_bits(LD2)) and np.array_equal(x.view(np.uint64), x2.view(np.uint64))
    assert path == 1 or np.array_equal(nz, nz2)
    Sg = S.copy()
    Sg[np.triu_indices(len(g), 1)] = np.nan
    LD3, x3, nz3 = fe.debug_ldlt(Sg, g, path)
    assert np.array_equal(_lower_bits(LD), _lower_bits(LD3)) and np.array_equal(x.view(np.uint64), x3.view(np.uint64))
    assert path == 1 or np.array_equal(nz, nz3)


BLOCKS = [(64, 0), (64, 1), (200, 0), (266, 0)]


@pytest.mark.parametrize("n6,path", BLOCKS, ids=[f"{a}-path{b}" for a, b in BLOCKS])
def test_block_diagonal_factors_bit_for_bit_like_each_block_alone(fe, n6, path):
    """Blocks of 192 = lcm(6, 64) rows start on tile boundaries: each block of L, D and x equals the call on that
    block alone (the last one partial), so every tile offset reaches the right rows and columns"""
    S, g, _, _, _ = _ref(lc.Case("blockdiag", "dominant", n6))
    LD, x, _ = fe.debug_ldlt(S, g, path)
    n = len(g)
    for b0 in range(0, n, lc.BLOCK):
        b1 = min(n, b0 + lc.BLOCK)
        LDb, xb, _ = fe.debug_ldlt(S[b0:b1, b0:b1], g[b0:b1], path)
        assert np.array_equal(_lower_bits(LD[b0:b1, b0:b1]), _lower_bits(LDb)), b0
        assert np.array_equal(x[b0:b1].view(np.uint64), xb.view(np.uint64)), b0
        assert not np.tril(LD[b1:, b0:b1]).view(np.uint64).any()


def _nonfinite(D):
    return ~((D > 0) & np.isfinite(D))   # k_pgo_step's test of a failed factorisation (cholmod's not-positive-definite)


# (n6, pattern, where, r, c): a lower entry in the last valid row, in a tile that is otherwise zero (band1 leaves tile
# (n_t - 1, 0) zero from n_t = 3); a diagonal entry; lower entries inside dense tiles; one in the strict upper triangle
PLANTS = []
for _n6 in (11, 64, 96):
    _n = 6 * _n6
    PLANTS += [(_n6, "band1", "zero_tile" if _n > 128 else "lower", _n - 1, 0),
               (_n6, "band1", "diagonal", _n // 2, _n // 2),
               (_n6, "dense", "lower", _n - 1, _n - 3), (_n6, "dense", "lower", min(70, _n - 1), 5),
               (_n6, "band1", "upper", 3, _n - 2)]
# inside the first 192-row block of a block-diagonal matrix: the dense factorisation spreads the NaN through its zero
# products into every later block, the tiled one skips those tiles and leaves the later blocks' pivots untouched
PLANTS += [(64, "blockdiag", "block", 100, 50), (96, "blockdiag", "block", 150, 149)]
NONFINITE = [(pl, v, p) for pl in PLANTS for v in (np.nan, np.inf) for p in _paths(pl[0])]


@pytest.mark.parametrize("plant,v,path", NONFINITE,
                         ids=[f"{pl[0]}-{pl[2]}-{pl[3]}-{pl[4]}-{v}-path{p}" for pl, v, p in NONFINITE])
def test_a_nan_or_inf_fails_its_own_pivot_and_no_pivot_the_dense_factorisation_keeps(fe, plant, v, path):
    """A NaN or +Inf at a lower entry (r, c) makes D_r fail k_pgo_step's test (!(D > 0 && D finite)), and every D that
    fails it also fails in the dense long-double factorisation (no zero skipped); one in the strict upper triangle
    changes nothing, bit for bit"""
    n6, pattern, where, r, c = plant
    S, g, _, _, _ = _ref(lc.Case(pattern, "dominant", n6))
    Sp = lc.plant(S, r, c, v)
    LD, x, _ = fe.debug_ldlt(Sp, g, path)
    D = LD.diagonal()
    if where == "upper":
        LD0, x0, _ = _dev(fe, lc.Case(pattern, "dominant", n6), path)
        assert np.array_equal(_lower_bits(LD), _lower_bits(LD0)) and np.array_equal(x.view(np.uint64), x0.view(np.uint64))
        return
    _, Dd = lc.ldlt(Sp, skip_zeros=False, dtype=np.float64)   # only which pivots stay finite matters here
    bad, bad_dense = _nonfinite(D), _nonfinite(np.asarray(Dd, np.float64))
    assert bad[r], (r, D[r])
    assert not np.any(bad & ~bad_dense), np.flatnonzero(bad & ~bad_dense)[:8]
    assert not bad[:min(r, c)].any()   # the pivots before the entry's row and column are the clean ones
    if where == "block" and path == 0:
        D0 = _dev(fe, lc.Case(pattern, "dominant", n6), path)[0].diagonal()
        assert bad_dense[lc.BLOCK:].all() and not bad[lc.BLOCK:].any()
        assert np.array_equal(D[lc.BLOCK:].view(np.uint64), D0[lc.BLOCK:].view(np.uint64))
    print(f"{plant} {v} path {path}: {bad.sum()} non-finite D of {len(D)}, dense {bad_dense.sum()}")


ZERO_PIVOT = [(n6, j, p) for n6, j in ((11, 0), (11, 65), (64, 63), (64, 383), (96, 300), (96, 575)) for p in _paths(n6)]


@pytest.mark.parametrize("n6,j,path", ZERO_PIVOT, ids=[f"{a}-{b}-path{c}" for a, b, c in ZERO_PIVOT])
def test_an_exactly_zero_pivot_gives_d_zero_and_a_non_finite_solution(fe, n6, j, path):
    S, g, _, _, _ = _ref(lc.Case("dense", "dominant", n6))
    LD, x, _ = fe.debug_ldlt(lc.zero_pivot(S, j), g, path)
    D = LD.diagonal()
    assert D[j] == 0.0 and np.all(D[:j] > 0) and np.all(np.isfinite(D[:j]))
    assert not np.all(np.isfinite(x))


def test_refuses_bad_arguments_and_stays_usable(fe):
    import plslam_b200 as plf
    n = 12
    S = np.eye(n)
    g = np.ones(n)
    x = np.zeros(n)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
    lib = fe.lib
    for path, n6 in ((2, 2), (-1, 2), (0, 0), (1, 0), (0, 4097), (1, 65), (0, -3)):
        assert lib.plf_debug_ldlt(fe._ctx, path, n6, dp(S), dp(g), dp(x), None) == -1, (path, n6)
        assert "plf_debug_ldlt" in lib.plf_last_error(fe._ctx).decode()
    for args in ((None, dp(g), dp(x)), (dp(S), None, dp(x)), (dp(S), dp(g), None)):
        assert lib.plf_debug_ldlt(fe._ctx, 0, 2, *args, None) == -1
    assert lib.plf_debug_ldlt(None, 0, 2, dp(S), dp(g), dp(x), None) == -1
    with pytest.raises(plf.PlfError):
        fe.debug_ldlt(np.eye(7), np.ones(7))
    for path in (0, 1):
        LD, xo, _ = fe.debug_ldlt(2 * np.eye(n), np.ones(n), path)
        assert np.array_equal(LD.diagonal(), np.full(n, 2.0)) and np.array_equal(xo, np.full(n, 0.5))


def test_max_size_banded_plus_loops():
    """n6 = 4096 (n = 24 576, n_t = 384, plf_global_ba's capacity) on the pose graph's shape: block tridiagonal plus 24
    loop blocks.  The zero flags equal the tile-level elimination's, flagged tiles hold +0.0, every D is positive and
    the solution's residual, by scipy.sparse, is within 3 n u ||S|| ||x||.  Its own context, closed afterwards, so that
    the 4.8 GB of scratch does not stay in the shared one; about 5 GB of host memory for the dense upload."""
    import plslam_b200 as plf
    n6 = lc.MAX_N6
    Ssp, g = lc.band_plus_loops(n6, 24, seed=4)
    n = 6 * n6
    nt = lc.n_tiles(n)
    tiles = lc.sparse_tiles(Ssp)
    exp = lc.tile_fill(tiles)
    Cl = Ssp.tocoo()
    keep = Cl.row >= Cl.col
    dense = np.zeros((n, n))
    dense[Cl.row[keep], Cl.col[keep]] = Cl.data[keep]
    with plf.Frontend(device=0) as big:
        t0 = time.perf_counter()
        LD, x, nz = big.debug_ldlt(dense, g, 0, overwrite_s=True)
        dt = time.perf_counter() - t0
    print(f"\nn6 = 4096: plf_debug_ldlt {dt:.2f} s including the 4.8 GB upload and download; "
          f"{int(exp.sum())} non-zero L tiles of {nt * (nt - 1) // 2}")
    assert np.array_equal(nz.astype(bool), exp)
    D = LD.diagonal()
    assert np.all(D > 0) and np.all(np.isfinite(D)) and np.all(np.isfinite(x))
    V = LD.reshape(nt, 64, nt, 64)
    for i in range(1, nt):   # tile row by tile row, to bound the temporaries
        z = np.flatnonzero(~exp[i, :i])
        if len(z):
            assert not V[i][:, z, :].view(np.uint64).any(), i
    Snorm = float(abs(Ssp).sum(axis=1).max())
    res = np.abs(Ssp @ x - g).max()
    assert res <= 3 * n * lc.U * Snorm * np.abs(x).max(), res
