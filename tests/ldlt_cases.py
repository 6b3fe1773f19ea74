"""Symmetric matrices built to reach what the BA / PGO systems leave to chance in the two dense LDL^T factorisations
(gbb_ldlt's gba_* stages and lba_solve, csrc/lba.cu): every pattern of zero 64 x 64 tiles the tiled one skips or fills, partial
last tiles, badly scaled and indefinite values, zero pivots and planted NaN / Inf; and the reference they are checked
against.  Pure numpy (mpmath for the smallest sizes), seeded; every generator returns (S, g, record) where the record
names the case and the tile pattern of S it is built to have.  tests/test_ldlt.py measures, without a GPU, that the
reference is right and that each matrix has the pattern its record claims; tests/test_ldlt_gpu.py runs the device on them.

The reference is the right-looking LDL^T without pivoting both kernels implement, in np.longdouble (64-bit significand
on x86-64, 11 bits more than the device's double), vectorised by column: after column j, A[i][j] = L_ij and
A[j][j] = D_j.  It reads only the lower triangle of S, as the kernels do."""
from dataclasses import dataclass

import numpy as np

T = 64                  # csrc/plf_internal.h PLF_LDLT_TILE
U = 2.0 ** -53          # unit roundoff of double
PATH_MAX_N6 = {0: 4096, 1: 64}   # plf_debug_ldlt: the tiled factorisation (plf_global_ba's capacity), the one-CTA one
BLOCK = 192             # lcm(6, 64): keyframe blocks and tiles both end on its multiples

# n_t = 1 without a panel launch, 1 -> 2 tiles with a 2-row last tile, 2 -> 6 tiles, the one-CTA path's capacity and one
# past it
SIZES_SMALL = (1, 10, 11, 21, 32, 64, 65)
SIZES_RESIDUE = tuple(range(65, 97))    # n = 6 n6 takes every even residue mod 64, at n_t >= 7
SIZES_LARGE = (200, 266)
MAX_N6 = 4096                           # n = 24 576, n_t = 384: 73 536 update CTAs at k = 0

PATTERNS = ("dense", "band1", "band5", "band15", "arrow", "rarrow", "blockdiag", "randmask", "single", "negative")
VALUES = ("dominant", "scaled", "quasi")


def n_tiles(n):
    return (n + T - 1) // T


# ---- tile patterns ----------------------------------------------------------------------------------------------------

def tile_any(M):
    """n_t x n_t: whether tile (I, K) of M holds an entry that is not +-0 (NaN counts), padded with zeros past n."""
    n = M.shape[0]
    nt = n_tiles(n)
    P = np.zeros((nt * T, nt * T), bool)
    P[:n, :n] = M != 0
    return P.reshape(nt, T, nt, T).any(axis=(1, 3))


def lower_tiles(M):
    """The strictly lower tiles (I > K) of M that hold an entry other than +-0 in its lower triangle: the zero flags
    gba_panel sets, as an n_t x n_t bool array (False on and above the tile diagonal)."""
    return np.tril(tile_any(np.tril(M)), -1)


def tile_fill(tiles):
    """The tile pattern of L from that of S by the elimination at tile granularity: L_IK != 0 iff S_IK != 0 or some
    J < K has L_IJ != 0 and L_KJ != 0.  Exact for the generators below, whose non-zero tiles fill every column they
    reach (tests/test_ldlt.py compares it with the reference's own zeros)."""
    P = np.tril(np.asarray(tiles, bool), -1).copy()
    for k in range(len(P)):
        r = np.flatnonzero(P[k + 1:, k]) + k + 1
        if len(r) > 1:
            P[np.ix_(r, r)] |= np.tril(np.ones((len(r), len(r)), bool), -1)
    return P


# ---- the reference ----------------------------------------------------------------------------------------------------

def ldlt(S, skip_zeros=True, dtype=np.longdouble):
    """(L, D) of S's lower triangle in `dtype`: L unit lower triangular, zeros above.  skip_zeros leaves out the trailing
    update of the rows whose L_ij is +-0, which changes nothing for finite S; a NaN or Inf spreads through those products
    only without it (the dense factorisation's behaviour)."""
    A = np.tril(np.asarray(S)).astype(dtype)
    n = len(A)
    with np.errstate(all="ignore"):
        for j in range(n - 1):
            dj = A[j, j]
            col = A[j + 1:, j]
            col /= dj
            if skip_zeros:
                idx = np.flatnonzero(col)
                if len(idx) == 0:
                    continue
                if len(idx) < len(col):
                    r = idx + j + 1
                    A[np.ix_(r, r)] -= np.multiply.outer(col[idx] * dj, col[idx])
                    continue
            A[j + 1:, j + 1:] -= np.multiply.outer(col * dj, col)   # (L_ij D_j) L_kj, as both kernels group it
    D = A.diagonal().copy()
    L = np.tril(A, -1)
    np.fill_diagonal(L, 1)
    return L, D


def solve(L, D, g):
    """x of L D L^T x = g in L's dtype: forward substitution by columns, scaling, backward substitution by rows."""
    y = np.array(g, L.dtype)
    n = len(y)
    with np.errstate(all="ignore"):
        for k in range(n - 1):
            y[k + 1:] -= L[k + 1:, k] * y[k]
        x = y / D
        for k in range(n - 1, 0, -1):
            x[:k] -= L[k, :k] * x[k]
    return x


def ldlt_mp(S, dps=50):
    """The same factorisation in mpmath at `dps` digits, element by element (small n only): (L, D) as lists of mpf."""
    import mpmath
    n = len(S)
    with mpmath.workdps(dps):
        A = [[mpmath.mpf(float(S[i][j])) if j <= i else mpmath.mpf(0) for j in range(n)] for i in range(n)]
        for j in range(n):
            dj = A[j][j]
            for i in range(j + 1, n):
                A[i][j] /= dj
            for i in range(j + 1, n):
                for k in range(j + 1, i + 1):
                    A[i][k] -= A[i][j] * dj * A[k][j]
    L = [[A[i][j] if j < i else mpmath.mpf(int(i == j)) for j in range(n)] for i in range(n)]
    return L, [A[j][j] for j in range(n)]


def product(L, D, dtype=np.longdouble):
    """Lower triangles of L D L^T and of |L| |D| |L|^T in `dtype`, summed tile by tile over the non-zero tiles of L."""
    n = len(D)
    nt = n_tiles(n)
    N = nt * T
    Lp = np.zeros((N, N), dtype)
    Lp[:n, :n] = L
    Dp = np.zeros(N, dtype)
    Dp[:n] = D
    W, Wa, La = Lp * Dp, np.abs(Lp) * np.abs(Dp), np.abs(Lp)
    nzt = tile_any(np.asarray(L, np.float64)) | np.eye(nt, dtype=bool)
    P = np.zeros((N, N), dtype)
    Q = np.zeros((N, N), dtype)
    t = lambda i: slice(T * i, T * i + T)   # noqa: E731
    for i in range(nt):
        for j in range(i + 1):
            for k in range(j + 1):
                if nzt[i, k] and nzt[j, k]:
                    P[t(i), t(j)] += W[t(i), t(k)] @ Lp[t(j), t(k)].T
                    Q[t(i), t(j)] += Wa[t(i), t(k)] @ La[t(j), t(k)].T
    return np.tril(P[:n, :n]), np.tril(Q[:n, :n])


def split(LD):
    """(L, D) of a device output: L strictly below the diagonal, 1 on it, zeros above; D the diagonal."""
    L = np.tril(LD, -1)
    np.fill_diagonal(L, 1.0)
    return L, LD.diagonal().copy()


# ---- generators -------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class Case:
    pattern: str
    values: str
    n6: int
    seed: int = 0

    @property
    def id(self):
        return f"{self.pattern}-{self.values}-{self.n6}"


def _block_band(n, w):
    b = np.arange(n) // 6
    return np.abs(b[:, None] - b[None, :]) <= w


def _expand(tiles, n):
    return np.kron(tiles, np.ones((T, T), bool))[:n, :n]


def pattern_mask(pattern, n6, rng):
    """(element mask of S, symmetric; tiles whose entries are all negative) of one pattern."""
    n = 6 * n6
    nt = n_tiles(n)
    I, K = np.meshgrid(np.arange(nt), np.arange(nt), indexing="ij")
    eye = I == K
    neg = []
    if pattern == "dense":
        m = np.ones((n, n), bool)
    elif pattern in ("band1", "band5", "band15"):           # block band of 1 / 5 keyframes (30 < 64 rows), 15 (90 > 64)
        m = _block_band(n, int(pattern[4:]))
    elif pattern == "arrow":                                 # dense last tile row: only the corner is updated
        m = _expand(eye | (I == nt - 1) | (K == nt - 1), n)
    elif pattern == "rarrow":                                # dense first tile column: everything else fills in
        m = _expand(eye | (K == 0) | (I == 0), n)
    elif pattern == "blockdiag":
        b = np.arange(n) // BLOCK
        m = b[:, None] == b[None, :]
    elif pattern == "randmask":
        r = np.tril(rng.random((nt, nt)) < 0.25, -1)
        m = _expand(eye | r | r.T, n)
    elif pattern == "single":                                # one entry at the last row and column of its tile
        m = _expand(eye, n)
        pts = []
        if nt >= 3:
            pts = [(2 * T - 1, T - 1), (n - 1, T * (nt - 2) + T - 1)]   # the second in the last valid row of the last tile
        elif nt == 2:
            pts = [(n - 1, T - 1)]
        for r, c in pts:
            m[r, c] = m[c, r] = True
    elif pattern == "negative":                              # one off-diagonal tile whose entries are all negative
        m = _expand(eye, n)
        if nt >= 2:
            ti, tk = nt - 1, max(0, nt - 3)
            m[T * ti:T * ti + T, T * tk:T * tk + T] = True
            m[T * tk:T * tk + T, T * ti:T * ti + T] = True
            neg = [(ti, tk)]
    else:
        raise ValueError(pattern)
    return m, neg


def values(mask, kind, rng, neg_tiles=()):
    """Symmetric S on mask.  dominant: off-diagonal entries uniform in (-1, 1), the diagonal one more than the row's
    absolute sum (strictly diagonally dominant SPD: growth <= 2, well conditioned); scaled: that, scaled on both sides by
    10^U(-3, 3), so that the diagonal spans 1e-6 .. 1e6 like the damped BA / PGO systems; quasi: dominant with random
    diagonal signs (quasi-definite, some D negative)."""
    n = len(mask)
    low = np.tril(mask, -1)
    off = np.where(low, rng.uniform(-1.0, 1.0, (n, n)), 0.0)
    for ti, tk in neg_tiles:
        blk = off[T * ti:T * ti + T, T * tk:T * tk + T]
        blk[...] = np.where(low[T * ti:T * ti + T, T * tk:T * tk + T], -rng.uniform(0.1, 1.0, blk.shape), 0.0)
    S = off + off.T
    d = np.abs(S).sum(axis=1) + rng.uniform(1.0, 2.0, n)
    if kind == "quasi":
        sgn = rng.choice([-1.0, 1.0], n)
        if n > 1:
            sgn[rng.permutation(n)[:2]] = (-1.0, 1.0)
        d *= sgn
    S[np.arange(n), np.arange(n)] = d
    if kind == "scaled":
        s = 10.0 ** rng.uniform(-3.0, 3.0, n)
        S = np.tril(s[:, None] * S * s[None, :])
        S = S + np.tril(S, -1).T                             # symmetric bit for bit
    elif kind not in ("dominant", "quasi"):
        raise ValueError(kind)
    return S


def make(case):
    """(S, g, record) of a Case: record = dict(case, tiles = the strictly lower tile pattern S is built to have)."""
    rng = np.random.default_rng([case.seed, case.n6, PATTERNS.index(case.pattern), VALUES.index(case.values)])
    m, neg = pattern_mask(case.pattern, case.n6, rng)
    S = values(m, case.values, rng, neg)
    g = rng.standard_normal(len(S))
    return S, g, dict(case=case, tiles=lower_tiles(np.where(m, 1.0, 0.0)), negative_tiles=neg)


def zero_pivot(S, j):
    """S with row and column j zero: D_j = 0 exactly, whatever came before it."""
    S = S.copy()
    S[j, :] = 0.0
    S[:, j] = 0.0
    return S


def plant(S, r, c, v):
    """S with S[r][c] = v only (r > c: lower, r == c: diagonal, r < c: strict upper)."""
    S = S.copy()
    S[r, c] = v
    return S


LOOP_SPAN = 256   # keyframes a loop block of band_plus_loops spans at most (see there)


def band_plus_loops(n6, n_loops, seed, max_span=LOOP_SPAN):
    """The pose graph's shape as scipy.sparse (CSR, both triangles): 6 x 6 blocks of neighbouring keyframes plus
    n_loops blocks between keyframes max_span / 2 .. max_span apart, strictly diagonally dominant SPD; and g.
    A loop fills its row from the older keyframe on, but the fill decays along the band by about 1e-0.46 per keyframe
    on these values, so a loop much longer than 256 keyframes fills with values that underflow to exact zeros in double
    and its tiles are (rightly) flagged zero: the tile pattern then depends on the values, not only on the structure."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    pairs = [(a + 1, a) for a in range(n6 - 1)]
    for _ in range(n_loops):
        a = int(rng.integers(0, n6 - max_span))
        pairs.append((a + int(rng.integers(max_span // 2, max_span + 1)), a))
    rows, cols, vals = [], [], []
    bi, bj = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
    for a, b in pairs:
        v = rng.uniform(-1.0, 1.0, 36)
        rows += [6 * a + bi.ravel(), 6 * b + bj.ravel()]
        cols += [6 * b + bj.ravel(), 6 * a + bi.ravel()]
        vals += [v, v]
    for a in range(n6):   # the diagonal blocks' off-diagonal entries
        v = rng.uniform(-1.0, 1.0, (6, 6))
        v = np.tril(v, -1) + np.tril(v, -1).T
        rows.append(6 * a + bi.ravel()); cols.append(6 * a + bj.ravel()); vals.append(v.ravel())
    n = 6 * n6
    S = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n)).tocsr()
    S.sum_duplicates()
    d = np.asarray(abs(S).sum(axis=1)).ravel() + rng.uniform(1.0, 2.0, n)
    S = (S + sp.diags(d)).tocsr()
    return S, rng.standard_normal(n)


def sparse_tiles(S):
    """lower_tiles of a scipy.sparse matrix."""
    C = S.tocoo()
    keep = (C.row > C.col) & (C.data != 0)
    nt = n_tiles(S.shape[0])
    P = np.zeros((nt, nt), bool)
    P[C.row[keep] // T, C.col[keep] // T] = True
    return np.tril(P, -1)


# ---- the sweep --------------------------------------------------------------------------------------------------------

def finite_cases():
    """Every finite case the device is run on: every pattern at the small sizes, the three value classes on three
    patterns there, one case per size of the residue sweep (patterns and value classes in turn), and the large sizes on
    the patterns whose fill stays sparse."""
    out = []
    for n6 in SIZES_SMALL:
        out += [Case(p, "dominant", n6) for p in PATTERNS]
        out += [Case(p, v, n6) for p in ("dense", "band5", "randmask") for v in ("scaled", "quasi")]
    for i, n6 in enumerate(SIZES_RESIDUE):
        c = Case(PATTERNS[i % len(PATTERNS)], VALUES[i % len(VALUES)], n6)
        if c not in out:
            out.append(c)
    out += [Case("blockdiag", "dominant", 200), Case("band15", "scaled", 200), Case("single", "quasi", 200),
            Case("blockdiag", "quasi", 266), Case("band5", "dominant", 266), Case("negative", "dominant", 266)]
    return out


def well_conditioned(case):
    return case.values in ("dominant", "quasi")


# ---- gba_update's block index -------------------------------------------------------------------------------------------

def update_pair(t):
    """gba_update's decode of its block index t (numpy int array) into the tile pair (a, b), 0 <= b <= a, restated:
    a = (int)((sqrt(8 t + 1) - 1) * 0.5) in double, each operation rounded (the library is built with --fmad=false), then
    the two correction loops in int."""
    t = np.asarray(t, np.int64)
    a = ((np.sqrt(8.0 * t.astype(np.float64) + 1.0) - 1.0) * 0.5).astype(np.int64)
    while True:
        up = (a + 1) * (a + 2) // 2 <= t
        if not up.any():
            break
        a = a + up
    while True:
        dn = a * (a + 1) // 2 > t
        if not dn.any():
            break
        a = a - dn
    return a, t - a * (a + 1) // 2
