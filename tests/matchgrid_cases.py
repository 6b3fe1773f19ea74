"""Windowed matcher cases built to reach the edges of both device paths of stvo-pl's matchGrid (csrc/matchgrid.cu): query
and train counts at the 4-query and 128-thread edges of the launches, column minima that tie across query blocks, ratio
tests that tie in f32, direction gates exactly on line_sim_th, windows that are asymmetric, empty or cover the grid, the
grids at the batched path's 4 096-cell query mask, lines in every octant and pixel-unit lines far outside the grid; and
the exact reference they are checked against.

The reference is oracle/matchgrid.py's greedy matcher, vectorised with numpy in exact integer arithmetic so that it runs
at 65 535 x 8 192:
  distances   256-bit Hamming by np.bitwise_count on uint64 views;
  candidates  points: the train cell inside the grid and inside GridStructure::get's window of the query cell; lines: one
              of the train line's Bresenham cells inside the grid and inside the window of one of the query's Bresenham
              cells, then the direction gate |v . t_dir| < line_sim_th in f64 (a NaN v passes it);
  column pass with best_lr: a candidate counts for query i1 only when its distance is below every earlier query's
              distance to that train feature, an exclusive prefix minimum down each column, taken over query blocks
              that carry the column minima forward; m21 is the earliest query reaching the column's minimum;
  row pass    best and second best in ascending train order with strict '<' (so best_d2 is the second smallest of the
              multiset, INT_MAX with one candidate), the ratio test best_d < best_d2 * nnr on an f32 product;
  mutual pass i1 keeps its match only when m21[m12[i1]] == i1.
The Bresenham walk is evaluated in closed form, y_n = y1 + ystep * ceil((n dy - dx / 2) / dx) at step n, and only over
the steps whose window can reach the grid (a cell further than the window from the grid adds nothing), so query lines
with end points at +-2^28 cost what their part near the grid costs.

A Case is a batch of problems at uniform capacities as plf_debug_match_grid_batch takes it.  Every generator is seeded
and takes small=True for the reduced instances tests/test_matchgrid_cases.py compares with oracle/matchgrid.py, whose
pure-Python grid and walk cannot take the full sizes."""
from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp

INT_MAX = 2 ** 31 - 1
MASK_CELLS = 4096            # the batched path's query mask (MGB_MASK_WORDS * 32 bits)
K_MAX, KT_MAX = 65535, 8192  # plf_debug_match_grid_batch's capacities, those of the keyframe matcher
SINGLE_MAX_N, SINGLE_MAX_SIDE = 8192, 4096   # plf_match_grid_points / _lines
QCELL = 2 ** 28              # the clamp of the keyframe matcher's pixel-unit query end points (plf_qcell)
CHUNK_BYTES = 2 ** 31        # the launcher's scratch per chunk of problems
COLS, ROWS = 64, 48          # stvo-pl's GRID_COLS x GRID_ROWS
RATIOS = (0.75, 0.9)         # min_ratio_12_p / _l of every configuration of tests/param_cases.py


# ---- the reference ------------------------------------------------------------------------------------------------------

def hamming(d1, d2):
    """int32 [n1, n2] Hamming distances of 32-byte descriptors."""
    a = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32).view(np.uint64)
    b = np.ascontiguousarray(d2, np.uint8).reshape(-1, 32).view(np.uint64)
    out = np.zeros((len(a), len(b)), np.int32)
    for k in range(4):
        out += np.bitwise_count(a[:, None, k] ^ b[None, :, k])
    return out


def walk(x1, y1, x2, y2, reach=None):
    """(x, y) int64 arrays of the cells of the Bresenham walk (x1,y1)-(x2,y2) in oracle.matchgrid.bresenham's order.
    reach = (w, cols, rows): only the steps whose major coordinate lies within the window of the grid."""
    x1, y1, x2, y2 = int(x1), int(y1), int(x2), int(y2)
    steep = abs(y2 - y1) > abs(x2 - x1)
    if steep:
        x1, y1, x2, y2 = y1, x1, y2, x2
    if x1 > x2:
        x1, x2, y1, y2 = x2, x1, y2, y1
    dx, dy = x2 - x1, abs(y2 - y1)
    lo, hi = 0, dx
    if reach is not None:
        w, cols, rows = reach
        m_lo, m_hi = (-w[3], rows - 1 + w[2]) if steep else (-w[1], cols - 1 + w[0])
        lo, hi = max(0, m_lo - x1), min(dx, m_hi - x1)
    n = np.arange(lo, hi + 1, dtype=np.int64)
    ystep = 1 if y1 < y2 else -1
    y = y1 + ystep * -((dx // 2 - n * dy) // dx) if dx > 0 else np.full(len(n), y1, np.int64)
    xx = x1 + n
    return (y, xx) if steep else (xx, y)


def _window_cells(cx, cy, w, cols, rows):
    """Sorted unique cell ids x * rows + y of the union of get()'s windows around the cells (cx, cy)."""
    ox = np.arange(-w[0], w[1] + 1)
    oy = np.arange(-w[2], w[3] + 1)
    X = (cx[:, None, None] + ox[None, :, None]) + 0 * oy[None, None, :]
    Y = (cy[:, None, None] + oy[None, None, :]) + 0 * ox[None, :, None]
    keep = (X >= 0) & (X < cols) & (Y >= 0) & (Y < rows)
    return np.unique(X[keep] * rows + Y[keep])


def _csr(rows_of_ids, ncell):
    ptr = np.zeros(len(rows_of_ids) + 1, np.int64)
    ptr[1:] = np.cumsum([len(r) for r in rows_of_ids])
    idx = np.concatenate(rows_of_ids) if rows_of_ids else np.zeros(0, np.int64)
    return sp.csr_matrix((np.ones(len(idx), np.float32), idx, ptr), shape=(len(rows_of_ids), ncell))


def train_line_cells(t, cols, rows):
    """Per train line, the sorted cell ids of its Bresenham cells inside the grid (where GridStructure holds it)."""
    out = []
    for ln in np.asarray(t, np.int64).reshape(-1, 4):
        x, y = walk(*ln, reach=((0, 0, 0, 0), cols, rows))
        keep = (x >= 0) & (x < cols) & (y >= 0) & (y < rows)
        out.append(np.unique(x[keep] * rows + y[keep]))
    return out


def greedy(n1, n2, cand_block, d1, d2, nnr, best_lr, block=2048):
    """matchGrid on candidates cand_block(s, e) -> bool [e - s, n2]: dict(m12, count, m21, best_d, best_d2, best_idx)."""
    run = np.full(n2, INT_MAX, np.int32)
    m21 = np.full(n2, -1, np.int64)
    best = np.full(n1, INT_MAX, np.int64)
    best2 = np.full(n1, INT_MAX, np.int64)
    idx = np.full(n1, -1, np.int64)
    for s in range(0, n1, block):
        e = min(n1, s + block)
        D = np.where(cand_block(s, e), hamming(d1[s:e], d2[:n2]), INT_MAX).astype(np.int32).reshape(e - s, n2)
        if n2 == 0:
            continue
        if best_lr:
            prev = np.minimum.accumulate(np.vstack([run[None], D[:-1]]), axis=0)   # exclusive prefix minimum
            bmin = D.min(axis=0)
            up = bmin < run
            m21[up] = s + D[:, up].argmin(axis=0)
            run = np.minimum(run, bmin)
            D = np.where(D < prev, D, INT_MAX)
        best[s:e] = D.min(axis=1)
        idx[s:e] = np.where(best[s:e] < INT_MAX, D.argmin(axis=1), -1)
        if n2 > 1:
            best2[s:e] = np.partition(D, 1, axis=1)[:, 1]
    acc = best.astype(np.float32) < best2.astype(np.float32) * np.float32(nnr)
    m12 = np.where(acc, idx, -1).astype(np.int32)
    count = int(acc.sum())
    if best_lr and n2 > 0:
        drop = (m12 >= 0) & (m21[np.maximum(m12, 0)] != np.arange(n1))
        m12[drop] = -1
        count -= int(drop.sum())
    return dict(m12=m12, count=count, m21=m21, best_d=best, best_d2=best2, best_idx=idx)


def line_dirs(q):
    """The normalised query directions in f64, as the device and the reference's normalize() compute them (NaN for a
    zero-length query)."""
    q = np.asarray(q, np.int64).reshape(-1, 4)
    vx, vy = (q[:, 2] - q[:, 0]).astype(np.float64), (q[:, 3] - q[:, 1]).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        nrm = np.sqrt(vx * vx + vy * vy)
        return vx / nrm, vy / nrm


def candidates(case, p):
    """(n1, n2, cand_block) of problem p."""
    n1, n2 = case.counts(p)
    q, t = case.q[p, :n1].astype(np.int64), case.t[p, :n2].astype(np.int64)
    w, cols, rows = case.w, case.cols, case.rows
    if not case.lines:
        t_in = (t[:, 0] >= 0) & (t[:, 0] < cols) & (t[:, 1] >= 0) & (t[:, 1] < rows)

        def cand(s, e):
            ddx = t[None, :, 0] - q[s:e, 0, None]
            ddy = t[None, :, 1] - q[s:e, 1, None]
            return t_in[None, :] & (ddx >= -w[0]) & (ddx <= w[1]) & (ddy >= -w[2]) & (ddy <= w[3])
        return n1, n2, cand
    ncell = cols * rows
    Tt = _csr(train_line_cells(t, cols, rows), ncell).T.tocsr()
    qc = [_window_cells(*walk(*ln, reach=(w, cols, rows)), w, cols, rows) for ln in q]
    Mq = _csr(qc, ncell)
    vx, vy = line_dirs(q)
    td = case.tdir[p, :n2]

    def cand(s, e):
        C = (Mq[s:e] @ Tt).toarray() > 0
        with np.errstate(invalid="ignore"):
            cosv = np.abs(vx[s:e, None] * td[None, :, 0] + vy[s:e, None] * td[None, :, 1])
            return C & ~(cosv < case.th)
    return n1, n2, cand


def reference(case, p):
    """The reference's result of problem p (see greedy)."""
    n1, n2, cand = candidates(case, p)
    s = case.slot(p)
    return greedy(n1, n2, cand, case.d1[s, :n1], case.d2[p, :n2], case.nnr, case.best_lr)


def grid_csr(case, p):
    """(cell_start, cell_items) of problem p's train features, the GridStructure the single path takes."""
    n1, n2 = case.counts(p)
    t = case.t[p, :n2].astype(np.int64)
    cols, rows = case.cols, case.rows
    if case.lines:
        per = train_line_cells(t, cols, rows)
    else:
        t_in = (t[:, 0] >= 0) & (t[:, 0] < cols) & (t[:, 1] >= 0) & (t[:, 1] < rows)
        per = [np.array([x * rows + y]) if k else np.zeros(0, np.int64) for (x, y), k in zip(t, t_in)]
    ids = np.concatenate(per) if per else np.zeros(0, np.int64)
    items = np.repeat(np.arange(len(per)), [len(c) for c in per])
    order = np.argsort(ids, kind="stable")
    start = np.zeros(cols * rows + 1, np.int32)
    start[1:] = np.cumsum(np.bincount(ids, minlength=cols * rows))
    return start, items[order].astype(np.int32)


def oracle_grid(case, p):
    """oracle.matchgrid's Grid over problem p's train features."""
    from oracle import matchgrid as mg
    n2 = case.counts(p)[1]
    f = mg.grid_from_lines if case.lines else mg.grid_from_points
    return f(case.t[p, :n2], case.rows, case.cols)


def chunks(case):
    """The number of chunks plf_launch_match_grid_batch splits the case's problems into (2 GB of scratch each)."""
    K, Kt = case.K, case.Kt
    al = lambda b: (b + 255) // 256 * 256   # noqa: E731
    per = al(2 * K * Kt) + al(4 * K * 128 if case.lines else 0) + al(4 * Kt)
    chunk = max(1, min(case.P, CHUNK_BYTES // per))
    return -(-case.P // chunk)


# ---- cases --------------------------------------------------------------------------------------------------------------

@dataclass(eq=False)
class Case:
    name: str
    lines: bool
    cols: int
    rows: int
    w: tuple
    nnr: float
    q: np.ndarray              # int32 [P, K, 2|4]
    t: np.ndarray              # int32 [P, Kt, 2|4]
    d1: np.ndarray             # uint8 [P, K, 32]
    d2: np.ndarray             # uint8 [P, Kt, 32]
    n1: np.ndarray             # int32 [P], may exceed K
    n2: np.ndarray             # int32 [P], may exceed Kt
    tdir: np.ndarray = None    # float64 [P, Kt, 2] (lines)
    th: float = 0.75
    best_lr: bool = True
    q_slot: np.ndarray = None  # int32 [P] or None
    far: bool = False          # query end points so far out that only the clipped walk may run them

    @property
    def P(self):
        return self.q.shape[0]

    @property
    def K(self):
        return self.q.shape[1]

    @property
    def Kt(self):
        return self.t.shape[1]

    def slot(self, p):
        return p if self.q_slot is None else int(self.q_slot[p])

    def counts(self, p):
        """The live query and train counts of problem p, clamped to the capacities."""
        return min(int(self.n1[self.slot(p)]), self.K), min(int(self.n2[p]), self.Kt)

    def fits_batch(self):
        return self.cols * self.rows <= MASK_CELLS

    def fits_single(self, p):
        n1, n2 = self.counts(p)
        return not self.far and max(n1, n2) <= SINGLE_MAX_N and max(self.cols, self.rows) <= SINGLE_MAX_SIDE

    def alone(self, p):
        """Problem p as a batch of its own."""
        s = self.slot(p)
        pick = lambda a, i: None if a is None else a[i:i + 1]   # noqa: E731
        return Case(f"{self.name}-p{p}", self.lines, self.cols, self.rows, self.w, self.nnr, self.q[p:p + 1],
                    self.t[p:p + 1], self.d1[s:s + 1], self.d2[p:p + 1], self.n1[s:s + 1], self.n2[p:p + 1],
                    pick(self.tdir, p), self.th, self.best_lr, None, self.far)


def _rng(name, seed=0):
    return np.random.default_rng([seed, *name.encode()])


def descs(rng, n, protos=None, flip=0.06):
    """n descriptors: uniform, or prototypes with each bit flipped with probability `flip` (near-duplicates and ties)."""
    if protos is None:
        return rng.integers(0, 256, (n, 32), dtype=np.uint8)
    bits = rng.random((n, 256)) < flip
    return (protos[rng.integers(0, len(protos), n)] ^ np.packbits(bits, axis=1)).astype(np.uint8)


def flip_bits(rng, d, k):
    """d with exactly k of its 256 bits flipped: at Hamming distance k from d."""
    bits = np.zeros(256, bool)
    bits[rng.choice(256, k, replace=False)] = True
    return d ^ np.packbits(bits)


def unit_dirs(t):
    """Unit directions of train lines [n, 4]; (1, 0) for a zero-length one."""
    v = (t[:, 2:] - t[:, :2]).astype(np.float64)
    nrm = np.linalg.norm(v, axis=1, keepdims=True)
    return np.where(nrm > 0, v / np.maximum(nrm, 1e-300), np.array([[1.0, 0.0]]))


def batch(name, lines, cols, rows, w, nnr, probs, K=None, Kt=None, n1=None, n2=None, **kw):
    """A Case from problems given as dicts (q, t, d1, d2[, tdir]) of any sizes, padded to capacities K / Kt (default: the
    largest), with counts n1 / n2 (default: the sizes)."""
    g = 4 if lines else 2
    K = max([len(p["q"]) for p in probs] + [0]) if K is None else K
    Kt = max([len(p["t"]) for p in probs] + [0]) if Kt is None else Kt
    P = len(probs)
    rng = _rng(name, 99)
    q = np.full((P, K, g), -7, np.int32)     # padding past the counts: geometry and descriptors the kernels never read
    t = np.full((P, Kt, g), -7, np.int32)
    d1 = rng.integers(0, 256, (P, K, 32), dtype=np.uint8)
    d2 = rng.integers(0, 256, (P, Kt, 32), dtype=np.uint8)
    td = np.zeros((P, Kt, 2)) if lines else None
    for i, pr in enumerate(probs):
        a, b = len(pr["q"]), len(pr["t"])
        q[i, :a], d1[i, :a], t[i, :b], d2[i, :b] = pr["q"], pr["d1"], pr["t"], pr["d2"]
        if lines:
            td[i, :b] = pr["tdir"] if "tdir" in pr else unit_dirs(np.asarray(pr["t"]))
    n1 = np.array([len(p["q"]) for p in probs] if n1 is None else n1, np.int32)
    n2 = np.array([len(p["t"]) for p in probs] if n2 is None else n2, np.int32)
    return Case(name, lines, cols, rows, tuple(w), float(nnr), q, t, d1, d2, n1, n2, td, **kw)


def random_points(rng, n1, n2, cols=COLS, rows=ROWS, protos=60, margin=2):
    pr = rng.integers(0, 256, (protos, 32), dtype=np.uint8)
    q = np.stack([rng.integers(-margin, cols + margin, n1), rng.integers(-margin, rows + margin, n1)], 1)
    t = np.stack([rng.integers(-1, cols + 1, n2), rng.integers(-1, rows + 1, n2)], 1)
    return dict(q=q, t=t, d1=descs(rng, n1, pr), d2=descs(rng, n2, pr))


def random_lines(rng, n1, n2, cols=COLS, rows=ROWS, span=(9, 9), protos=50, margin=2):
    pr = rng.integers(0, 256, (protos, 32), dtype=np.uint8)

    def lines(n):
        a = np.stack([rng.integers(-margin, cols + margin, n), rng.integers(-margin, rows + margin, n)], 1)
        return np.concatenate([a, a + np.stack([rng.integers(-s, s + 1, n) for s in span], 1)], 1)
    q, t = lines(n1), lines(n2)
    return dict(q=q, t=t, d1=descs(rng, n1, pr), d2=descs(rng, n2, pr))


N1 = (0, 1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 255, 256, 257, 8192)
N2 = (0, 1, 127, 128, 129, 8192)


def sizes(small=False):
    """Points at every query count of N1 (against 129 train points; 8192 against 8192) and every train count of N2
    (against 257 queries); lines at the counts up to 257.  Windows 1 and 2; best_lr on and off."""
    cap = (lambda n: min(n, 160)) if small else (lambda n: n)
    out = []
    for n1 in N1:
        rng = _rng(f"size-p-{n1}")
        n2 = 8192 if n1 == 8192 else 129
        out.append(batch(f"points-n1_{n1}", False, COLS, ROWS, (1, 1, 1, 1), 0.9, [random_points(rng, cap(n1), cap(n2))],
                         best_lr=n1 % 2 == 1 or n1 == 8192))
    for n2 in N2:
        rng = _rng(f"size-p2-{n2}")
        out.append(batch(f"points-n2_{n2}", False, COLS, ROWS, (2, 2, 2, 2), 0.9, [random_points(rng, cap(257), cap(n2))],
                         best_lr=n2 != 127))
    for n1 in N1[:-1]:
        rng = _rng(f"size-l-{n1}")
        n2 = (1, 128, 129)[n1 % 3]
        out.append(batch(f"lines-n1_{n1}", True, COLS, ROWS, (1, 1, 1, 1), 0.9, [random_lines(rng, cap(n1), cap(n2))],
                         best_lr=n1 != 33))
    for n2 in (0, 127, 128):
        rng = _rng(f"size-l2-{n2}")
        out.append(batch(f"lines-n2_{n2}", True, COLS, ROWS, (1, 1, 1, 1), 0.9, [random_lines(rng, cap(200), cap(n2))]))
    return out


TIE_PAIRS = ((127, 128), (255, 256))   # queries with identical descriptors across the 128- and 256-query boundaries


def ties(small=False):
    """300 queries in cell (5, 5) and every third one in an empty corner (non-candidates interleaved), against 64 train
    points around it: queries 127 / 128 and 255 / 256 are identical and each pair is at distance 0 from one train point, so
    its column minimum ties between the two and the earlier query must keep it; two identical train points give one
    query equal best and second best; a lone pair (query, complement) has distance 256."""
    out = []
    for best_lr in (True, False):
        rng = _rng("ties", best_lr)
        n1, n2 = 300, 64
        t = np.stack([rng.integers(4, 7, n2), rng.integers(4, 7, n2)], 1)
        d2 = descs(rng, n2)
        d2[21] = d2[20]
        q = np.tile([5, 5], (n1, 1))
        q[2::3] = (60, 45)
        d1 = np.stack([flip_bits(rng, d2[i % n2], int(rng.integers(8, 40))) for i in range(n1)])
        for (a, b), j in zip(TIE_PAIRS, (3, 7)):
            q[[a, b]] = (5, 5)
            d1[a] = d1[b] = d2[j]
        d1[10] = flip_bits(rng, d2[20], 12)                   # equal best and second best (train 20 and 21)
        t = np.concatenate([t, [[30, 30]]])                    # a lone train point ...
        d2 = np.concatenate([d2, [~d2[0]]])
        q[1] = (30, 30)                                        # ... whose only query is its complement: distance 256
        d1[1] = d2[0]
        out.append(batch(f"ties-lr{int(best_lr)}", False, COLS, ROWS, (1, 1, 1, 1), 0.9,
                         [dict(q=q, t=t, d1=d1, d2=d2)], best_lr=best_lr))
    return out


def f32_ties(b, b2, nnr):
    """Whether the f32 product of the ratio test rounds to best_d exactly."""
    return np.float32(b2) * np.float32(nnr) == np.float32(b)


def ratio_pairs(nnr, limit=256):
    """(best_d, best_d2) pairs with f32(best_d2 * nnr) == best_d, best_d2 <= 256."""
    out = []
    for b2 in range(1, limit + 1):
        b = int(np.rint(np.float32(b2) * np.float32(nnr)))
        if 0 <= b <= 256 and f32_ties(b, b2, nnr):
            out.append((b, b2))
    return out


def _pair_problem(rng, pairs, single=4):
    """Query i alone in its cell (window 0) with two train points at distances pairs[i] (the farther one first for odd
    i), then `single` queries with one train point each."""
    q, t, d1, d2 = [], [], [], []
    for i, (b, b2) in enumerate(pairs + [(int(rng.integers(0, 257)), None)] * single):
        cell = (i % COLS, i // COLS)
        x = descs(rng, 1)[0]
        q.append(cell)
        d1.append(x)
        near = [flip_bits(rng, x, b)] + ([] if b2 is None else [flip_bits(rng, x, b2)])
        for d in (near[::-1] if i % 2 else near):
            t.append(cell)
            d2.append(d)
    return dict(q=np.array(q), t=np.array(t), d1=np.array(d1), d2=np.array(d2))


def ratio_pins(small=False):
    """The ratio test at nnr where f32(best_d2 * nnr) == best_d (rejected by the strict '<'), one f32 ulp either side, at
    nnr = 1 with equal best and second best (one ulp above accepts the earlier train point), at the configurations'
    ratios; and single candidates (best_d2 = INT_MAX)."""
    out = []
    base = [np.float32(0.9), np.float32(0.75), np.float32(0.8), np.float32(1.0)]
    for k, nnr0 in enumerate(base):
        for side, nnr in (("at", nnr0), ("below", np.nextafter(nnr0, np.float32(0))),
                          ("above", np.nextafter(nnr0, np.float32(2)))):
            rng = _rng(f"ratio-{k}-{side}")
            pairs = ratio_pairs(nnr0)
            pairs = [pp for pp in pairs if pp[0] != pp[1]] if nnr0 != 1 else [(b, b) for b in range(0, 257, 4)]
            pairs = pairs[:40] if small else pairs
            pairs += [(b, b2) for b, b2 in zip(rng.integers(0, 200, 30), rng.integers(0, 257, 30))]
            out.append(batch(f"ratio-{float(nnr0):g}-{side}", False, COLS, ROWS, (0, 0, 0, 0), float(nnr),
                             [_pair_problem(rng, [(int(b), int(b2)) for b, b2 in pairs])]))
    for nnr in RATIOS:
        rng = _rng(f"ratio-cfg-{nnr}")
        n = 150 if small else 600
        out.append(batch(f"ratio-config-{nnr}", False, COLS, ROWS, (1, 1, 1, 1), nnr, [random_points(rng, n, n)]))
        out.append(batch(f"ratio-config-lines-{nnr}", True, COLS, ROWS, (1, 1, 1, 1), nnr,
                         [random_lines(rng, n // 2, n // 2)]))
    return out


WINDOWS = {"w0": (0, 0, 0, 0), "w1": (1, 1, 1, 1), "w2": (2, 2, 2, 2), "w3": (3, 3, 3, 3), "stereo": (10, 0, 0, 0),
           "stereo3": (3, 0, 0, 0), "asym": (1, 3, 0, 2), "asym2": (2, 0, 3, 1), "whole": (COLS, COLS, ROWS, ROWS)}


def windows(small=False):
    """Points (and lines, but for the whole-grid window) at every window of WINDOWS, with queries up to 4 cells outside
    the grid, train points outside it and train points on its last row and column."""
    out = []
    n1, n2 = (150, 120) if small else (500, 400)
    for name, w in WINDOWS.items():
        rng = _rng(f"win-{name}")
        pr = random_points(rng, n1, n2, margin=4)
        pr["t"][:40] = np.stack([np.full(40, COLS - 1), rng.integers(0, ROWS, 40)], 1)
        pr["t"][40:80] = np.stack([rng.integers(0, COLS, 40), np.full(40, ROWS - 1)], 1)
        pr["t"][80:90] = [(-1, 3), (COLS, 4), (5, -1), (6, ROWS), (-1, -1), (COLS, ROWS), (COLS - 1, ROWS - 1),
                          (0, 0), (COLS - 1, 0), (0, ROWS - 1)]
        out.append(batch(f"window-points-{name}", False, COLS, ROWS, w, 0.9, [pr], best_lr=name != "w2"))
        if name != "whole":
            rng = _rng(f"winl-{name}")
            pl = random_lines(rng, n1 // 2, n2 // 2, margin=5)
            pl["t"][:20] = np.array([(COLS - 1, y, COLS - 1, y + 3) for y in rng.integers(0, ROWS - 3, 20)])
            pl["t"][20:40] = np.array([(x, ROWS - 1, x + 4, ROWS - 1) for x in rng.integers(0, COLS - 4, 20)])
            out.append(batch(f"window-lines-{name}", True, COLS, ROWS, w, 0.9, [pl]))
    return out


GRIDS_BOTH = ((64, 48), (64, 64), (4096, 1), (1, 4096))
GRIDS_SINGLE = ((640, 480), (4096, 4096))
GRIDS_REFUSED = ((4097, 1), (1, 4097), (241, 17), (65, 64))   # one cell or more over the query mask


def grids(small=False):
    """Points and lines on the grids at the batched path's 4 096-cell mask, and larger grids for the single path."""
    out = []
    for cols, rows in GRIDS_BOTH + GRIDS_SINGLE:
        if small and cols * rows > MASK_CELLS * 64:
            cols, rows = 512, 512
        rng = _rng(f"grid-{cols}x{rows}")
        n = 120 if small else 400
        span = (max(cols // 8, 2), max(rows // 8, 2))
        w = (2, 1, 0, 1) if min(cols, rows) == 1 else (1, 1, 1, 1)
        pp = random_points(rng, n, n, cols, rows)
        pp["t"][:10] = np.stack([np.full(10, cols - 1), rng.integers(0, rows, 10)], 1)
        pp["t"][10:20] = np.stack([rng.integers(0, cols, 10), np.full(10, rows - 1)], 1)
        pp["q"][:20] = pp["t"][:20]
        out.append(batch(f"grid-points-{cols}x{rows}", False, cols, rows, w, 0.9, [pp]))
        nl = 60 if small else 200
        pl = random_lines(rng, nl, nl, cols, rows, span=span)
        out.append(batch(f"grid-lines-{cols}x{rows}", True, cols, rows, w, 0.9, [pl]))
    return out


def _octant_lines(c, r):
    """Lines from (c, c) to 16 directions (every octant, steep and shallow, the diagonals) at length r, each also with
    its end points reversed; horizontal, vertical and single-cell lines."""
    out = []
    for ax, ay in ((r, 0), (r, r // 3), (r, r), (r // 3, r), (0, r), (-r // 3, r), (-r, r), (-r, r // 3), (-r, 0),
                   (-r, -r // 3), (-r, -r), (-r // 3, -r), (0, -r), (r // 3, -r), (r, -r), (r, -r // 3)):
        out += [(c, c, c + ax, c + ay), (c + ax, c + ay, c, c)]
    return out + [(c, c, c, c), (c + 1, c - 2, c + 1, c - 2)]


def line_geometry(small=False):
    """Query lines in every octant (both end-point orders), horizontal, vertical and single-cell ones, lines entering and
    leaving the grid, against train lines of the same shapes shifted by a cell; and the direction gate exactly on
    line_sim_th: horizontal queries (v = (1, 0) exactly) against train directions (th, .), (-th, .) (kept) and
    (th - 1 ulp, .) (dropped), a zero-length query (NaN v, kept), and a slanted query whose th is its own |v . t_dir|."""
    out = []
    rng = _rng("octants")
    q = np.array(_octant_lines(20, 9) + _octant_lines(24, 4) + [(-6, 10, 8, 12), (50, 40, 75, 52), (30, -5, 33, 60),
                                                                 (-3, -3, 70, 55), (60, 47, 70, 47), (63, 0, 63, 60)])
    t = np.concatenate([q + [1, 0, 1, 0], q[::-1] + [0, 1, 0, 1]])
    pr = rng.integers(0, 256, (len(q), 32), dtype=np.uint8)
    d1 = np.stack([flip_bits(rng, pr[i], 10) for i in range(len(q))])
    d2 = np.concatenate([np.stack([flip_bits(rng, pr[i], 20) for i in range(len(q))]),
                         np.stack([flip_bits(rng, pr[i], 30) for i in range(len(q))[::-1]])])
    for w in ((0, 0, 0, 0), (1, 2, 0, 1)):
        out.append(batch(f"lines-octants-{''.join(map(str, w))}", True, COLS, ROWS, w, 0.9,
                         [dict(q=q, t=t, d1=d1, d2=d2)], th=0.0))
    th = float(np.float32(0.75))
    lo = np.nextafter(th, 0.0)
    qs, ts, tds, dq, dt = [], [], [], [], []
    for i, c in enumerate((th, -th, lo, -lo, th, 1.0, 0.0)):
        y = 2 + 3 * i
        qs.append((10, y, 16, y) if i != 4 else (12, y, 12, y))   # i = 4: zero length
        ts.append((11, y, 15, y + 1))
        tds.append((c, np.sqrt(1.0 - c * c)))
        x = descs(rng, 1)[0]
        dq.append(x)
        dt.append(flip_bits(rng, x, 5))
    out.append(batch("lines-gate-exact", True, COLS, ROWS, (0, 0, 0, 0), 0.9,
                     [dict(q=np.array(qs), t=np.array(ts), d1=np.array(dq), d2=np.array(dt), tdir=np.array(tds))], th=th))
    vx, vy = line_dirs([(0, 0, 3, 7)])
    tdir = np.array([[0.28, 0.96]])
    th2 = float(np.abs(vx * tdir[:, 0] + vy * tdir[:, 1])[0])
    x = descs(rng, 1)[0]
    for name, th_ in (("at", th2), ("above", np.nextafter(th2, 2.0))):
        out.append(batch(f"lines-gate-slanted-{name}", True, COLS, ROWS, (0, 0, 0, 0), 0.9,
                         [dict(q=np.array([(10, 10, 13, 17)]), t=np.array([(11, 11, 13, 16)]), d1=x[None],
                               d2=flip_bits(rng, x, 3)[None], tdir=tdir)], th=th_))
    return out


def pixel_lines(small=False):
    """Query lines with end points far outside the grid, as the keyframe matcher's pixel-unit projections: up to the
    +-2^28 clamp (clipped walk only; +-2^12 in the small instances), and up to +-4096 cells, which the full walk can
    still take.  Each crosses or passes the grid in some direction; the train lines lie inside it."""
    out = []
    for far, R in ((True, 4096 if small else QCELL), (False, 4096)):
        rng = _rng(f"pixel-{far}")
        n = 40 if small else 160
        cx, cy = rng.integers(-4, COLS + 4, n), rng.integers(-4, ROWS + 4, n)
        ang = rng.uniform(0, 2 * np.pi, n)
        a = np.round(np.stack([cx + R * np.cos(ang), cy + R * np.sin(ang)], 1)).astype(np.int64)
        b = np.round(np.stack([cx - R * np.cos(ang) * rng.uniform(0, 1, n), cy - R * np.sin(ang) * rng.uniform(0, 1, n)],
                              1)).astype(np.int64)
        q = np.clip(np.concatenate([a, b], 1), -R, R)
        q[:4] = [(-R, 10, R, 12), (20, -R, 22, R), (-R, -R, R, R), (-R, R, -R + 5, R)]   # the last never near the grid
        t = np.concatenate([np.stack([cx, cy], 1), np.stack([cx, cy], 1) + rng.integers(-3, 4, (n, 2))], 1)
        t = np.clip(t, 0, [COLS - 1, ROWS - 1, COLS - 1, ROWS - 1])
        pr = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        d1 = np.stack([flip_bits(rng, pr[i], 8) for i in range(n)])
        d2 = np.stack([flip_bits(rng, pr[i], 16) for i in range(n)])
        for w in ((0, 0, 0, 0), (3, 3, 3, 3), (1, 2, 3, 0)):
            out.append(batch(f"lines-pixel-{'far' if far else 'near'}-{''.join(map(str, w))}", True, COLS, ROWS, w,
                             0.9, [dict(q=q, t=t, d1=d1, d2=d2)], th=0.0, far=far and not small))
    return out


def batches(small=False):
    """Mixed sizes in one batch, counts above the capacities (clamped), several problems reading one query slot, and
    the same problems in a permuted order; points and lines."""
    out = []
    for lines in (False, True):
        rng = _rng(f"batch-{lines}")
        sz = [(0, 40), (5, 1), (300, 129), (129, 300), (1000, 700), (33, 0)]
        if small:
            sz = [(min(a, 120), min(b, 120)) for a, b in sz]
        gen = random_lines if lines else random_points
        probs = [gen(rng, a, b) for a, b in sz]
        kind = "lines" if lines else "points"
        out.append(batch(f"batch-{kind}-mixed", lines, COLS, ROWS, (2, 1, 1, 2), 0.9, probs))
        K, Kt = max(a for a, _ in sz), max(b for _, b in sz)
        n1 = [a for a, _ in sz]
        n2 = [b for _, b in sz]
        big = int(np.argmax(n1))
        n1[big] += 7                                         # counts above the capacities: clamped to K / Kt
        n2[int(np.argmax(n2))] += 3
        out.append(batch(f"batch-{kind}-over", lines, COLS, ROWS, (1, 1, 1, 1), 0.9, probs, K, Kt, n1, n2))
        slot = np.array([2, 2, 0, 4, 2, 2], np.int32)       # problem p reads the queries of slot q_slot[p]
        c = batch(f"batch-{kind}-slots", lines, COLS, ROWS, (1, 1, 1, 1), 0.9, probs, q_slot=slot)
        for p in range(c.P):                                 # query geometry stays per problem: give it the slot's count
            s = slot[p]
            c.q[p] = c.q[s]
            c.q[p, :, :2] += p % 2                           # ... shifted, so that the problems differ
        out.append(c)
        perm = rng.permutation(len(probs))
        out.append(batch(f"batch-{kind}-permuted", lines, COLS, ROWS, (2, 1, 1, 2), 0.9, [probs[i] for i in perm]))
    return out


def huge(small=False):
    """Three problems at the keyframe matcher's capacities, 65 535 queries by 8 192 train points: problem 0 has every
    query and train point live (the whole 1 GB distance matrix), 1 and 2 a few hundred.  One problem per 2 GB chunk."""
    K, Kt = (600, 200) if small else (K_MAX, KT_MAX)
    rng = _rng("huge")
    probs = [random_points(rng, K, Kt, protos=400), random_points(rng, 300, 150), random_points(rng, 257, 129)]
    return [batch("huge-65535x8192", False, COLS, ROWS, (1, 1, 1, 1), 0.9, probs, K, Kt)]


GENERATORS = {"sizes": sizes, "ties": ties, "ratio_pins": ratio_pins, "windows": windows, "grids": grids,
              "line_geometry": line_geometry, "pixel_lines": pixel_lines, "batches": batches, "huge": huge}


def all_cases(small=False):
    return [c for g in GENERATORS.values() for c in g(small)]
