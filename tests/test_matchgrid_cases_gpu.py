"""GPU tests of the windowed matcher's two device paths on tests/matchgrid_cases.py, bit for bit against its exact
reference: the single path (plf_match_grid_points / _lines, k_mg_columns) on every problem within its bounds, the batched
path (fe.debug_match_grid_batch, plf_launch_match_grid_batch) on every case within its 4 096-cell query mask with the
full and the clipped walk for lines, each problem of a batch against the same problem alone, and the hook's refusals."""
import ctypes as C
import functools
import time

import numpy as np
import pytest

import matchgrid_cases as mc

pytestmark = pytest.mark.gpu

CASES = mc.all_cases()
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)
_T0 = [None]


@pytest.fixture(scope="module", autouse=True)
def _wall():
    _T0[0] = time.perf_counter()
    yield
    print(f"\ntest_matchgrid_cases_gpu: {time.perf_counter() - _T0[0]:.1f} s over {len(CASES)} cases")


@functools.lru_cache(maxsize=None)
def _ref(name, p):
    return mc.reference(BY_NAME[name], p)


_RUNS = {}


def _batch(fe, case, clip):
    key = (case.name, clip)
    if key not in _RUNS:
        _RUNS[key] = fe.debug_match_grid_batch(case.q, case.t, case.d1, case.d2, case.n1, case.n2, case.cols, case.rows,
                                               case.w, case.nnr, t_dir=case.tdir, line_sim_th=case.th,
                                               best_lr=case.best_lr, clip=clip, q_slot=case.q_slot)
    return _RUNS[key]


def _check_batch(case, m, cnt, ref=None):
    assert m.shape == (case.P, case.K) and cnt.shape == (case.P,)
    for p in range(case.P):
        n1 = case.counts(p)[0]
        r = _ref(case.name, p) if ref is None else ref(p)
        bad = np.flatnonzero(m[p, :n1] != r["m12"])
        assert len(bad) == 0, (case.name, p, bad[:8], m[p, bad[:8]], r["m12"][bad[:8]])
        assert np.all(m[p, n1:] == -1), (case.name, p)
        assert cnt[p] == r["count"], (case.name, p, cnt[p], r["count"])


SINGLE = [(c.name, p) for c in CASES for p in range(c.P) if c.fits_single(p)]


@pytest.mark.parametrize("name,p", SINGLE, ids=[f"{n}-p{p}" for n, p in SINGLE])
def test_single_path_equals_the_reference(fe, name, p):
    c = BY_NAME[name]
    n1, n2 = c.counts(p)
    s = c.slot(p)
    cs, ci = mc.grid_csr(c, p)
    if c.lines:
        m, n = fe.match_grid_lines(c.q[p, :n1], c.d1[s, :n1], cs, ci, c.tdir[p, :n2], c.d2[p, :n2], c.cols, c.rows, c.w,
                                   c.nnr, c.th, c.best_lr)
    else:
        m, n = fe.match_grid_points(c.q[p, :n1], c.d1[s, :n1], cs, ci, c.d2[p, :n2], c.cols, c.rows, c.w, c.nnr,
                                    c.best_lr)
    r = _ref(name, p)
    bad = np.flatnonzero(m != r["m12"])
    assert len(bad) == 0 and n == r["count"], (bad[:8], n, r["count"])


# lines run with the full walk (clip 0) unless their end points are at the +-2^28 clamp, and with the clipped one
BATCH = [(c.name, clip) for c in CASES if c.fits_batch() for clip in ((0, 1) if c.lines else (0,)) if not (clip == 0 and c.far)]


@pytest.mark.parametrize("name,clip", BATCH, ids=[f"{n}-clip{k}" for n, k in BATCH])
def test_batched_path_equals_the_reference(fe, name, clip):
    c = BY_NAME[name]
    _check_batch(c, *_batch(fe, c, clip))


CLIPPED = [c.name for c in CASES if c.fits_batch() and c.lines and not c.far]


@pytest.mark.parametrize("name", CLIPPED)
def test_clipped_walk_equals_full_walk(fe, name):
    c = BY_NAME[name]
    (m0, n0), (m1, n1) = _batch(fe, c, 0), _batch(fe, c, 1)
    assert np.array_equal(m0, m1) and np.array_equal(n0, n1)


MULTI = [c.name for c in CASES if c.fits_batch() and c.P > 1]


@pytest.mark.parametrize("name", MULTI)
def test_each_problem_of_a_batch_equals_it_alone(fe, name):
    c = BY_NAME[name]
    for clip in (1, 0) if c.lines else (0,):
        m, cnt = _batch(fe, c, clip)
        for p in range(c.P):
            a = c.alone(p)
            ma, ca = fe.debug_match_grid_batch(a.q, a.t, a.d1, a.d2, a.n1, a.n2, a.cols, a.rows, a.w, a.nnr,
                                               t_dir=a.tdir, line_sim_th=a.th, best_lr=a.best_lr, clip=clip)
            assert np.array_equal(ma[0], m[p]) and ca[0] == cnt[p], (p, clip)


def test_refuses_bad_arguments_and_stays_usable(fe):
    """PLF_ERR_INVALID (-1) before any work, naming the hook, for each rule; then a valid call works."""
    import plslam_b200 as plf
    lib = fe.lib
    P, K, Kt = 2, 8, 8
    rng = np.random.default_rng(3)
    q = np.zeros((P, K, 4), np.int32)
    t = np.zeros((P, Kt, 4), np.int32)
    td = np.tile([1.0, 0.0], (P, Kt, 1))
    d1 = rng.integers(0, 256, (P, K, 32), dtype=np.uint8)
    d2 = rng.integers(0, 256, (P, Kt, 32), dtype=np.uint8)
    n1 = np.array([K, 3], np.int32)
    n2 = np.array([Kt, 2], np.int32)
    m = np.zeros((P, K), np.int32)
    cnt = np.zeros(P, np.int32)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))   # noqa: E731
    base = dict(P=P, K=K, Kt=Kt, q=ip(q), t=ip(t), td=td.ctypes.data_as(C.POINTER(C.c_double)),
                d1=d1.ctypes.data_as(C.POINTER(C.c_uint8)), d2=d2.ctypes.data_as(C.POINTER(C.c_uint8)), n1=ip(n1),
                n2=ip(n2), slot=None, cols=64, rows=48, lines=1, m=m.ctypes.data_as(C.POINTER(C.c_int32)), cnt=ip(cnt))

    def call(**kw):
        a = dict(base, **kw)
        return lib.plf_debug_match_grid_batch(fe._ctx, a["P"], a["K"], a["Kt"], a["q"], a["t"], a["td"], a["d1"], a["d2"],
                                              a["n1"], a["n2"], a["slot"], a["cols"], a["rows"],
                                              plf.plf_grid_window(1, 1, 1, 1), a["lines"], 1, 0.9, 0.75, 1, a["m"],
                                              a["cnt"])
    bad_slot = [np.array(v, np.int32) for v in ([0, 2], [-1, 0])]
    neg = [np.array(v, np.int32) for v in ([-1, 3], [3, -2])]
    refusals = [dict(P=-1), dict(P=65536), dict(K=-1), dict(K=65536), dict(Kt=-1), dict(Kt=8193), dict(cols=0),
                dict(rows=0), dict(cols=-64), *[dict(cols=a, rows=b) for a, b in mc.GRIDS_REFUSED],
                dict(slot=ip(bad_slot[0])), dict(slot=ip(bad_slot[1])), dict(n1=ip(neg[0])), dict(n2=ip(neg[1])),
                *[{k: None} for k in ("q", "t", "td", "d1", "d2", "n1", "n2", "m", "cnt")]]
    m[:] = 12345
    for kw in refusals:
        assert call(**kw) == -1, kw
        assert "plf_debug_match_grid_batch" in lib.plf_last_error(fe._ctx).decode(), kw
    assert np.all(m == 12345)   # nothing written
    assert call(td=None, lines=0) == 0                       # t_dir is read only for lines
    assert call(P=0) == 0
    assert call() == 0 and np.all(m[1, 3:] == -1)
    c = BY_NAME["ties-lr1"]
    _check_batch(c, *fe.debug_match_grid_batch(c.q, c.t, c.d1, c.d2, c.n1, c.n2, c.cols, c.rows, c.w, c.nnr))
