"""GPU tests of plf_pose_graph_batch: every problem of a batch gets, bit for bit, what plf_pose_graph gives it alone
(poses, scalars and trace rows), whatever its neighbours and their order; the batch agrees with oracle/pgo.py as the
single call does; refusals write nothing and leave the context usable; the launches are the header's count.  The
batches are the ones tests/test_pgo_batch.py checks on the oracle."""
import ctypes as C

import numpy as np
import pytest

import plslam_b200 as plf
from oracle import pgo
from oracle import synth as osynth
from plslam_b200 import synth
from test_pgo_batch import (FIRST_ITERS, documented_launches, edgeless_graph, graph, identity_graph, isolated_graph,
                            mixed_batch, overflow_graph)
from test_pgo_gpu import CASES, _compare, _final

pytestmark = pytest.mark.gpu
PLF_ERR_INVALID, PLF_ERR_CUDA, PLF_ERR_CAPACITY = -1, -3, -4
SCALARS = ("iters", "stop", "trials", "chi2_init", "chi2", "lambda_")


def bits(x):
    return np.asarray(x).tobytes()


def assert_same(got, want):
    """bit-identical poses, scalars and trace rows"""
    assert bits(got["T"]) == bits(want["T"])
    for k in SCALARS:
        assert bits(got[k]) == bits(want[k]), k
    assert bits(got.get("trace", [])) == bits(want.get("trace", []))


def run(fe, probs, **kw):
    """pose_graph_batch, with its launches checked against plslam_b200.h's count"""
    n0 = fe.launches
    got = fe.pose_graph_batch(probs, **kw)
    if kw.get("trace", True):
        assert fe.launches - n0 == documented_launches(probs, got)
    return got


def singles(fe, probs, **kw):
    return [fe.pose_graph(p, **kw) for p in probs]


def test_mixed_batch_is_each_single_call_bit_for_bit(fe):
    probs = [graph(n, w, l) for n, w, l in CASES] + mixed_batch()
    for g, w in zip(run(fe, probs), singles(fe, probs)):
        assert_same(g, w)


@pytest.mark.parametrize("order", ["reversed", "shuffled"])
def test_order_does_not_matter(fe, order):
    probs = mixed_batch()
    idx = list(range(len(probs)))[::-1] if order == "reversed" else list(np.random.default_rng(5).permutation(len(probs)))
    want = singles(fe, probs)
    got = run(fe, [probs[k] for k in idx])
    for g, k in zip(got, idx):
        assert_same(g, want[k])


def test_each_problem_alone_first_last_and_between_two_large_ones(fe):
    probs = mixed_batch()
    big = graph(684, 1, 1)
    for k, p in enumerate(probs):
        want = fe.pose_graph(p)
        others = probs[:k] + probs[k + 1:]
        assert_same(run(fe, [p])[0], want)
        assert_same(run(fe, [p] + others[:3])[0], want)
        assert_same(run(fe, others[-3:] + [p])[-1], want)
        assert_same(run(fe, [big, p, big])[1], want)


def test_sixteen_copies_launch_what_one_launches(fe):
    p = graph(101, 5, 1)
    n0 = fe.launches
    want = fe.pose_graph(p)
    one = fe.launches - n0
    n0 = fe.launches
    got = fe.pose_graph_batch([p] * 16)
    assert fe.launches - n0 == one == documented_launches([p], [want])
    for g in got:
        assert_same(g, want)


def test_a_batch_launches_no_more_than_its_longest_problem_plus_its_linearisations(fe):
    """the longest-running problem is also the largest here, so the others' rounds add only their linearisations"""
    big = graph(684, 5, 4)
    top = fe.pose_graph(big)["trials"]
    small = [graph(*c) for c in CASES if c[0] < 684]
    probs = [big] + [p for p, w in zip(small, singles(fe, small)) if w["trials"] < top]
    assert len(probs) >= 4
    want = singles(fe, probs)
    n0 = fe.launches
    fe.pose_graph(probs[0])
    alone = fe.launches - n0
    got = run(fe, probs)
    assert documented_launches(probs, got) <= alone + want[0]["trials"]
    for g, w in zip(got, want):
        assert_same(g, w)


@pytest.mark.parametrize("max_iters", [0, 1, FIRST_ITERS, 100])
def test_max_iters(fe, max_iters):
    probs = mixed_batch() + [graph(1001, 1, 1)]
    for g, w in zip(run(fe, probs, max_iters=max_iters), singles(fe, probs, max_iters=max_iters)):
        assert_same(g, w)


def test_the_stop_cases_and_the_isolated_vertex(fe):
    probs = [identity_graph(), overflow_graph(), isolated_graph(), edgeless_graph(), graph(65, 5, 0)]
    got = run(fe, probs)
    for g, w in zip(got, singles(fe, probs)):
        assert_same(g, w)
    assert [g["stop"] for g in got[:2]] == ["rho_zero", "lambda"] and got[1]["trials"] == 46
    assert got[3]["trials"] == 0 and got[3]["chi2"] == 0.0


def test_the_mixed_batch_matches_the_oracle(fe):
    probs = mixed_batch()
    for p, g in zip(probs, run(fe, probs)):
        ref = pgo.optimize(p)
        _compare(g, ref)
        _final(p, g, ref)


# ---- the C ABI directly: NULL and short traces, refusals -----------------------------------------------------------------
def raw_batch(fe, probs, caps=None, max_iters=100, lambda_init=1e-10, n=None, null=None, k_null=None, nulls=()):
    """plf_pose_graph_batch through ctypes: problem k's trace holds caps[k] rows (None: a NULL trace), and problem
    k_null's array `null` is passed as NULL (null = "trace": a NULL trace with its capacity; "n_v" / "n_e": that count
    passed as -1).  `nulls` names the call's own arguments passed as NULL ("opts", "problems", "out").  Returns (rc, out's bytes before and after the call, poses, traces, out)."""
    keep = []
    Ts, trs = [], []
    arr = (plf.plf_pgo_problem * max(len(probs), 1))()
    res = (plf.plf_pgo_result * max(len(probs), 1))()
    ad = lambda x: x.ctypes.data if x.size else None
    for k, p in enumerate(probs):
        T = np.ascontiguousarray(p["T"], np.float64).reshape(-1, 16).copy()
        a = {"fixed": np.ascontiguousarray(p["fixed"], np.uint8).ravel(),
             "from": np.ascontiguousarray(p["from"], np.int32).ravel(),
             "to": np.ascontiguousarray(p["to"], np.int32).ravel(),
             "Z": np.ascontiguousarray(p["Z"], np.float64).reshape(-1, 16)}
        keep.append(a)
        ptr = lambda name, x: None if (k == k_null and name == null) else ad(x)
        arr[k] = plf.plf_pgo_problem(len(T), len(a["from"]), ptr("T", T), *[ptr(m, a[m]) for m in ("fixed", "from", "to", "Z")])
        if k == k_null and null in ("n_v", "n_e"):
            setattr(arr[k], null, -1)
        cap = 10 * max_iters if caps is None else caps[k]
        tr = np.zeros(max(cap or 0, 0), plf.PGO_TRACE_DTYPE)
        res[k].trace = None if (k == k_null and null == "trace") else (ad(tr) if tr.size else None)
        res[k].trace_cap = cap or 0
        Ts.append(T); trs.append(tr)
    before = [bytes(r) for r in res][:len(probs)]
    opts = plf.plf_pgo_opts(max_iters, lambda_init)
    rc = fe.lib.plf_pose_graph_batch(fe._ctx, None if "opts" in nulls else C.byref(opts), len(probs) if n is None else n,
                                     None if "problems" in nulls else arr, None if "out" in nulls else res)
    return rc, before, [bytes(r) for r in res][:len(probs)], Ts, trs, res


def test_null_and_short_traces(fe):
    probs = mixed_batch()[:8]
    caps = [None, 0, 1, 5, None, 1000, 3, None]
    want = singles(fe, probs)
    rc, _, _, Ts, trs, res = raw_batch(fe, probs, caps)
    assert rc == 0
    for k, w in enumerate(want):
        assert bits(Ts[k].reshape(-1, 4, 4)) == bits(w["T"])
        r = res[k]
        for name in SCALARS:
            v = plf.PGO_STOP[r.stop] if name == "stop" else getattr(r, name)
            assert bits(v) == bits(w[name]), (k, name)
        m = min(w["trials"], caps[k] or 0)
        assert r.n_trace == m and bits(trs[k][:m]) == bits(w["trace"][:m])


def _bad_problems(p):
    """(name, problem, code) for plf_pose_graph's per-problem refusals"""
    out = []
    f = p["from"].copy(); f[3] = len(p["T"])
    out.append(("edge out of range", dict(p, **{"from": f}), PLF_ERR_INVALID))
    f = p["from"].copy(); f[3] = -1
    out.append(("negative vertex", dict(p, **{"from": f}), PLF_ERR_INVALID))
    t = p["to"].copy(); t[5] = p["from"][5]
    out.append(("self edge", dict(p, to=t), PLF_ERR_INVALID))
    T = p["T"].copy(); T[7, 1, 2] = np.nan
    out.append(("NaN pose", dict(p, T=T), PLF_ERR_INVALID))
    Z = p["Z"].copy(); Z[2, 0, 3] = np.inf
    out.append(("infinite measurement", dict(p, Z=Z), PLF_ERR_INVALID))
    n = len(p["T"])
    out.append(("component without a fixed vertex", {
        "T": np.concatenate([p["T"], p["T"][:2]]), "fixed": np.concatenate([p["fixed"], [0, 0]]),
        "from": np.append(p["from"], n).astype(np.int32), "to": np.append(p["to"], n + 1).astype(np.int32),
        "Z": np.concatenate([p["Z"], p["Z"][:1]])}, PLF_ERR_INVALID))
    out.append(("4097 free vertices", synth.pose_graph_problem(4098, 1, 0, drift=0.0, seed=1), PLF_ERR_CAPACITY))
    return out


def test_refusals_write_nothing_and_leave_the_context_usable(fe):
    good = [graph(12, 5, 1), graph(65, 5, 0), graph(101, 1, 4), graph(12, 1, 4)]
    want = singles(fe, good)
    p = graph(40, 3, 2)

    def usable():
        for g, w in zip(run(fe, good), want):
            assert_same(g, w)

    def refused(name, code, r, probs, k=2):
        rc, before, after, Ts, _, _ = r
        assert rc == code, name
        assert f"problem {k}: " in fe.lib.plf_last_error(fe._ctx).decode(), name
        assert before == after, name
        for T, q in zip(Ts, probs):
            assert bits(T) == bits(np.ascontiguousarray(q["T"], np.float64).reshape(-1, 16)), name
        usable()

    for name, bad, code in _bad_problems(p):
        probs = good[:2] + [bad] + good[2:]
        refused(name, code, raw_batch(fe, probs), probs)
    probs = good[:2] + [p] + good[2:]
    for null in ("T", "fixed", "from", "to", "Z"):
        refused(f"NULL {null}", PLF_ERR_INVALID, raw_batch(fe, probs, null=null, k_null=2), probs)
    refused("negative trace_cap", PLF_ERR_INVALID, raw_batch(fe, probs, caps=[10, 10, -1, 10, 10]), probs)
    refused("trace_cap without a trace", PLF_ERR_INVALID, raw_batch(fe, probs, null="trace", k_null=2), probs)
    for count in ("n_v", "n_e"):
        refused(f"negative {count}", PLF_ERR_INVALID, raw_batch(fe, probs, null=count, k_null=2), probs)
    # the first bad problem is named, whichever of its rules it breaks
    T = p["T"].copy(); T[7, 1, 2] = np.nan
    probs2 = good[:1] + [dict(p, T=T)] + good[1:3] + [p]
    refused("NaN pose before a negative count", PLF_ERR_INVALID, raw_batch(fe, probs2, null="n_v", k_null=4), probs2, k=1)
    # the batch's own arguments: NULL opts, problems or out with problems
    for arg in ("opts", "problems", "out"):
        rc, before, after, Ts, _, _ = raw_batch(fe, probs, nulls=(arg,))
        assert rc == PLF_ERR_INVALID and "bad arguments" in fe.lib.plf_last_error(fe._ctx).decode(), arg
        assert before == after, arg
        for T, q in zip(Ts, probs):
            assert bits(T) == bits(np.ascontiguousarray(q["T"], np.float64).reshape(-1, 16)), arg
        usable()
    # the batch's own rules, and n_problems = 0
    for n, code in ((-1, PLF_ERR_INVALID), (65536, PLF_ERR_CAPACITY)):
        rc, before, after, Ts, _, _ = raw_batch(fe, good, n=n)
        assert rc == code and before == after, n
        usable()
    rc, before, after, _, _, _ = raw_batch(fe, good, lambda_init=0.0)
    assert rc == PLF_ERR_INVALID and before == after and "lambda_init" in fe.lib.plf_last_error(fe._ctx).decode()
    n0 = fe.launches
    assert raw_batch(fe, good, n=0)[0] == 0 and fe.launches == n0
    assert fe.pose_graph_batch([]) == [] and fe.launches == n0
    usable()


def test_scratch_that_does_not_fit_fails_writes_nothing_and_the_context_stays_usable(fe):
    """twenty 4096-keyframe graphs: 20 x 288 x 4095^2 bytes = 97 GB of dense systems, more than the card holds"""
    big = synth.pose_graph_problem(4096, 1, 0, drift=0.01, seed=2)
    rc, before, after, Ts, _, _ = raw_batch(fe, [big] * 20, max_iters=2)
    assert rc == PLF_ERR_CUDA and "scratch" in fe.lib.plf_last_error(fe._ctx).decode()
    assert before == after
    assert all(bits(T) == bits(np.ascontiguousarray(big["T"], np.float64).reshape(-1, 16)) for T in Ts)
    probs = mixed_batch()
    for g, w in zip(run(fe, probs), singles(fe, probs)):
        assert_same(g, w)


def test_pose_graph_batch_between_batches_leaves_the_pipeline_unchanged(built):
    cam = dict(plf.KITTI_CAMERA, width=480, height=300, cx=240.0, cy=150.0, fx=400.0, fy=400.0)
    world = osynth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    frames = list(osynth.stream(cam, 8, world=world, seed=5, step=0.1))
    L = np.stack([f[0] for f in frames]); R = np.stack([f[1] for f in frames])
    lim = plf.default_limits(); lim.max_batch = 2
    probs = [graph(684, 5, 4), graph(65, 5, 0)]

    def run_pipe(with_pgo):
        with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=500, lsd_nfeatures=100) as f:
            out, pg = [], None
            for b in range(0, 8, 2):
                f.batch_upload(L[b:b + 2], R[b:b + 2])
                f.batch_run(2)
                if with_pgo and b == 4:   # two batches, pose_graph_batch with the third in flight, two batches
                    pg = f.pose_graph_batch(probs)
                res = f.batch_download_array(2)
                out += [np.ascontiguousarray(res[k]) for k in res.dtype.names]
                out += [np.ascontiguousarray(a) for a in f.get_frame(1).values() if isinstance(a, np.ndarray)]
            return out, pg

    (a, _), (b, pg) = run_pipe(False), run_pipe(True)
    assert len(a) == len(b) and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    with plf.Frontend(camera=cam) as f:
        for p, got in zip(probs, pg):
            assert_same(got, f.pose_graph(p))
