"""CPU tests of the motion model (plf_set_motion_model): the rule as oracle/motion_model.py restates it, at each edge
of stvo-pl's isGoodSolution, the oracle pipeline with the model off and with identity predictions, and the argument
checks of the C ABI, which run before the context is looked at."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from oracle import clib, synth
from oracle import frontend as ofe
from oracle.frontend import run_sequence
from oracle.motion_model import eig_range, prior

ROOT = Path(__file__).resolve().parent.parent
ULP0 = np.nextafter(0.0, 1.0)    # the smallest positive double
ONE_UP = np.nextafter(1.0, 2.0)
MOVED = clib.inverse_se3(clib.expmap_se3(np.array([0.02, -0.01, 0.9, 0.003, -0.002, 0.001])))   # a published DT
COV = np.diag([1e-4, 2e-4, 3e-4, 1e-5, 2e-5, 3e-5])


def cov_with(lo=None, hi=None):
    d = np.diag(COV).copy()
    if lo is not None:
        d[2] = lo
    if hi is not None:
        d[4] = hi
    return np.diag(d)


# (name, status, DT, DT_cov, err, good): every edge of the rule; shared with the device test (tests/test_motion_model_gpu.py)
EDGES = [
    ("good", 0, MOVED, COV, 0.5, True),
    ("eig_min_0", 0, MOVED, cov_with(lo=0.0), 0.5, True),
    ("eig_min_-ulp", 0, MOVED, cov_with(lo=-ULP0), 0.5, False),
    ("eig_min_-0", 0, MOVED, cov_with(lo=-0.0), 0.5, True),
    ("eig_max_1", 0, MOVED, cov_with(hi=1.0), 0.5, True),
    ("eig_max_1+ulp", 0, MOVED, cov_with(hi=ONE_UP), 0.5, False),
    ("err_-1", 0, MOVED, COV, -1.0, False),
    ("err_0", 0, MOVED, COV, 0.0, True),
    ("err_1", 0, MOVED, COV, 1.0, True),
    ("err_1+ulp", 0, MOVED, COV, ONE_UP, False),
    ("err_nan", 0, MOVED, COV, np.nan, True),
    ("DT_nan", 0, np.where(np.eye(4, k=1) > 0, np.nan, MOVED), COV, 0.5, False),
    ("DT_inf", 0, np.where(np.eye(4, k=-1) > 0, np.inf, MOVED), COV, 0.5, False),
    ("cov_nan", 0, MOVED, np.full((6, 6), np.nan), 0.5, True),
    ("cov_one_nan", 0, MOVED, np.where(np.eye(6, k=2) > 0, np.nan, COV), 0.5, True),
    ("status_1", 1, np.eye(4), np.zeros((6, 6)), -1.0, False),
    ("status_2", 2, np.eye(4), np.zeros((6, 6)), -1.0, False),
    ("status_1_good_fields", 1, MOVED, COV, 0.5, False),
    ("status_2_good_fields", 2, MOVED, COV, 0.5, False),
]


@pytest.mark.parametrize("name, status, DT, cov, err, good", EDGES, ids=[e[0] for e in EDGES])
def test_rule_at_each_edge(name, status, DT, cov, err, good):
    T, valid = prior(status, DT, cov, err)
    assert valid == good, name
    if good:
        assert np.array_equal(T, clib.inverse_se3(DT))
    else:
        assert np.array_equal(T, np.eye(4))


def test_diagonal_eigenvalues_are_exact():
    """The edge covariances are diagonal, so the eigenvalues the rule compares are the diagonal itself."""
    for lo in (0.0, -ULP0, -0.0, 1e-300):
        assert eig_range(cov_with(lo=lo))[0] == lo
    for hi in (1.0, ONE_UP):
        assert eig_range(cov_with(hi=hi))[1] == hi
    assert all(np.isnan(eig_range(np.where(np.eye(6, k=2) > 0, np.nan, COV))))


def test_prediction_is_the_optimisers_transform():
    """DT is the published increment inverse_se3(T_gn); the prediction is inverse_se3(DT), which maps the previous
    frame into the current one (the solver's own direction)."""
    T, valid = prior(0, MOVED, COV, 0.5)
    assert valid and np.allclose(T @ MOVED, np.eye(4), atol=1e-15)


CAM = dict(width=480, height=300, fx=400.0, fy=400.0, cx=240.0, cy=150.0, b=0.5)
PRM = dict(orb_nfeatures=500, lsd_nfeatures=100)


def _frames(n=3):
    world = synth.World(seed=3, length=40.0, n_quads=120, n_segs=60, half_width=6.0, half_height=3.0)
    return [(a, b) for a, b, _ in synth.stream(CAM, n, world=world, seed=5, step=0.1)]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x["status"] == y["status"] and x["DT"].tobytes() == y["DT"].tobytes() and x["Tfw"].tobytes() == y["Tfw"].tobytes()
        assert (x["n_pt"], x["n_ls"]) == (y["n_pt"], y["n_ls"])
        if x["res"] is not None:
            for k in ("T", "cov", "err", "iters", "inlier_pt", "inlier_ls"):
                assert np.asarray(x["res"][k]).tobytes() == np.asarray(y["res"][k]).tobytes(), k


@pytest.mark.parametrize("strategy", [0, 3])
def test_off_is_todays_oracle_pipeline(strategy):
    """With the model off the runner gives byte for byte what oracle/frontend.py run_sequence gives."""
    pairs = _frames()
    prm = dict(PRM, matching_strategy=strategy)
    today = ofe.run_sequence(CAM, pairs, dict(ofe.DEFAULTS, **prm))
    off = run_sequence(CAM, pairs, prm, motion_model=False, frames=[o["frame"] for o in today])
    _same(today, off)
    assert all(np.array_equal(o["T_pred"], np.eye(4)) for o in off)
    # identity predictions (finite points): the projection through I and the solver seeded with I change nothing
    ident = run_sequence(CAM, pairs, prm, motion_model=True, preds=[np.eye(4)] * len(pairs), frames=[o["frame"] for o in today])
    _same(today, ident)


def test_carried_prediction_and_restart():
    pairs = _frames(4)
    out = run_sequence(CAM, pairs, dict(PRM, matching_strategy=3), motion_model=True, restarts={2})
    assert [o["status"] for o in out] == [2, 0, 2, 0]
    assert not out[0]["valid_next"] and np.array_equal(out[1]["T_pred"], np.eye(4))
    assert out[1]["valid_next"] and np.array_equal(out[1]["T_next"], clib.inverse_se3(out[1]["DT"]))
    assert np.array_equal(out[2]["T_pred"], np.eye(4))    # a restart starts from identity
    assert np.array_equal(out[3]["T_pred"], out[2]["T_next"])


def _lib(built):
    import plslam_b200 as plf
    lib = plf.load_library()
    lib.plf_last_error.restype = C.c_char_p
    return plf, lib


def test_abi_declared(built):
    plf, _ = _lib(built)
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert "plf_status plf_set_motion_model(plf_ctx* ctx, int on);" in hdr
    assert "plf_status plf_get_sequence_motion(plf_ctx* ctx, int s, double T[16], int* valid);" in hdr
    assert re.search(r"plf_status plf_debug_motion_prior\(plf_ctx\* ctx, int n, const double\* DT, const double\* DT_cov, "
                     r"const double\* err,\s*const int32_t\* status, double\* T_out, int32_t\* valid_out\);", hdr)
    for m in ("set_motion_model", "sequence_motion", "debug_motion_prior"):
        assert callable(getattr(plf.Frontend, m))


def test_abi_null_context(built):
    _, lib = _lib(built)
    assert lib.plf_set_motion_model(None, 1) == -1
    assert "ctx is NULL" in lib.plf_last_error(None).decode()
    T = (C.c_double * 16)(*([7.0] * 16))
    v = C.c_int(7)
    assert lib.plf_get_sequence_motion(None, 0, T, C.byref(v)) == -1 and v.value == 7 and T[0] == 7.0
    assert lib.plf_debug_motion_prior(None, 0, None, None, None, None, None, None) == -1
