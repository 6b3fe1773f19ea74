"""CPU tests of the adaptive FAST threshold (plf_set_adaptive_fast): the rule as oracle/adaptive_fast.py restates it,
branch by branch, and the argument checks of the C ABI, which run before the context is looked at."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from oracle import frontend as ofe
from oracle.adaptive_fast import BRANCHES, fast_th_next

ROOT = Path(__file__).resolve().parent.parent
CFG = dict(min_th=5, max_th=50, inc_th=5, feat_th=50, err_th=0.5)   # config_euroc.yaml:36-41
I4 = np.eye(4)
MOVED = np.eye(4)
MOVED[0, 3] = 0.1


def nxt(th, n, status=0, DT=MOVED, err=0.1, cfg=CFG):
    return fast_th_next(th, status, DT, err, n, cfg, trace=True)


def test_every_branch():
    assert nxt(20, 500, status=2, DT=I4, err=-1.0) == (20, "first")      # no update on a first frame
    assert nxt(20, 0, status=1, DT=I4, err=-1.0) == (10, "bad_pose")     # too few rows: identity
    assert nxt(20, 500, DT=I4) == (10, "bad_pose")                        # an optimised pose that is exactly I
    assert nxt(20, 500, err=0.5000001) == (10, "bad_pose")
    assert nxt(20, 500, err=0.5) == (25, "many")                          # err == err_th is not > err_th
    assert nxt(20, 49) == (10, "few")
    assert nxt(20, 50) == (15, "some")
    assert nxt(20, 99) == (15, "some")
    assert nxt(20, 100) == (20, "keep")
    assert nxt(20, 150) == (20, "keep")
    assert nxt(20, 151) == (25, "many")
    assert nxt(20, 10 ** 6) == (25, "many")


def test_identity_compares_exactly():
    near = np.eye(4)
    near[2, 3] = 1e-300
    assert nxt(20, 500, DT=near) == (25, "many")
    neg0 = np.eye(4)
    neg0[0, 1] = -0.0
    assert nxt(20, 500, DT=neg0) == (10, "bad_pose")


def test_clamps():
    assert nxt(8, 0) == (5, "few") and nxt(5, 0) == (5, "few")
    assert nxt(7, 60) == (5, "some")
    assert nxt(48, 500) == (50, "many") and nxt(50, 500) == (50, "many")
    zero = dict(CFG, min_th=0)                                            # config_kitti.yaml
    assert nxt(3, 0, cfg=zero) == (0, "few") and nxt(0, 0, cfg=zero) == (0, "few")
    assert nxt(0, 500, cfg=zero) == (5, "many")
    # a start outside [min_th, max_th] is moved by the same rule: stvo-pl clamps only the result
    assert nxt(80, 500) == (50, "many") and nxt(2, 0) == (5, "few")


def test_the_fifth_branch_is_unreachable():
    """stvo-pl's "> 4 feat_th: + 2 inc_th" comes after "> 3 feat_th": no inlier count reaches it."""
    seen = set()
    for f in (0, 1, 2, 7, 50):
        for n in range(0, 5 * f + 20):
            for DT, err in ((MOVED, 0.1), (I4, 0.1), (MOVED, 1.0)):
                seen.add(nxt(20, n, DT=DT, err=err, cfg=dict(CFG, feat_th=f))[1])
    assert "very_many" not in seen
    assert seen == set(BRANCHES) - {"very_many", "first"}


def test_reset_on_restart(monkeypatch):
    """The stream runner detects every first frame at orb_fast_th and carries the rule's threshold otherwise."""
    used = []

    def extract(cam, L, R, prm, *_):
        used.append(prm["orb_fast_th"])
        return ofe.Frame()

    monkeypatch.setattr(ofe, "extract_stereo", extract)   # empty frames: status 1 after the first, th - 2 inc_th
    out = ofe.run_sequence({}, [(None, None)] * 6, dict(orb_fast_th=20), adaptive_fast=CFG, restarts={3})
    assert used == [20, 20, 10, 20, 20, 10]
    assert [o["status"] for o in out] == [2, 1, 1, 2, 1, 1]
    assert [o["branch"] for o in out] == ["first", "bad_pose", "bad_pose", "first", "bad_pose", "bad_pose"]
    used.clear()
    ofe.run_sequence({}, [(None, None)] * 3, dict(orb_fast_th=300), adaptive_fast=CFG)
    assert used == [255, 255, 245]   # orb_fast_th clamped to [0, 255] as the detector applies it
    used.clear()
    ofe.run_sequence({}, [(None, None)] * 3, dict(orb_fast_th=20), adaptive_fast=CFG, fast_th=[7, 30, 0])
    assert used == [7, 30, 0]


def _lib(built):
    import plslam_b200 as plf
    lib = plf.load_library()
    lib.plf_last_error.restype = C.c_char_p
    return plf, lib


def test_abi_declared_and_sized(built):
    plf, lib = _lib(built)
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"typedef struct plf_adaptive_fast \{\s*int min_th, max_th, inc_th, feat_th;\s*double err_th;\s*\} plf_adaptive_fast;", hdr)
    assert "plf_status plf_set_adaptive_fast(plf_ctx* ctx, const plf_adaptive_fast* cfg);" in hdr
    assert "plf_status plf_get_sequence_fast_th(plf_ctx* ctx, int s, int* th);" in hdr
    assert C.sizeof(plf.plf_adaptive_fast) == 24
    assert callable(plf.Frontend.set_adaptive_fast) and callable(plf.Frontend.sequence_fast_th)


@pytest.mark.parametrize("field, value", [("min_th", -1), ("max_th", 256), ("min_th", 51), ("inc_th", -1), ("feat_th", -1),
                                          ("err_th", float("nan")), ("err_th", float("inf")), ("err_th", -float("inf"))])
def test_abi_refuses_each_field(built, field, value):
    """Each invalid field is refused with PLF_ERR_INVALID and named, before the context is looked at."""
    plf, lib = _lib(built)
    a = plf.plf_adaptive_fast(**dict(CFG, **{field: value}))
    assert lib.plf_set_adaptive_fast(None, C.byref(a)) == -1
    msg = lib.plf_last_error(None).decode()
    assert msg.startswith("plf_set_adaptive_fast: ") and field in msg, msg


def test_abi_null_context(built):
    plf, lib = _lib(built)
    ok = plf.plf_adaptive_fast(**CFG)
    assert lib.plf_set_adaptive_fast(None, C.byref(ok)) == -1
    assert "ctx is NULL" in lib.plf_last_error(None).decode()
    assert lib.plf_set_adaptive_fast(None, None) == -1
    th = C.c_int(7)
    assert lib.plf_get_sequence_fast_th(None, 0, C.byref(th)) == -1 and th.value == 7
    edge = plf.plf_adaptive_fast(min_th=0, max_th=255, inc_th=0, feat_th=0, err_th=-1e300)   # every bound itself is valid
    assert lib.plf_set_adaptive_fast(None, C.byref(edge)) == -1
    assert "ctx is NULL" in lib.plf_last_error(None).decode()
