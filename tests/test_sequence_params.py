"""CPU tests of per-sequence front-end settings (plf_set_sequence_params): the header declares the calls and the library
exports them, the library's classification of plf_params' fields puts every field in exactly one class (the guard that
fails when a field is added without a class), the classes are the ones DESIGN.md section 8 gives reasons for, and the
binding builds the plf_params it passes from the context's settings and the named fields."""
import ctypes as C
import re
from pathlib import Path

import pytest

from param_cases import INVARIANT, REJECTED

ROOT = Path(__file__).resolve().parent.parent

SEQUENCE = {"orb_nfeatures", "orb_fast_th", "orb_nlevels", "lsd_nfeatures", "min_line_length", "best_lr_matches",
            "max_dist_epip", "min_disp", "min_ratio_12_p", "min_ratio_12_l", "line_sim_th", "stereo_overlap_th",
            "line_horiz_th", "ls_min_disp_ratio", "matching_strategy", "matching_s_ws", "matching_f2f_ws", "min_pt_matches",
            "min_ls_matches", "homog_th", "min_features", "max_iters", "max_iters_ref", "min_error", "min_error_change"}
IGNORED = {"inlier_k", "f2f_overlap_th"}


def test_symbols(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"plf_status plf_set_sequence_params\(plf_ctx\* ctx, int s, const plf_params\* p\);", hdr)
    assert re.search(r"plf_status plf_get_sequence_params\(const plf_ctx\* ctx, int s, plf_params\* out\);", hdr)
    assert re.search(r"int plf_sequence_param_fields\(const char\*\* names, int\* classes, int cap\);", hdr)
    lib = plf.load_library()
    # NULL context: PLF_ERR_INVALID, without a device
    assert lib.plf_set_sequence_params(None, 0, None) == -1
    assert lib.plf_get_sequence_params(None, 0, None) == -1
    assert callable(plf.Frontend.set_sequence_params) and callable(plf.Frontend.get_sequence_params)


def test_every_field_in_exactly_one_class(built):
    import plslam_b200 as plf
    lib = plf.load_library()
    n = lib.plf_sequence_param_fields(None, None, 0)
    names, classes = (C.c_char_p * n)(), (C.c_int * n)()
    assert lib.plf_sequence_param_fields(names, classes, n) == n
    listed = [names[i].decode() for i in range(n)]
    fields = [k for k, _ in plf.plf_params._fields_]
    assert len(listed) == len(set(listed)), "a field is listed twice"
    assert set(listed) == set(fields), (set(fields) - set(listed), set(listed) - set(fields))
    assert set(classes) <= set(plf.PARAM_CLASSES)
    # a short array gets the first entries only
    few = (C.c_int * 2)()
    assert lib.plf_sequence_param_fields(None, few, 2) == n and list(few) == list(classes)[:2]


def test_classes(built):
    import plslam_b200 as plf
    cls = plf.sequence_param_fields()
    assert {f for f, c in cls.items() if c == "sequence"} == SEQUENCE
    assert {f for f, c in cls.items() if c == "ignored"} == IGNORED
    context = {f for f, c in cls.items() if c == "context"}
    assert context == {f for f, _ in plf.plf_params._fields_} - SEQUENCE - IGNORED
    assert {"has_points", "has_lines", "orb_scale_factor", "orb_edge_th"} <= context
    assert all(f in context for f in cls if f.startswith("lsd_") and f != "lsd_nfeatures")
    # a field with a single supported value, or one that cannot change the output, never varies per sequence
    assert not (set(REJECTED) | set(INVARIANT)) & SEQUENCE


class _Lib:
    """Records plf_set_sequence_params' arguments."""
    def __init__(self):
        self.calls = []

    def plf_set_sequence_params(self, ctx, s, p):
        self.calls.append((s, None if p is None else {k: getattr(p._obj, k) for k, _ in type(p._obj)._fields_}))
        return 0


def test_binding_builds_the_params(built):
    import plslam_b200 as plf
    fe = object.__new__(plf.Frontend)
    fe.lib, fe._ctx = _Lib(), C.c_void_p()
    fe.params = plf.default_params()
    fe.params.orb_nfeatures = 700
    fe.set_sequence_params(2, lsd_nfeatures=300, matching_strategy=3)
    s, p = fe.lib.calls[-1]
    ctx = {k: getattr(fe.params, k) for k, _ in plf.plf_params._fields_}
    assert s == 2 and p == dict(ctx, lsd_nfeatures=300, matching_strategy=3)   # fields override the context's
    other = plf.default_params()
    other.max_iters = 100
    fe.set_sequence_params(1, other, max_iters_ref=100)
    assert fe.lib.calls[-1][1] == dict({k: getattr(other, k) for k, _ in plf.plf_params._fields_}, max_iters_ref=100)
    assert other.max_iters_ref != 100 or plf.default_params().max_iters_ref == 100   # the caller's params are not changed
    fe.set_sequence_params(0)
    assert fe.lib.calls[-1] == (0, None)
    n = len(fe.lib.calls)
    with pytest.raises(plf.PlfError, match="unknown parameter no_such_field"):
        fe.set_sequence_params(0, no_such_field=1)
    assert len(fe.lib.calls) == n
