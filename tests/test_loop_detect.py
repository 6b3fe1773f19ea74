"""CPU tests of loop-closure candidate detection (plf_bow_detect / plf_bow_detect_batch / plf_debug_loop_candidates):
the oracle (oracle/loopdetect.py) on hand-built columns covering every branch of lookForLoopCandidates
(src/mapHandler.cpp:3130-3190), the recalled vector_stdv and the conf_matrix combination, the decidability of the case
tables the device tests reuse, and the interface: declarations, exports, struct layouts and NULL-context refusals."""
import ctypes as C
import math
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from loopdetect_cases import cases
from oracle import loopdetect as old

ROOT = Path(__file__).resolve().parent.parent
CASES = cases()


def same_result(a, b):
    return all(a[k] == b[k] or (isinstance(b[k], float) and math.isnan(a[k]) and math.isnan(b[k])) for k in b)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_oracle_on_hand_built_columns(c):
    col = c["col"]
    got = old.look_for_loop_candidates(col["conf"], col["live"], col["covis"], col["kf_idx"], c["opts"])
    assert same_result(got, c["want"]), (got, c["want"])


def _near(s, t):
    return abs(s - t) <= 1e-6 * max(abs(t), 1e-3)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_case_tables_are_decidable(c):
    """Only the entries a case names sit within float rounding of a threshold: 0.001 for the entries that enter the
    minimum, the best score for ties, lc_min_score * 0.8 for the close keyframes, lc_min_score for the best."""
    col, o, r = c["col"], c["opts"], c["want"]
    kf, conf, live = col["kf_idx"], col["conf"], col["live"]
    cov = np.zeros(kf, np.uint32) if col["covis"] is None else col["covis"]
    if r["best"] < 0:
        return
    best, mn = r["best"], r["min_score"]
    bs = float(conf[best])
    if not math.isnan(bs) and best not in c["exact"]:
        assert not _near(bs, mn), best
    for i in range(kf + 1):
        s = float(conf[i])
        if not live[i] or math.isnan(s) or i in c["exact"]:
            continue
        if i < kf and (int(cov[i]) >= o["min_lm_cov_graph"] % (1 << 32) or kf - i <= o["min_kf_local_map"] + 3):
            assert not _near(s, 0.001), i
        if i < min(kf - o["lc_kf_dist"], kf + 1) and i != best:
            assert not _near(s, bs), i
            if abs(i - best) <= o["lc_kf_max_dist"]:
                assert not _near(s, mn * 0.8), i


def test_vector_stdv_edges():
    assert old.vector_stdv([]) == 0.0
    assert math.isnan(old.vector_stdv([3.5]))
    assert old.vector_stdv([1.0, 3.0]) == math.sqrt(2.0)


def test_vector_stdv_sums_in_index_order():
    """1 followed by 1023 values of 2^-60: sequentially each addend vanishes against 1, so the mean is 2^-10 exactly; a
    pairwise sum (numpy's) keeps them and gives another mean."""
    xs = [1.0] + [2.0 ** -60] * 1023
    seq_mean = 2.0 ** -10
    acc = 0.0
    for x in xs:
        acc += (x - seq_mean) * (x - seq_mean)
    want = math.sqrt(acc / 1023)
    assert old.vector_stdv(xs) == want
    pw_mean = float(np.sum(np.array(xs))) / 1024
    assert pw_mean != seq_mean


def test_conf_row_combinations():
    sp = np.array([0.5, np.nan, -0.0, 0.25])
    sl = np.array([0.25, np.nan, 0.125, 0.75])
    live = np.array([True, False, True, True])
    p = old.conf_row((1, 0), live, sp, sl)
    assert np.array_equal(p[[0, 2, 3]].view(np.uint32), np.float32(sp[[0, 2, 3]]).view(np.uint32)) and np.isnan(p[1])
    assert np.signbit(p[2])
    l = old.conf_row((0, 1), live, sp, sl)
    assert np.array_equal(l[[0, 2, 3]], np.float32(sl[[0, 2, 3]])) and np.isnan(l[1])
    pl = old.conf_row((1, 1), live, sp, sl, n_pt=3, n_ls=1, std_pt=2.0, std_ls=1.0)
    assert pl[0] == np.float32((0.0 + (0.5 * 3 + 0.25 * 1) / 4) + (0.5 * 2.0 + 0.25 * 1.0) / 3.0)
    assert np.isnan(pl[1])
    # no feature (n_pl = 0) and no dispersion (std_pl = 0): the whole column is NaN
    assert np.all(np.isnan(old.conf_row((1, 1), live, sp, sl, n_pt=0, n_ls=0, std_pt=0.0, std_ls=0.0)))
    assert np.all(np.isnan(old.conf_row((1, 1), live, sp, sl, n_pt=4, n_ls=2, std_pt=0.0, std_ls=0.0)))


def test_dispersions_of_points_and_line_midpoints():
    pt = np.array([[1.0, 2.0], [3.0, 6.0]])
    s, e = np.array([[0.0, 0.0], [2.0, 2.0], [4.0, 0.0]]), np.array([[2.0, 2.0], [4.0, 4.0], [6.0, 2.0]])
    std_pt, std_ls = old.dispersions(pt, s, e)
    assert std_pt == math.sqrt(2.0) + math.sqrt(8.0)
    assert std_ls == old.vector_stdv([1.0, 3.0, 5.0]) + old.vector_stdv([1.0, 3.0, 1.0])
    one_pt, no_ls = old.dispersions(pt[:1], s[:0], e[:0])
    assert math.isnan(one_pt) and no_ls == 0.0


DECLS = (r"plf_status plf_bow_detect\(plf_ctx\* ctx, const plf_lc_detect_opts\* opts, plf_lc_detect_problem\* problem\);",
         r"plf_status plf_bow_detect_batch\(plf_ctx\* ctx, const plf_lc_detect_opts\* opts, int n_problems,\s*"
         r"plf_lc_detect_problem\* problems, const int32_t\* seq\);",
         r"plf_status plf_debug_loop_candidates\(plf_ctx\* ctx, const plf_lc_detect_opts\* opts, int n, const int\* kf_idx,"
         r"\s*const float\* const\* conf, const uint8_t\* const\* live,\s*const uint32_t\* const\* covis, "
         r"plf_lc_detect_result\* out\);")


def test_declared_and_exported(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    for decl in DECLS:
        assert re.search(decl, hdr), decl
    lib = plf.load_library()
    for fn in ("plf_bow_detect", "plf_bow_detect_batch", "plf_debug_loop_candidates"):
        assert hasattr(lib, fn), fn
    for meth in ("bow_detect", "bow_detect_batch", "debug_loop_candidates"):
        assert callable(getattr(plf.Frontend, meth)), meth
    o = plf._lc_opts(None)
    assert lib.plf_bow_detect(None, C.byref(o), None) == -1
    assert lib.plf_bow_detect_batch(None, C.byref(o), 0, None, None) == -1
    assert lib.plf_debug_loop_candidates(None, C.byref(o), 0, None, None, None, None, None) == -1


def test_defaults_are_the_reference_config():
    import plslam_b200 as plf
    assert plf.LC_DETECT_DEFAULTS == old.DEFAULTS
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    for name, v in old.DEFAULTS.items():
        assert re.search(rf"int {name};.*\({v}\)", hdr), name


@pytest.mark.parametrize("struct,fields", [
    ("plf_lc_detect_opts", ("lc_kf_dist", "lc_kf_max_dist", "lc_nkf_closest", "min_lm_cov_graph", "min_kf_local_map")),
    ("plf_lc_detect_result", ("candidate", "best", "n_listed", "n_closest", "min_score")),
    ("plf_lc_detect_problem", ("kf_idx", "kf", "covis", "conf", "score_p", "score_l", "result"))])
def test_struct_layout(built, tmp_path, struct, fields):
    """sizeof and offsetof of every field, from a C program compiled against the header, equal the ctypes mirror's."""
    import plslam_b200 as plf
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layout"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "plslam_b200.h"', "int main(void) {",
             f'  printf("size %zu\\n", sizeof({struct}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f in fields]
    lines.append("  return 0;\n}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c11", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {a: int(b) for a, b in (ln.split() for ln in out if ln)}
    cls = getattr(plf, struct)
    assert [f for f, _ in cls._fields_] == list(fields)
    assert got["size"] == C.sizeof(cls)
    for f in fields:
        assert got[f] == getattr(cls, f).offset, f


@pytest.mark.parametrize("key,shape,msg", [("pt_pl", (2, 2), "pt_pl has 4 values for 3 rows of pdesc"),
                                           ("ls_spl", (4, 2), "ls_spl has 8 values for 5 rows of ldesc"),
                                           ("ls_epl", (5, 1), "ls_epl has 5 values for 5 rows of ldesc")])
def test_binding_refuses_coordinates_that_do_not_match_the_descriptors(built, key, shape, msg):
    """The refusal comes before any library call (the library would read n_pt / n_ls rows of each array): the Frontend
    here has no context."""
    import plslam_b200 as plf
    fe = object.__new__(plf.Frontend)
    fe.params = plf.default_params()
    pr = dict(kf_idx=0, pdesc=np.zeros((3, 32), np.uint8), ldesc=np.zeros((5, 32), np.uint8), pt_pl=np.zeros((3, 2)),
              ls_spl=np.zeros((5, 2)), ls_epl=np.zeros((5, 2)))
    pr[key] = np.zeros(shape)
    with pytest.raises(plf.PlfError, match=msg):
        fe.bow_detect(pr)
    with pytest.raises(plf.PlfError, match="problem 1: " + msg):
        fe.bow_detect_batch([dict(pr, **{key: np.zeros((3 if key == "pt_pl" else 5, 2))}), pr])


def test_integration_f8_snippet_is_the_compiled_block():
    """INTEGRATION.md §4 f8's code is, line for line, the BEGIN f8 / END f8 block vo_demo compiles and
    test_loop_detect_gpu.py runs."""
    src = (ROOT / "pl-slam_b200" / "cpp" / "vo_demo.cpp").read_text()
    block = src.split("// BEGIN f8\n", 1)[1].split("// END f8\n", 1)[0]
    doc = (ROOT / "INTEGRATION.md").read_text()
    sec = doc.split("* **f8 — loop-candidate detection**", 1)[1]
    code = sec.split("  ```cpp\n", 1)[1].split("  ```\n", 1)[0]
    assert [ln[2:] if ln.startswith("  ") else ln for ln in code.splitlines()] == block.splitlines()
