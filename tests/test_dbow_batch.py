"""CPU tests of the per-sequence bag-of-words interface (plf_bow_insert_batch / plf_bow_erase_seq / plf_bow_get_seq /
plf_bow_clear_sequence): the header declares the four calls and the library exports them, the binding exposes the
methods, a NULL context is refused without a device, the ctypes mirror of plf_bow_problem has the C layout, and the
binding refuses a malformed `seq` before any library call."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
FIELDS = ("kf_idx", "kf", "score_p", "score_l")


def test_declared_and_exported(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    for decl in (r"plf_status plf_bow_insert_batch\(plf_ctx\* ctx, int n_problems, plf_bow_problem\* problems, "
                 r"const int32_t\* seq\);",
                 r"plf_status plf_bow_erase_seq\(plf_ctx\* ctx, int s, int kf_idx\);",
                 r"plf_status plf_bow_get_seq\(plf_ctx\* ctx, int s, int kf_idx, int kind, int cap, uint32_t\* words, "
                 r"double\* values, int\* n\);",
                 r"plf_status plf_bow_clear_sequence\(plf_ctx\* ctx, int s\);"):
        assert re.search(decl, hdr), decl
    lib = plf.load_library()
    for fn in ("plf_bow_insert_batch", "plf_bow_erase_seq", "plf_bow_get_seq", "plf_bow_clear_sequence"):
        assert hasattr(lib, fn), fn
    for meth in ("bow_insert_batch", "bow_erase", "bow_vector", "bow_clear_sequence"):
        assert callable(getattr(plf.Frontend, meth)), meth
    # NULL context: PLF_ERR_INVALID, without a device
    n = C.c_int(0)
    assert lib.plf_bow_insert_batch(None, 0, None, None) == -1
    assert lib.plf_bow_erase_seq(None, 0, 0) == -1
    assert lib.plf_bow_get_seq(None, 0, 0, 0, 0, None, None, C.byref(n)) == -1
    assert lib.plf_bow_clear_sequence(None, 0) == -1


def test_seq_keyword_defaults_keep_the_single_calls():
    import inspect
    import plslam_b200 as plf
    for meth in ("bow_erase", "bow_vector", "bow_insert_batch"):
        assert inspect.signature(getattr(plf.Frontend, meth)).parameters["seq"].default is None, meth


def test_problem_struct_layout(built, tmp_path):
    """sizeof and offsetof of every field, from a C program compiled against the header, equal the ctypes mirror's."""
    import plslam_b200 as plf
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layout"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "plslam_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(plf_bow_problem));']
    lines += [f'  printf("{f} %zu\\n", offsetof(plf_bow_problem, {f}));' for f in FIELDS]
    lines.append("  return 0;\n}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c11", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {a: int(b) for a, b in (ln.split() for ln in out if ln)}
    assert [f for f, _ in plf.plf_bow_problem._fields_] == list(FIELDS)
    assert got["size"] == C.sizeof(plf.plf_bow_problem)
    for f in FIELDS:
        assert got[f] == getattr(plf.plf_bow_problem, f).offset, f


@pytest.mark.parametrize("seq,msg", [([0, 1], "3 entries"), (np.zeros((3, 1), np.int32), "3 entries"),
                                     (np.zeros(3, np.float64), "integer"), ([0, 1, 2 ** 40], "int32")])
def test_binding_refuses_a_malformed_seq(built, seq, msg):
    """The refusal comes before any library call: the Frontend here has no context, and the problems are never read."""
    import plslam_b200 as plf
    fe = object.__new__(plf.Frontend)
    with pytest.raises(plf.PlfError, match=msg):
        fe.bow_insert_batch([None, None, None], seq=seq)
