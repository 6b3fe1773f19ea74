"""CPU tests of the batched loop-closure and pose-refinement interface (plf_loop_closure_pose_batch / plf_gn_pose_batch):
the header declares both calls and the library exports them, a NULL context is refused, the ctypes mirrors of
plf_gn_problem / plf_lc_problem have the C layout, and the binding refuses a malformed `seq` before any library call."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
FIELDS = {"plf_gn_problem": ("P", "pl_obs", "inlier_pt", "np", "sP", "eP", "le_obs", "inlier_ls", "nl", "T_init", "out"),
          "plf_lc_problem": ("kf0", "kf1", "pt_pairs", "cap_pt", "ls_pairs", "cap_ls", "out", "status")}


def test_batch_symbols(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"plf_status plf_gn_pose_batch\(plf_ctx\* ctx, const plf_gn_opts\* opts, int n_problems, "
                     r"plf_gn_problem\* problems,\s+const int32_t\* seq\);", hdr)
    assert re.search(r"plf_status plf_loop_closure_pose_batch\(plf_ctx\* ctx, const plf_lc_params\* lc, int n_problems, "
                     r"plf_lc_problem\* problems,\s+const int32_t\* seq\);", hdr)
    lib = plf.load_library()
    for fn, meth in (("plf_gn_pose_batch", "gn_pose_batch"), ("plf_loop_closure_pose_batch", "loop_closure_pose_batch")):
        assert hasattr(lib, fn)
        assert callable(getattr(plf.Frontend, meth))
        assert getattr(lib, fn)(None, None, 0, None, None) == -1   # NULL context: PLF_ERR_INVALID, without a device


def test_problem_struct_layout(built, tmp_path):
    """sizeof and offsetof of every field, from a C program compiled against the header, equal the ctypes mirrors'."""
    import plslam_b200 as plf
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layout"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "plslam_b200.h"', "int main(void) {"]
    for st, fields in FIELDS.items():
        lines.append(f'  printf("{st} size %zu\\n", sizeof({st}));')
        lines += [f'  printf("{st} {f} %zu\\n", offsetof({st}, {f}));' for f in fields]
    lines.append("  return 0;\n}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c11", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {(a, b): int(c) for a, b, c in (ln.split() for ln in out if ln)}
    for st, fields in FIELDS.items():
        cls = getattr(plf, st)
        assert [f for f, _ in cls._fields_] == list(fields)
        assert got[(st, "size")] == C.sizeof(cls), st
        for f in fields:
            assert got[(st, f)] == getattr(cls, f).offset, (st, f)


@pytest.mark.parametrize("method", ["gn_pose_batch", "loop_closure_pose_batch"])
@pytest.mark.parametrize("seq,msg", [([0, 1], "3 entries"), (np.zeros((3, 1), np.int32), "3 entries"),
                                     (np.zeros(3, np.float64), "integer"), ([0, 1, 2 ** 40], "int32")])
def test_binding_refuses_a_malformed_seq(built, method, seq, msg):
    """The refusal comes before any library call: the Frontend here has no context (none can be created without a GPU),
    and the problems are never read."""
    import plslam_b200 as plf
    fe = object.__new__(plf.Frontend)
    with pytest.raises(plf.PlfError, match=msg):
        getattr(fe, method)([None, None, None], seq=seq)
