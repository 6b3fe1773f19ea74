"""CPU guard: every plf_params field is exercised somewhere.  A field must be varied by a case of tests/param_cases.py
(or named there as varied by another test), be listed as read-but-ignored (INVARIANT, whose tests assert the output does
not change), or be listed as accepting one value only (REJECTED, whose tests assert every other value is an error).  A new
parameter without coverage fails here."""
import numpy as np

import param_cases as pc
from oracle import frontend as ofe


def fields():
    import plslam_b200 as plf
    return [n for n, _ in plf.plf_params._fields_]


def test_every_plf_params_field_is_covered(built):
    varied = pc.varied_fields()
    uncovered = [f for f in fields() if f not in varied and f not in pc.INVARIANT and f not in pc.REJECTED]
    assert not uncovered, f"plf_params fields no test varies, checks for invariance or checks for rejection: {uncovered}"
    assert not set(pc.REJECTED) & varied, "a REJECTED field is run at a non-default value"
    assert not set(pc.INVARIANT) & set(pc.REJECTED)
    assert set(varied) | set(pc.INVARIANT) | set(pc.REJECTED) <= set(fields()), "a case names a field plf_params lacks"


def test_fields_varied_elsewhere_are_varied_there():
    """Each VARIED_ELSEWHERE entry names an existing test whose source sets the field."""
    import ast
    from pathlib import Path
    for field, where in pc.VARIED_ELSEWHERE.items():
        fname, test = where.split("::")
        src = (Path(__file__).parent / fname).read_text()
        fn = [n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == test]
        assert fn, f"{field}: {where} does not exist"
        body = ast.get_source_segment(src, fn[0])
        assert f"{field}=" in body, f"{field}: {where} does not set it"


def test_out_of_range_values_are_out_of_range():
    """OUT_OF_RANGE names fields that cases also run inside their range, and never a value a case runs."""
    varied = pc.varied_fields()
    for field, bad in pc.OUT_OF_RANGE.items():
        assert field in varied, field
        for case in [*pc.REFERENCE_CONFIGS.values(), *pc.ORB_CASES.values(), *pc.LSD_CASES.values()]:
            assert case.get(field) not in bad, (field, case)


def test_oracle_defaults_mirror_plf_default_params(built):
    """oracle/frontend.py DEFAULTS holds every field of plf_default_params() at the same value (f32 fields rounded)."""
    import ctypes as C

    import plslam_b200 as plf
    p = plf.default_params()
    assert set(ofe.DEFAULTS) == set(fields())
    for name, ctype in plf.plf_params._fields_:
        want = getattr(p, name)
        got = np.float32(ofe.DEFAULTS[name]) if ctype is C.c_float else ofe.DEFAULTS[name]
        assert got == want, name


def test_reference_configs_are_complete():
    """Each reference config names every front-end field; min_pt_matches / min_ls_matches come from SlamConfig, not
    from the config files."""
    want = set(ofe.DEFAULTS) - {"min_pt_matches", "min_ls_matches"}
    for name, cfg in pc.REFERENCE_CONFIGS.items():
        assert set(cfg) == want, name


def test_lsd_cases_cover_every_blur_kernel():
    """k_blur_q8_fast<5>, <7> and the generic k_blur_q8 at 3, 9, 11 and 15 taps all run in some LSD case."""
    sizes = {pc.lsd_ksize(dict(ofe.DEFAULTS, **c)) for c in pc.LSD_CASES.values()}
    assert {3, 5, 7, 9, 11, 15} <= sizes
