"""CPU test (static): the batched pipeline and the standalone detectors each own their ORB and LSD working state.  The
context holds no state that both use (no plf_ctx::orb / lsd, no lsd_keylines_wait hand-off), no translation unit reads
one, and a state no longer keeps a second batch parity just because an earlier owner asked for it."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parents[1] / "pl-slam_b200" / "csrc"


def struct_body(text, name):
    m = re.search(r"\bstruct\s+" + name + r"\s*\{", text)
    assert m, name
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[m.end():i - 1]


def test_context_holds_no_shared_detector_state():
    body = struct_body((CSRC / "plf_internal.h").read_text(), "plf_ctx")
    members = re.findall(r"(\w+)\s*(?:=[^;]*)?;", body)
    assert "orb" not in members and "lsd" not in members, members
    assert "lsd_keylines_wait" not in body


def test_no_translation_unit_reads_a_context_detector_state():
    for src in sorted(CSRC.glob("*.cu")):
        assert not re.search(r"ctx->(orb|lsd)\b", src.read_text()), src.name


def test_no_sticky_parities():
    for src in sorted(CSRC.glob("*.cu")):
        text = src.read_text()
        assert not re.search(r"if\s*\(\s*s\s*&&\s*s->two_parities\s*\)\s*two_parities\s*=\s*true", text), src.name
