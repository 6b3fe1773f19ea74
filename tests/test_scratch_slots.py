"""CPU test (static): the per-call device scratch of the operator entry points is taken only through the named slots of
plf_internal.h (enum plf_scratch_slot), and the 256-byte rounding of sub-allocations is written once, as plf_align256."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parents[1] / "pl-slam_b200" / "csrc"


def call_args(text, name):
    """(line, [top-level arguments]) of every call or definition `name(...)` in text."""
    out = []
    for m in re.finditer(r"\b" + re.escape(name) + r"\(", text):
        depth, args, cur = 1, [], ""
        for ch in text[m.end():]:
            if ch in "([{":
                depth += 1
            elif ch in ")]}":
                depth -= 1
                if depth == 0:
                    break
            if ch == "," and depth == 1:
                args.append(cur.strip())
                cur = ""
            else:
                cur += ch
        args.append(cur.strip())
        out.append((text.count("\n", 0, m.start()) + 1, args))
    return out


# a slot is named (PLF_SCR_*) or forwarded in a variable of the enum type; the definitions declare it as that type
SLOT = re.compile(r"(plf_scratch_slot\s+)?(PLF_SCR_[A-Z_]+|([A-Za-z_]\w*\.)?slot)")


def test_every_scratch_call_names_its_slot():
    seen = {"plf_scratch": 0, "carve": 0, "plf_launch_match_grid_batch": 0}
    for src in sorted(CSRC.glob("*.cu")):
        text = src.read_text()
        for name, pos in (("plf_scratch", 1), ("carve", 1), ("plf_launch_match_grid_batch", 5)):
            for line, args in call_args(text, name):
                seen[name] += 1
                assert len(args) > pos and SLOT.fullmatch(args[pos]), f"{src.name}:{line}: {name} slot {args[pos:pos + 1]}"
    assert all(seen.values()), seen


def test_the_256_byte_rounding_is_written_once():
    for src in sorted(CSRC.iterdir()):
        if src.name != "plf_internal.h":
            assert "& ~size_t(255)" not in src.read_text(), src.name
    assert "& ~size_t(255)" in (CSRC / "plf_internal.h").read_text()
