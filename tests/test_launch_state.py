"""CPU test (static): every launch is described by its call.  A launch helper takes its stream as an argument instead of
reading a current stream from the context, and a kernel reads no device table that a context writes at run time: tables
are compiled in (an initialised __constant__ or __device__ array) or passed with the launch, so contexts with different
parameters, or on different devices, can be alive in one process at once."""
import re
from pathlib import Path

CSRC = Path(__file__).resolve().parents[1] / "pl-slam_b200" / "csrc"


def sources():
    return sorted(p for p in CSRC.iterdir() if p.suffix in (".cu", ".h", ".cuh"))


def code(path):
    """The source text without comments."""
    text = re.sub(r"/\*.*?\*/", " ", path.read_text(), flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def struct_body(text, name):
    m = re.search(r"\bstruct\s+" + name + r"\s*\{", text)
    assert m, name
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[m.end():i - 1]


def test_context_holds_no_launch_state():
    body = struct_body(code(CSRC / "plf_internal.h"), "plf_ctx")
    members = re.findall(r"(\w+)\s*(?:\[[^\]]*\])?\s*(?:=[^;]*)?;", body)
    assert "stream" in members, members
    assert "cur" not in members and "lbd_tables" not in members, members


def test_no_current_stream_is_read():
    for src in sources():
        assert not re.search(r"->\s*cur\b", code(src)), src.name


def test_no_table_is_uploaded_at_run_time():
    for src in sources():
        text = code(src)
        assert "cudaMemcpyToSymbol" not in text, src.name
        assert not re.search(r'getenv\(\s*"PLF_G_PRIORITY"\s*\)', text), src.name


def test_every_constant_is_initialised():
    n = 0
    for src in sources():
        for m in re.finditer(r"__constant__[^;=]*([;=])", code(src)):
            n += 1
            assert m.group(1) == "=", f"{src.name}: {m.group(0)!r} has no initializer"
    assert n > 0


def test_no_namespace_scope_static_pointer():
    # a host-side static holding a device pointer is process-wide state that no context owns
    pattern = re.compile(r"^static\s+(?:const\s+)?[\w:<>]+(?:\s+const)?\s*\*+\s*(?:const\s+)?\w+\s*(?:=[^;]*)?;", re.M)
    for src in sources():
        m = pattern.search(code(src))
        assert not m, f"{src.name}: {m.group(0)!r}"
