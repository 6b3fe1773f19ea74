"""CPU tests of the per-sequence camera interface: the header declares plf_set_sequence_camera / plf_get_sequence_camera,
the library exports them, and the binding exposes them on Frontend."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_sequence_camera_symbols(built):
    import plslam_b200 as plf
    hdr = (ROOT / "include" / "plslam_b200.h").read_text()
    assert re.search(r"plf_status plf_set_sequence_camera\(plf_ctx\* ctx, int s, const plf_camera\* cam\);", hdr)
    assert re.search(r"plf_status plf_get_sequence_camera\(const plf_ctx\* ctx, int s, plf_camera\* out\);", hdr)
    lib = plf.load_library()
    assert hasattr(lib, "plf_set_sequence_camera") and hasattr(lib, "plf_get_sequence_camera")
    assert callable(plf.Frontend.set_sequence_camera) and callable(plf.Frontend.sequence_camera)
    # NULL context: PLF_ERR_INVALID, without a device
    assert lib.plf_set_sequence_camera(None, 0, None) == -1
    assert lib.plf_get_sequence_camera(None, 0, None) == -1
