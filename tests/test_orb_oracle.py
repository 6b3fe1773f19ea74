"""CPU tests: the C restatement of OpenCV's ORB pinned bit-exact against cv2 4.13 (live) and the golden."""
from pathlib import Path

import numpy as np
import pytest

import param_cases as pc
from oracle import clib, synth
from oracle import frontend as ofe
from oracle.cvref import orb_cv2

GOLD = Path(__file__).parent / "golden" / "orb_v1.npz"
FIELDS = ["x", "y", "size", "angle", "response", "octave"]


def same_kps(a, b):
    return len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in FIELDS)


@pytest.mark.parametrize("name,nf", [("l", 800), ("r", 800), ("l", 300), ("r", 300)])
def test_oracle_matches_golden(name, nf):
    g = np.load(GOLD)
    img = g["left"] if name == "l" else g["right"]
    kp, desc = clib.orb(img, nf)
    assert same_kps(kp, g[f"kp_{name}_{nf}"])
    assert np.array_equal(desc, g[f"desc_{name}_{nf}"])


def test_oracle_matches_cv2_live_full_size():
    pytest.importorskip("cv2")
    L, R = synth.scene_pair()
    for img in (L, R):
        kp, desc = clib.orb(img, 1500)
        rk, rd = orb_cv2(img, nfeatures=1500)
        assert same_kps(kp, rk) and np.array_equal(desc, rd)


def test_resize_exact_vs_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    for (sw, sh, dw, dh) in [(1242, 375, 1035, 312), (1035, 312, 862, 260), (752, 480, 627, 400), (53, 37, 64, 44)]:
        img = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        assert np.array_equal(clib.resize_linear_exact(img, dw, dh),
                              cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR_EXACT))


def test_fast_atan2_vs_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    for _ in range(2000):
        y, x = (float(v) for v in rng.integers(-200000, 200000, 2))
        assert np.float32(clib.fast_atan2(y, x)) == np.float32(cv2.fastAtan2(y, x))
    assert clib.fast_atan2(0.0, 0.0) == cv2.fastAtan2(0.0, 0.0)


@pytest.mark.parametrize("case", sorted(pc.ORB_CASES))
def test_oracle_matches_cv2_param_cases(case):
    """The ORB settings of tests/param_cases.py: the C restatement, called as the oracle front-end calls it, equals cv2."""
    pytest.importorskip("cv2")
    prm = dict(ofe.DEFAULTS, **pc.ORB_CASES[case])
    L, _ = synth.scene_pair(w=640, h=360, seed=3)
    kp, desc = ofe._orb_c(L, prm)
    rk, rd = orb_cv2(L, prm["orb_nfeatures"], prm["orb_scale_factor"], prm["orb_nlevels"], prm["orb_edge_th"],
                     prm["orb_wta_k"], prm["orb_patch_size"], prm["orb_fast_th"])
    assert len(rk) > 100 and same_kps(kp, rk) and np.array_equal(desc, rd)
