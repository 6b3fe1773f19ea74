"""CPU tests: the C restatement of OpenCV's LSD (refine = 0) pinned bit-exact — same segments, same order —
against cv2 4.13 (live) and the committed golden segments (tests/golden/lines_v1.npz was produced by cv2)."""
from pathlib import Path

import numpy as np
import pytest

import param_cases as pc
from oracle import clib, synth
from oracle import frontend as ofe
from oracle.cvref import lsd_cv2

GOLD = Path(__file__).parent / "golden" / "lines_v1.npz"


def test_lsd_oracle_matches_golden_cv2_segments():
    g = np.load(GOLD)
    for trig in (0, 1):
        segs = clib.lsd(g["left"], trig_mode=trig)
        assert segs.shape == g["segs"].shape and np.array_equal(segs, g["segs"])


@pytest.mark.parametrize("w,h,seed", [(1242, 375, 1), (752, 480, 9), (640, 360, 33)])
def test_lsd_oracle_matches_cv2_live(w, h, seed):
    pytest.importorskip("cv2")
    L, R = synth.scene_pair(w=w, h=h, seed=seed)
    for img in (L, R):
        ref = lsd_cv2(img)
        mine = clib.lsd(img)
        assert len(ref) > 100 and mine.shape == ref.shape and np.array_equal(mine, ref)


def test_lsd_scale_variants_vs_cv2():
    """scale 0.8 (OpenCV default; sigma = 0.6/0.8) and scale 1.0 (no resample) also match."""
    pytest.importorskip("cv2")
    L, _ = synth.scene_pair(w=500, h=300, seed=12, n_rect=80, n_lines=40)
    for sc in (0.8, 1.0):
        ref = lsd_cv2(L, scale=sc)
        mine = clib.lsd(L, scale=sc)
        assert mine.shape == ref.shape and np.array_equal(mine, ref)


def test_lsd_flat_image_has_no_segments():
    assert len(clib.lsd(np.full((100, 150), 90, np.uint8))) == 0


@pytest.mark.parametrize("case", sorted(pc.LSD_CASES))
def test_lsd_oracle_matches_cv2_param_cases(case):
    """The LSD settings of tests/param_cases.py (Gaussian kernels of 3 to 15 taps, quantisation, angle tolerance, bins)."""
    pytest.importorskip("cv2")
    prm = dict(ofe.DEFAULTS, **pc.LSD_CASES[case])
    L, _ = synth.scene_pair(w=640, h=360, seed=3)
    ref = lsd_cv2(L, scale=prm["lsd_scale"], sigma_scale=prm["lsd_sigma_scale"], quant=prm["lsd_quant"],
                  ang_th=prm["lsd_ang_th"], n_bins=prm["lsd_n_bins"])
    mine = clib.lsd(L, **ofe.lsd_kwargs(prm))
    assert len(ref) > 50 and mine.shape == ref.shape and np.array_equal(mine, ref)


def test_lsd_log_eps_density_th_have_no_effect_in_cv2():
    """Without refinement cv2 ignores log_eps and density_th, which is why the library may ignore them."""
    pytest.importorskip("cv2")
    L, _ = synth.scene_pair(w=640, h=360, seed=3)
    ref = lsd_cv2(L)
    for kw in (dict(log_eps=pc.INVARIANT["lsd_log_eps"]), dict(density_th=pc.INVARIANT["lsd_density_th"]),
               dict(log_eps=-2.0, density_th=0.1)):
        assert np.array_equal(lsd_cv2(L, **kw), ref), kw
