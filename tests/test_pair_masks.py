"""CPU tests of the pair-mask cases (tests/pair_mask_cases.py) the GPU tests of plf_batch_upload_masks run.

- The AND of a pair mask and a sequence mask is one mask: its cv2 pyramid (the one detectAndCompute applies) is the
  pyramid built from the ANDed level 0, and on the sparse pair an AND of the two masks' pyramids is another mask.
- The moving masks remove keypoints and cut lines in the rendered frames, so the GPU tests compare masked detection."""
import numpy as np
import pytest

import pair_mask_cases as pm
from oracle import cvref
from oracle import frontend as ofe
from oracle import masks as om

cv2 = pytest.importorskip("cv2")

KITTI = dict(width=1242, height=375, fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, b=0.537165719)
EUROC = dict(width=752, height=480, fx=458.654, fy=457.296, cx=367.215, cy=248.375, b=0.110077842)


@pytest.mark.parametrize("cam", [KITTI, EUROC], ids=["kitti", "euroc"])
@pytest.mark.parametrize("nlevels", [1, 4, 8])
def test_anded_mask_pyramid_is_cv2s(cam, nlevels):
    """detectAndCompute(img, S & P) keeps exactly the unmasked keypoints on a non-zero pixel of the pyramid built from
    S & P (no retainBest cut)."""
    h, w = cam["height"], cam["width"]
    img = pm.streams(cam, 1, 1)[0][0][0]
    N = 200000
    full, _ = cvref.orb_cv2(img, N, 1.2, nlevels)
    for S, P in ((pm.hood(h, w), pm.moving(h, w, 2, 0)), pm.sparse_pair(h, w)):
        m = S & P
        pyr = pm.mask_pyramid(m, nlevels)
        got, _ = om.orb(img, m, N, 1.2, nlevels)
        on = [pyr[k["octave"]][int(np.round(k["y"] / np.float32(1.2 ** int(k["octave"])))),
                                int(np.round(k["x"] / np.float32(1.2 ** int(k["octave"]))))] != 0 for k in full]
        ref = full[np.array(on, bool)]
        assert got[["x", "y", "octave"]].tobytes() == ref[["x", "y", "octave"]].tobytes()


def test_and_of_pyramids_is_another_mask():
    h, w = KITTI["height"], KITTI["width"]
    S, P = pm.sparse_pair(h, w)
    ps, pp, pa = pm.mask_pyramid(S, 4), pm.mask_pyramid(P, 4), pm.mask_pyramid(S & P, 4)
    assert all(np.array_equal(a, b) for a, b in zip(pa[:3], [x & y for x, y in zip(ps, pp)][:3]))
    diff = (ps[3] & pp[3]) != pa[3]
    assert diff.any()
    assert not pa[3][diff].any()   # the AND's pyramid masks them; the pyramids' AND allows them
    # the hood and a moving mask meet on wide edges only: there the two agree on every level
    H, M = pm.hood(h, w), pm.moving(h, w, 3, 1)
    assert all(np.array_equal(a & b, c) for a, b, c in zip(pm.mask_pyramid(H, 4), pm.mask_pyramid(M, 4), pm.mask_pyramid(H & M, 4)))


@pytest.mark.parametrize("cam", [KITTI, EUROC], ids=["kitti", "euroc"])
def test_moving_masks_remove_keypoints_and_lines(cam):
    h, w = cam["height"], cam["width"]
    prm = dict(ofe.DEFAULTS, orb_nfeatures=1500, lsd_nfeatures=200)
    frames = pm.streams(cam, 1, 5)[0]
    for i in (0, 4):
        for side in (0, 1):
            img, m = frames[i][side], pm.moving(h, w, i, side)
            kp, _ = ofe._orb_c(img, prm)
            mk, _ = om.orb(img, m, prm["orb_nfeatures"], 1.2, prm["orb_nlevels"])
            on = m[np.round(kp["y"]).astype(int), np.round(kp["x"]).astype(int)] == 0
            assert on.sum() >= 10 and not (m[np.round(mk["y"]).astype(int), np.round(mk["x"]).astype(int)] == 0).all()
            assert not np.array_equal(kp[["x", "y"]], mk[["x", "y"]])
            kl, _ = ofe.detect_lines(img, 0, prm["min_line_length"], ofe.lsd_kwargs(prm))
            kept = om.mask_keylines(kl, m)
            assert 0 < len(kept) < len(kl)
