"""Several image sizes in one batched context where some sizes run the fused LSD pre-grow kernel and others the
three-kernel chain (blur, resample, gradient): the states of all sizes share one set of LSD buffers, so each size must
still find its own buffers in it.  At lsd_scale 0.95 with lsd_sigma_scale 0.45 (5 taps) the narrow sizes fit the fused
kernel's box and the wide ones do not.  Every pair must give, bit for bit, what its sequence gives alone on a context
created at its size (the oracle of tests/test_image_sizes_gpu.py)."""
import numpy as np
import pytest

import plslam_b200 as plf
from test_image_sizes_gpu import CAMS, SEQS, alone, assert_same, packed, schedule, size_of

pytestmark = pytest.mark.gpu

MIXED = dict(lsd_scale=0.95, lsd_sigma_scale=0.45)


def fused_sizes(**prm):
    with plf.Frontend(device=0, **prm) as fe:
        return {size_of(s): fe.debug_lsd_pre(np.zeros((1, size_of(s)[1], size_of(s)[0]), np.uint8), None)["fused_applies"]
                for s in SEQS}


def test_mixed_fused_and_chain_sizes_equal_each_sequence_alone(built):
    kinds = fused_sizes(**MIXED)
    assert any(kinds.values()) and not all(kinds.values()), kinds
    ref = alone(SEQS, per=2, **MIXED)
    got = packed(SEQS, schedule(SEQS), **MIXED)
    assert_same(ref, got)
    assert sum(v[0]["n_stereo_ls"] > 0 for v in got.values()) >= 0.7 * len(got)


def test_default_sizes_all_fused(built):
    assert all(fused_sizes().values())
