"""Several image sizes in one batched context where the LSD pre-grow kernel cuts some sizes' row segments into one piece
and others' into two: the states of all sizes share one set of LSD buffers, so each size must still find its own buffers
in it.  At lsd_scale 0.95 with lsd_sigma_scale 0.45 (5 taps) the narrow sizes' segments fit one box and the wide ones'
do not.  Every pair must give, bit for bit, what its sequence gives alone on a context created at its size (the oracle of
tests/test_image_sizes_gpu.py)."""
import pytest

import plslam_b200 as plf
from test_image_sizes_gpu import SEQS, alone, assert_same, packed, schedule, size_of

pytestmark = pytest.mark.gpu

MIXED = dict(lsd_scale=0.95, lsd_sigma_scale=0.45)


def pieces(**prm):
    with plf.Frontend(device=0, **prm) as fe:
        return {size_of(s): fe.debug_lsd_pre_geometry(*size_of(s))["np"] for s in SEQS}


def test_mixed_piece_counts_equal_each_sequence_alone(built):
    kinds = pieces(**MIXED)
    assert set(kinds.values()) == {1, 2}, kinds
    ref = alone(SEQS, per=2, **MIXED)
    got = packed(SEQS, schedule(SEQS), **MIXED)
    assert_same(ref, got)
    assert sum(v[0]["n_stereo_ls"] > 0 for v in got.values()) >= 0.7 * len(got)


def test_default_sizes_one_piece(built):
    assert set(pieces().values()) == {1}
