"""The round-count replay of the LSD region growing (oracle/tools/grow_rounds_sim.py): handling 1, 2 or 3 queue entries
per round grows the same regions in the same order, and larger rounds shorten the chain (CPU simulation on a small crop
of the bench frame)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "oracle" / "tools"))


def test_round_sizes_keep_the_partition():
    pytest.importorskip("cv2")
    import grow_rounds_sim as sim
    import plslam_b200 as plf
    from plslam_b200 import synth
    L = next(iter(synth.stream(plf.KITTI_CAMERA, 1, world=synth.World(seed=7), seed=42)))[0]
    flat, seeds, W = sim.angle_map_deg(np.ascontiguousarray(L[100:260, 300:560]))
    c1, ref = sim.grow(flat, seeds, W, 1)
    assert len(ref) > 100 and sum(len(q) for q in ref) == len(seeds)   # every defined pixel in exactly one region
    prev = c1
    for n in (2, 3):
        c, regs = sim.grow(flat, seeds, W, n)
        assert regs == ref
        assert c["accept"] == c1["accept"] and c["starts"] == c1["starts"]
        assert c["rounds"] < prev["rounds"] and c["chain"] < prev["chain"]
        prev = c
