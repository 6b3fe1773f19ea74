#!/usr/bin/env python
"""bench_masks.py - the cost of per-sequence detector masks (plf_set_sequence_mask) in the batched front-end.

KITTI shape (1242 x 375), B = --batch pairs of bench.py's rendered stream, resident on the device (uploaded once), each
pair of its own sequence (seq = 0 .. B-1, one pair of every sequence per batch, up to three batches in flight).  Arms,
alternated --repeats times in one context:
  none    no sequence has a mask: the unmasked kernels, as bench.py runs them
  half    every image masked by a half-image mask (the left half allowed): the masked kernels, and fewer features
  all255  every image masked by an all-255 mask: the masked kernels with the feature counts of `none`, which isolates the
          cost of reading the masks from the change in feature counts
Reported: pairs/s and launches per step per arm, the mean keypoints and lines per image, and the one-time
plf_set_sequence_mask cost (ms per call, both images, the pyramid built on the device).  The GPU's name, power limit and
clocks are printed with the results.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench
from bench_color import fill, timed
from bench_multi_sequence import gpu_info, limits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3, help="alternations of the arms")
    ap.add_argument("--pool", type=int, default=12, help="rendered pairs")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_masks.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    cam, B = bench.CAM, args.batch
    h, w = cam["height"], cam["width"]
    L, R = fill(torch, bench.render_pool(cam, args.pool, seed=0), B, 1)
    seq = np.arange(B, dtype=np.int32)
    xx = np.arange(w)[None, :].repeat(h, 0)
    arms = {"none": None, "half": np.where(xx < w // 2, 255, 0).astype(np.uint8), "all255": np.full((h, w), 255, np.uint8)}
    sampler = bench.ClockSampler(0)
    sampler.start()
    try:
        with plf.Frontend(camera=cam, limits=limits(plf, B), max_sequences=B, **bench.PRM) as fe:
            fe.batch_upload_raw(B, L.data_ptr(), R.data_ptr())
            for rep in range(args.repeats):
                for arm, m in arms.items():
                    fe.sync()
                    t0 = time.perf_counter()
                    for s in range(B):
                        fe.set_sequence_mask(s, m, m)
                    set_ms = (time.perf_counter() - t0) * 1e3 / B
                    r = timed(fe, B, args.steps, args.warmup, None, seq)
                    n0 = fe.launches
                    fe.batch_run(B, seq=seq)
                    res = fe.batch_download_array(B)
                    launches = fe.launches - n0
                    print(json.dumps(dict(bench="masks", arm=arm, batch=B, width=w, height=h, repeat=rep, **r,
                                          launches_per_step=launches,
                                          kp_per_image=round(float((res["n_kp_l"] + res["n_kp_r"]).mean()) / 2, 1),
                                          lines_per_image=round(float((res["n_lines_l"] + res["n_lines_r"]).mean()) / 2, 1),
                                          set_mask_ms_per_call=round(set_ms, 3) if m is not None else None)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
