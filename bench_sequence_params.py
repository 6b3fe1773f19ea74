#!/usr/bin/env python
"""bench_sequence_params.py - KITTI-config and EuRoC-config recordings in one batched context (plf_set_sequence_params).

pl-slam's config_kitti.yaml and config_euroc.yaml differ in lsd_nfeatures, max_dist_epip, max_iters, max_iters_ref,
min_ratio_12_p and matching_strategy (KITTI below; EuRoC is the library's defaults with matching_strategy 3).  Each arm
runs --steps batches of B pairs at the KITTI shape, uploaded from pinned host memory every step, each pair of its own
sequence, half of the sequences with each config, up to three batches in flight:
  packed    one context of the EuRoC config whose first B / 2 sequences have the KITTI config: every batch holds both
  two       one context per config at B / 2 each, today's only way to run both configs; a step issues one batch on each
Reported per arm: pairs/s and the device memory in use once the pipelines exist (total - free, as cudaMemGetInfo reports
it).  The arms are alternated --repeats times.  The GPU's name, power limit and clocks are printed with the results.
"""
import argparse
import json
import sys

import numpy as np

import bench
from bench_color import fill
from bench_image_sizes import hbm_used, run_steps
from bench_multi_sequence import gpu_info, limits

SIZE = (1242, 375)
KITTI = dict(lsd_nfeatures=100, max_dist_epip=0.0, max_iters=100, max_iters_ref=100, min_ratio_12_p=0.75, matching_strategy=0)
EUROC = dict(matching_strategy=3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=2, help="alternations of the arms")
    ap.add_argument("--pool", type=int, default=6, help="rendered pairs")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequence_params.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    B, h = args.batch, args.batch // 2
    L, R = fill(torch, bench.render_pool(bench.CAM, args.pool, seed=0), B, 1)
    sampler = bench.ClockSampler(0)
    sampler.start()
    try:
        def packed():
            fe = plf.Frontend(camera=bench.CAM, limits=limits(plf, B), max_sequences=B, **dict(bench.PRM, **EUROC))
            for s in range(h):
                fe.set_sequence_params(s, **dict(bench.PRM, **KITTI))
            return [fe], [(fe, B, SIZE, L, R, np.arange(B, dtype=np.int32), True)]

        def two():
            fes = [plf.Frontend(camera=bench.CAM, limits=limits(plf, h), max_sequences=h, **dict(bench.PRM, **cfg))
                   for cfg in (KITTI, EUROC)]
            return fes, [(fe, h, SIZE, L, R, np.arange(h, dtype=np.int32), True) for fe in fes]

        for rep in range(args.repeats):
            for arm, make in (("packed", packed), ("two", two)):
                fes, ctxs = make()
                try:
                    for fe in fes:
                        fe.device_layout   # builds the pipeline
                    used = hbm_used(torch)
                    run_steps(torch, ctxs, args.warmup)
                    r = run_steps(torch, ctxs, args.steps)
                    print(json.dumps(dict(bench="sequence_params", arm=arm, batch=B, contexts=len(fes), repeat=rep,
                                          pairs_per_s=r["pairs_per_s"], hbm_used_GiB=used)), flush=True)
                finally:
                    for fe in fes:
                        fe.close()
                    torch.cuda.synchronize()
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
