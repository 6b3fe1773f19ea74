#!/usr/bin/env python
"""bench_adaptive_fast.py - the cost of stvo-pl's adaptative_fast (plf_set_adaptive_fast) in the batched front-end.

With the adaptation on, pair k of a sequence is detected at the threshold pair k-1's pose gives, so a batch holds one pair
of each sequence and the extraction (E) phase of batch t+1 waits for batch t's threshold update at the end of its match
(M) phase.  Without it, E(t+1) overlaps M(t).  This script measures what that wait costs.

For each shape in --configs (bench.py's kitti and lowtex workloads: their camera, parameters and rendered streams) and each
N in --sequences (default 256, 1024), one context with max_sequences = N runs round-robin batches: B = N, seq = 0..N-1,
sequence c at step t seeing frame t of its trajectory (bench_multi_sequence.py's ping-pong rows).  Two batches are kept in
flight (upload + run of batch t, then download of batch t-1), the pattern of a streaming caller.  Arms: off (no
adaptation), on (the reference configs' fast_*_th: min 5, max 50, inc 5, feat 50, err 0.5), and wait (the adaptation on
with min_th = max_th = orb_fast_th: every threshold stays put, so the pairs are detected as with it off and the difference
from off is the cost of the E-after-M wait and the two small kernels alone).

Reported per arm: pairs/s over the --steps timed batches after --warmup, the fraction of the last batch's pairs that
tracked, and for "on" where the thresholds settle (a histogram of every sequence's threshold after the last batch).  The
GPU's name, power limit and SM clocks sampled during the timed regions are printed with the results.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench
from bench_multi_sequence import gpu_info, limits, pingpong_frames

CFG = dict(min_th=5, max_th=50, inc_th=5, feat_th=50, err_th=0.5)   # config_euroc.yaml:36-41


def pinned(prm):
    th = prm.get("orb_fast_th", 20)
    return dict(CFG, min_th=th, max_th=th)


def run_arm(plf, L, R, period, N, steps, warmup, cfg):
    frame = L[0].numel()
    ptr = lambda t, A: A.data_ptr() + (t % period) * frame
    seq = np.arange(N, dtype=np.int32)
    with plf.Frontend(camera=bench.CAM, limits=limits(plf, N), max_sequences=N, adaptive_fast=cfg, **bench.PRM) as fe:
        t0, res = None, None
        for t in range(warmup + steps):
            if t == warmup:
                fe.sync()
                t0 = time.perf_counter()
            fe.batch_upload_raw(N, ptr(t, L), ptr(t, R))
            fe.batch_run(N, seq=seq)
            if t > 0:
                res = fe.batch_download_array(N)
        res = fe.batch_download_array(N)
        dt = time.perf_counter() - t0
        out = dict(pairs_per_s=round(N * steps / dt, 1), ms_per_batch=round(dt * 1e3 / steps, 3),
                   tracked=float(np.mean(res["status"] == 0)))
        if cfg is not None:
            th = np.array([fe.sequence_fast_th(s) for s in range(N)])
            vals, counts = np.unique(th, return_counts=True)
            out["thresholds"] = {int(v): int(c) for v, c in zip(vals, counts)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["kitti", "lowtex"], choices=["kitti", "lowtex"])
    ap.add_argument("--sequences", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--steps", type=int, default=30, help="timed batches per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2, help="off / on / wait alternations per (config, N)")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_adaptive_fast.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        for name in args.configs:
            bench.select_config(name)
            pool = bench.render_pool(bench.CAM, 24, seed=0)
            L, R, period = pingpong_frames(torch, pool, max(args.sequences))
            for N in args.sequences:
                for rep in range(args.repeats):
                    for arm, cfg in (("off", None), ("on", CFG), ("wait", pinned(bench.PRM))):
                        r = run_arm(plf, L, R, period, N, args.steps, args.warmup, cfg)
                        print(json.dumps(dict(bench="adaptive_fast", config=name, sequences=N, repeat=rep, arm=arm, **r)),
                              flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
