#!/usr/bin/env python
"""bench_motion_model.py - what stvo-pl's use_motion_model (plf_set_motion_model) changes in the batched front-end.

With the model on, each sequence's next pair starts from the prediction its last pair gave: the windowed frame-to-frame
matching (matching_strategy != 0) projects the previous frame through it, and the pose solver is seeded with it.  A
batch holds one pair of each sequence; the predictions are written and read on the match (M) stream, so no wait is added.

For each --strategies value (matching_strategy, default 0 and 3) and each N in --sequences (default 256, 1024), one
context at bench.py's kitti shape with max_sequences = N runs round-robin batches: B = N, seq = 0..N-1, sequence c at
step t seeing frame t of its trajectory (bench_multi_sequence.py's ping-pong rows; the trajectory turns back at both ends
of the rendered pool, where a constant-motion prediction points the wrong way).  Two batches are kept in flight.  Arms:
off and on.  Reported per arm: pairs/s over the --steps timed batches after --warmup, the fraction of tracked pairs, the
mean GN iterations (iters1 + iters2) and frame-to-frame point matches per tracked pair of the timed batches.

With a windowed strategy the oracle (oracle/frontend.py run_sequence, on the CPU) also runs --oracle-pairs consecutive
pairs of one camera off and on, and reports the windowed point matches per tracked pair and how many pairs fall back to
match().  The GPU's name, power limit and SM clocks sampled during the timed regions are printed with the results.
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

import bench
from bench_multi_sequence import gpu_info, limits, pingpong_frames

sys.path.insert(0, str(Path(__file__).resolve().parent / "tests"))


def run_arm(plf, L, R, period, N, steps, warmup, strategy, on):
    frame = L[0].numel()
    ptr = lambda t, A: A.data_ptr() + (t % period) * frame
    seq = np.arange(N, dtype=np.int32)
    prm = dict(bench.PRM, matching_strategy=strategy)
    timed = []
    with plf.Frontend(camera=bench.CAM, limits=limits(plf, N), max_sequences=N, motion_model=on, **prm) as fe:
        t0 = None
        for t in range(warmup + steps):
            if t == warmup:
                fe.sync()
                t0 = time.perf_counter()
            fe.batch_upload_raw(N, ptr(t, L), ptr(t, R))
            fe.batch_run(N, seq=seq)
            if t > 0:
                res = fe.batch_download_array(N)
                if t > warmup:
                    timed.append(res)
        timed.append(fe.batch_download_array(N))
        dt = time.perf_counter() - t0
    res = np.concatenate(timed)
    ok = res["status"] == 0
    return dict(pairs_per_s=round(N * steps / dt, 1), ms_per_batch=round(dt * 1e3 / steps, 3), tracked=float(np.mean(ok)),
                gn_iters=round(float(np.mean(res["iters1"][ok] + res["iters2"][ok])), 3),
                f2f_pt_matches=round(float(np.mean(res["n_matched_pt"][ok])), 1))


def oracle_counts(pool, n, strategy):
    """The oracle on the first n pairs of one camera's ping-pong order, off (identity predictions) and on: windowed
    point matches per tracked pair, pairs that fall back to match(), and GN iterations per tracked pair."""
    from oracle import frontend as ofe
    pairs = [pool[i] for i in (list(range(len(pool))) + list(range(len(pool) - 2, 0, -1)))[:n]]
    prm = dict(ofe.DEFAULTS, **bench.PRM, matching_strategy=strategy)
    frames = [ofe.extract_stereo(bench.CAM, L, R, prm) for L, R in pairs]
    out = {}
    for arm in ("off", "on"):
        preds = [np.eye(4)] * n if arm == "off" else None   # identity predictions: the off pipeline (finite points)
        r = [o for o in ofe.run_sequence(bench.CAM, pairs, prm, motion_model=True, preds=preds, frames=frames) if o["status"] == 0]
        out[arm] = dict(tracked=len(r), pt_window=round(float(np.mean([o["stats"]["pt_window"] for o in r])), 1),
                        pt_fallback=sum(o["stats"]["pt_fallback"] for o in r),
                        gn_iters=round(float(np.mean([sum(o["res"]["iters"]) for o in r])), 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strategies", type=int, nargs="+", default=[0, 3])
    ap.add_argument("--sequences", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--steps", type=int, default=30, help="timed batches per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2, help="off / on alternations per (strategy, N)")
    ap.add_argument("--oracle-pairs", type=int, default=8, help="consecutive pairs the CPU oracle runs (0: none)")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_motion_model.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    bench.select_config("kitti")
    pool = bench.render_pool(bench.CAM, 24, seed=0)
    L, R, period = pingpong_frames(torch, pool, max(args.sequences))
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        for strategy in args.strategies:
            for N in args.sequences:
                for rep in range(args.repeats):
                    for arm in ("off", "on"):
                        r = run_arm(plf, L, R, period, N, args.steps, args.warmup, strategy, arm == "on")
                        print(json.dumps(dict(bench="motion_model", config="kitti", strategy=strategy, sequences=N, repeat=rep,
                                              arm=arm, **r)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)
    if args.oracle_pairs > 1:
        for strategy in args.strategies:
            if strategy:
                print(json.dumps(dict(bench="motion_model_oracle", config="kitti", strategy=strategy, pairs=args.oracle_pairs,
                                      **oracle_counts(pool, args.oracle_pairs, strategy))), flush=True)


if __name__ == "__main__":
    sys.exit(main())
