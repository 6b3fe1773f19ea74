#!/usr/bin/env python
"""bench_multi_sequence.py - several stereo sequences through one front-end context (plf_batch_run_sequences).

At KITTI shape with bench.py's limits and parameters (1242x375, orb_nfeatures 1500, lsd_nfeatures 200, 4096 keypoints,
8192 segments, 1024 lines per image), on one GPU:

  1. live cameras: N cameras deliver one stereo pair each per step, for N in --cameras (default 1, 8, 64).  One context
     with max_sequences = N runs the N pairs as one batch (B = N, seq = 0..N-1) against N single-sequence contexts at
     B = 1, all uploaded and run before the first is downloaded (each context has its own streams, so their chains may
     overlap on the device).  A step = upload + run + download of every camera's pair; it ends with the downloads, which
     wait for the device.  Reported: pairs/s over the timed steps and the median / p90 step latency, from the host clock
     around each step (--steps after --warmup).
  2. packed recordings: B = 1024 as 8 sequences x 128 pairs (seq[k] = k // 128) against 1 sequence x 1024, the same
     images, in one context with max_sequences = 8, alternated --rounds times.  The batch stays resident in HBM and up to
     three batches are in flight, as bench.py's `value`; device time from CUDA events on the library's stream.

Camera c at step t shows frame t + c of bench.py's ping-pong over its rendered frames, so every camera follows a
trajectory and the per-image work matches bench.py's.  Prints the GPU's name, power limit and SM clocks sampled during
the timed regions, then one JSON line per measurement.
"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

import bench   # KITTI configuration, rendering, clock sampling (bench.py itself is not run)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, sm_max=sm_max)
    except Exception as e:   # the measurement still stands; the card is then named "unknown"
        return dict(name="unknown", error=str(e))


def pingpong_frames(torch, pool, n_extra):
    """Pinned [period + n_extra][h][w] left / right stacks of the ping-pong order, so rows t .. t + n - 1 (t < period) are
    n cameras' frames at step t, contiguous, and row t + c + 1 follows row t + c on camera c's trajectory."""
    n = len(pool)
    period = list(range(n)) + list(range(n - 2, 0, -1))
    rows = len(period) + n_extra
    h, w = pool[0][0].shape
    L = torch.empty((rows, h, w), dtype=torch.uint8, pin_memory=True)
    R = torch.empty((rows, h, w), dtype=torch.uint8, pin_memory=True)
    for j in range(rows):
        L[j].numpy()[:] = pool[period[j % len(period)]][0]
        R[j].numpy()[:] = pool[period[j % len(period)]][1]
    return L, R, len(period)


def limits(plf, B):
    lim = plf.default_limits()
    lim.max_batch = B; lim.max_keypoints = 4096; lim.max_segments = 8192; lim.max_lines = 1024
    return lim


def latency_stats(ms, pairs):
    ms = np.asarray(ms)
    return dict(pairs_per_s=round(pairs * len(ms) / (ms.sum() * 1e-3), 1), median_ms=round(float(np.median(ms)), 3),
                p90_ms=round(float(np.percentile(ms, 90)), 3))


def live_cameras(plf, L, R, period, N, steps, warmup):
    frame = L[0].numel()
    ptr = lambda t, A: A.data_ptr() + (t % period) * frame
    seq = np.arange(N, dtype=np.int32)
    out = {}
    with plf.Frontend(camera=bench.CAM, limits=limits(plf, N), max_sequences=N, **bench.PRM) as fe:
        ms = []
        for t in range(warmup + steps):
            t0 = time.perf_counter()
            fe.batch_upload_raw(N, ptr(t, L), ptr(t, R))
            fe.batch_run(N, seq=seq)
            res = fe.batch_download_array(N)
            if t >= warmup:
                ms.append((time.perf_counter() - t0) * 1e3)
        out["one_context"] = dict(latency_stats(ms, N), tracked=float(np.mean(res["status"] == 0)))
    fes = [plf.Frontend(camera=bench.CAM, limits=limits(plf, 1), **bench.PRM) for _ in range(N)]
    try:
        ms = []
        for t in range(warmup + steps):
            t0 = time.perf_counter()
            for c, fe in enumerate(fes):
                fe.batch_upload_raw(1, ptr(t, L) + c * frame, ptr(t, R) + c * frame)
                fe.batch_run(1)
            res = np.concatenate([fe.batch_download_array(1) for fe in fes])
            if t >= warmup:
                ms.append((time.perf_counter() - t0) * 1e3)
        out["n_contexts"] = dict(latency_stats(ms, N), tracked=float(np.mean(res["status"] == 0)))
    finally:
        for fe in fes:
            fe.close()
    return out


def packed(torch, plf, pool, steps, rounds):
    B, n_seq = 1024, 8
    h, w = bench.CAM["height"], bench.CAM["width"]
    hostL = torch.empty((B, h, w), dtype=torch.uint8, pin_memory=True)
    hostR = torch.empty((B, h, w), dtype=torch.uint8, pin_memory=True)
    bench.fill_batch(pool, B, hostL.numpy(), hostR.numpy())
    variants = {"1x1024": None, "8x128": (np.arange(B) // (B // n_seq)).astype(np.int32)}
    times = {k: [] for k in variants}
    with plf.Frontend(camera=bench.CAM, limits=limits(plf, B), max_sequences=n_seq, **bench.PRM) as fe:
        fe.batch_upload_raw(B, hostL.data_ptr(), hostR.data_ptr())
        ext = torch.cuda.ExternalStream(fe.stream)
        for name, seq in variants.items():   # warm-up of both
            for _ in range(3):
                fe.batch_run(B, seq=seq)
                fe.batch_download_array(B)
        for _ in range(rounds):
            for name, seq in variants.items():
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(ext)
                for _ in range(min(3, steps)):
                    fe.batch_run(B, seq=seq)
                for _ in range(steps - min(3, steps)):
                    fe.batch_download_array(B)
                    fe.batch_run(B, seq=seq)
                for _ in range(min(3, steps)):
                    fe.batch_download_array(B)
                e1.record(ext)
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) / steps)
    return {k: dict(ms_per_step=[round(x, 2) for x in v], median_ms=round(float(np.median(v)), 2),
                    pairs_per_s=round(B / (float(np.median(v)) * 1e-3), 1)) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--steps", type=int, default=200, help="timed steps per live-camera arm")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--packed-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two packed variants")
    ap.add_argument("--skip-packed", action="store_true")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_sequence.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    pool = bench.render_pool(bench.CAM, 24, seed=0)
    L, R, period = pingpong_frames(torch, pool, max(args.cameras))
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        for N in args.cameras:
            r = live_cameras(plf, L, R, period, N, args.steps, args.warmup)
            print(json.dumps(dict(bench="live_cameras", cameras=N, steps=args.steps, **r)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", part="live_cameras", gpu=info, **clocks)), flush=True)
    if not args.skip_packed:
        sampler = bench.ClockSampler(0)
        sampler.start()
        try:
            r = packed(torch, plf, pool, args.packed_steps, args.rounds)
        finally:
            clocks = sampler.stop()
        print(json.dumps(dict(bench="packed_1024", steps=args.packed_steps, rounds=args.rounds, **r)), flush=True)
        print(json.dumps(dict(bench="clocks", part="packed_1024", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
