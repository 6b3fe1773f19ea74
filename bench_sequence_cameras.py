#!/usr/bin/env python
"""bench_sequence_cameras.py - live cameras with distinct calibrations through one front-end context
(plf_set_sequence_camera), against the same cameras sharing one calibration.

At KITTI shape with bench.py's limits and parameters (1242x375, orb_nfeatures 1500, lsd_nfeatures 200, 4096 keypoints,
8192 segments, 1024 lines per image), on one GPU, for N in --cameras (default 1, 8, 64):

  shared:   bench_multi_sequence.py's live-camera arm as it is: every camera has bench.py's KITTI calibration.
  distinct: camera c has calibration c % 4 of CALIBRATIONS, four perturbations of the KITTI camera (fx, fy, cx, cy and b
            each moved by up to a few per cent), and sees frames rendered with that calibration from its own pool, so
            that every camera tracks.  One context with max_sequences = N and plf_set_sequence_camera(c, calibration)
            runs the N pairs as one batch (B = N, seq = 0..N-1), against N single-sequence contexts at B = 1, each
            created with its camera.

A step = upload + run + download of every camera's pair (bench_multi_sequence.py's definition).  Reported per arm:
pairs/s over the timed steps, median / p90 step latency from the host clock (--steps after --warmup), and the fraction
of the last step's pairs that tracked (status 0).  The arms of one N run one after the other, so that they share the
card's state; the GPU's name, power limit and SM clocks sampled during the timed regions are printed as by
bench_multi_sequence.py.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench   # KITTI configuration, rendering, clock sampling (bench.py itself is not run)
from bench_multi_sequence import gpu_info, latency_stats, limits, live_cameras, pingpong_frames

CALIBRATIONS = [dict(bench.CAM, fx=bench.CAM["fx"] * f, fy=bench.CAM["fy"] * g, cx=bench.CAM["cx"] + dx,
                     cy=bench.CAM["cy"] + dy, b=bench.CAM["b"] * s)
                for f, g, dx, dy, s in ((1.0, 1.0, 0.0, 0.0, 1.0), (0.97, 0.975, -6.5, 3.25, 0.96),
                                        (1.03, 1.025, 4.0, -2.5, 1.04), (0.985, 0.99, 9.0, 5.0, 1.02))]


def calibrated_frames(torch, pools, n_cameras):
    """Pinned [4 period + n_cameras][h][w] left / right stacks: row j holds calibration j % 4's rendering of frame
    period[j // 4 % period] (the ping-pong order over its pool).  Camera c at step t reads row 4 (t % period) + c: its
    calibration is c % 4 at every step, its frame follows the trajectory from step to step, and the N cameras of a step
    lie in N consecutive rows."""
    n = len(pools[0])
    order = list(range(n)) + list(range(n - 2, 0, -1))
    period = len(order)
    rows = 4 * period + n_cameras
    h, w = pools[0][0][0].shape
    L = torch.empty((rows, h, w), dtype=torch.uint8, pin_memory=True)
    R = torch.empty((rows, h, w), dtype=torch.uint8, pin_memory=True)
    for j in range(rows):
        f = pools[j % 4][order[(j // 4) % period]]
        L[j].numpy()[:] = f[0]
        R[j].numpy()[:] = f[1]
    return L, R, period


def live_cameras_calibrated(plf, L, R, period, N, steps, warmup):
    frame = L[0].numel()
    ptr = lambda t, A: A.data_ptr() + 4 * (t % period) * frame
    seq = np.arange(N, dtype=np.int32)
    out = {}
    with plf.Frontend(camera=bench.CAM, limits=limits(plf, N), max_sequences=N, **bench.PRM) as fe:
        for c in range(N):
            fe.set_sequence_camera(c, CALIBRATIONS[c % 4])
        ms = []
        for t in range(warmup + steps):
            t0 = time.perf_counter()
            fe.batch_upload_raw(N, ptr(t, L), ptr(t, R))
            fe.batch_run(N, seq=seq)
            res = fe.batch_download_array(N)
            if t >= warmup:
                ms.append((time.perf_counter() - t0) * 1e3)
        out["one_context"] = dict(latency_stats(ms, N), tracked=float(np.mean(res["status"] == 0)))
    fes = [plf.Frontend(camera=CALIBRATIONS[c % 4], limits=limits(plf, 1), **bench.PRM) for c in range(N)]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--steps", type=int, default=200, help="timed steps per arm")
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequence_cameras.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    print(json.dumps(dict(bench="calibrations", cameras=CALIBRATIONS)), flush=True)
    shared_pool = bench.render_pool(bench.CAM, 24, seed=0)
    Ls, Rs, period_s = pingpong_frames(torch, shared_pool, max(args.cameras))
    pools = [shared_pool] + [bench.render_pool(c, 24, seed=0) for c in CALIBRATIONS[1:]]   # CALIBRATIONS[0] is bench.CAM
    Ld, Rd, period_d = calibrated_frames(torch, pools, max(args.cameras))
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        for N in args.cameras:
            shared = live_cameras(plf, Ls, Rs, period_s, N, args.steps, args.warmup)
            distinct = live_cameras_calibrated(plf, Ld, Rd, period_d, N, args.steps, args.warmup)
            print(json.dumps(dict(bench="live_cameras", cameras=N, steps=args.steps, shared=shared, distinct=distinct)),
                  flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", part="live_cameras", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
