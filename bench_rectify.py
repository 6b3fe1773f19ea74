#!/usr/bin/env python
"""bench_rectify.py - the batched front-end on raw (distorted, unrectified) stereo pairs, with and without the device
rectification of plf_set_sequence_rectification.

For each shape in --shapes (EuRoC's 752 x 480 and KITTI's 1242 x 375) the maps are EuRoC's calibration through
cv2.stereoRectify + cv2.initUndistortRectifyMap(CV_16SC2), its intrinsics scaled to the shape (KITTI's own raw
calibration is not used: the distortion only sets where the taps land, not the work per pixel).  A pool of rectified
pairs is rendered with the rectified camera (oracle/synth.py) and distorted back into raw pairs.  For each N in
--sequences, one context with max_sequences = N runs round-robin batches: B = N, seq = 0..N-1, camera c at step t
seeing raw pair t + c of the pool's ping-pong order.  Two batches are kept in flight (upload + run of batch t, then
download of batch t-1), the pattern of a streaming caller.  Arms:
  rectified  every sequence has maps: raw pairs are uploaded and rectified on the device;
  none       no maps, fed the same pairs rectified beforehand (cv2.remap outside the timed loop): the same downstream
             work without any remap, the ceiling of the other two;
  host       cv2.remap of both images of every pair on the host (OpenCV's own threads), into pinned memory, then an
             upload to unrectified sequences: what a caller does without the device rectification.
Reported per arm: pairs/s over --steps timed batches after --warmup.  The GPU's name, power limit and SM clocks sampled
during the timed regions are printed with the results, and OpenCV's thread count with the host arm.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench
from bench_multi_sequence import gpu_info, limits, pingpong_frames

SHAPES = {"euroc": (752, 480), "kitti": (1242, 375)}
PRM = dict(bench.PRM)


def raw_pool(shape, n):
    from oracle import rectify, synth
    left, right, cam = rectify.stereo_maps(size=shape)
    world = synth.World(seed=1, length=60.0, n_quads=200, n_segs=100, half_width=8.0, half_height=3.5)
    pool = [rectify.distort(l, r) for l, r, _ in synth.stream(cam, n, world=world, seed=2, step=0.15)]
    return left, right, cam, pool


def run_arm(plf, cv2, arm, L, R, period, N, cam, maps, steps, warmup, pre=None):
    """pre: (L, R) stacks of the pairs rectified beforehand, uploaded by the "none" arm."""
    left, right = maps
    if arm == "none":
        L, R = pre
    frame = L[0].numel()
    h, w = L.shape[1:]
    seq = np.arange(N, dtype=np.int32)
    host = None
    if arm == "host":   # two pinned landing stacks: batch t is remapped into one while batch t-1 is uploaded from the other
        import torch
        host = [tuple(torch.empty((N, h, w), dtype=torch.uint8, pin_memory=True) for _ in range(2)) for _ in range(2)]
    with plf.Frontend(camera=cam, limits=limits(plf, N), max_sequences=N, **PRM) as fe:
        if arm == "rectified":
            for s in range(N):
                fe.set_sequence_rectification(s, left=left, right=right)
        t0 = None
        for t in range(warmup + steps):
            if t == warmup:
                fe.sync()
                t0 = time.perf_counter()
            r0 = t % period
            if host is None:
                fe.batch_upload_raw(N, L.data_ptr() + r0 * frame, R.data_ptr() + r0 * frame)
            else:
                hl, hr = host[t & 1]
                for c in range(N):
                    cv2.remap(L[r0 + c].numpy(), left[0], left[1], cv2.INTER_LINEAR, dst=hl[c].numpy())
                    cv2.remap(R[r0 + c].numpy(), right[0], right[1], cv2.INTER_LINEAR, dst=hr[c].numpy())
                fe.batch_upload_raw(N, hl.data_ptr(), hr.data_ptr())
            fe.batch_run(N, seq=seq)
            if t > 0:
                res = fe.batch_download_array(N)
        res = fe.batch_download_array(N)
        dt = time.perf_counter() - t0
    return dict(pairs_per_s=round(N * steps / dt, 1), ms_per_batch=round(dt * 1e3 / steps, 3),
                tracked=float(np.mean(res["status"] == 0)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["euroc", "kitti"], choices=sorted(SHAPES))
    ap.add_argument("--sequences", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=30, help="timed batches per arm")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2, help="alternations of the three arms per (shape, N)")
    ap.add_argument("--pool", type=int, default=12, help="rendered raw pairs per shape")
    args = ap.parse_args()
    import cv2
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_rectify.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        for name in args.shapes:
            left, right, cam, pool = raw_pool(SHAPES[name], args.pool)
            L, R, period = pingpong_frames(torch, pool, max(args.sequences))
            pre = [(cv2.remap(l, *left, cv2.INTER_LINEAR), cv2.remap(r, *right, cv2.INTER_LINEAR)) for l, r in pool]
            pre = pingpong_frames(torch, pre, max(args.sequences))[:2]
            for N in args.sequences:
                for rep in range(args.repeats):
                    for arm in ("rectified", "none", "host"):
                        r = run_arm(plf, cv2, arm, L, R, period, N, cam, (left, right), args.steps, args.warmup, pre)
                        extra = dict(cv2_threads=cv2.getNumThreads()) if arm == "host" else {}
                        print(json.dumps(dict(bench="rectify", shape=name, width=cam["width"], height=cam["height"],
                                              sequences=N, repeat=rep, arm=arm, **r, **extra)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
