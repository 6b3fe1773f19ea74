#!/usr/bin/env python
"""bench_color.py - the batched front-end on colour stereo pairs converted to grey on the device (plf_batch_upload_color),
against grey input and against converting on the host.

KITTI shape (1242 x 375), B = --batch pairs of bench.py's rendered stream, each frame colourised with a seeded per-channel
offset (every channel weight matters).  Arms, each in two modes:
  grey       plf_batch_upload of the grey pairs (bench.py's input): the baseline
  bgr, bgra  plf_batch_upload_color of 3 / 4-channel pairs, converted on the device
  host_bgr   cv2.cvtColor(COLOR_BGR2GRAY) of every image on the host (OpenCV's own threads) into pinned memory, then a
             grey upload: what a colour user does without the device conversion
Modes: "resident" = the upload done once, --steps runs with up to three in flight (the colour arms convert in every run);
"e2e" = from pinned host buffers, upload + run + download per step, up to three in flight.
Then --cameras round-robin rectified colour cameras (EuRoC's calibration scaled to the shape, oracle/rectify.py):
  rect_device  raw BGR pairs uploaded, remapped and converted on the device
  rect_host    cv2.remap of the BGR images then cv2.cvtColor on the host, then a grey upload to unrectified sequences
Reported: pairs/s per arm and mode, H2D bytes per pair, and k_color's device time (CUDA events of a profiled run) with the
HBM bytes it moves over that time.  The GPU's name, power limit and clocks are printed with the results.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

import bench
from bench_multi_sequence import gpu_info, limits


def colourise(g, seed, ch):
    rng = np.random.default_rng(seed)
    off = rng.integers(-24, 25, ch)
    out = np.clip(g[..., None].astype(np.int16) + off, 0, 255).astype(np.uint8)
    if ch == 4:
        out[..., 3] = 255
    return out


def pinned(torch, shape):
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True)


def fill(torch, pool, B, ch):
    """Pinned [B, h, w(, ch)] left / right stacks of bench.py's ping-pong order, colourised when ch > 1."""
    h, w = pool[0][0].shape
    shape = (B, h, w) if ch == 1 else (B, h, w, ch)
    L, R = pinned(torch, shape), pinned(torch, shape)
    n = len(pool)
    period = list(range(n)) + list(range(n - 2, 0, -1)) if n > 2 else list(range(n))
    frames = pool if ch == 1 else [(colourise(l, 2 * j, ch), colourise(r, 2 * j + 1, ch)) for j, (l, r) in enumerate(pool)]
    for k in range(B):
        L[k].numpy()[:], R[k].numpy()[:] = frames[period[k % len(period)]]
    return L, R


def pipelined(fe, B, steps, step_upload, seq=None):
    """steps x (upload + run), download, up to three batches in flight; step_upload(t) uploads batch t (None: no upload)."""
    issued = done = 0
    while done < steps:
        while issued < steps and issued - done < 3:
            if step_upload:
                step_upload(issued)
            fe.batch_run(B, seq=seq)
            issued += 1
        fe.batch_download_array(B)
        done += 1


def timed(fe, B, steps, warmup, step_upload, seq=None):
    pipelined(fe, B, warmup, step_upload, seq)
    fe.sync()
    t0 = time.perf_counter()
    pipelined(fe, B, steps, step_upload, seq)
    dt = time.perf_counter() - t0
    return dict(pairs_per_s=round(B * steps / dt, 1), ms_per_step=round(dt * 1e3 / steps, 2))


def kernel_time(fe, B, ch, upload):
    """k_color's device time (ms, CUDA events around it in a profiled run) and the HBM it moves, over 5 runs."""
    ms = []
    upload()
    for _ in range(5):
        fe.sync()
        fe.profile_enable(True)
        fe.batch_run(B)
        ms += [t for n, t in fe.profile_read() if n == "color.k_color"]
        fe.profile_enable(False)
        fe.batch_download_array(B)
    h, w = bench.CAM["height"], bench.CAM["width"]
    moved = 2 * B * h * w * (ch + 1)   # every colour byte read once, every grey byte written once
    t = float(np.median(ms))
    return dict(kernel_ms=round(t, 3), kernel_GBps=round(moved / (t * 1e-3) / 1e9, 1), kernel_bytes=moved)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--cameras", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=2, help="alternations of the arms")
    ap.add_argument("--pool", type=int, default=12, help="rendered pairs")
    args = ap.parse_args()
    import cv2
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_color.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    cam, B = bench.CAM, args.batch
    h, w = cam["height"], cam["width"]
    pool = bench.render_pool(cam, args.pool, seed=0)
    src = {ch: fill(torch, pool, B, ch) for ch in (1, 3, 4)}
    host_grey = [(pinned(torch, (B, h, w)), pinned(torch, (B, h, w))) for _ in range(2)]
    host = dict(cv2_threads=cv2.getNumThreads(), cpu_count=os.cpu_count())
    sampler = bench.ClockSampler(0)
    sampler.start()
    try:
        with plf.Frontend(camera=cam, limits=limits(plf, B), **bench.PRM) as fe:
            def up(ch):
                L, R = src[ch]
                return lambda t=0: fe.batch_upload_raw(B, L.data_ptr(), R.data_ptr(), channels=ch)

            def up_host(t):
                L, R = src[3]
                gl, gr = host_grey[t & 1]
                for k in range(B):
                    cv2.cvtColor(L[k].numpy(), cv2.COLOR_BGR2GRAY, dst=gl[k].numpy())
                    cv2.cvtColor(R[k].numpy(), cv2.COLOR_BGR2GRAY, dst=gr[k].numpy())
                fe.batch_upload_raw(B, gl.data_ptr(), gr.data_ptr())

            for rep in range(args.repeats):
                for arm, ch in (("grey", 1), ("bgr", 3), ("bgra", 4), ("host_bgr", 3)):
                    rows = []
                    if arm != "host_bgr":
                        up(ch)()
                        rows.append(("resident", timed(fe, B, args.steps, args.warmup, None)))
                    rows.append(("e2e", timed(fe, B, args.steps, args.warmup, up_host if arm == "host_bgr" else up(ch))))
                    for mode, r in rows:
                        extra = host if arm == "host_bgr" else {}
                        print(json.dumps(dict(bench="color", arm=arm, mode=mode, batch=B, width=w, height=h, repeat=rep,
                                              h2d_bytes_per_pair=2 * h * w * (1 if arm == "host_bgr" else ch), **r,
                                              **extra)), flush=True)
            for ch in (3, 4):
                print(json.dumps(dict(bench="color_kernel", channels=ch, batch=B, **kernel_time(fe, B, ch, up(ch)))),
                      flush=True)
        rect_cameras(plf, cv2, torch, args, host)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


def rect_cameras(plf, cv2, torch, args, host):
    """--cameras rectified colour cameras round-robin: one pair of each per batch, camera c at step t seeing raw pair
    t + c of the pool's ping-pong order."""
    from bench_rectify import raw_pool
    N = args.cameras
    cam0 = bench.CAM
    left, right, cam, pool = raw_pool((cam0["width"], cam0["height"]), args.pool)
    h, w = cam["height"], cam["width"]
    L, R = fill(torch, pool, len(pool) * 2 - 2 + N, 3)
    period = 2 * len(pool) - 2
    frame = h * w * 3
    seq = np.arange(N, dtype=np.int32)
    grey = [(pinned(torch, (N, h, w)), pinned(torch, (N, h, w))) for _ in range(2)]
    tmp = np.empty((h, w, 3), np.uint8)
    for rep in range(args.repeats):
        for arm in ("rect_device", "rect_host"):
            with plf.Frontend(camera=cam, limits=limits(plf, N), max_sequences=N, **bench.PRM) as fe:
                if arm == "rect_device":
                    for s in range(N):
                        fe.set_sequence_rectification(s, left=left, right=right)

                    def step(t):
                        r0 = t % period
                        fe.batch_upload_raw(N, L.data_ptr() + r0 * frame, R.data_ptr() + r0 * frame, channels=3)
                else:
                    def step(t):
                        r0 = t % period
                        gl, gr = grey[t & 1]
                        for c in range(N):
                            cv2.remap(L[r0 + c].numpy(), left[0], left[1], cv2.INTER_LINEAR, dst=tmp)
                            cv2.cvtColor(tmp, cv2.COLOR_BGR2GRAY, dst=gl[c].numpy())
                            cv2.remap(R[r0 + c].numpy(), right[0], right[1], cv2.INTER_LINEAR, dst=tmp)
                            cv2.cvtColor(tmp, cv2.COLOR_BGR2GRAY, dst=gr[c].numpy())
                        fe.batch_upload_raw(N, gl.data_ptr(), gr.data_ptr())
                r = timed(fe, N, args.steps * 4, args.warmup, step, seq)
            extra = host if arm == "rect_host" else {}
            print(json.dumps(dict(bench="color_rect", arm=arm, cameras=N, width=w, height=h, repeat=rep,
                                  h2d_bytes_per_pair=2 * h * w * (3 if arm == "rect_device" else 1), **r, **extra)),
                  flush=True)


if __name__ == "__main__":
    sys.exit(main())
