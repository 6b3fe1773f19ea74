#!/usr/bin/env python
"""bench_pair_masks.py - the cost of per-pair detector masks (plf_batch_upload_masks) in the batched front-end.

KITTI shape (1242 x 375), B = --batch pairs of bench.py's rendered stream, each pair of its own sequence (seq = 0 .. B-1),
up to three batches in flight.  Arms, alternated --repeats times in one context:
  none          no masks: the unmasked kernels, as bench.py runs them
  seq_half      every sequence masked by a half-image mask (plf_set_sequence_mask), set once before the arm
  pair_pinned   moving per-pair masks (a box and a disc per image) uploaded with every batch from pinned host memory
  pair_device   the same masks uploaded with every batch from a torch CUDA tensor (device to device)
  pair_all255   all-255 per-pair masks from pinned host memory: the pair-mask path with the feature counts of `none`
Reported per arm: pairs/s resident (the images uploaded once; the masks still with every batch) and end to end (the images
from pinned host memory with every batch too), launches per step, the mask upload's time (host clock around the copy,
between two device synchronisations) and the pyramid build's (the library's profiler marks, CUDA events on the upload
stream), and the device memory in use.  Then the live-camera case: --cameras sequences, one pair each per step, uploaded,
run and downloaded one step at a time, median and p90 step time without and with per-pair masks.  The GPU's name,
power limit and clocks are printed with the results.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench
from bench_color import fill, pinned, timed
from bench_multi_sequence import gpu_info, limits


def moving_masks(B, h, w):
    """[B, h, w] masks: 255 except a box and a disc at positions that differ per pair."""
    yy, xx = np.mgrid[:h, :w]
    out = np.full((B, h, w), 255, np.uint8)
    for k in range(B):
        bx, cx = (97 * k) % (w - w // 6), (w - 1 - (61 * k) % w)
        box = (xx >= bx) & (xx < bx + w // 6) & (yy >= h // 5) & (yy < h // 5 + h // 3)
        disc = (xx - cx) ** 2 + (yy - int(0.62 * h)) ** 2 < (h // 6) ** 2
        out[k][box | disc] = 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--cameras", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=2, help="alternations of the arms")
    ap.add_argument("--pool", type=int, default=12, help="rendered pairs")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_pair_masks.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    cam, B = bench.CAM, args.batch
    h, w = cam["height"], cam["width"]
    pool = bench.render_pool(cam, args.pool, seed=0)
    L, R = fill(torch, pool, B, 1)
    seq = np.arange(B, dtype=np.int32)
    mv = moving_masks(B, h, w)
    host = {"pair_pinned": pinned(torch, (B, h, w)), "pair_all255": pinned(torch, (B, h, w))}
    host["pair_pinned"].numpy()[:] = mv
    host["pair_all255"].numpy()[:] = 255
    dev = torch.from_numpy(mv).cuda()
    torch.cuda.synchronize()
    ptrs = {k: v.data_ptr() for k, v in host.items()}
    ptrs["pair_device"] = dev.data_ptr()
    half = np.where(np.arange(w)[None, :].repeat(h, 0) < w // 2, 255, 0).astype(np.uint8)
    arms = ["none", "seq_half", "pair_pinned", "pair_device", "pair_all255"]
    sampler = bench.ClockSampler(0)
    sampler.start()
    try:
        with plf.Frontend(camera=cam, limits=limits(plf, B), max_sequences=B, **bench.PRM) as fe:
            fe.batch_upload_raw(B, L.data_ptr(), R.data_ptr())
            for rep in range(args.repeats):
                for arm in arms:
                    fe.sync()
                    for s in range(B):
                        fe.set_sequence_mask(s, *((half, half) if arm == "seq_half" else (None, None)))
                    p = ptrs.get(arm)
                    masks = (lambda t: fe.batch_upload_masks_raw(B, p, p)) if p else None
                    resident = timed(fe, B, args.steps, args.warmup, masks, seq)

                    def images_and_masks(t):
                        fe.batch_upload_raw(B, L.data_ptr(), R.data_ptr())
                        if p:
                            fe.batch_upload_masks_raw(B, p, p)
                    e2e = timed(fe, B, args.steps, args.warmup, images_and_masks, seq)
                    # one step alone: launches, mask upload (host clock between device synchronisations), build (profiled)
                    fe.sync()
                    t0 = time.perf_counter()
                    if p:
                        fe.batch_upload_masks_raw(B, p, p)
                    fe.sync()
                    up_ms = (time.perf_counter() - t0) * 1e3
                    n0 = fe.launches
                    fe.profile_enable(True)
                    fe.batch_run(B, seq=seq)
                    prof = fe.profile_read()
                    fe.profile_enable(False)
                    res = fe.batch_download_array(B)
                    launches = fe.launches - n0
                    build = [t for n, t in prof if n == "masks.k_mask_pyramid"]
                    free, total = torch.cuda.mem_get_info()
                    print(json.dumps(dict(bench="pair_masks", arm=arm, batch=B, width=w, height=h, repeat=rep,
                                          resident=resident, end_to_end=e2e, launches_per_step=launches,
                                          mask_upload_ms=round(up_ms, 3) if p else None,
                                          pyramid_build_ms=round(float(build[0]), 3) if build else None,
                                          hbm_used_GB=round((total - free) / 1e9, 2),
                                          kp_per_image=round(float((res["n_kp_l"] + res["n_kp_r"]).mean()) / 2, 1),
                                          lines_per_image=round(float((res["n_lines_l"] + res["n_lines_r"]).mean()) / 2, 1))),
                          flush=True)
            for s in range(B):
                fe.set_sequence_mask(s)
        live(plf, torch, args, pool)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


def live(plf, torch, args, pool):
    """--cameras sequences, one pair each per step: upload, (masks,) run, download, one step at a time."""
    cam, N = bench.CAM, args.cameras
    h, w = cam["height"], cam["width"]
    L, R = fill(torch, pool, N, 1)
    mv = pinned(torch, (N, h, w))
    mv.numpy()[:] = moving_masks(N, h, w)
    dev = mv.cuda()
    torch.cuda.synchronize()
    seq = np.arange(N, dtype=np.int32)
    with plf.Frontend(camera=cam, limits=limits(plf, N), max_sequences=N, **bench.PRM) as fe:
        for rep in range(args.repeats):
            for arm, p in (("none", None), ("pair_pinned", mv.data_ptr()), ("pair_device", dev.data_ptr())):
                ms = []
                for t in range(args.warmup + 5 * args.steps):
                    fe.sync()
                    t0 = time.perf_counter()
                    fe.batch_upload_raw(N, L.data_ptr(), R.data_ptr())
                    if p:
                        fe.batch_upload_masks_raw(N, p, p)
                    fe.batch_run(N, seq=seq)
                    fe.batch_download_array(N)
                    if t >= args.warmup:
                        ms.append((time.perf_counter() - t0) * 1e3)
                print(json.dumps(dict(bench="pair_masks_live", arm=arm, cameras=N, repeat=rep,
                                      median_ms=round(float(np.median(ms)), 3), p90_ms=round(float(np.percentile(ms, 90)), 3))),
                      flush=True)


if __name__ == "__main__":
    sys.exit(main())
