#!/usr/bin/env python
"""bench_image_sizes.py - the KITTI odometry set's three image sizes packed into one batched context (plf_set_image_sizes).

The reference's calibration files use three KITTI sizes: 1241 x 376 (kitti00-02.yaml), 1242 x 375 (kitti03.yaml) and
1226 x 370 (kitti04-10.yaml).  Each arm runs --steps batches of B pairs uploaded from pinned host memory every step, each
pair of its own sequence, up to three batches in flight:
  packed    one context of camera 1242 x 375 that also accepts the other two sizes; the batches cycle through the three
            sizes, each batch full and of one size (B sequences per size)
  single    the single-size context at 1242 x 375, every batch of that size: the rate the packed context should match
  three     one context per size, each at the largest max_batch (of B, 3B/4, B/2, B/3) at which all three fit the card;
            a step issues one batch on each
Reported per arm: pairs/s, the batches run and the device memory in use once the pipelines exist (total - free, as
cudaMemGetInfo reports it).  The arms are alternated --repeats times.  The GPU's name, power limit and clocks are printed
with the results.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench
from bench_color import fill
from bench_multi_sequence import gpu_info, limits

SIZES = [(1242, 375), (1241, 376), (1226, 370)]


def camera(w, h):
    return dict(bench.CAM, width=w, height=h, cx=bench.CAM["cx"] * w / 1242, cy=bench.CAM["cy"] * h / 375)


def hbm_used(torch):
    free, total = torch.cuda.mem_get_info()
    return round((total - free) / 2**30, 2)


def run_steps(torch, ctxs, steps):
    """steps x (upload + run of ctxs[t % len] for entries without `every`, of every entry with it), at most three
    batches in flight per context; returns pairs/s."""
    pending = {}
    pairs = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        for i, (fe, B, size, L, R, seq, every) in enumerate(ctxs):
            if not every and i != t % len(ctxs):
                continue
            q = pending.setdefault(id(fe), (fe, []))[1]
            if len(q) == 3:
                fe.batch_download_array(q.pop(0))
            fe.batch_upload_raw(B, L.data_ptr(), R.data_ptr(), size=size)
            fe.batch_run(B, seq=seq)
            q.append(B)
            pairs += B
    for fe, q in pending.values():
        while q:
            fe.batch_download_array(q.pop(0))
    dt = time.perf_counter() - t0
    return dict(pairs_per_s=round(pairs / dt, 1), batches=pairs // ctxs[0][1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=2, help="alternations of the arms")
    ap.add_argument("--pool", type=int, default=6, help="rendered pairs per size")
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_sizes.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    B = args.batch
    stacks = {sz: fill(torch, bench.render_pool(camera(*sz), args.pool, seed=i), B, 1) for i, sz in enumerate(SIZES)}
    sampler = bench.ClockSampler(0)
    sampler.start()
    try:
        def packed():
            fe = plf.Frontend(camera=camera(*SIZES[0]), limits=limits(plf, B), max_sequences=3 * B,
                              image_sizes=SIZES[1:], **bench.PRM)
            for g, sz in enumerate(SIZES[1:], 1):
                for s in range(g * B, (g + 1) * B):
                    fe.set_sequence_camera(s, camera(*sz))
            return [fe], [(fe, B, sz, *stacks[sz], np.arange(g * B, (g + 1) * B, dtype=np.int32), False)
                          for g, sz in enumerate(SIZES)], B

        def single():
            fe = plf.Frontend(camera=camera(*SIZES[0]), limits=limits(plf, B), max_sequences=B, **bench.PRM)
            return [fe], [(fe, B, SIZES[0], *stacks[SIZES[0]], np.arange(B, dtype=np.int32), True)], B

        def three():
            for b in (B, 3 * B // 4, B // 2, B // 3):
                fes = []
                try:
                    for sz in SIZES:
                        fes.append(plf.Frontend(camera=camera(*sz), limits=limits(plf, b), max_sequences=b, **bench.PRM))
                        fes[-1].device_layout   # builds the pipeline: raises here when it does not fit
                    return fes, [(fe, b, sz, *stacks[sz], np.arange(b, dtype=np.int32), True)
                                 for fe, sz in zip(fes, SIZES)], b
                except plf.PlfError:
                    for fe in fes:
                        fe.close()
                    torch.cuda.empty_cache()
            raise SystemExit("bench_image_sizes.py: three contexts do not fit at B / 3")

        for rep in range(args.repeats):
            for arm, make in (("packed", packed), ("single", single), ("three", three)):
                fes, ctxs, b = make()
                try:
                    for fe in fes:
                        fe.device_layout
                    used = hbm_used(torch)
                    steps = lambda n: n * (len(ctxs) if arm == "packed" else 1)   # packed: a step is one batch of each size
                    run_steps(torch, ctxs, steps(args.warmup))
                    r = run_steps(torch, ctxs, steps(args.steps))
                    print(json.dumps(dict(bench="image_sizes", arm=arm, batch=b, contexts=len(fes), repeat=rep, **r,
                                          hbm_used_GiB=used)), flush=True)
                finally:
                    for fe in fes:
                        fe.close()
                    torch.cuda.synchronize()
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
