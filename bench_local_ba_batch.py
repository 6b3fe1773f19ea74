#!/usr/bin/env python
"""bench_local_ba_batch.py - P local bundle adjustments as P plf_local_ba calls, against one plf_local_ba_batch call.

Maps: synth.local_map_problem, shaped like the reference's local maps: n_kf from 5 to 10 local keyframes (map p has
5 + p % 6) and 2 fixed ones, --pts-per-kf points and --ls-per-kf lines created per keyframe, each seen by up to 3
keyframes.  Map p is generated with calibration p % 4 of bench_sequence_cameras.py's CALIBRATIONS (the KITTI camera
perturbed by a few per cent).  The default LBA options (max_iters 15, ref_quirks 1).

Arms, for each P in --batch (default 1, 8, 64, 256), alternated within each step so that they share the card's state:
  sequential: P plf_local_ba calls on one context, one after the other.  plf_local_ba projects with the context's camera.
  batch:      one plf_local_ba_batch call with seq = NULL: every problem with the context's camera, as the sequential arm.
  batch_seq:  one plf_local_ba_batch call on a context with max_sequences = 4 and sequence s set to CALIBRATIONS[s], with
              seq[p] = p % 4: every problem with the camera it was generated with (only this arm can do that).
Reported per arm: device ms (CUDA events on plf_stream around the arm), wall ms (host clock, including the binding's
marshalling), local maps per second over the wall time, and kernel launches per arm (plf_launch_count).  Medians over
--steps steps after --warmup.  The GPU's name, power limit and the SM clocks and throttle reasons sampled during the run
are printed as by bench_multi_sequence.py.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench   # clock sampling (bench.py itself is not run)
from bench_multi_sequence import gpu_info
from bench_sequence_cameras import CALIBRATIONS


def maps(synth, P, pts_per_kf, ls_per_kf):
    return [synth.local_map_problem(CALIBRATIONS[p % 4], n_kf=5 + p % 6, n_fixed=2, pts_per_kf=pts_per_kf,
                                    ls_per_kf=ls_per_kf, seed=1000 + p) for p in range(P)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 64, 256])
    ap.add_argument("--steps", type=int, default=10, help="timed steps per P")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pts-per-kf", type=int, default=100)
    ap.add_argument("--ls-per-kf", type=int, default=20)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_local_ba_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        with plf.Frontend(device=0, camera=bench.CAM) as fe, plf.Frontend(device=0, camera=bench.CAM, max_sequences=4) as fs:
            for s in range(4):
                fs.set_sequence_camera(s, CALIBRATIONS[s])
            for P in args.batch:
                probs = maps(synth, P, args.pts_per_kf, args.ls_per_kf)
                seq = np.arange(P, dtype=np.int32) % 4
                n_obs = sum(len(p["pt_obs_lm"]) + len(p["ls_obs_lm"]) for p in probs)
                arms = {"sequential": (fe, lambda: [fe.local_ba(p) for p in probs]),
                        "batch": (fe, lambda: fe.local_ba_batch(probs)),
                        "batch_seq": (fs, lambda: fs.local_ba_batch(probs, seq=seq))}
                rec = {k: dict(dev=[], wall=[], launches=0) for k in arms}
                for t in range(args.warmup + args.steps):
                    for name, (f, run) in arms.items():
                        stream = torch.cuda.ExternalStream(f.stream)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        f.sync()
                        n0 = f.launches
                        w0 = time.perf_counter()
                        e0.record(stream)
                        res = run()
                        e1.record(stream)
                        wall = (time.perf_counter() - w0) * 1e3
                        e1.synchronize()
                        if name != "sequential":
                            assert all(r["status"] == 0 for r in res)
                        if t >= args.warmup:
                            rec[name]["dev"].append(e0.elapsed_time(e1))
                            rec[name]["wall"].append(wall)
                            rec[name]["launches"] = f.launches - n0
                out = {}
                for name, r in rec.items():
                    wall = float(np.median(r["wall"]))
                    out[name] = dict(device_ms=round(float(np.median(r["dev"])), 3), wall_ms=round(wall, 3),
                                     maps_per_s=round(P / (wall * 1e-3), 1), launches=r["launches"])
                print(json.dumps(dict(bench="local_ba_batch", P=P, observations=n_obs, steps=args.steps, **out)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
