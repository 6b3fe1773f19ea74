#!/usr/bin/env python
"""bench_loop_closure_batch.py - P loop-closure checks as P single calls (plf_loop_closure_pose) against one
plf_loop_closure_pose_batch call, and P keyframe refinements as P plf_gn_pose calls against one plf_gn_pose_batch call.

Inputs: for each of bench_sequence_cameras.py's four CALIBRATIONS, 8 candidate pairs rendered with that calibration by
synth.loop_closure_keyframes at about the reference's sizes (1 500 points and 200 lines per keyframe, 10 % planted
outliers): 6 true revisits (accepted), one with a translation beyond lc_trs and one with unrelated point descriptors
(both rejected).  Problem p uses calibration c = p % 4 and its pair (p // 4) % 8.  The refinement problems are the
same pairs' solver rows (synth.gn_problem's points and lines with their observations).  bench.py's front-end parameters.

Arms, for each P in --batch (default 1, 8, 64, 256), alternated within each step so that they share the card's state:
  sequential: P single calls on one context, with the context's camera.
  batch:      one batch call with seq = NULL: the context's camera, as the sequential arm.
  batch_seq:  the same call on a context with max_sequences = 4 and sequence c set to CALIBRATIONS[c], with seq[p] = p % 4:
              every problem solved with the camera it was rendered with.
Reported per operator and arm: device ms (CUDA events on plf_stream around the arm), wall ms (host clock, including the
binding's marshalling), problems per second over the wall time, and kernel launches per arm (plf_launch_count).  Medians
over --steps steps after --warmup.  The batch arm's results are asserted bit-identical to the sequential arm's.  The
GPU's name, power limit and the SM clocks and throttle reasons sampled during the run are printed as by
bench_kf_matching_batch.py.  Writes nothing into the tree.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench   # clock sampling (bench.py itself is not run)
from bench_multi_sequence import gpu_info
from bench_sequence_cameras import CALIBRATIONS

N_PAIRS = 8
REVISIT = np.array([0.08, -0.03, 0.4, 0.01, -0.04, 0.006])


def pairs_of(synth, cam, c, n_pts, n_lines):
    """(lc pair, gn problem) x N_PAIRS rendered with `cam`."""
    out = []
    for k in range(N_PAIRS):
        x = np.array([0.5, 0.2, 1.9, 0.02, 0.05, 0.0]) if k == 6 else REVISIT
        kf0, kf1, g, _, _ = synth.loop_closure_keyframes(cam, seed=100 * c + k, x_true=x, n_pts=n_pts, n_lines=n_lines)
        if k == 7:
            kf1 = dict(kf1, pdesc=np.random.default_rng(k).integers(0, 256, kf1["pdesc"].shape, dtype=np.uint8))
        out.append(((kf0, kf1), dict(P=g["P"], pl_obs=g["obs"], sP=g["sP"], eP=g["eP"], le_obs=g["le"])))
    return out


def same(a, b):
    return all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a if k != "status")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 64, 256])
    ap.add_argument("--steps", type=int, default=10, help="timed steps per P")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--points", type=int, default=1500)
    ap.add_argument("--lines", type=int, default=200)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_loop_closure_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    data = [pairs_of(synth, cam, c, args.points, args.lines) for c, cam in enumerate(CALIBRATIONS)]
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        with plf.Frontend(device=0, camera=bench.CAM, **bench.PRM) as fe, \
                plf.Frontend(device=0, camera=bench.CAM, max_sequences=4, **bench.PRM) as fs:
            for c in range(4):
                fs.set_sequence_camera(c, CALIBRATIONS[c])
            for P in args.batch:
                probs = [data[p % 4][(p // 4) % N_PAIRS] for p in range(P)]
                lcp, gnp = [q[0] for q in probs], [q[1] for q in probs]
                seq = np.arange(P, dtype=np.int32) % 4
                gn1 = lambda f, d: f.gn_pose(d["P"], d["pl_obs"], d["sP"], d["eP"], d["le_obs"])
                ops = {"loop_closure": {"sequential": (fe, lambda: [fe.loop_closure_pose(*q) for q in lcp]),
                                        "batch": (fe, lambda: fe.loop_closure_pose_batch(lcp)),
                                        "batch_seq": (fs, lambda: fs.loop_closure_pose_batch(lcp, seq=seq))},
                       "gn_pose": {"sequential": (fe, lambda: [gn1(fe, d) for d in gnp]),
                                   "batch": (fe, lambda: fe.gn_pose_batch(gnp)),
                                   "batch_seq": (fs, lambda: fs.gn_pose_batch(gnp, seq=seq))}}
                for op, arms in ops.items():
                    rec = {k: dict(dev=[], wall=[], launches=0) for k in arms}
                    results = {}
                    for t in range(args.warmup + args.steps):
                        for name, (f, run) in arms.items():
                            stream = torch.cuda.ExternalStream(f.stream)
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            f.sync()
                            n0 = f.launches
                            w0 = time.perf_counter()
                            e0.record(stream)
                            results[name] = run()
                            e1.record(stream)
                            wall = (time.perf_counter() - w0) * 1e3
                            e1.synchronize()
                            if t >= args.warmup:
                                rec[name]["dev"].append(e0.elapsed_time(e1))
                                rec[name]["wall"].append(wall)
                                rec[name]["launches"] = f.launches - n0
                    # the batch returns what the single calls return (same camera)
                    assert all(same(b, a) for a, b in zip(results["sequential"], results["batch"])), op
                    out = {}
                    for name, r in rec.items():
                        wall = float(np.median(r["wall"]))
                        out[name] = dict(device_ms=round(float(np.median(r["dev"])), 3), wall_ms=round(wall, 3),
                                         problems_per_s=round(P / (wall * 1e-3), 1), launches=r["launches"])
                    extra = {}
                    if op == "loop_closure":
                        extra["accepted"] = int(sum(r["accepted"] for r in results["batch_seq"]))
                    print(json.dumps(dict(bench=f"{op}_batch", P=P, points=args.points, lines=args.lines, steps=args.steps,
                                          **extra, **out)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
