#!/usr/bin/env python
"""bench_kf_matching_batch.py - the keyframe matching of P new keyframes as 2 P single calls (plf_match_kf2kf and
plf_match_map2kf), against one plf_match_kf2kf_batch and one plf_match_map2kf_batch call.

Keyframes: four synthetic KITTI-shape streams (synth.stream, bench.py's front-end parameters), stream c rendered with
calibration c of bench_sequence_cameras.py's CALIBRATIONS and its features taken from a context with that camera.
Keyframe p belongs to stream c = p % 4 and has
  - a KF-to-KF problem: frames k and k + 5 of its stream, k = (p // 4) % 7;
  - a map-to-KF problem: frame 8 of its stream against a local map of about --landmarks landmarks built from frames 0-7
    as bench_map_matching.py builds them (lines in the stream's proportion).
fast_matching = 1, as every reference configuration sets it, and the default parameters otherwise.

Arms, for each P in --batch (default 1, 8, 64, 256), alternated within each step so that they share the card's state:
  sequential: P plf_match_kf2kf then P plf_match_map2kf calls on one context, with the context's camera.
  batch:      one plf_match_kf2kf_batch and one plf_match_map2kf_batch call with seq = NULL: the context's camera, as the
              sequential arm.
  batch_seq:  the same two calls on a context with max_sequences = 4 and sequence c set to CALIBRATIONS[c], with
              seq[p] = p % 4: every keyframe matched with the camera it was rendered with.
Reported per arm: device ms (CUDA events on plf_stream around the arm), wall ms (host clock, including the binding's
marshalling), keyframes per second over the wall time, and kernel launches per arm (plf_launch_count).  Medians over
--steps steps after --warmup.  The GPU's name, power limit and the SM clocks and throttle reasons sampled during the run
are printed as by bench_local_ba_batch.py.  Writes nothing into the tree.
"""
import argparse
import json
import sys
import time

import numpy as np

import bench   # clock sampling (bench.py itself is not run)
from bench_map_matching import build_map
from bench_multi_sequence import gpu_info
from bench_sequence_cameras import CALIBRATIONS

N_FRAMES = 12


def streams(plf, synth):
    """Per calibration: (T_wc, get_frame dicts) of N_FRAMES frames."""
    out = []
    lim = plf.default_limits()
    lim.max_batch = N_FRAMES
    for c, cam in enumerate(CALIBRATIONS):
        frames = list(synth.stream(cam, N_FRAMES, seed=c))
        with plf.Frontend(device=0, camera=cam, limits=lim, **bench.PRM) as fe:
            fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
            out.append(([f[2] for f in frames], [fe.get_frame(k) for k in range(N_FRAMES)]))
    return out


def problems(data, maps, P):
    kf2kf, map2kf = [], []
    for p in range(P):
        T_wc, feats = data[p % 4]
        k = (p // 4) % 7
        kf2kf.append(dict(prev=feats[k], curr=feats[k + 5], DT=np.linalg.inv(T_wc[k + 5]) @ T_wc[k]))
        map2kf.append(dict(local_map=maps[p % 4], Twf=np.linalg.inv(T_wc[8]), kf=feats[8]))
    return kf2kf, map2kf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 64, 256])
    ap.add_argument("--steps", type=int, default=10, help="timed steps per P")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--landmarks", type=int, default=2000)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_kf_matching_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    data = streams(plf, synth)
    rng = np.random.default_rng(0)
    maps = [build_map(T_wc[:8], feats[:8], args.landmarks, rng) for T_wc, feats in data]
    sampler = bench.ClockSampler(0)   # nvidia-smi in the background: stopped on every way out
    sampler.start()
    try:
        with plf.Frontend(device=0, camera=bench.CAM, **bench.PRM) as fe, \
                plf.Frontend(device=0, camera=bench.CAM, max_sequences=4, **bench.PRM) as fs:
            for c in range(4):
                fs.set_sequence_camera(c, CALIBRATIONS[c])
            for P in args.batch:
                kp, mp = problems(data, maps, P)
                seq = np.arange(P, dtype=np.int32) % 4

                def sequential():
                    return ([fe.match_kf2kf(q["prev"], q["curr"], q["DT"]) for q in kp],
                            [fe.match_map2kf(q["local_map"], q["Twf"], q["kf"]) for q in mp])
                arms = {"sequential": (fe, sequential),
                        "batch": (fe, lambda: (fe.match_kf2kf_batch(kp), fe.match_map2kf_batch(mp))),
                        "batch_seq": (fs, lambda: (fs.match_kf2kf_batch(kp, seq=seq), fs.match_map2kf_batch(mp, seq=seq)))}
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
                for a, b in zip(results["sequential"][0] + results["sequential"][1], results["batch"][0] + results["batch"][1]):
                    assert all(np.array_equal(a[k], b[k]) for k in a)
                out = {}
                for name, r in rec.items():
                    wall = float(np.median(r["wall"]))
                    out[name] = dict(device_ms=round(float(np.median(r["dev"])), 3), wall_ms=round(wall, 3),
                                     keyframes_per_s=round(P / (wall * 1e-3), 1), launches=r["launches"])
                n_pt = int(np.mean([r["n_pt"] for r in results["batch_seq"][1]]))
                print(json.dumps(dict(bench="kf_matching_batch", P=P, landmarks=args.landmarks, map_pt_matches=n_pt,
                                      steps=args.steps, **out)), flush=True)
    finally:
        clocks = sampler.stop()
    print(json.dumps(dict(bench="clocks", gpu=info, **clocks)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
