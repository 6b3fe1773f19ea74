#!/usr/bin/env python
"""bench_global_ba_batch.py - P global bundle adjustments as P plf_global_ba calls, against one plf_global_ba_batch call.

Maps: synth.gba_problem at --sizes optimised keyframes (default 32, 256 and 1024: one CTA's solve, and the tiled LDL^T
at 24 and 96 tile columns), ~100 points and 15 lines created per keyframe, each seen by three consecutive keyframes,
with a loop closure; map p of a row has seed 1000 + p.  P in --batch (default 1, 4 and 16, and 64 at the smallest size:
more small maps fit where each costs little).  The reference's settings: ref_quirks = 1, max_iters = 15, DBL_EPSILON stop
thresholds, so every run takes its 15 iterations (g3) unless |DX| vanishes.

Arms, alternated within each step so that they share the card's state:
  single: P plf_global_ba calls on one context, one after the other;
  batch:  one plf_global_ba_batch call on the same maps, seq = NULL (the context's camera, as the single calls).
Per row: device ms of each arm (CUDA events on plf_stream around the arm; median of --steps after --warmup), the ratio,
kernel launches per arm (plf_launch_count), the batch call's scratch bytes (plf_global_ba_batch's staged layout, as the
header lists it), and the largest difference between the batch's and the single calls' outputs, relative to the step
(max |batch - single| / max |single - input| over every block of every map).  The card's name, power limit and maximum
SM clock are read in the same command.  Prints one JSON line per row.  Writes nothing to the tree.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "pl-slam_b200"))

from bench_multi_sequence import gpu_info  # noqa: E402


def a256(b):
    return (b + 255) // 256 * 256


def scratch_bytes(probs):
    """plf_global_ba_batch's staged layout for these maps (csrc/lba.cu, lbb_run): inputs, outputs and device work"""
    P = len(probs)
    kf = [len(p["kf_pose"]) for p in probs]
    obs = sum(len(p["pt_obs_lm"]) + len(p["ls_obs_lm"]) for p in probs)
    lm = sum(len(p["pt"]) + len(p["ls"]) for p in probs)
    N = sum(6 * len(p["kf_pose"]) + 3 * len(p["pt"]) + 6 * len(p["ls"]) for p in probs)
    fix = sum(len(p["fixed_T"]) for p in probs)
    nt = [(6 * k + 63) // 64 for k in kf if k > 64]
    tkf, tG, tS = sum(kf), 6 * sum(kf), sum(36 * k * k for k in kf)
    parts = [120 * P, 8 * N, 128 * fix, 4 * obs, 4 * obs, 24 * obs, 4 * (lm + P), 48 * len(nt),          # inputs
             8 * N, lm, 40 * P,                                                                      # outputs
             128 * tkf, 128 * fix, 48 * obs, 48 * obs, 16 * obs, 288 * lm, 288 * lm, 48 * lm, 8 * tG, 8 * N,
             8 * sum(t * 4096 for t in nt), sum(t * t for t in nt), 288 * tkf, 48 * tkf, 8 * tS, 8 * tG, 64 * P]
    return sum(a256(b) for b in parts)


def rel_diff(inputs, single, batch):
    out = 0.0
    for p, a, b in zip(inputs, single, batch):
        for k in ("kf_pose", "pt", "ls"):
            if a[k].size:
                step = max(np.abs(a[k] - p[k]).max(), 1e-300)
                out = max(out, float(np.abs(b[k] - a[k]).max() / step))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[32, 256, 1024])
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--small-extra", type=int, default=64, help="an extra P at the smallest size (0: none)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_global_ba_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    cam = plf.KITTI_CAMERA
    with plf.Frontend(device=0, camera=cam) as fe:
        stream = torch.cuda.ExternalStream(fe.stream)
        for n_kf in args.sizes:
            Ps = list(args.batch) + ([args.small_extra] if n_kf == min(args.sizes) and args.small_extra else [])
            pool = [synth.gba_problem(cam, n_kf=n_kf, seed=1000 + p) for p in range(max(Ps))]
            for P in Ps:
                probs = pool[:P]
                arms = {"single": lambda: [fe.global_ba(p) for p in probs], "batch": lambda: fe.global_ba_batch(probs)}
                rec = {k: dict(dev=[], launches=0, res=None) for k in arms}
                for t in range(args.warmup + args.steps):
                    for name, run in arms.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        fe.sync()
                        n0 = fe.launches
                        e0.record(stream)
                        res = run()
                        e1.record(stream)
                        e1.synchronize()
                        if t >= args.warmup:
                            rec[name]["dev"].append(e0.elapsed_time(e1))
                            rec[name]["launches"] = fe.launches - n0
                            rec[name]["res"] = res
                assert all(r["status"] == 0 for r in rec["batch"]["res"])
                assert [r["iters"] for r in rec["batch"]["res"]] == [r["iters"] for r in rec["single"]["res"]]
                ms = {k: float(np.median(r["dev"])) for k, r in rec.items()}
                print(json.dumps(dict(bench="global_ba_batch", n_kf=n_kf, P=P, steps=args.steps,
                                      observations=sum(len(p["pt_obs_lm"]) + len(p["ls_obs_lm"]) for p in probs),
                                      single_ms=round(ms["single"], 3), batch_ms=round(ms["batch"], 3),
                                      single_over_batch=round(ms["single"] / ms["batch"], 3),
                                      single_launches=rec["single"]["launches"], batch_launches=rec["batch"]["launches"],
                                      scratch_bytes=scratch_bytes(probs),
                                      max_rel_diff=rel_diff(probs, rec["single"]["res"], rec["batch"]["res"]),
                                      gpu=info)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
