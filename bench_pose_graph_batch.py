#!/usr/bin/env python
"""bench_pose_graph_batch.py - P loop-closure pose graphs as P plf_pose_graph calls, against one plf_pose_graph_batch call.

Graphs: synth.pose_graph_problem (keyframe 0 fixed, drift 0.01) at the reference's settings (max_iters = maxItersPGO =
100, lambda_init = 1e-10).  Graph p of a row has 100-300 keyframes, a kf2kf window of 1-5 and 0-4 loop edges, drawn from
seed 2000 + p, so the graphs of a row finish after different numbers of trials.  Rows:
  P = 1, 4, 16 and 64 such graphs (--batch);
  one 2048-keyframe graph (window 5, 4 loop edges) among 15 of them (--big; 0: no such row).

Arms, alternated within each step so that they share the card's state:
  single: P plf_pose_graph calls on one context, one after the other;
  batch:  one plf_pose_graph_batch call on the same graphs.
Per row: device ms of each arm (CUDA events on plf_stream around the arm; median of --steps after --warmup), the ratio,
the batch's rounds (1 + the largest trial count), the host synchronisations of each arm as the header documents them
(not counted: derived from the trial counts, once per round and once for the download, so P single calls sum 2 + trials
over the graphs and the batch takes 2 + the largest; keys *_syncs_derived), kernel launches per arm (counted with
plf_launch_count), and whether every output of the batch (poses, scalars, trace rows) is
bit-identical to the single calls'.  The card's name, power limit and maximum SM clock are read in the same command.
Prints one JSON line per row.  Writes nothing to the tree.
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


def graphs(synth, n):
    out = []
    for p in range(n):
        rng = np.random.default_rng(2000 + p)
        out.append(synth.pose_graph_problem(int(rng.integers(100, 301)), int(rng.integers(1, 6)), int(rng.integers(0, 5)),
                                            drift=0.01, seed=2000 + p))
    return out


def identical(a, b):
    keys = ("T", "iters", "stop", "trials", "chi2_init", "chi2", "lambda_", "trace")
    return all(np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes() for x, y in zip(a, b) for k in keys)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--big", type=int, default=2048, help="keyframes of the large graph among 15 small ones (0: no row)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_pose_graph_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    pool = graphs(synth, max(args.batch + [15]))
    rows = [(f"P={P}", pool[:P]) for P in args.batch]
    if args.big:
        rows.append((f"{args.big} among 15", [synth.pose_graph_problem(args.big, 5, 4, drift=0.01, seed=1)] + pool[:15]))
    with plf.Frontend(device=0) as fe:
        stream = torch.cuda.ExternalStream(fe.stream)
        for name, probs in rows:
            arms = {"single": lambda: [fe.pose_graph(p) for p in probs], "batch": lambda: fe.pose_graph_batch(probs)}
            rec = {k: dict(dev=[], launches=0, res=None) for k in arms}
            for t in range(args.warmup + args.steps):
                for arm, run in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    fe.sync()
                    n0 = fe.launches
                    e0.record(stream)
                    res = run()
                    e1.record(stream)
                    e1.synchronize()
                    if t >= args.warmup:
                        rec[arm]["dev"].append(e0.elapsed_time(e1))
                        rec[arm]["launches"] = fe.launches - n0
                        rec[arm]["res"] = res
            ms = {k: float(np.median(r["dev"])) for k, r in rec.items()}
            trials = [r["trials"] for r in rec["batch"]["res"]]
            print(json.dumps(dict(bench="pose_graph_batch", row=name, P=len(probs), steps=args.steps,
                                  n_kf=[len(p["T"]) for p in probs], trials=trials,
                                  single_ms=round(ms["single"], 3), batch_ms=round(ms["batch"], 3),
                                  single_over_batch=round(ms["single"] / ms["batch"], 3),
                                  rounds=1 + max(trials), single_syncs_derived=sum(2 + t for t in trials),
                                  batch_syncs_derived=2 + max(trials),
                                  single_launches=rec["single"]["launches"], batch_launches=rec["batch"]["launches"],
                                  bit_identical=identical(rec["single"]["res"], rec["batch"]["res"]), gpu=info)),
                  flush=True)


if __name__ == "__main__":
    sys.exit(main())
