"""Loop-closure pose-graph benchmark: one plf_pose_graph (g2o's computeInitialGuess + Levenberg-Marquardt in
MapHandler::loopClosureOptimizationCovGraphG2O) on synthetic loops of 256, 1024, 2048 and 4096 keyframes
(synth.pose_graph_problem: kf2kf edges within a window of 5, 4 loop edges, keyframe 0 fixed), at the reference's settings
(max_iters = maxItersPGO = 100, lambda_init = 1e-10).

Per size it reports:
  - device ms per call (CUDA events on plf_stream around the call, median of --timed calls after one warm-up call);
  - iterations and trials of the call;
  - the per-trial split from torch.profiler (a separate call): linearisation (k_pgo_linearize, once per iteration),
    assembly (k_pgo_assemble and the zeroing of the dense system: k_pgo_zero, a memset before it), factorisation
    (k_gbb_diag / panel / update, k_gba_* before the batched driver), substitution (k_gbb_fwd / dscale / bwd, k_gba_*
    likewise), step and chi2 (k_pgo_step, k_pgo_edge_chi2, k_pgo_reduce), each summed
    over the call and divided by the number of trials;
  - factorisation FLOPs: n^3 / 3 for a dense LDL^T (n = 6 n_free) and the count the tiled path executes after skipping
    exactly-zero tiles, from the tile-level symbolic factorisation of H's block pattern (64^3 / 3 per diagonal tile,
    64^3 per panel tile, 2 * 64^3 per trailing tile update); achieved TFLOP/s = executed FLOPs over the factorisation
    kernels' time, against the data-sheet 67 TFLOP/s FP64 tensor-core figure of the H100 SXM;
  - the scratch bytes the call carves (plf_pgo_result.scratch_bytes);
  - oracle/pgo.py CPU time for the same call, at every size expected to finish within --oracle-budget seconds (the
    smallest size always runs; a larger one when the last measured time, scaled by the ratio of the edge counts, fits).
Prints the card name and power limit, one JSON line per size, then one JSON summary line.  Writes nothing to the tree."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "pl-slam_b200"))

import plslam_b200 as plf  # noqa: E402
from oracle import pgo  # noqa: E402
from plslam_b200 import synth  # noqa: E402

T = 64
GROUPS = {
    "linearize": ("k_pgo_linearize",),
    "assembly": ("k_pgo_assemble", "k_pgo_zero", "Memset"),
    "factorisation": ("k_gba_diag", "k_gba_panel", "k_gba_update", "k_gbb_diag", "k_gbb_panel", "k_gbb_update"),
    "substitution": ("k_gba_fwd", "k_gba_dscale", "k_gba_bwd", "k_gbb_fwd", "k_gbb_dscale", "k_gbb_bwd"),
    "step_chi2": ("k_pgo_step", "k_pgo_edge_chi2", "k_pgo_reduce"),
}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def tile_flops(p):
    """(dense n^3/3, executed) factorisation FLOPs of the tiled LDL^T, from the symbolic factorisation of the tile pattern"""
    fixed, frm, to = np.asarray(p["fixed"]).astype(bool), np.asarray(p["from"]), np.asarray(p["to"])
    fidx = pgo.free_index(fixed, frm, to)
    nf = int((fidx >= 0).sum())
    n = 6 * nf
    nt = (n + T - 1) // T
    P = np.eye(nt, dtype=bool)
    a, b = fidx[frm], fidx[to]
    keep = (a >= 0) & (b >= 0)
    a, b = a[keep], b[keep]
    for ra in (6 * a // T, (6 * a + 5) // T):
        for rb in (6 * b // T, (6 * b + 5) // T):
            P[np.maximum(ra, rb), np.minimum(ra, rb)] = True
    executed = 0.0
    for k in range(nt):
        R = k + 1 + np.nonzero(P[k + 1:, k])[0]
        if len(R):
            P[np.ix_(R, R)] |= np.tril(np.ones((len(R), len(R)), bool))
        executed += T ** 3 / 3 + len(R) * T ** 3 + len(R) * (len(R) + 1) / 2 * 2 * T ** 3
    return nf, n ** 3 / 3, executed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,1024,2048,4096")
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--loops", type=int, default=4)
    ap.add_argument("--drift", type=float, default=0.01)
    ap.add_argument("--timed", type=int, default=3, help="calls timed at each size")
    ap.add_argument("--oracle-budget", type=float, default=60.0, help="seconds an oracle/pgo.py call may be expected to take")
    args = ap.parse_args()
    import torch
    print("card:", card(), flush=True)
    res = []
    oracle_last = None   # (seconds, edges) of the last oracle run
    with plf.Frontend() as fe:
        stream = torch.cuda.ExternalStream(fe.stream)
        for nkf in [int(s) for s in args.sizes.split(",")]:
            p = synth.pose_graph_problem(nkf, args.window, args.loops, drift=args.drift, seed=1)
            r = fe.pose_graph(p, trace=False)   # warm-up (scratch allocation)
            dev_ms = []
            for _ in range(args.timed):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                r = fe.pose_graph(p, trace=False)
                e1.record(stream)
                e1.synchronize()
                dev_ms.append(e0.elapsed_time(e1))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fe.pose_graph(p, trace=False)
                torch.cuda.synchronize()
            ev = prof.key_averages()
            tot = {g: sum(e.device_time_total for e in ev if any(k in e.key for k in ks)) / 1e3 for g, ks in GROUPS.items()}
            per_trial = {g: v / max(r["trials"], 1) for g, v in tot.items()}
            nf, dense, executed = tile_flops(p)
            fact_s = per_trial["factorisation"] * 1e-3
            entry = dict(n_kf=nkf, n_free=nf, n=6 * nf, n_e=len(p["from"]), window=args.window, loops=args.loops,
                         iters=r["iters"], trials=r["trials"], stop=r["stop"], chi2_init=r["chi2_init"], chi2=r["chi2"],
                         device_ms=float(np.median(dev_ms)), per_trial_ms=per_trial,
                         fact_flop_dense=dense, fact_flop_executed=executed,
                         fact_TFLOPs=executed / fact_s / 1e12 if fact_s > 0 else None,
                         fact_share_of_67TFLOPs=executed / fact_s / 67e12 if fact_s > 0 else None,
                         scratch_bytes=r["scratch_bytes"])
            if oracle_last is None or oracle_last[0] * (entry["n_e"] / oracle_last[1]) <= args.oracle_budget:
                t0 = time.perf_counter()
                pgo.optimize(p)
                entry["oracle_cpu_s"] = time.perf_counter() - t0
                oracle_last = (entry["oracle_cpu_s"], entry["n_e"])
            print(json.dumps(entry), flush=True)
            res.append(entry)
    print(json.dumps(dict(bench="pose_graph", card=card(), results=res)))


if __name__ == "__main__":
    main()
