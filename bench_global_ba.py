"""Global bundle adjustment benchmark: one plf_global_ba (MapHandler::levMarquardtOptimizationGBA) on synthetic maps of
32, 256, 1024, 2048 and 4096 optimised keyframes (synth.gba_problem: ~100 points and 15 lines created per keyframe,
each seen by three consecutive keyframes, with a loop closure), at the reference's settings (ref_quirks = 1,
max_iters = 15, DBL_EPSILON stop thresholds).

Per size it reports:
  - device ms per call (CUDA events on plf_stream around the call, median of --timed calls after one warm-up call);
  - the per-iteration split from torch.profiler (a separate call): rows / landmark blocks (k_lbb_rows, k_lbb_lm_accum,
    the diagonal maxima), Schur assembly (k_lbb_schur), factorisation (k_lbb_solve up to 64 keyframes, which also does
    the substitutions; k_gbb_damp / diag / panel / update beyond), substitution (k_gbb_fwd / dscale / bwd), step
    (k_lbb_backsub, k_lbb_apply), zeroing of the next round's system (k_gbb_zero, memsets), each summed over the call
    and divided by the number of solves (Schur launches).  Each group also lists the kernels of the earlier driver
    (k_lba_*, k_gba_*), so that the script times builds from before and after it alike;
  - factorisation FLOPs: n^3 / 3 for a dense LDL^T (n = 6 n_kf), and the count the tiled path executes after skipping
    exactly-zero tiles, from the tile-level symbolic factorisation of the reduced system's pattern (64^3 / 3 per
    diagonal tile, 64^3 per panel tile, 2 * 64^3 per trailing tile update); achieved TFLOP/s = executed FLOPs over the
    factorisation kernels' time, against the data-sheet 67 TFLOP/s FP64 tensor-core figure of the H100 SXM;
  - oracle/gba.py CPU time for the same call, at every size where it is expected to finish within --oracle-budget seconds
    (the smallest size always runs; a larger one runs when the last measured time, scaled by the square of the ratio
    of the observation counts, is within the budget: the sparse LU's time grows faster than the map);
  - the bytes the reference's H.reserve(VectorXi::Constant(N, 5000)) asks for (:2112): N * 5000 * (8 + 4), computed.
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
from oracle import gba  # noqa: E402
from plslam_b200 import synth  # noqa: E402

T = 64
GROUPS = {
    "rows_landmark_blocks": ("k_lba_rows", "k_lba_lm_accum", "k_lba_kf_diagmax", "k_gba_hmax_int",
                             "k_lbb_rows", "k_lbb_lm_accum", "k_lbb_kf_diagmax", "k_gbb_hmax_int"),
    "schur": ("k_lba_lm_schur", "k_lbb_schur"),
    "factorisation": ("k_lba_solve", "k_gba_damp", "k_gba_diag", "k_gba_panel", "k_gba_update",
                      "k_lbb_solve", "k_gbb_damp", "k_gbb_diag", "k_gbb_panel", "k_gbb_update"),
    "substitution": ("k_gba_fwd", "k_gba_dscale", "k_gba_bwd", "k_gbb_fwd", "k_gbb_dscale", "k_gbb_bwd"),
    "step": ("k_lba_backsub", "k_lba_apply", "k_lbb_backsub", "k_lbb_apply"),
    "zero": ("k_gbb_zero", "Memset"),
}
SCHUR = GROUPS["schur"]   # one launch per solve


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def tile_flops(p):
    """(dense n^3/3, executed) factorisation FLOPs of the tiled LDL^T, from the symbolic factorisation of the tile pattern"""
    nkf = len(p["kf_pose"])
    n = 6 * nkf
    nt = (n + T - 1) // T
    P = np.eye(nt, dtype=bool)
    for kind in ("pt", "ls"):
        lm, kf = p[kind + "_obs_lm"], p[kind + "_obs_kf"]
        keep = kf >= 0
        lm, kf = lm[keep], kf[keep]
        for d in range(1, 16):   # keyframe pairs sharing a landmark (observations are grouped per landmark)
            same = lm[d:] == lm[:-d]
            if not same.any():
                break
            a, b = kf[d:][same], kf[:-d][same]
            for ra in (6 * a // T, (6 * a + 5) // T):
                for rb in (6 * b // T, (6 * b + 5) // T):
                    P[np.maximum(ra, rb), np.minimum(ra, rb)] = True
    executed = 0.0
    for k in range(nt):
        R = k + 1 + np.nonzero(P[k + 1:, k])[0]
        if len(R):
            P[np.ix_(R, R)] |= np.tril(np.ones((len(R), len(R)), bool))
        executed += T ** 3 / 3 + len(R) * T ** 3 + len(R) * (len(R) + 1) / 2 * 2 * T ** 3
    return n ** 3 / 3, executed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32,256,1024,2048,4096")
    ap.add_argument("--pts", type=int, default=100)
    ap.add_argument("--ls", type=int, default=15)
    ap.add_argument("--timed", type=int, default=3, help="calls timed at each size")
    ap.add_argument("--oracle-budget", type=float, default=60.0, help="seconds an oracle/gba.py call may be expected to take")
    args = ap.parse_args()
    import torch
    cam = plf.KITTI_CAMERA
    print("card:", card(), flush=True)
    res = []
    oracle_last = None   # (seconds, observations) of the last oracle run
    with plf.Frontend() as fe:
        stream = torch.cuda.ExternalStream(fe.stream)
        for nkf in [int(s) for s in args.sizes.split(",")]:
            p = synth.gba_problem(cam, n_kf=nkf, pts_per_kf=args.pts, ls_per_kf=args.ls, seed=1)
            N = 6 * nkf + 3 * len(p["pt"]) + 6 * len(p["ls"])
            r = fe.global_ba(p)   # warm-up (scratch allocation)
            dev_ms, wall_ms = [], []
            for _ in range(args.timed):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                t0 = time.perf_counter()
                r = fe.global_ba(p)
                t1 = time.perf_counter()
                e1.record(stream)
                e1.synchronize()
                dev_ms.append(e0.elapsed_time(e1)); wall_ms.append((t1 - t0) * 1e3)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fe.global_ba(p)
                torch.cuda.synchronize()
            ev = prof.key_averages()
            tot = {g: sum(e.device_time_total for e in ev if any(k in e.key for k in ks)) / 1e3 for g, ks in GROUPS.items()}
            solves = sum(e.count for e in ev if any(k in e.key for k in SCHUR))
            per_iter = {g: v / max(solves, 1) for g, v in tot.items()}
            dense, executed = tile_flops(p)
            fact_s = per_iter["factorisation"] * 1e-3
            entry = dict(n_kf=nkf, n=6 * nkf, n_pt=len(p["pt"]), n_ls=len(p["ls"]),
                         n_obs=int(len(p["pt_obs_lm"]) + len(p["ls_obs_lm"])), N=N, iters=r["iters"], solves=solves,
                         solver="one CTA" if 6 * nkf <= 384 else "tiled LDL^T",
                         device_ms=float(np.median(dev_ms)), wall_ms=float(np.median(wall_ms)),
                         per_iter_ms=per_iter, fact_flop_dense=dense,
                         fact_flop_executed=executed if 6 * nkf > 384 else None,
                         fact_TFLOPs=(executed / fact_s / 1e12) if 6 * nkf > 384 and fact_s > 0 else None,
                         fact_share_of_67TFLOPs=(executed / fact_s / 67e12) if 6 * nkf > 384 and fact_s > 0 else None,
                         ref_reserve_bytes=N * 5000 * 12)
            if oracle_last is None or oracle_last[0] * (entry["n_obs"] / oracle_last[1]) ** 2 <= args.oracle_budget:
                t0 = time.perf_counter()
                gba.global_ba(cam, p)
                entry["oracle_cpu_s"] = time.perf_counter() - t0
                oracle_last = (entry["oracle_cpu_s"], entry["n_obs"])
            print(json.dumps(entry), flush=True)
            res.append(entry)
    print(json.dumps(dict(bench="global_ba", card=card(), results=res)))


if __name__ == "__main__":
    main()
