"""Counts the serial chain of the LSD region growing (k_lsd_grow) when one warp round handles 1, 2 or 3 queue entries.

The growing warp walks each region's queue.  A round takes the E = min(n, nreg - r) entries r .. r+E-1 that exist when
it starts, puts the 9 records of each entry's 3x3 neighbourhood on lanes 9e + kk, and decides them in lane order, which
is the reference's order of tests: one decision-loop iteration per acceptance, per evaluation of the region angle and per
exact f64 test, and one terminating iteration when everything left is clearly not aligned.  Cells accepted in a round
join the queue and are handled by a later round.  Besides its iterations, a round pays a fixed cost (queue-entry loads,
the look-ahead rotation, the first ballot, a warp barrier).

The replay follows the kernel's deferred region angle: the angle th is evaluated only when the first undecided candidate
sits in the band prec -/+ m around it (m = 0.05 deg after an evaluation, m += min(d + m, prec + 0.05) / |S| per
acceptance), and inside the 0.05 deg band the exact test decides.  It works in float64 on cv2's level-line angles, so
its partition can differ from the kernel's in a few borderline pixels; the counts are statistics, not a parity check.
It does check that every round size grows the same regions in the same order (the round structure must not change
the result).

Columns per image: region starts, rounds, "cold" rounds (an entry of the round did not exist when the previous round
started, so a look-ahead issued at round starts alone could not have covered it; the kernel loads such an entry's
records when its cell is accepted), decision-loop iterations by outcome (acceptance, terminating, angle evaluation,
exact f64 test) and their sum, and the chain = rounds + iterations.

Usage: python oracle/tools/grow_rounds_sim.py [--configs kitti,lowtex] [--frames 3]
"""
import argparse
import math
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "pl-slam_b200")); sys.path.insert(0, str(Path(__file__).resolve().parent))

NOTDEF = -1024.0
MARGIN0 = 0.05
KINDS = ("starts", "rounds", "cold", "accept", "terminate", "band_atan2", "band_f64", "iterations")


def angle_map_deg(img, scale=1.2):
    """Level-line angles in degrees [0, 360) (NOTDEF where undefined), with W + 1 NOTDEF guard records in front as in
    the kernel's record map, and the seeds (linear indices into the guarded map) in pseudo-order."""
    from spec_grow_sim import level_lines
    ang, order = level_lines(img, scale)
    H, W = ang.shape
    deg = np.where(ang == NOTDEF, NOTDEF, np.mod(np.degrees(ang), 360.0))
    g = W + 1
    flat = [NOTDEF] * g + deg.ravel().tolist()
    return flat, [g + y * W + x for (x, y) in order], W


def grow(flat, seeds, W, n, prec_deg=22.5):
    """Replays the growing with n queue entries per round; returns (counts, regions)."""
    a = list(flat)                      # a used cell is set to NOTDEF, as in the kernel
    offs = [dy * W + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    dmax = prec_deg + MARGIN0
    c = dict.fromkeys(KINDS, 0)
    regions = []
    for s in seeds:
        if a[s] == NOTDEF:
            continue
        c["starts"] += 1
        th = a[s]
        sx, sy = math.cos(math.radians(th)), math.sin(math.radians(th))
        margin, inv0, fresh = MARGIN0, 1.02, True
        a[s] = NOTDEF
        queue = [s]
        r, seen = 0, 0                   # seen: queue length when the previous round started
        while r < len(queue):
            E = min(n, len(queue) - r)
            c["rounds"] += 1
            c["cold"] += r + E > seen        # an entry the previous round could not look ahead to
            seen = len(queue)
            cells = [queue[r + e] + o for e in range(E) for o in offs]
            rem = [a[ci] != NOTDEF for ci in cells]
            rec = [a[ci] for ci in cells]
            r += E
            while any(rem):
                c["iterations"] += 1
                lo, hi = prec_deg - margin, prec_deg + margin
                k = -1
                for j, ci in enumerate(cells):
                    if rem[j]:
                        d = abs(rec[j] - th)
                        if d > 180.0:
                            d = 360.0 - d
                        if d <= hi:
                            k, dk = j, d
                            break
                if k < 0:
                    c["terminate"] += 1
                    break
                if dk >= lo:                        # the first candidate sits in the band
                    if not fresh:
                        c["band_atan2"] += 1
                        th = math.degrees(math.atan2(sy, sx)) % 360.0
                        inv0 = 1.02 / math.hypot(sx, sy)
                        margin, fresh = MARGIN0, True
                        continue
                    c["band_f64"] += 1
                    if not dk <= prec_deg:
                        for j in range(k + 1):
                            rem[j] = False
                        continue
                else:
                    c["accept"] += 1
                for j in range(k + 1):
                    rem[j] = False
                ai = cells[k]
                for j in range(k + 1, len(cells)):  # the same cell seen from a later entry of the round is used now
                    if cells[j] == ai:
                        rem[j] = False
                a[ai] = NOTDEF
                queue.append(ai)
                sx += math.cos(math.radians(rec[k])); sy += math.sin(math.radians(rec[k]))
                margin += min(dk + margin, dmax) * inv0
                fresh = False
        regions.append(queue)
    c["chain"] = c["rounds"] + c["iterations"]
    return c, regions


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="kitti,lowtex")
    ap.add_argument("--frames", type=int, default=3, help="frames of the bench pool replayed per config")
    ap.add_argument("--scale", type=float, default=1.2)
    args = ap.parse_args()
    import bench
    for cfg in args.configs.split(","):
        bench.select_config(cfg)
        pool = bench.render_pool(bench.CAM, args.frames, seed=0)
        tot = {n: dict.fromkeys(KINDS + ("chain",), 0) for n in (1, 2, 3)}
        for fi, (L, R) in enumerate(pool):
            for side, img in (("L", L), ("R", R)):
                flat, seeds, W = angle_map_deg(img, args.scale)
                ref = None
                for n in (1, 2, 3):
                    cnt, regs = grow(flat, seeds, W, n)
                    if ref is None:
                        ref = regs
                    assert regs == ref, f"{cfg} frame {fi}{side}: {n} entries per round changed the partition"
                    for k, v in cnt.items():
                        tot[n][k] += v
        nimg = 2 * len(pool)
        print(f"{cfg}: {nimg} images {bench.CAM['width']}x{bench.CAM['height']} at scale {args.scale}, per image:")
        print("  entries/round " + " ".join(f"{k:>11s}" for k in KINDS + ("chain",)))
        for n in (1, 2, 3):
            print(f"  {n:13d} " + " ".join(f"{tot[n][k] / nimg:11.0f}" for k in KINDS + ("chain",)))
        for n in (2, 3):
            it = 1 - tot[n]["iterations"] / tot[1]["iterations"]
            ch = 1 - tot[n]["chain"] / tot[1]["chain"]
            print(f"  {n} entries per round: decision-loop iterations -{100 * it:.1f} %, chain (rounds + iterations) -{100 * ch:.1f} %")


if __name__ == "__main__":
    main()
