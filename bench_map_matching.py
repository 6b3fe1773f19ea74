#!/usr/bin/env python
"""bench_map_matching.py - keyframe matching on the device (plf_match_kf2kf / plf_match_map2kf) against the host
composition it replaces, on the synthetic KITTI-shape stream.

Cases: KF-to-KF on keyframe pairs 5 frames apart, and map-to-KF with local maps of about 2k, 8k and 32k landmarks (lines
in the stream's proportion), each with fast_matching 0 and 1.  Per case:
  dev_ms    device time per call (CUDA events on plf_stream around the call).  With fast_matching = 1 this includes the
            brute-force match() pass whenever the host-known sizes allow the fallback: the call computes it before the
            device decides whether the windowed result stands
  wall_ms   host wall time per call, ending at the call's own synchronise
  host_ms   the same inputs through the host composition: numpy projection / visibility / grids -> plf_match_grid_* ->
            plf_match when the fallback is taken -> numpy gate (wall time)
  cv2_ms    cv2.BFMatcher(NORM_HAMMING).knnMatch(k=2) on the brute-force-sized problem (points and lines), CPU
The card name and power limit are printed with the table.  Writes nothing into the tree."""
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
from oracle import kfmatching as kfm  # noqa: E402
from oracle import matchgrid as mg  # noqa: E402
from oracle import synth  # noqa: E402
from oracle.frontend import GRID_COLS, GRID_ROWS  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi gave no output"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fe, fn, reps):
    import torch
    s = torch.cuda.ExternalStream(fe.stream)
    dev, wall = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        t0 = time.perf_counter()
        fn()
        wall.append((time.perf_counter() - t0) * 1e3)
        b.record(s)
        b.synchronize()
        dev.append(a.elapsed_time(b))
    return float(np.median(dev)), float(np.median(wall))


def host_kind(fe, cam, prm, lines, q_px, d1, t_geo, d2, ws, kmin, n_cond, fast):
    """The host composition of one kind: grids on the host, plf_match_grid_*, plf_match on fallback."""
    iw, ih = GRID_COLS / cam["width"], GRID_ROWS / cam["height"]
    nnr = prm["min_ratio_12_l"] if lines else prm["min_ratio_12_p"]
    m12, n = np.full(len(d1), -1, np.int32), 0
    if fast:
        w = (ws, ws, ws, ws)
        if lines:
            q = kfm.qcell(q_px * np.array([iw, ih, iw, ih]))
            t_line, t_dir = t_geo
            cs, ci = mg.grid_from_lines(t_line, GRID_ROWS, GRID_COLS).csr()
            m12, n = fe.match_grid_lines(q, d1, cs, ci, t_dir, d2, GRID_COLS, GRID_ROWS, w, nnr, prm["line_sim_th"])
        else:
            q = kfm.qcell(q_px * np.array([iw, ih]))
            cs, ci = mg.grid_from_points(t_geo, GRID_ROWS, GRID_COLS).csr()
            m12, n = fe.match_grid_points(q, d1, cs, ci, d2, GRID_COLS, GRID_ROWS, w, nnr)
    if n_cond > kmin and n < kmin:
        m12, n = fe.match(d1, d2, nnr)
    return m12, n


def host_map2kf(fe, cam, prm, lmap, Twf, kf, fast):
    """matchMap2KFPoints / Lines composed on the host around plf_match_grid_* / plf_match (points and lines)."""
    iw, ih = GRID_COLS / cam["width"], GRID_ROWS / cam["height"]
    ws = prm["matching_f2f_ws"]
    out = []
    for lines in (False, True):
        key = "ls" if lines else "pt"
        X = lmap[key + "_X"]
        if lines:
            ps, pe = kfm.project(cam, kfm.rigid(Twf, X[:, :3])), kfm.project(cam, kfm.rigid(Twf, X[:, 3:]))
            Zs, Ze = kfm.rigid(Twf, X[:, :3])[:, 2], kfm.rigid(Twf, X[:, 3:])[:, 2]
            vis = kfm._visible(cam, ps, Zs) & kfm._visible(cam, pe, Ze)
            q_px = np.concatenate([ps, pe], 1)[vis]
            t_geo = kfm._train_lines(cam, kf["ls_spl"], kf["ls_epl"])
            d2 = kf["ldesc"]
        else:
            P = kfm.rigid(Twf, X)
            ps = kfm.project(cam, P)
            vis = kfm._visible(cam, ps, P[:, 2])
            q_px = ps[vis]
            pl = kf["pt_pl"]
            t_geo = np.stack([kfm.tcell(pl[:, 0] * iw), kfm.tcell(pl[:, 1] * ih)], 1)
            d2 = kf["pdesc"]
        d1 = lmap[key + "_desc"][vis]
        kmin = prm["min_ls_matches" if lines else "min_pt_matches"]
        m12, n = host_kind(fe, cam, prm, lines, q_px, d1, t_geo, d2, ws, kmin, len(q_px), fast)
        j = np.nonzero(m12 >= 0)[0]
        if lines:
            le = kf["ls_le"][m12[j]]
            e0 = le[:, 0] * q_px[j, 0] + le[:, 1] * q_px[j, 1] + le[:, 2]
            e1 = le[:, 0] * q_px[j, 2] + le[:, 1] * q_px[j, 3] + le[:, 2]
            ok = (e0 < 1.0) & (e1 < 1.0)
        else:
            ok = np.hypot(q_px[j, 0] - kf["pt_pl"][m12[j], 0], q_px[j, 1] - kf["pt_pl"][m12[j], 1]) < 1.0
        out.append(n - int((~ok).sum()))
    return out


def host_kf2kf(fe, cam, prm, prev, curr, DT, fast):
    iw, ih = GRID_COLS / cam["width"], GRID_ROWS / cam["height"]
    ws = prm["matching_f2f_ws"]
    ps = kfm.project(cam, kfm.rigid(DT, prev["pt_P"]))
    t = np.stack([kfm.tcell(curr["pt_pl"][:, 0] * iw), kfm.tcell(curr["pt_pl"][:, 1] * ih)], 1)
    host_kind(fe, cam, prm, False, ps, prev["pdesc"], t, curr["pdesc"], ws, prm["min_pt_matches"],
              min(len(prev["pdesc"]), len(curr["pdesc"])), fast)
    s, e = kfm.project(cam, kfm.rigid(DT, prev["ls_sP"])), kfm.project(cam, kfm.rigid(DT, prev["ls_eP"]))
    # matchKF2KFLines' queries stay in pixels: pass them through unscaled
    q = np.concatenate([s, e], 1) * np.array([cam["width"] / GRID_COLS, cam["height"] / GRID_ROWS] * 2)
    host_kind(fe, cam, prm, True, q, prev["ldesc"], kfm._train_lines(cam, curr["ls_spl"], curr["ls_epl"]), curr["ldesc"], ws,
              prm["min_ls_matches"], min(len(prev["ldesc"]), len(curr["ldesc"])), fast)


def cv2_ms(d1, d2, reps):
    import cv2
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        bf.knnMatch(d1, d2, k=2)
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def build_map(T_wc, feats, n_target, rng):
    """About n_target landmarks (lines in the stream's proportion): the keyframes' features in world coordinates, repeated
    with jittered positions and a few flipped descriptor bits."""
    pX = np.concatenate([(T_wc[k][:3, :3] @ f["pt_P"].T).T + T_wc[k][:3, 3] for k, f in enumerate(feats)])
    pD = np.concatenate([f["pdesc"] for f in feats])
    lX = np.concatenate([np.concatenate([(T_wc[k][:3, :3] @ f[s].T).T + T_wc[k][:3, 3] for s in ("ls_sP", "ls_eP")], 1)
                         for k, f in enumerate(feats)])
    lD = np.concatenate([f["ldesc"] for f in feats])
    n_ls = max(1, int(round(n_target * len(lX) / len(pX))))

    def grow(X, D, n):
        i = rng.integers(0, len(X), n)
        flips = np.packbits(rng.random((n, 256)) < 0.03, axis=1)
        return X[i] + rng.normal(0, 0.05, (n, X.shape[1])), (D[i] ^ flips).astype(np.uint8)
    pX, pD = grow(pX, pD, n_target)
    lX, lD = grow(lX, lD, min(n_ls, 65535))
    return dict(pt_X=pX, pt_desc=pD, ls_X=lX, ls_desc=lD)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="2000,8000,32000")
    a = ap.parse_args()
    cam = plf.KITTI_CAMERA
    n_frames = 12
    frames = list(synth.stream(cam, n_frames))
    T_wc = [f[2] for f in frames]
    lim = plf.default_limits(); lim.max_batch = n_frames
    rows = []
    print(f"card: {card()}")
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=1500, lsd_nfeatures=200) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        feats = [fe.get_frame(k) for k in range(n_frames)]
        prm = {k: getattr(fe.params, k) for k, _ in plf.plf_params._fields_}
        for fast in (0, 1):
            pairs = [(k, k + 5) for k in range(n_frames - 5)]
            dev, wall, host = [], [], []
            for (i, j) in pairs:
                DT = np.linalg.inv(T_wc[j]) @ T_wc[i]
                d, w = timed(fe, lambda: fe.match_kf2kf(feats[i], feats[j], DT, fast_matching=fast), a.reps)
                t0 = time.perf_counter()
                for _ in range(3):
                    host_kf2kf(fe, cam, prm, feats[i], feats[j], DT, fast)
                dev.append(d); wall.append(w); host.append((time.perf_counter() - t0) / 3 * 1e3)
            cv = cv2_ms(feats[0]["pdesc"], feats[5]["pdesc"], 5) + cv2_ms(feats[0]["ldesc"], feats[5]["ldesc"], 5)
            rows.append(dict(case="kf2kf d=5", n_query=len(feats[0]["pdesc"]), fast=fast, dev_ms=np.median(dev),
                             wall_ms=np.median(wall), host_ms=np.median(host), cv2_ms=cv))
        rng = np.random.default_rng(0)
        kf = feats[8]
        Twf = np.linalg.inv(T_wc[8])
        for n in [int(s) for s in a.sizes.split(",")]:
            lmap = build_map(T_wc[:8], feats[:8], n, rng)
            for fast in (0, 1):
                d, w = timed(fe, lambda: fe.match_map2kf(lmap, Twf, kf, fast_matching=fast), a.reps)
                try:   # plf_match_grid_* takes at most 8192 queries: larger visible maps have no host composition
                    t0 = time.perf_counter()
                    for _ in range(3):
                        host_map2kf(fe, cam, prm, lmap, Twf, kf, fast)
                    h = (time.perf_counter() - t0) / 3 * 1e3
                except plf.PlfError:
                    h = None
                P = kfm.rigid(Twf, lmap["pt_X"])
                vis = kfm._visible(cam, kfm.project(cam, P), P[:, 2])
                cv = cv2_ms(lmap["pt_desc"][vis], kf["pdesc"], 3)
                rows.append(dict(case=f"map2kf {n}", n_query=int(vis.sum()), n_ls=len(lmap["ls_X"]), fast=fast, dev_ms=d,
                                 wall_ms=w, host_ms=h, cv2_ms=cv))
    print("| case | visible queries (points) | fast_matching | device ms | wall ms | host composition ms | cv2 knnMatch ms |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['case']} | {r['n_query']} | {r['fast']} | {r['dev_ms']:.3f} | {r['wall_ms']:.3f} | "
              f"{'n/a (> 8192 queries)' if r['host_ms'] is None else format(r['host_ms'], '.2f')} | "
              f"{r['cv2_ms']:.2f} |")
    for r in rows:
        print(json.dumps({k: (float(v) if isinstance(v, (np.floating, float)) else v) for k, v in r.items()}))


if __name__ == "__main__":
    main()
