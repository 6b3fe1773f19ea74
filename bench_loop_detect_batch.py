#!/usr/bin/env python
"""bench_loop_detect_batch.py - loop-closure candidate detection for the new keyframes of P sequences: the scores
downloaded and combined and searched on the host, against one plf_bow_detect_batch call.

Inputs: those of bench_place_recognition_batch.py (the real-shape synthetic vocabularies, 16 frames of the synthetic
KITTI-shape stream cycled as keyframe d of sequence p = frame (7 p + d) mod 16), with each frame's stereo coordinates.
Every sequence holds D earlier keyframes before the timed steps; both kinds are enabled, so the PL combination applies.
Covisibility is all zero and the options are SlamConfig's defaults.

Arms, for each P in --batch (default 1, 8, 64, 256) and D in --depth (default 100, 1000), alternated within each step,
each on its own context holding the same databases:
  host:   plf_bow_insert_batch with both rows, then the dispersions, the conf column and lookForLoopCandidates restated
          in numpy (sequential sums via cumsum; ties at the maximum to the lowest index, as the device);
  device: one plf_bow_detect_batch returning the results only.
Reported per arm: device ms (CUDA events on plf_stream around the arm; the host arm's numpy runs inside it), wall ms
(host clock around the arm), the bytes of the call's one device-to-host copy (download_bytes, from its staged layout:
each region starts at a 256-byte boundary; the host arm copies the counts' region and every row of kf_idx + 1 doubles,
the device arm the counts' and the results' regions) and kernel launches; medians over --steps steps after --warmup.  The candidates of the two arms are asserted
equal.  Prints the GPU's name and power limit, then one JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import sys
import time

import numpy as np

from bench_multi_sequence import gpu_info

N_FRAMES = 16
FILL_CHUNK = 2048


def align256(b):
    return (b + 255) // 256 * 256


def download_bytes(P, kf_idx, detect):
    """The one device-to-host copy of plf_bow_insert_batch with both rows (detect False) or of plf_bow_detect_batch
    with no row and no column requested (detect True), for P problems at kf_idx: the per-problem counts (8 bytes each),
    then the rows, or then the results (24 bytes each), every region 256-byte aligned."""
    return align256(8 * P) + (align256(24 * P) if detect else 2 * 8 * (kf_idx + 1) * P)


def stream_keyframes(plf, synth):
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, N_FRAMES))
    lim = plf.default_limits(); lim.max_batch = N_FRAMES
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=1500, lsd_nfeatures=200) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        return [{k: v for k, v in fe.get_frame(i).items() if k in ("pdesc", "ldesc", "pt_pl", "ls_spl", "ls_epl")}
                for i in range(N_FRAMES)]


def kf(frames, p, d, idx):
    return dict(frames[(7 * p + d) % N_FRAMES], kf_idx=idx)


def stdv(x):
    n = len(x)
    if n == 0:
        return 0.0
    mean = np.cumsum(x)[-1] / n
    with np.errstate(all="ignore"):
        return float(np.sqrt(np.cumsum((x - mean) * (x - mean))[-1] / np.float64(n - 1)))


def host_detect(pr, sp, sl, o):
    """The conf column of insertKFBowVectorPL and lookForLoopCandidates, in numpy; returns the candidate."""
    k = pr["kf_idx"]
    pt, s, e = pr["pt_pl"], pr["ls_spl"], pr["ls_epl"]
    mid = (s + e) * 0.5
    std_pt, std_ls = stdv(pt[:, 0]) + stdv(pt[:, 1]), stdv(mid[:, 0]) + stdv(mid[:, 1])
    n_pt, n_ls = len(pt), len(mid)
    live = ~np.isnan(sp) & ~np.isnan(sl)
    with np.errstate(all="ignore"):
        score = (0.0 + (sp * n_pt + sl * n_ls) / np.float64(n_pt + n_ls)) + (sp * std_pt + sl * std_ls) / (std_ls + std_pt)
    conf = np.where(live, score, np.nan).astype(np.float32).astype(np.float64)
    idx = np.arange(k + 1)
    listed = live & (idx < k - o["lc_kf_dist"])
    if listed.sum() <= o["lc_kf_max_dist"]:
        return -1
    sc = np.where(live, conf, 0.0)
    near = (idx < k) & ((k - idx) <= o["min_kf_local_map"] + 3)   # covisibility all zero
    cand = sc[near & (sc > 0.001) & (sc < 1.0)]
    mn = float(cand.min()) if len(cand) else 1.0
    ls = np.where(listed & ~np.isnan(conf), conf, -np.inf)
    best = int(np.argmax(ls)) if np.any(listed & ~np.isnan(conf)) else int(np.argmax(listed))
    if not conf[best] >= mn:
        return -1
    close = listed & (idx != best) & (np.abs(idx - best) <= o["lc_kf_max_dist"]) & (conf >= mn * 0.8)
    return best if int(close.sum()) >= o["lc_nkf_closest"] else -1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 64, 256])
    ap.add_argument("--depth", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--steps", type=int, default=5, help="timed steps per (P, D)")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import plslam_b200 as plf
    from oracle import dbow
    from plslam_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_loop_detect_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", file=sys.stderr, flush=True)
    frames = stream_keyframes(plf, synth)
    vocs = [dbow.synth_vocab(5), dbow.synth_vocab(6)]
    o = dict(plf.LC_DETECT_DEFAULTS)
    results = []
    for D in args.depth:
        for P in args.batch:
            with plf.Frontend(device=0, max_sequences=P) as fa, plf.Frontend(device=0, max_sequences=P) as fb:
                seq = list(range(P))
                for f in (fa, fb):
                    for c in range(2):
                        f.bow_set_vocabulary(c, vocs[c])
                    probs = [kf(frames, p, d, d) for d in range(D) for p in range(P)]
                    sq = [p for d in range(D) for p in range(P)]
                    for i in range(0, len(probs), FILL_CHUNK):
                        f.bow_insert_batch(probs[i:i + FILL_CHUNK], seq=sq[i:i + FILL_CHUNK], rows=(False, False))
                rec = {k: dict(dev=[], wall=[], launches=0, bytes=[]) for k in ("host", "device")}
                n_cand = 0
                for t in range(args.warmup + args.steps):
                    d = D + t
                    new = [kf(frames, p, d, d) for p in range(P)]
                    out = {}

                    def host():
                        rows = fa.bow_insert_batch(new, seq=seq)
                        return rows, [host_detect(pr, r[0], r[1], o) for pr, r in zip(new, rows)]

                    def device():
                        return fb.bow_detect_batch(new, o, seq=seq, conf=False), None
                    for name, (f, run) in (("host", (fa, host)), ("device", (fb, device))):
                        stream = torch.cuda.ExternalStream(f.stream)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        f.sync()
                        n0 = f.launches
                        w0 = time.perf_counter()
                        e0.record(stream)
                        a, b = run()
                        e1.record(stream)
                        wall = (time.perf_counter() - w0) * 1e3
                        e1.synchronize()
                        out[name] = b if name == "host" else [r["candidate"] for r in a]
                        if t >= args.warmup:
                            rec[name]["dev"].append(e0.elapsed_time(e1))
                            rec[name]["wall"].append(wall)
                            rec[name]["launches"] = f.launches - n0
                            rec[name]["bytes"].append(download_bytes(P, d, name == "device"))
                    assert out["host"] == out["device"], (P, D, t, out["host"], out["device"])
                    n_cand += sum(c >= 0 for c in out["device"])
                entry = dict(P=P, D=D, steps=args.steps, candidates=n_cand)
                for name, r in rec.items():
                    entry[name] = dict(device_ms=round(float(np.median(r["dev"])), 3),
                                       wall_ms=round(float(np.median(r["wall"])), 3),
                                       download_bytes=int(np.median(r["bytes"])),
                                       launches=r["launches"])
                print(json.dumps(entry), file=sys.stderr, flush=True)
                results.append(entry)
    print(json.dumps(dict(bench="loop_detect_batch", gpu=info, results=results)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
