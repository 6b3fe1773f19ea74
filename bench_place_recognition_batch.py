#!/usr/bin/env python
"""bench_place_recognition_batch.py - the new keyframes of P sequences inserted and scored one call each in one shared
database (plf_bow_insert), against one plf_bow_insert_batch call into each sequence's own database.

Inputs: the real-shape synthetic vocabularies (oracle.dbow.synth_vocab(5) for points, (6) for lines; k 9, L 6, about
560 k nodes each) and the stereo descriptors of 16 frames of the synthetic KITTI-shape stream, cycled: keyframe d of
sequence p uses frame (7 p + d) mod 16.  Every sequence holds D earlier keyframes before the timed steps.

Arms, for each P in --batch (default 1, 8, 64, 256) and D in --depth (default 100, 1000), alternated within each step so
that they share the card's state:
  shared: one context whose single database holds all P * D keyframes, sequence p's keyframe d at index d * P + p (the
          multi-sequence workaround: every row covers every sequence); the step's P keyframes are P plf_bow_insert calls.
  batch:  a context with max_sequences = P, sequence p's keyframes at 0 .. D - 1 of its own database; the step's P
          keyframes are one plf_bow_insert_batch with seq[p] = p.
Both arms request both rows (points and lines).  Reported per arm: device ms (CUDA events on plf_stream around the
arm), wall ms (host clock, including the binding's marshalling), keyframes inserted per second over the wall time and
kernel launches per arm (plf_launch_count); medians over --steps steps after --warmup.  Also the vocabulary bytes one
context holds on the device (48 per node and kind) and what P contexts, one per sequence, would hold (computed, not
allocated).  Every batch row is asserted bit-identical to the shared arm's row restricted to that sequence's indices.
Prints the GPU's name and power limit, then one JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import sys
import time

import numpy as np

from bench_multi_sequence import gpu_info

N_FRAMES = 16
FILL_CHUNK = 2048   # problems per filling call


def stream_descriptors(plf, synth):
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, N_FRAMES))
    lim = plf.default_limits(); lim.max_batch = N_FRAMES
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=1500, lsd_nfeatures=200) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        return [(fe.get_frame(k)["pdesc"], fe.get_frame(k)["ldesc"]) for k in range(N_FRAMES)]


def kf(descs, p, d, idx):
    pd, ld = descs[(7 * p + d) % N_FRAMES]
    return dict(kf_idx=idx, pdesc=pd, ldesc=ld)


def fill(fe, problems, seq):
    for i in range(0, len(problems), FILL_CHUNK):
        fe.bow_insert_batch(problems[i:i + FILL_CHUNK], seq=None if seq is None else seq[i:i + FILL_CHUNK],
                            rows=(False, False))


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
        raise SystemExit("bench_place_recognition_batch.py: no CUDA device; the library has no CPU fallback")
    info = gpu_info()
    print(f"GPU: {info}", file=sys.stderr, flush=True)
    descs = stream_descriptors(plf, synth)
    vocs = [dbow.synth_vocab(5), dbow.synth_vocab(6)]
    voc_bytes = 48 * sum(len(v["node_id"]) for v in vocs)
    results = []
    for D in args.depth:
        for P in args.batch:
            with plf.Frontend(device=0) as fa, plf.Frontend(device=0, max_sequences=P) as fb:
                for f in (fa, fb):
                    for c in range(2):
                        f.bow_set_vocabulary(c, vocs[c])
                fill(fa, [kf(descs, p, d, d * P + p) for d in range(D) for p in range(P)], None)
                fill(fb, [kf(descs, p, d, d) for d in range(D) for p in range(P)], [p for d in range(D) for p in range(P)])
                seq = list(range(P))
                rec = {k: dict(dev=[], wall=[], launches=0) for k in ("shared", "batch")}
                for t in range(args.warmup + args.steps):
                    d = D + t
                    new = [kf(descs, p, d, 0) for p in range(P)]
                    arms = {"shared": (fa, lambda: [fa.bow_insert(d * P + p, new[p]["pdesc"], new[p]["ldesc"]) for p in range(P)]),
                            "batch": (fb, lambda: fb.bow_insert_batch([dict(x, kf_idx=d) for x in new], seq=seq))}
                    out = {}
                    for name, (f, run) in arms.items():
                        stream = torch.cuda.ExternalStream(f.stream)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        f.sync()
                        n0 = f.launches
                        w0 = time.perf_counter()
                        e0.record(stream)
                        out[name] = run()
                        e1.record(stream)
                        wall = (time.perf_counter() - w0) * 1e3
                        e1.synchronize()
                        if t >= args.warmup:
                            rec[name]["dev"].append(e0.elapsed_time(e1))
                            rec[name]["wall"].append(wall)
                            rec[name]["launches"] = f.launches - n0
                    # each sequence's batch row is the shared row at that sequence's indices, bit for bit
                    for p in range(P):
                        for c in range(2):
                            a, b = out["shared"][p][c][p::P], out["batch"][p][c]
                            assert a.tobytes() == b.tobytes(), (P, D, t, p, c)
                entry = dict(P=P, D=D, steps=args.steps, vocab_bytes_one_context=voc_bytes,
                             vocab_bytes_P_contexts=P * voc_bytes)
                for name, r in rec.items():
                    wall = float(np.median(r["wall"]))
                    entry[name] = dict(device_ms=round(float(np.median(r["dev"])), 3), wall_ms=round(wall, 3),
                                       keyframes_per_s=round(P / (wall * 1e-3), 1), launches=r["launches"])
                print(json.dumps(entry), file=sys.stderr, flush=True)
                results.append(entry)
    print(json.dumps(dict(bench="place_recognition_batch", gpu=info, results=results)), flush=True)


if __name__ == "__main__":
    sys.exit(main())
