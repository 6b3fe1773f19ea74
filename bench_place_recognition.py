"""Place-recognition benchmark: one plf_bow_insert (MapHandler::insertKFBowVectorPL's transform + score rows, points and
lines) at database sizes of 100, 1 k, 5 k and 20 k keyframes, against the same work on the host.

The vocabularies are real-shape synthetic ones (k 9, L 6, ~560 k nodes, oracle.dbow.synth_vocab); the keyframes are the
stereo descriptors of frames of the synthetic KITTI-shape stream, cycled.  Per size it reports the device time (CUDA
events on plf_stream around the call) and wall time per insert, the score kernel's time (torch.profiler, a separate run)
and its achieved GB/s over the bytes it must read: per earlier keyframe its 8-byte index entry and its 4-byte words, plus
8 bytes per common word (that keyframe's value).  The host side runs the same per-keyframe work with DBoW2 compiled from
the reference (oracle/_ref/libdbow_ref.so) when it was built, else with oracle/dbow.c, and says which.  Prints the card
name and power limit, then one JSON line.  Writes nothing to the tree."""
import argparse
import ctypes as C
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
from oracle import dbow, synth  # noqa: E402
from oracle.clib import _p, lib as oracle_lib  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def stream_descriptors(n_frames):
    cam = plf.KITTI_CAMERA
    frames = list(synth.stream(cam, n_frames))
    lim = plf.default_limits(); lim.max_batch = n_frames
    with plf.Frontend(camera=cam, limits=lim, orb_nfeatures=1500, lsd_nfeatures=200) as fe:
        fe.process_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        return [(fe.get_frame(k)["pdesc"], fe.get_frame(k)["ldesc"]) for k in range(n_frames)]


class HostDb:
    """insertKFBowVectorP + L on the host: DBoW2 itself when oracle/_ref was built, else oracle/dbow.c."""

    def __init__(self, vocs):
        self.use_ref = dbow.ref_available()
        self.vocs = [dbow.RefVocab(v) if self.use_ref else dbow.Vocab(v) for v in vocs]
        if self.use_ref:
            from oracle import dbow as d
            self.L = d._ref
            self.handles = [v._r for v in self.vocs]
        else:
            self.L = oracle_lib()
            self.handles = [v._h for v in self.vocs]
        self.L_new = self.L.ref_dbow_db_new if self.use_ref else self.L.orc_dbow_db_new
        self.L_new.restype = C.c_void_p
        self.ins = self.L.ref_dbow_db_insert if self.use_ref else self.L.orc_dbow_db_insert
        self.dbs = [C.c_void_p(self.L_new()), C.c_void_p(self.L_new())]
        self.name = "DBoW2 (oracle/_ref/libdbow_ref.so)" if self.use_ref else "oracle/dbow.c (DBoW2 not built)"

    def insert(self, k, descs, score=True):
        for c in range(2):
            d = np.ascontiguousarray(descs[c], np.uint8)
            row = np.empty(k + 1)
            self.ins(self.handles[c], self.dbs[c], _p(d), len(d), _p(row) if score else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100,1000,5000,20000")
    ap.add_argument("--timed", type=int, default=20, help="inserts timed at each size")
    ap.add_argument("--frames", type=int, default=16, help="stream frames whose descriptors are cycled")
    ap.add_argument("--host-max", type=int, default=20000, help="largest size also measured on the host")
    args = ap.parse_args()
    sizes = [int(s) for s in args.sizes.split(",")]
    import torch
    print("card:", card(), flush=True)
    descs = stream_descriptors(args.frames)
    vocs = [dbow.synth_vocab(5), dbow.synth_vocab(6)]
    host = HostDb(vocs)
    print("host:", host.name, flush=True)
    res = []
    with plf.Frontend() as fe:
        for c in range(2):
            fe.bow_set_vocabulary(c, vocs[c])
        stream = torch.cuda.ExternalStream(fe.stream)
        k = 0
        host_k = 0
        for n in sizes:
            while k < n:
                fe.bow_insert(k, *descs[k % len(descs)], rows=(False, False))
                k += 1
            dev_ms, wall_ms = [], []
            for _ in range(args.timed):
                d = descs[k % len(descs)]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                t0 = time.perf_counter()
                fe.bow_insert(k, *d)
                t1 = time.perf_counter()
                e1.record(stream)
                e1.synchronize()
                dev_ms.append(e0.elapsed_time(e1)); wall_ms.append((t1 - t0) * 1e3)
                k += 1
            # score-kernel time and the bytes it must read, at this size
            d = descs[k % len(descs)]
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fe.bow_insert(k, *d)
                torch.cuda.synchronize()
            ktime = sum(e.device_time_total for e in prof.key_averages() if "k_bow_score" in e.key) / 1e3   # ms
            nbytes = 0
            for c in range(2):
                ws = set(fe.bow_vector(k, c)[0].tolist())
                for i in range(k + 1):
                    w = fe.bow_vector(i, c)[0]
                    nbytes += 8 + 4 * len(w) + 8 * len(ws.intersection(w.tolist()))
            k += 1
            entry = dict(size=n, device_ms=float(np.median(dev_ms)), wall_ms=float(np.median(wall_ms)),
                         score_kernel_ms=ktime, score_bytes_est=int(nbytes),
                         score_GBps=(nbytes / (ktime * 1e-3) / 1e9) if ktime > 0 else None)
            if n <= args.host_max:
                while host_k < k - 1:                      # fill: transforms only
                    host.insert(host_k, descs[host_k % len(descs)], score=False)
                    host_k += 1
                ht = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    host.insert(host_k, descs[host_k % len(descs)])
                    ht.append((time.perf_counter() - t0) * 1e3)
                    host_k += 1
                entry["host_ms"] = float(np.median(ht))
            print(json.dumps(entry), flush=True)
            res.append(entry)
    print(json.dumps(dict(bench="place_recognition", card=card(), host=host.name, results=res)))


if __name__ == "__main__":
    main()
