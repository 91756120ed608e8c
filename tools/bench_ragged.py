"""Frames of different sizes in one batch: what one ragged runner gains over one runner per frame size.

    python tools/bench_ragged.py [--frames 20 --warmup 3 --reps 3] [--baseline-tracker FILE]

Dataset case: 64 synthetic VOT sequences (tools/bench_vot.py's make_sequences: a textured rectangle drifting over a
textured background whose gt quad jumps to a far corner every 7th frame) over 8 frame sizes in unequal groups
24/12/8/6/6/4/2/2.  Stream-frames/s of one `VotRunner` over all 64 (frames given as lists) against one `VotRunner` per
size group run one after another on the same frames (today's only option), alternated --reps times.  Packing overhead:
`BatchTracker.track(mask=False)` on 64 streams of one size with the frames given as a list (packed) and as one
[64,H,W,3] tensor.  With --baseline-tracker (siammask_b200/tracker.py of another revision) it also runs bench.py's
`loop` leg with that tracker and with this one, alternated.  Prints one JSON line with the card name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import siammask_b200 as smb                                     # noqa: E402
from siammask_b200.tracker import BatchTracker, TrackerParams   # noqa: E402
from bench_vos import gpu_info, loop_legs                       # noqa: E402
from bench_vot import make_sequences                            # noqa: E402

GROUPS = [((1080, 1920), 24), ((720, 1280), 12), ((480, 854), 8), ((576, 1024), 6), ((360, 640), 6),
          ((540, 960), 4), ((404, 720), 2), ((288, 352), 2)]


def dataset_legs(net, params, T, warmup, reps):
    """Per group: frames [T][n,H,W,3] and gt.  Times frames warmup+1 .. T-1 of one ragged runner and of the per-size
    runners in sequence."""
    groups = []
    for i, ((H, W), n) in enumerate(GROUPS):
        frames, gt = make_sequences(n, T, H, W, seed=i)
        groups.append((frames, gt))
    G = sum(n for _, n in GROUPS)
    timed_frames = T - 1 - warmup

    def ragged():
        r = smb.VotRunner(net, params)
        lists = [[frames[t][j] for frames, _ in groups for j in range(frames[t].shape[0])] for t in range(T)]
        r.open(lists[0], [g for _, gt in groups for g in gt])
        for t in range(1, 1 + warmup):
            r.frame(lists[t])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(1 + warmup, T):
            r.frame(lists[t])
        torch.cuda.synchronize()
        return G * timed_frames / (time.perf_counter() - t0)

    def per_size():
        total = 0.0
        for frames, gt in groups:
            r = smb.VotRunner(net, params)
            r.open(frames[0], gt)
            for t in range(1, 1 + warmup):
                r.frame(frames[t])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for t in range(1 + warmup, T):
                r.frame(frames[t])
            torch.cuda.synchronize()
            total += time.perf_counter() - t0
        return G * timed_frames / total

    out = {"sequences": G, "groups": [[h, w, n] for (h, w), n in GROUPS], "timed_frames": timed_frames,
           "unit": "stream-frames/s", "ragged": [], "per_size": []}
    for _ in range(reps):
        out["ragged"].append(ragged())
        out["per_size"].append(per_size())
    for k in ("ragged", "per_size"):
        out[f"median_{k}"] = float(np.median(out[k]))
        out[f"range_{k}"] = [float(min(out[k])), float(max(out[k]))]
    out["speedup_median"] = out["median_ragged"] / out["median_per_size"]
    return out


def packing_legs(net, params, T, warmup, reps, H=720, W=1280, B=64):
    frames, gt = make_sequences(B, T, H, W, seed=50)
    box = np.asarray([[g[0, 0], g[0, 1], g[0, 2] - g[0, 0], g[0, 5] - g[0, 1]] for g in gt])

    def run(as_list):
        bt = BatchTracker(net, params)
        fr = [[f[j] for j in range(B)] for f in frames] if as_list else frames
        bt.add(fr[0], box)
        for t in range(1, 1 + warmup):
            bt.track(fr[t], mask=False)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(1 + warmup, T):
            bt.track(fr[t], mask=False)
        torch.cuda.synchronize()
        return B * (T - 1 - warmup) / (time.perf_counter() - t0)

    out = {"streams": B, "frame_hw": [H, W], "unit": "stream-frames/s", "list": [], "tensor": []}
    for _ in range(reps):
        out["list"].append(run(True))
        out["tensor"].append(run(False))
    for k in ("list", "tensor"):
        out[f"median_{k}"] = float(np.median(out[k]))
        out[f"range_{k}"] = [float(min(out[k])), float(max(out[k]))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    T = 1 + args.warmup + args.frames
    torch.cuda.set_device(0)
    res = {"metric": "ragged_vot_stream_frames_per_s", **gpu_info()}
    from oracle.calibrate import calibrated_state_dict
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=64, num_slots=64)
    net.load_state_dict(calibrated_state_dict(0)).eval().to("cuda")
    params = TrackerParams(instance_size=255)
    res["dataset"] = dataset_legs(net, params, T, args.warmup, args.reps)
    res["value"] = res["dataset"]["median_ragged"]
    res["unit"] = "stream-frames/s"
    res["packing"] = packing_legs(net, params, T, args.warmup, args.reps)
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
