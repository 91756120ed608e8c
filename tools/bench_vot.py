"""Throughput of the VOT protocol on the device (siammask_b200.VotRunner) against the tracker step it wraps, and of the
region overlap `sm_vot_overlap` against the reference's host path (copy the predictions to the host, then call the
compiled region.c once per pair).

    python tools/bench_vot.py [--sequences 4 --combos 16 --frames 30 --warmup 5 --reps 3] [--baseline-tracker FILE]

G synthetic 1280x720 sequences (one textured rectangle drifting over a textured background; its gt quad jumps to a far
corner every 7th frame, so each stream fails, skips and re-initialises several times) x K hyper-parameter combinations,
64 streams by default.  Prints one JSON line: the card name and power limit (read-only nvidia-smi query),
stream-frames/s of `VotRunner.frame` and of `BatchTracker.track(mask=False)` alone on the same frames, alternated
--reps times (medians and ranges), and the time of one 256-pair overlap call on the device against the D2H copy plus the
host loop (skipped, and said so, when oracle/_ref/libvot_region.so was not built).  With --baseline-tracker (a
siammask_b200/tracker.py from another revision) it also runs bench.py's `loop` leg with that tracker and with this one,
alternated.
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
from siammask_b200 import ops                                   # noqa: E402
from siammask_b200.tracker import BatchTracker, TrackerParams   # noqa: E402
from siammask_b200.tune import grid                             # noqa: E402
from bench_vos import gpu_info, loop_legs, timed                # noqa: E402


def make_sequences(G, T, H, W, seed=0, fail_every=7):
    """uint8 frames [T][G,H,W,3] on the device and gt float64 [G][T,8] (axis-aligned quads of the rectangle)."""
    rng = np.random.RandomState(seed)
    bg = torch.from_numpy(np.kron((rng.rand(G, H // 8 + 1, W // 8 + 1, 3) * 255).astype(np.uint8),
                                  np.ones((1, 8, 8, 1), np.uint8))[:, :H, :W]).to("cuda")
    size = rng.randint(70, 130, (G, 2))
    start = rng.rand(G, 2) * [W - 300, H - 250] + [60, 50]
    vel = rng.randn(G, 2) * 4
    tex = [torch.from_numpy(np.kron((rng.rand(size[g, 1] // 8 + 1, size[g, 0] // 8 + 1, 3) * 255).astype(np.uint8),
                                    np.ones((8, 8, 1), np.uint8))[:size[g, 1], :size[g, 0]]).to("cuda") for g in range(G)]
    frames, gt = [], np.zeros((G, T, 8))
    for t in range(T):
        f = bg.clone()
        for g in range(G):
            x, y = np.clip(start[g] + vel[g] * t, 0, [W - size[g, 0], H - size[g, 1]]).astype(int)
            f[g, y:y + size[g, 1], x:x + size[g, 0]] = tex[g]
            w, h = size[g]
            gt[g, t] = [x, y, x + w, y, x + w, y + h, x, y + h]
            if t and (t + g) % fail_every == 0:
                gt[g, t] = [0, 0, 10, 0, 10, 10, 0, 10]
        frames.append(f)
    return frames, list(gt)


def throughput_legs(net, params, combos, frames, gt, warmup, reps):
    """Alternated runs of VotRunner.frame and of BatchTracker.track(mask=False) over the same frames."""
    G, K, T = len(gt), combos.shape[0], len(frames)
    n = T - 1 - warmup

    def runner():
        r = smb.VotRunner(net, params, combos)
        r.open(frames[0], gt)
        for f in range(1, 1 + warmup):
            r.frame(frames[f])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in range(1 + warmup, T):
            r.frame(frames[f])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        _, lost = r.result()
        return G * K * n / dt, int(lost.sum())

    def tracker():
        bt = BatchTracker(net, params)
        video = np.repeat(np.arange(G), K)
        box = np.asarray([[g[0, 0], g[0, 1], g[0, 2] - g[0, 0], g[0, 5] - g[0, 1]] for g in gt])
        bt.add(frames[0], box[video], frame_index=video, hp=np.tile(combos, (G, 1)))
        for f in range(1, 1 + warmup):
            bt.track(frames[f], mask=False)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in range(1 + warmup, T):
            bt.track(frames[f], mask=False)
        torch.cuda.synchronize()
        return G * K * n / (time.perf_counter() - t0)

    out = {"runner": [], "track_only": [], "unit": "stream-frames/s", "timed_frames": n}
    for _ in range(reps):
        v, lost = runner()
        out["runner"].append(v)
        out["track_only"].append(tracker())
    out["lost_times_total"] = lost
    for k in ("runner", "track_only"):
        out[f"median_{k}"] = float(np.median(out[k]))
        out[f"range_{k}"] = [float(min(out[k])), float(max(out[k]))]
    return out


def overlap_legs(H, W, B=256, reps=200):
    rng = np.random.RandomState(1)
    cx, cy = rng.uniform(100, W - 100, B), rng.uniform(100, H - 100, B)
    w, h = rng.uniform(20, 200, B), rng.uniform(20, 200, B)
    gt = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy - h / 2, cx + w / 2, cy + h / 2, cx - w / 2, cy + h / 2], 1)
    pred = gt + rng.uniform(-15, 15, (B, 8))
    a = torch.from_numpy(gt.astype(np.float32)).cuda()
    b = torch.from_numpy(pred.astype(np.float32)).cuda()
    dev = ops.vot_overlap(a, b, (H, W))
    out = {"pairs": B, "frame_hw": [H, W], "device_ms": timed(lambda: ops._vot_overlap(a, b, (H, W)), reps)}
    from oracle import build_ref
    lib = build_ref.load()
    if lib is None:
        out["host_ms"] = "not measured: oracle/_ref/libvot_region.so was not built (no reference tree)"
        return out

    def host():
        pa, pb = a.cpu().numpy(), b.cpu().numpy()
        return np.asarray([lib.overlap(pa[i], pb[i], W, H) for i in range(B)], np.float32)
    host()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        ref = host()
    out["host_ms"] = 1e3 * (time.perf_counter() - t0) / 5
    out["identical"] = bool((dev.cpu().numpy().view(np.uint32) == ref.view(np.uint32)).all())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=4)
    ap.add_argument("--combos", type=int, default=16)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    G, H, W = args.sequences, args.height, args.width
    combos = grid([0.04, 0.1, 0.2, 0.3], [0.3, 0.4], [0.35, 0.45])[:args.combos]
    K = combos.shape[0]
    T = 1 + args.warmup + args.frames
    torch.cuda.set_device(0)
    res = {"metric": "vot_stream_frames_per_s", **gpu_info(), "sequences": G, "combinations": K, "streams": G * K,
           "frame_hw": [H, W]}
    from oracle.calibrate import calibrated_state_dict
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=G * K, num_slots=G * K)
    net.load_state_dict(calibrated_state_dict(0)).eval().to("cuda")
    frames, gt = make_sequences(G, T, H, W)
    res["frame"] = throughput_legs(net, TrackerParams(instance_size=255), combos, frames, gt, args.warmup, args.reps)
    res["value"] = res["frame"]["median_runner"]
    res["unit"] = "stream-frames/s"
    res["overlap"] = overlap_legs(H, W)
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
