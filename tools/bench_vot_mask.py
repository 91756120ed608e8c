"""Throughput of VOT in mask mode (siammask_b200.VotRunner(mask=True, refine=True)) with the rotated box on the device,
against the same runner with the rotated box done on the host by cv2 per stream from D2H'd masks (what a user would
otherwise write), against box-mode VotRunner, and the rotated-box kernel's own time per call.

    python tools/bench_vot_mask.py [--sequences 4 --combos 16 --frames 30 --warmup 5 --reps 3]

The workload is tools/bench_vot.py's: G synthetic 1280x720 sequences whose gt quad jumps to a far corner every 7th
frame (each stream fails, skips and re-initialises several times) x K hyper-parameter combinations, 64 streams by
default.  The three runner legs alternate --reps times (medians and ranges, stream-frames/s).  The kernel leg times
`ops._rotated_box` with CUDA events on the 64 pasted 1280x720 masks of one tracked frame.  Prints one JSON line with
the card name and power limit.
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
from siammask_b200 import ops, vot                              # noqa: E402
from siammask_b200.tracker import TrackerParams                 # noqa: E402
from siammask_b200.tune import grid                             # noqa: E402
from bench_vos import gpu_info, timed                           # noqa: E402
from bench_vot import make_sequences                            # noqa: E402


def host_rotated_box(flat, desc, N, max_hw, fallback):
    """The rotated box with cv2 on the host (tools/test.py:284-303 per stream), from the D2H'd packed masks."""
    import cv2
    H, W = max_hw
    masks = flat.view(N, H, W).cpu().numpy().astype(np.uint8)      # one frame size in this workload
    fb = fallback.cpu().numpy()
    out = np.zeros((N, 8))
    for i in range(N):
        cs = cv2.findContours(masks[i], cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)[-2]
        areas = [cv2.contourArea(c) for c in cs]
        if cs and max(areas) > 100:
            out[i] = cv2.boxPoints(cv2.minAreaRect(cs[int(np.argmax(areas))].reshape(-1, 2))).reshape(-1)
        else:
            cx, cy, w, h = fb[i]
            x0, y0 = cx - w / 2, cy - h / 2
            out[i] = [x0, y0, x0 + w, y0, x0 + w, y0 + h, x0, y0 + h]
    dev = flat.device
    return (torch.from_numpy(out).to(dev), torch.zeros(N, dtype=torch.int32, device=dev),
            torch.zeros(N, dtype=torch.int64, device=dev))


def run_leg(net, params, combos, frames, gt, warmup, mask, host=False):
    G, K, T = len(gt), combos.shape[0], len(frames)
    saved = ops._rotated_box
    if host:
        ops._rotated_box = host_rotated_box
    try:
        r = smb.VotRunner(net, params, combos, mask=mask)
        r.open(frames[0], gt)
        for f in range(1, 1 + warmup):
            r.frame(frames[f])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in range(1 + warmup, T):
            r.frame(frames[f])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        ops._rotated_box = saved
    _, lost = r.result()
    return G * K * (T - 1 - warmup) / dt, int(lost.sum())


def kernel_leg(net, params, frames, gt, reps=50):
    """ops._rotated_box on one frame's pasted masks of every stream: ms per call (CUDA events) and the flags."""
    G = len(gt)
    combos = grid([0.04, 0.1, 0.2, 0.3], [0.3, 0.4], [0.35, 0.45])
    r = smb.VotRunner(net, params, combos, mask=True)
    r.open(frames[0], gt)
    res = r.frame(frames[1])
    flat, desc, max_hw = res.extras["packed_mask"]
    N = r.tracker.N
    fb = res.extras["unclamped"].clone()
    for _ in range(5):
        ops._rotated_box(flat, desc, N, max_hw, fb)
    ms = timed(lambda: ops._rotated_box(flat, desc, N, max_hw, fb), reps)
    _, flag, _ = ops._rotated_box(flat, desc, N, max_hw, fb)
    return {"streams": N, "frame_hw": list(max_hw), "ms_per_call": ms, "contour_results": int(flag.sum()),
            "sequences": G}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=4)
    ap.add_argument("--combos", type=int, default=16)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    args = ap.parse_args()
    G, H, W = args.sequences, args.height, args.width
    combos = grid([0.04, 0.1, 0.2, 0.3], [0.3, 0.4], [0.35, 0.45])[:args.combos]
    K = combos.shape[0]
    T = 1 + args.warmup + args.frames
    torch.cuda.set_device(0)
    res = {"metric": "vot_mask_stream_frames_per_s", **gpu_info(), "sequences": G, "combinations": K,
           "streams": G * K, "frame_hw": [H, W], "unit": "stream-frames/s"}
    from oracle.calibrate import calibrated_state_dict
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=G * K, num_slots=G * K)
    net.load_state_dict(calibrated_state_dict(0)).eval().to("cuda")
    frames, gt = make_sequences(G, T, H, W)
    params = TrackerParams(instance_size=255)
    legs = {"mask_device": [], "mask_host_cv2": [], "box": []}
    lost = {}
    for _ in range(args.reps):
        for name, mask, host in (("mask_device", True, False), ("mask_host_cv2", True, True), ("box", False, False)):
            v, lost[name] = run_leg(net, params, combos, frames, gt, args.warmup, mask, host)
            legs[name].append(v)
    for k, v in legs.items():
        res[k] = {"runs": v, "median": float(np.median(v)), "range": [float(min(v)), float(max(v))],
                  "lost_times_total": lost[k]}
    res["value"] = res["mask_device"]["median"]
    res["timed_frames"] = args.frames
    res["kernel"] = kernel_leg(net, params, frames, gt)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
