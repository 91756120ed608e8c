"""Whole VOS datasets through one engine: `VideoSegmenter.open_queue` against what a user must do without it, one
`open` per (length, frame size) group run one after another, on the same seeded workloads in the same process.

    python tools/bench_vos_queue.py [--reps 3 --max-batch 64] [--baseline-tracker FILE]
    python tools/bench_vos_queue.py --count-only          # host only: the step counts of both plans, no GPU

Both workloads use the seeded synthetic video of oracle/synthetic_video.py: each video cycles a pool of 8 frames of a
textured 48x64 target drifting over a textured background, kept on the device (decoding and host memory stay out of the
timing).  The target is cut into horizontal stripes, one object per stripe (ids 1..n), drawn in every annotation.
  davis: 30 videos of 25-105 frames with 1-5 objects, all starting at frame 0, mostly 854x480 plus 960x540 and 640x360,
         score="whole".  Baseline: one `open` per (length, size) group.
  ytvos: 40 videos of 20-100 frames with 1-6 objects that start and end part-way through their video, 1280x720,
         854x480 and 640x360, score="spans"; more objects than max_batch.  Baseline: one `open` per (length, size)
         group, split into chunks whose objects fit the engine at once.

Prints one JSON line: the card name and power limit (read-only nvidia-smi query in the same call), per workload the
step counts of both plans, the wall times of --reps alternated runs (host clock around work that ends in a device
synchronise; medians and ranges), object-frames/s (an object-frame: one object initialised or tracked at one frame),
and whether both give identical scores and label maps (checked in one more, untimed run of each).  With
--baseline-tracker (a siammask_b200/tracker.py from another revision) it also runs bench.py's `loop` leg with that
tracker and with this one, alternated.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle.synthetic_video import make_frames                 # noqa: E402
from siammask_b200 import schedule                              # noqa: E402
from siammask_b200.vos import peak_width                        # noqa: E402

POOL = [0, 1, 2, 3, 4, 5, 6, 7, 6, 5, 4, 3, 2, 1]          # frame t of a video is pool frame POOL[t % 14]


def davis_workload():
    """(lengths [G], sizes [G] of (H, W), objects (video, id, start, end))."""
    rng = np.random.default_rng(0)
    G = 30
    T = rng.integers(25, 106, G)
    sizes = [(540, 960) if g % 15 == 7 else (360, 640) if g % 15 == 14 else (480, 854) for g in range(G)]
    objs = [(g, k + 1, 0, int(T[g]) - 1) for g in range(G) for k in range(int(rng.integers(1, 6)))]
    return T.astype(np.int64), sizes, objs


def ytvos_workload():
    rng = np.random.default_rng(1)
    G = 40
    T = rng.integers(20, 101, G)
    all_sizes = [(720, 1280), (480, 854), (360, 640)]
    sizes = [all_sizes[g % 3] for g in range(G)]
    objs = []
    for g in range(G):
        for k in range(int(rng.integers(1, 7))):
            s = 0 if k == 0 else int(rng.integers(0, T[g] * 2 // 3))
            e = int(T[g]) - 1 if rng.random() < 0.6 else int(rng.integers(s, T[g]))
            objs.append((g, k + 1, s, e))
    return T.astype(np.int64), sizes, objs


def widths(T, objs):
    return np.array([peak_width([o[2] for o in objs if o[0] == g], [o[3] for o in objs if o[0] == g])
                     for g in range(len(T))], np.int64)


def groups(T, sizes, objs, capacity):
    """The baseline's runs: videos grouped by (length, size) in index order, each group cut into chunks whose summed
    peak widths fit the engine.  Returns lists of video indices."""
    w = widths(T, objs)
    keyed = {}
    for g in range(len(T)):
        keyed.setdefault((int(T[g]), sizes[g]), []).append(g)
    runs = []
    for vids in keyed.values():
        cur, used = [], 0
        for g in vids:
            if cur and used + w[g] > capacity:
                runs.append(cur)
                cur, used = [], 0
            cur.append(g)
            used += int(w[g])
        runs.append(cur)
    return runs


def counts(T, sizes, objs, capacity) -> dict:
    w = widths(T, objs)
    steps = schedule.plan(T, 1, capacity, w)
    runs = groups(T, sizes, objs, capacity)
    active = [sum(1 for o in objs if o[0] == g and o[2] <= t <= o[3]) for st in steps for g, t in st.need]
    return {"videos": len(T), "objects": len(objs), "frames": int(T.sum()),
            "object_frames": int(sum(o[3] - o[2] + 1 for o in objs)), "peak_widths_sum": int(w.sum()),
            "queue_steps": len(steps), "grouped_runs": len(runs),
            "grouped_steps": int(sum(int(T[r[0]]) for r in runs)),
            "queue_mean_objects_per_step": float(np.sum(active) / len(steps))}


# ---------------------------------------------------------------------------------------------- GPU legs
def make_pools(T, sizes, objs):
    """Per video: 8 uint8 CUDA frames [H,W,3] and their label maps [H,W] (the target cut into one stripe per object)."""
    import torch
    pools = []
    for g in range(len(T)):
        H, W = sizes[g]
        frames, boxes = make_frames(n=8, h=H, w=W, seed=g)
        n = sum(1 for o in objs if o[0] == g)
        annos = []
        for (x, y, w, h) in boxes:
            a = np.zeros((H, W), np.uint8)
            cut = np.linspace(0, h, n + 1).round().astype(int)
            for k in range(n):
                a[y + cut[k]:y + cut[k + 1], x:x + w] = k + 1
            annos.append(torch.from_numpy(a).cuda())
        pools.append(([torch.from_numpy(f).cuda() for f in frames], annos))
    return pools


def frame_of(pools, g, t):
    return pools[g][0][POOL[t % len(POOL)]]


def anno_of(pools, g, t):
    return pools[g][1][POOL[t % len(POOL)]]


def run_queue(net, params, T, objs, pools, score, check=False):
    """One queue run; returns (result(), per-video label checksums or None)."""
    import torch
    import siammask_b200 as smb
    seg = smb.VideoSegmenter(net, params).open_queue(objs, T, score=score)
    sums = [torch.zeros((), dtype=torch.int64, device="cuda") for _ in T] if check else None
    while seg.pending:
        need, want = seg.needed(), seg.needs_anno()
        labels = seg.step([frame_of(pools, g, t) for g, t in need],
                          [anno_of(pools, g, t) if w else None for (g, t), w in zip(need, want)])
        if check:
            for (g, t), lab in zip(need, labels):
                sums[g] += _checksum(lab, t)
    return seg.result(), sums


def _checksum(lab, t):
    import torch
    idx = torch.arange(1, lab.numel() + 1, device=lab.device, dtype=torch.int64)
    return ((lab.reshape(-1).to(torch.int64) * idx).sum() * (t + 1)) % 1000000007


def run_grouped(net, params, T, objs, pools, runs, score, check=False):
    """One `open` per run of videos of one (length, size), frames stacked per video; returns per-video results and
    label checksums as `run_queue`."""
    import torch
    import siammask_b200 as smb
    res, sums = [None] * len(T), [torch.zeros((), dtype=torch.int64, device="cuda") for _ in T] if check else None
    for vids in runs:
        local = {g: i for i, g in enumerate(vids)}
        ol = [(local[o[0]],) + tuple(o[1:]) for o in objs if o[0] in local]
        seg = smb.VideoSegmenter(net, params).open(ol, num_frames=int(T[vids[0]]), num_videos=len(vids), score=score)
        for t in range(int(T[vids[0]])):
            lab = seg.frame(torch.stack([frame_of(pools, g, t) for g in vids]),
                            torch.stack([anno_of(pools, g, t) for g in vids]))
            if check:
                for i, g in enumerate(vids):
                    sums[g] += _checksum(lab[i], t)
        for i, g in enumerate(vids):
            res[g] = seg.result()[i]
    return res, sums


def alternate(legs, reps):
    import torch
    times = {k: [] for k in legs}
    for _ in range(reps):
        for name, fn in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            print(f"{name}: {times[name][-1]:.2f} s", file=sys.stderr, flush=True)
    return times


def summary(times, object_frames):
    out = {}
    for name, ts in times.items():
        out[name] = {"seconds": ts, "median_s": float(np.median(ts)), "range_s": [min(ts), max(ts)],
                     "object_frames_per_s": object_frames / float(np.median(ts)),
                     "range_object_frames_per_s": [object_frames / max(ts), object_frames / min(ts)]}
    return out


def leg(net, params, B, workload, score, reps):
    import torch
    T, sizes, objs = workload
    out = counts(T, sizes, objs, B)
    runs = groups(T, sizes, objs, B)
    pools = make_pools(T, sizes, objs)
    wT = np.array([min(int(T[g]), 12) for g in range(3)], np.int64)         # warm-up: the first 3 videos, cut short
    wobjs = [(g, k, s, min(e, int(wT[g]) - 1)) for (g, k, s, e) in objs if g < 3 and s < wT[g]]
    run_queue(net, params, wT, wobjs, pools, score)
    run_grouped(net, params, wT, wobjs, pools, groups(wT, sizes[:3], wobjs, B), score)
    times = alternate({"queue": lambda: run_queue(net, params, T, objs, pools, score),
                       "grouped": lambda: run_grouped(net, params, T, objs, pools, runs, score)}, reps)
    out.update(summary(times, out["object_frames"]))
    (qr, qs), (gr, gs) = (run_queue(net, params, T, objs, pools, score, check=True),
                          run_grouped(net, params, T, objs, pools, runs, score, check=True))
    out["identical_scores"] = bool(all(np.array_equal(a, b, equal_nan=True) for a, b in zip(qr, gr)))
    out["identical_labels"] = bool(all(int(a) == int(b) for a, b in zip(qs, gs)))
    out["nan_rows"] = int(sum(np.isnan(r).all(1).sum() for r in qr))
    del pools
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count-only", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--legs", default="davis,ytvos", help="comma-separated subset of davis, ytvos")
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    work = {"davis": (davis_workload(), "whole"), "ytvos": (ytvos_workload(), "spans")}
    legs = args.legs.split(",")
    res = {"metric": "vos_queue_vs_grouped", "max_batch": args.max_batch}
    if args.count_only:
        for name in legs:
            res[name] = counts(*work[name][0], args.max_batch)
        print(json.dumps(res))
        return
    import torch
    from bench_queue import build_net
    from bench_vos import gpu_info, loop_legs
    from siammask_b200.tracker import TrackerParams
    torch.cuda.set_device(0)
    res.update(gpu_info())
    net, B = build_net(args.max_batch)
    res["max_batch"], res["reps"] = B, args.reps
    params = TrackerParams(instance_size=255, out_size=127)
    for name in legs:
        res[name] = leg(net, params, B, work[name][0], work[name][1], args.reps)
        res[name]["score"] = work[name][1]
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
