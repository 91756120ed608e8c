"""Throughput of multi-object video segmentation (siammask_b200.VideoSegmenter) on one GPU, and the fused label map
(`sm_paste_labels`) against the unfused path (per-object `sm_warp_affine` frames + torch stack / argmax / threshold).

    python tools/bench_vos.py [--videos 16 --objects 4 --frames 20 --warmup 3] [--baseline-tracker FILE]

G videos x K objects at 854x480 (DAVIS resolution), synthetic textured frames and label maps.  Prints one JSON line:
the card name and power limit (read-only nvidia-smi query), object-frames/s of the whole `VideoSegmenter.frame`, the
time of the fused and the unfused label map and whether their labels are identical.  With --baseline-tracker (a
siammask_b200/tracker.py from another revision) it also runs bench.py's `loop` leg (BatchTracker, 64 streams) with
that tracker and with this one, alternated, --loop-reps times each.

Traffic of the label map, from shapes only: the unfused path writes and re-reads a f32 frame per object (4*H*W bytes,
1.6 MB at 854x480); the fused path writes H*W bytes per video and reads the 64 KB 127x127 mask of each object.
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import siammask_b200 as smb                                     # noqa: E402
from siammask_b200 import ops                                   # noqa: E402
from siammask_b200.ops import OBJ_TRACKED                       # noqa: E402
from siammask_b200.tracker import TrackerParams                 # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as exc:                                   # the numbers are still reported, marked unidentified
        return {"gpu": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(exc)}


def make_videos(G, K, T, H, W, seed=0):
    """uint8 frames [T][G,H,W,3] on the device and the frame-0 label maps [G,H,W]: K textured rectangles per video
    drifting over a textured background."""
    rng = np.random.RandomState(seed)
    dev = "cuda"
    bg = torch.from_numpy(np.kron((rng.rand(G, H // 8 + 1, W // 8 + 1, 3) * 255).astype(np.uint8),
                                  np.ones((1, 8, 8, 1), np.uint8))[:, :H, :W]).to(dev)
    start = rng.rand(G, K, 2) * [W - 160, H - 140] + [20, 20]
    vel = rng.randn(G, K, 2) * 3
    size = rng.randint(50, 110, (G, K, 2))
    tex = [[torch.from_numpy((rng.rand(size[g, k, 1], size[g, k, 0], 3) * 255).astype(np.uint8)).to(dev)
            for k in range(K)] for g in range(G)]
    frames, anno0 = [], torch.zeros(G, H, W, dtype=torch.uint8, device=dev)
    for t in range(T):
        f = bg.clone()
        for g in range(G):
            for k in range(K):
                x, y = np.clip(start[g, k] + vel[g, k] * t, 0, [W - size[g, k, 0], H - size[g, k, 1]]).astype(int)
                f[g, y:y + size[g, k, 1], x:x + size[g, k, 0]] = tex[g][k]
                if t == 0:
                    anno0[g, y:y + size[g, k, 1], x:x + size[g, k, 0]] = k + 1
        frames.append(f)
    return frames, anno0


def timed(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def label_map_legs(seg, G, K, H, W, thr, reps=50):
    r = seg.last
    masks, maps = r.extras["mask_prob"], r.extras["maps"].clone()
    rows = {sid: i for i, sid in enumerate(r.extras["ids"])}
    order = [rows[seg._sid[k]] for k in seg.order]              # row of each (video, object) in video-major order
    table = torch.tensor([(OBJ_TRACKED, i) for i in order], dtype=torch.int32, device="cuda")
    off = torch.arange(0, G * K + 1, K, dtype=torch.int32, device="cuda")
    perm = torch.tensor(order, device="cuda")

    def fused():                     # the tables are fixed: no per-call host check of the offsets (as VideoSegmenter)
        return ops._paste_labels(masks, maps, None, off, table, (H, W), thr)

    def unfused():
        pasted = ops.warp_affine(masks, maps, (W, H), -1.0)[perm].view(G, K, H, W)
        mx, am = pasted.max(dim=1)
        return ((am + 1) * (mx.double() > thr)).to(torch.uint8)

    same = bool(torch.equal(fused(), unfused()))
    return {"fused_ms": timed(fused, reps), "unfused_ms": timed(unfused, reps), "labels_identical": same}


def loop_legs(path, reps):
    """bench.py's `loop` leg (64 streams, 480x640) with the tracker in `path` and with this tree's, alternated."""
    import bench
    import siammask_b200.tracker as cur
    spec = importlib.util.spec_from_file_location("siammask_b200._tracker_baseline", path)
    base = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = base                               # dataclasses look their module up while it loads
    spec.loader.exec_module(base)
    B = 64
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, search_size=255, max_batch=B, num_slots=2 * B)
    m.load_state_dict(smb.synthetic_state_dict(0)).eval().to("cuda")
    args = argparse.Namespace(search=255)
    mine = cur.BatchTracker
    out = {"baseline": [], "this": []}
    try:
        for _ in range(reps):
            for name, cls in (("baseline", base.BatchTracker), ("this", mine)):
                cur.BatchTracker = cls
                out[name].append(bench.tracker_loop_rate(args, m, B, torch.device("cuda", 0))["value"])
    finally:
        cur.BatchTracker = mine
    out["unit"] = "frames/s"
    out["median_baseline"], out["median_this"] = float(np.median(out["baseline"])), float(np.median(out["this"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--objects", type=int, default=4)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=854)
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    G, K, H, W = args.videos, args.objects, args.height, args.width
    T = args.warmup + args.frames + 1
    torch.cuda.set_device(0)
    res = {"metric": "vos_object_frames_per_s", **gpu_info(), "videos": G, "objects_per_video": K, "frame_hw": [H, W]}
    from oracle.calibrate import calibrated_state_dict
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=G * K, num_slots=G * K)
    net.load_state_dict(calibrated_state_dict(0)).eval().to("cuda")
    p = TrackerParams(instance_size=255, out_size=127)
    frames, anno0 = make_videos(G, K, T, H, W)
    seg = smb.VideoSegmenter(net, p).open([(g, k + 1, 0) for g in range(G) for k in range(K)], num_frames=T)
    seg.frame(frames[0], anno0)
    for f in range(1, 1 + args.warmup):
        seg.frame(frames[f])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(1 + args.warmup, T):
        labels = seg.frame(frames[f])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res["value"] = G * K * args.frames / dt
    res["unit"] = "object-frames/s"
    res["frame_ms"] = 1e3 * dt / args.frames
    res["labelled_fraction"] = float((labels > 0).float().mean())
    res["label_map"] = label_map_legs(seg, G, K, H, W, p.seg_thr)
    res["label_map"]["traffic_bytes_shapes_only"] = {"unfused": 2 * 4 * H * W * G * K,
                                                      "fused": H * W * G + 4 * 127 * 127 * G * K}
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
