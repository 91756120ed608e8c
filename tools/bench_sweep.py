"""Throughput of the hyper-parameter sweep (siammask_b200.ParamSweep) on one GPU, the fused IoU counts (`sm_mask_iou`)
against the unfused path (`sm_warp_affine` frames + torch compare / sum per threshold), and the same combinations run
one B=1 tracker stream after another, as tools/tune_vos.py runs them.

    python tools/bench_sweep.py [--videos 2 --frames 12 --warmup 3 --serial-frames 3] [--baseline-tracker FILE]

tune_vos's default 4 x 5 x 5 = 100-combination grid on G synthetic 854x480 videos (DAVIS resolution: one textured
rectangle drifting over a textured background, with its label map).  Prints one JSON line: the card name and power
limit (read-only nvidia-smi query), combination-frames/s through `ParamSweep.frame`, the time of the fused and the
unfused scoring of one frame and whether their counts are identical, and combination-frames/s of the serial B=1 run
(CUDA graphs on).  With --baseline-tracker (a siammask_b200/tracker.py from another revision) it also runs bench.py's
`loop` leg with that tracker and with this one, alternated, --loop-reps times each.

Traffic of the scoring, from shapes only: the unfused path writes a f32 frame per stream and re-reads it once per
threshold (4*H*W*(1+T) bytes, 18 MB per stream at 854x480 with 11 thresholds); the fused path reads the 64 KB mask of
each stream, the pixels of the pasted mask's bounding rectangle of the annotation and each video's annotation once.
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
from siammask_b200.tune import THRESHOLDS, grid                 # noqa: E402
from bench_vos import gpu_info, loop_legs, timed                # noqa: E402


def make_videos(G, T, H, W, seed=0):
    """uint8 frames [T][G,H,W,3] and label maps [T][G,H,W] on the device, plus the frame-0 boxes [G,4] (x, y, w, h)."""
    rng = np.random.RandomState(seed)
    dev = "cuda"
    bg = torch.from_numpy(np.kron((rng.rand(G, H // 8 + 1, W // 8 + 1, 3) * 255).astype(np.uint8),
                                  np.ones((1, 8, 8, 1), np.uint8))[:, :H, :W]).to(dev)
    size = rng.randint(70, 130, (G, 2))
    start = rng.rand(G, 2) * [W - 300, H - 250] + [60, 50]
    vel = rng.randn(G, 2) * 4
    tex = [torch.from_numpy(np.kron((rng.rand(size[g, 1] // 8 + 1, size[g, 0] // 8 + 1, 3) * 255).astype(np.uint8),
                                    np.ones((8, 8, 1), np.uint8))[:size[g, 1], :size[g, 0]]).to(dev) for g in range(G)]
    frames, annos, boxes = [], [], np.zeros((G, 4))
    for t in range(T):
        f, a = bg.clone(), torch.zeros(G, H, W, dtype=torch.uint8, device=dev)
        for g in range(G):
            x, y = np.clip(start[g] + vel[g] * t, 0, [W - size[g, 0], H - size[g, 1]]).astype(int)
            f[g, y:y + size[g, 1], x:x + size[g, 0]] = tex[g]
            a[g, y:y + size[g, 1], x:x + size[g, 0]] = 1
            if t == 0:
                boxes[g] = [x, y, size[g, 0], size[g, 1]]
        frames.append(f)
        annos.append(a)
    return frames, annos, boxes


def scoring_legs(r, anno, video, thrs, W, H, reps=50):
    masks, maps = r.extras["mask_prob"], r.extras["maps"].clone()
    thrs_dev = torch.as_tensor(thrs, device="cuda")
    # float32 v > float64 t  <=>  v > the largest float32 <= t: the unfused path compares in float32 exactly
    lo = [np.float32(t) if np.float32(t) <= t else np.nextafter(np.float32(t), np.float32(-np.inf)) for t in thrs]
    tgt = anno.index_select(0, video.long()) > 0

    def fused():                     # the tables are fixed: no per-call host checks (as ParamSweep)
        return ops._mask_iou(masks, maps, anno, video, thrs_dev)

    def unfused():
        pasted = ops.warp_affine(masks, maps, (W, H), -1.0)
        out = []
        for f in lo:
            pred = pasted > float(f)
            out.append(torch.stack([(pred & tgt).sum((1, 2)), (pred | tgt).sum((1, 2))], -1))
        return torch.stack(out, 1).to(torch.int32)

    same = bool(torch.equal(fused(), unfused()))
    return {"fused_ms": timed(fused, reps), "unfused_ms": timed(unfused, reps), "counts_identical": same}


def serial_leg(sd, combos, frames, boxes, n_frames, base):
    """Each combination as its own B=1 BatchTracker stream on video 0 (CUDA graphs on), one after another."""
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=1, num_slots=1, graphs=True)
    net.load_state_dict(sd).eval().to("cuda")

    def run(cs):
        for pk, wi, lr in cs:
            p = TrackerParams(**{**base, "penalty_k": float(pk), "window_influence": float(wi), "lr": float(lr)})
            bt = BatchTracker(net, p).init(frames[0][0:1], boxes[0:1])
            for f in range(1, 1 + n_frames):
                bt.track(frames[f][0:1], paste=True)
    run(combos[:2])                                              # warm-up: graph capture
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(combos)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"value": len(combos) * n_frames / dt, "unit": "combination-frames/s", "frames_per_combination": n_frames}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=2)
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=854)
    ap.add_argument("--serial-frames", type=int, default=3)
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    G, H, W = args.videos, args.height, args.width
    combos = grid()
    K = combos.shape[0]
    T = 1 + args.warmup + args.frames + 1                       # init frame, warm-up, timed frames, last (unscored)
    torch.cuda.set_device(0)
    res = {"metric": "sweep_combination_frames_per_s", **gpu_info(), "videos": G, "combinations": K,
           "streams": G * K, "frame_hw": [H, W], "thresholds": len(THRESHOLDS)}
    from oracle.calibrate import calibrated_state_dict
    sd = calibrated_state_dict(0)
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=G * K, num_slots=G * K)
    net.load_state_dict(sd).eval().to("cuda")
    base = dict(instance_size=255, out_size=127)
    frames, annos, boxes = make_videos(G, T, H, W)
    sweep = smb.ParamSweep(net, TrackerParams(**base), combos)
    sweep.open(frames[0], boxes, num_frames=T)
    for f in range(1, 1 + args.warmup):
        sweep.frame(frames[f], annos[f])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(1 + args.warmup, T - 1):
        r = sweep.frame(frames[f], annos[f])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res["value"] = G * K * args.frames / dt
    res["unit"] = "combination-frames/s"
    res["frame_ms"] = 1e3 * dt / args.frames
    iou_list, _ = sweep.result()
    res["best_mean_iou"] = float(iou_list.max())
    video = torch.arange(G, dtype=torch.int32, device="cuda").repeat_interleave(K)     # stream g*K + k scores video g
    res["scoring"] = scoring_legs(r, annos[T - 2], video, THRESHOLDS, W, H)
    res["scoring"]["traffic_bytes_shapes_only"] = {"unfused": 4 * H * W * (1 + len(THRESHOLDS)) * G * K}
    res["serial_b1"] = serial_leg(sd, combos, frames, boxes, args.serial_frames, base)
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
