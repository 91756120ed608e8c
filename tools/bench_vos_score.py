"""Cost of scoring multi-object video segmentation on the device: the fused label map + per-object IoU counts
(`sm_paste_labels_iou`) against the label map alone (`sm_paste_labels`) and against an unfused scorer, and
`VideoSegmenter.frame` with score=None against score="whole".

    python tools/bench_vos_score.py [--videos 16 --objects 4 --frames 20 --warmup 3 --reps 3]

G videos x K objects at 854x480 (DAVIS resolution) with tools/test.py's 4 thresholds, the synthetic videos of
tools/bench_vos.py, scored against their frame-0 label maps.  Prints one JSON line: the card name and power limit
(read-only nvidia-smi query); the kernel times (CUDA events, averaged over --kernel-reps calls on the last frame's
masks) of the fused labels + counts, of the label map alone, and of the unfused path (`sm_paste_labels` once per
threshold, then per-object intersection / union in torch) with whether its counts equal the fused ones; and the
object-frames/s of `VideoSegmenter.frame` without and with scoring, alternated --reps times each (medians).
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

import siammask_b200 as smb                                     # noqa: E402
from siammask_b200 import ops                                   # noqa: E402
from siammask_b200.ops import OBJ_TRACKED                       # noqa: E402
from siammask_b200.tracker import TrackerParams                 # noqa: E402
from siammask_b200.vos import VOS_THRESHOLDS                    # noqa: E402
from bench_vos import gpu_info, make_videos, timed              # noqa: E402


def kernel_legs(seg, anno, G, K, H, W, thr, reps):
    r = seg.last
    masks, maps = r.extras["mask_prob"], r.extras["maps"].clone()
    rows = {sid: i for i, sid in enumerate(r.extras["ids"])}
    order = [rows[seg._sid[k]] for k in seg.order]              # row of each (video, object) in video-major order
    table = torch.tensor([(OBJ_TRACKED, i) for i in order], dtype=torch.int32, device="cuda")
    off = torch.arange(0, G * K + 1, K, dtype=torch.int32, device="cuda")
    ids = torch.arange(1, K + 1, dtype=torch.int32, device="cuda").repeat(G)           # "whole": k-th object -> k+1
    thrs = torch.as_tensor(VOS_THRESHOLDS, device="cuda")
    T = thrs.numel()
    counts = torch.empty(G * K, T, 2, dtype=torch.int32, device="cuda")

    def fused():
        return ops._paste_labels_iou(masks, maps, anno, off, table, ids, (H, W), thr, thrs, counts=counts)

    def labels_only():
        return ops._paste_labels(masks, maps, None, off, table, (H, W), thr)

    kk = torch.arange(1, K + 1, device="cuda", dtype=torch.uint8).view(1, K, 1, 1)
    tgt = anno.unsqueeze(1) == ids.view(G, K, 1, 1).to(torch.uint8)                    # [G,K,H,W]

    def unfused():
        out = []
        for t in VOS_THRESHOLDS:
            pred = ops._paste_labels(masks, maps, None, off, table, (H, W), float(t)).unsqueeze(1) == kk
            out.append(torch.stack([(pred & tgt).sum((2, 3)), (pred | tgt).sum((2, 3))], -1).view(G * K, 2))
        return torch.stack(out, 1).to(torch.int32)

    _, c = fused()
    same = bool(torch.equal(c, unfused())) and bool(torch.equal(fused()[0], labels_only()))
    return {"fused_labels_counts_ms": timed(fused, reps), "labels_only_ms": timed(labels_only, reps),
            "unfused_ms": timed(unfused, reps), "counts_and_labels_identical": same, "thresholds": T}


def frame_rate(net, p, frames, anno0, G, K, warmup, n, score):
    T = warmup + n + 1
    seg = smb.VideoSegmenter(net, p).open([(g, k + 1, 0) for g in range(G) for k in range(K)], num_frames=T,
                                          score=score)
    seg.frame(frames[0], anno0)
    for f in range(1, 1 + warmup):
        seg.frame(frames[f], anno0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(1 + warmup, T):
        seg.frame(frames[f], anno0)
    torch.cuda.synchronize()
    return G * K * n / (time.perf_counter() - t0), seg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--objects", type=int, default=4)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=854)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=100)
    args = ap.parse_args()
    G, K, H, W = args.videos, args.objects, args.height, args.width
    torch.cuda.set_device(0)
    res = {"metric": "vos_score_object_frames_per_s", **gpu_info(), "videos": G, "objects_per_video": K,
           "frame_hw": [H, W], "thresholds": [float(t) for t in VOS_THRESHOLDS]}
    from oracle.calibrate import calibrated_state_dict
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=G * K, num_slots=G * K)
    net.load_state_dict(calibrated_state_dict(0)).eval().to("cuda")
    p = TrackerParams(instance_size=255, out_size=127)
    frames, anno0 = make_videos(G, K, args.warmup + args.frames + 1, H, W)
    rates = {"none": [], "whole": []}
    for _ in range(args.reps):
        for name, score in (("none", None), ("whole", "whole")):
            rate, seg = frame_rate(net, p, frames, anno0, G, K, args.warmup, args.frames, score)
            rates[name].append(rate)
    res["frame"] = {"unit": "object-frames/s", "score_none": rates["none"], "score_whole": rates["whole"],
                    "median_score_none": float(np.median(rates["none"])),
                    "median_score_whole": float(np.median(rates["whole"]))}
    res["value"] = res["frame"]["median_score_whole"]
    res["unit"] = "object-frames/s"
    res["kernels"] = kernel_legs(seg, anno0, G, K, H, W, p.seg_thr, args.kernel_reps)
    res["score_whole_mean_iou"] = [float(v) for v in np.mean(np.concatenate(seg.result()), axis=0)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
