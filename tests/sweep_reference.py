"""TEST INFRASTRUCTURE ONLY (checker) for the hyper-parameter sweep (siammask_b200/tune.py).  Nothing under
`siammask_b200/` imports this module.

`tune_run` restates `tune()` of tools/tune_vos.py for one video and one (penalty_k, window_influence, lr) combination
statement for statement on top of `oracle.ref_loop.siamese_init` / `siamese_track` (mask and refine on, one
single-stream net), and `IouMeter` restates utils/average_meter_helper.py:71-113 as that loop uses it.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ref_loop


class IouMeter:
    """utils/average_meter_helper.py:71-113 (add and value('mean'))."""

    def __init__(self, thrs, sz):
        self.sz = sz
        self.iou = np.zeros((sz, len(thrs)), dtype=np.float32)
        self.thrs = thrs
        self.n = 0

    def add(self, output, target):
        if self.n >= len(self.iou):
            return
        target, output = target.squeeze(), output.squeeze()
        for i, thr in enumerate(self.thrs):
            pred = output > thr
            mask_sum = (pred == 1).astype(np.uint8) + (target > 0).astype(np.uint8)
            intxn = np.sum(mask_sum == 2)
            union = np.sum(mask_sum > 0)
            if union > 0:
                self.iou[self.n, i] = intxn / union
            elif union == 0 and intxn == 0:
                self.iou[self.n, i] = 1
        self.n += 1

    def value_mean(self):
        nb = max(int(np.sum(self.iou > 0)), 1)
        return np.mean(self.iou[:nb], axis=0)


def tune_run(model, frames, annos, box_xywh, hp, thrs, device="cuda"):
    """tools/tune_vos.py tune() with --mask --refine for one video: frames (numpy HWC or uint8 CUDA tensors), annos
    (uint8 label maps), the frame-0 box x, y, w, h and the hp dict of one combination.  Returns the IouMeter matrix
    float32 [T-2, len(thrs)], its value('mean') and target_pos float64 [T, 2]."""
    iou = IouMeter(thrs, len(frames) - 2)
    start_frame, end_frame = 0, len(frames) - 1
    positions = np.zeros((len(frames), 2))
    x, y, w, h = box_xywh
    for f, (im, anno) in enumerate(zip(frames, annos)):
        if f == start_frame:  # init
            target_pos = np.array([x + w / 2, y + h / 2])
            target_sz = np.array([w, h])
            state = ref_loop.siamese_init(im, target_pos, target_sz, model, hp, device=device)
        elif f > start_frame:  # tracking
            state = ref_loop.siamese_track(state, im, True, True, device=device, device_paste=True)
            mask = state["mask"]
            if torch.is_tensor(mask):
                mask = mask.cpu().numpy()
        positions[f] = state["target_pos"]
        if start_frame < f < end_frame:
            iou.add(mask, anno)
    return iou.iou, iou.value_mean(), positions
