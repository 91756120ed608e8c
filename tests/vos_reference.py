"""TEST INFRASTRUCTURE ONLY (checker) for the multi-object VOS path (siammask_b200/vos.py).  Nothing under
`siammask_b200/` imports this module.

`track_vos` restates tools/test.py:459-530 statement for statement on top of `oracle.ref_loop.siamese_init` /
`siamese_track`: object-outer / frame-inner loops, one single-stream net, float64 `pred_masks` initialised to -1, and
the fused label map of :521-523.  `make_multi_frames` is a deterministic synthetic multi-object video.
"""
from __future__ import annotations

import cv2
import numpy as np
import torch

from oracle import ref_loop


def schedule_ref(start: int, end: int, f: int) -> str:
    """The reference's per-frame branch for one object (tools/test.py:492-501)."""
    if f == start:
        return "init"
    elif end >= f > start:
        return "track"
    return "idle"


def fuse_labels(pred: np.ndarray, seg_thr: float) -> np.ndarray:
    """tools/test.py:521-523 for one frame: pred float64 [K,H,W] -> uint8 [H,W]."""
    pred = np.asarray(pred, dtype=np.float64)
    if pred.shape[0] == 0:
        return np.zeros(pred.shape[1:], np.uint8)
    return (np.argmax(pred, axis=0).astype("uint8") + 1) * (np.max(pred, axis=0) > seg_thr).astype("uint8")


def label_box(anno: np.ndarray, obj_id: int):
    """The min / max reduction of sm_label_boxes in numpy: x, y, w, h of the pixels equal to obj_id, or 0, 0, 0, 0."""
    ys, xs = np.nonzero(anno == obj_id)
    if xs.size == 0:
        return 0, 0, 0, 0
    return int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1)


def track_vos(model, frames, annos_init, object_ids, starts, ends, hp, seg_thr, device="cuda", device_paste=True):
    """tools/test.py:459-530 for one video with mask_enable = refine_enable = True.  frames: list of frames (numpy HWC or
    uint8 CUDA tensors); annos_init[k]: label map object k is initialised from; starts / ends: per-object frames.
    Returns pred_masks float64 [K,F,H,W], labels uint8 [F,H,W] and target_pos float64 [K,F,2] (NaN where idle)."""
    H, W = annos_init[0].shape
    object_num = len(object_ids)
    pred_masks = np.zeros((object_num, len(frames), H, W)) - 1
    positions = np.full((object_num, len(frames), 2), np.nan)
    for obj_id, o_id in enumerate(object_ids):
        start_frame, end_frame = starts[obj_id], ends[obj_id]
        state = None
        for f, im in enumerate(frames):
            if f == start_frame:  # init
                mask = annos_init[obj_id] == o_id
                x, y, w, h = cv2.boundingRect((mask).astype(np.uint8))
                cx, cy = x + w / 2, y + h / 2
                target_pos = np.array([cx, cy])
                target_sz = np.array([w, h])
                state = ref_loop.siamese_init(im, target_pos, target_sz, model, hp, device=device)
            elif end_frame >= f > start_frame:  # tracking
                state = ref_loop.siamese_track(state, im, True, True, device=device, device_paste=device_paste)
                mask = state["mask"]
                if torch.is_tensor(mask):
                    mask = mask.cpu().numpy()
            if end_frame >= f >= start_frame:
                pred_masks[obj_id, f, :, :] = mask
                positions[obj_id, f] = state["target_pos"]
    labels = np.stack([fuse_labels(pred_masks[:, f], seg_thr) for f in range(len(frames))], 0)
    return pred_masks, labels, positions


def make_multi_frames(n=8, h=240, w=320, seed=0, objects=None):
    """Textured rectangles drifting over a textured background; they overlap at some frame, and each exists only from
    its start to its end frame.  Returns frames (list of uint8 BGR [h,w,3]), annos (list of uint8 label maps [h,w],
    later objects drawn over earlier ones) and the objects as (id, start, end)."""
    rng = np.random.RandomState(seed)
    bg = (rng.rand(h // 8 + 1, w // 8 + 1, 3) * 255).astype(np.uint8)
    bg = np.kron(bg, np.ones((8, 8, 1), np.uint8))[:h, :w]
    if objects is None:
        # id, start, end, (x, y), (vx, vy), (cells w, cells h)
        objects = [(1, 0, n - 1, (60.0, 70.0), (9.0, 2.0), (7, 6)),
                   (2, 1, n - 2, (200.0, 90.0), (-9.0, 1.0), (6, 7)),
                   (3, 2, n - 1, (130.0, 150.0), (2.0, -3.0), (8, 5))]
    tex = [np.kron((rng.rand(ch, cw, 3) * 255).astype(np.uint8), np.ones((8, 8, 1), np.uint8))
           for (_, _, _, _, _, (cw, ch)) in objects]
    frames, annos = [], []
    for f in range(n):
        img, anno = bg.copy(), np.zeros((h, w), np.uint8)
        for (oid, s, e, (x, y), (vx, vy), _), t in zip(objects, tex):
            if not s <= f <= e:
                continue
            xi, yi = int(round(x + vx * f)), int(round(y + vy * f))
            x0, y0, x1, y1 = max(xi, 0), max(yi, 0), min(xi + t.shape[1], w), min(yi + t.shape[0], h)
            if x1 <= x0 or y1 <= y0:
                continue
            img[y0:y1, x0:x1] = t[y0 - yi:y1 - yi, x0 - xi:x1 - xi]
            anno[y0:y1, x0:x1] = oid
        frames.append(img)
        annos.append(anno)
    return frames, annos, [(o[0], o[1], o[2]) for o in objects]
