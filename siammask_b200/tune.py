"""Hyper-parameter sweeps on the device: the grid search of tools/tune_vos.py for G videos at once.

The reference re-runs the whole `siamese_init` / `siamese_track` loop on the same frames once per combination of
(penalty_k, window_influence, lr), one stream at a time, and scores frames start < f < end of each run with `IouMeter`
(utils/average_meter_helper.py:71-113): the pasted soft mask thresholded at each of `np.arange(0.3, 0.81, 0.05)`
against `anno > 0`.  Here the K combinations x G videos are one batch of tracker streams: stream (g, k) reads video g's
frames in place and carries combination k in the tracker's per-stream hyper-parameter table (`sm_step_slots_hp`,
`sm_tracker_update_hp`).  Each frame is scored by one fused paste-back + count kernel (`sm_mask_iou`) without
materialising a frame-sized mask per stream, and the IoU rows stay on the device until `ParamSweep.result`.

The rotated box of `siamese_track` (contours / minAreaRect) is not computed: tune_vos never scores it.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .tracker import BatchTracker, TrackerParams

# tools/tune_vos.py's default ranges (--penalty-k 0.0,0.1,0.03 --window-influence 0.3,0.5,0.04 --lr 0.8,1.01,0.05)
# and IouMeter thresholds: a 4 x 5 x 5 grid, 11 thresholds
DEFAULT_PENALTY_K = np.arange(0.0, 0.1, 0.03)
DEFAULT_WINDOW_INFLUENCE = np.arange(0.3, 0.5, 0.04)
DEFAULT_LR = np.arange(0.8, 1.01, 0.05)
THRESHOLDS = np.arange(0.3, 0.81, 0.05)


def grid(penalty_k=DEFAULT_PENALTY_K, window_influence=DEFAULT_WINDOW_INFLUENCE, lr=DEFAULT_LR) -> np.ndarray:
    """float64 [n,3] rows (penalty_k, window_influence, lr) in tune_vos's nested-loop order (penalty_k outermost, lr
    innermost), without the shuffles it applies to each range first."""
    rows = [(pk, wi, r) for pk in np.asarray(penalty_k, np.float64).reshape(-1)
            for wi in np.asarray(window_influence, np.float64).reshape(-1)
            for r in np.asarray(lr, np.float64).reshape(-1)]
    return np.asarray(rows, dtype=np.float64).reshape(-1, 3)


def iou_mean(iou) -> np.ndarray:
    """IouMeter.value('mean') of one run: iou float32 [rows, thresholds], one row per scored frame.  Like the reference it
    averages the first nb = max(number of positive cells of the whole matrix, 1) rows, not the rows that were filled."""
    iou = np.ascontiguousarray(iou, dtype=np.float32)
    nb = max(int(np.sum(iou > 0)), 1)
    return np.mean(iou[:nb], axis=0)


def _check_thresholds(thrs) -> np.ndarray:
    t = np.asarray(thrs, dtype=np.float64).reshape(-1)
    if not 1 <= t.size <= 32:
        raise ValueError("1 to 32 thresholds expected")
    if not (t >= -1.0).all():
        raise ValueError("thresholds must be >= -1")
    return t


def _one_size(frames, fr) -> bool:
    """Whether `frames` (fr: the tracker's `Packed` of them) is a [G,H,W,3] batch or a list of frames of one size:
    `sm_mask_iou` scores same-size videos only."""
    if isinstance(frames, (list, tuple)):
        return None not in fr.shapes and len(set(fr.shapes)) == 1
    return np.ndim(frames) == 4


class ParamSweep:
    """tune_vos's grid search over `combos` (float64 [K,3] = penalty_k, window_influence, lr; default `grid()`) for G
    videos on one engine.  `net` is a `siammask_b200.Custom` whose max_batch and num_slots cover G*K streams; `params`
    holds the settings the combinations do not (context_amount, out_size, ...).  Masks come from the refine module when
    params.out_size is 127 and from the mask head when it is 63."""

    def __init__(self, net, params: TrackerParams | None = None, combos=None, thrs=THRESHOLDS):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        c = grid() if combos is None else np.asarray(combos, dtype=np.float64)
        if c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0:
            raise ValueError(f"combos must be [K, 3] (penalty_k, window_influence, lr), got {c.shape}")
        if not np.isfinite(c).all():
            raise ValueError("combos must be finite")
        self.combos = c
        self.thrs = _check_thresholds(thrs)
        self._thrs_dev = torch.as_tensor(self.thrs, device=self.dev)
        self.G = 0
        self.f = self.T = 0

    @property
    def K(self) -> int:
        return int(self.combos.shape[0])

    @torch.no_grad()
    def open(self, frames0, boxes_xywh, num_frames: int):
        """siamese_init of every (video, combination) stream on frame 0.  frames0: uint8 [G,H,W,3] (BGR); boxes_xywh:
        [G,4] top-left x, y, w, h of each video's target; num_frames: T, the videos' length.  Frames 1 .. T-2 are scored
        (tune_vos's start_frame < f < end_frame).  Stream (g, k) is row g*K + k of every per-frame output."""
        fr = self.tracker._input(frames0)
        if not _one_size(frames0, fr):
            raise ValueError("frames0 must be [G,H,W,3]")
        G, K, T = len(fr.shapes), self.K, int(num_frames)
        boxes = np.asarray(boxes_xywh, dtype=np.float64)
        if boxes.shape != (G, 4):
            raise ValueError(f"boxes_xywh must be [{G}, 4]")
        if T < 3:
            raise ValueError("num_frames must be >= 3 (the first and the last frame are not scored)")
        net = self.tracker.net
        if G * K > net.max_batch or G * K > net.num_slots - self.tracker.slot0:
            raise ValueError(f"{G} videos x {K} combinations = {G * K} streams exceed the engine's max_batch "
                             f"({net.max_batch}) or free slots ({net.num_slots - self.tracker.slot0}); split the grid")
        video = np.repeat(np.arange(G), K)
        self.tracker._clear()
        self.tracker.add(fr, np.repeat(boxes, K, axis=0), frame_index=video, hp=np.tile(self.combos, (G, 1)))
        self._video = torch.as_tensor(video.astype(np.int32), device=self.dev)
        self._iou = torch.zeros(T - 2, G * K, self.thrs.size, dtype=torch.float32, device=self.dev)
        self.G, self.T, self.f = G, T, 1
        return self

    @torch.no_grad()
    def frame(self, frames, annos=None):
        """Track frame f (the next one) of every video: frames uint8 [G,H,W,3]; annos uint8 [G,H,W] annotation label maps
        of this frame, required when it is scored (0 < f < T-1).  The frame's IoU rows (float32(intersection / union),
        1 where the union is empty) are written into a device buffer.  Returns the tracker's `TrackResult`."""
        f = self.f
        if not 1 <= f < self.T:
            raise ValueError("call open() first; at most num_frames - 1 frames follow it")
        fr = self.tracker._input(frames)
        if not _one_size(frames, fr) or len(fr.shapes) != self.G:
            raise ValueError(f"frames must be [{self.G},H,W,3]")
        H, W = fr.shapes[0]
        scored = f < self.T - 1
        anno = None
        if scored:
            if annos is None:
                raise ValueError(f"frame {f} is scored: annotations are required")
            anno = torch.as_tensor(annos).to(self.dev).contiguous()
            if anno.dtype != torch.uint8 or tuple(anno.shape) != (self.G, H, W):
                raise ValueError(f"annos must be uint8 [{self.G},{H},{W}]")
        r = self.tracker.track(fr, mask=True, refine=self.p.out_size == 127, paste=False)
        if scored:
            cnt = ops._mask_iou(r.extras["mask_prob"], r.extras["maps"], anno, self._video, self._thrs_dev)
            inter, union = cnt[..., 0].double(), cnt[..., 1].double()
            # IouMeter.add: intxn / union in float64, stored into a float32 matrix; 1 when the union is empty
            self._iou[f - 1] = torch.where(union > 0, (inter / union).float(), torch.ones_like(union, dtype=torch.float32))
        self.f += 1
        return r

    def result(self):
        """One D2H copy.  Returns (iou_list float32 [G,K,T] = IouMeter.value('mean') of every stream, per-frame IoU
        float32 [num_frames-2, G, K, T]); rows of frames not tracked yet are 0, as in a partly filled IouMeter."""
        per_frame = self._iou.cpu().numpy()
        G, K, n = self.G, self.K, self.thrs.size
        means = np.stack([iou_mean(per_frame[:, s]) for s in range(G * K)]).reshape(G, K, n)
        return means, per_frame.reshape(-1, G, K, n)
