"""Multi-object video object segmentation on the device: the `track_vos` loop of tools/test.py:459-542 (also driven by
tools/tune_vos.py) for G videos of one frame size at once.

In the reference every object of a video is a separate tracker run with its own lifetime: it is initialised from the
annotation label map at its `start_frame` with `cv2.boundingRect(anno == id)` (:483-498), tracked while
`end_frame >= f > start_frame` (:499-501) and idle otherwise.  Its entry of the float64 `pred_masks` (initialised to -1)
is the GT mask at the start frame and the pasted soft mask (border -1) on tracked frames, and the output of a frame is
one label map, `(argmax_k + 1) * (max_k > seg_thr)` (:480, :504, :521-523).

`VideoSegmenter` restates that over a `BatchTracker`: all objects of all videos that are tracked at a frame advance
as one batch (each stream crops its own video's frame in place), objects join at their start frame (`add`, init boxes
from `sm_label_boxes`) and leave after their end frame (`remove`), and the label maps of all videos come from one fused
paste-back + argmax kernel (`sm_paste_labels`): the per-object float frames are never materialised.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED
from .tracker import BatchTracker, TrackerParams

UNBOUNDED = np.iinfo(np.int64).max


def schedule(start, end, f: int) -> np.ndarray:
    """What each object does at frame f (tools/test.py:492-501): OBJ_INIT where f == start, OBJ_TRACKED where
    end >= f > start, OBJ_IDLE otherwise.  start, end: per-object frame numbers."""
    start, end = np.asarray(start, dtype=np.int64), np.asarray(end, dtype=np.int64)
    kind = np.full(start.shape, OBJ_IDLE, dtype=np.int32)
    kind[(end >= f) & (f > start)] = OBJ_TRACKED
    kind[f == start] = OBJ_INIT
    return kind


class VideoSegmenter:
    """track_vos for G videos on one engine.  `net` is a `siammask_b200.Custom` whose max_batch / num_slots cover the
    largest number of objects tracked at once; `params` the tracker hyper-parameters (seg_thr included)."""

    def __init__(self, net, params: TrackerParams | None = None):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        self.objects: list[tuple[int, int, int, int]] = []

    def open(self, objects, num_frames: int | None = None, num_videos: int | None = None):
        """objects: (video, object_id, start_frame[, end_frame]) per object, in the reference's object order;
        end_frame defaults to the last frame (num_frames - 1, or never when num_frames is None).  Within a video the
        k-th object (in this order) gets label k + 1.  num_videos (default: largest video index + 1) is the G of every
        later `frame` call.  Resets the frame counter to 0."""
        last = UNBOUNDED if num_frames is None else int(num_frames) - 1
        objs = []
        for o in objects:
            o = tuple(int(v) for v in o)
            if len(o) == 3:
                o = o + (last,)
            if len(o) != 4 or o[0] < 0 or not 0 <= o[1] <= 255:
                raise ValueError(f"bad object entry {o}: (video >= 0, id in 0..255, start[, end])")
            if o[3] < o[2]:
                # the reference would initialise such an object and then never write its pred_masks entry
                # (tools/test.py:502-503), so it could never appear in a label map
                raise ValueError(f"object {o}: end_frame {o[3]} is before start_frame {o[2]}")
            objs.append(o)
        self.G = max((o[0] for o in objs), default=-1) + 1 if num_videos is None else int(num_videos)
        if self.G < 1 or any(o[0] >= self.G for o in objs):
            raise ValueError("every object's video index must be < num_videos")
        counts = np.bincount([o[0] for o in objs], minlength=self.G)
        if (counts > 255).any():
            raise ValueError("at most 255 objects per video (labels are uint8)")
        # objects grouped by video (stable): entry i of the kernel's table is object order[i]
        self.order = sorted(range(len(objs)), key=lambda k: objs[k][0])
        self.objects = objs
        self._start = np.array([o[2] for o in objs], dtype=np.int64)
        self._end = np.array([o[3] for o in objs], dtype=np.int64)
        self._sid: list[int | None] = [None] * len(objs)     # tracker stream of each object (None: not tracked)
        self._offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int32, device=self.dev)
        self._table_key, self._table = None, None
        self.tracker._clear()
        self.f = 0
        return self

    def _entries(self, kinds, rows) -> torch.Tensor:
        ent = []
        for k in self.order:
            if kinds[k] == OBJ_TRACKED:
                ent.append((OBJ_TRACKED, rows[self._sid[k]]))
            elif kinds[k] == OBJ_INIT:
                ent.append((OBJ_INIT, self.objects[k][1]))
            else:
                ent.append((OBJ_IDLE, 0))
        key = tuple(ent)
        if key != self._table_key:            # the table changes only when an object starts, stops or a row moves
            self._table_key = key
            self._table = torch.tensor(ent if ent else [(OBJ_IDLE, 0)], dtype=torch.int32, device=self.dev).reshape(-1, 2)
        return self._table

    @torch.no_grad()
    def frame(self, frames, annos=None) -> torch.Tensor:
        """Advance every video by one frame.  frames: uint8 [G,H,W,3] (BGR); annos: uint8 [G,H,W] annotation label maps
        of this frame, needed only when some object starts here.  Returns labels uint8 [G,H,W] on the device."""
        f = self.f
        fr = self.tracker._frames(frames)
        if fr.dim() != 4 or fr.shape[0] != self.G:
            raise ValueError(f"frames must be [{self.G},H,W,3]")
        G, H, W = int(fr.shape[0]), int(fr.shape[1]), int(fr.shape[2])
        kinds = schedule(self._start, self._end, f)
        starting = [k for k in range(len(self.objects)) if kinds[k] == OBJ_INIT]
        anno = None
        if starting:
            if annos is None:
                raise ValueError(f"frame {f}: objects start here, annotation label maps are required")
            anno = torch.as_tensor(annos).to(self.dev).contiguous()
            if anno.dtype != torch.uint8 or tuple(anno.shape) != (G, H, W):
                raise ValueError(f"annos must be uint8 [{G},{H},{W}]")
            # init boxes (:494-496): one D2H copy, at init frames only
            boxes = ops.label_boxes(anno, [(self.objects[k][0], self.objects[k][1]) for k in starting]).cpu().numpy()
            missing = [self.objects[k][:2] for k, b in zip(starting, boxes) if b[2] == 0]
            if missing:
                raise ValueError(f"frame {f}: (video, id) {missing} not in the annotation")
        bt = self.tracker
        leaving = [k for k, s in enumerate(self._sid) if s is not None and kinds[k] != OBJ_TRACKED]
        if leaving:
            bt.remove([self._sid[k] for k in leaving])
            for k in leaving:
                self._sid[k] = None
        masks = maps = None
        rows = {}
        if bt.N:
            r = bt.track(fr, mask=True, refine=self.p.out_size == 127, paste=False)
            masks, maps = r.extras["mask_prob"], r.extras["maps"]
            rows = {sid: i for i, sid in enumerate(r.extras["ids"])}
            self.last = r
        table = self._entries(kinds, rows)
        if starting:
            xywh = boxes.astype(np.float64)
            ids = bt.add(fr, xywh, frame_index=[self.objects[k][0] for k in starting])
            for k, sid in zip(starting, ids):
                self._sid[k] = sid
        labels = ops._paste_labels(masks, maps, anno, self._offsets, table, (H, W), self.p.seg_thr)
        self.f += 1
        return labels

    def state(self):
        """Per-object tracker state after the last frame: target_pos f64 [n,2], target_sz f64 [n,2] (NaN for objects
        that are not active), in the order of `open`.  One D2H copy."""
        n = len(self.objects)
        pos, sz = np.full((n, 2), np.nan), np.full((n, 2), np.nan)
        s = self.tracker.state.cpu().numpy()
        rows = {sid: i for i, sid in enumerate(self.tracker.ids)}
        for k, sid in enumerate(self._sid):
            if sid is not None:
                pos[k], sz[k] = s[rows[sid], 0:2], s[rows[sid], 2:4]
        return {"target_pos": pos, "target_sz": sz}
