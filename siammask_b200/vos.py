"""Multi-object video object segmentation on the device: the `track_vos` loop of tools/test.py:459-542 (also driven by
tools/tune_vos.py) for G videos at once, which may differ in frame size (pass the frames and annotations as lists:
the label maps then come back as a list).  Frames and annotations reach the kernels as `tracker.Packed` buffers with
an sm_image_desc table, so the label map, its scores and the init boxes always run through the *_ragged kernels.

In the reference every object of a video is a separate tracker run with its own lifetime: it is initialised from the
annotation label map at its `start_frame` with `cv2.boundingRect(anno == id)` (:483-498), tracked while
`end_frame >= f > start_frame` (:499-501) and idle otherwise.  Its entry of the float64 `pred_masks` (initialised to -1)
is the GT mask at the start frame and the pasted soft mask (border -1) on tracked frames, and the output of a frame is
one label map, `(argmax_k + 1) * (max_k > seg_thr)` (:480, :504, :521-523).

`VideoSegmenter` restates that over a `BatchTracker`: all objects of all videos that are tracked at a frame advance
as one batch (each stream crops its own video's frame in place), objects join at their start frame (`add`, init boxes
from `sm_label_boxes_ragged`) and leave after their end frame (`remove`), and the label maps of all videos come from one
fused paste-back + argmax kernel (`sm_paste_labels_ragged`): the per-object float frames are never materialised.

With `open(..., score=...)` it also computes the score `track_vos` returns for a video, `MultiBatchIouMeter`
(tools/test.py:421-456): per object and threshold of `VOS_THRESHOLDS`, the mean over the object's scored frames of the IoU
between the fused label `== k+1` and the object's annotation.  Scored frames go through `sm_paste_labels_iou_ragged`,
the same kernel pass with (intersection, union) counts per object and threshold; the counts stay on the device until
`result`.
The reference has two branches, both restated as they are:
  score="whole": no start_frame dict (DAVIS 2016/2017).  The k-th object of a video is scored against annotation id
                 k+1 (by position, whatever id it was tracked with) on frames 1 .. num_frames-2;
  score="spans": start_frame / end_frame dicts.  Each object is scored against its own id on frames
                 start+1 .. end-2 (an empty window gives NaN).
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED
from .tracker import BatchTracker, TrackerParams
from .tune import _check_thresholds

UNBOUNDED = np.iinfo(np.int64).max
VOS_THRESHOLDS = np.arange(0.3, 0.5, 0.05)         # tools/test.py:30 thrs
SCORE_MODES = (None, "whole", "spans")


def schedule(start, end, f: int) -> np.ndarray:
    """What each object does at frame f (tools/test.py:492-501): OBJ_INIT where f == start, OBJ_TRACKED where
    end >= f > start, OBJ_IDLE otherwise.  start, end: per-object frame numbers."""
    start, end = np.asarray(start, dtype=np.int64), np.asarray(end, dtype=np.int64)
    kind = np.full(start.shape, OBJ_IDLE, dtype=np.int32)
    kind[(end >= f) & (f > start)] = OBJ_TRACKED
    kind[f == start] = OBJ_INIT
    return kind


def score_windows(objects, num_frames: int, score: str):
    """MultiBatchIouMeter's scoring plan for objects (video, id, start, end) in open order: target_ids int [n] (the
    annotation value each object is scored against) and its scored frames [lo, hi) as int arrays [n].
    "whole": the k-th object of a video (in this order) against id k+1 on [1, num_frames - 1);
    "spans": each object against its own id on [start + 1, end - 1)."""
    n, T = len(objects), int(num_frames)
    if score == "whole":
        seen = {}
        ids = []
        for o in objects:
            seen[o[0]] = seen.get(o[0], 0) + 1
            ids.append(seen[o[0]])
        return np.array(ids, np.int64), np.full(n, 1, np.int64), np.full(n, T - 1, np.int64)
    if score == "spans":
        return (np.array([o[1] for o in objects], np.int64), np.array([o[2] + 1 for o in objects], np.int64),
                np.array([o[3] - 1 for o in objects], np.int64))
    raise ValueError(f"score must be one of {SCORE_MODES}, got {score!r}")


def score_row(counts, lo: int, hi: int) -> np.ndarray:
    """One object's row of MultiBatchIouMeter from its integer counts int [frames, thrs, 2] (intersection, union):
    per threshold, np.mean of [intxn / union (float64), or 1 where union == 0] over frames lo .. hi-1, as float32; NaN for
    an empty window."""
    c = np.asarray(counts, dtype=np.int64)
    res = np.full(c.shape[1], np.nan, dtype=np.float32)
    if hi <= lo:
        return res
    inter, union = c[lo:hi, :, 0], c[lo:hi, :, 1]
    iou = np.where(union > 0, inter / np.maximum(union, 1), 1.0)
    for t in range(c.shape[1]):
        res[t] = np.mean(np.ascontiguousarray(iou[:, t]))        # the 1-D reduction order of np.mean(list)
    return res


class VideoSegmenter:
    """track_vos for G videos on one engine.  `net` is a `siammask_b200.Custom` whose max_batch / num_slots cover the
    largest number of objects tracked at once; `params` the tracker hyper-parameters (seg_thr included)."""

    def __init__(self, net, params: TrackerParams | None = None):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        self.objects: list[tuple[int, int, int, int]] = []
        self.score = None

    def open(self, objects, num_frames: int | None = None, num_videos: int | None = None, score: str | None = None,
             thrs=VOS_THRESHOLDS):
        """objects: (video, object_id, start_frame[, end_frame]) per object, in the reference's object order;
        end_frame defaults to the last frame (num_frames - 1, or never when num_frames is None).  Within a video the
        k-th object (in this order) gets label k + 1.  num_videos (default: largest video index + 1) is the G of every
        later `frame` call.  score: None, "whole" or "spans" (module docstring) scores every video with the reference's
        MultiBatchIouMeter at the thresholds thrs (1..32 values >= -1); it needs num_frames, and `result()` returns the
        scores.  Resets the frame counter to 0."""
        if score not in SCORE_MODES:
            raise ValueError(f"score must be one of {SCORE_MODES}, got {score!r}")
        if score is not None and num_frames is None:
            raise ValueError("scoring needs num_frames (the scored windows end relative to the last frame)")
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
        self.score = score
        if score is not None:
            if any(o[3] > last for o in objs):
                raise ValueError(f"scoring: every end_frame must be <= num_frames - 1 ({last})")
            self.thrs = _check_thresholds(thrs)
            target, self._lo, self._hi = score_windows(objs, int(num_frames), score)
            for g in range(self.G):
                v = target[[k for k in range(len(objs)) if objs[k][0] == g]]
                if np.unique(v).size != v.size:
                    raise ValueError(f"video {g}: scored object ids must be unique within a video")
            self._target = target
            self._thrs_dev = torch.as_tensor(self.thrs, device=self.dev)
            self._tid_key, self._tid = None, None
            # counts of frame f, entry i (kernel order, self.order[i]) and threshold t: (intersection, union)
            self._counts = torch.zeros(int(num_frames), len(objs), self.thrs.size, 2, dtype=torch.int32, device=self.dev)
        self.tracker._clear()
        self.f = 0
        return self

    def _target_ids(self, scored) -> torch.Tensor:
        key = tuple(int(self._target[k]) if scored[k] else -1 for k in self.order)
        if key != self._tid_key:              # changes only when an object's window opens or closes
            self._tid_key = key
            self._tid = torch.tensor(key, dtype=torch.int32, device=self.dev)
        return self._tid

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
        of this frame, needed when some object starts here or, when scoring, when the frame lies in some object's
        scored window.  Returns labels uint8 [G,H,W] on the device.  frames may instead be a list of G frames
        [H_g,W_g,3] of different sizes, with annos a list of G maps [H_g,W_g]; labels are then a list of G uint8
        [H_g,W_g] views of one packed buffer."""
        f, G = self.f, self.G
        # the schedule and scoring checks need no frames: they fail before any frame reaches the device
        kinds = schedule(self._start, self._end, f)
        starting = [k for k in range(len(self.objects)) if kinds[k] == OBJ_INIT]
        scored = None
        if self.score is not None:
            if f >= self._counts.shape[0]:
                raise ValueError(f"scoring: at most num_frames ({self._counts.shape[0]}) frames")
            scored = (self._lo <= f) & (f < self._hi)
            if scored.any() and annos is None:
                raise ValueError(f"frame {f} is scored: annotation label maps are required")
            if not scored.any():
                scored = None
        listed = isinstance(frames, (list, tuple))
        fr = self.tracker._input(frames)
        if listed and (len(fr.shapes) != G or any(s is None for s in fr.shapes)):
            raise ValueError(f"frames must be a list of {G} frames")
        if not listed and (np.ndim(frames) != 4 or len(fr.shapes) != G):
            raise ValueError(f"frames must be [{G},H,W,3]")
        H, W = max(s[0] for s in fr.shapes), max(s[1] for s in fr.shapes)      # the grid of the label kernels
        if listed and annos is not None:                # host check from shapes alone, before any device work
            if not isinstance(annos, (list, tuple)) or len(annos) != G:
                raise ValueError(f"annos must be a list of {G} label maps, one per frame")
            shp = [None if a is None else tuple(int(v) for v in a.shape) for a in annos]
            if shp != [tuple(s) for s in fr.shapes]:
                raise ValueError(f"each anno must be [H_g, W_g] of its frame: {shp} vs {fr.shapes}")
        anno = None
        if starting or scored is not None:
            if annos is None:
                raise ValueError(f"frame {f}: objects start here, annotation label maps are required")
            if listed:
                pa = self.tracker.packer.pack(annos, 1)
                if pa.shapes != fr.shapes:
                    raise ValueError(f"each anno must match its frame's size: {pa.shapes} vs {fr.shapes}")
            else:
                a = torch.as_tensor(annos)
                if a.dtype != torch.uint8 or tuple(a.shape) != (G, H, W):
                    raise ValueError(f"annos must be uint8 [{G},{H},{W}]")
                pa = self.tracker.packer.wrap(a, 1)
            anno = pa.data
        # sm_image_desc of the G label maps (and annotations)
        desc, ptable = self.tracker.packer.table(fr.shapes, 1)
        plane = (desc, int(ptable["offset"][-1]) + fr.shapes[-1][0] * fr.shapes[-1][1])
        if starting:
            # init boxes (:494-496): one D2H copy, at init frames only
            queries = [(self.objects[k][0], self.objects[k][1]) for k in starting]
            boxes = ops._label_boxes_ragged(anno, desc, G, queries).cpu().numpy()
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
        if scored is None:
            labels = ops._paste_labels(masks, maps, anno, self._offsets, table, (H, W), self.p.seg_thr, ragged=plane)
        else:
            labels, _ = ops._paste_labels_iou(masks, maps, anno, self._offsets, table, self._target_ids(scored), (H, W),
                                              self.p.seg_thr, self._thrs_dev, counts=self._counts[f], ragged=plane)
        self.f += 1
        if listed:
            return [labels[int(o):int(o) + h * w].view(h, w) for o, (h, w) in zip(ptable["offset"], fr.shapes)]
        return labels.view(G, H, W)

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

    def result(self) -> list[np.ndarray]:
        """MultiBatchIouMeter of every video: a list of G float32 arrays [objects of video g, thresholds], the objects in
        `open` order, from the counts of the frames processed so far.  One D2H copy; the IoU and the means are computed
        from the integer counts with the reference's float64 arithmetic (`score_row`); NaN for an empty window."""
        if self.score is None:
            raise ValueError("open(..., score='whole' | 'spans') first")
        counts = self._counts.cpu().numpy()
        entry = {k: i for i, k in enumerate(self.order)}
        rows = [score_row(counts[:, entry[k]], int(self._lo[k]), min(int(self._hi[k]), self.f))
                for k in range(len(self.objects))]
        out = []
        for g in range(self.G):
            r = [rows[k] for k in range(len(self.objects)) if self.objects[k][0] == g]
            out.append(np.stack(r) if r else np.zeros((0, self.thrs.size), np.float32))
        return out
