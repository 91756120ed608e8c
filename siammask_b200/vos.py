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

A whole dataset (videos of any length, frame size and object count) goes through `open_queue` / `needed` / `step`: the
videos are queued by `schedule.Scheduler`, each holding as many slots as it has objects active at once (`peak_width`)
from its admission until its last frame, and each admitted video advances one frame of its own per step.  `frame` is a
step of the same kind in which every video reads frame f, so one code path runs the loop in both.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED
from .schedule import QueueRun
from .tracker import BatchTracker, TrackerParams, upload
from .tune import _check_thresholds

UNBOUNDED = np.iinfo(np.int64).max
VOS_THRESHOLDS = np.arange(0.3, 0.5, 0.05)         # tools/test.py:30 thrs
SCORE_MODES = (None, "whole", "spans")


def schedule(start, end, f) -> np.ndarray:
    """What each object does at frame f (tools/test.py:492-501): OBJ_INIT where f == start, OBJ_TRACKED where
    end >= f > start, OBJ_IDLE otherwise.  start, end: per-object frame numbers; f: one frame, or one per object."""
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


def peak_width(start, end) -> int:
    """The most objects active at one frame: object k is active at frame f when start[k] <= f <= end[k] (it joins at
    its start frame after the objects that stopped the frame before have left).  The slots a video holds in a queue."""
    s, e = np.asarray(start, np.int64).reshape(-1), np.asarray(end, np.int64).reshape(-1)
    return max((int(((s <= f) & (f <= e)).sum()) for f in s), default=0)


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


class VideoSegmenter(QueueRun):
    """track_vos for G videos on one engine.  `net` is a `siammask_b200.Custom` whose max_batch / num_slots cover the
    largest number of objects tracked at once; `params` the tracker hyper-parameters (seg_thr included)."""

    def __init__(self, net, params: TrackerParams | None = None):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        self.objects: list[tuple[int, int, int, int]] = []
        self.score = None

    def _reset(self, objs, G: int, lengths, score, thrs):
        """The state of a run over objs (checked (video, id, start, end) tuples) in G videos of lengths[g] frames (None:
        unbounded, without scoring): every object idle, no frame processed.  Checks the per-video object count and the
        scored ids."""
        members = [[k for k, o in enumerate(objs) if o[0] == g] for g in range(G)]
        for g, ks in enumerate(members):
            if len(ks) > 255:
                raise ValueError(f"video {g}: at most 255 objects per video (labels are uint8)")
        if score is not None:
            self.thrs = _check_thresholds(thrs)
            target, lo, hi = (np.zeros(len(objs), np.int64) for _ in range(3))
            for g, ks in enumerate(members):
                target[ks], lo[ks], hi[ks] = score_windows([objs[k] for k in ks], int(lengths[g]), score)
                if np.unique(target[ks]).size != len(ks):
                    raise ValueError(f"video {g}: scored object ids must be unique within a video")
            self._target, self._lo, self._hi = target, lo, hi
            n_rows = np.maximum(hi - lo, 0)
            self._row0 = np.concatenate([[0], np.cumsum(n_rows)[:-1]]).astype(np.int64)
            self._thrs_dev = torch.as_tensor(self.thrs, device=self.dev)
            # (intersection, union) of object k at frame lo[k] + j, threshold t: row _row0[k] + j
            self._rows = torch.zeros(int(n_rows.sum()), self.thrs.size, 2, dtype=torch.int32, device=self.dev)
        self.objects, self.score, self.G, self._T = objs, score, G, lengths
        self.order = [k for ks in members for k in ks]          # the objects grouped by video, each video's in order
        self._members = members
        self._video = np.array([o[0] for o in objs], np.int64)
        self._start = np.array([o[2] for o in objs], np.int64)
        self._end = np.array([o[3] for o in objs], np.int64)
        self._sid: list[int | None] = [None] * len(objs)     # tracker stream of each object (None: not tracked)
        self._hw: list = [None] * G                  # frame size of each video, from its frame 0
        self._admitted = np.full(G, -1, np.int64)   # the step that read each video's frame 0
        self._done = np.zeros(G, np.int64)          # frames of each video processed
        self._table_key = self._tid_key = self._off_key = self._copy_key = None
        self._sched = self._plan = None
        self.tracker._clear()
        self.f = 0

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
        G = max((o[0] for o in objs), default=-1) + 1 if num_videos is None else int(num_videos)
        if G < 1 or any(o[0] >= G for o in objs):
            raise ValueError("every object's video index must be < num_videos")
        if score is not None and any(o[3] > last for o in objs):
            raise ValueError(f"scoring: every end_frame must be <= num_frames - 1 ({last})")
        self._reset(objs, G, None if num_frames is None else [int(num_frames)] * G, score, thrs)
        return self

    def _target_ids(self, scored, order) -> torch.Tensor:
        key = tuple(int(self._target[k]) if scored[k] else -1 for k in order)
        if key != self._tid_key:              # changes only when an object's window opens or closes
            self._tid_key = key
            self._tid = upload(np.asarray(key, np.int64), torch.int32, self.dev)
        return self._tid

    def _entries(self, kinds, rows, order) -> torch.Tensor:
        """The kernel's object table: one (kind, arg) entry per object of `order`."""
        ent = []
        for k in order:
            if kinds[k] == OBJ_TRACKED:
                ent.append((OBJ_TRACKED, rows[self._sid[k]]))
            elif kinds[k] == OBJ_INIT:
                ent.append((OBJ_INIT, self.objects[k][1]))
            else:
                ent.append((OBJ_IDLE, 0))
        key = tuple(ent)
        if key != self._table_key:            # the table changes only when an object starts, stops or a row moves
            self._table_key = key
            self._table = upload(np.asarray(ent if ent else [(OBJ_IDLE, 0)], np.int64).reshape(-1, 2), torch.int32,
                                 self.dev)
        return self._table

    @torch.no_grad()
    def frame(self, frames, annos=None) -> torch.Tensor:
        """Advance every video by one frame.  frames: uint8 [G,H,W,3] (BGR); annos: uint8 [G,H,W] annotation label maps
        of this frame, needed when some object starts here or, when scoring, when the frame lies in some object's
        scored window.  Returns labels uint8 [G,H,W] on the device.  frames may instead be a list of G frames
        [H_g,W_g,3] of different sizes, with annos a list of G maps [H_g,W_g]; labels are then a list of G uint8
        [H_g,W_g] views of one packed buffer."""
        if self._sched is not None:
            raise ValueError("a queue run advances with step(); frame() belongs to open()")
        f, G = self.f, self.G
        # the scoring checks need no frames: they fail before any frame reaches the device
        scored = False
        if self.score is not None:
            if f >= self._T[0]:
                raise ValueError(f"scoring: at most num_frames ({self._T[0]}) frames")
            scored = bool(((self._lo <= f) & (f < self._hi)).any())
            if scored and annos is None:
                raise ValueError(f"frame {f} is scored: annotation label maps are required")
        listed = isinstance(frames, (list, tuple))
        fr = self.tracker._input(frames)
        if listed and (len(fr.shapes) != G or any(s is None for s in fr.shapes)):
            raise ValueError(f"frames must be a list of {G} frames")
        if not listed and (np.ndim(frames) != 4 or len(fr.shapes) != G):
            raise ValueError(f"frames must be [{G},H,W,3]")
        H, W = max(s[0] for s in fr.shapes), max(s[1] for s in fr.shapes)
        if listed and annos is not None:                # host check from shapes alone, before any device work
            if not isinstance(annos, (list, tuple)) or len(annos) != G:
                raise ValueError(f"annos must be a list of {G} label maps, one per frame")
            shp = [None if a is None else tuple(int(v) for v in a.shape) for a in annos]
            if shp != [tuple(s) for s in fr.shapes]:
                raise ValueError(f"each anno must be [H_g, W_g] of its frame: {shp} vs {fr.shapes}")
        anno = None
        if scored or (self._start == f).any():
            if annos is None:
                raise ValueError(f"frame {f}: objects start here, annotation label maps are required")
            if listed:                                  # their shapes were checked above
                pa = self.tracker.packer.pack(annos, 1)
            else:
                a = torch.as_tensor(annos)
                if a.dtype != torch.uint8 or tuple(a.shape) != (G, H, W):
                    raise ValueError(f"annos must be uint8 [{G},{H},{W}]")
                pa = self.tracker.packer.wrap(a, 1)
            anno = pa.data
        labels, offsets = self._run(fr, anno, [(g, f) for g in range(G)])
        if listed:
            return [labels[int(o):int(o) + h * w].view(h, w) for o, (h, w) in zip(offsets, fr.shapes)]
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
            raise ValueError("open(..., score='whole' | 'spans') or open_queue(..., score=...) first")
        counts = self._rows.cpu().numpy()
        out = []
        for g, ks in enumerate(self._members):
            # frames lo .. min(hi, frames processed) - 1 of each object
            out.append(np.stack([score_row(counts[self._row0[k]:self._row0[k] + max(self._hi[k] - self._lo[k], 0)], 0,
                                           min(int(self._hi[k]), int(self._done[g])) - int(self._lo[k]))
                                 for k in ks]) if ks else np.zeros((0, self.thrs.size), np.float32))
        return out

    # ------------------------------------------------------------------ queue mode
    def open_queue(self, objects, num_frames, score: str | None = None, thrs=VOS_THRESHOLDS):
        """Queues G videos of any length, frame size and object count through the engine (`schedule.Scheduler`, K = 1):
        video g holds `peak_width` of its objects' (start, end) slots from its admission until its last frame, and a
        video waits until that many of min(max_batch, free slots) are free.  num_frames: [G] the videos' lengths;
        objects: (video, object_id, start_frame[, end_frame]) as in `open`, end_frame defaulting to T_g - 1, with
        0 <= start <= end <= T_g - 1; every video needs one object.  score: as in `open`, each video scored on its own
        length ("whole": frames 1 .. T_g - 2).  Drive it with

            while seg.pending:
                need = seg.needed()
                want = seg.needs_anno()
                labels = seg.step([frames[g][t] for g, t in need],
                                  [annos[g][t] if w else None for (g, t), w in zip(need, want)])

        and read `result()` (G float32 arrays [objects of g, thresholds], objects in open order)."""
        T = np.asarray(num_frames).reshape(-1)
        if T.size == 0 or not np.issubdtype(T.dtype, np.integer) or (T < 1).any():
            raise ValueError("num_frames must be one integer >= 1 per video")
        G = int(T.size)
        objs = []
        for o in objects:
            o = tuple(int(v) for v in o)
            if len(o) not in (3, 4) or not 0 <= o[0] < G or not 0 <= o[1] <= 255:
                raise ValueError(f"bad object entry {o}: (video in 0..{G - 1}, id in 0..255, start[, end])")
            if len(o) == 3:
                o = o + (int(T[o[0]]) - 1,)
            if not 0 <= o[2] <= o[3] <= T[o[0]] - 1:
                raise ValueError(f"object {o}: needs 0 <= start_frame <= end_frame <= {int(T[o[0]]) - 1} "
                                 f"(video {o[0]}'s last frame)")
            objs.append(o)
        self._reset(objs, G, T.astype(np.int64), score, thrs)
        if [] in self._members:
            raise ValueError(f"video {self._members.index([])} has no object")
        width = [peak_width(self._start[ks], self._end[ks]) for ks in self._members]
        self._queue(T, 1, width)                     # ValueError for a video wider than the engine
        return self

    def _wants_anno(self, g: int, t: int) -> bool:
        ks = self._members[g]
        if (self._start[ks] == t).any():
            return True
        return self.score is not None and bool(((self._lo[ks] <= t) & (t < self._hi[ks])).any())

    def needs_anno(self) -> list:
        """Per `needed()` entry (g, t): whether `step` needs frame t's annotation of video g (an object of g starts at
        t, or t lies in some object's scored window)."""
        return [self._wants_anno(g, t) for g, t in self.needed()]

    @staticmethod
    def _size_of(im, what: str):
        shape = tuple(int(v) for v in im.shape)
        if len(shape) != (3 if what == "frame" else 2) or (what == "frame" and shape[2] != 3):
            raise ValueError(f"each {what} must be {'[H,W,3]' if what == 'frame' else '[H,W]'}, got {shape}")
        return shape[:2]

    @torch.no_grad()
    def step(self, frames, annos):
        """One step of a queue run: frames[i] is frame t of video g for (g, t) = needed()[i] (uint8 [H_g,W_g,3], BGR),
        annos[i] its uint8 [H_g,W_g] annotation label map where needs_anno()[i] (ignored elsewhere; None will do).  Does
        for every admitted video what `frame` does at its frame t: objects start, are tracked and leave, and the fused
        label map (with the scored objects' counts) comes from one ragged kernel pass over the step's videos.  Returns
        the label maps, a list of uint8 [H_g,W_g] device views in needed() order."""
        st = self._pending_step(frames=frames, annos=annos)
        # every check reads shapes on the host, before any device work
        want = [self._wants_anno(g, t) for g, t in st.need]
        for i, (g, t) in enumerate(st.need):
            if frames[i] is None:
                raise ValueError(f"frame {t} of video {g} is missing")
            hw = self._size_of(frames[i], "frame")
            if t > 0 and hw != self._hw[g]:
                raise ValueError(f"frame {t} of video {g} is {hw[0]}x{hw[1]}, its frame 0 "
                                 f"{self._hw[g][0]}x{self._hw[g][1]}")
            if want[i]:
                a = annos[i]
                if a is None:
                    raise ValueError(f"frame {t} of video {g}: an object starts or is scored, its annotation is "
                                     "required")
                if a.dtype not in (np.uint8, torch.uint8) or self._size_of(a, "annotation") != hw:
                    raise ValueError(f"the annotation of frame {t} of video {g} must be uint8 [{hw[0]},{hw[1]}]")
        fr = self.tracker._input(frames)
        anno = None
        if any(want):
            # every video of the step gets a map in the frames' layout (the kernels read both through one table)
            fill = [annos[i] if want[i] else
                    (torch.zeros(hw, dtype=torch.uint8, device=frames[i].device) if torch.is_tensor(frames[i])
                     else np.zeros(hw, np.uint8)) for i, hw in enumerate(fr.shapes)]
            anno = self.tracker.packer.pack(fill, 1).data
        labels, offsets = self._run(fr, anno, st.need)
        self._advance()
        return [labels[int(o):int(o) + h * w].view(h, w) for o, (h, w) in zip(offsets, fr.shapes)]

    def _run(self, fr, anno, need):
        """One step over the frames fr of `need` ((video g, frame t) pairs in frame-list order): every video of it does
        at its frame t what the reference's loop does: objects start, are tracked and leave, and the fused label map
        (with the scored objects' counts) comes from one ragged kernel pass.  anno: the packed annotations in the
        frames' layout, None when no object starts or is scored.  Returns (packed labels, each video's offset)."""
        f, bt, n = self.f, self.tracker, len(need)
        for i, (g, t) in enumerate(need):
            if t == 0:
                self._hw[g], self._admitted[g] = fr.shapes[i], f
        order = [k for g, _ in need for k in self._members[g]]
        tv = np.full(self.G, -1, np.int64)
        tv[[g for g, _ in need]] = [t for _, t in need]
        t_obj = tv[self._video]                   # each object's frame in this step, -1 where its video is not in it
        # objects of videos that are not in the step (ended, or not admitted yet) are idle
        kinds = np.where(t_obj >= 0, schedule(self._start, self._end, t_obj), OBJ_IDLE)
        scored = np.zeros(len(self.objects), bool)
        if self.score is not None:
            scored = (t_obj >= 0) & (self._lo <= t_obj) & (t_obj < self._hi)
        entry = {g: i for i, (g, _) in enumerate(need)}
        starting = [k for k in order if kinds[k] == OBJ_INIT]
        desc, ptable = bt.packer.table(fr.shapes, 1)
        plane = (desc, int(ptable["offset"][-1]) + fr.shapes[-1][0] * fr.shapes[-1][1])
        H, W = max(s[0] for s in fr.shapes), max(s[1] for s in fr.shapes)      # the grid of the label kernels
        if starting:
            # init boxes (:494-496): one D2H copy, at steps where objects start
            queries = [(entry[self.objects[k][0]], self.objects[k][1]) for k in starting]
            boxes = ops._label_boxes_ragged(anno, desc, n, queries).cpu().numpy()
            missing = [self.objects[k][:2] for k, b in zip(starting, boxes) if b[2] == 0]
            if missing:
                raise ValueError(f"(video, id) {missing} not in the annotation of their start frame")
        # objects that stopped and the objects of videos that ended in the last step leave
        leaving = [k for k, s in enumerate(self._sid) if s is not None and kinds[k] != OBJ_TRACKED]
        if leaving:
            bt.remove([self._sid[k] for k in leaving])
            for k in leaving:
                self._sid[k] = None
        masks = maps = None
        rows = {}
        if bt.N:
            video = {self._sid[k]: self.objects[k][0] for k in order if self._sid[k] is not None}
            self._repoint([entry[video[i]] for i in bt.ids])
            r = bt.track(fr, mask=True, refine=self.p.out_size == 127, paste=False)
            masks, maps = r.extras["mask_prob"], r.extras["maps"]
            rows = {sid: i for i, sid in enumerate(r.extras["ids"])}
            self.last = r
        table = self._entries(kinds, rows, order)
        if starting:
            ids = bt.add(fr, boxes.astype(np.float64), frame_index=[entry[self.objects[k][0]] for k in starting])
            for k, sid in zip(starting, ids):
                self._sid[k] = sid
        per = tuple(len(self._members[g]) for g, _ in need)
        if per != self._off_key:                         # changes only when a video is admitted or retires
            self._off_key = per
            self._offsets = upload(np.concatenate([[0], np.cumsum(per)]), torch.int32, self.dev)
        if not scored.any():
            labels = ops._paste_labels(masks, maps, anno, self._offsets, table, (H, W), self.p.seg_thr, ragged=plane)
        else:
            labels, cnt = ops._paste_labels_iou(masks, maps, anno, self._offsets, table, self._target_ids(scored, order),
                                                (H, W), self.p.seg_thr, self._thrs_dev, ragged=plane)
            # object k's counts at its frame t = f - admitted go to row _row0[k] + t - lo[k]: a constant plus f
            src = [i for i, k in enumerate(order) if scored[k]]
            key = (tuple(src), tuple(int(self._row0[order[i]] - self._lo[order[i]]
                                         - self._admitted[self.objects[order[i]][0]]) for i in src))
            if key != self._copy_key:                    # changes only when a window opens or closes, or entries move
                self._copy_key = key
                self._copy_src = upload(np.asarray(key[0], np.int64), torch.long, self.dev)
                self._copy_dst = upload(np.asarray(key[1], np.int64), torch.long, self.dev)
            self._rows.index_copy_(0, self._copy_dst + f, cnt.index_select(0, self._copy_src))
        for g, t in need:
            self._done[g] = t + 1
        self.f += 1
        return labels, ptable["offset"]
