"""Hyper-parameter sweeps on the device: the grid search of tools/tune_vos.py for G videos at once.

The reference re-runs the whole `siamese_init` / `siamese_track` loop on the same frames once per combination of
(penalty_k, window_influence, lr), one stream at a time, and scores frames start < f < end of each run with `IouMeter`
(utils/average_meter_helper.py:71-113): the pasted soft mask thresholded at each of `np.arange(0.3, 0.81, 0.05)`
against `anno > 0`.  Here the K combinations x G videos are one batch of tracker streams: stream (g, k) reads video g's
frames in place and carries combination k in the tracker's per-stream hyper-parameter table (`sm_step_slots_hp`,
`sm_tracker_update_hp`).  Each frame is scored by one fused paste-back + count kernel (`sm_mask_iou_ragged`, over
the frame's packed annotations) without materialising a frame-sized mask per stream, and the IoU rows stay on the
device until `ParamSweep.result`.

`open_queue` / `needed` / `step` run a sweep of any size, with videos of different lengths and frame sizes, through a
queue of streams (`schedule.Scheduler`).  `open` / `frame` run G same-size videos as one step of that kind each, all
streams admitted at once.

The rotated box of `siamese_track` (contours / minAreaRect) is not computed: tune_vos never scores it.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .schedule import QueueRun, Step
from .tracker import BatchTracker, FramePacker, TrackerParams

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


def _check_combos(combos) -> np.ndarray:
    c = np.asarray(combos, dtype=np.float64)
    if c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0:
        raise ValueError(f"combos must be [K, 3] (penalty_k, window_influence, lr), got {c.shape}")
    if not np.isfinite(c).all():
        raise ValueError("combos must be finite")
    return c


def _one_size(frames, fr) -> bool:
    """Whether `frames` (fr: the tracker's `Packed` of them) is a [G,H,W,3] batch or a list of frames of one size:
    `open` / `frame` take same-size videos only."""
    if isinstance(frames, (list, tuple)):
        return None not in fr.shapes and len(set(fr.shapes)) == 1
    return np.ndim(frames) == 4


class ParamSweep(QueueRun):
    """tune_vos's grid search over `combos` (float64 [K,3] = penalty_k, window_influence, lr; default `grid()`) for G
    videos on one engine.  `net` is a `siammask_b200.Custom` whose max_batch and num_slots cover G*K streams; `params`
    holds the settings the combinations do not (context_amount, out_size, ...).  Masks come from the refine module when
    params.out_size is 127 and from the mask head when it is 63."""

    def __init__(self, net, params: TrackerParams | None = None, combos=None, thrs=THRESHOLDS):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        self.combos = _check_combos(grid() if combos is None else combos)
        self.thrs = _check_thresholds(thrs)
        self._thrs_dev = torch.as_tensor(self.thrs, device=self.dev)
        self.G = 0
        self.f = self.T = 0

    @property
    def K(self) -> int:
        return int(self.combos.shape[0])

    def _reset(self, boxes_xywh, lengths):
        """The state of a run over len(lengths) videos of lengths[g] frames: no stream admitted yet, every IoU row 0."""
        G, K = len(lengths), self.K
        boxes = np.asarray(boxes_xywh, dtype=np.float64)
        if boxes.shape != (G, 4):
            raise ValueError(f"boxes_xywh must be [{G}, 4]")
        self._boxes, self._hw = boxes, [None] * G
        self._video = np.repeat(np.arange(G), K)
        self._vT = np.asarray(lengths, np.int64)[self._video]
        self._off = np.concatenate([[0], np.cumsum(self._vT - 2)[:-1]])      # stream s owns IoU rows off[s] ..
        self._iou = torch.zeros(int((self._vT - 2).sum()), self.thrs.size, dtype=torch.float32, device=self.dev)
        self._admit = np.full(G * K, -1, np.int64)     # the step at which each stream was templated
        self._annos = FramePacker(self.dev)
        self.tracker._clear()
        self._stream_of, self._id_of = {}, [None] * (G * K)
        self._sched = self._plan = None
        self.G, self.f = G, 0
        self._index_rows()

    @torch.no_grad()
    def open(self, frames0, boxes_xywh, num_frames: int):
        """siamese_init of every (video, combination) stream on frame 0.  frames0: uint8 [G,H,W,3] (BGR); boxes_xywh:
        [G,4] top-left x, y, w, h of each video's target; num_frames: T, the videos' length.  Frames 1 .. T-2 are scored
        (tune_vos's start_frame < f < end_frame).  Stream (g, k) is row g*K + k of every per-frame output."""
        fr = self.tracker._input(frames0)
        if not _one_size(frames0, fr):
            raise ValueError("frames0 must be [G,H,W,3]")
        G, K, T = len(fr.shapes), self.K, int(num_frames)
        if T < 3:
            raise ValueError("num_frames must be >= 3 (the first and the last frame are not scored)")
        net = self.tracker.net
        if G * K > net.max_batch or G * K > net.num_slots - self.tracker.slot0:
            raise ValueError(f"{G} videos x {K} combinations = {G * K} streams exceed the engine's max_batch "
                             f"({net.max_batch}) or free slots ({net.num_slots - self.tracker.slot0}); split the grid")
        self._reset(boxes_xywh, [T] * G)
        self.T = T
        self._run(fr, None, Step([(g, 0) for g in range(G)], {s: s // K for s in range(G * K)}, [],
                                 list(range(G * K)), []))
        return self

    @torch.no_grad()
    def frame(self, frames, annos=None):
        """Track frame f (the next one) of every video: frames uint8 [G,H,W,3]; annos uint8 [G,H,W] annotation label maps
        of this frame, required when it is scored (0 < f < T-1).  The frame's IoU rows (float32(intersection / union),
        1 where the union is empty) are written into a device buffer.  Returns the tracker's `TrackResult`.  The streams
        leave the engine after the last frame."""
        f = self.f
        if self._sched is not None:
            raise ValueError("a queue run advances with step(); frame() belongs to open()")
        if not 1 <= f < self.T:
            raise ValueError("call open() first; at most num_frames - 1 frames follow it")
        fr = self.tracker._input(frames)
        if not _one_size(frames, fr) or len(fr.shapes) != self.G:
            raise ValueError(f"frames must be [{self.G},H,W,3]")
        H, W = fr.shapes[0]
        anno = None
        if f < self.T - 1:
            if annos is None:
                raise ValueError(f"frame {f} is scored: annotations are required")
            a = torch.as_tensor(annos).to(self.dev).contiguous()
            if a.dtype != torch.uint8 or tuple(a.shape) != (self.G, H, W):
                raise ValueError(f"annos must be uint8 [{self.G},{H},{W}]")
            anno = self._annos.wrap(a, 1)
        S, K = self.G * self.K, self.K
        return self._run(fr, anno, Step([(g, f) for g in range(self.G)], {s: s // K for s in range(S)},
                                        self._row_streams, [], list(range(S)) if f == self.T - 1 else []))

    def result(self):
        """One D2H copy.  Returns (iou_list float32 [G,K,T] = IouMeter.value('mean') of every stream, per-frame IoU
        float32 [num_frames-2, G, K, T]); rows of frames not tracked yet are 0, as in a partly filled IouMeter.  After
        a queue run the per-frame IoU is a list of G arrays float32 [T_g-2, K, T], one per video."""
        G, K, n = self.G, self.K, self.thrs.size
        flat = self._iou.cpu().numpy()
        rows = [flat[o:o + m] for o, m in zip(self._off, self._vT - 2)]
        means = np.stack([iou_mean(r) for r in rows]).reshape(G, K, n)
        per_video = [np.stack(rows[g * K:(g + 1) * K], 1) for g in range(G)]
        return means, np.stack(per_video, 1) if np.ndim(self.T) == 0 else per_video

    # ------------------------------------------------------------------ queue mode
    @torch.no_grad()
    def open_queue(self, boxes_xywh, num_frames):
        """Queues every (video, combination) stream of a sweep of any size through the engine (`schedule.Scheduler`,
        as `VotRunner.open_queue`): videos of different lengths and frame sizes, at most min(max_batch, free slots)
        streams active, a stream admitted the step after a slot frees.  boxes_xywh: [G,4] top-left x, y, w, h of each
        video's target on its frame 0; num_frames: [G] the videos' lengths (each >= 3).  Each stream scores its own
        video's frames 1 .. T_g-2, as tune_vos's IouMeter(thrs, len(ims) - 2).  Drive it with

            while sweep.pending:
                need = sweep.needed()
                sweep.step([frames[g][t] for g, t in need],
                           [annos[g][t] if 0 < t < T[g] - 1 else None for g, t in need])

        and read `result()`: iou_list [G,K,T] and one per-frame array [T_g-2, K, T] per video."""
        T = np.asarray(num_frames).reshape(-1)
        if T.size == 0:
            raise ValueError("open_queue needs at least one video")
        if not np.issubdtype(T.dtype, np.integer) or (T < 3).any():
            raise ValueError("num_frames must be integers >= 3 (the first and the last frame are not scored)")
        self._reset(boxes_xywh, T)
        self.T = T
        self._queue(T, self.K)
        return self

    def _index_rows(self):
        """Each active tracker row's stream and the IoU row it writes at step 0 (add the step): uploaded only when the
        set of active streams changes."""
        self._row_streams = [self._stream_of[i] for i in self.tracker.ids]
        s = np.asarray(self._row_streams, np.int64)
        self._row_dest = torch.as_tensor(self._off[s] - 1 - self._admit[s], dtype=torch.long, device=self.dev)

    @torch.no_grad()
    def step(self, frames, annos):
        """One step of a queue run: frames[i] / annos[i] are frame t of video g and its uint8 [H,W] annotation for
        (g, t) = needed()[i]; an annotation is required where 0 < t < T_g - 1 and ignored elsewhere (None will do).
        Tracks every running stream one frame of its own video, scores it against the packed annotations, retires the
        streams whose video ends, then templates the admitted streams from their frame 0.  Returns the tracker's
        `TrackResult` of the streams that tracked a frame, or None when none did."""
        st = self._pending_step(frames=frames, annos=annos)
        scored = [0 < t < self.T[g] - 1 for g, t in st.need]
        fr = self.tracker._input(frames)
        for i, (g, t) in enumerate(st.need):
            hw = fr.shapes[i]
            if self._hw[g] is not None and hw != self._hw[g]:
                h, w = hw if hw is not None else (0, 0)
                raise ValueError(f"frame {t} of video {g} is {h}x{w}, its frame 0 {self._hw[g][0]}x{self._hw[g][1]}")
            if scored[i]:
                a = annos[i]
                if a is None:
                    raise ValueError(f"frame {t} of video {g} is scored: its annotation is required")
                if a.dtype not in (np.uint8, torch.uint8) or tuple(a.shape) != tuple(hw):
                    raise ValueError(f"the annotation of frame {t} of video {g} must be uint8 [{hw[0]},{hw[1]}]")
        r = self._run(fr, self._annos.pack([a if s else None for a, s in zip(annos, scored)], 1), st)
        self._advance()
        return r

    def _run(self, fr, anno, st):
        """Step st over the step's frames fr and annotations anno (a `Packed` in frame-list order, skipped where no
        stream is scored; None when none is): tracks every running stream one frame of its own video, scores the rows
        that are not on their video's last frame, retires the streams whose video ends, then templates the admitted
        streams from their frame 0."""
        f, bt = self.f, self.tracker
        r = None
        if st.track:
            self._repoint([st.entry[self._stream_of[i]] for i in bt.ids])
            r = bt.track(fr, mask=True, refine=self.p.out_size == 127, paste=False)
            masks, maps, video, dest = r.extras["mask_prob"], r.extras["maps"], bt._fidx_dev, self._row_dest + f
            last = set(st.retire)
            if last:                                    # rows on their video's last frame are not scored
                keep = [j for j, s in enumerate(self._row_streams) if s not in last]
                sel = torch.tensor(keep, dtype=torch.long, device=self.dev)
                masks, maps, video, dest = masks[sel], maps[sel], video[sel], dest[sel]
            if dest.numel():
                hs, ws = zip(*[s for s in anno.shapes if s is not None])
                cnt = ops._mask_iou_ragged(masks, maps, anno.data, anno.desc, video, (max(hs), max(ws)),
                                           self._thrs_dev)
                inter, union = cnt[..., 0].double(), cnt[..., 1].double()
                # IouMeter.add: intxn / union in float64, stored into a float32 matrix; 1 when the union is empty
                iou = torch.where(union > 0, (inter / union).float(), torch.ones_like(union, dtype=torch.float32))
                self._iou.index_copy_(0, dest, iou)
        gone = [self._id_of[s] for s in st.retire if self._id_of[s] is not None]
        if gone:
            bt.remove(gone)
        for s in st.admit:
            g = int(self._video[s])
            if self._hw[g] is None:
                self._hw[g] = fr.shapes[st.entry[s]]
            self._admit[s] = f
        if st.admit:
            ids = bt.add(fr, self._boxes[self._video[st.admit]], frame_index=[st.entry[s] for s in st.admit],
                         hp=self.combos[[s % self.K for s in st.admit]])
            for s, i in zip(st.admit, ids):
                self._stream_of[i], self._id_of[s] = s, i
        if gone or st.admit:
            self._index_rows()
        self.f += 1
        return r
