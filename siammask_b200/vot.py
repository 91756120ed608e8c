"""The VOT supervised protocol on the device: track_vot of tools/test.py:318-418 (and its grid search,
tools/tune_vot.py) for N sequences at once.

Per sequence, the reference initialises the tracker on frame 0 from `get_axis_aligned_bbox(gt[0])`, then tracks each
frame without masks and scores it with pyvotkit's `vot_overlap(gt polygon, predicted rectangle, (W, H))`.  An overlap
of 0 is a failure: the frame's entry is 2, `lost_times` grows, the next 4 frames are skipped (entry 0) and the tracker
is initialised again from the ground truth on the 5th (entry 1).  Any other overlap, NaN included, keeps the
prediction `cxy_wh_2_rect(target_pos, target_sz)` as the entry.

Here every sequence (x every hyper-parameter combination) is one stream of a `BatchTracker`:
    1. `track(mask=False)` advances all active streams;
    2. `sm_vot_overlap` scores each stream's clamped-state rectangle against its sequence's ground truth of the frame
       (`sm_vot_overlap_sized` with each sequence's own (W, H) when the sequences differ in frame size);
    3. device tensors keep each stream's start frame, entry codes, float64 locations and lost_times, without a host
       sync;
    4. streams whose start frame is this frame are templated again in their own engine slots (`BatchTracker.reinit`);
    5. streams whose sequence has ended leave the batch.
A lost stream stays in the batch through its 4 skipped frames: its outputs are discarded and the device writes 0 for
them.  The host learns of a failure only when it must re-initialise, 5 frames later: each frame's loss flags travel to
pinned memory behind an event, and frame f + 5 reads frame f's flags, which are long complete.  A frame therefore
queues its work without waiting for the device, unless it re-initialises streams or one of its sequences ends: those
upload small tables (the template rows, the active set) once.

Sequences of different frame sizes run in one batch: pass each frame as a list of G frames (`BatchTracker` packs them;
the entry of a sequence that has ended may be None).

Mask-mode VOT (the rotated box of tools/test.py:284-303), EAO / accuracy-robustness and the OTB branch are not here.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .tracker import BatchTracker, Packed, TrackerParams

# tools/tune_vot.py's argparse defaults: a 9 x 14 x 3 grid of (penalty_k, window_influence, lr)
DEFAULT_PENALTY_K = np.arange(0.05, 0.5, 0.05)
DEFAULT_WINDOW_INFLUENCE = np.arange(0.1, 0.8, 0.05)
DEFAULT_LR = np.arange(0.35, 0.5, 0.05)

CODE_SKIP, CODE_INIT, CODE_LOST, CODE_LOCATION = 0, 1, 2, 3
SKIP_FRAMES = 5                   # start_frame = f + 5 after a failure (tools/test.py:362)


def get_axis_aligned_bbox(region):
    """utils/bbox_helper.py:52-75 for an 8-value polygon, in the same float64 numpy arithmetic: (cx, cy, w, h), the
    centre of the vertices and the axis-aligned box scaled to the polygon's area, plus one pixel."""
    r = np.asarray(region, dtype=np.float64).reshape(-1)
    if r.size != 8:
        raise ValueError("get_axis_aligned_bbox expects an 8-value polygon")
    xs, ys = r[0::2], r[1::2]
    x_lo, x_hi, y_lo, y_hi = min(xs), max(xs), min(ys), max(ys)
    side_a = np.linalg.norm(r[0:2] - r[2:4])
    side_b = np.linalg.norm(r[2:4] - r[4:6])
    s = np.sqrt(side_a * side_b / ((x_hi - x_lo) * (y_hi - y_lo)))
    return np.mean(xs), np.mean(ys), s * (x_hi - x_lo) + 1, s * (y_hi - y_lo) + 1


def check_gt(gt) -> list[np.ndarray]:
    """Each sequence's ground truth as float64 [T, 8]; ValueError unless every row has 8 values, finite and within
    +-2^20 px (sm_vot_overlap's precondition)."""
    out = []
    for g, a in enumerate(gt):
        a = np.asarray(a, dtype=np.float64)
        if a.ndim != 2 or a.shape[1] != 8 or a.shape[0] < 1:
            raise ValueError(f"gt[{g}] must be float64 [T, 8] with T >= 1 (4-point polygons; convert 4-value "
                             f"rectangles to 8 values first, as utils/benchmark_helper.py does), got {a.shape}")
        if not np.isfinite(a).all():
            raise ValueError(f"gt[{g}] must be finite")
        if (np.abs(a) > ops.VOT_COORD_LIMIT).any():
            raise ValueError(f"gt[{g}]: coordinates must lie within +-2^20 px")
        out.append(a)
    return out


def regions_from_record(rec: np.ndarray, T: int) -> list:
    """One stream's regions in the reference's form from its rows rec float64 [>=T, 5] = (code, location[4])."""
    regions = []
    for f in range(T):
        c = int(rec[f, 0])
        regions.append(rec[f, 1:5].copy() if c == CODE_LOCATION else c)
    return regions


def write_result(path, regions) -> None:
    """The result file of track_vot (tools/test.py:402-406): "{:d}" for an integer entry, else the location's values
    rounded to a C float and printed with "%.4f" (pyvotkit's vot_float2str), joined by commas."""
    lines = []
    for x in regions:
        if isinstance(x, (int, np.integer)):
            lines.append("{:d}".format(int(x)))
        else:
            lines.append(",".join("%.4f" % float(np.float32(v)) for v in np.asarray(x).reshape(-1)))
    with open(path, "w") as f:
        f.write("".join(line + "\n" for line in lines))


class VotRunner:
    """track_vot for G sequences on one engine; their frames may differ in size.  With combos=None
    each sequence is one stream with `params`' hyper-parameters; with combos float64 [K,3] = (penalty_k,
    window_influence, lr) rows (tune_vot's grid is `tune.grid(DEFAULT_PENALTY_K, DEFAULT_WINDOW_INFLUENCE,
    DEFAULT_LR)`, in its nested-loop order) each sequence runs every combination, and stream (g, k) is row g*K + k of
    every output, as in `ParamSweep`.  `net` is a `siammask_b200.Custom` (with or without the mask branch) whose
    max_batch and num_slots cover G*K streams."""

    def __init__(self, net, params: TrackerParams | None = None, combos=None):
        self.tracker = BatchTracker(net, params)
        self.p = self.tracker.p
        self.dev = self.tracker.dev
        self.combos = None
        if combos is not None:
            c = np.asarray(combos, dtype=np.float64)
            if c.ndim != 2 or c.shape[1] != 3 or c.shape[0] == 0:
                raise ValueError(f"combos must be [K, 3] (penalty_k, window_influence, lr), got {c.shape}")
            if not np.isfinite(c).all():
                raise ValueError("combos must be finite")
            self.combos = c
        self.G = 0
        self.f = 0

    @property
    def K(self) -> int:
        return 1 if self.combos is None else int(self.combos.shape[0])

    @torch.no_grad()
    def open(self, frames0, gt):
        """siamese_init of every stream on frame 0.  frames0: uint8 [G,H,W,3] (BGR) frame 0 of each sequence, or a list
        of G frames [H_g,W_g,3] whose sizes may differ; gt: G float64 arrays [T_g, 8], each sequence's ground-truth
        polygons (lengths may differ).  Every gt row is checked and uploaded here, once."""
        fr = self.tracker._input(frames0)
        if isinstance(fr, Packed):
            if any(s is None for s in fr.shapes):
                raise ValueError("frames0 must hold frame 0 of every sequence")
            G, self._hw = len(fr.shapes), list(fr.shapes)
        else:
            if fr.dim() != 4:
                raise ValueError("frames0 must be [G,H,W,3]")
            G, self._hw = int(fr.shape[0]), [self.tracker._hw(fr)] * int(fr.shape[0])
        K = self.K
        gts = check_gt(gt)
        if len(gts) != G:
            raise ValueError(f"one gt array per sequence expected ({G})")
        net, S = self.tracker.net, G * K
        if S > net.max_batch or S > net.num_slots - self.tracker.slot0:
            raise ValueError(f"{G} sequences x {K} combinations = {S} streams exceed the engine's max_batch "
                             f"({net.max_batch}) or free slots ({net.num_slots - self.tracker.slot0}); split the run")
        self.T = np.array([a.shape[0] for a in gts])
        Tmax = int(self.T.max())
        # get_axis_aligned_bbox of every gt row, on the host in the reference's arithmetic: (cx, cy, w, h) [G, Tmax, 4]
        self._init = np.zeros((G, Tmax, 4))
        polys = np.zeros((G, Tmax, 8), np.float32)
        for g, a in enumerate(gts):
            with np.errstate(divide="ignore", invalid="ignore"):
                self._init[g, :len(a)] = [get_axis_aligned_bbox(row) for row in a]
            polys[g, :len(a)] = a                            # Polygon() stores C floats
        self._gt = torch.from_numpy(polys).to(self.dev)
        video = np.repeat(np.arange(G), K)
        self._video = video
        c0 = self._init[video, 0]
        self.tracker._clear()
        ids = self.tracker.add_state(fr, c0[:, 0:2], c0[:, 2:4], frame_index=video,
                                     hp=None if self.combos is None else np.tile(self.combos, (G, 1)))
        self._stream_of = {i: s for s, i in enumerate(ids)}          # tracker id -> stream
        self._id_of = ids
        # rows [0, Tmax) of stream s: (entry code, location x, y, w, h); row Tmax: (lost_times, 0, 0, 0, 0)
        self._rec = torch.zeros(Tmax + 1, S, 5, dtype=torch.float64, device=self.dev)
        self._rec[0, :, 0] = CODE_INIT
        self._start = torch.zeros(S, dtype=torch.int32, device=self.dev)
        self._flags = torch.zeros(S, dtype=torch.uint8, device=self.dev)
        self._pinned = [torch.zeros(S, dtype=torch.uint8).pin_memory() for _ in range(SKIP_FRAMES + 1)]
        self._events = [None] * (SKIP_FRAMES + 1)
        self.G, self.f = G, 0
        self._index_rows()
        self._retire()
        self.f = 1
        return self

    def _index_rows(self):
        """Stream and sequence of each active tracker row: a host list and device indices.  The upload waits for the
        copy, so it runs only when the set of active streams changes."""
        self._row_streams = [self._stream_of[i] for i in self.tracker.ids]
        self._row_dev = torch.tensor(self._row_streams, dtype=torch.long, device=self.dev)
        self._row_video = torch.as_tensor(self._video[self._row_streams], dtype=torch.long, device=self.dev)
        if len(set(self._hw)) > 1:                      # each row's own (W, H) for sm_vot_overlap_sized
            wh = [self._hw[self._video[s]][::-1] for s in self._row_streams]
            self._row_wh = torch.tensor(wh, dtype=torch.int32, device=self.dev).reshape(-1, 2)

    def _retire(self):
        """Step 5: streams whose sequence ends with frame self.f leave the batch."""
        done = [i for i in self.tracker.ids if self.T[self._video[self._stream_of[i]]] == self.f + 1]
        if done:
            self.tracker.remove(done)
            self._index_rows()

    @torch.no_grad()
    def frame(self, frames):
        """Frame f (the next one) of every sequence: frames uint8 [G,H,W,3], or a list of G frames [H_g,W_g,3] in which
        the entry of a sequence that has ended may be None; the slots of sequences that have ended are not read (any
        frame of the right size will do).  Returns the tracker's `TrackResult` of the streams that were active, whose
        rows are skipped or re-initialised streams too."""
        f = self.f
        if self.G == 0 or self.tracker.N == 0:
            raise ValueError("call open() first; every sequence has ended")
        fr = self.tracker._input(frames)
        if isinstance(fr, Packed):
            if len(fr.shapes) != self.G:
                raise ValueError(f"frames must be a list of {self.G} frames")
        elif fr.dim() != 4 or fr.shape[0] != self.G:
            raise ValueError(f"frames must be [{self.G},H,W,3]")
        rows = self._row_dev
        # 1. track every active stream (skipped ones too: their outputs are discarded below)
        r = self.tracker.track(fr, mask=False)
        st = r.state
        # 2. overlap of the gt polygon with the rectangle of the clamped state: float64 vertices, stored as C floats
        x0 = st[:, 0] - st[:, 2] / 2
        y0 = st[:, 1] - st[:, 3] / 2
        x1, y1 = x0 + st[:, 2], y0 + st[:, 3]
        loc = torch.stack([x0, y0, st[:, 2], st[:, 3]], 1)
        pred = torch.stack([x0, y0, x1, y0, x1, y1, x0, y1], 1).float()
        if len(set(self._hw)) > 1:
            ov = ops._vot_overlap_sized(self._gt[self._row_video, f], pred, self._row_wh)
        else:
            ov = ops._vot_overlap(self._gt[self._row_video, f], pred, self._hw[0])
        # 3. bookkeeping on the device: init / track / skip by the stream's start frame; only an overlap of exactly 0
        #    is a failure (NaN is truthy)
        start = self._start[rows]
        tracking = start < f
        lost = tracking & (ov == 0)
        code = torch.where(start == f, CODE_INIT, torch.where(lost, CODE_LOST, CODE_LOCATION * tracking.long()))
        self._rec[f, rows, 0] = code.double()
        self._rec[f, rows, 1:5] = torch.where(tracking & ~lost, 1, 0).unsqueeze(1) * loc
        self._rec[-1, rows, 0] += lost.double()
        self._start[rows] = torch.where(lost, f + SKIP_FRAMES, start)
        self._flags.zero_()
        self._flags[rows] = lost.to(torch.uint8)
        slot = f % len(self._pinned)
        self._pinned[slot].copy_(self._flags, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        self._events[slot] = ev
        # 4. re-initialise the streams lost at frame f - 5 (their start frame is f), from the gt of frame f
        if f > SKIP_FRAMES:                              # nothing is lost on frame 0
            old = (f - SKIP_FRAMES) % len(self._pinned)
            self._events[old].synchronize()
            again = np.nonzero(self._pinned[old].numpy())[0]
            active = set(self._row_streams)
            again = [int(s) for s in again if int(s) in active]
            if again:
                c = self._init[self._video[again], f]
                self.tracker.reinit([self._id_of[s] for s in again], fr, c[:, 0:2], c[:, 2:4])
        # 5. sequences that end with this frame leave the batch
        self._retire()
        self.f += 1
        return r

    def result(self):
        """One D2H copy.  Returns (regions, lost_times): regions[g][k] is stream (g, k)'s list in the reference's form
        (1 init, 2 lost, 0 skipped, or a float64 [4] location x, y, w, h) over the frames tracked so far; lost_times
        int [G, K]."""
        rec = self._rec.cpu().numpy()
        G, K = self.G, self.K
        n = np.minimum(self.T, self.f)
        regions = [[regions_from_record(rec[:, g * K + k], int(n[g])) for k in range(K)] for g in range(G)]
        return regions, rec[-1, :, 0].astype(np.int64).reshape(G, K)

