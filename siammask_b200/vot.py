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

`VotScore` scores finished runs the way tools/eval.py does for VOT2016/2017/2018/2019 ('all' tag): pysot's
AccuracyRobustnessBenchmark (accuracy, robustness, lost number) and EAOBenchmark (expected-overlap curve and EAO), for
every hyper-parameter combination at once, from the runner's device record and without result files:
    1. `sm_vot_trajectory_overlap` reads each frame's entry as load_tracker would read it back from the result file
       ("%.4f" of the float32 value) and computes both per-frame overlaps: bounds (W, H) with burn-in 10 for accuracy,
       bounds (W-1, H-1) for EAO;
    2. `sm_vot_eao_accumulate` turns them into per-combination float64 sums: accuracy sum and count, lost entries and
       frames, and the numerator / denominator of every column of the expected-overlap curve over the fragments pysot
       cuts at each failure.  A column's sums depend only on its index, so runs of any split of the dataset (by
       sequence or by combination) add up; the curve is read out up to the longest sequence added.

Mask-mode VOT (the rotated box of tools/test.py:284-303), per-attribute EAO tags and the OTB branch are not here.
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



# EAOBenchmark's (low, high) per dataset (utils/pysot/evaluation/eao_benchmark.py): EAO averages curve[low-1 .. high-1]
EAO_BOUNDS = {"VOT2016": (100, 356), "VOT2017": (100, 356), "VOT2018": (100, 356), "VOT2019": (46, 291)}


class VotScore:
    """tools/eval.py's VOT numbers ('all' tag) for `num_combos` hyper-parameter combinations, accumulated on the device.

        score = VotScore(K, dataset="VOT2018")          # or low=, high= for other EAO bounds
        score.add(runner)                                # a finished VotRunner; combo_index maps its k to score rows
        r = score.result()                               # accuracy, robustness, lost_number, eao, expected_overlaps

    Every combination's row gathers all sequences added to it; add() may be called per batch of sequences or per chunk
    of the grid.  Sequences must be at least 2 x 2 pixels (EAO scores them with bounds (W-1, H-1))."""

    def __init__(self, num_combos: int, dataset: str | None = "VOT2018", low: int | None = None,
                 high: int | None = None, device=None):
        K = int(num_combos)
        if not 1 <= K <= 65535:
            raise ValueError(f"num_combos must be in [1, 65535], got {num_combos}")
        if low is None and high is None:
            if dataset not in EAO_BOUNDS:
                raise ValueError(f"unknown dataset {dataset!r}: pass low= and high= (known: {sorted(EAO_BOUNDS)})")
            low, high = EAO_BOUNDS[dataset]
        elif low is None or high is None or not 1 <= int(low) <= int(high):
            raise ValueError(f"EAO bounds need 1 <= low <= high, got low={low}, high={high}")
        self.K, self.low, self.high = K, int(low), int(high)
        self.dev = torch.device(device if device is not None else "cuda")
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float64, device=self.dev)      # noqa: E731
        self._num, self._den = z(K, 0), z(K, 0)
        self._tail, self._tail_next = z(K, 2), z(K, 2)
        self._stats = z(K, 4)                       # accuracy sum, accuracy count, lost entries, frames
        self._sequences = np.zeros(K, np.int64)

    @property
    def cap(self) -> int:
        return int(self._num.shape[1])

    def _rows(self, combo_index, K: int) -> np.ndarray:
        ci = np.arange(K) if combo_index is None else np.asarray(combo_index)
        if ci.shape != (K,) or not np.issubdtype(ci.dtype, np.integer):
            raise ValueError(f"combo_index must be {K} integers (one score row per combination of the run)")
        if (ci < 0).any() or (ci >= self.K).any():
            raise ValueError(f"combo_index entries must lie in [0, {self.K})")
        if len(set(ci.tolist())) != K:
            raise ValueError("combo_index entries must be distinct")
        return ci.astype(np.int64)

    @torch.no_grad()
    def add(self, runner: VotRunner, combo_index=None):
        """Adds every stream of a VotRunner whose sequences have all ended: stream (g, k) goes to score row
        combo_index[k] (default k).  Reads the runner's device record in place; no host sync."""
        if runner.G == 0:
            raise ValueError("the runner has not been opened")
        if (runner.T > runner.f).any():
            raise ValueError(f"every sequence must have ended: frame {runner.f} of lengths {runner.T.tolist()}")
        sizes = [(int(h), int(w)) for h, w in runner._hw]
        self._add(runner._rec, runner._gt, runner.T, sizes, runner.K, combo_index)
        return self

    @torch.no_grad()
    def add_regions(self, regions, gt, sizes, combo_index=None):
        """Adds trajectories in the form `VotRunner.result()` returns: regions[g][k] is the list of sequence g under
        combination k (1 init, 2 lost, 0 skipped, or a location x, y, w, h), gt[g] its float64 [T_g, 8] polygons and
        sizes[g] its frame (H, W).  Every list must have T_g entries."""
        gts = check_gt(gt)
        G = len(gts)
        if len(regions) != G or len(sizes) != G or G == 0:
            raise ValueError("regions, gt and sizes need one entry per sequence")
        K = len(regions[0])
        if K == 0 or any(len(r) != K for r in regions):
            raise ValueError("every sequence needs the same number of combinations")
        T = np.array([len(a) for a in gts])
        Tmax = int(T.max())
        rec = np.zeros((Tmax, G * K, 5))
        for g in range(G):
            for k in range(K):
                traj = regions[g][k]
                if len(traj) != T[g]:
                    raise ValueError(f"regions[{g}][{k}] has {len(traj)} entries, the sequence {T[g]} frames")
                for f, x in enumerate(traj):
                    if isinstance(x, (int, np.integer)):
                        if x not in (CODE_SKIP, CODE_INIT, CODE_LOST):
                            raise ValueError(f"regions[{g}][{k}][{f}]: integer entries are 0, 1 or 2")
                        rec[f, g * K + k, 0] = x
                    else:
                        loc = np.asarray(x, np.float64).reshape(-1)
                        if loc.size != 4 or not np.isfinite(loc).all():
                            raise ValueError(f"regions[{g}][{k}][{f}]: a location is 4 finite values")
                        rec[f, g * K + k] = (CODE_LOCATION, *loc)
        locs = rec[..., 1:]
        if (np.abs(locs[..., :2]) + np.abs(locs[..., 2:]) > ops.VOT_COORD_LIMIT / 2).any():
            raise ValueError("locations must lie within +-2^19 px")
        polys = np.zeros((G, Tmax, 8), np.float32)
        for g, a in enumerate(gts):
            polys[g, :len(a)] = a
        self._add(torch.from_numpy(rec).to(self.dev), torch.from_numpy(polys).to(self.dev), T,
                  [(int(h), int(w)) for h, w in sizes], K, combo_index)
        return self

    def _add(self, rec, gt, T, sizes, K, combo_index):
        rows = self._rows(combo_index, K)
        G = len(T)
        wh = np.array([(w, h) for h, w in sizes], np.int64)
        if (wh < 2).any() or ((wh[:, 0] + 1) * (wh[:, 1] + 1) > 2 ** 31 - 1).any():
            raise ValueError("frames must be at least 2 x 2 px (EAO uses bounds (W-1, H-1)) and (W+1)*(H+1) < 2^31")
        Tmax, S = int(np.max(T)), G * K
        if 2 * Tmax * S > 2 ** 31 - 1:
            raise ValueError(f"{S} streams x {Tmax} frames is too large for one add(); add the run in parts")
        if self.dev.type != "cuda":
            raise RuntimeError("VotScore runs on a CUDA device only; there is no CPU path")
        seq = np.repeat(np.arange(G), K)
        table = np.concatenate([seq, np.asarray(T)[seq], np.tile(rows, G), wh[seq].ravel()]).astype(np.int32)
        t = torch.from_numpy(table).to(self.dev)                       # one upload: seq, lengths, combo, (W, H)
        seq_d, len_d, combo_d, wh_d = t[:S], t[S:2 * S], t[2 * S:3 * S], t[3 * S:]
        with torch.cuda.device(self.dev):
            acc, eao = ops._vot_trajectory_overlap(rec, Tmax, S, gt, seq_d, wh_d, len_d)
            old = self.cap
            if Tmax > old:                                             # grow: earlier fragments reach the new columns
                num = torch.zeros(self.K, Tmax, dtype=torch.float64, device=self.dev)
                den = torch.zeros_like(num)
                num[:, :old], den[:, :old] = self._num, self._den
                self._num, self._den = num, den
            ops._vot_eao_accumulate(eao, acc, rec, len_d, combo_d, old, self._tail, self._tail_next, self._num,
                                    self._den, self._stats)
        self._tail, self._tail_next = self._tail_next, self._tail
        self._sequences[rows] += G

    def result(self) -> dict:
        """One D2H copy.  Per combination (arrays [K]): accuracy (nan-mean of the burn-in overlaps), robustness (lost
        entries per 100 frames), lost_number, eao, and expected_overlaps float32 [K, max_T] (the curve, entry 0 = 1);
        sequences: how many sequences each row has gathered.  Rows without sequences are NaN."""
        cap = self.cap
        h = torch.cat([self._num, self._den, self._stats], 1).cpu().numpy()
        num, den, st = h[:, :cap], h[:, cap:2 * cap], h[:, 2 * cap:]
        with np.errstate(divide="ignore", invalid="ignore"):
            curve = np.where(den > 0, num / np.where(den > 0, den, 1), 0.0).astype(np.float32)
            if cap:
                curve[:, 0] = 1
            seg = curve[:, self.low - 1:min(self.high, cap)].astype(np.float64)
            valid = ~np.isnan(seg)
            eao = np.where(valid, seg, 0.0).sum(1) / valid.sum(1)
            return {"accuracy": st[:, 0] / st[:, 1], "robustness": st[:, 2] / st[:, 3] * 100,
                    "lost_number": st[:, 2].astype(np.int64), "eao": eao, "expected_overlaps": curve,
                    "sequences": self._sequences.copy()}
