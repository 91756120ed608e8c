"""Queue scheduling of (sequence, combination) streams through one engine: the admission plan `VotRunner.open_queue`,
`ParamSweep.open_queue` and `VideoSegmenter.open_queue` follow, and the plumbing those classes share (`QueueRun`).

A benchmark run is G sequences x K hyper-parameter combinations, one tracker stream each, and the engine holds at most
`capacity` of them.  Run in fixed chunks, every stream of a chunk starts on frame 0 and the batch only shrinks, so a
chunk lasts as long as its longest sequence.  The queue instead refills a slot as soon as it frees:

  - streams are admitted in a fixed order, sequences by descending length (ties by index), each sequence's
    combinations in order;
  - at step f, waiting streams are admitted in that order while the next one fits into the free slots: the slots
    that streams leaving at step f-1 freed (and, at step 0, all of them).  A stream holds one slot, or its sequence's
    width (`widths`: a video whose objects are tracked at once holds as many slots as it has objects at its peak) from
    its admission until it leaves.  A stream that does not fit waits, and so does every stream behind it: the plan
    stays a pure function of the lengths, widths and capacity.  An admitted stream is templated from frame 0 of its sequence at step f
    and tracks frame t of its own sequence at step f + t;
  - a stream leaves after the step that reads its sequence's last frame.

Every stream advances one frame per step, so the streams of one sequence admitted at the same step read the same frame
at every step: they form a group and share one entry of the step's frame list (also when a sequence's combinations are
spread over several admissions).  The frame list (`Step.need`) holds one (sequence, frame) pair per group, in the order
the groups were admitted; it changes only in the steps that admit streams or follow a departure.  Everything here is
known on the host from the lengths: no device result decides an admission or a departure."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class Step:
    """One step of the plan.  need: the distinct (sequence g, frame t) pairs the step reads, in frame-list order;
    entry: the position in `need` of every stream that is tracked or admitted in the step; track: the streams that
    track a frame (t >= 1), in admission order; admit: the streams templated from frame 0 in the step; retire: the
    streams whose last frame the step reads (tracked or, for one-frame sequences, admitted): they leave after it."""
    need: list
    entry: dict
    track: list
    admit: list
    retire: list


class Scheduler:
    """The plan for sequences of `lengths` frames x K combinations through `capacity` slots, one `Step` per call of
    `step()`; stream (g, k) is number g*K + k.  widths (optional): the slots each stream of sequence g holds, one
    integer >= 1 per sequence (default 1); a width above the capacity is a ValueError."""

    def __init__(self, lengths, K: int, capacity: int, widths=None):
        T = np.asarray(lengths).reshape(-1)
        if T.size == 0 or not np.issubdtype(T.dtype, np.integer) or (T < 1).any():
            raise ValueError("lengths must be one integer >= 1 per sequence (every sequence has a frame 0)")
        if int(K) < 1 or int(capacity) < 1:
            raise ValueError("K and capacity must be >= 1")
        w = np.ones(T.size, np.int64) if widths is None else np.asarray(widths).reshape(-1)
        if w.size != T.size or not np.issubdtype(w.dtype, np.integer) or (w < 1).any():
            raise ValueError("widths must be one integer >= 1 per sequence")
        if (w > int(capacity)).any():
            g = int(np.argmax(w > int(capacity)))
            raise ValueError(f"sequence {g} needs {int(w[g])} slots at once; the engine has {int(capacity)}")
        self.T, self.K, self.capacity = T.astype(np.int64), int(K), int(capacity)
        self.width = w.astype(np.int64)
        seqs = sorted(range(T.size), key=lambda g: (-int(T[g]), g))
        self.order = [g * self.K + k for g in seqs for k in range(self.K)]
        self._next = 0                          # position in `order` of the next stream to admit
        self._groups: list[tuple[int, int, list]] = []         # (sequence, admission step, streams), in admission order
        self._active = 0
        self.f = 0

    @property
    def done(self) -> bool:
        return self._next == len(self.order) and not self._groups

    def step(self) -> Step:
        if self.done:
            raise ValueError("every stream has finished")
        f = self.f
        new, free = [], self.capacity - self._active
        while self._next < len(self.order) and self.width[self.order[self._next] // self.K] <= free:
            new.append(self.order[self._next])
            free -= int(self.width[self.order[self._next] // self.K])
            self._next += 1
        track = [s for _, _, streams in self._groups for s in streams]
        for s in new:
            g = s // self.K
            if self._groups and self._groups[-1][0] == g and self._groups[-1][1] == f:
                self._groups[-1][2].append(s)
            else:
                self._groups.append((g, f, [s]))
        self._active = self.capacity - free
        need = [(g, f - a) for g, a, _ in self._groups]
        entry = {s: i for i, (_, _, streams) in enumerate(self._groups) for s in streams}
        ending = [i for i, (g, a, _) in enumerate(self._groups) if f - a == self.T[g] - 1]
        retire = [s for i in ending for s in self._groups[i][2]]
        self._groups = [grp for i, grp in enumerate(self._groups) if i not in set(ending)]
        self._active -= int(sum(self.width[s // self.K] for s in retire))
        self.f += 1
        return Step(need, entry, track, list(new), retire)


class QueueRun:
    """The queue plumbing of `VotRunner`, `ParamSweep` and `VideoSegmenter`, whose `open` / `frame` and `open_queue` /
    `step` feed one step body per class.  `tracker` is the run's `BatchTracker`; `_sched` is None outside a queue run."""

    _sched = None
    _plan = None

    @property
    def pending(self) -> bool:
        """Whether a queue run has steps left."""
        return self._sched is not None and self._plan is not None

    def needed(self) -> list:
        """The distinct (sequence, frame) pairs the next `step` reads, in the order its lists follow."""
        return list(self._pending_step().need)

    def _pending_step(self, **lists) -> Step:
        """The next step of the plan; ValueError unless a queue run is pending and every list (frames, annos) holds one
        entry per needed() entry."""
        if not self.pending:
            raise ValueError("no queue step is pending: call open_queue() first; the run has finished")
        n = len(self._plan.need)
        for name, v in lists.items():
            if not isinstance(v, (list, tuple)) or len(v) != n:
                raise ValueError(f"{name} must be a list of {n} entries, one per needed() entry")
        return self._plan

    def _queue(self, lengths, K: int, widths=None):
        """Plans a queue run through min(max_batch, free slots) engine slots and takes its first step."""
        net = self.tracker.net
        cap = min(net.max_batch, net.num_slots - self.tracker.slot0)
        if cap < 1:
            raise ValueError("the engine has no free slot")
        self._sched = Scheduler(lengths, K, cap, widths)
        self._plan = self._sched.step()

    def _advance(self):
        self._plan = self._sched.step() if not self._sched.done else None

    def _repoint(self, want: list):
        """Points the tracker's rows at their entries (`want`, in row order) of the step's frame list.  The list moves
        only after admissions or departures, so the table is uploaded only then."""
        bt = self.tracker
        if want != bt._fidx:
            bt.set_frame_index(bt.ids, want)


MAX_LANES = 2         # engine.cu kMaxLanes
LANE_MIN_B = 8        # engine.cu kLaneMinB: a lane gets at least this many streams


def lane_split(B: int, max_batch: int) -> list[int]:
    """The streams each execution lane of an engine built for `max_batch` runs in a call of batch B, lane 0 first
    (engine.cu lanes_for / chunk): B splits over two lanes once both get at least LANE_MIN_B streams, lane 0 taking the
    odd one.  Every search-side and refine launch of the call runs once per lane with M = (lane streams) x Ho x Wo;
    template calls are not split."""
    if not 1 <= int(B) <= int(max_batch):
        raise ValueError("need 1 <= B <= max_batch")
    n = max(1, min(MAX_LANES, int(max_batch) // LANE_MIN_B))
    n = max(1, min(n, int(B) // LANE_MIN_B))
    return [int(B) // n + (1 if lane < int(B) % n else 0) for lane in range(n)]


def plan(lengths, K: int, capacity: int, widths=None) -> list[Step]:
    """Every step of the queue, as a pure function of the lengths (and widths)."""
    s = Scheduler(lengths, K, capacity, widths)
    out = []
    while not s.done:
        out.append(s.step())
    return out


def chunked_steps(lengths, K: int, capacity: int) -> int:
    """Steps of the same run in fixed chunks of capacity // K sequences in index order, each chunk opened on frame 0 and
    run until its longest sequence ends (one `VotRunner.open` per chunk); requires K <= capacity."""
    per = int(capacity) // int(K)
    if per < 1:
        raise ValueError("a chunk must hold every combination of one sequence (K <= capacity)")
    T = np.asarray(lengths, np.int64).reshape(-1)
    return int(sum(T[i:i + per].max() for i in range(0, T.size, per)))
