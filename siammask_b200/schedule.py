"""Queue scheduling of (sequence, combination) streams through one engine: the admission plan `VotRunner.open_queue`
and `ParamSweep.open_queue` follow.

A benchmark run is G sequences x K hyper-parameter combinations, one tracker stream each, and the engine holds at most
`capacity` of them.  Run in fixed chunks, every stream of a chunk starts on frame 0 and the batch only shrinks, so a
chunk lasts as long as its longest sequence.  The queue instead refills a slot as soon as it frees:

  - streams are admitted in a fixed order, sequences by descending length (ties by index), each sequence's
    combinations in order;
  - at step f, as many waiting streams are admitted as there are free slots: the slots that streams leaving at step
    f-1 freed (and, at step 0, all of them).  An admitted stream is templated from frame 0 of its sequence at step f
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
    `step()`; stream (g, k) is number g*K + k."""

    def __init__(self, lengths, K: int, capacity: int):
        T = np.asarray(lengths).reshape(-1)
        if T.size == 0 or not np.issubdtype(T.dtype, np.integer) or (T < 1).any():
            raise ValueError("lengths must be one integer >= 1 per sequence (every sequence has a frame 0)")
        if int(K) < 1 or int(capacity) < 1:
            raise ValueError("K and capacity must be >= 1")
        self.T, self.K, self.capacity = T.astype(np.int64), int(K), int(capacity)
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
        new = self.order[self._next:self._next + self.capacity - self._active]
        self._next += len(new)
        track = [s for _, _, streams in self._groups for s in streams]
        for s in new:
            g = s // self.K
            if self._groups and self._groups[-1][0] == g and self._groups[-1][1] == f:
                self._groups[-1][2].append(s)
            else:
                self._groups.append((g, f, [s]))
        self._active += len(new)
        need = [(g, f - a) for g, a, _ in self._groups]
        entry = {s: i for i, (_, _, streams) in enumerate(self._groups) for s in streams}
        ending = [i for i, (g, a, _) in enumerate(self._groups) if f - a == self.T[g] - 1]
        retire = [s for i in ending for s in self._groups[i][2]]
        self._groups = [grp for i, grp in enumerate(self._groups) if i not in set(ending)]
        self._active -= len(retire)
        self.f += 1
        return Step(need, entry, track, list(new), retire)


def plan(lengths, K: int, capacity: int) -> list[Step]:
    """Every step of the queue, as a pure function of the lengths."""
    s = Scheduler(lengths, K, capacity)
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
