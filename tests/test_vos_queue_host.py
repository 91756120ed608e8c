"""The VOS queue on the host (no GPU): the scheduler with per-sequence widths against the one-slot plan, the peak width
of a video's objects against brute force, `VideoSegmenter.needs_anno` over the "whole" / "spans" windows, and the
argument checks `open_queue` and `step` make before any device work."""
import numpy as np
import pytest
import torch

from siammask_b200 import schedule
from siammask_b200.vos import VideoSegmenter, peak_width


def _one_slot_plan(lengths, K, cap):
    """The one-slot admission rule as a plain restatement: at each step take as many streams as slots are free."""
    T = np.asarray(lengths, np.int64)
    order = [g * K + k for g in sorted(range(T.size), key=lambda g: (-int(T[g]), g)) for k in range(K)]
    nxt, groups, active, f, out = 0, [], 0, 0, []
    while nxt < len(order) or groups:
        new = order[nxt:nxt + cap - active]
        nxt += len(new)
        track = [s for _, _, ss in groups for s in ss]
        for s in new:
            if groups and groups[-1][0] == s // K and groups[-1][1] == f:
                groups[-1][2].append(s)
            else:
                groups.append((s // K, f, [s]))
        active += len(new)
        need = [(g, f - a) for g, a, _ in groups]
        ending = [i for i, (g, a, _) in enumerate(groups) if f - a == T[g] - 1]
        retire = [s for i in ending for s in groups[i][2]]
        groups = [grp for i, grp in enumerate(groups) if i not in ending]
        active -= len(retire)
        out.append((need, track, list(new), retire))
        f += 1
    return out


def _key(steps):
    return [(st.need, st.entry, st.track, st.admit, st.retire) for st in steps]


def test_width_one_plans_equal_one_slot_plans():
    rng = np.random.RandomState(0)
    for _ in range(60):
        T = rng.randint(1, 30, size=rng.randint(1, 12))
        K, cap = int(rng.randint(1, 5)), int(rng.randint(1, 12))
        default = schedule.plan(T, K, cap)
        assert _key(default) == _key(schedule.plan(T, K, cap, np.ones(T.size, np.int64)))
        assert [(st.need, st.track, st.admit, st.retire) for st in default] == _one_slot_plan(T, K, cap)


def _replay_widths(T, widths, cap):
    steps = schedule.plan(T, 1, cap, widths)
    order = schedule.Scheduler(T, 1, cap, widths).order
    admitted, active, used = [], set(), 0
    for f, st in enumerate(steps):
        assert st.track == [s for s in admitted if s in active]
        used += sum(widths[s] for s in st.admit)
        assert used <= cap                                      # never more slots than the engine has
        admitted += st.admit
        assert admitted == order[:len(admitted)]                # in order, nobody skips ahead
        if len(admitted) < len(order):                          # the next one waits only when it does not fit
            assert widths[order[len(admitted)]] > cap - used
        for g in st.admit + st.track:
            assert st.need[st.entry[g]][0] == g
        active |= set(st.admit)
        for g in st.retire:
            assert st.need[st.entry[g]] == (g, T[g] - 1)
        active -= set(st.retire)
        used -= sum(widths[s] for s in st.retire)
    assert not active and sorted(admitted) == list(range(len(T)))
    return steps


def test_width_plans_respect_capacity_and_order():
    rng = np.random.RandomState(1)
    for _ in range(60):
        G = rng.randint(1, 14)
        T, cap = rng.randint(1, 40, size=G), int(rng.randint(1, 9))
        widths = rng.randint(1, cap + 1, size=G)
        steps = _replay_widths(T, widths, cap)
        assert _key(steps) == _key(schedule.plan(T.copy(), 1, cap, widths.copy()))      # a pure function


def test_a_wide_sequence_blocks_narrower_ones_behind_it():
    # order: video 1 (length 9, width 3), video 0 (8, 1), video 2 (5, 2), video 3 (2, 1)
    steps = _replay_widths(np.array([8, 9, 5, 2]), np.array([1, 3, 2, 1]), 4)
    assert steps[0].admit == [1, 0]
    # after video 0 leaves, video 2 (width 2) does not fit into the one free slot, and video 3 may not overtake it
    assert steps[7].retire == [0] and steps[8].retire == [1]
    assert all(not st.admit for st in steps[1:9]) and steps[9].admit == [2, 3]


def test_width_checks():
    with pytest.raises(ValueError, match="slots"):
        schedule.Scheduler([4, 5], 1, 3, [2, 4])
    for bad in ([1], [0, 1], [1.5, 1]):
        with pytest.raises(ValueError, match="widths"):
            schedule.Scheduler([4, 5], 1, 3, bad)


def _brute_peak(start, end):
    hi = max(end, default=-1)
    return max([sum(s <= f <= e for s, e in zip(start, end)) for f in range(hi + 1)], default=0)


def test_peak_width_equals_brute_force():
    cases = [([0, 3], [2, 5]),                      # the second starts on the frame after the first ends
             ([0, 2], [2, 5]),                      # ... or on its last frame
             ([4], [4]), ([0, 4, 4], [9, 4, 6]),    # start == end
             ([0, 0, 0], [0, 0, 0]), ([], [])]
    rng = np.random.RandomState(2)
    for _ in range(200):
        n = rng.randint(1, 8)
        s = rng.randint(0, 20, size=n)
        cases.append((list(s), list(s + rng.randint(0, 8, size=n))))
    for s, e in cases:
        assert peak_width(s, e) == _brute_peak(s, e), (s, e)
    assert peak_width([0, 3], [2, 5]) == 1 and peak_width([0, 2], [2, 5]) == 2


class _Net:
    max_batch, num_slots = 4, 6


class _HostTracker:
    """Just enough of BatchTracker for what VideoSegmenter does before any device work."""
    dev = torch.device("cpu")
    net, slot0, p = _Net(), 0, None

    def _clear(self):
        pass


def _segmenter():
    seg = VideoSegmenter.__new__(VideoSegmenter)
    seg.tracker, seg.p, seg.dev, seg.objects, seg.score, seg._sched = _HostTracker(), None, torch.device("cpu"), [], \
        None, None
    return seg


OBJS = [(0, 1, 0), (0, 2, 3, 5), (1, 7, 2, 4), (1, 3, 0, 1), (2, 1, 0)]
T = [8, 6, 3]


def _all_wants(seg):
    return {(g, t): seg._wants_anno(g, t) for g in range(len(T)) for t in range(T[g])}


def test_needs_anno_follows_starts_and_windows():
    seg = _segmenter()
    seg.open_queue(OBJS, T)
    assert seg.needed() == [(0, 0), (1, 0), (2, 0)] and seg.needs_anno() == [True, True, True]
    starts = {(0, 0), (0, 3), (1, 2), (1, 0), (2, 0)}
    assert {k for k, v in _all_wants(seg).items() if v} == starts
    seg.open_queue(OBJS, T, score="whole")
    whole = {(g, t) for g in range(3) for t in range(1, T[g] - 1)}
    assert {k for k, v in _all_wants(seg).items() if v} == starts | whole
    seg.open_queue(OBJS, T, score="spans")
    # windows [start + 1, end - 1): video 0 [1, 6), [4, 4); video 1 [3, 3), [1, 0); video 2 [1, 1)
    spans = {(0, t) for t in range(1, 6)}
    assert {k for k, v in _all_wants(seg).items() if v} == starts | spans
    # needs_anno() of every step of the plan follows the same rule
    while seg._plan is not None:
        assert seg.needs_anno() == [_all_wants(seg)[gt] for gt in seg.needed()]
        seg._plan = seg._sched.step() if not seg._sched.done else None


def test_open_queue_checks():
    seg = _segmenter()
    for num_frames in ([], [3, 0], [2.0, 3]):
        with pytest.raises(ValueError, match="num_frames"):
            seg.open_queue([(0, 1, 0)], num_frames)
    with pytest.raises(ValueError, match="score"):
        seg.open_queue([(0, 1, 0)], [3], score="all")
    for o in ((1, 1, 0), (-1, 1, 0), (0, 256, 0), (0, 1)):
        with pytest.raises(ValueError, match="object entry"):
            seg.open_queue([o], [3])
    for o in ((0, 1, 3), (0, 1, 2, 3), (0, 1, 2, 1), (0, 1, -1, 1)):
        with pytest.raises(ValueError, match="start_frame"):
            seg.open_queue([o], [3])
    with pytest.raises(ValueError, match="no object"):
        seg.open_queue([(0, 1, 0)], [3, 4])
    with pytest.raises(ValueError, match="255"):
        seg.open_queue([(0, i % 200 + 1, 0, 0) for i in range(256)], [3])
    # five objects at once in video 1: wider than the engine's 4
    with pytest.raises(ValueError, match="slots"):
        seg.open_queue([(0, 1, 0)] + [(1, i + 1, 1, 2) for i in range(5)], [3, 4])
    seg.open_queue([(0, 1, 0)] + [(1, i + 1, i, i) for i in range(5)], [3, 5])       # one at a time: width 1
    with pytest.raises(ValueError, match="unique"):
        seg.open_queue([(0, 1, 0), (0, 1, 1)], [4], score="spans")
    seg.open_queue([(0, 1, 0), (0, 1, 1)], [4], score="whole")                       # positional ids 1, 2
    with pytest.raises(ValueError, match="thresholds"):
        seg.open_queue([(0, 1, 0)], [4], score="whole", thrs=np.linspace(0, 1, 40))


def test_step_checks_before_device_work():
    seg = _segmenter()
    seg.open_queue(OBJS, T, score="whole")
    need = seg.needed()
    fr = [np.zeros((4, 4, 3), np.uint8) for _ in need]
    an = [np.zeros((4, 4), np.uint8) for _ in need]
    with pytest.raises(ValueError, match="frames"):
        seg.step(fr[:-1], an)                                   # one frame short
    with pytest.raises(ValueError, match="annos"):
        seg.step(fr, an[:-1])
    with pytest.raises(ValueError, match="required"):
        seg.step(fr, [an[0], None, an[2]])                      # an object of video 1 starts at frame 0
    with pytest.raises(ValueError, match="uint8"):
        seg.step(fr, [an[0], an[1].astype(np.int32), an[2]])
    with pytest.raises(ValueError, match="uint8"):
        seg.step(fr, [an[0], an[1][:3], an[2]])                 # not the frame's size
    with pytest.raises(ValueError, match="frame"):
        seg.step([fr[0], fr[1][..., :2], fr[2]], an)
    with pytest.raises(ValueError, match="frame"):
        seg.frame(np.stack(fr), np.stack(an))                   # frame() belongs to open()
    # a later frame must have its video's frame-0 size
    seg._hw = [(4, 4), (4, 4), (4, 4)]
    seg._plan = seg._sched.step()
    need = seg.needed()
    fr = [np.zeros((4, 4, 3), np.uint8) for _ in need]
    fr[1] = np.zeros((5, 4, 3), np.uint8)
    with pytest.raises(ValueError, match="frame 0"):
        seg.step(fr, [np.zeros((4, 4), np.uint8) for _ in need])
    with pytest.raises(ValueError, match="score"):
        _segmenter().open_queue(OBJS, T).result()
