"""The queue scheduler of VotRunner.open_queue / ParamSweep.open_queue as a pure function of the lengths (no GPU):
admission order, frame lists, frame sharing, K > capacity, and the step counts of tools/bench_queue.py."""
import importlib.util
import os

import numpy as np
import pytest

from siammask_b200 import schedule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _replay(lengths, K, cap):
    """Runs the plan and checks every invariant a runner relies on; returns (steps, admission step per stream)."""
    T = np.asarray(lengths)
    steps = schedule.plan(T, K, cap)
    admit, left, active = {}, {}, set()
    for f, st in enumerate(steps):
        assert set(st.track) == active                         # exactly the streams admitted earlier and not gone
        assert len(st.need) == len(set(st.need))                # distinct (sequence, frame) pairs
        for s in st.admit:
            assert s not in admit
            admit[s] = f
        for s in st.track + st.admit:
            g, t = st.need[st.entry[s]]
            assert g == s // K and t == f - admit[s]            # each stream reads its own sequence's frame t
        assert {st.need[st.entry[s]] for s in st.track + st.admit} == set(st.need)
        assert len(active) + len(st.admit) <= cap
        for s in st.retire:
            assert f - admit[s] == T[s // K] - 1                # after its sequence's last frame
            left[s] = f
        active = (active | set(st.admit)) - set(st.retire)
        if f and st.admit:                                      # admitted into slots freed by the previous step
            assert len(st.admit) <= cap - len(st.track)
    assert not active and set(admit) == set(left) == set(range(T.size * K))
    return steps, admit


def test_admission_order_is_longest_sequence_first():
    T = [5, 9, 9, 3]
    s = schedule.Scheduler(T, 2, 3)
    assert s.order == [2, 3, 4, 5, 0, 1, 6, 7]                 # lengths 9 (index 1), 9 (2), 5, 3; combos in order
    steps, admit = _replay(T, 2, 3)
    assert steps[0].admit == [2, 3, 4]
    steps_in_order = [admit[x] for x in s.order]
    assert steps_in_order == sorted(steps_in_order)              # nobody overtakes a stream ahead of it


def test_need_lists_and_frame_sharing():
    steps, admit = _replay([4, 2], 2, 4)
    assert [st.need for st in steps] == [[(0, 0), (1, 0)], [(0, 1), (1, 1)], [(0, 2)], [(0, 3)]]
    assert steps[0].entry == {0: 0, 1: 0, 2: 1, 3: 1}          # streams of one sequence share an entry
    assert steps[1].retire == [2, 3] and steps[3].retire == [0, 1]


def test_k_above_capacity_spreads_one_sequence_over_admissions():
    steps, admit = _replay([6], 5, 2)
    assert [sorted(s for s in admit if admit[s] == f) for f in sorted(set(admit.values()))] == [[0, 1], [2, 3], [4]]
    assert sorted(set(admit.values())) == [0, 6, 12]
    # one group per admission step: the combinations admitted together share a frame entry, later ones get their own
    assert steps[6].need == [(0, 0)] and steps[12].need == [(0, 0)]


def test_refill_the_step_after_a_slot_frees():
    steps, admit = _replay([3, 10, 2, 8, 1, 4], 1, 2)
    # 10 and 8 start at 0; 8 ends at step 7, 4 enters at 8; 10 ends at 9, 3 at 10 ...
    assert admit[1] == admit[3] == 0 and admit[5] == 8 and admit[0] == 10 and admit[2] == 12
    assert admit[4] == 13 and steps[13].admit == [4] and 4 in steps[13].retire     # one frame: in and out at once


def test_random_plans_keep_the_invariants():
    rng = np.random.default_rng(3)
    for _ in range(20):
        T = rng.integers(1, 30, rng.integers(1, 12))
        _replay(T, int(rng.integers(1, 5)), int(rng.integers(1, 9)))


def test_scheduler_rejects_bad_arguments():
    for args in (([], 1, 1), ([3, 0], 1, 2), ([3.5], 1, 1), ([3], 0, 1), ([3], 1, 0)):
        with pytest.raises(ValueError):
            schedule.Scheduler(*args)
    s = schedule.Scheduler([1], 1, 1)
    s.step()
    assert s.done
    with pytest.raises(ValueError):
        s.step()
    with pytest.raises(ValueError):
        schedule.chunked_steps([3], 4, 2)


def test_bench_workload_queue_beats_the_chunks():
    spec = importlib.util.spec_from_file_location("bench_queue", os.path.join(ROOT, "tools", "bench_queue.py"))
    bq = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bq)
    L = bq.vot_lengths()
    assert (L.min(), L.max(), L.sum()) == (53, 1067, 20768)
    c = bq.counts(L, bq.K_VOT, bq.CAPACITY)
    assert c["chunked_steps"] == 3399
    assert c["queue_steps"] < c["chunked_steps"]
    assert c["queue_steps"] == len(schedule.plan(L, 16, 256))
    _replay(L, 16, 256)
