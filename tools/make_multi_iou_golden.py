"""Generates tests/golden/multi_iou.npz by running the reference's own, unmodified `MultiBatchIouMeter`
(tools/test.py:421-456) on seeded inputs.  TEST INFRASTRUCTURE ONLY; it needs the reference source tree
(SIAMMASK_REFERENCE, imported read-only through the shims of `oracle.make_golden.reference_loop_functions`):

    python tools/make_multi_iou_golden.py

Two cases, one per branch of the meter:
  whole: no start / end dicts.  Three objects tracked with the non-consecutive annotation ids 2, 5 and 7, which the
         meter compares against the positional ids 1, 2, 3; -1 idle stretches, ties (values on a 1/8 grid), NaN values,
         and test.py's thresholds.
  spans: start / end dicts in a non-sorted key order, one object whose window is empty (NaN row), six thresholds
         including -1 and values that occur in the outputs.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "multi_iou.npz")


def _outputs(rng, K, F, H, W):
    out = rng.randint(-8, 9, (K, F, H, W)).astype(np.float64) / 8.0     # [-1, 1] on a 1/8 grid: many ties
    out[0, 3:5] = -1.0                                                  # idle stretches
    out[-1, :2] = -1.0
    out[1, 2, rng.rand(H, W) < 0.05] = np.nan
    return out


def _targets(rng, ids, F, H, W):
    t = np.zeros((F, H, W), np.uint8)
    for f in range(F):
        for i in ids:
            x, y = rng.randint(0, W - 8), rng.randint(0, H - 6)
            t[f, y:y + rng.randint(3, 12), x:x + rng.randint(4, 16)] = i
    return t


def main():
    from oracle.make_golden import reference_loop_functions
    reference_loop_functions()                                          # shims; imports tools.test from the reference
    from tools.test import MultiBatchIouMeter, thrs                     # noqa: the reference's own meter
    warnings.filterwarnings("ignore")                                   # np.mean of an empty window
    rng = np.random.RandomState(20)
    F, H, W = 7, 24, 32
    whole_out = _outputs(rng, 3, F, H, W)
    whole_tgt = _targets(rng, (2, 5, 7), F, H, W)
    whole_tgt[4] = 0                                                    # a frame without targets
    whole_thrs = np.asarray(thrs, np.float64)
    whole_res = MultiBatchIouMeter(whole_thrs, whole_out, whole_tgt)

    spans_out = _outputs(rng, 4, F, H, W)
    spans_tgt = _targets(rng, (3, 1, 6, 9), F, H, W)
    start = {"3": 0, "1": 1, "6": 2, "9": 4}                            # dict order = object order
    end = {"3": 6, "1": 5, "6": 6, "9": 5}                              # id 9: range(5, 4) is empty -> NaN
    spans_thrs = np.array([-1.0, 0.0, 0.25, 0.3, 0.5, 0.75])
    spans_res = MultiBatchIouMeter(spans_thrs, spans_out, spans_tgt, start=start, end=end)

    np.savez_compressed(OUT, whole_outputs=whole_out, whole_targets=whole_tgt, whole_thrs=whole_thrs,
                        whole_res=whole_res, spans_outputs=spans_out, spans_targets=spans_tgt, spans_thrs=spans_thrs,
                        spans_ids=np.array([int(k) for k in start]), spans_start=np.array(list(start.values())),
                        spans_end=np.array([end[k] for k in start]), spans_res=spans_res)
    print(OUT, os.path.getsize(OUT))
    print("whole", whole_res)
    print("spans", spans_res)


if __name__ == "__main__":
    main()
