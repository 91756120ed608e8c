"""TEST INFRASTRUCTURE ONLY (checker) for `siammask_b200.VotScore` (C ABI `sm_vot_trajectory_overlap`,
`sm_vot_eao_accumulate`).  Nothing under `siammask_b200/` imports this module.

A numpy restatement of what tools/eval.py computes for VOT with pysot ('all' tag): `read_back` is load_tracker reading a
result file written by track_vot, `trajectory_overlaps` is calculate_accuracy (pyvotkit's vot_overlap through the
polygon restatement of tests/vot_reference.py), `accuracy_robustness` the figures AccuracyRobustnessBenchmark prints and
`expected_overlaps` / `eao` EAOBenchmark's fragments, curve and mean.  The curve's fragment means come from cumulative
sums (pysot re-sums every prefix), so entries may differ from pysot's in the last float32 bit.
"""
from __future__ import annotations

import numpy as np

import vot_reference

BURNIN, SKIPPING = 10, 5


def result_value(v) -> float:
    """float("%.4f" % float32(v)): one location value written to and read back from a result file."""
    return float("%.4f" % float(np.float32(v)))


def read_back(regions) -> list:
    """load_tracker's list of float lists for the regions write_result writes."""
    return [[float(x)] if isinstance(x, (int, np.integer)) else [result_value(v) for v in x] for x in regions]


def trajectory_overlaps(traj, gt, W: int, H: int, burnin: int = 0) -> np.ndarray:
    """calculate_accuracy(traj, gt, burnin, bound=(W, H))[1] as float32 [T]: a 1-element entry is NaN (0x7FC00000)."""
    traj = list(traj)
    if burnin:
        for i in [i for i, x in enumerate(traj) if len(x) == 1 and x[0] == 1]:
            for j in range(i, min(i + burnin, len(traj))):
                traj[j] = [0]
    out = np.full(min(len(traj), len(gt)), np.nan, np.float32)
    for f in range(len(out)):
        x = traj[f]
        if len(x) == 4:
            rect = [x[0], x[1], x[0] + x[2], x[1], x[0] + x[2], x[1] + x[3], x[0], x[1] + x[3]]
            out[f] = vot_reference.polygon_overlap(rect, gt[f], W, H)
    return out


def failures(traj) -> list:
    return [i for i, x in enumerate(traj) if len(x) == 1 and x[0] == 2]


def accuracy_robustness(acc_overlaps, lost_counts):
    """(accuracy, robustness, lost_number) over the sequences' burn-in overlaps and lost counts."""
    ov = np.concatenate([np.asarray(o, np.float64) for o in acc_overlaps])
    with np.errstate(invalid="ignore"):
        acc = np.nanmean(ov) if np.isfinite(ov).any() else np.nan
    n = int(np.sum(lost_counts))
    return acc, n / len(ov) * 100, n


def expected_overlaps(eao_overlaps, fails, max_len: int) -> np.ndarray:
    """EAOBenchmark's fragments of each sequence (its EAO overlaps and failure frames) and calculate_expected_overlap's
    float32 curve of length max_len."""
    frags, weights = [], []
    for ov, fl in zip(eao_overlaps, fails):
        ov = np.asarray(ov, np.float64)
        T = len(ov)
        if not fl:
            row = np.full(max_len, np.nan)
            row[:T] = ov
            frags.append(row)
            weights.append(1.0)
            continue
        points = [0] + [f + SKIPPING for f in fl if f + SKIPPING <= T]
        for i, p in enumerate(points):
            last = i == len(points) - 1
            frag = np.nan_to_num(ov[p:] if last else ov[p:points[i + 1] + 1], nan=0.0)
            row = np.full(max_len, np.nan) if last else np.zeros(max_len)
            row[:len(frag)] = frag
            frags.append(row)
            weights.append(len(frag) / (T - p + 1e-16) if last else len(frag) / (points[i + 1] - p + 1))
    F = np.asarray(frags)
    w = np.asarray(weights)[:, None]
    alive = ~np.isnan(F[:, 1:])
    mean = np.cumsum(F[:, 1:], axis=1) / np.arange(1, max_len)
    with np.errstate(invalid="ignore"):
        num = np.where(alive, mean * w, 0.0).sum(0)
        den = np.where(alive, w, 0.0).sum(0)
        curve = np.zeros(max_len, np.float32)
        curve[0] = 1
        curve[1:] = np.where(alive.any(0), num / np.where(den > 0, den, 1), 0.0)
    return curve


def eao(curve, low: int, high: int) -> float:
    seg = np.asarray(curve, np.float64)[low - 1:high]
    valid = ~np.isnan(seg)
    with np.errstate(invalid="ignore", divide="ignore"):
        return seg[valid].sum() / valid.sum()
