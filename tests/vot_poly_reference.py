"""TEST INFRASTRUCTURE ONLY (checker) for `VotScore` with polygon entries (C ABI `sm_vot_trajectory_overlap_poly`):
pysot's calculate_accuracy over a read-back trajectory whose locations are 8-value lines, which load_tracker reads and
vot_overlap builds as a Polygon of C floats.  Read-back (`vot_eval_reference.read_back`), failures and the aggregate
figures are those of tests/vot_eval_reference.py; only the per-frame overlap differs from its 4-value form."""
from __future__ import annotations

import numpy as np

import vot_reference


def trajectory_overlaps(traj, gt, W: int, H: int, burnin: int = 0) -> np.ndarray:
    """calculate_accuracy(traj, gt, burnin, bound=(W, H))[1] as float32 [T] for read-back entries of 1 or 8 values: the
    burn-in turns the `burnin` entries from every init entry into [0]; a 1-value entry is NaN (0x7FC00000), an
    8-value entry the overlap of its polygon (as C floats) with the gt."""
    traj = list(traj)
    if burnin:
        for i in [i for i, x in enumerate(traj) if len(x) == 1 and x[0] == 1]:
            for j in range(i, min(i + burnin, len(traj))):
                traj[j] = [0]
    out = np.full(min(len(traj), len(gt)), np.nan, np.float32)
    for f in range(len(out)):
        if len(traj[f]) == 8:
            out[f] = vot_reference.polygon_overlap(np.asarray(traj[f], np.float32), gt[f], W, H)
    return out
