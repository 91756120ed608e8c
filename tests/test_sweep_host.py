"""Host logic of the hyper-parameter sweep (siammask_b200/tune.py) without a GPU: the grid order of tools/tune_vos.py,
the IouMeter.value('mean') restatement, and the host-side argument checks."""
import numpy as np
import pytest
import torch

import siammask_b200 as smb
from siammask_b200 import tune
from siammask_b200.ops import mask_iou
from sweep_reference import IouMeter


def test_grid_follows_tune_vos_nested_loops():
    pk, wi, lr = np.arange(0.0, 0.1, 0.03), np.arange(0.3, 0.5, 0.04), np.arange(0.8, 1.01, 0.05)
    want = []
    for penalty_k in pk:
        for window_influence in wi:
            for r in lr:
                want.append((penalty_k, window_influence, r))
    got = tune.grid()
    assert got.shape == (100, 3) and got.dtype == np.float64
    np.testing.assert_array_equal(got, np.array(want))
    np.testing.assert_array_equal(tune.grid([0.1], [0.2, 0.3], [0.9]), [[0.1, 0.2, 0.9], [0.1, 0.3, 0.9]])
    assert len(tune.THRESHOLDS) == 11


def _meter(rows):
    m = IouMeter(np.arange(0.3, 0.81, 0.05), rows.shape[0])
    m.iou[:] = rows
    return m.value_mean()


@pytest.mark.parametrize("case", ["dense", "zero_cells", "nb_below_rows", "all_zero", "nb_above_rows"])
def test_iou_mean_equals_iou_meter(case):
    rng = np.random.RandomState(len(case))
    rows = rng.rand(9, 11).astype(np.float32)
    if case == "zero_cells":
        rows[rng.rand(9, 11) < 0.4] = 0
    elif case == "nb_below_rows":
        rows[:] = 0
        rows[5, 3:7] = rng.rand(4)                       # 4 positive cells: the first 4 rows are averaged
    elif case == "all_zero":
        rows[:] = 0
    elif case == "nb_above_rows":
        rows[:, :2] = 0
    got = tune.iou_mean(rows)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, _meter(rows))
    nb = max(int((rows > 0).sum()), 1)
    np.testing.assert_allclose(got, rows[:nb].astype(np.float64).mean(0), rtol=1e-6)


def test_host_argument_checks():
    for bad in ([], [-1.01], [0.3, np.nan], np.linspace(0, 1, 33)):
        with pytest.raises(ValueError):
            tune._check_thresholds(bad)
    np.testing.assert_array_equal(tune._check_thresholds([-1.0, 0.5]), [-1.0, 0.5])
    cpu = torch.zeros(2, 127, 127)
    with pytest.raises(ValueError):                      # operators take CUDA tensors only
        mask_iou(cpu, torch.zeros(2, 6, dtype=torch.float64), torch.zeros(1, 8, 8, dtype=torch.uint8), [0, 0], [0.5])
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=2)
    with pytest.raises(ValueError):
        net._check_hp(torch.zeros(2, 3, dtype=torch.float64), 2)
