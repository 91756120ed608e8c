import os
import sys
import warnings

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
warnings.filterwarnings("ignore", category=UserWarning)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90a) device")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def max_rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """The parity metric (SURVEY §7): max|a-b| / max|b| per tensor."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def assert_close(a, b, tol, what=""):
    err = max_rel(a, b)
    print(f"[parity] {what:32s} max|a-b|/max|b| = {err:.3e} (tol {tol:g})")
    assert tuple(a.shape) == tuple(b.shape), f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    assert err <= tol, f"{what}: {err:.3e} > {tol:g}"
    # and element-wise: rtol = tol, atol = tol * max|b|
    bb = b.detach().double().cpu()
    assert torch.allclose(a.detach().double().cpu(), bb, rtol=tol, atol=tol * float(bb.abs().max()))


@pytest.fixture(scope="session")
def calib_sd():
    from oracle.calibrate import calibrated_state_dict
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    return calibrated_state_dict(0)
