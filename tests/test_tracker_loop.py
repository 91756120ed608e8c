"""The tracker loop around the hot path (SURVEY §8f): the host restatement of the reference loop (oracle/ref_loop.py)
against the golden trajectory produced by the reference's OWN loop (tools/test.py siamese_init/siamese_track,
oracle/make_golden.py::tracker_loop_golden), first driven by the CPU oracle network (tight), then — on the GPU —
by the CUDA engine with the on-device score/box post-processing `sm_select` (network parity tolerance)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.siammask_oracle import Oracle
from oracle.synthetic_video import make_frames
from oracle import ref_loop as tracker

HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}


def _run(net, device):
    frames, boxes = make_frames()
    x, y, w, h = boxes[0]
    state = tracker.siamese_init(frames[0], np.array([x + w / 2, y + h / 2]), np.array([w, h]), net, HP, device=device)
    out = {"pos": [], "sz": [], "score": [], "mask_area": [], "polygon": [], "best": []}
    for f in frames[1:]:
        state = tracker.siamese_track(state, f, mask_enable=True, refine_enable=True, device=device)
        out["pos"].append(state["target_pos"].copy())
        out["sz"].append(state["target_sz"].copy())
        out["score"].append(state["score"])
        out["mask_area"].append(float((state["mask"] > HP["seg_thr"]).sum()))
        out["polygon"].append(np.asarray(state["ploygon"], dtype=np.float64))
        out["best"].append(state["best_id"])
    return {k: np.asarray(v) for k, v in out.items()}


def test_generate_anchor_layout():
    from siammask_b200 import anchors
    cfg = {"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8], "round_dight": 0}
    for R in (25, 41):       # the product's table == the restatement of tools/test.py:113-129
        assert np.array_equal(anchors.generate_anchor(cfg, R), tracker.generate_anchor(cfg, R))
    assert np.array_equal(anchors.cosine_window(25, 5), np.tile(np.outer(np.hanning(25), np.hanning(25)).flatten(), 5))
    a = anchors.generate_anchor({"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8], "round_dight": 0}, 25)
    assert a.shape == (5 * 25 * 25, 4) and a.dtype == np.float32
    # order (anchor, y, x); centres on a stride-8 grid centred at 0; sizes from int(sqrt(64/r)) * 8
    assert tuple(a[0]) == (-96.0, -96.0, 104.0, 32.0)
    assert tuple(a[1][:2]) == (-88.0, -96.0) and tuple(a[25][:2]) == (-96.0, -88.0)
    assert tuple(a[2 * 625][2:]) == (64.0, 64.0)


def test_host_loop_matches_reference_loop_golden(calib_sd):
    g = np.load(os.path.join(GOLDEN, "tracker_loop.npz"))
    out = _run(Oracle(calib_sd), "cpu")
    # same network (oracle), same arithmetic: differences only from CPU conv kernels of the regenerated checkpoint
    np.testing.assert_allclose(out["pos"], g["pos"], rtol=0, atol=2e-2)
    np.testing.assert_allclose(out["sz"], g["sz"], rtol=0, atol=2e-2)
    np.testing.assert_allclose(out["score"], g["score"], rtol=0, atol=1e-3)
    assert np.all(np.abs(out["mask_area"] - g["mask_area"]) <= 0.01 * g["mask_area"] + 20)


@pytest.mark.gpu
def test_device_select_matches_numpy(calib_sd):
    import siammask_b200 as smb
    from oracle.calibrate import synthetic_inputs
    z, x = synthetic_inputs(31, 3)
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=3).load_state_dict(calib_sd).eval().to("cuda")
    m.template(z.cuda())
    cls, loc, _ = m.track_mask(x.cuda(), mask_head=False)
    anchor = tracker.generate_anchor(smb.DEFAULT_ANCHORS, 25)
    window = np.tile(np.outer(np.hanning(25), np.hanning(25)).flatten(), 5)
    tsz = np.array([[60.0, 40.0], [35.5, 80.25], [100.0, 100.0]])
    best, pos, rec = m.select(cls, loc, torch.from_numpy(anchor), torch.from_numpy(window),
                              torch.from_numpy(tsz), 0.04, 0.4)
    best, pos, rec = best.cpu().numpy(), pos.cpu().numpy(), rec.cpu().numpy()
    for b in range(3):
        bid, box, score, pen, ps = tracker.select_numpy(cls[b:b + 1].cpu(), loc[b:b + 1].cpu(), anchor, window, tsz[b],
                                                        0.04, 0.4)
        assert best[b] == bid and int(rec[b, 7]) == bid
        assert tuple(pos[b]) == tuple(np.unravel_index(bid, (5, 25, 25))[1:])
        np.testing.assert_allclose(rec[b, :4], box, rtol=2e-5, atol=1e-4)
        np.testing.assert_allclose(rec[b, 4:7], [score, pen, ps], rtol=2e-5, atol=1e-6)


@pytest.mark.gpu
def test_engine_loop_matches_reference_loop_golden(calib_sd):
    import siammask_b200 as smb
    g = np.load(os.path.join(GOLDEN, "tracker_loop.npz"))
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS).load_state_dict(calib_sd).eval().to("cuda")
    out = _run(m, "cuda")
    print("[loop] max |pos - ref| =", np.abs(out["pos"] - g["pos"]).max(), "px; max |score - ref| =",
          np.abs(out["score"] - g["score"]).max())
    np.testing.assert_allclose(out["pos"], g["pos"], rtol=0, atol=0.1)
    np.testing.assert_allclose(out["sz"], g["sz"], rtol=0, atol=0.1)
    np.testing.assert_allclose(out["score"], g["score"], rtol=0, atol=2e-3)
    assert np.all(np.abs(out["mask_area"] - g["mask_area"]) <= 0.02 * g["mask_area"] + 30)
