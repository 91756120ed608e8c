"""The batched device-resident tracker (siammask_b200/tracker.py, C ABI sm_tracker_prepare / sm_tracker_update) against
(i) single-stream runs of the host restatement of the reference loop (oracle/ref_loop.py, numpy float64 selection and
state update exactly as tools/test.py does them) driven by the same engine, and (ii) the golden trajectory that the
reference's OWN siamese_init / siamese_track produced (oracle/make_golden.py::tracker_loop_golden)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import siammask_b200 as smb
from siammask_b200.tracker import BatchTracker, TrackerParams
from oracle import ref_loop
from oracle.synthetic_video import make_frames

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}


class _NoSelect:
    """The engine behind the reference's plain model API only (no `select`): ref_loop then runs the numpy float64
    post-processing of tools/test.py:205-254 on the engine's cls / loc."""
    def __init__(self, net):
        self._n = net
        self.anchors, self.anchor_num = net.anchors, net.anchor_num

    def template(self, z):
        return self._n.template(z)

    def track_mask(self, x):
        return self._n.track_mask(x)

    def track(self, x):
        return self._n.track(x)

    def track_refine(self, pos):
        return self._n.track_refine(pos)


def _videos(n):
    vids = [make_frames(seed=s) for s in range(n)]
    frames = [np.stack([v[0][t] for v in vids], 0) for t in range(len(vids[0][0]))]       # per time step: [N,H,W,3]
    boxes = np.array([v[1][0] for v in vids], dtype=np.float64)
    return vids, frames, boxes


def test_batched_tracker_equals_single_stream_reference_loops(calib_sd):
    N = 4
    vids, frames, boxes = _videos(N)
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=N).load_state_dict(calib_sd).eval().to("cuda")
    bt = BatchTracker(net, TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                                         window_influence=HP["window_influence"], lr=HP["lr"]))
    bt.init(frames[0], boxes)
    got = []
    for f in frames[1:]:
        r = bt.track(f, mask=True, refine=True)
        c = r.cpu()
        c["mask"] = r.mask.cpu().numpy()
        got.append(c)
    # single-stream runs of the reference-loop restatement with the same engine, device crop and device paste-back
    single = smb.Custom(anchors=smb.DEFAULT_ANCHORS).load_state_dict(calib_sd).eval().to("cuda")
    for b in range(N):
        fs, bx = vids[b]
        fdev = [torch.from_numpy(f).cuda() for f in fs]
        x, y, w, h = bx[0]
        st = ref_loop.siamese_init(fdev[0], np.array([x + w / 2, y + h / 2]), np.array([w, h]), _NoSelect(single), HP,
                                   device="cuda")
        for t, f in enumerate(fdev[1:]):
            st = ref_loop.siamese_track(st, f, mask_enable=True, refine_enable=True, device="cuda", device_paste=True)
            np.testing.assert_allclose(got[t]["target_pos"][b], st["target_pos"], rtol=0, atol=1e-5)
            # w, h pass through exp(): the device evaluates numpy's float32 exp algorithm (simt_kernels.cu np_expf)
            np.testing.assert_allclose(got[t]["target_sz"][b], st["target_sz"], rtol=1e-6, atol=0)
            assert abs(got[t]["score"][b] - st["score"]) < 1e-6 and got[t]["best_id"][b] == st["best_id"]
            ref_mask = (st["mask"] > HP["seg_thr"]).cpu().numpy() if torch.is_tensor(st["mask"]) else st["mask"] > HP["seg_thr"]
            assert (got[t]["mask"][b] != ref_mask).mean() < 1e-3, f"stream {b} frame {t}: pasted masks differ"


def test_batched_tracker_follows_reference_loop_golden(calib_sd):
    """Stream 0 of a batch is the synthetic video of the golden file: trajectory within the engine's network tolerance."""
    g = np.load(os.path.join(GOLDEN, "tracker_loop.npz"))
    N = 3
    vids, frames, boxes = _videos(N)
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=N, num_slots=N + 2).load_state_dict(calib_sd).eval().to("cuda")
    bt = BatchTracker(net, TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                                         window_influence=HP["window_influence"], lr=HP["lr"]), slot0=2)
    bt.init(frames[0], boxes)
    pos, sz, score, area = [], [], [], []
    for f in frames[1:]:
        r = bt.track(f)
        c = r.cpu()
        pos.append(c["target_pos"][0]); sz.append(c["target_sz"][0]); score.append(c["score"][0])
        area.append(float(r.mask[0].sum()))
    np.testing.assert_allclose(np.array(pos), g["pos"], rtol=0, atol=0.1)
    np.testing.assert_allclose(np.array(sz), g["sz"], rtol=0, atol=0.1)
    np.testing.assert_allclose(np.array(score), g["score"], rtol=0, atol=2e-3)
    assert np.all(np.abs(np.array(area) - g["mask_area"]) <= 0.02 * g["mask_area"] + 30)


def test_tracker_state_kernels_match_numpy():
    """sm_tracker_prepare / sm_tracker_update against the reference arithmetic written out in numpy float64."""
    import ctypes as C
    from siammask_b200 import _lib
    lib = _lib.load()
    rng = np.random.RandomState(0)
    B = 37
    state = np.stack([rng.rand(B) * 300, rng.rand(B) * 200, rng.rand(B) * 80 + 12, rng.rand(B) * 80 + 12], 1)
    avg = rng.randint(0, 256, (B, 3)).astype(np.int32)
    hp = _lib.SmTrackerHp(0.5, 0.04, 0.4, 0.9, 127, 255, 8, 8, 127, 0)
    sd, ad = torch.from_numpy(state).cuda(), torch.from_numpy(avg).cuda()
    boxes = torch.zeros(B, 8, dtype=torch.int32, device="cuda")
    tsz = torch.zeros(B, 2, dtype=torch.float64, device="cuda")
    aux = torch.zeros(B, 4, dtype=torch.float64, device="cuda")
    _lib.check(lib.sm_tracker_prepare(B, sd.data_ptr(), ad.data_ptr(), C.byref(hp), boxes.data_ptr(), tsz.data_ptr(),
                                      aux.data_ptr(), None))
    torch.cuda.synchronize()
    for b in range(B):
        px, py, sw, sh = state[b]
        wc_x = sh + 0.5 * (sw + sh); hc_x = sw + 0.5 * (sw + sh)
        s_x = np.sqrt(wc_x * hc_x); scale_x = 127 / s_x
        s_x = s_x + 2 * ((255 - 127) / 2 / scale_x)
        want = ref_loop.subwindow_box([px, py], round(s_x), avg[b].astype(np.float64))
        assert boxes[b, :6].tolist() == want
        np.testing.assert_allclose(tsz[b].cpu().numpy(), np.array([sw, sh]) * scale_x, rtol=1e-14)
        np.testing.assert_allclose(aux[b].cpu().numpy(), [scale_x, round(s_x), px - round(s_x) / 2, py - round(s_x) / 2],
                                   rtol=1e-14)
    # update: winner records as sm_select writes them
    rec = np.zeros((B, 8), np.float32)
    rec[:, 0:2] = rng.randn(B, 2) * 20
    rec[:, 2:4] = rng.rand(B, 2) * 80 + 20
    rec[:, 4] = rng.rand(B)
    rec[:, 7] = rng.randint(0, 3125, B)
    im = np.array([[320, 240]] * B, np.int32)
    rd, imd = torch.from_numpy(rec).cuda(), torch.from_numpy(im).cuda()
    maps = torch.zeros(B, 6, dtype=torch.float64, device="cuda")
    out = torch.zeros(B, 8, dtype=torch.float64, device="cuda")
    _lib.check(lib.sm_tracker_update(B, sd.data_ptr(), rd.data_ptr(), aux.data_ptr(), imd.data_ptr(), C.byref(hp), 5, 25,
                                     maps.data_ptr(), out.data_ptr(), None))
    torch.cuda.synchronize()
    auxh = aux.cpu().numpy()
    for b in range(B):
        px, py, sw, sh = state[b]
        scale_x, sxr, cx0, cy0 = auxh[b]
        tszc = np.array([sw, sh]) * scale_x
        w, h = rec[b, 2], rec[b, 3]                      # float32, as the reference's delta array

        def szf(w_, h_):
            pad = (w_ + h_) * 0.5
            return np.sqrt((w_ + pad) * (h_ + pad))
        s_c = szf(w, h) / szf(tszc[0], tszc[1]); s_c = max(s_c, 1 / s_c)
        r_c = (tszc[0] / tszc[1]) / (w / h); r_c = max(r_c, 1 / r_c)
        pen = np.exp(-(r_c * s_c - 1) * 0.04)
        lr = pen * rec[b, 4] * 0.9
        pred = rec[b, :4].astype(np.float64) / scale_x
        res = [pred[0] + px, pred[1] + py, sw * (1 - lr) + pred[2] * lr, sh * (1 - lr) + pred[3] * lr]
        want = [max(0, min(320, res[0])), max(0, min(240, res[1])), max(10, min(320, res[2])), max(10, min(240, res[3]))]
        np.testing.assert_allclose(out[b, :4].cpu().numpy(), want, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sd[b].cpu().numpy(), want, rtol=1e-12, atol=1e-12)
        # crop_back mapping (tools/test.py:263-282)
        idx = int(rec[b, 7]); dy, dx = (idx % 625) // 25, idx % 25
        s = sxr / 255
        sub = [cx0 + (dx - 4) * 8 * s, cy0 + (dy - 4) * 8 * s, s * 127, s * 127]
        s2 = 127 / sub[2]
        back = [-sub[0] * s2, -sub[1] * s2, 320 * s2, 240 * s2]
        a_, b_ = (320 - 1) / back[2], (240 - 1) / back[3]
        np.testing.assert_allclose(maps[b].cpu().numpy(), [a_, 0, -a_ * back[0], 0, b_, -b_ * back[1]], rtol=1e-12, atol=1e-9)
