"""Parity at the shapes the benchmark actually runs (VERDICT r01 "missing 1"): the B=64 default tile /
two-lane path, the sharp path at search 383 (R=41), SiamRPN-only at B=256, and the fused frame entry points
`sm_step` / `sm_step_host_async`.  All against the CPU oracle / the reference goldens, tolerance 1e-3."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, assert_close
import siammask_b200 as smb
from siammask_b200 import _lib, anchors as anc
from oracle.calibrate import synthetic_inputs
from oracle.ref_loop import select_numpy
from oracle.siammask_oracle import Oracle

pytestmark = pytest.mark.gpu
TOL = 1e-3
PK, WI = 0.04, 0.4


def _engine(sd, **kw):
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, **kw)
    m.load_state_dict(sd)
    return m.eval().to("cuda")


def _consts(R, B, seed=3):
    a = anc.generate_anchor(smb.DEFAULT_ANCHORS, R)
    w = anc.cosine_window(R, 5)
    g = np.random.RandomState(seed)
    tsz = g.rand(B, 2) * 60 + 30
    return a, w, tsz


def _check_stream(o, out, b, z, x, a, w, tsz, sharp=True, mask_head=True):
    o.template(z[b:b + 1])
    if sharp:
        ocls, oloc, omask = o.track_mask(x[b:b + 1], with_mask_head=mask_head)
    else:
        ocls, oloc = o.track(x[b:b + 1])
    assert_close(out["cls"][b:b + 1], ocls, TOL, f"cls stream {b}")
    assert_close(out["loc"][b:b + 1], oloc, TOL, f"loc stream {b}")
    # the engine's selection on ITS cls/loc must be what the reference arithmetic (numpy, float64) selects on them
    bid, box, score, pen, ps = select_numpy(out["cls"][b:b + 1].cpu(), out["loc"][b:b + 1].cpu(), a, w, tsz[b], PK, WI)
    assert int(out["best"][b]) == bid and int(out["records"][b, 7]) == bid
    R = out["cls"].shape[-1]
    pos = tuple(int(v) for v in out["pos"][b].cpu())
    assert pos == tuple(int(v) for v in np.unravel_index(bid, (5, R, R))[1:])
    np.testing.assert_allclose(out["records"][b, :4].cpu().numpy(), box, rtol=2e-5, atol=1e-4)
    if sharp:
        assert_close(out["refine"][b:b + 1], o.track_refine(pos), TOL, f"refine stream {b} at {pos}")
        if mask_head:
            assert_close(out["mask"][b:b + 1], omask, TOL, f"mask head stream {b}")
            assert torch.equal(out["mask_col"][b], out["mask"][b, :, pos[0], pos[1]])


def test_b64_default_path_matches_oracle(calib_sd):
    """BASELINE configs[1] exactly as bench.py runs it: B=64, default env (the tiles the launcher
    picks, two lanes of 32), one `sm_step` per frame incl. the mask head; streams at both ends of both lanes."""
    B = 64
    z, x = synthetic_inputs(71, B)
    a, w, tsz = _consts(25, B)
    m = _engine(calib_sd, max_batch=B)
    m.template(z.cuda())
    out = m.step(x.cuda(), torch.from_numpy(a), torch.from_numpy(w.astype(np.float32)), torch.from_numpy(tsz), PK, WI,
                 refine=True, mask_head=True, mask_col=True)
    torch.cuda.synchronize()
    o = Oracle(calib_sd)
    for b in (0, 31, 32, 63):
        _check_stream(o, out, b, z, x, a, w, tsz)
    # the fused frame == the three separate calls (track_mask / select / track_refine), bit for bit
    cls, loc, mask = m.track_mask(x.cuda())
    best, pos, rec = m.select(cls, loc, torch.from_numpy(a), torch.from_numpy(w.astype(np.float32)),
                              torch.from_numpy(tsz), PK, WI)
    ref = m.track_refine(pos)
    for got, want, n in ((out["cls"], cls, "cls"), (out["loc"], loc, "loc"), (out["pos"], pos, "pos"),
                         (out["records"], rec, "records"), (out["refine"], ref, "refine")):
        assert torch.equal(got, want), n


def test_step_host_async_matches_device_step(calib_sd):
    """The host-buffer frame (bench.py's e2e) == the device-pointer frame, for two alternating stream groups."""
    B = 18                                   # two lanes (9 + 9)
    z, x = synthetic_inputs(72, 2 * B)
    a, w, tsz = _consts(25, 2 * B)
    m = _engine(calib_sd, max_batch=B, num_slots=2 * B)
    ad, wd = torch.from_numpy(a).cuda(), torch.from_numpy(w.astype(np.float32)).cuda()
    m.template(z[:B].cuda(), slot0=0)
    m.template(z[B:].cuda(), slot0=B)
    want = []
    for g in range(2):
        out = m.step(x[g * B:(g + 1) * B].cuda(), ad, wd, torch.from_numpy(tsz[g * B:(g + 1) * B]), PK, WI, slot0=g * B,
                     refine=True, mask_head=True, mask_col=True)
        want.append({k: v.cpu().clone() for k, v in out.items() if v is not None})
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bufs, tickets, keep = [], [], []
    for g in range(2):
        xh = x[g * B:(g + 1) * B].contiguous().pin_memory()
        th = torch.from_numpy(tsz[g * B:(g + 1) * B].copy()).pin_memory()
        o = {"records": torch.empty(B, 8).pin_memory(), "refine": torch.empty(B, 127 * 127).pin_memory(),
             "mask_col": torch.empty(B, 3969).pin_memory(), "cls": torch.empty(B, 10, 25, 25).pin_memory(),
             "loc": torch.empty(B, 20, 25, 25).pin_memory()}
        io = _lib.SmStepIO()
        io.x_host, io.tsz_host = xh.data_ptr(), th.data_ptr()
        io.anchors_dev, io.window_dev = ad.data_ptr(), wd.data_ptr()
        io.penalty_k, io.window_influence = PK, WI
        io.flags = _lib.SM_TRACK_MASK_FEATURES | _lib.SM_TRACK_MASK_HEAD
        io.records_host, io.refine_host, io.mask_col_host = o["records"].data_ptr(), o["refine"].data_ptr(), o["mask_col"].data_ptr()
        io.cls_host, io.loc_host = o["cls"].data_ptr(), o["loc"].data_ptr()
        tk = C.c_int32()
        _lib.check(lib.sm_step_host_async(m.handle, g * B, B, C.byref(io), st, C.byref(tk)))
        tickets.append(tk.value); bufs.append(o); keep.append((xh, th, io))
    for g in range(2):
        _lib.check(lib.sm_track_host_wait(m.handle, tickets[g]))
        for k, v in bufs[g].items():
            assert torch.equal(v, want[g][k]), f"group {g} {k}"
    # without refine / mask head (SiamRPN-style frame through the same entry point)
    io = _lib.SmStepIO()
    io.x_host, io.tsz_host = keep[0][0].data_ptr(), keep[0][1].data_ptr()
    io.anchors_dev, io.window_dev, io.penalty_k, io.window_influence, io.flags = ad.data_ptr(), wd.data_ptr(), PK, WI, 0
    rec = torch.empty(B, 8).pin_memory()
    io.records_host = rec.data_ptr()
    tk = C.c_int32()
    _lib.check(lib.sm_step_host_async(m.handle, 0, B, C.byref(io), st, C.byref(tk)))
    _lib.check(lib.sm_track_host_wait(m.handle, tk.value))
    assert torch.equal(rec, want[0]["records"])


def test_sharp_383_matches_oracle_and_golden(calib_sd):
    """BASELINE configs[4] geometry: search 383 -> 189/95/47-px pyramids, 45x45 search feature, 41x41 response
    (the 16-channel xcorr variant), refine positions up to 40."""
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLDEN, "sharp_b1_s383.npz")).items()}
    z, x = synthetic_inputs(3, 1, search=383)
    m = _engine(calib_sd, search_size=383)
    m.template(z.cuda())
    cls, loc, mask = m.track_mask(x.cuda())
    assert mask.shape == (1, 3969, 41, 41)
    o = Oracle(calib_sd)
    o.template(z)
    ocls, oloc, omask = o.track_mask(x)
    for i, name in enumerate(("p0", "p1", "p2", "p3")):
        assert_close(m.export(name), o.feature[i], TOL, name + " @383")
        assert_close(m.export(name).flatten().cpu()[::509], g[name], 2e-3, name + " @383 vs reference golden")
    assert_close(m.export("search"), o.search, TOL, "search feature @383")
    assert_close(m.export("corr_mask"), o.corr_feature, TOL, "mask corr feature @383")
    assert_close(cls, ocls, TOL, "cls @383")
    assert_close(loc, oloc, TOL, "loc @383")
    assert_close(mask, omask, TOL, "mask head @383")
    assert_close(mask[:, slice(0, 3969, 193)], g["mask_sub"], 2e-3, "mask head @383 vs reference golden")
    for pos in ((0, 0), (40, 40), (7, 33)):
        r = m.track_refine(pos)
        assert_close(r, o.track_refine(pos), TOL, f"refine {pos} @383")
        assert_close(r, g[f"refine_{pos[0]}_{pos[1]}"], 2e-3, f"refine {pos} @383 vs reference golden")
    with pytest.raises(IndexError):
        m.track_refine((41, 0))


def test_sharp_383_batched_lanes(calib_sd):
    """search 383 with a two-lane batch (the config the 1->8 GPU sweep runs per GPU, scaled down)."""
    B = 16
    z, x = synthetic_inputs(73, B, search=383)
    a, w, tsz = _consts(41, B)
    m = _engine(calib_sd, search_size=383, max_batch=B)
    m.template(z.cuda())
    out = m.step(x.cuda(), torch.from_numpy(a), torch.from_numpy(w.astype(np.float32)), torch.from_numpy(tsz), PK, WI,
                 refine=True, mask_head=False)
    torch.cuda.synchronize()
    o = Oracle(calib_sd)
    for b in (0, 7, 8, 15):
        _check_stream(o, out, b, z, x, a, w, tsz, mask_head=False)


def test_rpn_only_b256(calib_sd):
    """BASELINE configs[2]: SiamRPN-only engine at B=256 (two lanes of 128), sampled streams vs the oracle."""
    B = 256
    sd = {k: v for k, v in calib_sd.items() if not k.startswith(("mask_model", "refine_model"))}
    z, x = synthetic_inputs(74, B)
    a, w, tsz = _consts(25, B)
    m = _engine(sd, mask=False, max_batch=B)
    m.template(z.cuda())
    out = m.step(x.cuda(), torch.from_numpy(a), torch.from_numpy(w.astype(np.float32)), torch.from_numpy(tsz), PK, WI,
                 refine=False, mask_head=False)
    torch.cuda.synchronize()
    o = Oracle(calib_sd)
    for b in (0, 127, 128, 255):
        _check_stream(o, out, b, z, x, a, w, tsz, sharp=False)


def test_select_is_nan_safe(calib_sd):
    """np.argmax semantics with NaN scores: the first NaN wins, the indices stay in range (no out-of-bounds gather)."""
    m = _engine(calib_sd, max_batch=2)
    a, w, tsz = _consts(25, 2)
    cls = torch.randn(2, 10, 25, 25, device="cuda")
    loc = torch.randn(2, 20, 25, 25, device="cuda") * 0.1
    cls[0, 5 + 2, 7, 9] = float("nan")           # stream 0: one NaN score at (anchor 2, y 7, x 9)
    cls[1] = float("nan")                         # stream 1: everything NaN
    best, pos, rec = m.select(cls, loc, torch.from_numpy(a), torch.from_numpy(w.astype(np.float32)),
                              torch.from_numpy(tsz), PK, WI)
    assert int(best[0]) == 2 * 625 + 7 * 25 + 9 and tuple(pos[0].tolist()) == (7, 9)
    assert int(best[1]) == 0 and tuple(pos[1].tolist()) == (0, 0)
    z, x = synthetic_inputs(75, 2)
    m.template(z.cuda())
    m.track_mask(x.cuda(), mask_head=False)
    bad = torch.tensor([[-5, 99], [1000, -1]], dtype=torch.int32, device="cuda")
    r = m.track_refine(bad)                       # device positions are clamped to the response map, not trusted
    torch.cuda.synchronize()
    assert torch.isfinite(r).all()
    assert torch.equal(r, m.track_refine(torch.tensor([[0, 24], [24, 0]], dtype=torch.int32, device="cuda")))


def test_step_graph_replay_matches_eager(calib_sd):
    """`sm_step` under CUDA-graph replay (call 1 eager, call 2 captured, then replayed) == eager, fresh inputs honoured."""
    B = 2
    a, w, tsz = _consts(25, B)
    ad, wd = torch.from_numpy(a).cuda(), torch.from_numpy(w.astype(np.float32)).cuda()
    z, x1 = synthetic_inputs(76, B)
    _, x2 = synthetic_inputs(77, B)
    eager = _engine(calib_sd, max_batch=B)
    graph = _engine(calib_sd, max_batch=B, graphs=True)
    eager.template(z.cuda()); graph.template(z.cuda())
    for it, xin in enumerate([x1, x2, x1, x2]):
        t = torch.from_numpy(tsz + it)
        oe = eager.step(xin.cuda(), ad, wd, t, PK, WI, refine=True, mask_head=False)
        og = graph.step(xin.cuda(), ad, wd, t, PK, WI, refine=True, mask_head=False)
        for k in ("cls", "loc", "pos", "records", "refine"):
            assert torch.equal(oe[k], og[k]), f"call {it}: {k}"
