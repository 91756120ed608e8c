"""Entry-point combinations that share the engine's lane dispatch and host staging: the host-buffer calls on a
graph-replay engine (one and two lanes, both staging sets seen, captured and replayed), the launch count of one
frame through every frame entry point, and the per-lane cached tensors after a decoupled host-buffer frame."""
import ctypes as C

import numpy as np
import pytest
import torch

import siammask_b200 as smb
from siammask_b200 import _lib, anchors as anc
from oracle.calibrate import synthetic_inputs

pytestmark = pytest.mark.gpu
PK, WI = 0.04, 0.4
R = 25
STEP_FLAGS = _lib.SM_TRACK_MASK_FEATURES | _lib.SM_TRACK_MASK_HEAD


def _engine(sd, **kw):
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, **kw)
    m.load_state_dict(sd)
    return m.eval().to("cuda")


def _consts(B, seed=5):
    a = torch.from_numpy(anc.generate_anchor(smb.DEFAULT_ANCHORS, R)).float().cuda()
    w = torch.from_numpy(anc.cosine_window(R, 5).astype(np.float32)).cuda()
    tsz = np.random.RandomState(seed).rand(B, 2) * 60 + 30
    return a, w, tsz


def _host_step(lib, m, st, B, xh, th, a, w):
    """Submits one sm_step_host_async frame (refine, mask head, mask column, cls, loc); returns (ticket, outputs)."""
    o = {"records": torch.empty(B, 8).pin_memory(), "refine": torch.empty(B, 127 * 127).pin_memory(),
         "mask_col": torch.empty(B, 3969).pin_memory(), "cls": torch.empty(B, 10, R, R).pin_memory(),
         "loc": torch.empty(B, 20, R, R).pin_memory()}
    io = _lib.SmStepIO()
    io.x_host, io.tsz_host = xh.data_ptr(), th.data_ptr()
    io.anchors_dev, io.window_dev = a.data_ptr(), w.data_ptr()
    io.penalty_k, io.window_influence, io.flags = PK, WI, STEP_FLAGS
    io.records_host, io.refine_host, io.mask_col_host = o["records"].data_ptr(), o["refine"].data_ptr(), o["mask_col"].data_ptr()
    io.cls_host, io.loc_host = o["cls"].data_ptr(), o["loc"].data_ptr()
    tk = C.c_int32()
    _lib.check(lib.sm_step_host_async(m.handle, 0, B, C.byref(io), st, C.byref(tk)))
    return tk.value, o


def _device_step(m, x, a, w, tsz):
    return m.step(x.cuda(), a, w, torch.from_numpy(tsz), PK, WI, refine=True, mask_head=True, mask_col=True)


@pytest.mark.parametrize("B", [2, 17])
def test_track_host_async_on_graph_engine(calib_sd, B):
    """B=2 (one lane) and B=17 (two lanes, joined: graphs keep the host path coupled): six calls alternate the two
    staging sets, so each set's track and refine are run eagerly, captured and replayed."""
    lib = _lib.load()
    z, x = synthetic_inputs(81, B)
    _, x2 = synthetic_inputs(82, B)
    pos = torch.tensor([[(5 * b) % R, (3 * b + 4) % R] for b in range(B)], dtype=torch.int32)
    eager = _engine(calib_sd, max_batch=B, num_slots=B)
    eager.template(z.cuda())
    want = []
    for xin in (x, x2):
        cls, loc, _ = eager.track_mask(xin.cuda(), mask_head=False)
        want.append((cls.cpu(), loc.cpu(), eager.track_refine(pos.cuda()).cpu()))
    g = _engine(calib_sd, max_batch=B, num_slots=B, graphs=True)
    g.template(z.cuda())
    torch.cuda.synchronize()
    st = g._stream()
    xs = [x.contiguous().pin_memory(), x2.contiguous().pin_memory()]
    posh = pos.contiguous().pin_memory()
    for rnd in range(3):
        tickets, outs = [], []
        for i in range(2):
            o = (torch.empty(B, 10, R, R).pin_memory(), torch.empty(B, 20, R, R).pin_memory(),
                 torch.empty(B, 127 * 127).pin_memory())
            tk = C.c_int32()
            _lib.check(lib.sm_track_host_async(g.handle, 0, B, xs[i].data_ptr(), o[0].data_ptr(), o[1].data_ptr(),
                                               posh.data_ptr(), o[2].data_ptr(), st, C.byref(tk)))
            tickets.append(tk.value)
            outs.append(o)
        for i in range(2):
            _lib.check(lib.sm_track_host_wait(g.handle, tickets[i]))
            for got, ref, n in zip(outs[i], want[i], ("cls", "loc", "refine")):
                assert torch.equal(got, ref), f"B={B} round {rnd} input {i} {n}"


def test_step_host_async_on_graph_engine(calib_sd):
    """B=18 frames through sm_step_host_async on a graph-replay engine (coupled path, two joined lanes) == the eager
    device-pointer sm_step, over six calls (both staging sets eager, captured, replayed)."""
    B = 18
    lib = _lib.load()
    z, x = synthetic_inputs(83, B)
    _, x2 = synthetic_inputs(84, B)
    a, w, tsz = _consts(B)
    eager = _engine(calib_sd, max_batch=B)
    eager.template(z.cuda())
    want = []
    for xin in (x, x2):
        out = _device_step(eager, xin, a, w, tsz)
        want.append({k: v.cpu().clone() for k, v in out.items() if v is not None})
    g = _engine(calib_sd, max_batch=B, graphs=True)
    g.template(z.cuda())
    torch.cuda.synchronize()
    st = g._stream()
    xs = [x.contiguous().pin_memory(), x2.contiguous().pin_memory()]
    th = torch.from_numpy(tsz.copy()).pin_memory()
    for rnd in range(3):
        subs = [_host_step(lib, g, st, B, xs[i], th, a, w) for i in range(2)]
        for i, (tk, o) in enumerate(subs):
            _lib.check(lib.sm_track_host_wait(g.handle, tk))
            for k, v in o.items():
                assert torch.equal(v, want[i][k]), f"round {rnd} input {i} {k}"


def test_frame_launch_count_is_the_same_on_every_entry_point(calib_sd):
    """One B=18 frame adds the same launch count through sm_step eager, sm_step replayed from a graph and
    sm_step_host_async (decoupled lanes on the eager engine, coupled and replayed on the graph engine)."""
    B = 18
    lib = _lib.load()
    z, x = synthetic_inputs(85, B)
    a, w, tsz = _consts(B)
    eager = _engine(calib_sd, max_batch=B)
    g = _engine(calib_sd, max_batch=B, graphs=True)
    for m in (eager, g):
        m.template(z.cuda())
    torch.cuda.synchronize()

    def delta(m, fn):
        n0 = m.launch_count
        fn()
        torch.cuda.synchronize()
        return m.launch_count - n0

    xh = x.contiguous().pin_memory()
    th = torch.from_numpy(tsz.copy()).pin_memory()

    def host(m):
        tk, _ = _host_step(lib, m, m._stream(), B, xh, th, a, w)
        _lib.check(lib.sm_track_host_wait(m.handle, tk))

    counts = {"step eager": delta(eager, lambda: _device_step(eager, x, a, w, tsz))}
    for _ in range(2):                                       # first sight eager, then captured
        _device_step(g, x, a, w, tsz)
    counts["step replayed"] = delta(g, lambda: _device_step(g, x, a, w, tsz))
    counts["host decoupled"] = delta(eager, lambda: host(eager))
    for _ in range(4):                                       # both staging sets eager, then captured
        host(g)
    counts["host replayed"] = delta(g, lambda: host(g))
    assert len(set(counts.values())) == 1, counts
    assert counts["step eager"] > 0


def test_exports_after_decoupled_host_step(calib_sd):
    """After a decoupled sm_step_host_async and its wait, export() joins the lanes and gathers each lane's cached
    tensors: the same as after the device-pointer step on the same inputs."""
    B = 18
    lib = _lib.load()
    z, x = synthetic_inputs(86, B)
    a, w, tsz = _consts(B)
    m = _engine(calib_sd, max_batch=B)
    m.template(z.cuda())
    _device_step(m, x, a, w, tsz)
    want = {k: m.export(k).clone() for k in ("search", "p2")}
    _, x2 = synthetic_inputs(87, B)
    _device_step(m, x2, a, w, tsz)                           # different cached tensors in between
    torch.cuda.synchronize()
    xh = x.contiguous().pin_memory()
    th = torch.from_numpy(tsz.copy()).pin_memory()
    tk, _ = _host_step(lib, m, C.c_void_p(torch.cuda.current_stream().cuda_stream), B, xh, th, a, w)
    _lib.check(lib.sm_track_host_wait(m.handle, tk))
    for k, v in want.items():
        got = m.export(k)
        assert got.shape[0] == B
        assert torch.equal(got, v), k
