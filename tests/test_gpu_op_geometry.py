"""The standalone convolution and cross-correlation operators against float64 over the geometries and ranges they
accept (case list, routes and gates: op_geometry_reference.py).

* Every conv case runs on its route (resident patch, GEMM with tiled or im2col operands, SIMT) in exact and fast mode
  (SIMT: exact), with and without ReLU, into the middle of a NaN-filled buffer whose guard elements must survive.
* Every xcorr case runs through `smb.conv2d_dw_group`, bulk pipeline, one-warp-per-plane and generic kernels.
* A range sweep: inputs with max |x| from 2^-30 to 2^30 against weights whose per-channel max runs from 2^-40 to 2^40
  (shift scaled alike), on every route, so the patch route's outputs reach far past fp16's 65504.  Each case must
  pass the gate; a wrong or infinite result must never come back.

Run with -s for the per-route table of measured gammas.  Worst measured on one H100 80GB HBM3 (700 W): conv exact
4.0e-7 (im2col), 3.8e-7 (tiled), 3.1e-7 (patch), SIMT 1.5e-7; fast 2.9e-4 (tiled), 2.9e-4 (im2col), 1.7e-4 (patch);
xcorr 2.6e-7 (one warp per plane), 2.4e-7 (bulk), 1.6e-7 (generic).  The file takes about 16 s.
"""
import collections

import pytest
import torch

import op_geometry_reference as R
import siammask_b200 as smb
from siammask_b200.ops import conv2d_route

pytestmark = pytest.mark.gpu

GUARD = 1024
TABLE = collections.defaultdict(float)      # (op, route, precision) -> worst measured gamma
NAN_BITS = torch.tensor([float("nan")], dtype=torch.float32).view(torch.int32)


def _guarded_conv(x, w, sc, sh, c, relu, precision, shape):
    n = int(torch.Size(shape).numel())
    buf = torch.full((GUARD + n + GUARD,), float("nan"), device="cuda")
    out = buf[GUARD:GUARD + n].view(shape)
    smb.conv2d(x, w, sc, sh, c.stride, c.pad, c.dil, relu=relu, backend=c.backend, precision=precision, out=out)
    torch.cuda.synchronize()
    bits = buf.view(torch.int32).cpu()
    guards_ok = torch.equal(bits[:GUARD], NAN_BITS.expand(GUARD)) and torch.equal(bits[-GUARD:],
                                                                                  NAN_BITS.expand(GUARD))
    return out.cpu(), guards_ok


def _check(c, x, w, sc, sh, precisions, relus, label):
    wf = R.folded(w, sc)
    base, scale = R.conv_ref(c, x, wf, sh)
    xd = x.cuda()
    fails = []
    for precision in precisions:
        route = R.conv_route(c, precision)
        assert conv2d_route(x.shape, w.shape, c.stride, c.pad, c.dil, c.backend, precision) == route
        for relu in relus:
            ref = base.relu() if relu else base
            got, guards_ok = _guarded_conv(xd, w, sc, sh, c, relu, precision, ref.shape)
            if not guards_ok:
                fails.append(f"{precision} relu={relu}: guard elements overwritten")
            raw, use = R.conv_gate(c, precision, got, ref, scale)
            TABLE[("conv2d", route, precision)] = max(TABLE[("conv2d", route, precision)], raw)
            if not use <= 1.0:            # NaN fails too
                d = ((got.double() - ref).abs() - R.conv_rho(c, precision) * ref.abs()) / scale.clamp_min(1e-300)
                d = torch.nan_to_num(d, nan=float("inf"))
                i = tuple(int(v) for v in torch.unravel_index(d.argmax(), ref.shape))
                fails.append(f"{label} {route} {precision} relu={relu}: measured gamma {raw:.3e} = {use:.2f} x the gate;"
                             f" worst at {i}: got {float(got[i]):.6e} ref {float(ref[i]):.6e} scale "
                             f"{float(scale[i]):.3e}")
    return fails


@pytest.mark.parametrize("i", range(len(R.CONV_CASES)),
                         ids=[f"{R.conv_route(c)}-{i}" for i, c in enumerate(R.CONV_CASES)])
def test_conv_geometry(i):
    c = R.CONV_CASES[i]
    x, w, sc, sh = R.conv_inputs(c, i)
    precisions = ("exact",) if c.backend == "simt" else ("exact", "fast")
    fails = _check(c, x, w, sc, sh, precisions, (False, True), str(c))
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("i", range(len(R.XCORR_CASES)), ids=[str(tuple(x)) for x in R.XCORR_CASES])
def test_xcorr_geometry(i):
    xc = R.XCORR_CASES[i]
    x, k = R.xcorr_inputs(xc, i)
    ref, scale = R.xcorr_ref(x, k)
    got = smb.conv2d_dw_group(x.cuda(), k.cuda()).cpu()
    raw, use = R.xcorr_gate(xc, got, ref, scale)
    bulk, rest = R.xcorr_route(xc)
    TABLE[("xcorr", f"bulk={int(bool(bulk))} rest={rest}", "f32")] = max(
        TABLE[("xcorr", f"bulk={int(bool(bulk))} rest={rest}", "f32")], raw)
    assert use <= 1.0, f"{xc}: measured gamma {raw:.3e} = {use:.2f} x the gate (n u / (1 - n u))"


RANGE_CASES = {"gemm_tiled": R.Conv(1, 64, 6, 10, 64, 1, 1, 1, 0, 1, "tensor"),
               "gemm_im2col": R.Conv(1, 64, 7, 9, 64, 3, 3, 1, 1, 1, "tensor"),
               "patch": R.Conv(1, 64, 9, 9, 64, 3, 3, 1, 1, 1, "tensor"),
               "simt": R.Conv(1, 16, 6, 7, 16, 3, 3, 1, 1, 1, "simt")}
X_EXPS = (-30, -15, 0, 15, 30)


@pytest.mark.parametrize("route", list(RANGE_CASES))
@pytest.mark.parametrize("xe", X_EXPS)
def test_conv_range(route, xe):
    """max |x| = 2^xe (about), channel n's weights and shift at 2^(-40 + 10 (n % 9)): every result within the gate."""
    c = RANGE_CASES[route]
    x, w, sc, sh = R.conv_inputs(c, 1000 + xe)
    t = torch.tensor([-40.0 + 10 * (n % 9) for n in range(c.Cout)])
    x = x * 2.0 ** xe
    w = w * torch.exp2(t).view(-1, 1, 1, 1)
    sh = sh * torch.exp2(t + xe)
    precisions = ("exact",) if c.backend == "simt" else ("exact", "fast")
    fails = _check(c, x, w, sc, sh, precisions, (False,), f"range 2^{xe}")
    assert not fails, "\n".join(fails)


@pytest.fixture(scope="module", autouse=True)
def _table():
    TABLE.clear()
    yield
    if TABLE:
        print("\n[op-geometry] op      route                        mode    measured gamma")
        for (op, route, mode), v in sorted(TABLE.items()):
            print(f"[op-geometry] {op:7s} {route:28s} {mode:6s} {v:.3e}")
