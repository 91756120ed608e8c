"""Host-only checks of the standalone operators' geometry tests (op_geometry_reference.py): the route restatement
against the library's own rule, the coverage of the case list, the gates against plausible kernel defects, and the
argument checks of the C ABI, which run before the library looks for a device."""
import ctypes as C
import itertools

import pytest
import torch

import op_geometry_reference as R
from siammask_b200 import _lib, ops


def _lib_route(c, precision="exact"):
    try:
        return ops.conv2d_route((c.B, c.Cin, c.H, c.W), (c.Cout, c.Cin, c.KH, c.KW), c.stride, c.pad, c.dil, c.backend,
                                precision)
    except RuntimeError:
        return None


def _table():
    """Accepted and rejected geometries around every limit of the rule, plus the case list."""
    rows = list(R.CONV_CASES)
    for W, cin, cout, k, s, p, d in itertools.product((1, 7, 8, 16, 23, 24, 63, 64), (64, 128, 96), (64, 128), (1, 3),
                                                      (0, 1, 2, 8, 9), (-1, 0, 1, 2), (0, 1, 3)):
        rows.append(R.Conv(1, cin, W, W, cout, k, k, s, p, d, "tensor"))
    rows.append(R.Conv(1, 64, 9, 8, 64, 3, 3, 1, 1, 1, "tensor"))                 # not square: GEMM
    for p, k, d in ((128, 3, 1), (129, 3, 1), (0, 3, 65), (0, 3, 64), (1, 130, 1), (127, 1, 1), (128, 1, 1),
                    (130, 3, 1)):
        rows.append(R.Conv(1, 64, 300, 300, 8, k, k, 1, p, d, "tensor"))          # im2col corners
        rows.append(R.Conv(1, 64, 300, 300, 8, k, k, 1, p, d, "simt"))
    rows += [R.Conv(0, 64, 4, 4, 8, 1, 1, 1, 0, 1, "tensor"), R.Conv(1, 64, 4, 4, 0, 1, 1, 1, 0, 1, "tensor"),
             R.Conv(1, 64, 0, 4, 8, 1, 1, 1, 0, 1, "tensor"), R.Conv(1, 64, 4, 4, 8, 0, 1, 1, 0, 1, "tensor"),
             R.Conv(1, 64, 4, 4, 8, 5, 5, 1, 0, 1, "tensor"), R.Conv(1, 64, 4, 4, 8, 5, 5, 1, 0, 1, "simt"),
             R.Conv(1, 64, 4, 4, 8, 5, 5, 1, 1, 1, "tensor"), R.Conv(1, 16, 4, 4, 8, 1, 1, 1, 0, 1, "tensor"),
             R.Conv(1, 64, 4, 4, 8, 1, 1, 9, 0, 1, "simt"), R.Conv(2 ** 16, 64, 256, 256, 8, 1, 1, 1, 0, 1, "simt")]
    return rows


def test_route_restatement_matches_the_library():
    mismatch = []
    for c, p in itertools.product(_table(), R.PRECISIONS):
        want = R.conv_route(c, p) if R.conv_accepts(c) else None
        if _lib_route(c, p) != want:
            mismatch.append((c, p, want, _lib_route(c, p)))
    assert not mismatch, mismatch[:10]


def test_patch_widths():
    """The resident-patch kernel takes square W in {1..15, 24..31, 56..63} at Cin == Cout in {64, 128}, except 128
    channels at W 56..63 in exact mode, whose two split-plane patch buffers do not fit shared memory (the GEMM takes
    those)."""
    want = set(range(1, 16)) | set(range(24, 32)) | set(range(56, 64))
    for cm, p in itertools.product((64, 128), R.PRECISIONS):
        got = {W for W in range(1, 130) if _lib_route(R.Conv(1, cm, W, W, cm, 3, 3, 1, 1, 1, "tensor"), p) == "patch"}
        assert got == (want - set(range(56, 64)) if (cm, p) == (128, "exact") else want), (cm, p)
        assert {W for W in range(1, 130) if R.patch_ok(W, cm, p)} == got


def test_case_list_covers_every_route_and_class():
    cov = {}
    for c, p in itertools.product(R.CONV_CASES, R.PRECISIONS):
        assert R.conv_accepts(c) and _lib_route(c, p) == R.conv_route(c, p), c
        cov.setdefault(R.conv_route(c, p), set()).update(R.conv_classes(c, p))
    assert set(cov) == {"simt", "gemm_tiled", "gemm_im2col", "patch"}
    for route, got in cov.items():
        need = R.CONV_CLASSES | (R.PATCH_CLASSES if route == "patch" else set())
        missing = {k for k in need - got if (route, k) not in R.NOT_APPLICABLE}
        assert not missing, f"{route}: no case in classes {sorted(missing)}"
        assert not {k for k in got if (route, k) in R.NOT_APPLICABLE}, f"{route}: a class listed as impossible occurs"
    assert any(c.KH * c.KW * c.Cin > R.K_ENGINE_MAX for c in R.CONV_CASES if R.conv_route(c) == "gemm_im2col")
    xcov = set().union(*(R.xcorr_classes(x) for x in R.XCORR_CASES))
    assert not R.XCORR_REQUIRED - xcov, f"xcorr classes without a case: {sorted(R.XCORR_REQUIRED - xcov)}"
    assert {R.xcorr_route(x)[1] for x in R.XCORR_CASES} == {None, "one_warp", "generic"}
    assert any(R.xcorr_route(x)[0] and R.xcorr_route(x)[1] for x in R.XCORR_CASES)


def _mutant_cases():
    """Per route, the cases with the fewest output elements (cheap in float64)."""
    by_route = {}
    for i, c in enumerate(R.CONV_CASES):
        by_route.setdefault(R.conv_route(c), []).append((c.B * c.Cout * R.out_hw(c)[0] * R.out_hw(c)[1], i, c))
    return [(i, c) for v in by_route.values() for _, i, c in sorted(v)[:4]]


@pytest.mark.parametrize("i,c", _mutant_cases(), ids=lambda v: str(v) if isinstance(v, int) else R.conv_route(v))
def test_conv_gate_rejects_mutants(i, c):
    """The exact-mode gate of each route rejects an H / W mix-up, a dilation off by one, a missing last k-block and a
    dropped lo plane of the input (where the geometry lets the defect change the output)."""
    x, w, sc, sh = R.conv_inputs(c, i)
    wf = R.folded(w, sc)
    ref, scale = R.conv_ref(c, x, wf, sh)
    assert R.conv_gate(c, "exact", ref, ref, scale)[1] <= 0.0
    Ho, Wo = R.out_hw(c)
    muts = {"lo dropped": R.mut_lo_dropped(c, x, wf, sh), "last k-block": R.mut_last_kblock(c, x, wf, sh)}
    if Ho > 1 and Wo > 1:
        muts["H/W transposed"] = R.mut_transposed(ref)
    if c.KH * c.KW > 1:
        muts["dilation + 1"] = R.mut_dilation(c, x, wf, sh)
    for name, m in muts.items():
        if torch.equal(m, ref):              # e.g. the last tap of a 3x3 on a 1 x 1 image reads padding only
            continue
        assert R.conv_gate(c, "exact", m, ref, scale)[1] > 1.0, f"gate does not reject {name}"


@pytest.mark.parametrize("i", range(len(R.XCORR_CASES)))
def test_xcorr_gate_rejects_shifted_kernel(i):
    x = R.XCORR_CASES[i]
    xs, ks = R.xcorr_inputs(x, i)
    ref, scale = R.xcorr_ref(xs, ks)
    assert R.xcorr_gate(x, ref, ref, scale)[1] <= 0.0
    if x.kw > 1:
        assert R.xcorr_gate(x, R.mut_xcorr_shift(xs, ks), ref, scale)[1] > 1.0


def test_gamma_scales_with_k_beyond_the_engine():
    c = R.Conv(1, 576, 6, 5, 24, 3, 3, 1, 1, 1, "tensor")
    assert R.conv_gamma(c, "exact") == R.GAMMA[("gemm", "exact")] * 5184 / 4864
    assert R.conv_gamma(c._replace(Cin=64), "fast") == R.GAMMA[("gemm", "fast")]


BAD_CONV = [  # (B, Cin, H, W, Cout, KH, KW, stride, pad, dil, backend, precision)
    (1, 64, 8, 8, 8, 3, 3, 0, 1, 1, 0, 0), (1, 64, 8, 8, 8, 3, 3, -1, 1, 1, 0, 0), (1, 64, 8, 8, 8, 3, 3, 1, -1, 1, 0, 0),
    (1, 64, 8, 8, 8, 3, 3, 1, 1, 0, 0, 0), (1, 64, 8, 8, 8, 3, 3, 1, 1, 0, 1, 0), (1, 64, 2, 8, 8, 5, 3, 1, 0, 1, 0, 0),
    (1, 64, 8, 2, 8, 3, 5, 1, 0, 1, 1, 0), (1, 64, 8, 8, 8, 3, 3, 9, 1, 1, 0, 0), (1, 64, 300, 300, 8, 3, 3, 1, 129, 1, 0, 0),
    (1, 64, 300, 300, 8, 3, 3, 1, 0, 65, 0, 0), (1, 64, 300, 300, 8, 3, 3, 1, 130, 1, 0, 0), (0, 64, 8, 8, 8, 1, 1, 1, 0, 1, 0, 0),
    (1, 0, 8, 8, 8, 1, 1, 1, 0, 1, 1, 0), (1, 64, 8, 8, 0, 1, 1, 1, 0, 1, 0, 0), (1, 64, 8, 8, 8, 0, 1, 1, 0, 1, 0, 0),
    (1, 48, 8, 8, 8, 1, 1, 1, 0, 1, 0, 0), (1, 64, 8, 8, 8, 1, 1, 1, 0, 1, 2, 0), (1, 64, 8, 8, 8, 1, 1, 1, 0, 1, 0, 2),
    (2 ** 16, 64, 256, 256, 8, 1, 1, 1, 0, 1, 1, 0),
]
BAD_XCORR = [(0, 1, 8, 8, 3, 3), (1, 0, 8, 8, 3, 3), (1, 1, 8, 8, 0, 3), (1, 1, 8, 8, 3, 0), (1, 1, 2, 8, 3, 3),
             (1, 1, 8, 2, 3, 3), (1, 1, 8, 8, -1, 3), (2 ** 16, 2 ** 10, 64, 64, 5, 5)]


def test_route_query_rejects_bad_arguments():
    lib = _lib.load()
    r = C.c_int32(-1)
    for a in BAD_CONV:
        assert lib.sm_conv2d_route(*a, C.byref(r)) != 0, a
        assert b"no CUDA device" not in lib.sm_last_error()
    assert lib.sm_conv2d_route(1, 64, 8, 8, 8, 1, 1, 1, 0, 1, 0, 0, None) != 0
    assert lib.sm_conv2d_route(1, 64, 8, 8, 64, 3, 3, 1, 1, 1, 0, 0, C.byref(r)) == 0
    assert r.value == _lib.SM_CONV_ROUTE_PATCH


@pytest.mark.skipif(torch.cuda.is_available(), reason="calls the operators with host buffers: only WITHOUT a GPU")
def test_operators_check_arguments_before_the_device():
    """On a machine without a GPU the argument checks answer first; accepted arguments reach the device check."""
    lib = _lib.load()
    buf = (C.c_float * 16)()
    for a in BAD_CONV:
        assert lib.sm_conv2d(buf, buf, None, None, buf, *a[:10], 0, *a[10:], None) != 0, a
        assert b"no CUDA device" not in lib.sm_last_error(), a
    for a in BAD_XCORR:
        assert lib.sm_xcorr_depthwise(buf, buf, buf, *a, None) != 0, a
        assert b"no CUDA device" not in lib.sm_last_error(), a
    assert lib.sm_conv2d(buf, buf, None, None, buf, 1, 64, 8, 8, 8, 1, 1, 1, 0, 1, 0, 0, 0, None) != 0
    assert b"no CUDA device" in lib.sm_last_error()
    assert lib.sm_xcorr_depthwise(buf, buf, buf, 1, 1, 8, 8, 3, 3, None) != 0
    assert b"no CUDA device" in lib.sm_last_error()


def test_conv2d_checks_arguments_first():
    """ops.conv2d rejects a bad geometry with the library's message (stride 0 used to be a ZeroDivisionError)."""
    x, w = torch.zeros(1, 64, 8, 8), torch.zeros(8, 64, 3, 3)
    for kw in (dict(stride=0), dict(padding=-1), dict(dilation=0), dict(stride=9, padding=1), dict(padding=200)):
        with pytest.raises(RuntimeError, match="check failed"):
            ops.conv2d(x, w, **kw)
    with pytest.raises(RuntimeError, match="weight"):
        ops.conv2d(x, torch.zeros(8, 32, 3, 3))
    with pytest.raises(RuntimeError, match="scale"):
        ops.conv2d(x, w, torch.ones(7))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.conv2d(x, w, stride=2)                        # accepted geometry: only now the missing device
