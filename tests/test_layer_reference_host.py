"""The per-layer float64 references (tests/layer_reference.py), chained layer by layer, reproduce the CPU oracle: this
pins the wiring table to `Oracle`, which tests/golden pins to the reference.  And the mutation helpers produce errors
of the size their docstrings claim."""
import numpy as np
import pytest
import torch

import layer_reference as lr
from oracle.calibrate import synthetic_inputs
from oracle.siammask_oracle import Oracle

TOL = 1e-6


def _oracle64(sd):
    """The oracle evaluated in float64, so that only a wiring difference can exceed TOL."""
    return Oracle({k: v.double() for k, v in sd.items()})


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def chain(sd, z, x, pos, backend="tensor", with_mask=True):
    """Every tap's float64 reference, each fed the previous references."""
    refs = {"z": z.double(), "x": x.double(), "pos": np.asarray(pos)}
    for t in lr.template_taps(backend, with_mask):
        refs["template:" + t.name] = lr.evaluate(sd, t, lambda n: refs["template:" + n] if n != "z" else refs["z"])[0]
    for t in lr.search_taps(backend=backend, with_mask=with_mask):
        refs[t.name] = lr.evaluate(sd, t, refs.__getitem__)[0]
    if with_mask:
        for t in lr.refine_taps():
            refs[t.name] = lr.evaluate(sd, t, refs.__getitem__)[0]
    return refs


@pytest.mark.parametrize("search,backend", [(255, "tensor"), (383, "tensor"), (255, "simt")])
def test_chain_reproduces_oracle(calib_sd, search, backend):
    z, x = synthetic_inputs(5, 1, search)
    R = (search - 127) // 8 + 1 + 8
    o = _oracle64(calib_sd)
    o.template(z.double())
    cls, loc, mask = o.track_mask(x.double())
    for pos in [(0, 0), (R - 1, R - 1), (R // 2, 3)]:
        refs = chain(calib_sd, z, x, [pos], backend)
        assert _rel(refs["template:crop_center"], o.zf) < TOL
        assert _rel(refs["features.downsample.downsample.0"], o.search) < TOL
        for i, n in enumerate(("stem", "features.features.layer1.2.conv3", "features.features.layer2.3.conv3",
                               "features.features.layer3.5.conv3")):
            assert _rel(refs[n], o.feature[i]) < TOL, n
        assert _rel(refs["corr_mask"], o.corr_feature) < TOL
        if backend == "simt":                         # unfused downsample, per-branch conv_search
            assert "features.features.layer1.0.downsample.0" in refs and "heads.conv_search_cat" not in refs
        assert _rel(refs["cls"], cls) < TOL and _rel(refs["loc"], loc) < TOL and _rel(refs["mask"], mask) < TOL
        assert _rel(refs["refine"].reshape(1, -1), o.track_refine(pos)) < TOL, pos
        if backend == "simt" or search == 383:
            break                                     # the refine positions are covered once


def test_chain_rpn_only(calib_sd):
    sd = {k: v for k, v in calib_sd.items() if not k.startswith(("mask_model.", "refine_model."))}
    z, x = synthetic_inputs(6, 2)
    o = _oracle64(sd)
    o.template(z.double())
    cls, loc = o.track(x.double())
    refs = chain(sd, z, x, None, with_mask=False)
    assert refs["heads.conv_search_cat"].shape[1] == 512
    assert _rel(refs["cls"], cls) < TOL and _rel(refs["loc"], loc) < TOL


def test_round_sig_error_size():
    t = torch.randn(10000, dtype=torch.float64) * 10.0 ** torch.randint(-30, 30, (10000,)).double()
    r = lr.round_sig(t, 11)
    rel = ((r - t).abs() / t.abs()).max()
    assert 2.0 ** -13 < rel <= 2.0 ** -11                # at most half an ulp of an 11-bit significand, and not less
    assert (r != 0).all()                                # no flush: the exponent range is unlimited
    # an 11-bit value survives unchanged (an fp16-representable hi plane loses nothing)
    h = torch.randn(1000).half().double()
    assert torch.equal(lr.round_sig(h, 11), h)


def test_drop_k_block_error_size():
    g = torch.Generator().manual_seed(0)
    w = torch.rand(8, 256, 3, 3, generator=g, dtype=torch.float64)
    x = torch.rand(1, 256, 6, 6, generator=g, dtype=torch.float64)
    full = torch.nn.functional.conv2d(x, w)
    cut = torch.nn.functional.conv2d(x, lr.drop_k_block(w, (1, 2), 64))
    # one of 36 equal-sized k-blocks of positive terms is missing: about 1/36 of every output element
    frac = (full - cut) / full
    assert float(frac.min()) > 0.5 / 36 and float(frac.max()) < 2.0 / 36


def test_drop_xcorr_tap_error_size():
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 4, 9, 9, generator=g, dtype=torch.float64)
    k = torch.rand(1, 4, 5, 5, generator=g, dtype=torch.float64)
    frac = (lr.xcorr(x, k) - lr.xcorr(x, lr.drop_xcorr_tap(k))) / lr.xcorr(x, k)
    # one of 25 taps of positive terms: 1/25 of an output element on average, never more than a few times that
    assert 0.5 / 25 < float(frac.mean()) < 2.0 / 25 and float(frac.min()) > 0 and float(frac.max()) < 5.0 / 25


def test_gate_rejects_and_accepts():
    ref = torch.tensor([1.0, -2.0, 1e-3], dtype=torch.float64)
    scale = torch.tensor([2.0, 3.0, 1e-3], dtype=torch.float64)
    ok = ref + 1e-7 * scale
    assert lr.ratio(ok, ref, scale, 1e-6, 0.0, 0.0)[1] <= 1.0
    bad = ref.clone()
    bad[2] += 1e-8                                        # small against the tensor, 1e-5 of its own element's scale
    raw, gated = lr.ratio(bad, ref, scale, 1e-6, 0.0, 0.0)
    assert gated > 1.0 and raw == pytest.approx(1e-5, rel=1e-6)
