"""The host restatement of the tracker's glue (tests/tracker_glue_reference.py) against the reference loop's own numpy
(oracle/ref_loop.py), and the proof that the bit-exact assertions of tests/test_gpu_tracker_glue.py reject the
arithmetic variants a kernel can fall into: a float32 window, a fused pscore, a correctly rounded expf, truncation in
place of round(), and an FMA in crop_back's sub-box."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tracker_glue_reference as ref
from oracle import ref_loop


def _random_stream(R, seed):
    g = np.random.RandomState(seed)
    n = 5 * R * R
    cls = g.randn(1, 10, R, R).astype(np.float32) * 3
    loc = g.randn(1, 20, R, R).astype(np.float32) * 0.5
    anchor = ref_loop.generate_anchor({"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8]}, R)
    tsz = g.rand(2) * 60 + 20
    return cls, loc, anchor, tsz, n


@pytest.mark.parametrize("R", [25, 41])
def test_restatement_equals_reference_select(R):
    for seed in range(3):
        cls, loc, anchor, tsz, n = _random_stream(R, seed)
        # select_numpy decodes into its loc argument in place (a batch-1 permute is contiguous): hand it a copy
        want = ref_loop.select_numpy(torch.from_numpy(cls), torch.from_numpy(loc.copy()), anchor, ref.window(R, 5), tsz,
                                     0.04, 0.4)
        score = F.softmax(torch.from_numpy(cls).permute(1, 2, 3, 0).reshape(2, -1).permute(1, 0), dim=1)[:, 1].numpy()
        best, box, pen, ps = ref.select(score[None], loc.reshape(1, 4, n), anchor, ref.window(R, 5), tsz[None], 0.04, 0.4)
        assert best[0] == want[0]
        assert np.array_equal(box[0, :, best[0]], want[1].astype(np.float32))
        assert pen[0, best[0]] == want[3] and ps[0, best[0]] == want[4]


def test_window_tie_pairs():
    pairs = ref.window_tie_pairs(25)
    assert (60, 104) in pairs and len(pairs) >= 5
    w = np.outer(np.hanning(25), np.hanning(25)).flatten()
    assert w[60] == 0.06249999999999998 and w[104] == 0.06250000000000006
    assert ref.window_tie_pairs(41) == []


def tie_inputs(R, B, seed=0):
    """B streams, each one window-tie pair with equal cls / loc and a score in [0.63, 1); every other candidate has a
    score of ~2e-9 (window influence 0.4 then keeps it below the pair)."""
    g = np.random.RandomState(seed)
    pairs = ref.window_tie_pairs(R)
    n, RR = 5 * R * R, R * R
    cls = np.zeros((B, 2, n), np.float32)
    cls[:, 1] = -20
    loc = (g.randn(B, 4, n) * 0.1).astype(np.float32)
    for b in range(B):
        p, q = pairs[b % len(pairs)]
        a = g.randint(5)
        t = np.float32(g.uniform(0.6, 12))
        for i in (a * RR + p, a * RR + q):
            cls[b, 1, i] = t
            loc[b, :, i] = loc[b, :, a * RR + p]
    return cls, loc


def _score(cls):
    return torch.softmax(torch.from_numpy(cls), dim=1)[:, 1].numpy()


def test_mutations_of_the_selection_are_rejected():
    R, B = 25, 2048
    cls, loc = tie_inputs(R, B)
    anchor = ref_loop.generate_anchor({"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8]}, R)
    tsz = np.full((B, 2), 40.0)
    s = _score(cls)
    good = ref.select(s, loc, anchor, ref.window(R, 5), tsz, 0.0, 0.4)[0]
    # numpy ranks each pair through the float64 window: the first member wins some streams, the second others
    firsts = [p for p, _ in ref.window_tie_pairs(R)]
    assert np.isin(good % 625, firsts).any() and (~np.isin(good % 625, firsts)).any()
    w32 = ref.select(s, loc, anchor, ref.window(R, 5), tsz, 0.0, 0.4, window32=True)[0]
    assert (w32 != good).sum() > 0, "a float32 window must change some winners"
    for form in ("window", "score"):
        fz = ref.select(s, loc, anchor, ref.window(R, 5), tsz, 0.0, 0.4, fused=form)[0]
        assert (fz != good).sum() > 0, f"a fused pscore ({form}) must change some winners"


def expf_sweep():
    """~10^6 float32 arguments: the neighbourhoods of the overflow and underflow thresholds, the subnormal results,
    signed zeros, and a spread over the whole finite range of results."""
    g = np.random.RandomState(7)
    hi, lo = np.float32(88.72283935546875), np.float32(-103.97208404541015625)
    steps = np.arange(-3000, 3001, dtype=np.int32)
    nb = [(np.array([c], np.float32).view(np.int32) + steps).view(np.float32) for c in (hi, lo)]
    nb.append((np.array([-0.0], np.float32).view(np.int32) + np.arange(0, 2000, dtype=np.int32)).view(np.float32))
    x = np.concatenate(nb + [np.array([0.0, -0.0], np.float32),
                             g.uniform(-103.98, -87.3, 200_000).astype(np.float32),       # subnormal results
                             g.uniform(-104, 89, 780_000).astype(np.float32)])
    return x


def numpy_expf_is_simd():
    """numpy's float32 exp is the SIMD algorithm the device restates (not correctly rounded) when it differs from the
    correctly rounded result on part of the sweep; the device comparison is only meaningful then."""
    x = expf_sweep()
    with np.errstate(over="ignore", under="ignore"):
        return bool((np.exp(x) != ref.expf_cr(x)).any())


def test_correctly_rounded_expf_is_rejected():
    if not numpy_expf_is_simd():
        pytest.skip("this numpy's float32 exp is correctly rounded: not the SIMD algorithm the device restates")
    x = expf_sweep()
    with np.errstate(over="ignore", under="ignore"):
        assert (np.exp(x) != ref.expf_cr(x)).mean() > 1e-3


def edge_states():
    """(x, y, w, h) states on a 320 x 240 frame that reach both sides of every clamp and round() exactly at .5."""
    g = np.random.RandomState(3)
    rows = [[160.0, 120.0, 10.0, 10.0], [0.0, 0.0, 320.0, 240.0], [-50.0, 400.0, 12.0, 80.0], [1e4, -1e4, 30.0, 30.0],
            [319.5, 239.5, 200.0, 11.0], [3.0, 7.0, 64.0, 64.0]]
    # px - c exactly at .5: integer px, even round(s_x) (c = (s_x + 1) / 2 ends in .5)
    for w in range(10, 120, 7):
        rows.append([100.0 + w, 50.0, float(w), float(w) + 3])
    rows += list(np.stack([g.rand(40) * 400 - 40, g.rand(40) * 300 - 30, g.rand(40) * 300 + 2, g.rand(40) * 250 + 2], 1))
    return np.array(rows, np.float64)


def test_dropped_round_is_rejected():
    st = edge_states()
    good = ref.prepare(st, 0.45)[0]
    bad = ref.prepare(st, 0.45, trunc=True)[0]
    assert (good != bad).any()
    # the .5 cases of round(): px - c exactly halfway, round half to even
    assert any((st[i, 0] - (good[i, 2] + 1) / 2) % 1 == 0.5 for i in range(len(st)))


def test_prepare_matches_subwindow_box():
    st = edge_states()
    boxes, tsz, aux = ref.prepare(st)
    for i, (px, py, _, _) in enumerate(st):
        assert ref_loop.subwindow_box([px, py], int(boxes[i, 2]), [1, 2, 3])[:3] == list(boxes[i])


def update_inputs(R, B, seed=5):
    g = np.random.RandomState(seed)
    st = edge_states()[:B]
    B = len(st)
    _, _, aux = ref.prepare(st, 0.45)
    rec = np.zeros((B, 8), np.float32)
    rec[:, 0:2] = g.randn(B, 2) * 30
    rec[:, 2:4] = g.rand(B, 2) * 150 + 1
    rec[:, 4] = g.rand(B)
    rec[:, 7] = g.randint(0, 5 * R * R, B)
    return st, aux, rec


def test_fused_subbox_is_rejected():
    st, aux, rec = update_inputs(25, 100)
    im = np.tile([320, 240], (len(st), 1))
    _, good = ref.update(st, rec, aux, im, 0.0, 1.0, 25)
    _, bad = ref.update(st, rec, aux, im, 0.0, 1.0, 25, fused_subbox=True)
    assert (good != bad).any()
