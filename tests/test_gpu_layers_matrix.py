"""Every engine layer against float64 at the batch sizes a running engine sees, and the standalone conv per element.

A queued engine runs every batch from 1 to max_batch, and every search-side launch runs once per lane with
M = (lane streams) x Ho x Wo rows.  M decides which tiles of the wgmma conv GEMM, the resident-patch conv, the stem
and the xcorr are ragged and whether persistent CTAs take a second tile, so the batch sizes checked here are chosen
from the launch shapes (layer_reference.launches, lane split from siammask_b200.schedule) such that every launch of
a frame ends its last tile in the first warpgroup's rows (a), in the second's (b), and has more tiles than the SMs
(c).  Each such batch runs in both precision modes at both search sizes through the per-layer gate and mutation check
of test_gpu_layers.py, on the streams at the lane boundaries.  The remaining configurations: fast mode with
calibrated activation scales and with the adversarial checkpoint, the SIMT backend and the RPN-only engine batched
over two lanes.  Run with -s for the per-layer table.
"""
import collections

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_reference as lr
import siammask_b200 as smb
from oracle.calibrate import calibrated_state_dict, synthetic_inputs
from siammask_b200.schedule import lane_split
from test_gpu_layers import GAMMA, RHO, TABLE, Run, _assert, _engine, _frame, adversarial_sd, check, print_table

gpu = pytest.mark.gpu

# The family gammas of test_gpu_layers.GAMMA hold for every configuration here.  Worst measured |got - ref| / scale on
# one H100 (700 W): gemm exact 1.4e-6 (383 B=43, layer3.0.conv3), gemm fast 2.4e-4 (383 B=43, layer1.1.conv3; fast
# calib -10: 1.4e-4 at the stem), simt exact 3.3e-7 (simt B=59, mask), xcorr exact 1.4e-7 (rpn B=59); the conv2d sweep:
# exact 4.8e-7 (Cout 3969, K 1152, M 225), fast 3.1e-4 (Cout 3969, K 64, M 625: 160 tiles).
NUM_SMS = 132                       # H100 SXM
MAX_BATCH = 64                      # the streams per GPU of the default benchmark configuration
SEARCH_SIZES = (255, 383)

# (side, name, class) no batch up to MAX_BATCH reaches, per search size.  (c): the tile count stays <= NUM_SMS:
# template-side layer2 (225 B rows, one N tile: needs B >= 76), the 5x5 conv_kernel outputs (25 B rows, two N tiles:
# B >= 338) and refine v2.0 / v2.2 (225 rows per lane stream, one N tile: 76 streams per lane).  (b) at 255: the
# search side's 63 x 63 layers hold 31 x 128 + 1 rows per stream, so their last tile has as many rows as the lane has
# streams, at most 32 (two lanes of 32 at B = 64).
_NO_C = {("template", "features.features.layer2.0.conv2", "c")} | {
    ("template", f"features.features.layer2.{i}.conv{j}", "c") for i in (1, 2, 3) for j in (1, 2)} | {
    ("template", b + "conv_kernel.0", "c") for b in lr.BRANCHES} | {("refine", "refine_model.v2.0", "c"),
                                                                    ("refine", "refine_model.v2.2", "c")}
UNREACHABLE = {255: _NO_C | {("search", f"features.features.layer1.{i}.conv{j}", "b") for i in range(3)
                             for j in (1, 2, 3)} | {("search", "features.features.layer2.0.conv1", "b")},
               383: _NO_C}


def _coverage(search_size, batches, with_mask=True):
    """(side, name) -> {tile class: first batch in `batches` that exercises it}, classes (a)-(c).  Class (d), a third
    tile per persistent CTA, is planned and asserted up to the benchmark's batch sizes in test_gpu_layers_large.py."""
    cov = collections.defaultdict(dict)
    for B in batches:
        for launch in lr.launches(search_size, B, with_mask=with_mask, refine=with_mask):
            for c in lr.tile_classes(launch, NUM_SMS) - {"d"}:
                cov[(launch["side"], launch["name"])].setdefault(c, B)
    return cov


def batch_plan(search_size, with_mask=True):
    """A few batch sizes that together put every launch in every tile class it can reach up to MAX_BATCH: greedy set
    cover over 1..MAX_BATCH, the batch covering the most missing (launch, class) pairs first, the smaller on ties."""
    per_b = {B: {(k, c) for k, cs in _coverage(search_size, [B], with_mask).items() for c in cs}
             for B in range(1, MAX_BATCH + 1)}
    left, plan = set().union(*per_b.values()), []
    while left:
        B = max(per_b, key=lambda b: (len(per_b[b] & left), -b))
        plan.append(B)
        left -= per_b[B]
    return sorted(plan)


BATCHES = {S: batch_plan(S) for S in SEARCH_SIZES}


def boundary_streams(B):
    """The first and last stream of each lane (engine built with max_batch = B)."""
    off = np.cumsum([0] + lane_split(B, B))
    return sorted({int(s) for a, b in zip(off[:-1], off[1:]) for s in (a, b - 1)})


def test_batch_plan_covers_every_tile_class():
    """Host only.  Every conv / stem / xcorr launch of a frame is checked in tile classes (a), (b) and (c) at both search
    sizes, except the listed (launch, class) pairs no batch up to MAX_BATCH reaches; a new layer or a change to the lane
    split that leaves a class unchecked fails here."""
    for S in SEARCH_SIZES:
        cov = _coverage(S, BATCHES[S])
        print(f"\n[tiles] search {S}: batches {BATCHES[S]} (lanes {[lane_split(B, B) for B in BATCHES[S]]})")
        for (side, name), cs in sorted(cov.items()):
            print(f"[tiles]   {side:8s} {name:42s} " + "  ".join(f"{c}: B={cs[c]:2d}" for c in sorted(cs)))
        assert len(BATCHES[S]) <= 4 and any(len(lane_split(B, B)) > 1 for B in BATCHES[S])
        assert len(cov) == len({(d["side"], d["name"]) for d in lr.launches(S, 1)})
        missing = [(*k, c) for k, cs in cov.items() for c in "abc" if c not in cs and (*k, c) not in UNREACHABLE[S]]
        assert not missing, f"search {S}: launches without a checked tile class: {missing}"
        reach = _coverage(S, range(1, MAX_BATCH + 1))
        assert {(*k, c) for k, cs in reach.items() for c in "abc" if c not in cs} == UNREACHABLE[S]


def test_batch_plan_rpn_only_crosses_lanes():
    assert any(len(lane_split(B, B)) > 1 for B in batch_plan(255, with_mask=False))


def _pos(B, S):
    R = (S - 127) // 8 + 1 + 8
    return np.array([[(5 * b) % R, (11 * b + 3) % R] for b in range(B)])


@gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("S,B", [(S, B) for S in SEARCH_SIZES for B in BATCHES[S]])
def test_batched_layers(calib_sd, S, B, precision):
    m = _engine(calib_sd, search_size=S, max_batch=B, precision=precision)
    z, x = synthetic_inputs(40 + B, B, S)
    pos = _pos(B, S)
    run = Run(m, z, x, boundary_streams(B), pos, _frame(m, z, x, pos))
    _assert(*check(f"{precision} {S} B={B}", run, calib_sd, precision))


@gpu
@pytest.mark.parametrize("log2_scale", [10, -10])
def test_fast_calibrated_scales(log2_scale):
    sd = calibrated_state_dict(0, log2_scale)
    m = _engine(sd, precision="fast")
    z, x = synthetic_inputs(36, 1)
    m.calibrate(z.cuda(), x.cuda())
    pos = np.array([[12, 7]])
    run = Run(m, z, x, [0], pos, _frame(m, z, x, pos), calibrated=True)
    _assert(*check(f"fast calib {log2_scale:+d}", run, sd, "fast"))


@gpu
def test_fast_adversarial_checkpoint(calib_sd):
    sd = adversarial_sd(calib_sd)
    m = _engine(sd, precision="fast")
    z, x = synthetic_inputs(39, 1)
    m.calibrate(z.cuda(), x.cuda())
    pos = np.array([[6, 18]])
    run = Run(m, z, x, [0], pos, _frame(m, z, x, pos), calibrated=True)
    _assert(*check("fast adversarial", run, sd, "fast"))


@gpu
def test_simt_batched(calib_sd):
    B = max(BATCHES[255])
    m = _engine(calib_sd, backend="simt", max_batch=B)
    z, x = synthetic_inputs(41, B)
    pos = _pos(B, 255)
    run = Run(m, z, x, boundary_streams(B), pos, _frame(m, z, x, pos))
    _assert(*check(f"simt B={B}", run, calib_sd, "exact", backend="simt"))


@gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_rpn_only_batched(calib_sd, precision):
    B = max(batch_plan(255, with_mask=False))
    sd = {k: v for k, v in calib_sd.items() if not k.startswith(("mask_model.", "refine_model."))}
    m = _engine(sd, max_batch=B, mask=False, precision=precision)
    z, x = synthetic_inputs(42, B)
    m.template(z.cuda())
    cls, loc = m.track(x.cuda())
    torch.cuda.synchronize()
    run = Run(m, z, x, boundary_streams(B), np.zeros((B, 2), int), {"cls": cls, "loc": loc})
    _assert(*check(f"{precision} rpn B={B}", run, sd, precision, with_mask=False, refine=False))


@pytest.fixture(scope="module", autouse=True)
def _table():
    TABLE.clear()
    yield
    print_table()


# ---------------------------------------------------------------------------------------------------- smb.conv2d
# M classes (B, H): (a) 147 rows = 1 tile + 19; (b) 225 = 1 tile + 97; (c) more than NUM_SMS tiles (17298 rows with one
# N tile, 8649 rows with two, 625 rows with the 32 N tiles of Cout 3969)
COUTS = (1, 3, 10, 17, 33, 100, 129, 3969)
M_SHAPES = {"a": (3, 7), "b": (1, 15)}
C_SHAPES = {1: (2, 93), 2: (1, 93), 32: (1, 25)}         # N tiles -> (B, H) with more tiles than SMs
K_SHAPES = {"k64": (64, 1), "k1152": (128, 3)}            # one 64-channel k-block; 18 of them (3x3, pad 1)
CONV_SWEEP = [(co, mc, kc) for co in COUTS for mc in "abc" for kc in K_SHAPES]
GUARD = 4096                                              # NaN elements before and after the output


def _conv_shape(cout, mclass):
    if mclass != "c":
        return M_SHAPES[mclass]
    pad = lr._cout_pad(cout)
    return C_SHAPES[pad // min(pad, 128)]


@gpu
@pytest.mark.parametrize("cout,mclass,kclass", CONV_SWEEP, ids=[f"cout{c}-{m}-{k}" for c, m, k in CONV_SWEEP])
def test_conv2d_per_element(cout, mclass, kclass):
    """smb.conv2d against float64 F.conv2d with the layer gate |got - ref| <= gamma * scale + rho |ref| per element
    (scale = sum |x||w| over the window + |shift|), both precisions, with and without ReLU; the gate must reject a
    dropped lo plane of the input or the weights (exact) and a missing k-block; the output is written into the middle
    of a NaN-filled buffer whose guard elements must survive."""
    B, H = _conv_shape(cout, mclass)
    cin, k = K_SHAPES[kclass]
    g = torch.Generator().manual_seed(cout * 7 + ord(mclass) + k)
    x = torch.randn(B, cin, H, H, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    sc = torch.rand(cout, generator=g) + 0.5
    sh = torch.randn(cout, generator=g) * 0.1
    pad = k // 2
    wf = w.double() * sc.double().view(-1, 1, 1, 1)
    xd = x.double()

    def conv(xx, ww):
        return F.conv2d(xx, ww, None, 1, pad)
    ref = conv(xd, wf) + sh.double().view(1, -1, 1, 1)
    scale = conv(xd.abs(), wf.abs()) + sh.double().abs().view(1, -1, 1, 1)
    n = ref.numel()
    launch = dict(M=B * H * H, tiles=-(-B * H * H // 128) * (lr._cout_pad(cout) // min(lr._cout_pad(cout), 128)))
    assert mclass in lr.tile_classes(launch, NUM_SMS)
    muts = {"c: one k-block missing": conv(xd, lr.drop_k_block(wf, (1, 1), 0, 64)) + sh.double().view(1, -1, 1, 1),
            "a: input lo dropped": conv(lr.round_sig(xd), wf) + sh.double().view(1, -1, 1, 1),
            "b: weight lo dropped": conv(xd, lr.round_sig(wf)) + sh.double().view(1, -1, 1, 1)}
    nan_bits = torch.tensor([float("nan")], dtype=torch.float32).view(torch.int32)
    fails = []
    for precision in ("exact", "fast"):
        gamma = GAMMA[("gemm", precision)]
        for relu in (False, True):
            buf = torch.full((GUARD + n + GUARD,), float("nan"), device="cuda")
            out = buf[GUARD:GUARD + n].view(ref.shape)
            smb.conv2d(x.cuda(), w, sc, sh, 1, pad, 1, relu=relu, precision=precision, out=out)
            torch.cuda.synchronize()
            bits = buf.view(torch.int32).cpu()
            if not (torch.equal(bits[:GUARD], nan_bits.expand(GUARD)) and torch.equal(bits[-GUARD:],
                                                                                     nan_bits.expand(GUARD))):
                fails.append(f"{precision} relu={relu}: guard elements overwritten")
            r = ref.relu() if relu else ref
            got = out.cpu()
            raw, gated = lr.ratio(got, r, scale, gamma, RHO["f32"], 1e-30)
            TABLE.append((f"conv2d {mclass} {kclass} B={B} H={H}", f"Cout {cout} relu={int(relu)}", "gemm",
                          precision, raw, gated))
            if not gated <= 1.0:
                d = ((got.double() - r).abs() - RHO["f32"] * r.abs()) / scale
                i = np.unravel_index(int(d.argmax()), tuple(r.shape))
                fails.append(f"{precision} relu={relu}: measured gamma {raw:.3e}, {gated:.2f} x the gate; worst at "
                             f"{i}: got {float(got[i]):.6e} ref {float(r[i]):.6e} scale {float(scale[i]):.3e}")
            for label, mut in muts.items():
                if precision == "fast" and label[0] in "ab":
                    continue
                if lr.ratio(mut.relu() if relu else mut, r, scale, gamma, RHO["f32"], 1e-30)[1] <= 1.0:
                    fails.append(f"{precision} relu={relu}: gate does not reject {label}")
    assert not fails, "\n".join(fails)
