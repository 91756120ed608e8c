"""Every engine layer on its own against a float64 reference (tests/layer_reference.py), in both precision modes.

Each configuration runs once (template -> track_mask -> track_refine, or step); then every recorded tensor is checked
against its layer's float64 reference, computed from the engine's own exported inputs, with the per-element gate
|got - ref| <= gamma * scale + rho * |ref| + tau.  Copies (max-pool, crops, the corr gather) must match bit for bit.
For B > 2 only the streams at lane boundaries are checked (0, last of lane 0, first of lane 1, last), which keeps
the float64 CPU work bounded.  Run with -s for the per-layer worst-ratio table.
"""
import collections

import numpy as np
import pytest
import torch

import layer_reference as lr
import siammask_b200 as smb
from oracle.calibrate import calibrated_state_dict, synthetic_inputs
from siammask_b200 import anchors as anc

pytestmark = pytest.mark.gpu

# (family, mode) -> gamma: the accumulation / operand-quantisation term, in units of the element's scale.  Set at
# >= 4x the worst measured |got - ref| / scale on one H100 (700 W), measured value beside it.
GAMMA = {
    ("gemm", "exact"): 2.0 ** -17,      # measured 1.6e-6 (2^-19.2): 383 B=1, layer3.0.conv3 (K = 256 + 4608)
    ("gemm", "fast"): 2.0 ** -9,        # measured 2.6e-4 (2^-11.9): fast B=2, layer1.1.conv3
    ("xcorr", "exact"): 2.0 ** -20,     # measured 1.7e-7 (2^-22.5)
    ("xcorr", "fast"): 2.0 ** -20,      # measured <= 0: the fp16 output rounding (rho) covers it
    ("simt", "exact"): 2.0 ** -19,      # measured 3.4e-7 (2^-21.5): SIMT backend, layer3.0.downsample.0 (K = 4608)
    ("simt", "fast"): 2.0 ** -19,       # measured 3.7e-7 (2^-21.4): refine post0 (fp32 kernels in both modes)
}
# output storage -> rho: relative rounding of the stored value
RHO = {"split": 2.0 ** -22, "hi": 2.0 ** -11, "f32": 2.0 ** -24}

# launch names of one profiled frame that this file does not check per layer, and why
SKIP = {
    "select": "score/box selection, checked against its float64 numpy restatement in test_gpu_shapes.py",
    "scatter_slots": "a copy; checked through the xcorr of the slot-table config, which reads the scattered rows",
    "mask_col": "a copy of one mask-head column, compared bit for bit with the head output in test_gpu_shapes.py",
    "export": "the copy these checks read every tensor through",
}
# profiled launch name -> tap that checks it (conv launches are named by their checkpoint key)
LAUNCH_TAP = {"crop_p0": "refine:crop_p0", "crop_p1": "refine:crop_p1", "crop_p2": "refine:crop_p2",
              "deconv": "refine:deconv"}

# (config, tap, mutation) the family gate cannot reject because the layer's output there is almost all shift, so no
# operand error is visible against its scale.  The same layers reject every mutation in the other configurations.
# Measured on one H100: the kernel's own error at these layers is within rho and tau (measured gamma <= 0); the
# mutation, in units of scale, against gamma = 2^-17 = 7.6e-6:
#  * calib -10: calibrated_state_dict(0, -10) floors the head BN variances at 1e-4, so the heads are 32-96 % shift,
#    K = 256:
#    cls head.0 (a) 6.6e-6 (b) 5.8e-6; cls head.3 (a) 5.3e-6 (b) 7.1e-6; loc head.0 (a) 2.8e-6 (b) 1.5e-6;
#    loc head.3 (a) 8.4e-7 (b) 1.2e-6.
#  * adversarial: layer2.2.conv2 reads the 1e-6 layer, so it is 99.8 % shift, K = 1152: (a) and (b) <= 0.
#  * fast adversarial, the same layer: (c) changes it by at most 1.0e-4 of scale (template 9.9e-5, search 1.0e-4; the
#    float64 chain from the same inputs), below the fp16 output rounding rho = 2^-11 = 4.9e-4 of |ref| ~ scale.
SHIFT_DOMINATED = {("exact calib -10", n, m) for n in ("rpn_model.cls.head.0", "cls", "rpn_model.loc.head.0", "loc")
                   for m in "ab"} | {(cfg, p + "features.features.layer2.2.conv2", m)
                                     for p in ("", "template:")
                                     for cfg, m in (("exact adversarial", "a"), ("exact adversarial", "b"),
                                                    ("fast adversarial", "c"))}

TABLE = []          # (config, tap, family, mode, measured gamma, gate use)


def print_table():
    """The per-layer measured gammas of every configuration checked so far, and the worst per (family, mode)."""
    if not TABLE:
        return
    print("\n[layers] config                 tap                                         family mode   "
          "measured gamma  gate use")
    for cfg, name, fam, mode, raw, gated in TABLE:
        print(f"[layers] {cfg:22s} {name:43s} {fam:6s} {mode:6s} {raw:13.3e}  {gated:8.3f}")
    worst = collections.defaultdict(float)
    for cfg, name, fam, mode, raw, gated in TABLE:
        worst[(fam, mode)] = max(worst[(fam, mode)], raw)
    for k, v in sorted(worst.items()):
        print(f"[layers] max over layers {k[0]:6s} {k[1]:6s} {v:.3e}  (gamma {GAMMA.get(k, 0):.3e})")


@pytest.fixture(scope="module", autouse=True)
def _table():
    yield
    print_table()


def _engine(sd, **kw):
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, **kw)
    m.load_state_dict(sd)
    return m.eval().to("cuda")


def _rows(t, rows):
    return t.detach()[list(rows)].cpu().double()


class Run:
    """The exported tensors of one engine call sequence, restricted to the checked streams.  tap_streams (optional):
    tap name -> the subset of `streams` checked at that tap (default: all of them); mutation_streams (optional): the
    subset of `streams` every tap's mutations are evaluated at (default: the tap's checked streams)."""

    def __init__(self, m, z, x, streams, pos, outputs, kernel_rows=None, calibrated=False, tap_streams=None,
                 mutation_streams=None):
        self.m, self.streams, self.outputs, self.calibrated = m, list(streams), outputs, calibrated
        self.kernel_rows = list(kernel_rows) if kernel_rows is not None else self.streams
        self.base = {"z": _rows(z, streams), "x": _rows(x, streams), "pos": np.asarray(pos)[self.streams]}
        self.cache = {}
        self.tap_streams, self.mutation_streams = tap_streams, mutation_streams

    def select(self, name, mutation=False):
        """Positions in `streams` of the streams checked at tap `name` (mutation: of the streams its mutations are
        evaluated at), or None for all of them."""
        if mutation and self.mutation_streams is not None:
            return [self.streams.index(s) for s in sorted(self.mutation_streams)]
        if self.tap_streams is None or name not in self.tap_streams:
            return None
        return [self.streams.index(s) for s in sorted(self.tap_streams[name])]

    def get(self, name, for_xcorr=False):
        if name in self.base:
            return self.base[name]
        key = (name, for_xcorr)
        if key not in self.cache:
            if name in self.outputs:
                t = self.outputs[name]
                if name == "mask":
                    t = t.reshape(t.shape[0], 3969, *t.shape[-2:])
                elif name == "refine":
                    t = t.reshape(-1, 1, 127, 127)
            else:
                t = self.m.export(name)
            self.cache[key] = _rows(t, self.kernel_rows if for_xcorr else self.streams)
        return self.cache[key]


def _tap_list(backend, with_mask, mask_head, refine):
    taps = [(t, "template:") for t in lr.template_taps(backend, with_mask)]
    taps += [(t, "") for t in lr.search_taps(backend=backend, with_mask=with_mask, mask_head=mask_head)]
    if refine:
        taps += [(t, "") for t in lr.refine_taps()]
    return taps


def check(cfg, run, sd, precision, backend="tensor", with_mask=True, mask_head=True, refine=True, stale=None):
    """Check every tap, and that its gate rejects every mutation of the layer; returns (failures, mutations the gate
    accepts).  The measured numbers go to TABLE.  stale (optional): stale(name, tap, fetch, streams) -> a fetch that
    returns the tap's inputs (rows: `streams`) with some rows of the previous engine call in place of this call's, or
    None; the gate must reject that as well (mutation d)."""
    mode = "exact" if precision == "exact" else "fast"
    fails, insensitive = [], []
    taps = _tap_list(backend, with_mask, mask_head, refine)
    # backbone layers run on both sides under one activation scale
    shared = {t.name for t, p in taps if p} & {t.name for t, p in taps if not p and t.op == "conv"}
    for tap, prefix in taps:
        name = prefix + tap.name

        def fetcher(sel, prefix=prefix, tap=tap):
            def fetch(n):
                if n in ("z", "x", "pos"):
                    t = run.get(n)
                elif prefix and n != "z":
                    t = run.get(prefix + n)
                else:
                    t = run.get(n, for_xcorr=tap.op == "xcorr" and n.startswith("template:"))
                return t if sel is None else t[sel]
            return fetch
        sel, msel = run.select(name), run.select(name, mutation=True)
        fetch = fetcher(sel)
        ref, scale = lr.evaluate(sd, tap, fetch)
        got = run.get(name) if sel is None else run.get(name)[sel]
        fam = lr.family(tap, backend)
        if fam == "exact":
            if not torch.equal(got.float(), ref.float().reshape(got.shape)):
                fails.append(f"{name}: not bit-exact")
            continue
        gamma, rho = GAMMA[(fam, mode)], RHO[lr.out_format(tap, precision)]
        peak = float(ref.abs().max())
        if run.calibrated and tap.name in shared:
            peak = max(peak, float(run.get(tap.name if prefix else "template:" + tap.name).abs().max()))
        tau = lr.tau_for(peak, lr.out_format(tap, precision), run.calibrated)
        raw, gated = lr.ratio(got, ref, scale, gamma, rho, tau)
        TABLE.append((cfg, name, fam, mode, raw, gated))
        if not gated <= 1.0:
            d = ((got.reshape(ref.shape) - ref).abs() - rho * ref.abs() - tau) / scale.clamp_min(1e-300)
            i = np.unravel_index(int(d.argmax()), tuple(ref.shape))
            fails.append(f"{name} ({fam}/{mode}): measured gamma {raw:.3e}, {gated:.2f} x the gate; worst at {i}: "
                         f"got {float(got.reshape(ref.shape)[i]):.6e} ref {float(ref[i]):.6e} scale "
                         f"{float(scale[i]):.3e} (max|ref| {float(ref.abs().max()):.3e})")
        if msel != sel:                                           # the mutations at other (fewer) streams
            fetch = fetcher(msel)
            ref, scale = lr.evaluate(sd, tap, fetch)
        stale_fetch = None if stale is None else stale(name, tap, fetch,
                                                       run.streams if msel is None else [run.streams[i] for i in msel])
        insensitive += [f"{name}: {m}" for m in _mutations_passing(sd, tap, fetch, ref, scale, gamma, rho, tau,
                                                                    fam, precision, stale_fetch)
                        if (cfg, name, m[0]) not in SHIFT_DOMINATED]
    return fails, insensitive


def _split(n):
    """Whether the tensor named n reaches its consumer as fp16 planes (hi + lo in exact mode) rather than as fp32."""
    return n not in ("x", "z", "pos") and n not in lr.F32_OUT


def _mutations_passing(sd, tap, fetch, ref, scale, gamma, rho, tau, fam, precision, stale_fetch=None):
    """Mutations of the layer that its gate fails to reject.  (a) exact mode: the lo plane of every split-fp16 input is
    dropped (the xcorr's search input and kernel separately); (b) exact mode, tensor-core convs: the weight lo plane is
    dropped; (c) one 64-channel k-block of one kernel tap of the (first) conv is missing; for the fp32 SIMT convs and
    the deconv one input channel, for xcorr one of the 25 taps; (d) with stale_fetch: input rows the previous engine
    call left behind read in place of this call's."""
    muts = {}
    if stale_fetch is not None:
        muts["d: stale rows of the previous call"] = dict(fetch=stale_fetch)
    if precision == "exact":
        if tap.op == "xcorr":
            muts["a: search lo dropped"] = dict(fetch=lambda n: lr.round_sig(fetch(n)) if n == tap.inputs[0]
                                                else fetch(n))
            muts["a: kernel lo dropped"] = dict(k_mut=lr.round_sig)
        elif any(_split(n) for n in tap.inputs):                # not the stem: 0..255 pixels are exact in fp16
            muts["a: input lo dropped"] = dict(fetch=lambda n: lr.round_sig(fetch(n)) if _split(n) else fetch(n))
        if fam == "gemm":
            muts["b: weight lo dropped"] = dict(w_mut=lr.round_sig, w2_mut=lr.round_sig)
    # (c) removes the block / channel that carries the most input (a missing channel of zeros is no defect)
    if tap.op == "xcorr":
        muts["c: one xcorr tap missing"] = dict(k_mut=lr.drop_xcorr_tap)
    else:
        xin = fetch(tap.inputs[0]).abs()
        if tap.op == "small" and len(tap.inputs) == 2:
            xin = xin + fetch(tap.inputs[1]).abs()
        mass = xin.reshape(xin.shape[0], xin.shape[1], -1).sum((0, 2))       # per input channel
        if fam == "gemm":                                     # the stem's 3 channels sit in one k-block
            c0 = 64 * int(mass.reshape(-1, 64).sum(1).argmax()) if mass.numel() % 64 == 0 else 0
            muts["c: one k-block missing"] = dict(w_mut=lambda w: lr.drop_k_block(w, (1, 1), c0, 64))
        else:
            c, dim = int(mass.argmax()), 0 if tap.op == "deconv" else 1   # ConvTranspose2d weights: [Cin, Cout, ..]
            muts["c: one input channel missing"] = dict(w_mut=lambda w: w.index_fill(dim, torch.tensor([c]), 0.0))
    passing = []
    for label, kw in muts.items():
        f = kw.pop("fetch", fetch)
        mut, _ = lr.evaluate(sd, tap, f, **kw)
        if lr.ratio(mut, ref, scale, gamma, rho, tau)[1] <= 1.0:
            passing.append(label)
    return passing


def _assert(fails, insensitive=()):
    assert not fails, "\n".join(fails)
    assert not insensitive, "gate does not reject: " + "\n".join(insensitive)


def _frame(m, z, x, pos, mask_head=True, refine=True):
    m.template(z.cuda())
    cls, loc, mask = m.track_mask(x.cuda(), mask_head=mask_head)
    out = {"cls": cls, "loc": loc}
    if mask_head:
        out["mask"] = mask
    if refine:
        out["refine"] = m.track_refine(pos)
    torch.cuda.synchronize()
    return out


def test_exact_255_b1(calib_sd):
    m = _engine(calib_sd)
    z, x = synthetic_inputs(31, 1)
    pos = np.array([[0, 24]])
    run = Run(m, z, x, [0], pos, _frame(m, z, x, pos))
    _assert(*check("exact 255 B=1", run, calib_sd, "exact"))


def test_every_launch_is_checked(calib_sd):
    """Coverage by construction: every launch of one profiled frame is checked here or skip-listed with a reason.  The
    engine times every launch under a name when profiling, so a kernel added later shows up here."""
    m = _engine(calib_sd)
    z, x = synthetic_inputs(32, 1)
    m.profile(True)
    try:
        _frame(m, z, x, np.array([[3, 4]]))
        names = {r[0] for r in m.profile_dump()}
    finally:
        m.profile(False)
    checked = set()
    for tap, _ in _tap_list("tensor", True, True, True):
        checked.add(tap.name)
        checked.update(k for k, _ in tap.keys)
        if tap.name == "refine":
            checked.add("refine_model.post2")
    missing = sorted(n for n in names if n not in checked and LAUNCH_TAP.get(n) not in checked and n not in SKIP)
    assert not missing, f"launches without a layer check or a skip reason: {missing}"


def _consts(B, R=25):
    a = torch.from_numpy(anc.generate_anchor(smb.DEFAULT_ANCHORS, R)).float().cuda()
    w = torch.from_numpy(anc.cosine_window(R, 5).astype(np.float32)).cuda()
    tsz = np.random.RandomState(B).rand(B, 2) * 60 + 30
    return a, w, torch.from_numpy(tsz)


def test_exact_255_b17_slot_table_step(calib_sd):
    """Two lanes (9 + 8), reverse M over several persistent tiles, xcorr slot indexing and the slot scatter."""
    B = 17
    m = _engine(calib_sd, max_batch=B, num_slots=B + 3)
    z, x = synthetic_inputs(33, B)
    rs = np.random.RandomState(0)
    t_slots = rs.permutation(B + 3)[:B]                        # template stream j -> slot t_slots[j]
    s_slots = t_slots[rs.permutation(B)]                       # step stream b reads slot s_slots[b]
    m.template(z.cuda(), slots=torch.from_numpy(t_slots.astype(np.int32)).cuda())
    a, w, tsz = _consts(B)
    out = m.step(x.cuda(), a, w, tsz, 0.04, 0.4, refine=True, mask_head=True,
                 slots=torch.from_numpy(s_slots.astype(np.int32)).cuda())
    torch.cuda.synchronize()
    pos = out["pos"].cpu().numpy()
    streams = (0, 8, 9, 16)
    row_of_slot = {int(s): j for j, s in enumerate(t_slots)}
    run = Run(m, z, x, streams, pos, {k: out[k] for k in ("cls", "loc", "mask", "refine")},
              kernel_rows=[row_of_slot[int(s_slots[b])] for b in streams])
    # template-side taps are in template stream order: check the same rows there
    _assert(*check("exact 255 B=17 slots", run, calib_sd, "exact"))


def test_exact_383_b1_far_edge(calib_sd):
    m = _engine(calib_sd, search_size=383)
    z, x = synthetic_inputs(34, 1, 383)
    pos = np.array([[40, 40]])
    _assert(*check("exact 383 B=1", Run(m, z, x, [0], pos, _frame(m, z, x, pos)), calib_sd, "exact"))


@pytest.mark.parametrize("B", [2, 17])
def test_fast(calib_sd, B):
    m = _engine(calib_sd, max_batch=B, precision="fast")
    z, x = synthetic_inputs(35, B)
    pos = np.array([[(5 * b) % 25, (11 * b + 3) % 25] for b in range(B)])
    streams = (0, 1) if B == 2 else (0, 8, 9, 16)
    run = Run(m, z, x, streams, pos, _frame(m, z, x, pos))
    _assert(*check(f"fast 255 B={B}", run, calib_sd, "fast"))


@pytest.mark.parametrize("log2_scale", [10, -10])
def test_exact_calibrated_scales(log2_scale):
    """Non-zero activation scales: the fused second conv at 2^(s_in - s_in2), identity diagonal != 1."""
    sd = calibrated_state_dict(0, log2_scale)
    m = _engine(sd)
    z, x = synthetic_inputs(36, 1)
    m.calibrate(z.cuda(), x.cuda())
    pos = np.array([[12, 7]])
    run = Run(m, z, x, [0], pos, _frame(m, z, x, pos), calibrated=True)
    _assert(*check(f"exact calib {log2_scale:+d}", run, sd, "exact"))


def test_exact_rpn_only(calib_sd):
    sd = {k: v for k, v in calib_sd.items() if not k.startswith(("mask_model.", "refine_model."))}
    m = _engine(sd, max_batch=2, mask=False)
    z, x = synthetic_inputs(37, 2)
    m.template(z.cuda())
    cls, loc = m.track(x.cuda())
    torch.cuda.synchronize()
    run = Run(m, z, x, (0, 1), np.zeros((2, 2), int), {"cls": cls, "loc": loc})
    _assert(*check("exact rpn B=2", run, sd, "exact", with_mask=False, refine=False))


def test_simt_b1(calib_sd):
    m = _engine(calib_sd, backend="simt")
    z, x = synthetic_inputs(38, 1)
    pos = np.array([[24, 0]])
    _assert(*check("simt B=1", Run(m, z, x, [0], pos, _frame(m, z, x, pos)), calib_sd, "exact", backend="simt"))


def adversarial_sd(sd):
    """calib_sd with BN gamma = 0 on a few channels (weight amax 0), gamma and beta of a backbone 1x1 conv and of a head
    scaled by 1e-6 (weights far below fp16's normal range at the per-channel exponent clamp), another layer's by 1e2,
    and one mask-head output column all zero.  With the 1e2 layer some tensors overflow fp16 at scale 0 while the
    1e-6 backbone layer sits near fp16's subnormal floor: calibrate() has to move their scales in opposite directions."""
    sd = {k: v.clone() for k, v in sd.items()}
    sd["features.features.layer2.1.bn2.weight"][:5] = 0
    sd["rpn_model.cls.head.1.weight"][7:9] = 0
    for k in ("features.features.layer2.2.bn1", "rpn_model.loc.head.1"):
        sd[k + ".weight"] *= 1e-6
        sd[k + ".bias"] *= 1e-6
    sd["features.features.layer3.1.bn2.weight"] *= 1e2
    sd["features.features.layer3.1.bn2.bias"] *= 1e2
    sd["mask_model.mask.head.3.weight"][100] = 0
    return sd


def test_exact_adversarial_checkpoint(calib_sd):
    sd = adversarial_sd(calib_sd)
    m = _engine(sd)
    z, x = synthetic_inputs(39, 1)
    m.calibrate(z.cuda(), x.cuda())
    pos = np.array([[6, 18]])
    run = Run(m, z, x, [0], pos, _frame(m, z, x, pos), calibrated=True)
    _assert(*check("exact adversarial", run, sd, "exact"))
