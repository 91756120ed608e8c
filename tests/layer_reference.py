"""Float64 restatement of the engine's layers, one op at a time, with a per-element error bound.  TEST SUPPORT ONLY.

Three parts:

* `wiring(...)`: for every tensor the engine records under a name (`Custom.export`), the op that produced it, the
  names of the tensors that feed it (the block input as residual or as the fused downsample input included) and the
  checkpoint keys and geometry.  Built by walking `oracle.siammask_oracle._LAYERS` the way `Oracle.features` /
  `Oracle.refine` do, not from the engine's layer table.
* `run(tap, inputs)`: the op in float64 on the CPU, returning `(ref, scale)`, where `scale` is the same op on absolute
  values (sum |x||w| + |shift| + |residual|).  It restates what the layer computes, not the kernel's arithmetic: BN is
  folded in float64 as the engine's `fold_affine` does, nothing is rounded.
* `ratio(got, ref, scale, gamma, rho, tau)`: the gate |got - ref| <= gamma * scale + rho * |ref| + tau per element.
  gamma covers operand quantisation and accumulation, rho the output's storage format, tau the fp16 subnormal floor.
  Because the bound is per element and scaled by that element's own terms, a low-magnitude channel, a ragged tile or
  one stream's rows in a shared tile count as much as the tensor's maximum.

The mutation helpers (`round_sig`, `drop_k_block`, ...) build what a plausible kernel defect would produce from the
same inputs; the GPU tests assert that each layer's gate rejects them.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

from oracle.siammask_oracle import BN_EPS, _LAYERS, nearest_upsample_index

BRANCHES = ("rpn_model.cls.", "rpn_model.loc.", "mask_model.mask.")
CORR = {"rpn_model.cls.": "corr_cls", "rpn_model.loc.": "corr_loc", "mask_model.mask.": "corr_mask"}
SEARCH_CAT = "heads.conv_search_cat"
HEAD_OUT = {"rpn_model.cls.": "cls", "rpn_model.loc.": "loc", "mask_model.mask.": "mask"}


@dataclass
class Tap:
    """One recorded tensor.  `inputs` name the tensors it reads ('x' / 'z': the API input; 'pos': refine positions)."""
    name: str
    op: str                      # conv | maxpool | crop_center | refine_crop | gather | deconv | small | xcorr
    inputs: tuple
    keys: tuple = ()             # conv: ((conv_key, bn_key or None), ...) concatenated along Cout
    stride: int = 1
    pad: int = 0
    dil: int = 1
    relu: bool = False
    second: tuple | None = None  # fused second conv: (conv_key, bn_key, stride, pad, dil), input = inputs[1]
    residual: bool = False       # inputs[-1] is added before the ReLU
    c_off: int = 0               # xcorr: channel offset into the (concatenated) search-side conv output
    geom: dict = field(default_factory=dict)   # crops / small convs: sizes


def fold(sd, conv_key, bn_key):
    """Folded weight (OIHW) and shift in float64: y = conv(x, w) + shift (engine.cu fold_affine)."""
    w = sd[conv_key + ".weight"].double()
    if bn_key is None:
        return w, sd[conv_key + ".bias"].double()
    eps = float(np.float32(BN_EPS))
    scale = sd[bn_key + ".weight"].double() / torch.sqrt(sd[bn_key + ".running_var"].double() + eps)
    shift = sd[bn_key + ".bias"].double() - sd[bn_key + ".running_mean"].double() * scale
    return w * scale.view(-1, 1, 1, 1), shift


# ---------------------------------------------------------------------------------------------------- wiring table
def backbone_taps(search: bool, backend: str = "tensor"):
    """ResNet.forward + ResDownS (Oracle.features / resdown).  Returns (taps, name of the backbone output)."""
    P = "features.features."
    taps = [Tap("stem", "conv", ("x" if search else "z",), ((P + "conv1", P + "bn1"),), 2, 0, 1, True),
            Tap("maxpool", "maxpool", ("stem",))]
    y = "maxpool"
    for name, planes, blocks, stride, dilation in _LAYERS:
        for i in range(blocks):
            p = f"{P}{name}.{i}."
            if i == 0:                                   # Oracle.features: the first block's dilation and downsample
                if stride == 1 and dilation == 1:
                    ds, d0 = (1, 1, 0), 1
                elif dilation > 1:
                    ds, d0 = (3, stride, dilation // 2), dilation // 2
                else:
                    ds, d0 = (3, stride, 0), 1
                s, d = stride, d0
            else:
                ds, s, d = None, 1, dilation
            pad = d if d > 1 else 2 - s                   # Oracle._bottleneck
            taps.append(Tap(p + "conv1", "conv", (y,), ((p + "conv1", p + "bn1"),), 1, 0, 1, True))
            taps.append(Tap(p + "conv2", "conv", (p + "conv1",), ((p + "conv2", p + "bn2"),), s, pad, d, True))
            c3 = ((p + "conv3", p + "bn3"),)
            if ds is None:
                taps.append(Tap(p + "conv3", "conv", (p + "conv2", y), c3, relu=True, residual=True))
            elif backend == "tensor":                    # conv3 and the downsample branch in one GEMM
                taps.append(Tap(p + "conv3", "conv", (p + "conv2", y), c3, relu=True,
                                second=(p + "downsample.0", p + "downsample.1", ds[1], ds[2], 1)))
            else:
                taps.append(Tap(p + "downsample.0", "conv", (y,), ((p + "downsample.0", p + "downsample.1"),),
                                ds[1], ds[2], 1, False))
                taps.append(Tap(p + "conv3", "conv", (p + "conv2", p + "downsample.0"), c3, relu=True, residual=True))
            y = p + "conv3"
    D = "features.downsample.downsample."
    taps.append(Tap(D + "0", "conv", (y,), ((D + "0", D + "1"),)))
    out = D + "0"
    if not search:                                       # ResDownS: x[:, :, 4:-4, 4:-4] when W < 20
        taps.append(Tap("crop_center", "crop_center", (out,)))
        out = "crop_center"
    return taps, out


def template_taps(backend="tensor", with_mask=True):
    """Template side, names without the 'template:' prefix."""
    taps, zf = backbone_taps(False, backend)
    for br in BRANCHES[:3 if with_mask else 2]:
        taps.append(Tap(br + "conv_kernel.0", "conv", (zf,), ((br + "conv_kernel.0", br + "conv_kernel.1"),),
                        relu=True))
    return taps


def search_taps(anchor_num=5, backend="tensor", with_mask=True, mask_head=True):
    """Search side of track / track_mask (all branches the engine runs when the mask features are requested)."""
    taps, xf = backbone_taps(True, backend)
    branches = BRANCHES[:3 if with_mask else 2]
    cat = backend == "tensor"
    if cat:
        taps.append(Tap(SEARCH_CAT, "conv", (xf,), tuple((b + "conv_search.0", b + "conv_search.1") for b in branches),
                        relu=True))
    for i, br in enumerate(branches):
        cs = SEARCH_CAT if cat else br + "conv_search.0"
        if not cat:
            taps.append(Tap(cs, "conv", (xf,), ((br + "conv_search.0", br + "conv_search.1"),), relu=True))
        taps.append(Tap(CORR[br], "xcorr", (cs, "template:" + br + "conv_kernel.0"), c_off=256 * i if cat else 0))
        if br == "mask_model.mask." and not mask_head:
            continue
        taps.append(Tap(br + "head.0", "conv", (CORR[br],), ((br + "head.0", br + "head.1"),), relu=True))
        taps.append(Tap(HEAD_OUT[br], "conv", (br + "head.0",), ((br + "head.3", None),)))
    return taps


def refine_taps():
    """Refine.forward(test=True) as Oracle.refine restates it; 'post2' is the API output of track_refine."""
    R = "refine_model."
    src = {"p0": "features.features.conv1", "p1": "features.features.layer1.2.conv3",
           "p2": "features.features.layer2.3.conv3"}
    taps = []
    for lvl, (scale, pad, size) in {"p0": (4, 16, 61), "p1": (2, 8, 31), "p2": (1, 4, 15)}.items():
        taps.append(Tap("refine:crop_" + lvl, "refine_crop", (src[lvl] if lvl != "p0" else "stem", "pos"),
                        geom=dict(scale=scale, pad=pad, size=size)))
    taps.append(Tap("refine:p3", "gather", ("corr_mask", "pos")))
    taps.append(Tap("refine:deconv", "deconv", ("refine:p3",)))

    def c3(name, inp, relu=True, other=None, out=None):
        ins = (inp,) if other is None else (inp, other)
        taps.append(Tap(R + name if out is None else out, "small", ins, ((R + name, None),), 1, 1, 1, relu,
                        geom=dict(up=0)))
    c3("v2.0", "refine:crop_p2"); c3("v2.2", R + "v2.0")
    c3("v1.0", "refine:crop_p1"); c3("v1.2", R + "v1.0")
    c3("v0.0", "refine:crop_p0"); c3("v0.2", R + "v0.0")
    c3("h2.0", "refine:deconv"); c3("h2.2", R + "h2.0")
    c3("post0", R + "h2.2", False, R + "v2.2")
    taps[-1].geom = dict(up=31)
    c3("h1.0", R + "post0"); c3("h1.2", R + "h1.0")
    c3("post1", R + "h1.2", False, R + "v1.2")
    taps[-1].geom = dict(up=61)
    c3("h0.0", R + "post1"); c3("h0.2", R + "h0.0")
    c3("post2", R + "h0.2", False, R + "v0.2", out="refine")
    taps[-1].geom = dict(up=127)
    return taps


# ---------------------------------------------------------------------------------------------------- the ops
def _conv_terms(sd, tap, x, x2=None, res=None, w_mut=None, w2_mut=None):
    """(ref, scale) of conv [+ second conv] + shift [+ residual], before the ReLU.  w_mut(w) mutates the weights of the
    first conv, w2_mut those of the fused second conv."""
    ws, shifts = zip(*(fold(sd, c, b) for c, b in tap.keys))
    w, shift = torch.cat(ws, 0), torch.cat(shifts, 0)
    if w_mut is not None:
        w = w_mut(w)
    ref = F.conv2d(x, w, None, tap.stride, tap.pad, tap.dil)
    scale = F.conv2d(x.abs(), w.abs(), None, tap.stride, tap.pad, tap.dil)
    if tap.second is not None:
        c, b, s, p, d = tap.second
        w2, sh2 = fold(sd, c, b)
        if w2_mut is not None:
            w2 = w2_mut(w2)
        ref = ref + F.conv2d(x2, w2, None, s, p, d)
        scale = scale + F.conv2d(x2.abs(), w2.abs(), None, s, p, d)
        shift = shift + sh2
    ref = ref + shift.view(1, -1, 1, 1)
    scale = scale + shift.abs().view(1, -1, 1, 1)
    if res is not None:
        ref = ref + res
        scale = scale + res.abs()
    return ref, scale


def refine_crop(f, pos, scale, pad, size):
    """pad(f, pad)[:, :, scale*dy : scale*dy + size, scale*dx : ...] per stream (Oracle.refine, custom.py:133-135)."""
    out = []
    for b in range(f.shape[0]):
        dy, dx = int(pos[b][0]), int(pos[b][1])
        out.append(F.pad(f[b:b + 1], [pad] * 4)[:, :, scale * dy:scale * dy + size, scale * dx:scale * dx + size])
    return torch.cat(out, 0)


def nearest_up(t, size):
    """F.interpolate(size=(size, size)) through the oracle's index table."""
    idx = torch.from_numpy(nearest_upsample_index(size, t.shape[-1]))
    return t[:, :, idx][:, :, :, idx]


def xcorr(x, k):
    """Depthwise valid cross-correlation (conv2d_dw_group, rpn.py:32-38), paired batch."""
    b, c = k.shape[:2]
    out = F.conv2d(x.reshape(1, b * c, *x.shape[2:]), k.reshape(b * c, 1, *k.shape[2:]), groups=b * c)
    return out.view(b, c, *out.shape[2:])


def run(sd, tap, ins, w_mut=None, k_mut=None, w2_mut=None):
    """Float64 reference of one tap: (ref, scale) with the op's own output nonlinearity applied to ref.
    ins: name -> tensor (float64 NCHW; 'pos': int array [B,2]).  Exact ops return scale None."""
    a = [ins[n] for n in tap.inputs]
    if tap.op == "conv":
        x2 = a[1] if tap.second is not None else None
        res = a[-1] if tap.residual else None
        ref, scale = _conv_terms(sd, tap, a[0], x2, res, w_mut, w2_mut)
    elif tap.op == "small":
        # conv3x3(nearest_up(a (+ b))) + bias: the add happens in fp32 before the conv, so scale takes |a| + |b|
        x = a[0] if len(a) == 1 else a[0] + a[1]
        xs = a[0].abs() if len(a) == 1 else a[0].abs() + a[1].abs()
        if tap.geom.get("up"):
            x, xs = nearest_up(x, tap.geom["up"]), nearest_up(xs, tap.geom["up"])
        ref, _ = _conv_terms(sd, tap, x, w_mut=w_mut)
        _, scale = _conv_terms(sd, tap, xs, w_mut=w_mut)
    elif tap.op == "deconv":
        w = sd["refine_model.deconv.weight"].double()
        b = sd["refine_model.deconv.bias"].double()
        if w_mut is not None:
            w = w_mut(w)
        p3 = a[0].reshape(-1, 256, 1, 1)
        ref = F.conv_transpose2d(p3, w, b, 15)
        scale = F.conv_transpose2d(p3.abs(), w.abs(), b.abs(), 15)
    elif tap.op == "xcorr":
        x = a[0][:, tap.c_off:tap.c_off + 256]
        k = a[1] if k_mut is None else k_mut(a[1])
        if w_mut is not None:
            x = w_mut(x)
        ref, scale = xcorr(x, k), xcorr(x.abs(), k.abs())
        return ref, scale
    elif tap.op == "maxpool":
        return F.max_pool2d(a[0], 3, 2, 1), None
    elif tap.op == "crop_center":
        return a[0][:, :, 4:-4, 4:-4], None
    elif tap.op == "refine_crop":
        return refine_crop(a[0], a[1], **tap.geom), None
    elif tap.op == "gather":
        pos = a[1]
        return torch.stack([a[0][b, :, int(pos[b][0]), int(pos[b][1])] for b in range(a[0].shape[0])])\
            .reshape(-1, 256, 1, 1), None
    else:
        raise ValueError(tap.op)
    if tap.relu:
        ref = ref.relu()
    return ref, scale


# ---------------------------------------------------------------------------------------------------- the gate
# refine convs the engine runs on the fp32 small_conv3x3 kernels (Cin not a multiple of 64; upsample maps, two operands)
SMALL_SIMT = {"refine_model." + k for k in ("v0.2", "h2.0", "h2.2", "h1.0", "h1.2", "h0.0", "h0.2", "post0", "post1")} | {
    "refine"}
F32_OUT = SMALL_SIMT | {"refine_model.v2.2", "refine_model.v1.2", "refine_model.v0.0", "refine:deconv", "refine:p3",
                        "cls", "loc", "mask"}


def family(tap, backend="tensor"):
    """Which kernel family computes the tap: 'gemm' (tensor-core conv, patch conv, stem), 'simt' (fp32 CUDA-core convs,
    deconv), 'xcorr', or 'exact' (copies: must match bit for bit)."""
    if tap.op in ("maxpool", "crop_center", "refine_crop", "gather"):
        return "exact"
    if tap.op == "xcorr":
        return "xcorr"
    if tap.op == "deconv" or backend != "tensor" or tap.name in SMALL_SIMT:
        return "simt"
    return "gemm"


def out_format(tap, precision):
    """Storage of the tap's output: 'f32', 'split' (exact mode hi + lo) or 'hi' (fast mode, fp16 only)."""
    if tap.name in F32_OUT:
        return "f32"
    return "split" if precision == "exact" else "hi"


def evaluate(sd, tap, fetch, **mut):
    """run() with the tap's inputs taken from fetch(name) (float64 NCHW) and 'pos' from fetch('pos')."""
    return run(sd, tap, {n: fetch(n) for n in tap.inputs}, **mut)


def ratio(got, ref, scale, gamma, rho, tau):
    """(measured gamma, gate use): the worst (|got - ref| - rho|ref| - tau) / scale over the elements, i.e. the error
    left for the gamma term in units of each element's own scale, and that number over gamma.  The gate holds when the
    gate use is <= 1."""
    got, ref = got.double().reshape(ref.shape), ref.double()
    excess = ((got - ref).abs() - rho * ref.abs() - tau) / scale.clamp_min(1e-300)
    worst = float(excess.max())
    return worst, worst / gamma


def tau_for(peak, fmt, calibrated):
    """Subnormal floor of the output's storage: fp16 planes hold value * 2^s, so one fp16 subnormal step is 2^-24 * 2^-s.
    Uncalibrated, s = 0.  After calibrate() every tensor's stored maximum lies in [2^8, 2^12], so 2^-s <= peak / 2^8,
    where peak is the tensor's max |value| over everything that shares its scale (template and search side of a
    backbone layer).  fp32 outputs: none."""
    if fmt == "f32":
        return 1e-30
    return 2.0 ** -24 * (peak / 256.0 if calibrated else 1.0)


# ---------------------------------------------------------------------------------------------------- launch shapes
def _patch_ro(w):
    """conv3x3_patch_sm90.cu patch_pw / patch_ro: image rows per 128-pixel tile (0: the geometry is not supported)."""
    pw = (w + 1 + 7) // 8 * 8
    return 128 // pw if pw <= 64 and 128 % pw == 0 else 0


def _cout_pad(cout):
    """conv_gemm_sm90.cu gemm_cout_pad."""
    for p in (16, 32, 64, 128):
        if cout <= p:
            return p
    return (cout + 255) // 256 * 256


def launches(search_size, B, max_batch=None, with_mask=True, refine=True):
    """Every tensor-core conv, stem and engine-xcorr launch of one template + track_mask + track_refine at batch B on
    the tensor backend, as dicts (side, name, kernel, lane, M, tiles, s0, hw, ho, ntile).  Template launches run once
    over all B streams; search-side and refine launches run once per lane on that lane's streams (schedule.lane_split).
    M is the launch's output rows (streams x Ho x Wo); tiles counts the persistent kernels' work items (GEMM / stem:
    128-row M tiles x N tiles; patch conv: RO-row blocks per image; xcorr: its blocks of 32 channels x row band per
    stream).  s0 is the lane's first stream, hw = ho * ho the output rows per stream, ntile the GEMM's N tiles (the
    patch conv's row blocks per image)."""
    from siammask_b200.checkpoint import expected_keys
    from siammask_b200.schedule import lane_split

    shapes = expected_keys(with_mask, refine)
    sides = [("template", template_taps("tensor", with_mask), [B])]
    lanes = lane_split(B, max_batch or B)
    sides.append(("search", search_taps(backend="tensor", with_mask=with_mask, mask_head=with_mask), lanes))
    if refine:
        sides.append(("refine", refine_taps(), lanes))
    out, size = [], {}
    for side, taps, chunks in sides:
        if side != "refine":                                   # refine reads the search side's tensors
            size = {"x": search_size, "z": 127}
        for t in taps:
            h = size[t.inputs[0]]
            kernel = None
            if t.op in ("conv", "small"):
                co = sum(shapes[k + ".weight"][0] for k, _ in t.keys)
                _, ci, kh, kw = shapes[t.keys[0][0] + ".weight"]
                if t.op == "small":
                    h = t.geom["up"] or h
                ho = (h + 2 * t.pad - t.dil * (kh - 1) - 1) // t.stride + 1
                if family(t) == "gemm":
                    if t.name == "stem":
                        kernel, ntile = "stem", 1
                    elif (kh == kw == 3 and t.stride == 1 and t.pad == 1 and t.dil == 1 and ci == co in (64, 128)
                          and t.second is None and not t.residual and t.name not in F32_OUT and _patch_ro(h)):
                        kernel = "patch"
                    else:
                        kernel, ntile = "gemm", _cout_pad(co) // min(_cout_pad(co), 128)
            elif t.op == "maxpool":
                ho = (h + 2 - 3) // 2 + 1
            elif t.op == "crop_center":
                ho = h - 8
            elif t.op == "xcorr":
                ho, kernel = h - 4, "xcorr"
                bands = 1
                while (-(-ho // bands) + 4) * h * 32 * 4 > 160 * 1024:        # launch_xcorr_nhwc's row bands
                    bands += 1
            elif t.op == "refine_crop":
                ho = t.geom["size"]
            elif t.op == "gather":
                ho = 1
            else:                                                           # deconv
                ho = 15
            size[t.name] = ho
            if kernel is None:
                continue
            if kernel == "patch":
                ntile = -(-ho // _patch_ro(ho))
            elif kernel == "xcorr":
                ntile = 8 * bands
            s0 = 0
            for lane, b in enumerate(chunks):
                M = b * ho * ho
                tiles = b * ntile if kernel in ("patch", "xcorr") else -(-M // 128) * ntile
                out.append(dict(side=side, name=t.name, kernel=kernel, lane=lane, M=M, tiles=tiles, s0=s0,
                                hw=ho * ho, ho=ho, ntile=ntile))
                s0 += b
    return out


def tile_classes(launch, num_sms=132):
    """The ragged-tile classes a launch exercises: 'a' when its last 128-row tile ends in the first warpgroup's 64 rows
    (the second consumer warpgroup has no row to store), 'b' when it ends in the second's, 'c' when there are more
    tiles than SMs (persistent CTAs take a second tile), 'd' when there are more than two tiles per CTA of the
    persistent grid, min(tiles, num_sms) (conv_gemm_sm90.cu launch_cfg, stem_sm90.cu, conv3x3_patch_sm90.cu
    launch_patch): only from the third tile on do the producer's stage ring and the mbarrier phase parities, the
    epilogue's per-warpgroup staging buffers and the patch conv's cross-tile patch prefetch come back round to the state
    they started from.  The xcorr is not persistent: one block per work item, nothing carried from one to the next, so
    it has no (d); its (c) means a second wave of blocks."""
    r, cls = launch["M"] % 128, set()
    if 0 < r <= 64:
        cls.add("a")
    elif r > 64:
        cls.add("b")
    if launch["tiles"] > num_sms:
        cls.add("c")
        if launch.get("kernel") != "xcorr" and launch["tiles"] > 2 * num_sms:
            cls.add("d")
    return cls


def work_rows(launch, t, reverse_m=False):
    """Output rows [r0, r1) of the launch (lane-local) that work item t computes.  GEMM / stem: M block t // ntile,
    counted from the end with reverse_m (conv_gemm_sm90.cu m_block); patch conv: image t // ntile, its RO-row block
    t % ntile (conv3x3_patch_sm90.cu)."""
    M, hw, ho = launch["M"], launch["hw"], launch["ho"]
    if launch["kernel"] == "patch":
        b, blk = divmod(t, launch["ntile"])
        ro = _patch_ro(ho)
        return b * hw + blk * ro * ho, b * hw + min(ho, (blk + 1) * ro) * ho
    mb = t // launch["ntile"]
    if reverse_m:
        mb = -(-M // 128) - 1 - mb
    return mb * 128, min(M, (mb + 1) * 128)


def rows_streams(launch, r0, r1):
    """The streams (global index) holding the lane-local output rows [r0, r1)."""
    return set(range(launch["s0"] + r0 // launch["hw"], launch["s0"] + (r1 - 1) // launch["hw"] + 1))


def last_tile_streams(launch):
    """The streams holding rows of the launch's last 128-row M tile (the ragged one, wherever a CTA meets it)."""
    return rows_streams(launch, (-(-launch["M"] // 128) - 1) * 128, launch["M"])


def pass_streams(launch, num_sms=132):
    """The streams holding the first rows of the work items a persistent CTA takes on its second and third pass (work
    items grid and 2 grid, grid = min(tiles, num_sms)), for the GEMM in both M orders: the engine picks reverse_m per
    launch from where the layer's biggest input was last written (engine.cu conv_into, last_end_), which is keyed by
    buffer address and so depends on the calls an engine ran before.  The xcorr has no passes."""
    if launch["kernel"] == "xcorr":
        return set()
    grid, out = min(launch["tiles"], num_sms), set()
    for t in (grid, 2 * grid):
        if t < launch["tiles"]:
            for rev in ((False, True) if launch["kernel"] == "gemm" else (False,)):
                r0 = work_rows(launch, t, rev)[0]
                out |= rows_streams(launch, r0, r0 + 1)
    return out


# ---------------------------------------------------------------------------------------------------- mutations
def round_sig(t, bits=11):
    """Round the significand to `bits` significant bits, round-to-nearest-even, no exponent range (nothing is flushed):
    what dropping the lo plane of a hi+lo pair leaves.  The error is at most 2^-bits relative."""
    t = t.double()
    m, e = torch.frexp(t)                       # t = m * 2^e, 0.5 <= |m| < 1
    return torch.ldexp(torch.round(torch.ldexp(m, torch.full_like(e, bits))), e - bits)


def drop_k_block(w, tap_yx=(0, 0), c0=0, width=64):
    """Weights (OIHW) with one `width`-channel k-block of one kernel tap missing: a skipped K tile."""
    w = w.clone()
    ky, kx = min(tap_yx[0], w.shape[2] - 1), min(tap_yx[1], w.shape[3] - 1)
    w[:, c0:c0 + width, ky, kx] = 0
    return w


def drop_xcorr_tap(k, u=2, v=2):
    """Template kernel with one of its 5 x 5 taps missing."""
    k = k.clone()
    k[:, :, u, v] = 0
    return k
