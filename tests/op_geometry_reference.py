"""Float64 references, error gates, route rule and case list of the standalone operators `smb.conv2d` and
`smb.conv2d_dw_group`.  TEST SUPPORT ONLY.

* `conv_ref` / `xcorr_ref`: the op in float64 on the CPU, with `scale` = the same op on absolute values.
* Gates, per element, through `layer_reference.ratio`:
  - conv: |got - ref| <= gamma * sum|x||w| (+ |shift|) + rho * |ref|.  gamma is the family gamma of
    test_gpu_layers.GAMMA (tensor routes: 'gemm', SIMT: 'simt'), measured up to the engine's largest reduction,
    K = 4864.  Beyond it gamma grows linearly with K: the accumulation error of a K-term dot product is bounded by
    gamma_K * sum|x||w| with gamma_K = K u / (1 - K u) (Higham, Accuracy and Stability, Thm. 3.1), linear in K, and
    the operand quantisation part does not grow with K, so scaling the whole gamma by K / 4864 over-covers both.
    rho is the output's storage: the patch route stores fp16 split planes (exact) or the hi plane (fast) and
    re-expands them, every other route writes fp32.
  - xcorr: every output is a sequence of kh*kw fp32 FMAs starting from 0, so |got - ref| <= gamma_n * sum|x||k| with
    gamma_n = n u / (1 - n u), n = kh*kw, u = 2^-24.
* `conv_route` / `xcorr_route`: which kernel the operators run (conv: pinned to the library's `sm_conv2d_route` by
  test_op_geometry_host.py).
* `CONV_CASES` / `XCORR_CASES`: a fixed case list, and `conv_classes` / `xcorr_classes`, the geometry classes each
  case exercises (the host test asserts every route meets every class it can).
* Mutations: what a plausible kernel defect would return, computed in float64 from the same inputs.
"""
from __future__ import annotations

from collections import namedtuple

import torch
import torch.nn.functional as F

import layer_reference as lr
from test_gpu_layers import GAMMA, RHO

K_ENGINE_MAX = 4864                 # the engine's largest conv reduction (layer3.0.conv3 + its downsample)
NUM_SMS = 132                       # H100 SXM
U32 = 2.0 ** -24

Conv = namedtuple("Conv", "B Cin H W Cout KH KW stride pad dil backend")
Xcorr = namedtuple("Xcorr", "B C H W kh kw")


def out_size(n, k, stride, pad, dil):
    return (n + 2 * pad - dil * (k - 1) - 1) // stride + 1


def out_hw(c):
    return out_size(c.H, c.KH, c.stride, c.pad, c.dil), out_size(c.W, c.KW, c.stride, c.pad, c.dil)


# ---------------------------------------------------------------------------------------------------- route rules
PRECISIONS = ("exact", "fast")


def patch_smem(W, cm, precision):
    """conv3x3_patch_sm90.cu patch_smem_bytes: two patch buffers of (RO+2) x PW pixel rows plus 2 x 8 slack rows of
    128 bytes per plane, a 3-stage weight ring, barriers and alignment slack."""
    nsplit = 2 if precision == "exact" else 1
    pw = (W + 8) // 8 * 8
    panel = ((lr._patch_ro(W) + 2) * pw + 16) * 128
    return 2 * nsplit * panel + 3 * nsplit * cm * 128 + 256 + 1024


def patch_ok(W, cm=64, precision="exact"):
    """conv3x3_patch_sm90.cu: a square image of width W with cm channels fits the resident-patch kernel."""
    return lr._patch_ro(W) > 0 and patch_smem(W, cm, precision) <= 227 * 1024


def conv_route(c: Conv, precision="exact") -> str:
    """engine.cu conv2d_route for an accepted geometry: 'simt', 'patch', 'gemm_tiled' (mode 0) or 'gemm_im2col'."""
    if c.backend == "simt":
        return "simt"
    if (c.KH == c.KW == 3 and c.stride == 1 and c.pad == 1 and c.dil == 1 and c.Cin == c.Cout in (64, 128)
            and c.H == c.W and patch_ok(c.W, c.Cin, precision)):
        return "patch"
    if c.KH == c.KW == 1 and c.stride == 1 and c.pad == 0:
        return "gemm_tiled"
    return "gemm_im2col"


def conv_accepts(c: Conv) -> bool:
    """The arguments sm_conv2d accepts (engine.cu conv2d_route)."""
    if min(c.B, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, c.stride, c.dil) < 1 or c.pad < 0:
        return False
    Ho, Wo = out_hw(c)
    if Ho < 1 or Wo < 1 or max(c.B * c.Cin * c.H * c.W, c.Cout * c.Cin * c.KH * c.KW, c.B * c.Cout * Ho * Wo) >= 2 ** 31:
        return False
    if c.backend == "simt":
        return True
    if c.Cin % 64:
        return False
    if conv_route(c) != "gemm_im2col":
        return True
    ups = (c.pad - (c.KW - 1) * c.dil, c.pad - (c.KH - 1) * c.dil)
    return c.stride <= 8 and c.pad <= 128 and all(-128 <= u <= 127 for u in ups)


def block_k(precision, cout):
    """conv_gemm_sm90.cu Cfg::BLOCK_K: 32-wide k-blocks only in exact mode at a 128-wide N tile."""
    return 32 if precision == "exact" and lr._cout_pad(cout) >= 128 else 64


def tiles_and_tail(c: Conv, precision):
    """(work tiles of the persistent kernel, rows of its last 128-row tile) for the tensor routes."""
    Ho, Wo = out_hw(c)
    if conv_route(c, precision) == "patch":
        ro, pw = lr._patch_ro(c.W), (c.W + 8) // 8 * 8
        per_img = -(-c.H // ro)
        return c.B * per_img, (c.H - (per_img - 1) * ro) * pw
    pad = lr._cout_pad(c.Cout)
    M = c.B * Ho * Wo
    return -(-M // 128) * (pad // min(pad, 128)), M - (M - 1) // 128 * 128


XCORR_TILE = {29: 32, 45: 8}        # xcorr_bulk.cu: planes per pipeline stage at 29 x 29 and 45 x 45


def xcorr_route(x: Xcorr):
    """sm_xcorr_depthwise on 16-byte aligned tensors: (planes on the bulk pipeline, kernel of the rest: 'one_warp',
    'generic' or None)."""
    planes = x.B * x.C
    bulk = 0
    if x.kh == x.kw == 5 and x.H == x.W and x.H in XCORR_TILE:
        bulk = planes // XCORR_TILE[x.H] * XCORR_TILE[x.H]
    rest = None if bulk == planes else ("one_warp" if x.kh == x.kw == 5 else "generic")
    return bulk, rest


# ---------------------------------------------------------------------------------------------------- case lists
def _t(B, Cin, H, W, Cout, K, stride=1, pad=0, dil=1):
    KH, KW = (K, K) if isinstance(K, int) else K
    return Conv(B, Cin, H, W, Cout, KH, KW, stride, pad, dil, "tensor")


def _s(B, Cin, H, W, Cout, K, stride=1, pad=0, dil=1):
    return _t(B, Cin, H, W, Cout, K, stride, pad, dil)._replace(backend="simt")


CONV_CASES = [
    # wgmma GEMM, 2-D tiled operands (1x1, stride 1, pad 0)
    _t(1, 64, 5, 40, 48, 1),                     # H != W, last tile 72 rows (b)
    _t(3, 64, 1, 1, 8, 1),                       # 1 x 1 image
    _t(1, 192, 7, 9, 100, 1),                    # 3 k-blocks
    _t(1, 64, 131, 131, 64, 1),                  # 135 tiles
    _t(2, 128, 11, 13, 3969, 1),                 # 16 N tiles, the last ragged
    _t(1, 5120, 3, 5, 16, 1),                    # K 5120 > the engine's largest
    # wgmma GEMM, im2col operands
    _t(2, 64, 9, 23, 32, 3, 1, 1),               # H != W
    _t(1, 64, 11, 17, 40, (1, 5), 1, 2),         # KH != KW, pad beyond the kernel's reach on H
    _t(2, 64, 17, 12, 48, 3, 2, 1),
    _t(1, 64, 20, 17, 40, 3, 3, 1),
    _t(2, 64, 13, 19, 24, 1, 4, 0),              # strided 1x1
    _t(1, 64, 23, 31, 16, (2, 3), 5, 1),
    _t(1, 128, 25, 14, 20, 3, 6, 2, 2),
    _t(2, 64, 30, 22, 12, 5, 7, 2),
    _t(1, 64, 33, 41, 32, 7, 8, 3),
    _t(2, 64, 15, 21, 64, 3, 1, 2, 2),           # Cin == Cout, dilated: not the patch kernel
    _t(1, 64, 16, 16, 17, 3, 1, 3, 3),
    _t(1, 64, 13, 21, 33, 3, 1, 0, 4),
    _t(1, 64, 6, 9, 8, 3, 1, 3),                 # output larger than the input
    _t(2, 64, 5, 7, 16, 1, 1, 2),                # padded 1x1
    _t(1, 64, 4, 4, 8, 3, 2, 4, 2),
    _t(3, 64, 3, 9, 24, 3, 1, 0),                # Ho = 1
    _t(2, 64, 1, 1, 8, 3, 1, 1),                 # 1 x 1 image, 3x3 pad 1
    _t(1, 192, 9, 13, 40, 3, 1, 1),              # 27 k-blocks
    _t(1, 576, 6, 5, 24, 3, 1, 1),               # K 5184 > the engine's largest
    _t(1, 64, 12, 11, 130, 3, 1, 1),             # two N tiles, exact mode's 32-wide k-blocks
    _t(2, 64, 186, 185, 64, 1, 2, 0),            # 136 tiles, H != W
    # resident-patch 3x3 (square W in {1..15, 24..31, 56..63}, Cin == Cout in {64, 128})
    _t(1, 64, 1, 1, 64, 3, 1, 1),                # PW 8
    _t(2, 128, 5, 5, 128, 3, 1, 1),
    _t(133, 64, 7, 7, 64, 3, 1, 1),              # 133 tiles of one image each
    _t(1, 64, 8, 8, 64, 3, 1, 1),                # PW 16: W = PW - 8
    _t(2, 128, 12, 12, 128, 3, 1, 1),
    _t(1, 64, 24, 24, 64, 3, 1, 1),              # PW 32: W = PW - 8
    _t(1, 128, 27, 27, 128, 3, 1, 1),
    _t(1, 64, 56, 56, 64, 3, 1, 1),              # PW 64: W = PW - 8
    _t(1, 64, 57, 57, 64, 3, 1, 1),
    _t(1, 128, 60, 60, 128, 3, 1, 1),            # fast mode only: exact mode's patch buffers exceed shared memory
    # SIMT reference conv (any Cin)
    _s(1, 16, 9, 13, 8, 3, 1, 1),
    _s(1, 8, 12, 7, 4, (2, 5), 2, 2),
    _s(1, 4, 20, 23, 3, 3, 3, 1),
    _s(1, 4, 17, 9, 5, 1, 4, 0),
    _s(1, 3, 23, 31, 2, (2, 3), 5, 1),
    _s(1, 4, 25, 14, 3, 3, 6, 2, 2),
    _s(1, 2, 30, 22, 3, 5, 7, 2),
    _s(1, 3, 33, 41, 4, 7, 8, 3),
    _s(1, 4, 16, 16, 5, 3, 1, 3, 3),
    _s(1, 4, 13, 21, 6, 3, 1, 0, 4),
    _s(2, 5, 1, 1, 3, 3, 1, 1),
]

XCORR_CASES = [
    # 29 x 29 (search 255): 32 planes per bulk stage, the rest one warp per plane
    Xcorr(1, 31, 29, 29, 5, 5), Xcorr(1, 32, 29, 29, 5, 5), Xcorr(1, 33, 29, 29, 5, 5),
    Xcorr(3, 21, 29, 29, 5, 5), Xcorr(2, 32, 29, 29, 5, 5), Xcorr(5, 13, 29, 29, 5, 5),
    # 45 x 45 (search 383): 8 planes per bulk stage
    Xcorr(1, 7, 45, 45, 5, 5), Xcorr(1, 8, 45, 45, 5, 5), Xcorr(3, 3, 45, 45, 5, 5),
    Xcorr(1, 15, 45, 45, 5, 5), Xcorr(2, 8, 45, 45, 5, 5), Xcorr(1, 17, 45, 45, 5, 5),
    # one warp per plane: 28 output columns per pass, 32 (H <= 32) or 24 rows per load batch
    Xcorr(2, 3, 31, 31, 5, 5), Xcorr(1, 4, 32, 32, 5, 5), Xcorr(1, 5, 33, 33, 5, 5),
    Xcorr(1, 3, 9, 61, 5, 5), Xcorr(2, 2, 40, 7, 5, 5), Xcorr(1, 2, 5, 5, 5, 5),
    # generic kernel (kh, kw != 5 x 5)
    Xcorr(2, 3, 12, 17, 3, 7), Xcorr(1, 4, 7, 7, 7, 7), Xcorr(1, 2, 6, 9, 1, 1), Xcorr(3, 2, 10, 4, 6, 2),
]


# ---------------------------------------------------------------------------------------------------- classes
def conv_classes(c: Conv, precision="exact"):
    """The geometry classes a conv case exercises in one precision mode."""
    Ho, Wo = out_hw(c)
    cls = {f"stride{c.stride}"}
    if c.H != c.W:
        cls.add("h_ne_w")
    if c.KH != c.KW:
        cls.add("kh_ne_kw")
    if max(c.KH, c.KW) > 1:
        cls.add(f"dil{c.dil}")
    if 2 * c.pad > (c.KH - 1) * c.dil or 2 * c.pad > (c.KW - 1) * c.dil:
        cls.add("pad_gt_half")
    if Ho == 1 or Wo == 1:
        cls.add("out1")
    route = conv_route(c, precision)
    if route == "simt":
        return cls
    if (c.Cin // block_k("fast", c.Cout)) % 2:
        cls.add("cin_kb_odd")
    tiles, tail = tiles_and_tail(c, precision)
    cls |= {"tail_a"} if tail <= 64 else {"tail_b"} if tail < 128 else set()
    if tiles > NUM_SMS:
        cls.add("tiles_c")
    if route == "patch":
        pw = (c.W + 8) // 8 * 8
        cls.add(f"pw{pw}")
        if c.W == pw - 8:
            cls.add("w_pw_minus_8")
    return cls


CONV_CLASSES = ({"h_ne_w", "kh_ne_kw", "pad_gt_half", "out1", "cin_kb_odd", "tail_a", "tail_b", "tiles_c"}
                | {f"stride{s}" for s in range(1, 9)} | {f"dil{d}" for d in range(1, 5)})
PATCH_CLASSES = {"pw8", "pw16", "pw32", "pw64", "w_pw_minus_8"}
# (route, class) pairs no accepted geometry has, and why
_FIXED_PATCH = {"h_ne_w", "kh_ne_kw", "pad_gt_half"} | {f"stride{s}" for s in range(2, 9)} | {
    f"dil{d}" for d in range(2, 5)}
_FIXED_TILED = {"kh_ne_kw", "pad_gt_half"} | {f"stride{s}" for s in range(2, 9)} | {f"dil{d}" for d in range(1, 5)}
NOT_APPLICABLE = {
    **{("patch", k): "the patch kernel takes square 3x3 / stride 1 / pad 1 / dilation 1 only" for k in _FIXED_PATCH},
    **{("gemm_tiled", k): "the tiled path is 1x1 / stride 1 / pad 0: no taps to dilate or pad" for k in _FIXED_TILED},
    **{("simt", k): "one thread per output element: no tiles and no k-blocks"
       for k in ("cin_kb_odd", "tail_a", "tail_b", "tiles_c")},
}


def xcorr_classes(x: Xcorr):
    bulk, rest = xcorr_route(x)
    cls = set()
    if x.H in XCORR_TILE and x.H == x.W and x.kh == x.kw == 5:
        t, planes = XCORR_TILE[x.H], x.B * x.C
        for d in (-1, 0, 1):
            if planes % t == (d % t) and planes >= t + d:
                cls.add(f"{x.H}:{'tile' + ('%+d' % d if d else '')}")
        if planes > 2 * t:
            cls.add(f"{x.H}:tiles>2")
    if rest == "one_warp":
        if x.W - 4 in (27, 28, 29):                      # around one 28-column pass
            cls.add(f"wo{x.W - 4}")
        if x.W - 4 > 28:
            cls.add("one_warp:multi_pass")
        cls.add("one_warp:rb32" if x.H <= 32 else "one_warp:rb24")
    if rest == "generic":
        cls.add("generic")
    if x.H != x.W:
        cls.add(f"{rest}:h_ne_w")
    if x.kh != x.kw:
        cls.add("kh_ne_kw")
    return cls


XCORR_REQUIRED = ({f"{h}:{t}" for h in XCORR_TILE for t in ("tile-1", "tile", "tile+1", "tiles>2")}
                  | {"wo27", "wo28", "wo29", "one_warp:multi_pass", "one_warp:rb32", "one_warp:rb24",
                     "one_warp:h_ne_w", "generic", "generic:h_ne_w", "kh_ne_kw"})


# ---------------------------------------------------------------------------------------------------- data
def conv_inputs(c: Conv, seed):
    """Deterministic x, w, scale, shift for a case: He-scaled weights, per-channel affine."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c.B, c.Cin, c.H, c.W, generator=g)
    w = torch.randn(c.Cout, c.Cin, c.KH, c.KW, generator=g) * (2.0 / (c.Cin * c.KH * c.KW)) ** 0.5
    sc = torch.rand(c.Cout, generator=g) + 0.5
    sh = torch.randn(c.Cout, generator=g) * 0.1
    return x, w, sc, sh


def xcorr_inputs(x: Xcorr, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(x.B, x.C, x.H, x.W, generator=g), torch.randn(x.B, x.C, x.kh, x.kw, generator=g)


# ---------------------------------------------------------------------------------------------------- references
def folded(w, sc):
    return w.double() * sc.double().view(-1, 1, 1, 1)


def conv_ref(c: Conv, x, wf, sh, relu=False):
    """(ref, scale) in float64: conv(x, wf) + shift (ReLU on ref), scale = conv(|x|, |wf|) + |shift|."""
    xd, shd = x.double(), sh.double().view(1, -1, 1, 1)
    ref = F.conv2d(xd, wf, None, c.stride, c.pad, c.dil) + shd
    scale = F.conv2d(xd.abs(), wf.abs(), None, c.stride, c.pad, c.dil) + shd.abs()
    return (ref.relu() if relu else ref), scale


def xcorr_ref(x, k):
    xd, kd = x.double(), k.double()
    return lr.xcorr(xd, kd), lr.xcorr(xd.abs(), kd.abs())


def conv_gamma(c: Conv, precision):
    fam = "simt" if c.backend == "simt" else "gemm"
    return GAMMA[(fam, precision)] * max(1.0, c.KH * c.KW * c.Cin / K_ENGINE_MAX)


def conv_rho(c: Conv, precision):
    if conv_route(c, precision) == "patch":
        return RHO["split" if precision == "exact" else "hi"]
    return RHO["f32"]


def xcorr_gamma(x: Xcorr):
    n = x.kh * x.kw
    return n * U32 / (1 - n * U32)


def conv_gate(c: Conv, precision, got, ref, scale):
    """(measured gamma, gate use) of the conv gate."""
    return lr.ratio(got, ref, scale, conv_gamma(c, precision), conv_rho(c, precision), 0.0)


def xcorr_gate(x: Xcorr, got, ref, scale):
    return lr.ratio(got, ref, scale, xcorr_gamma(x), 0.0, 0.0)


# ---------------------------------------------------------------------------------------------------- mutations
def mut_transposed(ref):
    """The output with H and W exchanged in its layout (an H / W mix-up in an index computation)."""
    return ref.transpose(-1, -2).contiguous().reshape(ref.shape)


def mut_dilation(c: Conv, x, wf, sh):
    """Taps read at dilation dil + 1 from the same window origin."""
    xp = F.pad(x.double(), [c.pad, c.pad + c.KW - 1, c.pad, c.pad + c.KH - 1])
    Ho, Wo = out_hw(c)
    return F.conv2d(xp, wf, None, c.stride, 0, c.dil + 1)[:, :, :Ho, :Wo] + sh.double().view(1, -1, 1, 1)


def mut_last_kblock(c: Conv, x, wf, sh):
    """The last 64-channel k-block of the last tap missing."""
    w = lr.drop_k_block(wf, (c.KH - 1, c.KW - 1), max(c.Cin - 64, 0), 64)
    return conv_ref(c, x, w, sh)[0]


def mut_lo_dropped(c: Conv, x, wf, sh):
    """The input's lo plane dropped: x rounded to fp16's 11 significant bits."""
    return conv_ref(c, lr.round_sig(x.double()), wf, sh)[0]


def mut_xcorr_shift(x, k):
    """The template kernel shifted by one tap along the columns."""
    ks = torch.zeros_like(k)
    ks[..., 1:] = k[..., :-1]
    return lr.xcorr(x.double(), ks.double())
