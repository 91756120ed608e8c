"""CPU oracle for the SiamMask per-frame inference hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package (`siammask_b200/`)
may import this module; only `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py` use it, and only as the
checker / the timed CPU baseline.

It is a plain restatement, in torch fp32 functional calls on the CPU, of what
the reference computes on the path (all citations into foolwood/SiamMask):

  * `conv2d_dw_group`                      models/rpn.py:32-38
  * `DepthCorr.forward_corr / .head`       models/rpn.py:41-72
  * `Bottleneck.forward`                   experiments/siammask_sharp/resnet.py:80-103
  * `ResNet.forward / _make_layer`         experiments/siammask_sharp/resnet.py:151-227
  * `ResDownS`, `ResDown.forward_all`      experiments/siammask_sharp/custom.py:12-66
  * `UP.forward`                           experiments/siammask_sharp/custom.py:83-86
  * `Refine.forward(test=True)`            experiments/siammask_sharp/custom.py:131-154
  * `Custom.template/track/track_mask/track_refine`
                                           experiments/siammask_sharp/custom.py:173-190

The reference holds no tests and no golden vectors for this path (SURVEY §4),
so the oracle is pinned the other way round: `oracle/make_golden.py` imports
the *unmodified* reference model from /root/reference, runs it on a seeded
checkpoint and commits its outputs under `tests/golden/`; `tests/test_oracle.py`
checks this restatement against those vectors.

The arithmetic itself (conv / batch-norm / max-pool / nearest upsample) lives
in PyTorch, which the reference pins as torch==0.4.1 (requirements.txt); here it
is torch 2.x — the eval-mode semantics of these ops are unchanged.

`emulate` (None | 'fp16' | 'bf16' | 'tf32') optionally rounds every conv input
and every conv weight to that format before an fp32-accumulated convolution.
It predicts what a single-pass tensor-core implementation delivers and is used
by tests to separate kernel bugs from precision effects; with emulate=None the
oracle is the fp32 reference semantics.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5  # nn.BatchNorm2d default, used by every BN on the path

# (name, planes, blocks, stride of block 0, dilation of blocks 1..)   resnet.py:159-165
_LAYERS = (("layer1", 64, 3, 1, 1), ("layer2", 128, 4, 2, 1), ("layer3", 256, 6, 1, 2))


def _round_to(x: torch.Tensor, fmt: str | None) -> torch.Tensor:
    if fmt is None:
        return x
    if fmt == "fp16":
        return x.to(torch.float16).to(torch.float32)
    if fmt == "bf16":
        return x.to(torch.bfloat16).to(torch.float32)
    if fmt == "tf32":  # round-to-nearest-even on the 13 dropped mantissa bits
        i = x.contiguous().view(torch.int32)
        lsb = (i >> 13) & 1
        i = (i + 0xFFF + lsb) & ~0x1FFF
        return i.view(torch.float32)
    raise ValueError(fmt)


class Oracle:
    """Functional SiamMask-sharp over a reference-keyed state dict (SURVEY App. B)."""

    def __init__(self, state_dict, anchors=None, emulate: str | None = None, bn_hook=None):
        self.sd = state_dict
        self.anchors = anchors or {"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8], "round_dight": 0}
        self.anchor_num = len(self.anchors["ratios"]) * len(self.anchors["scales"])  # siammask_sharp.py:17
        self.emulate = emulate
        self.bn_hook = bn_hook
        self.has_mask = "mask_model.mask.head.3.weight" in state_dict
        self.has_refine = "refine_model.deconv.weight" in state_dict

    # -- primitives ---------------------------------------------------------
    def _conv(self, x, wkey, bkey=None, stride=1, pad=0, dil=1):
        w = self.sd[wkey]
        b = self.sd[bkey] if bkey is not None else None
        return F.conv2d(_round_to(x, self.emulate), _round_to(w, self.emulate), b, stride, pad, dil)

    def _bn(self, x, key):
        if self.bn_hook is not None:
            self.bn_hook(key, x, self.sd)
        g, b = self.sd[key + ".weight"], self.sd[key + ".bias"]
        m, v = self.sd[key + ".running_mean"], self.sd[key + ".running_var"]
        scale = g / torch.sqrt(v + BN_EPS)
        return x * scale.view(1, -1, 1, 1) + (b - m * scale).view(1, -1, 1, 1)

    # -- backbone -----------------------------------------------------------
    def _bottleneck(self, x, p, stride, dilation, ds):
        """resnet.py:80-103.  ds: None | (kernel, stride, pad) of the downsample conv."""
        out = F.relu(self._bn(self._conv(x, p + "conv1.weight"), p + "bn1"))
        pad = dilation if dilation > 1 else 2 - stride          # resnet.py:66-70
        out = F.relu(self._bn(self._conv(out, p + "conv2.weight", None, stride, pad, dilation), p + "bn2"))
        out = self._bn(self._conv(out, p + "conv3.weight"), p + "bn3")
        res = x
        if ds is not None:
            k, s, pd = ds
            res = self._bn(self._conv(x, p + "downsample.0.weight", None, s, pd, 1), p + "downsample.1")
        return F.relu(out + res)

    def features(self, x):
        """ResNet.forward, resnet.py:217-227 -> (p0, p1, p2, p3)."""
        P = "features.features."
        p0 = F.relu(self._bn(self._conv(x, P + "conv1.weight", None, 2, 0, 1), P + "bn1"))
        y = F.max_pool2d(p0, 3, 2, 1)
        outs = [p0]
        for name, planes, blocks, stride, dilation in _LAYERS:
            for i in range(blocks):
                p = f"{P}{name}.{i}."
                if i == 0:
                    # _make_layer, resnet.py:184-215: first block gets dilation dd
                    if stride == 1 and dilation == 1:
                        ds, d0 = (1, 1, 0), 1
                    elif dilation > 1:
                        ds, d0 = (3, stride, dilation // 2), dilation // 2
                    else:
                        ds, d0 = (3, stride, 0), 1
                    y = self._bottleneck(y, p, stride, d0, ds)
                else:
                    y = self._bottleneck(y, p, 1, dilation, None)
            outs.append(y)
        return tuple(outs)

    def resdown(self, p3):
        """ResDownS.forward, custom.py:19-25."""
        x = self._bn(self._conv(p3, "features.downsample.downsample.0.weight"), "features.downsample.downsample.1")
        if x.size(3) < 20:
            x = x[:, :, 4:-4, 4:-4]
        return x

    # -- correlation heads ---------------------------------------------------
    @staticmethod
    def xcorr_depthwise(x, kernel):
        """conv2d_dw_group, models/rpn.py:32-38 (paired batch, valid, no flip)."""
        b, c = kernel.shape[:2]
        out = F.conv2d(x.reshape(1, b * c, x.size(2), x.size(3)),
                       kernel.reshape(b * c, 1, kernel.size(2), kernel.size(3)), groups=b * c)
        return out.view(b, c, out.size(2), out.size(3))

    def conv_kernel(self, zf, p):
        return F.relu(self._bn(self._conv(zf, p + "conv_kernel.0.weight"), p + "conv_kernel.1"))

    def conv_search(self, xf, p):
        return F.relu(self._bn(self._conv(xf, p + "conv_search.0.weight"), p + "conv_search.1"))

    def forward_corr(self, zf, xf, p):
        """DepthCorr.forward_corr, rpn.py:63-67."""
        return self.xcorr_depthwise(self.conv_search(xf, p), self.conv_kernel(zf, p))

    def head(self, feat, p):
        """DepthCorr.head, rpn.py:56-61."""
        h = F.relu(self._bn(self._conv(feat, p + "head.0.weight"), p + "head.1"))
        return self._conv(h, p + "head.3.weight", p + "head.3.bias")

    # -- refine ---------------------------------------------------------------
    def _seq2(self, x, p):
        x = F.relu(self._conv(x, p + ".0.weight", p + ".0.bias", 1, 1))
        return F.relu(self._conv(x, p + ".2.weight", p + ".2.bias", 1, 1))

    def refine(self, f, corr_feature, pos):
        """Refine.forward(test=True), custom.py:131-154.  pos = (dy, dx) shared by the batch."""
        R = "refine_model."
        dy, dx = int(pos[0]), int(pos[1])
        p0 = F.pad(f[0], [16, 16, 16, 16])[:, :, 4 * dy:4 * dy + 61, 4 * dx:4 * dx + 61]
        p1 = F.pad(f[1], [8, 8, 8, 8])[:, :, 2 * dy:2 * dy + 31, 2 * dx:2 * dx + 31]
        p2 = F.pad(f[2], [4, 4, 4, 4])[:, :, dy:dy + 15, dx:dx + 15]
        p3 = corr_feature[:, :, dy, dx].reshape(-1, 256, 1, 1)
        out = F.conv_transpose2d(_round_to(p3, self.emulate), _round_to(self.sd[R + "deconv.weight"], self.emulate),
                                 self.sd[R + "deconv.bias"], 15)
        out = F.interpolate(self._seq2(out, R + "h2") + self._seq2(p2, R + "v2"), size=(31, 31))
        out = self._conv(out, R + "post0.weight", R + "post0.bias", 1, 1)
        out = F.interpolate(self._seq2(out, R + "h1") + self._seq2(p1, R + "v1"), size=(61, 61))
        out = self._conv(out, R + "post1.weight", R + "post1.bias", 1, 1)
        out = F.interpolate(self._seq2(out, R + "h0") + self._seq2(p0, R + "v0"), size=(127, 127))
        out = self._conv(out, R + "post2.weight", R + "post2.bias", 1, 1)
        return out.reshape(-1, 127 * 127)

    # -- the boundary: Custom.* ------------------------------------------------
    @torch.no_grad()
    def template(self, z):
        self.zf = self.resdown(self.features(z)[-1])

    @torch.no_grad()
    def track(self, x):
        xf = self.resdown(self.features(x)[-1])
        cls = self.head(self.forward_corr(self.zf, xf, "rpn_model.cls."), "rpn_model.cls.")
        loc = self.head(self.forward_corr(self.zf, xf, "rpn_model.loc."), "rpn_model.loc.")
        return cls, loc

    @torch.no_grad()
    def track_mask(self, x, with_mask_head=True):
        self.feature = self.features(x)
        self.search = self.resdown(self.feature[-1])
        cls = self.head(self.forward_corr(self.zf, self.search, "rpn_model.cls."), "rpn_model.cls.")
        loc = self.head(self.forward_corr(self.zf, self.search, "rpn_model.loc."), "rpn_model.loc.")
        self.corr_feature = self.forward_corr(self.zf, self.search, "mask_model.mask.")
        mask = self.head(self.corr_feature, "mask_model.mask.") if with_mask_head else None
        return cls, loc, mask

    @torch.no_grad()
    def track_refine(self, pos):
        """pos: (dy, dx) shared by the batch (reference semantics), or an int [B,2] array giving
        one position per stream (the batched extension, SURVEY §8b) — evaluated sample by sample."""
        pos_arr = np.asarray(pos)
        if pos_arr.ndim == 1:
            return self.refine(self.feature, self.corr_feature, pos_arr)
        outs = []
        for b in range(pos_arr.shape[0]):
            f = [t[b:b + 1] for t in self.feature]
            outs.append(self.refine(f, self.corr_feature[b:b + 1], pos_arr[b]))
        return torch.cat(outs, 0)


# ---- independent plain-loop restatements (cross-checks of the oracle itself) ----

def xcorr_depthwise_loops(x: np.ndarray, k: np.ndarray) -> np.ndarray:
    """out[b,c,i,j] = sum_{u,v} x[b,c,i+u,j+v] * k[b,c,u,v]  (models/rpn.py:32-38, float64 accumulate)."""
    B, C, H, W = x.shape
    kh, kw = k.shape[2:]
    out = np.zeros((B, C, H - kh + 1, W - kw + 1), np.float64)
    for u in range(kh):
        for v in range(kw):
            out += x[:, :, u:u + out.shape[2], v:v + out.shape[3]].astype(np.float64) * k[:, :, u:u + 1, v:v + 1]
    return out


def nearest_upsample_index(out_size: int, in_size: int) -> np.ndarray:
    """Source index of F.upsample(mode='nearest') as used at custom.py:150-152:
    src = min(floor(dst * in / out), in - 1)  (float32 scale, as ATen computes it)."""
    scale = np.float32(in_size) / np.float32(out_size)
    return np.minimum(np.floor(np.arange(out_size, dtype=np.float32) * scale).astype(np.int64), in_size - 1)
