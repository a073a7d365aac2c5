"""NYUv2 DenseDepth-style wavelet decoders with the reference's contract, on libwmd.

Mirrors NYUv2/networks/layers.py:11-79 (``Conv3x3``, ``upsample``, ``UpSampleBlock``, ``depthwise``,
``pointwise``) and NYUv2/networks/decoders/densedepth_decoder.py:92-148 (``DecoderWave``), :151-221
(``DecoderWave224``), :224-409 (``SparseDecoderWave``).  The three share one native level engine, driven by a per-class
level table (``_NyuWaveBase._LEVELS``).  State-dict names (``conv2.conv.weight``, ``up1.convA.conv.weight``,
``wave1_ll.conv.weight`` ..., ``iwt.*`` / ``iwt_LL.*`` buffers), constructor and forward signatures and the
output-dict keys are the reference's.  The functional ``sparse_*`` ops of NYUv2/networks/layers.py:82-223
are the KITTI ones minus the 1x1 branch; they are re-exported from ``kitti_layers`` (whose
``sparse_conv3x3`` accepts this file's ``Conv3x3`` as well).

As for KITTI: inference runs natively and batched in the pixel-major row layout; grad-enabled calls of a non-depthwise
``DecoderWave`` or ``DecoderWave224`` (NYUv2/train.py:293-327 trains through them) run every convolution forward and
backward on libwmd when fp32 convolutions are requested (``torch.backends.cudnn.allow_tf32`` False, train_native.py),
else the differentiable cuDNN + native-IDWT path.  The DenseDepth baselines ``Decoder`` and ``Decoder224``
(densedepth_decoder.py:15-89) select their path the same way; their depthwise variants keep the cuDNN module graph.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import opcount, ops, train_native
from .opsfuture import OpsFuture
from ._lib import ACT_LRELU, ACT_NONE, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO, WmdError
from .kitti_decoders import _PackedModule, _need_cuda, _needs_grad, _pm
from .kitti_layers import (make_result, mask2idxmap, mask2yx, sparse_conv3x3, sparse_select,  # noqa: F401
                           sparse_upsample)
from .wavelets import IDWT

_PAD_CODE = {"reflection": PAD_REFLECT, "replicate": PAD_REPLICATE, "zero": PAD_ZERO}


def depthwise(in_channels, kernel_size):
    """[NYUv2/networks/layers.py:70-75]"""
    return nn.Sequential(
        nn.Conv2d(in_channels, in_channels, kernel_size, stride=1, padding=0, bias=False, groups=in_channels),
        nn.ReLU(inplace=True),
    )


def pointwise(in_channels, out_channels):
    """[NYUv2/networks/layers.py:78-79]"""
    return nn.Conv2d(in_channels, out_channels, 1, 1, 0, bias=False)


class Conv3x3(nn.Module):
    """Pad (reflection / replicate / zero) and convolve.  [NYUv2/networks/layers.py:11-32]"""

    def __init__(self, in_channels, out_channels, padding="zero", stride=1, is_depthwise=False):
        super().__init__()
        if padding == "reflection":
            self.pad = nn.ReflectionPad2d(1)
        elif padding == "replicate":
            self.pad = nn.ReplicationPad2d(1)
        else:
            self.pad = nn.ZeroPad2d(1)
        self.padding = padding if padding in ("reflection", "replicate") else "zero"
        self.is_depthwise = bool(is_depthwise)
        if is_depthwise:
            self.conv = nn.Sequential(depthwise(int(in_channels), kernel_size=3),
                                      pointwise(int(in_channels), int(out_channels)))
        else:
            self.conv = nn.Conv2d(int(in_channels), int(out_channels), 3, stride=stride, padding=0)

    def forward(self, x):
        return self.conv(self.pad(x))


def upsample(x):
    """[NYUv2/networks/layers.py:35-36]"""
    return F.interpolate(x, scale_factor=2, mode="nearest")


class UpSampleBlock(nn.Sequential):
    """nearest x2, concat skip, convA, LeakyReLU(0.2).  [NYUv2/networks/layers.py:57-67]"""

    def __init__(self, skip_input, output_features, padding="zero", is_depthwise=False):
        super().__init__()
        self.convA = Conv3x3(skip_input, output_features, padding=padding, is_depthwise=is_depthwise)
        self.leakyreluA = nn.LeakyReLU(0.2)
        self.upsample = nn.Upsample(scale_factor=2, mode="nearest")

    def forward(self, x, concat_with):
        return self.leakyreluA(self.convA(torch.cat([self.upsample(x), concat_with], dim=1)))


class _NyuPacks(_PackedModule):
    """Packed weights of the NYU engines.  The NYU decoders do not track their sources' maxima, so their tensor-core
    convolutions run the tf32x3 operand form: no fp16-pair image."""

    def _gemm(self, name, layer, c1=0):
        conv = layer.conv
        return self._packs.get(("gemm", name), [conv.weight],
                               lambda: ops.pack_weight(conv.weight, c1, precision="tf32x3")), conv.bias.detach()

    def _head(self, name, layer):
        conv = layer.conv
        return self._packs.get(("head", name), [conv.weight], lambda: ops.pack_head_weight(conv.weight)), conv.bias.detach()


class _NyuWaveBase(_NyuPacks):
    # Level table of the native engine and of the native training forward (train_native.nyu_forward).
    # _LL_HEAD: (LL scale, k) - LL = scale * wave1_ll(up1 output), and ("disp", k) is the raw LL head (k None: no such
    # output).  _LEVELS: one (j, s, disp) per IDWT level, coarse to fine: the level reads up<j>'s output (up1 for j = 1,
    # shared with the LL head), its details are 2**s * wave<j>, and ("disp", s) is "div" ll / 2**s, "floor" ll // 2 or
    # "last" ll itself (with depth_epilogue's ("depth", s)).  Sparse decoders run the levels j > 1 on active lists.
    _LL_HEAD = (2 ** 3, 3)                                        # densedepth_decoder.py:122-123
    _LEVELS = ((1, 2, "div"), (2, 1, "div"), (3, 0, "last"))     # densedepth_decoder.py:124-146

    def _build(self, enc_features, decoder_width, dw_waveconv=False, dw_upconv=False):
        features = int(enc_features[-1] * decoder_width)
        self.features = features
        self.enc_features = list(enc_features)
        wave_pad = "zero"
        padding = "reflection"
        self.iwt = IDWT(wave="haar", mode=wave_pad)
        self.iwt_LL = IDWT(wave="haar", mode="zero")
        self.conv2 = Conv3x3(enc_features[-1], features, padding="replicate")
        self.up1 = UpSampleBlock(skip_input=features // 1 + enc_features[-2], output_features=features // 2,
                                 padding=padding, is_depthwise=dw_upconv)
        self.wave1_ll = Conv3x3(features // 2, 1, padding="replicate")
        self.wave1 = Conv3x3(features // 2, 3, padding=wave_pad, is_depthwise=dw_waveconv)
        for j in range(2, len(self._LEVELS) + 1):                 # up2, wave2, up3, wave3 [, up4, wave4]
            setattr(self, "up%d" % j, UpSampleBlock(skip_input=features // 2 ** (j - 1) + enc_features[-1 - j],
                                                    output_features=features // 2 ** j, padding=padding,
                                                    is_depthwise=dw_upconv))
            setattr(self, "wave%d" % j, Conv3x3(features // 2 ** j, 3, padding=wave_pad, is_depthwise=dw_waveconv))
        self._depthwise = bool(dw_waveconv or dw_upconv)
        # optional consumer epilogue of ("disp", 0), off by default: (div, lo, hi) adds ("depth", 0) =
        # clamp(("disp", 0) / div, lo, hi) - NYUv2/utils.py:219,229 uses (100, 0.4, 10) - fused into the last IDWT
        self.depth_epilogue = None
        self._init_packs()

    def _forward(self, x_blocks):
        """Dense decoders: the cuDNN module graph for depthwise variants and for training with TF32 allowed, the native
        training forward for training with fp32 convolutions, the native engine otherwise (no_grad / inference)."""
        _need_cuda(x_blocks)
        needs_grad = _needs_grad(self, x_blocks)
        if self._depthwise or (needs_grad and not train_native.fp32_convs_requested()):
            return self._autograd_forward(x_blocks)
        if needs_grad:
            # fp32 convolutions requested: forward and backward of every convolution on libwmd
            return train_native.nyu_forward(self, x_blocks)
        out, _ = self._native_forward(x_blocks, 0.0, sparse=False)
        return out

    @torch.no_grad()
    @ops._on_device
    def _native_forward(self, blocks, thresh_ratio, sparse):
        """conv2/up1 and the first level dense, then the levels of _LEVELS dense or on active lists.

        Returns (outputs, counts): counts = int32 device tensor (2, 2, N+1), row offsets of S4 / S5 of the two sparse
        blocks (None on the dense path)."""
        _need_cuda(blocks)
        if self._depthwise:
            raise NotImplementedError("depthwise-separable variants only run on the differentiable cuDNN path")
        out = {}
        xb = blocks[-1]
        n, _, h, w = xb.shape
        f = self.features
        counts = []
        wp, b = self._gemm("conv2", self.conv2)
        d0 = ops.conv_rows(ops.nchw_to_rows(xb), xb.shape[1], wp, b, f, n, h, w, pad=PAD_REPLICATE, act=ACT_NONE)
        skip = blocks[-2]
        if tuple(skip.shape[2:]) != (2 * h, 2 * w):
            raise WmdError("skip block has shape %s, expected spatial %s" % (tuple(skip.shape), (2 * h, 2 * w)))
        wp, b = self._gemm("up1", self.up1.convA, skip.shape[1])
        d1 = ops.conv_rows(d0, f, wp, b, f // 2, n, 2 * h, 2 * w, pad=PAD_REFLECT, act=ACT_LRELU, act_param=0.2,
                           shift0=1, x1=ops.nchw_to_rows(skip), c1=skip.shape[1])
        h, w = 2 * h, 2 * w
        ll_scale, ll_disp = self._LL_HEAD
        wl, bl = self._head("wave1_ll", self.wave1_ll)
        raw = ops.head_conv3x3(d1, f // 2, 0, wl, bl, n, h, w, 1, scale=1.0, act=ACT_NONE, pad=PAD_REPLICATE)
        ll = raw * float(ll_scale)           # exact power-of-two scaling of a (N,1,H/16,W/16) map
        if ll_disp is not None:
            out[("disp", ll_disp)] = raw     # == ll / ll_scale (densedepth_decoder.py:123)

        x_rows, x_c, prev_map, hcoef = d1, f // 2, None, None
        for j, s, disp_form in self._LEVELS:
            scale = float(2 ** s)
            wave = getattr(self, "wave%d" % j)
            if j == 1:
                # the first level's details come from up1's output, like the LL head
                wh, bh = self._head("wave1", wave)
                hcoef = ops.head_conv3x3(d1, f // 2, 0, wh, bh, n, h, w, 3, scale=scale, act=ACT_NONE, pad=PAD_ZERO)
                if sparse:
                    # the reference builds this one as ones_like(h[:, 0]) with h already (N,1,3,H,W): a 3-channel map
                    # (densedepth_decoder.py:301-303); kept as is
                    out[("wavelet_mask", s)] = torch.ones((n, 3, h, w), dtype=torch.float32, device=xb.device)
                out[("wavelets", s, "LL")] = ll
            else:
                name = "up%d" % j
                up = getattr(self, name)
                skip = blocks[-1 - j]
                cs = skip.shape[1]
                cout = up.convA.conv.weight.shape[0]
                wp, b = self._gemm(name, up.convA, cs)
                wh, bh = self._head("wave%d" % j, wave)
                if tuple(skip.shape[2:]) != (2 * h, 2 * w):
                    raise WmdError("skip block has shape %s, expected spatial %s" % (tuple(skip.shape), (2 * h, 2 * w)))
                if sparse:
                    thresh = ops.range_thresh(ll, thresh_ratio)
                    masks = ops.level_masks(hcoef, thresh, want=("S2", "S3", "S4", "S5"))
                    gmap = ops.gate_map(masks["S2"], prev_map)
                    map4, pix4, off4 = ops.compact(masks["S4"])
                    _, pix5, off5 = ops.compact(masks["S5"], want_idxmap=False)
                    counts.append((off4, off5))
                    out[("wavelet_mask", s)] = masks["S5"].to(torch.float32)
                    xa = ops.conv_rows(x_rows, x_c, wp, b, cout, n, 2 * h, 2 * w, pad=PAD_REFLECT, act=ACT_LRELU,
                                       act_param=0.2, map0=gmap, shift0=1, x1=ops.nchw_to_rows(skip), c1=cs,
                                       gate=masks["S3"], pixels=pix4, count=off4[n:],
                                       m_in0=_pm(lambda: (gmap >= 0).sum()), m_in1=_pm(lambda: masks["S3"].sum()))
                    hcoef = ops.head_conv3x3(xa, cout, 0, wh, bh, n, 2 * h, 2 * w, 3, scale=scale, act=ACT_NONE,
                                             pad=PAD_ZERO, idxmap=map4, pixels=pix5, count=off5[n:])
                    prev_map = map4
                else:
                    xa = ops.conv_rows(x_rows, x_c, wp, b, cout, n, 2 * h, 2 * w, pad=PAD_REFLECT, act=ACT_LRELU,
                                       act_param=0.2, shift0=1, x1=ops.nchw_to_rows(skip), c1=cs)
                    hcoef = ops.head_conv3x3(xa, cout, 0, wh, bh, n, 2 * h, 2 * w, 3, scale=scale, act=ACT_NONE,
                                             pad=PAD_ZERO)
                x_rows, x_c = xa, cout
                h, w = 2 * h, 2 * w
            for k, band in enumerate(("LH", "HL", "HH")):
                out[("wavelets", s, band)] = hcoef[:, k:k + 1]
            if disp_form == "div":
                ll, disp = ops.idwt_haar(ll, hcoef.unsqueeze(1), disp_scale=1.0 / 2 ** s, clamp01=False)
                out[("disp", s)] = disp
            elif disp_form == "floor":
                ll = ops.idwt_haar(ll, hcoef.unsqueeze(1))
                out[("disp", s)] = ll // 2           # torch's floor division, as the reference computes it
            elif self.depth_epilogue is not None:
                ll, depth = ops.idwt_haar(ll, hcoef.unsqueeze(1), epilogue=("div_clamp",) + tuple(self.depth_epilogue))
                out[("disp", s)], out[("depth", s)] = ll, depth
            else:
                ll = ops.idwt_haar(ll, hcoef.unsqueeze(1))
                out[("disp", s)] = ll
        return out, (torch.stack([torch.stack(c) for c in counts]) if counts else None)


class DecoderWave(_NyuWaveBase):
    """Dense wavelet decoder.  [densedepth_decoder.py:92-148]"""

    def __init__(self, enc_features=[96, 96, 192, 384, 2208], decoder_width=0.5, dw_waveconv=False, dw_upconv=False):
        super().__init__()
        self._build(enc_features, decoder_width, dw_waveconv, dw_upconv)

    def _autograd_forward(self, x_blocks):
        outputs = {}
        x_d0 = self.conv2(x_blocks[-1])
        x_d1 = self.up1(x_d0, x_blocks[-2])
        ll = (2 ** 3) * self.wave1_ll(x_d1)
        outputs[("disp", 3)] = ll / (2 ** 3)
        h = (2 ** 2) * self.wave1(x_d1).unsqueeze(1)
        outputs[("wavelets", 2, "LL")] = ll
        for k, band in enumerate(("LH", "HL", "HH")):
            outputs[("wavelets", 2, band)] = h[:, :, k]
        ll = self.iwt((ll, list([h])))
        outputs[("disp", 2)] = ll / (2 ** 2)
        x_d2 = self.up2(x_d1, x_blocks[-3])
        h = (2 ** 1) * self.wave2(x_d2).unsqueeze(1)
        for k, band in enumerate(("LH", "HL", "HH")):
            outputs[("wavelets", 1, band)] = h[:, :, k]
        ll = self.iwt((ll, list([h])))
        outputs[("disp", 1)] = ll / (2 ** 1)
        x_d3 = self.up3(x_d2, x_blocks[-4])
        h = self.wave3(x_d3).unsqueeze(1)
        for k, band in enumerate(("LH", "HL", "HH")):
            outputs[("wavelets", 0, band)] = h[:, :, k]
        ll = self.iwt((ll, list([h])))
        outputs[("disp", 0)] = ll
        return outputs

    def forward(self, x_blocks):
        return self._forward(x_blocks)


class SparseDecoderWave(_NyuWaveBase):
    """Threshold-gated sparse decoder (levels 1 and 0 sparse), batched.  [densedepth_decoder.py:224-409]"""

    def __init__(self, enc_features=[96, 96, 192, 384, 2208], decoder_width=0.5):
        super().__init__()
        self._build(enc_features, decoder_width)
        self.sparse_padding = "reflect"
        self.sparse_wave_pad = "constant"
        self.leakyreluA = nn.LeakyReLU(0.2)
        self.maxpool3 = nn.MaxPool2d(3, stride=1, padding=1)
        self.maxpool5 = nn.MaxPool2d(5, stride=1, padding=2)
        self.maxpool7 = nn.MaxPool2d(7, stride=1, padding=3)
        self.count_ops = True

    def forward(self, x_blocks, thresh_ratio=0.1):
        out, counts = self._native_forward(x_blocks, float(thresh_ratio), sparse=True)
        if self.count_ops:
            fut = self.ops_future(counts, x_blocks)
            if self.count_ops == "async":
                out["total_ops"] = fut                       # OpsFuture: nothing waits (see opsfuture.py)
            else:
                out.update(fut.result())
        return out

    def ops_future(self, counts, x_blocks):
        """OpsFuture of one forward: enqueues the count read-back on the current stream (no host wait)."""
        n, cin, h, w = (int(v) for v in x_blocks[-1].shape)
        f = self.features
        c2, c3, c4 = (int(x_blocks[k].shape[1]) for k in (-2, -3, -4))

        def finish(host):                                    # host: (2, 2, N+1) offsets of S4 / S5 per sparse block
            per_sample = []
            for b in range(n):
                v = opcount.nyu_dense_part_ops(cin, h, w, f, c2)
                m4, m5 = (int(host[0][k][b + 1] - host[0][k][b]) for k in range(2))
                v += opcount.nyu_sparse_block_ops(2 * h, 2 * w, f // 2 + c3, f // 4, m4, m5, False)
                m4, m5 = (int(host[1][k][b + 1] - host[1][k][b]) for k in range(2))
                v += opcount.nyu_sparse_block_ops(4 * h, 4 * w, f // 4 + c4, f // 8, m4, m5, True)
                per_sample.append(v)
            res = {"total_ops": sum(per_sample)}
            if n > 1:
                res["total_ops_per_sample"] = per_sample
            return res

        return OpsFuture(counts, finish)


# ------------------------------------------------------------------------------------------------------------------
# The DenseDepth baseline decoders (NYUv2/model.py:47-64 builds them without --use_wavelets).
# ------------------------------------------------------------------------------------------------------------------
class _BaselineDecoder(_NyuPacks):
    """conv2 -> four UpSampleBlocks -> [x2 + conv5 + LeakyReLU(0.2)] -> conv3; zero padding everywhere.

    ``no_grad`` calls run the native engine: conv2, up1..up4 and conv5 on the gather-GEMM engine (tf32x3 operands),
    conv3 on head_conv3x3.  Grad-enabled calls with fp32 convolutions requested (``torch.backends.cudnn.allow_tf32``
    False) run ``train_native.nyu_baseline_forward``.  Training with TF32 allowed and the depthwise variants run the cuDNN
    module graph."""

    def _build(self, enc_features, decoder_width, is_depthwise, extra_stage):
        f = int(enc_features[-1] * decoder_width)
        self.conv2 = Conv3x3(enc_features[-1], f, padding="zero")
        for k in range(1, 5):
            setattr(self, "up%d" % k, UpSampleBlock(skip_input=f // 2 ** (k - 1) + enc_features[-1 - k],
                                                    output_features=f // 2 ** k, padding="zero",
                                                    is_depthwise=is_depthwise))
        last = f // 16
        if extra_stage:
            self.conv5 = nn.Sequential(Conv3x3(f // 16, f // 32, is_depthwise=is_depthwise), nn.LeakyReLU(0.2))
            last = f // 32
        if is_depthwise:
            self.conv3 = Conv3x3(last, 1, is_depthwise=True)
        else:
            self.conv3 = nn.Conv2d(last, 1, kernel_size=3, stride=1, padding=1, padding_mode="zeros")
        if extra_stage:
            self.upsample = nn.Upsample(scale_factor=2, mode="nearest")
        self._extra_stage = extra_stage
        self._depthwise = bool(is_depthwise)
        self._init_packs()

    def forward(self, features):
        blocks = tuple(features)
        if len(blocks) != 5:
            raise ValueError("expected the five encoder blocks, fine to coarse")
        needs_grad = _needs_grad(self, blocks)
        if self._depthwise or (needs_grad and not train_native.fp32_convs_requested()):
            return self._autograd_forward(blocks)
        _need_cuda(blocks)
        if needs_grad:
            return train_native.nyu_baseline_forward(self, blocks)
        return self._native_forward(blocks)

    @torch.no_grad()
    @ops._on_device
    def _native_forward(self, blocks):
        xb = blocks[4]
        n, c, h, w = (int(v) for v in xb.shape)
        up = 32 if self._extra_stage else 16
        if n == 0:
            return {("disp", 0): torch.zeros((0, 1, up * h, up * w), dtype=torch.float32, device=xb.device)}
        wp, b = self._gemm("conv2", self.conv2)
        f = int(self.conv2.conv.weight.shape[0])
        d = ops.conv_rows(ops.nchw_to_rows(xb), c, wp, b, f, n, h, w, pad=PAD_ZERO, act=ACT_NONE)
        c = f
        for k in range(1, 5):
            skip = blocks[4 - k]
            if tuple(skip.shape[2:]) != (2 * h, 2 * w):
                raise WmdError("skip block has shape %s, expected spatial %s" % (tuple(skip.shape), (2 * h, 2 * w)))
            conv = getattr(self, "up%d" % k).convA
            cout = int(conv.conv.weight.shape[0])
            wp, b = self._gemm("up%d" % k, conv, int(skip.shape[1]))
            d = ops.conv_rows(d, c, wp, b, cout, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_LRELU, act_param=0.2, shift0=1,
                              x1=ops.nchw_to_rows(skip), c1=int(skip.shape[1]))
            c, h, w = cout, 2 * h, 2 * w
        if self._extra_stage:
            cout = int(self.conv5[0].conv.weight.shape[0])
            wp, b = self._gemm("conv5", self.conv5[0])
            d = ops.conv_rows(d, c, wp, b, cout, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_LRELU, act_param=0.2, shift0=1)
            c, h, w = cout, 2 * h, 2 * w
        w3 = self._packs.get(("head", "conv3"), [self.conv3.weight], lambda: ops.pack_head_weight(self.conv3.weight))
        return {("disp", 0): ops.head_conv3x3(d, c, 0, w3, self.conv3.bias.detach(), n, h, w, 1, act=ACT_NONE,
                                              pad=PAD_ZERO)}

    def _autograd_forward(self, blocks):
        x = self.conv2(blocks[4])
        for k in range(1, 5):
            x = getattr(self, "up%d" % k)(x, blocks[4 - k])
        if self._extra_stage:
            x = self.conv5(self.upsample(x))
        return {("disp", 0): self.conv3(x)}


class Decoder(_BaselineDecoder):
    """DenseDepth baseline decoder (no wavelets).  [densedepth_decoder.py:15-47]"""

    def __init__(self, enc_features=[96, 96, 192, 384, 2208], decoder_width=0.5, is_depthwise=False):
        super().__init__()
        self._build(enc_features, decoder_width, is_depthwise, extra_stage=False)


class Decoder224(_BaselineDecoder):
    """Baseline decoder for 224-pixel inputs: one more x2 + conv stage.  [densedepth_decoder.py:50-89]"""

    def __init__(self, enc_features=[96, 96, 192, 384, 2208], decoder_width=0.5, is_depthwise=False):
        super().__init__()
        self._build(enc_features, decoder_width, is_depthwise, extra_stage=True)


class DecoderWave224(_NyuWaveBase):
    """Four-level wavelet decoder for 224-pixel inputs (NYUv2/train.py --use_224).  [densedepth_decoder.py:151-221]

    Same state-dict names and order as the reference (conv2, up1..up4, wave1_ll, wave1..wave4, iwt / iwt_LL buffers, the
    unused sigmoid).  Runs like ``DecoderWave``: the native engine at inference, the native training forward when fp32
    convolutions are requested, the cuDNN module graph for depthwise variants and for training with TF32 allowed.  Like
    every NYU engine launch, the tensor-core convolutions take the tf32x3 operand form: the engine does not track its
    sources' maxima, which the fp16-pair form needs.  ``depth_epilogue`` works as in ``DecoderWave``: with the reference's
    224 evaluation (NYUv2/utils.py:215-229, no resize) it is ``(100, 0.4, 10)``.

    Keeps the reference's quirks (:181-221): ``("wavelets", 3, "LL")`` is 16 * wave1_ll with details scaled 8, 4, 2, 1;
    ``("disp", 3)`` is taken after the first IDWT; ``("disp", 1)`` is FLOOR-divided (:212, SURVEY A.5) - by torch on the
    level's LL, so that it equals the reference's given the same LL; the native training step gives it a zero gradient
    (train_native._FloorHalfFn); nothing is clamped."""

    _LL_HEAD = (2 ** 4, None)
    _LEVELS = ((1, 3, "div"), (2, 2, "div"), (3, 1, "floor"), (4, 0, "last"))

    def __init__(self, enc_features=[96, 96, 192, 384, 2208], decoder_width=0.5, dw_waveconv=False, dw_upconv=False):
        super().__init__()
        self._build(enc_features, decoder_width, dw_waveconv, dw_upconv)
        self.sigmoid = nn.Sigmoid()

    def _autograd_forward(self, x_blocks):
        out = {}
        x = self.up1(self.conv2(x_blocks[-1]), x_blocks[-2])
        ll = (2 ** 4) * self.wave1_ll(x)
        out[("wavelets", 3, "LL")] = ll
        for k in range(1, 5):                                # level k emits scale 4 - k
            s = 4 - k
            if k > 1:
                x = getattr(self, "up%d" % k)(x, x_blocks[-1 - k])
            hcoef = (2 ** s) * getattr(self, "wave%d" % k)(x).unsqueeze(1)
            for j, band in enumerate(("LH", "HL", "HH")):
                out[("wavelets", s, band)] = hcoef[:, :, j]
            ll = self.iwt((ll, [hcoef]))
            out[("disp", s)] = ll // 2 if s == 1 else ll / (2 ** s)
        return out

    def forward(self, x_blocks):
        return self._forward(x_blocks)
