"""Native training step of the dense wavelet decoders and the baseline decoders: every convolution runs forward and
backward on libwmd.

Selected by the decoders for a grad-enabled call when ``torch.backends.cudnn.allow_tf32`` is False, which is how a PyTorch
user asks for fp32 convolutions; with TF32 allowed they keep the cuDNN path.  Each decoder convolution is one
``_ConvRowsFn`` on pixel-major rows: its forward is ``ops.conv_rows`` (source maxima tracked for the fp16-pair operand
form), its backward the activation backward with the bias gradient, the tensor-core weight gradient and the data gradient
(the forward engine over the ring-extended grid plus the fold).  The glue stays torch autograd: NCHW <-> rows moves (the
reverse move is the adjoint), the power-of-two scalings and the sigma difference, the native IDWT, the clamp.  The fused
inference kernels (head_mlp, head_idwt, the baseline's disp_tail16) are not used: they do not keep the intermediates a
backward needs.
"""
import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import ops
from ._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO


def fp32_convs_requested():
    """True when PyTorch is asked for fp32 (not TF32) convolutions: the native training path computes exactly that."""
    return not torch.backends.cudnn.allow_tf32


class _ToRowsFn(torch.autograd.Function):
    """NCHW -> pixel-major rows (raising `amax` to max |x|); the adjoint is the reverse move."""

    @staticmethod
    def forward(ctx, x, amax):
        ctx.shape = tuple(x.shape)
        return ops.nchw_to_rows(x, amax=amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.rows_to_nchw(g, *ctx.shape), None


class _ToNchwFn(torch.autograd.Function):
    """Pixel-major rows -> NCHW (N, C, H, W); the adjoint is the reverse move."""

    @staticmethod
    def forward(ctx, rows, n, c, h, w):
        ctx.ld = rows.shape[1]
        return ops.rows_to_nchw(rows, n, c, h, w)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.nchw_to_rows(g.contiguous(), ld=ctx.ld), None, None, None, None


class _ConvRowsFn(torch.autograd.Function):
    """y = act(bias + A W) on rows, A gathered from x0 rows (shift0: the nearest x2 upsample) and the NCHW skip x1."""

    @staticmethod
    def forward(ctx, x0, x1, weight, bias, cfg):
        n, h, w, taps, pad, act, act_param, shift0, amax0, amax_out = cfg
        cout, cin = int(weight.shape[0]), int(weight.shape[1])
        c1 = int(x1.shape[1]) if x1 is not None else 0
        c0 = cin - c1
        amax1 = torch.zeros(1, dtype=torch.float32, device=x0.device) if x1 is not None else None
        x1r = ops.nchw_to_rows(x1, amax=amax1) if x1 is not None else None
        wp = ops.pack_weight(weight.detach(), c1)
        y = ops.conv_rows(x0, c0, wp, bias.detach(), cout, n, h, w, taps=taps, pad=pad, act=act, act_param=act_param,
                          shift0=shift0, x1=x1r, c1=c1, amax0=amax0, amax1=amax1, amax_out=amax_out)
        ctx.cfg = (n, h, w, taps, pad, act, act_param, shift0, c0, c1, cout)
        ctx.save_for_backward(x0, x1r, weight, y)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        n, h, w, taps, pad, act, act_param, shift0, c0, c1, cout = ctx.cfg
        x0, x1r, weight, y = ctx.saved_tensors
        need_x0, need_x1, need_w, need_b = ctx.needs_input_grad[:4]
        amax_dz = torch.zeros(1, dtype=torch.float32, device=y.device)
        dz, db = ops.act_backward(y, gy, cout, act, act_param, want_bias=need_b, amax=amax_dz)
        dw = ops.conv_wgrad(x0, c0, dz, cout, n, h, w, taps=taps, pad=pad, shift0=shift0, x1=x1r, c1=c1) if need_w else None
        dx0 = dx1 = None
        if need_x0 or need_x1:
            wt = ops.pack_weight(weight.detach().transpose(0, 1).flip(2, 3))
            dx0, dx1 = ops.conv_dgrad(dz, cout, wt, c0, n, h, w, taps=taps, pad=pad, shift0=shift0, c1=c1, amax=amax_dz,
                                      want_x1=need_x1)
        return dx0 if need_x0 else None, dx1, dw, db, None


class _FloorHalfFn(torch.autograd.Function):
    """ll // 2 (torch's floor division) with a zero gradient: DecoderWave224's ("disp", 1) (densedepth_decoder.py:212).

    A floor is flat wherever it is differentiable, so a loss on that output trains nothing; the native step keeps it that
    way rather than giving it the gradient of ll / 2.  (Recent torch has no derivative for floor division at all: the
    cuDNN path's backward raises when ("disp", 1) is in the loss.)"""

    @staticmethod
    def forward(ctx, ll):
        return ll // 2

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return torch.zeros_like(g)


def _amax(dev):
    return torch.zeros(1, dtype=torch.float32, device=dev)


def conv(x0, amax0, x1, weight, bias, n, h, w, taps=9, pad=PAD_REFLECT, act=ACT_NONE, act_param=0.0, shift0=0):
    """One differentiable decoder convolution on rows -> (y rows, device scalar max |y|)."""
    amax_out = _amax(x0.device)
    y = _ConvRowsFn.apply(x0, x1, weight, bias, (n, h, w, taps, pad, act, act_param, shift0, amax0, amax_out))
    return y, amax_out


def to_rows(x):
    """Differentiable NCHW -> rows with the map's max |x| -> (rows, amax)."""
    amax = _amax(x.device)
    return _ToRowsFn.apply(x, amax), amax


def to_nchw(rows, n, c, h, w):
    return _ToNchwFn.apply(rows, n, c, h, w)


def _block_diag_3x3(weights):
    """(sum co, sum ci, 3, 3) weight of independent 3x3 heads that read consecutive channel ranges of one row tensor."""
    ctot = sum(int(wt.shape[1]) for wt in weights)
    parts, off = [], 0
    for wt in weights:
        ci = int(wt.shape[1])
        parts.append(F.pad(wt, (0, 0, 0, 0, off, ctot - off - ci)))
        off += ci
    return torch.cat(parts, 0)


def kitti_forward(dec, feats):
    """DepthWaveProgressiveDecoder's outputs (the reference's keys) with every convolution on libwmd, differentiable."""
    out = {}
    n = int(feats[-1].shape[0])
    h, w = (int(v) for v in feats[4].shape[2:])
    x, x_amax = to_rows(feats[4])
    yl = None
    for i in range(4, 0, -1):
        conv0 = dec.convs[("upconv", i, 0)].conv.conv
        conv1 = dec.convs[("upconv", i, 1)].conv.conv
        xa, a_amax = conv(x, x_amax, None, conv0.weight, conv0.bias, n, h, w, act=ACT_ELU)
        skip = feats[i - 1] if dec.use_skips else None
        xb, b_amax = conv(xa, a_amax, skip, conv1.weight, conv1.bias, n, 2 * h, 2 * w, act=ACT_ELU, shift0=1)
        h, w = 2 * h, 2 * w
        # the level's coefficient heads: their 1x1 stages as one launch, their 3x3 stages as one block-diagonal launch
        names = ([0] if i == 4 else []) + [1, -1]
        s1 = [dec.convs[("waveconv", i, j)][0].conv for j in names]
        s3 = [dec.convs[("waveconv", i, j)][2].conv for j in names]
        t, t_amax = conv(xb, b_amax, None, torch.cat([m.weight for m in s1], 0), torch.cat([m.bias for m in s1], 0),
                         n, h, w, taps=1, act=ACT_LRELU, act_param=0.1)
        cz = sum(int(m.weight.shape[0]) for m in s3)
        z, _ = conv(t, t_amax, None, _block_diag_3x3([m.weight for m in s3]), torch.cat([m.bias for m in s3], 0),
                    n, h, w, act=ACT_SIGMOID)
        sig = to_nchw(z, n, cz, h, w)
        k = 0
        if i == 4:
            yl = 2 ** i * sig[:, 0:1]
            k = 1
        yh = (2 ** (i - 1) * sig[:, k:k + 3] - 2 ** (i - 1) * sig[:, k + 3:k + 6]).unsqueeze(1)
        out[("wavelets", i - 1, "LL")] = yl
        out[("wavelets", i - 1, "LH")] = yh[:, :, 0]
        out[("wavelets", i - 1, "HL")] = yh[:, :, 1]
        out[("wavelets", i - 1, "HH")] = yh[:, :, 2]
        yl = dec.inverse_wt((yl, [yh]))
        out[("disp", i - 1)] = torch.clamp(yl / 2 ** (i - 1), 0, 1)
        x, x_amax = xb, b_amax
    return out


def nyu_forward(dec, blocks):
    """DecoderWave's / DecoderWave224's outputs (the reference's keys) with every convolution on libwmd, differentiable.

    Follows the decoder's level table (nyu_decoders._NyuWaveBase._LEVELS).  A "floor" level's ("disp", s) is ll // 2
    with a zero gradient (_FloorHalfFn)."""
    out = {}
    n, _, h, w = (int(v) for v in blocks[-1].shape)
    x, x_amax = to_rows(blocks[-1])
    c = dec.conv2.conv
    d, d_amax = conv(x, x_amax, None, c.weight, c.bias, n, h, w, pad=PAD_REPLICATE)
    c = dec.up1.convA.conv
    d, d_amax = conv(d, d_amax, blocks[-2], c.weight, c.bias, n, 2 * h, 2 * w, act=ACT_LRELU, act_param=0.2, shift0=1)
    h, w = 2 * h, 2 * w
    ll_scale, ll_disp = dec._LL_HEAD
    c = dec.wave1_ll.conv
    ll = ll_scale * to_nchw(conv(d, d_amax, None, c.weight, c.bias, n, h, w, pad=PAD_REPLICATE)[0], n, 1, h, w)
    if ll_disp is not None:
        out[("disp", ll_disp)] = ll / ll_scale
    out[("wavelets", dec._LEVELS[0][1], "LL")] = ll
    for j, s, disp_form in dec._LEVELS:
        if j > 1:
            c = getattr(dec, "up%d" % j).convA.conv
            d, d_amax = conv(d, d_amax, blocks[-1 - j], c.weight, c.bias, n, 2 * h, 2 * w, act=ACT_LRELU, act_param=0.2,
                             shift0=1)
            h, w = 2 * h, 2 * w
        c = getattr(dec, "wave%d" % j).conv
        hc = to_nchw(conv(d, d_amax, None, c.weight, c.bias, n, h, w, pad=PAD_ZERO)[0], n, 3, h, w).unsqueeze(1)
        if s:
            hc = 2 ** s * hc
        for k, band in enumerate(("LH", "HL", "HH")):
            out[("wavelets", s, band)] = hc[:, :, k]
        ll = dec.iwt((ll, [hc]))
        if disp_form == "floor":
            out[("disp", s)] = _FloorHalfFn.apply(ll)
        else:
            out[("disp", s)] = ll / 2 ** s if s else ll
    return out


def kitti_baseline_forward(dec, feats):
    """DepthDecoder's outputs with every convolution on libwmd, differentiable: ELU ConvBlocks with zero padding,
    reflection-padded dispconvs with the sigmoid in their epilogue.  Levels finer than the finest requested scale are
    not run (no output depends on them)."""
    out = {}
    n = int(feats[-1].shape[0])
    h, w = (int(v) for v in feats[4].shape[2:])
    x, x_amax = to_rows(feats[4])
    cout = int(dec.num_output_channels)
    for i in range(4, min(dec.scales) - 1, -1):
        conv0 = dec.convs[("upconv", i, 0)].conv.conv
        conv1 = dec.convs[("upconv", i, 1)].conv.conv
        xa, a_amax = conv(x, x_amax, None, conv0.weight, conv0.bias, n, h, w, pad=PAD_ZERO, act=ACT_ELU)
        skip = feats[i - 1] if (dec.use_skips and i > 0) else None
        x, x_amax = conv(xa, a_amax, skip, conv1.weight, conv1.bias, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_ELU, shift0=1)
        h, w = 2 * h, 2 * w
        if i in dec.scales:
            d = dec.convs[("dispconv", i)].conv
            z, _ = conv(x, x_amax, None, d.weight, d.bias, n, h, w, pad=PAD_REFLECT, act=ACT_SIGMOID)
            out[("disp", i)] = to_nchw(z, n, cout, h, w)
    return out


def nyu_baseline_forward(dec, blocks):
    """Decoder's / Decoder224's ("disp", 0) with every convolution on libwmd, differentiable (zero padding throughout)."""
    n, _, h, w = (int(v) for v in blocks[4].shape)
    x, x_amax = to_rows(blocks[4])
    c = dec.conv2.conv
    x, x_amax = conv(x, x_amax, None, c.weight, c.bias, n, h, w, pad=PAD_ZERO)
    for k in range(1, 5):
        c = getattr(dec, "up%d" % k).convA.conv
        x, x_amax = conv(x, x_amax, blocks[4 - k], c.weight, c.bias, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_LRELU,
                         act_param=0.2, shift0=1)
        h, w = 2 * h, 2 * w
    if dec._extra_stage:
        c = dec.conv5[0].conv
        x, x_amax = conv(x, x_amax, None, c.weight, c.bias, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_LRELU, act_param=0.2,
                         shift0=1)
        h, w = 2 * h, 2 * w
    z, _ = conv(x, x_amax, None, dec.conv3.weight, dec.conv3.bias, n, h, w, pad=PAD_ZERO)
    return {("disp", 0): to_nchw(z, n, 1, h, w)}
