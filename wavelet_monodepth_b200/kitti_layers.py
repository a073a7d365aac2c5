"""KITTI layer / op library of the decoder hot path, on libwmd kernels.

Mirrors the public names and signatures of the reference's KITTI/layers.py:120-173,
233-236,335-508 (``ConvBlock``, ``Conv3x3``, ``Conv1x1``, ``upsample`` and the functional
``sparse_*`` ops) so code written against the reference reads the same here.

* The module classes keep the reference's sub-module structure (``.conv.conv.weight`` ...), so
  state dicts are interchangeable and ``pyt_utils.group_weight`` (KITTI/pyt_utils.py:12-29) still
  finds only Conv2d parameters.  Their ``forward`` is the dense, differentiable path (cuDNN) used
  for training; the decoders bypass it at inference and run the native gather-GEMM kernels.
* The functional ops keep the reference's batch-1 wire format (flat channel-major ``xvals``, int64
  ``xidxmap``, (1,1,H,W) masks) at their boundary and convert to the native pixel-major row layout
  inside; they exist for drop-in compatibility (the notebooks and the NYUv2 decoder call them
  directly).  The decoders do not go through them: they stay in the native layout end to end.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from ._lib import PAD_BY_NAME, WmdError


class Conv3x3(nn.Module):
    """Pad (reflect or zero) and convolve.  [KITTI/layers.py:146-161]"""

    def __init__(self, in_channels, out_channels, use_refl=True, stride=1, use_bias=True):
        super().__init__()
        self.pad = nn.ReflectionPad2d(1) if use_refl else nn.ZeroPad2d(1)
        self.conv = nn.Conv2d(int(in_channels), int(out_channels), 3, stride=stride, bias=use_bias)
        self.use_refl = bool(use_refl)

    def forward(self, x):
        return self.conv(self.pad(x))


class Conv1x1(nn.Module):
    """[KITTI/layers.py:164-173]"""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv = nn.Conv2d(int(in_channels), int(out_channels), 1, stride=1, padding=0)

    def forward(self, x):
        return self.conv(x)


class ConvBlock(nn.Module):
    """Convolution followed by ELU.  [KITTI/layers.py:120-143]"""

    def __init__(self, in_channels, out_channels, kernel_size=3, norm_layer=None, use_refl=False):
        super().__init__()
        if kernel_size == 3:
            self.conv = Conv3x3(in_channels, out_channels, use_refl=use_refl)
        elif kernel_size == 1:
            self.conv = Conv1x1(in_channels, out_channels)
        else:
            raise NotImplementedError
        self.nonlin = nn.ELU(inplace=True)
        self.norm_layer = norm_layer(out_channels) if norm_layer is not None else nn.Identity()

    def forward(self, x):
        return self.nonlin(self.norm_layer(self.conv(x)))


def upsample(x):
    """Nearest x2.  [KITTI/layers.py:233-236]"""
    return F.interpolate(x, scale_factor=2, mode="nearest")


# ----------------------------------------------------------------------------------------------
# functional sparse ops, reference wire format at the boundary
# ----------------------------------------------------------------------------------------------
def _single(mask):
    assert mask.shape[0] == 1 and mask.shape[1] == 1          # layers.py:372-373,383-384
    return mask


def _mask_u8(mask):
    m = mask if mask.dtype == torch.bool else (mask > 0.5)
    return m.to(torch.uint8).contiguous()


def _cm_to_rows(xvals, chn):
    """flat channel-major (C*M,) -> rows (M, pad4(C))."""
    m = xvals.numel() // chn
    if m == 0:
        return torch.zeros((1, ops.pad4(chn)), dtype=torch.float32, device=xvals.device), 0
    return ops.nchw_to_rows(xvals.reshape(1, chn, m, 1)), m


def _rows_to_cm(rows, chn, m):
    if m == 0:
        return torch.zeros((0,), dtype=torch.float32, device=rows.device)
    return ops.rows_to_nchw(rows[:m], 1, chn, m, 1).reshape(-1)


def _act_of(nonlin):
    """Translate the reference's nonlinearity argument into a libwmd activation code."""
    from ._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID
    if nonlin is None or isinstance(nonlin, nn.Identity):
        return ACT_NONE, 0.0
    if isinstance(nonlin, nn.ELU):
        if nonlin.alpha != 1.0:
            raise NotImplementedError("ELU alpha != 1")
        return ACT_ELU, 0.0
    if isinstance(nonlin, nn.LeakyReLU):
        return ACT_LRELU, float(nonlin.negative_slope)
    if isinstance(nonlin, nn.Sigmoid) or nonlin is torch.sigmoid:
        return ACT_SIGMOID, 0.0
    raise NotImplementedError("unsupported nonlinearity for the native sparse conv: %r" % (nonlin,))


def mask2yx(mask):
    """(2, M) int64 row/col of active pixels, row-major.  [KITTI/layers.py:371-379]"""
    _single(mask)
    h, w = mask.shape[2:]
    _, pixels, offsets = ops.compact(_mask_u8(mask), want_idxmap=False)
    m = int(offsets[1])
    p = pixels[:m].long()
    return torch.stack([p // w, p % w], 0)


def mask2idxmap(xmask):
    """(1,1,H,W) int64 index map (-1 inactive) and the reference's op count H*W.  [KITTI/layers.py:382-389]"""
    _single(xmask)
    idxmap, _, _ = ops.compact(_mask_u8(xmask), want_pixels=False)
    return idxmap.long().reshape(1, 1, *xmask.shape[2:]), xmask.shape[2] * xmask.shape[3]


def make_result(xvals, xchn, mask):
    """Scatter sparse values to a dense (1,C,H,W) map.  [KITTI/layers.py:365-368]"""
    _single(mask)
    h, w = mask.shape[2:]
    _, pixels, offsets = ops.compact(_mask_u8(mask), want_idxmap=False)
    rows, m = _cm_to_rows(xvals, xchn)
    return ops.scatter_rows(rows, xchn, pixels, offsets[1:], 1, h, w, max_rows=min(rows.shape[0], h * w))


def sparse_select(xvals, xchn, xidxmap, ymask, ufactor=1, pad=False):
    """Re-index sparse features onto ``ymask``'s active set.  [KITTI/layers.py:337-362]

    Misses read a zero row (the reference's pad=True; without pad the reference would fault).
    """
    from ._lib import ACT_NONE, PAD_ZERO
    xh, xw = xidxmap.shape[2:]
    yh, yw = ymask.shape[2:]
    assert xh * ufactor == yh and xw * ufactor == yw
    rows, _ = _cm_to_rows(xvals, xchn)
    _, pixels, offsets = ops.compact(_mask_u8(ymask), want_idxmap=False)
    eye = _identity_weight(xchn, rows.device)
    out = ops.conv_rows(rows, xchn, eye, None, xchn, 1, yh, yw, taps=1, pad=PAD_ZERO, act=ACT_NONE,
                        map0=xidxmap.reshape(1, xh, xw).to(torch.int32).contiguous(),
                        shift0=1 if ufactor == 2 else 0, pixels=pixels, count=offsets[1:])
    return _rows_to_cm(out, xchn, int(offsets[1]))


_eye_cache = {}


def _identity_weight(c, device, c1=0):
    # exact copies need the fp32 FMA engine (1.0 * x + 0 is exact; a tf32 split is not a copy)
    key = (c, c1, str(device))
    if key not in _eye_cache:
        _eye_cache[key] = ops.pack_weight(torch.eye(c, device=device).reshape(c, c, 1, 1), c1, kind="simt")
    return _eye_cache[key]


def sparse_conv1x1(conv_layer, xvals, nonlin):
    """Per-active-pixel 1x1 convolution.  [KITTI/layers.py:392-406]  Returns (vals (Cout,M), Cout, ops)."""
    if not isinstance(conv_layer, Conv1x1):
        raise NotImplementedError()
    wt, bias = conv_layer.conv.weight, conv_layer.conv.bias
    ochn, ichn = wt.shape[:2]
    rows, m = _cm_to_rows(xvals, ichn)
    act, ap = _act_of(nonlin)
    wp = ops.pack_weight(wt, precision="tf32x3")     # no source maxima here: tf32x3 operands, no fp16-pair image
    out = ops.conv_rows(rows, ichn, wp, bias.detach(), ochn, 1, 1, max(m, 1), taps=1, act=act,
                        act_param=ap, max_rows=m)
    return _rows_to_cm(out, ochn, m).reshape(ochn, m), ochn, m * ichn * ochn + m * ochn


def sparse_conv3x3(conv_layer, xvals, xidxmap, mask, nonlin=nn.Identity(), padding="reflect", make_result=True):
    """Sparse 3x3 convolution.  [KITTI/layers.py:409-480]

    Same dispatch as the reference: ``Conv3x3`` -> (W,b); ``ConvBlock`` -> its conv and ITS OWN ELU;
    ``nn.Sequential(Conv1x1, LeakyReLU, Conv3x3)`` -> 1x1 over all active inputs first.
    """
    ops_count = 0
    if isinstance(conv_layer, ConvBlock):
        nonlin = conv_layer.nonlin
        conv_layer = conv_layer.conv
    if isinstance(conv_layer, nn.Sequential):
        if isinstance(conv_layer[0], Conv1x1):
            mid, ichn, ops_count = sparse_conv1x1(conv_layer[0], xvals, conv_layer[1])
            xvals = mid.reshape(-1)
        conv = conv_layer[2].conv
    elif hasattr(conv_layer, "conv") and isinstance(conv_layer.conv, nn.Conv2d):
        conv = conv_layer.conv
    else:
        raise NotImplementedError()
    ochn, ichn = conv.weight.shape[:2]
    h, w = mask.shape[2:]
    if padding not in PAD_BY_NAME:
        raise WmdError("unknown padding %r" % (padding,))
    rows, _ = _cm_to_rows(xvals, ichn)
    _, pixels, offsets = ops.compact(_mask_u8(mask), want_idxmap=False)
    act, ap = _act_of(nonlin)
    wp = ops.pack_weight(conv.weight, precision="tf32x3")     # no source maxima here: tf32x3 operands
    out = ops.conv_rows(rows, ichn, wp, conv.bias.detach(), ochn, 1, h, w, taps=9,
                        pad=PAD_BY_NAME[padding], act=act, act_param=ap,
                        map0=xidxmap.reshape(1, h, w).to(torch.int32).contiguous(), pixels=pixels, count=offsets[1:])
    m_out = int(offsets[1])
    ops_count += ichn * 9 * m_out + (1 + 9 * ichn) * m_out * ochn
    if make_result:
        return ops.scatter_rows(out, ochn, pixels, offsets[1:], 1, h, w), ops_count
    return _rows_to_cm(out, ochn, m_out), ochn, ops_count


def sparse_upsample(xvals, xchn, xidxmap, skip, mask, make_result=True):
    """Nearest x2 of sparse features + skip concat at ``mask``.  [KITTI/layers.py:483-508]"""
    from ._lib import ACT_NONE, PAD_ZERO
    xh, xw = xidxmap.shape[2:]
    oh, ow = 2 * xh, 2 * xw
    cs = skip.shape[1]
    ochn = xchn + cs
    rows, _ = _cm_to_rows(xvals, xchn)
    _, pixels, offsets = ops.compact(_mask_u8(mask), want_idxmap=False)
    # identity 1x1 over the concatenated (upsampled | skip) channels
    eye = _identity_weight(ochn, rows.device, cs)
    out = ops.conv_rows(rows, xchn, eye, None, ochn, 1, oh, ow, taps=1, pad=PAD_ZERO, act=ACT_NONE,
                        map0=xidxmap.reshape(1, xh, xw).to(torch.int32).contiguous(), shift0=1,
                        x1=ops.nchw_to_rows(skip), c1=cs, pixels=pixels, count=offsets[1:])
    m = int(offsets[1])
    if make_result:
        return ops.scatter_rows(out, ochn, pixels, offsets[1:], 1, oh, ow)
    return _rows_to_cm(out, ochn, m), ochn
