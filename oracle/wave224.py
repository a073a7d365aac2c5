"""Oracle: the two dense wavelet decoders oracle.nyu and oracle.kitti do not restate, on torch-CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py).
* ``nyu224_dense_forward``  NYUv2/networks/decoders/densedepth_decoder.py:151-221 (DecoderWave224), the four-level
  decoder NYUv2/model.py:47-57 builds for ``--use_224``.
* ``kitti_dense_noskip_forward``  KITTI/networks/decoders/depth_decoder.py:72-168 (DepthWaveProgressiveDecoder) with
  ``use_skips=False``: only the coarsest feature map is read (:145-148).
Parameters are plain state dicts with the reference's key names, as for oracle.nyu / oracle.kitti, whose building
blocks these reuse.  Pinned against the unmodified reference by oracle/pin_wave224.py.
"""
import torch

from . import kitti as okitti
from . import nyu as onyu


def nyu224_dense_forward(params, blocks):
    """DecoderWave224.forward (densedepth_decoder.py:181-221): four IDWT levels, LL scaled by 2**4, detail scales 8,
    4, 2, 1; ("disp", 3) taken after the first IDWT and ("disp", 1) FLOOR-divided (:212), as the reference does."""
    out = {}
    d = onyu._up_block(params, "up1", onyu._conv3(blocks[-1], *onyu._p(params, "conv2"), "replicate"), blocks[-2])
    ll = (2 ** 4) * onyu._conv3(d, *onyu._p(params, "wave1_ll"), "replicate")
    out[("wavelets", 3, "LL")] = ll
    for k in range(1, 5):
        s = 4 - k
        if k > 1:
            d = onyu._up_block(params, "up%d" % k, d, blocks[-1 - k])
        h = onyu._conv3(d, *onyu._p(params, "wave%d" % k), "zero").unsqueeze(1)
        if s:
            h = (2 ** s) * h
        for j, band in enumerate(("LH", "HL", "HH")):
            out[("wavelets", s, band)] = h[:, :, j]
        ll = onyu._idwt(ll, h)
        out[("disp", s)] = ll // 2 if s == 1 else ll / (2 ** s)
    return out


def kitti_dense_noskip_forward(params, feats):
    """DepthWaveProgressiveDecoder(use_skips=False).forward (depth_decoder.py:138-168): upconv(i,1) reads only the
    upsampled upconv(i,0) output."""
    out = {}
    x = feats[-1]
    yl = None
    for i in range(4, 0, -1):
        x = okitti._conv_block(x, *okitti._block(params, okitti.slot(i, "upconv0")))
        x = okitti._conv_block(okitti._up2(x), *okitti._block(params, okitti.slot(i, "upconv1")))
        if i == 4:
            yl = (2 ** i) * torch.sigmoid(okitti._dense_head(x, *okitti._head(params, okitti.slot(i, "ll"))))
        pos = torch.sigmoid(okitti._dense_head(x, *okitti._head(params, okitti.slot(i, "pos"))))
        neg = torch.sigmoid(okitti._dense_head(x, *okitti._head(params, okitti.slot(i, "neg"))))
        yh = (2 ** (i - 1)) * pos.unsqueeze(1) - (2 ** (i - 1)) * neg.unsqueeze(1)   # :133-135
        out[("wavelets", i - 1, "LL")] = yl
        out[("wavelets", i - 1, "LH")] = yh[:, :, 0]
        out[("wavelets", i - 1, "HL")] = yh[:, :, 1]
        out[("wavelets", i - 1, "HH")] = yh[:, :, 2]
        yl = okitti._idwt(yl, yh)
        out[("disp", i - 1)] = torch.clamp(yl / 2 ** (i - 1), 0, 1)
    return out
