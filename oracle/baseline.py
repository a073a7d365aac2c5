"""Oracle: the baseline (non-wavelet) depth decoders, restated functionally on torch-CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py).
* ``kitti_baseline_forward``  KITTI/networks/decoders/depth_decoder.py:18-69 (monodepth2's DepthDecoder).  Its ConvBlocks
  pad with ZEROS (``use_refl=False`` by default, KITTI/layers.py:123), its dispconvs (``Conv3x3``) by REFLECTION
  (layers.py:149).
* ``nyu_baseline_forward``  NYUv2/networks/decoders/densedepth_decoder.py:15-47 (Decoder) and, with ``extra_stage``,
  :50-89 (Decoder224).  Every convolution pads with zeros; conv2 and conv3 have no activation.
Parameters are plain state dicts with the reference's key names, as for oracle.kitti / oracle.nyu, whose building
blocks these reuse.  Pinned against the unmodified reference by oracle/pin_baseline.py.
"""
import torch
import torch.nn.functional as F

from . import kitti as okitti
from . import nyu as onyu

NUM_CH_DEC = okitti.NUM_CH_DEC


def kitti_slots(scales):
    """Index of each module in the DepthDecoder's ModuleList (depth_decoder.py:32-48): upconv(i,0), upconv(i,1) for
    i = 4..0, then the dispconvs in the order of ``scales``."""
    slots = {}
    for i in range(4, -1, -1):
        slots[("upconv", i, 0)] = 2 * (4 - i)
        slots[("upconv", i, 1)] = 2 * (4 - i) + 1
    for k, s in enumerate(scales):
        slots[("dispconv", s)] = 10 + k
    return slots


def _kitti_conv(params, k):
    """ConvBlock k's convolution (``decoder.k.conv.conv``); a dispconv is a bare Conv3x3 (``decoder.k.conv``)."""
    if "decoder.%d.conv.weight" % k in params:
        return params["decoder.%d.conv.weight" % k], params["decoder.%d.conv.bias" % k]
    return params["decoder.%d.conv.conv.weight" % k], params["decoder.%d.conv.conv.bias" % k]


def _conv3_zero(x, w, b):
    return F.conv2d(F.pad(x, (1, 1, 1, 1)), w, b)


def kitti_baseline_forward(params, feats, scales=range(4), use_skips=True):
    """DepthDecoder.forward (depth_decoder.py:51-69): ELU ConvBlocks with zero padding, sigmoid of a reflection-padded
    dispconv at every requested scale."""
    slots = kitti_slots(scales)
    out = {}
    x = feats[-1]
    for i in range(4, -1, -1):
        x = F.elu(_conv3_zero(x, *_kitti_conv(params, slots[("upconv", i, 0)])))
        x = [okitti._up2(x)]
        if use_skips and i > 0:
            x += [feats[i - 1]]
        x = F.elu(_conv3_zero(torch.cat(x, 1), *_kitti_conv(params, slots[("upconv", i, 1)])))
        if i in scales:
            out[("disp", i)] = torch.sigmoid(okitti._conv3_reflect(x, *_kitti_conv(params, slots[("dispconv", i)])))
    return out


def nyu_baseline_forward(params, blocks, extra_stage=False):
    """Decoder.forward (densedepth_decoder.py:36-47); with extra_stage, Decoder224.forward (:78-89): nearest x2, conv5 +
    LeakyReLU(0.2), then conv3."""
    x = _conv3_zero(blocks[4], *onyu._p(params, "conv2"))
    for k in range(1, 5):
        x = torch.cat([okitti._up2(x), blocks[4 - k]], 1)
        x = F.leaky_relu(_conv3_zero(x, *onyu._p(params, "up%d.convA" % k)), 0.2)
    if extra_stage:
        x = F.leaky_relu(_conv3_zero(okitti._up2(x), *onyu._p(params, "conv5.0")), 0.2)
    return {("disp", 0): _conv3_zero(x, params["conv3.weight"], params["conv3.bias"])}
