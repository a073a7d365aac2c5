"""KITTI depth decoders with the reference's constructor / forward / state-dict contract, on libwmd.

Mirrors KITTI/networks/decoders/depth_decoder.py:
  * ``DepthDecoder``                       (:18-69)   baseline, API surface only (cuDNN convs)
  * ``DepthWaveProgressiveDecoder``        (:72-168)  dense wavelet decoder
  * ``SparseDepthWaveProgressiveDecoder``  (:171-428) threshold-gated sparse decoder

Contract kept (SURVEY 8b): ``.convs`` OrderedDict keyed by tuples, ``.decoder = ModuleList(convs.values())``
(state-dict names ``decoder.0 .. decoder.16``), ``inverse_wt`` sub-module with the IDWT tap buffers,
``forward(input_features[, thresh_ratio[, sparse_scales]]) -> dict`` with the reference's keys, ``self.outputs``.

What is different underneath (H100-native, DESIGN.md):
  * inference runs natively end to end in a pixel-major row layout: encoder maps are transposed once
    (or used zero-copy when channels_last), every conv is the gather-GEMM kernel, heads + IDWT + disp are
    fused kernels, and no intermediate dense tensor or index tensor of the reference is materialised;
  * the sparse decoder is BATCHED (the reference asserts batch 1, :297): thresholds, masks and active
    lists are per sample, rows of all samples are concatenated, counts stay on the device, and the only
    host sync is one read of the counts at the end for ``total_ops``;
  * training (grad enabled) uses the differentiable path: cuDNN convs + the native IDWT with its adjoint.
"""
import os
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import opcount, ops
from .opsfuture import OpsFuture
from ._lib import ACT_ELU, ACT_LRELU, ACT_SIGMOID, PAD_REFLECT, WmdError
from .kitti_layers import Conv1x1, Conv3x3, ConvBlock, upsample
from .wavelets import IDWT


def _version_of(t):
    try:
        return t._version
    except RuntimeError:          # inference tensors do not track versions
        return -1


class _PackCache:
    """Packed-weight cache keyed by (data_ptr, version, device) of the source parameters.

    In-place updates through autograd-visible ops (optimizer steps, ``p.mul_()``) bump the version counter and
    repack on the next forward.  Updates the counter cannot see - ``p.data.copy_()``, an EMA swap through ``.data``,
    tensors created under ``inference_mode`` - need ``invalidate()``; the decoders call it from ``_apply`` (``.to()``,
    ``.cuda()``, ``.half()``...) and from a ``load_state_dict`` post-hook, and expose it as ``invalidate_packs()``."""

    def __init__(self):
        self._c = {}

    def invalidate(self):
        self._c.clear()

    def get(self, key, tensors, build):
        ver = tuple((t.data_ptr(), _version_of(t), str(t.device)) for t in tensors)
        ent = self._c.get(key)
        if ent is None or ent[0] != ver:
            with torch.no_grad():
                ent = (ver, build())
            self._c[key] = ent
        return ent[1]


def _pm(fn):
    """Active-row counts for the profiler's byte accounting; evaluated only while a profiler is installed."""
    return fn() if ops._profiler is not None else None


_SIDE_STREAMS = {}


def _side_stream(device, which=0):
    """Side streams per device (0: layout moves, 1-2: compactions), created lazily and reused: CUDA graphs fork/join
    through them."""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device(), which)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def _need_cuda(feats, host_ok=()):
    """host_ok: indices of feature maps that may instead be pinned host tensors (read in place by the gated move)."""
    for k, f in enumerate(feats):
        if not f.is_cuda and k in host_ok and f.is_pinned():
            continue
        if not f.is_cuda:
            raise WmdError("wavelet_monodepth_b200 decoders run on CUDA tensors only: the native kernels have no "
                           "CPU fallback (got a feature map on %s)" % f.device)


class DepthDecoder(nn.Module):
    """monodepth2 baseline decoder (sigmoid disparity at 4 scales).  [depth_decoder.py:18-69]"""

    def __init__(self, num_ch_enc, scales=range(4), num_output_channels=1, use_skips=True):
        super().__init__()
        self.num_output_channels = num_output_channels
        self.use_skips = use_skips
        self.upsample_mode = "nearest"
        self.scales = scales
        self.num_ch_enc = num_ch_enc
        self.num_ch_dec = np.array([16, 32, 64, 128, 256])
        self.convs = OrderedDict()
        for i in range(4, -1, -1):
            cin = self.num_ch_enc[-1] if i == 4 else self.num_ch_dec[i + 1]
            self.convs[("upconv", i, 0)] = ConvBlock(cin, self.num_ch_dec[i])
            cin = self.num_ch_dec[i]
            if self.use_skips and i > 0:
                cin += self.num_ch_enc[i - 1]
            self.convs[("upconv", i, 1)] = ConvBlock(cin, self.num_ch_dec[i])
        for s in self.scales:
            self.convs[("dispconv", s)] = Conv3x3(self.num_ch_dec[s], self.num_output_channels)
        self.decoder = nn.ModuleList(list(self.convs.values()))
        self.sigmoid = nn.Sigmoid()

    def forward(self, input_features):
        self.outputs = {}
        x = input_features[-1]
        for i in range(4, -1, -1):
            x = self.convs[("upconv", i, 0)](x)
            x = [upsample(x)]
            if self.use_skips and i > 0:
                x += [input_features[i - 1]]
            x = self.convs[("upconv", i, 1)](torch.cat(x, 1))
            if i in self.scales:
                self.outputs[("disp", i)] = self.sigmoid(self.convs[("dispconv", i)](x))
        return self.outputs


class _WaveDecoderBase(nn.Module):
    """Shared module structure + native level engine of the two wavelet decoders."""

    def _build(self, num_ch_enc, scales, num_output_channels, use_skips):
        self.num_output_channels = num_output_channels
        self.use_skips = use_skips
        self.upsample_mode = "nearest"
        self.scales = scales
        self.num_ch_enc = num_ch_enc
        self.num_ch_dec = np.array([16, 32, 64, 128, 256])
        self.J = 1
        self.inverse_wt = IDWT(wave="haar", mode="zero")
        self.convs = OrderedDict()
        for i in range(4, 0, -1):
            c = self.num_ch_dec[i]
            cin = self.num_ch_enc[-1] if i == 4 else self.num_ch_dec[i + 1]
            self.convs[("upconv", i, 0)] = ConvBlock(cin, c, use_refl=True)
            cin = c + (self.num_ch_enc[i - 1] if self.use_skips and i > 0 else 0)
            self.convs[("upconv", i, 1)] = ConvBlock(cin, c, use_refl=True)
            if i == 4:
                self.convs[("waveconv", i, 0)] = nn.Sequential(Conv1x1(c, c // 4), nn.LeakyReLU(0.1, inplace=True),
                                                               Conv3x3(c // 4, 1, use_refl=True))
            self.convs[("waveconv", i, 1)] = nn.Sequential(Conv1x1(c, c), nn.LeakyReLU(0.1, inplace=True),
                                                           Conv3x3(c, 3, use_refl=True))
            self.convs[("waveconv", i, -1)] = nn.Sequential(Conv1x1(c, c), nn.LeakyReLU(0.1, inplace=True),
                                                            Conv3x3(c, 3, use_refl=True))
        self.decoder = nn.ModuleList(list(self.convs.values()))
        self.sigmoid = nn.Sigmoid()
        self._packs = _PackCache()
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packs())
        # optional fused consumer epilogue (not part of the reference's decoder, off by default): when set to (H, W),
        # inference also returns ("disp_full", s) = F.interpolate(("disp", s), (H, W), mode="bilinear",
        # align_corners=False) for s = 1..3 - what KITTI/trainer.py:338-339 computes from every scale - produced
        # straight from the coefficients by the fused IDWT+bilinear kernel
        self.full_res_size = None
        # run the skip maps' layout transposes on a side stream (WMD_OVERLAP_LAYOUT=0/1 sets the default)
        self.overlap_layout = os.environ.get("WMD_OVERLAP_LAYOUT", "0") == "1"
        # transpose a sparse level's skip map only under its upsample mask (WMD_GATED_LAYOUT=0/1 sets the default).  On since
        # the gated move issues all its loads before using any (72 us against 175 before and ~110 for the whole level-3 map)
        self.gated_layout = os.environ.get("WMD_GATED_LAYOUT", "1") == "1"
        # run the two 1x1 head stages of the fine levels as one fused kernel (WMD_FUSED_HEADS=0/1 sets the default)
        self.fused_heads = os.environ.get("WMD_FUSED_HEADS", "1") == "1"
        # level 4: the LL head's 3x3 stage rides in the tap-product GEMM of the +/- heads (WMD_FACTORED_LL=0/1)
        self.factored_ll = os.environ.get("WMD_FACTORED_LL", "1") == "1"
        # compactions of the level's three active sets on parallel streams (WMD_OVERLAP_COMPACTION=0/1)
        self.overlap_compaction = os.environ.get("WMD_OVERLAP_COMPACTION", "1") == "1"
        # sparse levels keep their skip map COMPACT: only the rows of the upsample mask S3 are moved out of the NCHW map
        # (list-based gather-transpose: bytes scale with the mask density, 16-50 % on the bench) and upconv(i,1) reaches them
        # through S3's index map (wmd_conv_desc.map1).  The skip map may then be a pinned HOST tensor.  WMD_COMPACT_SKIP=0/1
        self.compact_skip = os.environ.get("WMD_COMPACT_SKIP", "1") == "1"
        # ... at the levels where it pays on a device-resident map: the list-based gather moves fewer useful bytes per second
        # than the whole-map transpose (scripts/probe_gather.py), so it wins only at low mask density - levels 2 and 1
        # (16-28 % on the bench), not level 3 (50 %).  A pinned-host skip map always takes it.
        self.compact_skip_levels = tuple(int(v) for v in os.environ.get("WMD_COMPACT_SKIP_LEVELS", "1,2").split(",") if v)
        # tail of every level as one kernel: head gather-sum -> yh -> IDWT -> disp -> next level's threshold
        # (wmd_head_idwt_f32; WMD_FUSED_TAIL=0/1).  Bit-identical to the head_gather + idwt_haar + range_thresh chain.
        self.fused_tail = os.environ.get("WMD_FUSED_TAIL", "1") == "1"
        # optional consumer epilogue of ("disp", 0), off by default: (min_depth, max_depth) adds ("scaled_disp", 0) and
        # ("depth", 0) = disp_to_depth(("disp", 0), min_depth, max_depth) (KITTI/layers.py:16-25; evaluate_depth.py:193,
        # test_simple.py:151), produced by the last level's fused tail
        self.depth_range = None

    # ---- packed parameters ------------------------------------------------------------------
    def invalidate_packs(self):
        """Drop the packed copies of the weights (they are rebuilt on the next native forward).  Needed only after a
        weight update the version counters cannot see, e.g. ``p.data.copy_(...)``."""
        self._packs.invalidate()

    def _apply(self, fn, *args, **kwargs):
        if hasattr(self, "_packs"):
            self._packs.invalidate()
        return super()._apply(fn, *args, **kwargs)

    def _upconv(self, i, j):
        conv = self.convs[("upconv", i, j)].conv.conv
        c1 = int(self.num_ch_enc[i - 1]) if j == 1 else 0          # upconv(i,1) reads the skip map as gather source 1
        kind = ops.default_conv_kind()
        return self._packs.get(("upconv", i, j, kind), [conv.weight], lambda: ops.pack_weight(conv.weight, c1)), conv.bias.detach()

    def _head_1x1(self, i):
        """Concatenated 1x1 stages of the level's heads: [LL (i==4) | + | -] -> (packed (C, ld), bias, offsets)."""
        names = ([0] if i == 4 else []) + [1, -1]
        convs = [self.convs[("waveconv", i, j)][0].conv for j in names]
        wts = [c.weight for c in convs]
        packed = self._packs.get(("head1x1", i, ops.default_conv_kind()), wts,
                                 lambda: ops.pack_weight(torch.cat([w.detach() for w in wts], 0)))
        bias = self._packs.get(("head1x1b", i), [c.bias for c in convs],
                               lambda: torch.cat([c.bias.detach() for c in convs], 0).contiguous())
        offs, run = {}, 0
        for j, c in zip(names, convs):
            offs[j] = run
            run += c.weight.shape[0]
        return packed, bias, offs, run

    def _head_taps(self, i, offs, ctot):
        """Factored +/- 3x3 stage: packed (54, ctot) tap-product weight and the 6 biases [+ | -].

        With factored_ll, level 4 appends the LL head's nine tap filters as columns 54..62 (same 64-wide GEMM tile)."""
        cp, cn = self.convs[("waveconv", i, 1)][2].conv, self.convs[("waveconv", i, -1)][2].conv
        kind = ops.default_conv_kind()
        if i == 4 and self.factored_ll:
            cl = self.convs[("waveconv", i, 0)][2].conv
            wz = self._packs.get(("headtaps+ll", i, kind), [cp.weight, cn.weight, cl.weight],
                                 lambda: ops.pack_weight(torch.cat([
                                     ops.head_tap_weight([cp.weight, cn.weight], [offs[1], offs[-1]], ctot),
                                     ops.head_tap_weight([cl.weight], [offs[0]], ctot)], 0)))
            bz = self._packs.get(("headtapsb", i), [cp.bias, cn.bias],
                                 lambda: torch.cat([cp.bias.detach(), cn.bias.detach()]).contiguous())
            return wz, bz
        wz = self._packs.get(("headtaps", i, kind), [cp.weight, cn.weight],
                             lambda: ops.pack_weight(ops.head_tap_weight([cp.weight, cn.weight], [offs[1], offs[-1]], ctot)))
        bz = self._packs.get(("headtapsb", i), [cp.bias, cn.bias],
                             lambda: torch.cat([cp.bias.detach(), cn.bias.detach()]).contiguous())
        return wz, bz

    def _head_mlp(self, i):
        """Fused 1x1 stages of the + / - heads (levels without an LL head): packed [W1 | Wz | b1] image or None."""
        c = int(self.num_ch_dec[i])
        if i == 4 or not self.fused_heads or not ops.head_mlp_supported(c, 2 * c):
            return None
        c1p, c1n = self.convs[("waveconv", i, 1)][0].conv, self.convs[("waveconv", i, -1)][0].conv
        c3p, c3n = self.convs[("waveconv", i, 1)][2].conv, self.convs[("waveconv", i, -1)][2].conv
        return self._packs.get(("headmlp", i), [c1p.weight, c1n.weight, c1p.bias, c1n.bias, c3p.weight, c3n.weight],
                               lambda: ops.pack_head_mlp(torch.cat([c1p.weight.detach(), c1n.weight.detach()], 0),
                                                         torch.cat([c1p.bias.detach(), c1n.bias.detach()], 0),
                                                         ops.head_tap_weight([c3p.weight, c3n.weight], [0, c], 2 * c)))

    def _head_3x3(self, i, j):
        conv = self.convs[("waveconv", i, j)][2].conv
        return self._packs.get(("head3x3", i, j), [conv.weight], lambda: ops.pack_head_weight(conv.weight)), conv.bias.detach()

    # ---- native engine ------------------------------------------------------------------------
    @torch.no_grad()
    def _native_forward(self, feats, thresh_ratio, sparse_levels, with_masks):
        """Runs levels 4..1 on libwmd.  sparse_levels: set of levels i executed on active lists.

        Returns (outputs, counts): counts = int32 device tensor (levels, 3, N+1) with the row offsets of the compacted
        sets S2, S4, S5 of every sparse level, sparse levels in descending order (None without sparse levels)."""
        dev = next(f.device for f in feats if f.is_cuda) if any(f.is_cuda for f in feats) else None
        if dev is not None and dev.index is not None and dev.index != torch.cuda.current_device():
            with torch.cuda.device(dev):       # libwmd launches on the current device: make the tensors' device current
                return self._native_forward_on_device(feats, thresh_ratio, sparse_levels, with_masks)
        return self._native_forward_on_device(feats, thresh_ratio, sparse_levels, with_masks)

    def _empty_outputs(self, feats, sparse_levels, with_masks):
        """Outputs of an empty batch (a rank whose shard is empty: world size > batch) - right keys, N = 0."""
        dev = feats[-1].device
        out = {}
        h, w = (int(v) for v in feats[4].shape[2:])
        for i in range(4, 0, -1):
            if with_masks:
                for name, up in (("lowres_mask", 0), ("upconv0_mask", 0), ("upsample_mask", 1), ("upconv1_mask", 1),
                                 ("wavelet_mask", 1)):
                    out[(name, i - 1)] = torch.zeros((0, 1, h << up, w << up), dtype=torch.bool, device=dev)
            for band in ("LL", "LH", "HL", "HH"):
                out[("wavelets", i - 1, band)] = torch.zeros((0, 1, 2 * h, 2 * w), dtype=torch.float32, device=dev)
            out[("disp", i - 1)] = torch.zeros((0, 1, 4 * h, 4 * w), dtype=torch.float32, device=dev)
            h, w = 2 * h, 2 * w
        counts = torch.zeros((len(sparse_levels), 3, 1), dtype=torch.int32, device=dev) if sparse_levels else None
        return out, counts

    def _native_forward_on_device(self, feats, thresh_ratio, sparse_levels, with_masks):
        # with gated_layout the skip map of a sparse level i (feats[i-1]) may live in pinned host memory
        _need_cuda(feats, host_ok=tuple(i - 1 for i in sparse_levels) if (self.gated_layout or self.compact_skip) else ())
        out = {}
        n = feats[-1].shape[0]
        dev = feats[-1].device
        if n == 0:
            return self._empty_outputs(feats, sparse_levels, with_masks)
        # max |x| of every tensor a tensor-core conv reads (device scalars, zeroed here, raised by the producers): the
        # fp16-pair operand form scales by a power of two chosen from them (ops.default_conv_precision)
        track = ops.default_conv_precision() == "f16x3"
        amax = torch.zeros(24, dtype=torch.float32, device=dev) if track else None
        slot = (lambda k: amax[k:k + 1]) if track else (lambda k: None)
        x_rows, x_c, prev_map = ops.nchw_to_rows(feats[4], amax=slot(0)), feats[4].shape[1], None
        x_amax = slot(0)
        # layout moves of the skip maps (NCHW -> pixel-major rows), two options on top of the plain in-order transpose:
        #  gated_layout   a sparse level reads its skip map only under the upsample mask S3 (sparse_upsample:
        #                 skip[mask], layers.py:500), so only those rows are produced - the move scales with density;
        #  overlap_layout the move runs on a side stream next to the level's upconv(i,0), which does not need it
        #                 (HBM-bound transposes fill the tails of the tensor-bound convolution), joined by an event.
        side = _side_stream(dev) if self.overlap_layout else None
        h, w = feats[4].shape[2:]
        yl = yh = None
        counts = {}
        next_thresh = None                 # per-sample threshold of the coming level, when the fused tail produced it
        for i in range(4, 0, -1):
            c = int(self.num_ch_dec[i])
            sparse = i in sparse_levels
            skip = feats[i - 1]
            cs = skip.shape[1]
            if tuple(skip.shape[2:]) != (2 * h, 2 * w):
                raise WmdError("skip feature %d has shape %s, expected spatial %s" % (i - 1, tuple(skip.shape), (2 * h, 2 * w)))
            masks = None
            if with_masks:
                if i == 4:
                    masks = ops.level_masks(None, None, n=n, h=h, w=w, device=dev)
                else:
                    thresh = next_thresh if next_thresh is not None else ops.range_thresh(yl, thresh_ratio)
                    masks = ops.level_masks(yh, thresh)
            skip_gate = masks["S3"] if (sparse and self.gated_layout) else None
            skip_done = None
            map3 = None
            if sparse and self.compact_skip and (i in self.compact_skip_levels or not skip.is_cuda) and \
                    ops.rows_view(skip) is None:                         # channels_last maps are used in place instead
                # S3's compaction and the gather of exactly its rows, on a side stream next to gate_map / compact(S2) / upconv(i,0)
                s3 = _side_stream(dev, 3) if self.overlap_compaction else None
                if s3 is not None:
                    (map3, pix3, off3), _ = ops.compact(masks["S3"], stream=s3, ws_slot=3)
                    skip_rows, skip_done = ops.gather_rows_list(skip, pix3, off3[n:], stream=s3, amax=slot(i))
                else:
                    map3, pix3, off3 = ops.compact(masks["S3"], ws_slot=3)
                    skip_rows = ops.gather_rows_list(skip, pix3, off3[n:], amax=slot(i))
                skip_amax = slot(i)
            else:
                skip_amax = slot(i)
                if side is not None:
                    skip_rows, skip_done = ops.nchw_to_rows(skip, stream=side, gate=skip_gate, amax=skip_amax)
                else:
                    skip_rows = ops.nchw_to_rows(skip, gate=skip_gate, amax=skip_amax)
            if with_masks:
                for name, key in (("lowres_mask", "S1"), ("upconv0_mask", "S2"), ("upsample_mask", "S3"),
                                  ("upconv1_mask", "S4"), ("wavelet_mask", "S5")):
                    out[(name, i - 1)] = masks[key].view(torch.bool)
            wp0, b0 = self._upconv(i, 0)
            wp1, b1 = self._upconv(i, 1)
            w1x1, b1x1, offs, c1x1 = self._head_1x1(i)
            mlp = self._head_mlp(i)                      # fused 1x1 stages (then t is never materialised)
            t = None
            if sparse:
                if yl is None:
                    raise WmdError("a sparse level needs a previous dense level (depth_decoder.py:344)")
                ev4 = ev5 = None
                if self.overlap_compaction:
                    # the three compactions are independent: S4 / S5 go to two side streams (own workspaces) and are
                    # joined where their lists are first read (upconv(i,1) / the head scatter)
                    (map4, pix4, off4), ev4 = ops.compact(masks["S4"], stream=_side_stream(dev, 1), ws_slot=1)
                    (_, pix5, off5), ev5 = ops.compact(masks["S5"], want_idxmap=False, want_pixels=not self.fused_tail,
                                                       stream=_side_stream(dev, 2), ws_slot=2)   # fused tail: the count only
                gmap = ops.gate_map(masks["S1"], prev_map)
                map2, pix2, off2 = ops.compact(masks["S2"])
                if not self.overlap_compaction:
                    map4, pix4, off4 = ops.compact(masks["S4"])
                    _, pix5, off5 = ops.compact(masks["S5"], want_idxmap=False, want_pixels=not self.fused_tail)
                counts[i] = (off2, off4, off5)
                xa = ops.conv_rows(x_rows, x_c, wp0, b0, c, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, map0=gmap,
                                   pixels=pix2, count=off2[n:], m_in0=_pm(lambda: (gmap >= 0).sum()),
                                   amax0=x_amax, amax_out=slot(4 + i))
                if skip_done is not None:
                    torch.cuda.current_stream(dev).wait_event(skip_done)
                if ev4 is not None:
                    torch.cuda.current_stream(dev).wait_event(ev4)
                    torch.cuda.current_stream(dev).wait_event(ev5)
                xb = ops.conv_rows(xa, c, wp1, b1, c, n, 2 * h, 2 * w, pad=PAD_REFLECT, act=ACT_ELU, map0=map2,
                                   shift0=1, x1=skip_rows, c1=cs, map1=map3, gate=masks["S3"], pixels=pix4, count=off4[n:],
                                   m_in0=off2[n:], m_in1=_pm(lambda: masks["S3"].sum()),
                                   amax0=slot(4 + i), amax1=skip_amax, amax_out=slot(8 + i))
                if mlp is None:
                    t = ops.conv_rows(xb, c, w1x1, b1x1, c1x1, n, 2 * h, 2 * w, taps=1, act=ACT_LRELU, act_param=0.1,
                                      pixels=pix4, count=off4[n:], m_in0=off4[n:], amax0=slot(8 + i), amax_out=slot(12 + i))
                head_kw = dict(idxmap=map4, pixels=pix5, count=off5[n:])
                prev_map = map4
            else:
                xa = ops.conv_rows(x_rows, x_c, wp0, b0, c, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, map0=prev_map,
                                   amax0=x_amax, amax_out=slot(4 + i))
                if skip_done is not None:
                    torch.cuda.current_stream(dev).wait_event(skip_done)
                xb = ops.conv_rows(xa, c, wp1, b1, c, n, 2 * h, 2 * w, pad=PAD_REFLECT, act=ACT_ELU, shift0=1,
                                   x1=skip_rows, c1=cs, amax0=slot(4 + i), amax1=skip_amax, amax_out=slot(8 + i))
                if mlp is None:
                    t = ops.conv_rows(xb, c, w1x1, b1x1, c1x1, n, 2 * h, 2 * w, taps=1, act=ACT_LRELU, act_param=0.1,
                                      amax0=slot(8 + i), amax_out=slot(12 + i))
                head_kw = {}
                if with_masks and i != 4:
                    # dense level under a thresholded mask: yh * wavelet_mask (depth_decoder.py:271-272)
                    _, pix5, off5 = ops.compact(masks["S5"], want_idxmap=False)
                    head_kw = dict(pixels=pix5, count=off5[n:])
                prev_map = None
            ll_in_gemm = i == 4 and self.factored_ll
            if i == 4 and not ll_in_gemm:
                wl, bl = self._head_3x3(i, 0)
                yl = ops.head_conv3x3(t, c // 4, offs[0], wl, bl, n, 2 * h, 2 * w, 1, scale=float(2 ** i),
                                      act=ACT_SIGMOID, pad=PAD_REFLECT)
            # +/- heads, factored: per-row tap products on the GEMM engine, then a 9 x 6 float gather-sum per pixel
            wz, bz = self._head_taps(i, offs, c1x1)
            if mlp is not None:
                z = ops.head_mlp(xb, c, mlp, c1x1, 0.1, count=off4[n:] if sparse else None, max_rows=n * 4 * h * w)
            elif sparse:
                z = ops.conv_rows(t, c1x1, wz, None, 54, n, 2 * h, 2 * w, taps=1, pixels=pix4, count=off4[n:], m_in0=off4[n:],
                                  amax0=slot(12 + i))
            else:
                z = ops.conv_rows(t, c1x1, wz, None, 63 if ll_in_gemm else 54, n, 2 * h, 2 * w, taps=1, amax0=slot(12 + i))
            if ll_in_gemm:
                yl = ops.head_gather(z, 1, self.convs[("waveconv", i, 0)][2].conv.bias.detach(), n, 2 * h, 2 * w, 1,
                                     scale=float(2 ** i), act=ACT_SIGMOID, pad=PAD_REFLECT, col0=54)
            next_thresh = None
            epi = ("disp_to_depth",) + tuple(self.depth_range) if (self.depth_range is not None and i == 1) else None
            if self.fused_tail and (2 * w) % 4 == 0:
                tail = ops.head_idwt(z, bz, yl, float(2 ** (i - 1)), 1.0 / 2 ** (i - 1), idxmap=head_kw.get("idxmap"),
                                     mask=masks["S5"] if head_kw else None, pad=PAD_REFLECT, clamp01=True,
                                     thresh_ratio=thresh_ratio if (with_masks and i > 1) else None, epilogue=epi)
                yh, yl_next, disp = tail["yh"], tail["out"], tail["disp"]
                next_thresh = tail.get("thresh")
                if epi is not None:
                    out[("scaled_disp", 0)], out[("depth", 0)] = tail["scaled_disp"], tail["depth"]
            else:
                if epi is not None:
                    raise WmdError("depth_range needs the fused tail (fused_tail = True, even width)")
                yh = ops.head_gather(z, 6, bz, n, 2 * h, 2 * w, 3, scale=float(2 ** (i - 1)), act=ACT_SIGMOID, dual=True,
                                     pad=PAD_REFLECT, **head_kw)
                yl_next, disp = ops.idwt_haar(yl, yh.unsqueeze(1), disp_scale=1.0 / 2 ** (i - 1), clamp01=True)
            out[("wavelets", i - 1, "LL")] = yl
            out[("wavelets", i - 1, "LH")] = yh[:, 0:1]
            out[("wavelets", i - 1, "HL")] = yh[:, 1:2]
            out[("wavelets", i - 1, "HH")] = yh[:, 2:3]
            if self.full_res_size is not None and i > 1:
                out[("disp_full", i - 1)] = ops.idwt_bilinear(yl, yh.unsqueeze(1), self.full_res_size,
                                                               disp_scale=1.0 / 2 ** (i - 1), clamp01=True)
            yl = yl_next
            out[("disp", i - 1)] = disp
            x_rows, x_c, x_amax = xb, c, slot(8 + i)
            h, w = 2 * h, 2 * w
        stacked = torch.stack([torch.stack(counts[i]) for i in sorted(counts, reverse=True)]) if counts else None
        return out, stacked


class DepthWaveProgressiveDecoder(_WaveDecoderBase):
    """Dense wavelet decoder.  [depth_decoder.py:72-168]"""

    def __init__(self, num_ch_enc, scales=range(4), num_output_channels=1, use_skips=True):
        super().__init__()
        self._build(num_ch_enc, scales, num_output_channels, use_skips)
        self.tanh = nn.Tanh()

    def get_coefficients(self, input_features, scale=1, return_ll=False):
        """(LL, [LH, HL, HH]) from feature maps at ``scale`` - differentiable path.  [:126-136]"""
        yl = None
        if return_ll:
            yl = 2 ** scale * self.sigmoid(self.convs[("waveconv", scale, 0)](input_features))
        yh = 2 ** (scale - 1) * self.sigmoid(self.convs[("waveconv", scale, 1)](input_features)).unsqueeze(1) - \
            2 ** (scale - 1) * self.sigmoid(self.convs[("waveconv", scale, -1)](input_features)).unsqueeze(1)
        return yl, yh

    def _autograd_forward(self, input_features):
        out = {}
        x = input_features[-1]
        yl = None
        for i in range(4, 0, -1):
            x = self.convs[("upconv", i, 0)](x)
            x = [upsample(x)]
            if self.use_skips and i > 0:
                x += [input_features[i - 1]]
            x = self.convs[("upconv", i, 1)](torch.cat(x, 1))
            if i == 4:
                yl, yh = self.get_coefficients(x, scale=i, return_ll=True)
            else:
                _, yh = self.get_coefficients(x, scale=i, return_ll=False)
            out[("wavelets", i - 1, "LL")] = yl
            out[("wavelets", i - 1, "LH")] = yh[:, :, 0]
            out[("wavelets", i - 1, "HL")] = yh[:, :, 1]
            out[("wavelets", i - 1, "HH")] = yh[:, :, 2]
            yl = self.inverse_wt((yl, list([yh])))
            out[("disp", i - 1)] = torch.clamp(yl / 2 ** (i - 1), 0, 1)
        return out

    def forward(self, input_features):
        _need_cuda(input_features)
        needs_grad = torch.is_grad_enabled() and (
            any(p.requires_grad for p in self.parameters()) or any(f.requires_grad for f in input_features))
        if needs_grad:
            self.outputs = self._autograd_forward(input_features)
        else:
            self.outputs, _ = self._native_forward(input_features, 0.0, sparse_levels=(), with_masks=False)
        return self.outputs


class SparseDepthWaveProgressiveDecoder(_WaveDecoderBase):
    """Threshold-gated sparse wavelet decoder, batched.  [depth_decoder.py:171-428]

    Inference only, like the reference (KITTI/trainer.py:35-36).  ``count_ops``: True (default) returns the
    reference's ``total_ops`` keys as Python ints, which waits for this forward's active counts; ``"async"`` returns
    ``out["total_ops"]`` as an ``OpsFuture`` instead and never blocks the host (serving / multi-GPU: the next step
    and the all-gather are enqueued while this one runs); False skips op counting.
    """

    def __init__(self, num_ch_enc, scales=range(4), num_output_channels=1, use_skips=True):
        super().__init__()
        self._build(num_ch_enc, scales, num_output_channels, use_skips)
        self.maxpool3 = nn.MaxPool2d(3, stride=1, padding=1)
        self.maxpool5 = nn.MaxPool2d(5, stride=1, padding=2)
        self.maxpool7 = nn.MaxPool2d(7, stride=1, padding=3)
        self.count_ops = True

    @staticmethod
    def my_iwt_once(coeffs):
        """One Haar synthesis level (the reference's closed form, :225-239) on the native kernel."""
        yl, [yh] = coeffs
        return ops.idwt_haar(yl, yh)

    def forward(self, input_features, thresh_ratio=0.05, sparse_scales=[0, 1, 2, 3]):
        assert self.use_skips
        sparse_levels = self._sparse_levels(sparse_scales)
        out, counts = self._native_forward(input_features, float(thresh_ratio), sparse_levels, with_masks=True)
        self._attach_total_ops(out, counts, input_features, sparse_levels)
        self.outputs = out
        return out

    @staticmethod
    def _sparse_levels(sparse_scales):
        sparse_levels = tuple(i for i in range(1, 4) if i in sparse_scales)
        if any((i + 1) in sparse_levels and i not in sparse_levels for i in range(1, 4)):
            raise NotImplementedError("a dense level below a sparse level is not defined by the reference either")
        return sparse_levels

    def _attach_total_ops(self, out, counts, feats, sparse_levels):
        """count_ops True: the reference's keys as Python ints (one wait for this forward's counts);
        "async": out["total_ops"] = OpsFuture, nothing waits; False: no op counting."""
        if not self.count_ops:
            return
        fut = self.ops_future(counts, feats, sparse_levels)
        if self.count_ops == "async":
            out["total_ops"] = fut
        else:
            out.update(fut.result())

    def ops_future(self, counts, feats, sparse_levels):
        """OpsFuture of one forward: enqueues the count read-back on the current stream (no host wait)."""
        n = int(feats[-1].shape[0])
        h4, w4 = (int(v) for v in feats[-1].shape[2:])
        levels = sorted(sparse_levels, reverse=True)
        ch_enc = [int(v) for v in self.num_ch_enc]
        ch_dec = [int(v) for v in self.num_ch_dec]

        def finish(host):
            res = {}
            per_sample = [0] * n
            for i in range(4, 0, -1):
                h, w = h4 << (4 - i), w4 << (4 - i)
                cin0 = ch_enc[-1] if i == 4 else ch_dec[i + 1]
                c, cs = ch_dec[i], ch_enc[i - 1]
                level_total = 0
                for b in range(n):
                    if i in levels:
                        row = host[levels.index(i)]                                  # (3, N+1) offsets of S2, S4, S5
                        m2, m4, m5 = (int(row[k][b + 1] - row[k][b]) for k in range(3))
                        v = opcount.kitti_level_ops(i, h, w, cin0, c, cs, True, m2, m4, m5)
                    else:
                        v = opcount.kitti_level_ops(i, h, w, cin0, c, cs, False)
                    per_sample[b] += v
                    level_total += v
                res[("total_ops", i - 1)] = level_total
            res["total_ops"] = sum(per_sample)
            if n > 1:
                res["total_ops_per_sample"] = per_sample
            return res

        return OpsFuture(counts if levels else None, finish)
