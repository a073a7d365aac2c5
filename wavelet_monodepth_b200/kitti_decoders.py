"""KITTI depth decoders with the reference's constructor / forward / state-dict contract, on libwmd.

Mirrors KITTI/networks/decoders/depth_decoder.py:
  * ``DepthDecoder``                       (:18-69)   monodepth2 baseline decoder
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
  * training (grad enabled) of the dense decoder runs every convolution forward and backward on libwmd when fp32
    convolutions are requested (torch.backends.cudnn.allow_tf32 False, train_native.py); with TF32 allowed it takes the
    differentiable cuDNN path.  Both train through the native IDWT with its adjoint;
  * the baseline ``DepthDecoder`` runs the same way: natively at inference (its full-resolution level 0 as one fused
    kernel, wmd_disp_tail16_f32), natively in training with fp32 convolutions, the cuDNN module graph with TF32 allowed
    and whenever ``num_output_channels > 4``.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import opcount, ops, train_native
from .opsfuture import OpsFuture
from ._lib import ACT_ELU, ACT_LRELU, ACT_SIGMOID, PAD_REFLECT, PAD_ZERO, WmdError
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


def _side_stream(device, which):
    """Side streams per device (1-2: compactions of S4 / S5, 3: S3's compaction and skip-row gather), created lazily and
    reused: CUDA graphs fork/join through them."""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device(), which)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def _fused_tail_fits(width):
    """Whether a level's tail runs as one kernel (wmd_head_idwt_f32: head gather-sum -> yh -> IDWT -> disp -> next level's
    threshold, bit-identical to the head_gather + idwt_haar + range_thresh chain).  The kernel needs the width of the
    level's coefficient maps to be a multiple of 4; other widths (level 4 of small frames) take the chain."""
    return width % 4 == 0


def _need_cuda(feats, host_ok=()):
    """host_ok: indices of feature maps that may instead be pinned host tensors (read in place by the gated move)."""
    for k, f in enumerate(feats):
        if not f.is_cuda and k in host_ok and f.is_pinned():
            continue
        if not f.is_cuda:
            raise WmdError("wavelet_monodepth_b200 decoders run on CUDA tensors only: the native kernels have no "
                           "CPU fallback (got a feature map on %s)" % f.device)


class _PackedModule(nn.Module):
    """A decoder that keeps packed copies of its weights for the native engine (see _PackCache)."""

    def _init_packs(self):
        self._packs = _PackCache()
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packs())

    def invalidate_packs(self):
        """Drop the packed copies of the weights (they are rebuilt on the next native forward).  Needed only after a
        weight update the version counters cannot see, e.g. ``p.data.copy_(...)``."""
        self._packs.invalidate()

    def _apply(self, fn, *args, **kwargs):
        if hasattr(self, "_packs"):
            self._packs.invalidate()
        return super()._apply(fn, *args, **kwargs)


def _needs_grad(module, feats):
    return torch.is_grad_enabled() and (
        any(p.requires_grad for p in module.parameters()) or any(f.requires_grad for f in feats))


class DepthDecoder(_PackedModule):
    """monodepth2 baseline decoder (sigmoid disparity at 4 scales).  [depth_decoder.py:18-69]

    Same module structure, state dict and outputs as the reference.  Selects its path like the dense wavelet decoder:
    ``no_grad`` calls run the native engine, grad-enabled calls with fp32 convolutions requested
    (``torch.backends.cudnn.allow_tf32`` False) run ``train_native.kitti_baseline_forward``, and training with TF32
    allowed - or any call with ``num_output_channels > 4`` - runs the cuDNN module graph.  The native engine follows
    the reference's padding: zeros in the ELU ConvBlocks, reflection in the dispconvs (KITTI/layers.py:123,149).
    Levels finer than the finest requested scale feed no output and are not run."""

    NATIVE_MAX_OUTPUT_CHANNELS = 4         # the dispconv kernels (head_conv3x3, the fused tail) take 1..4 channels

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
        self._init_packs()

    def forward(self, input_features):
        needs_grad = _needs_grad(self, input_features)
        if self.num_output_channels > self.NATIVE_MAX_OUTPUT_CHANNELS or \
                (needs_grad and not train_native.fp32_convs_requested()):
            self.outputs = self._autograd_forward(input_features)
        elif needs_grad:
            _need_cuda(input_features)
            self.outputs = train_native.kitti_baseline_forward(self, input_features)
        else:
            self.outputs = self._native_forward(input_features)
        return self.outputs

    def _autograd_forward(self, input_features):
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

    # ---- native engine ------------------------------------------------------------------------
    def _upconv(self, i, j):
        conv = self.convs[("upconv", i, j)].conv.conv
        c1 = int(self.num_ch_enc[i - 1]) if (j == 1 and self.use_skips and i > 0) else 0
        return self._packs.get(("upconv", i, j), [conv.weight], lambda: ops.pack_weight(conv.weight, c1)), conv.bias.detach()

    def _dispconv(self, s):
        conv = self.convs[("dispconv", s)].conv
        return self._packs.get(("dispconv", s), [conv.weight], lambda: ops.pack_head_weight(conv.weight)), conv.bias.detach()

    def _tail(self):
        """Packed weights of the fused level-0 tail: upconv(0,1) and dispconv(0)."""
        c1, cd = self.convs[("upconv", 0, 1)].conv.conv, self.convs[("dispconv", 0)].conv
        return self._packs.get(("tail",), [c1.weight, c1.bias, cd.weight, cd.bias],
                               lambda: ops.pack_disp_tail16(c1.weight, c1.bias, cd.weight, cd.bias))

    @torch.no_grad()
    @ops._on_device
    def _native_forward(self, feats):
        """upconv(i,0) / upconv(i,1) on the gather-GEMM engine, dispconv(s) on head_conv3x3, ("disp", 0) on the fused
        tail.  Operands in the fp16-pair form with tracked maxima, as in the wavelet engine."""
        _need_cuda(feats)
        n = int(feats[-1].shape[0])
        dev = feats[-1].device
        h, w = (int(v) for v in feats[4].shape[2:])
        finest = min(self.scales)
        cout = int(self.num_output_channels)
        out = {}
        if n == 0:
            for s in self.scales:
                out[("disp", s)] = torch.zeros((0, cout, h << (5 - s), w << (5 - s)), dtype=torch.float32, device=dev)
            return out
        amax = torch.zeros(16, dtype=torch.float32, device=dev)

        def slot(k):
            return amax[k:k + 1]
        x_rows, x_c, x_amax = ops.nchw_to_rows(feats[4], amax=slot(0)), int(feats[4].shape[1]), slot(0)
        for i in range(4, finest - 1, -1):
            c = int(self.num_ch_dec[i])
            k = 1 + 3 * (4 - i)
            wp0, b0 = self._upconv(i, 0)
            xa = ops.conv_rows(x_rows, x_c, wp0, b0, c, n, h, w, pad=PAD_ZERO, act=ACT_ELU, amax0=x_amax, amax_out=slot(k))
            if i == 0:
                # upconv(0,1) -> dispconv(0) -> sigmoid in one kernel: the full-resolution 16-channel map stays on chip
                out[("disp", 0)] = ops.disp_tail16(xa, self._tail(), cout, n, h, w)
                break
            skip_rows, cs = None, 0
            if self.use_skips:
                skip = feats[i - 1]
                if tuple(skip.shape[2:]) != (2 * h, 2 * w):
                    raise WmdError("skip feature %d has shape %s, expected spatial %s" % (i - 1, tuple(skip.shape), (2 * h, 2 * w)))
                skip_rows, cs = ops.nchw_to_rows(skip, amax=slot(k + 1)), int(skip.shape[1])
            wp1, b1 = self._upconv(i, 1)
            xb = ops.conv_rows(xa, c, wp1, b1, c, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_ELU, shift0=1, x1=skip_rows, c1=cs,
                               amax0=slot(k), amax1=slot(k + 1) if skip_rows is not None else None, amax_out=slot(k + 2))
            h, w = 2 * h, 2 * w
            if i in self.scales:
                wd, bd = self._dispconv(i)
                out[("disp", i)] = ops.head_conv3x3(xb, c, 0, wd, bd, n, h, w, cout, act=ACT_SIGMOID, pad=PAD_REFLECT)
            x_rows, x_c, x_amax = xb, c, slot(k + 2)
        return out


class _WaveDecoderBase(_PackedModule):
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
        self._init_packs()
        # optional fused consumer epilogue (not part of the reference's decoder, off by default): when set to (H, W),
        # inference also returns ("disp_full", s) = F.interpolate(("disp", s), (H, W), mode="bilinear",
        # align_corners=False) for s = 1..3 - what KITTI/trainer.py:338-339 computes from every scale - produced
        # straight from the coefficients by the fused IDWT+bilinear kernel
        self.full_res_size = None
        # transpose a sparse level's skip map only under its upsample mask.  On since the gated move issues all its loads
        # before using any (72 us against 175 before and ~110 for the whole level-3 map)
        self.gated_layout = True
        # run the two 1x1 head stages of the fine levels as one fused kernel
        self.fused_heads = True
        # sparse levels keep their skip map COMPACT: only the rows of the upsample mask S3 are moved out of the NCHW map
        # (list-based gather-transpose: bytes scale with the mask density, 16-50 % on the bench) and upconv(i,1) reaches them
        # through S3's index map (wmd_conv_desc.map1).  The skip map may then be a pinned HOST tensor.
        self.compact_skip = True
        # ... at the levels where it pays on a device-resident map: the list-based gather moves fewer useful bytes per second
        # than the whole-map transpose (scripts/probe_gather.py), so it wins only at low mask density - levels 2 and 1
        # (16-28 % on the bench), not level 3 (50 %).  A pinned-host skip map always takes it.
        self.compact_skip_levels = (1, 2)
        # optional consumer epilogue of ("disp", 0), off by default: (min_depth, max_depth) adds ("scaled_disp", 0) and
        # ("depth", 0) = disp_to_depth(("disp", 0), min_depth, max_depth) (KITTI/layers.py:16-25; evaluate_depth.py:193,
        # test_simple.py:151), produced by the last level's fused tail
        self.depth_range = None

    # ---- packed parameters ------------------------------------------------------------------
    def _upconv(self, i, j):
        conv = self.convs[("upconv", i, j)].conv.conv
        # upconv(i,1) reads the skip map as gather source 1; without skips it reads only the upsampled upconv(i,0)
        c1 = int(self.num_ch_enc[i - 1]) if (j == 1 and self.use_skips) else 0
        return self._packs.get(("upconv", i, j), [conv.weight], lambda: ops.pack_weight(conv.weight, c1)), conv.bias.detach()

    def _head_1x1(self, i):
        """Concatenated 1x1 stages of the level's heads: [LL (i==4) | + | -] -> (packed (C, ld), bias, offsets)."""
        names = ([0] if i == 4 else []) + [1, -1]
        convs = [self.convs[("waveconv", i, j)][0].conv for j in names]
        wts = [c.weight for c in convs]
        packed = self._packs.get(("head1x1", i), wts,
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

        Level 4 appends the LL head's nine tap filters as columns 54..62 (same 64-wide GEMM tile)."""
        cp, cn = self.convs[("waveconv", i, 1)][2].conv, self.convs[("waveconv", i, -1)][2].conv
        if i == 4:
            cl = self.convs[("waveconv", i, 0)][2].conv
            wz = self._packs.get(("headtaps+ll", i), [cp.weight, cn.weight, cl.weight],
                                 lambda: ops.pack_weight(torch.cat([
                                     ops.head_tap_weight([cp.weight, cn.weight], [offs[1], offs[-1]], ctot),
                                     ops.head_tap_weight([cl.weight], [offs[0]], ctot)], 0)))
            bz = self._packs.get(("headtapsb", i), [cp.bias, cn.bias],
                                 lambda: torch.cat([cp.bias.detach(), cn.bias.detach()]).contiguous())
            return wz, bz
        wz = self._packs.get(("headtaps", i), [cp.weight, cn.weight],
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

    # ---- native engine ------------------------------------------------------------------------
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

    @torch.no_grad()
    @ops._on_device
    def _native_forward(self, feats, thresh_ratio, sparse_levels, with_masks):
        """Runs levels 4..1 on libwmd.  sparse_levels: set of levels i executed on active lists.

        Returns (outputs, counts): counts = int32 device tensor (levels, 3, N+1) with the row offsets of the compacted
        sets S2, S4, S5 of every sparse level, sparse levels in descending order (None without sparse levels)."""
        # with gated_layout the skip map of a sparse level i (feats[i-1]) may live in pinned host memory
        _need_cuda(feats, host_ok=tuple(i - 1 for i in sparse_levels) if (self.gated_layout or self.compact_skip) else ())
        out = {}
        n = feats[-1].shape[0]
        dev = feats[-1].device
        if n == 0:
            return self._empty_outputs(feats, sparse_levels, with_masks)
        # max |x| of every tensor a tensor-core conv reads (device scalars, zeroed here, raised by the producers): the
        # fp16-pair operand form scales by a power of two chosen from them.  A skip map's maximum covers exactly the
        # pixels upconv(i,1) reads, so every layout option picks the same scale.
        amax = torch.zeros(24, dtype=torch.float32, device=dev)

        def slot(k):
            return amax[k:k + 1]
        x_rows, x_c, prev_map = ops.nchw_to_rows(feats[4], amax=slot(0)), feats[4].shape[1], None
        x_amax = slot(0)
        h, w = feats[4].shape[2:]
        yl = yh = None
        counts = {}
        next_thresh = None                 # per-sample threshold of the coming level, when the fused tail produced it
        for i in range(4, 0, -1):
            c = int(self.num_ch_dec[i])
            sparse = i in sparse_levels
            one_kernel_tail = _fused_tail_fits(2 * w)
            # without skips the maps feats[0..3] are never read: no layout move, gate, compaction or maximum for them
            skip = feats[i - 1] if self.use_skips else None
            cs = skip.shape[1] if self.use_skips else 0
            if self.use_skips and tuple(skip.shape[2:]) != (2 * h, 2 * w):
                raise WmdError("skip feature %d has shape %s, expected spatial %s" % (i - 1, tuple(skip.shape), (2 * h, 2 * w)))
            masks = None
            if with_masks:
                if i == 4:
                    masks = ops.level_masks(None, None, n=n, h=h, w=w, device=dev)
                else:
                    thresh = next_thresh if next_thresh is not None else ops.range_thresh(yl, thresh_ratio)
                    masks = ops.level_masks(yh, thresh)
            skip_rows = skip_amax = skip_done = map3 = None
            if self.use_skips:
                skip_amax = slot(i)
                if sparse and self.compact_skip and (i in self.compact_skip_levels or not skip.is_cuda) and \
                        ops.rows_view(skip) is None:                         # channels_last maps are used in place instead
                    # S3's compaction and the gather of exactly its rows, on a side stream next to gate_map / compact(S2) / upconv(i,0)
                    s3 = _side_stream(dev, 3)
                    (map3, pix3, off3), _ = ops.compact(masks["S3"], stream=s3, ws_slot=3)
                    skip_rows, skip_done = ops.gather_rows_list(skip, pix3, off3[n:], stream=s3, amax=skip_amax)
                else:
                    # layout move of the skip map (NCHW -> pixel-major rows).  gated_layout: a sparse level reads its skip
                    # map only under the upsample mask S3 (sparse_upsample: skip[mask], layers.py:500), so only those rows
                    # are produced - the move scales with density.  A sparse level's maximum covers S3 only, the rows
                    # upconv(i,1) reads, whether the move is gated or not
                    skip_gate = masks["S3"] if (sparse and self.gated_layout) else None
                    skip_rows = ops.nchw_to_rows(skip, gate=skip_gate, amax=skip_amax, amax_mask=masks["S3"] if sparse else None)
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
                # the three compactions are independent: S4 / S5 go to two side streams (own workspaces) and are joined
                # where their lists are first read (upconv(i,1) / the head scatter)
                (map4, pix4, off4), ev4 = ops.compact(masks["S4"], stream=_side_stream(dev, 1), ws_slot=1)
                (_, pix5, off5), ev5 = ops.compact(masks["S5"], want_idxmap=False, want_pixels=not one_kernel_tail,
                                                   stream=_side_stream(dev, 2), ws_slot=2)   # fused tail: the count only
                gmap = ops.gate_map(masks["S1"], prev_map)
                map2, pix2, off2 = ops.compact(masks["S2"])
                counts[i] = (off2, off4, off5)
                xa = ops.conv_rows(x_rows, x_c, wp0, b0, c, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, map0=gmap,
                                   pixels=pix2, count=off2[n:], m_in0=_pm(lambda: (gmap >= 0).sum()),
                                   amax0=x_amax, amax_out=slot(4 + i))
                if skip_done is not None:
                    torch.cuda.current_stream(dev).wait_event(skip_done)
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
            # +/- heads, factored: per-row tap products on the GEMM engine, then a 9 x 6 float gather-sum per pixel.  Level 4's
            # LL head rides in the same GEMM as nine more tap-product columns (54..62), then a 9-float gather-sum
            wz, bz = self._head_taps(i, offs, c1x1)
            if mlp is not None:
                z = ops.head_mlp(xb, c, mlp, c1x1, 0.1, count=off4[n:] if sparse else None, max_rows=n * 4 * h * w)
            elif sparse:
                z = ops.conv_rows(t, c1x1, wz, None, 54, n, 2 * h, 2 * w, taps=1, pixels=pix4, count=off4[n:], m_in0=off4[n:],
                                  amax0=slot(12 + i))
            else:
                z = ops.conv_rows(t, c1x1, wz, None, 63 if i == 4 else 54, n, 2 * h, 2 * w, taps=1, amax0=slot(12 + i))
            if i == 4:
                yl = ops.head_gather(z, 1, self.convs[("waveconv", i, 0)][2].conv.bias.detach(), n, 2 * h, 2 * w, 1,
                                     scale=float(2 ** i), act=ACT_SIGMOID, pad=PAD_REFLECT, col0=54)
            next_thresh = None
            epi = ("disp_to_depth",) + tuple(self.depth_range) if (self.depth_range is not None and i == 1) else None
            if one_kernel_tail:
                tail = ops.head_idwt(z, bz, yl, float(2 ** (i - 1)), 1.0 / 2 ** (i - 1), idxmap=head_kw.get("idxmap"),
                                     mask=masks["S5"] if head_kw else None, pad=PAD_REFLECT, clamp01=True,
                                     thresh_ratio=thresh_ratio if (with_masks and i > 1) else None, epilogue=epi)
                yh, yl_next, disp = tail["yh"], tail["out"], tail["disp"]
                next_thresh = tail.get("thresh")
                if epi is not None:
                    out[("scaled_disp", 0)], out[("depth", 0)] = tail["scaled_disp"], tail["depth"]
            else:
                if epi is not None:
                    raise WmdError("depth_range needs the fused level tail, which takes coefficient maps whose width is a "
                                   "multiple of 4 (got %d)" % (2 * w))
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
        needs_grad = _needs_grad(self, input_features)
        if needs_grad and train_native.fp32_convs_requested():
            # fp32 convolutions requested: forward and backward of every convolution on libwmd
            self.outputs = train_native.kitti_forward(self, input_features)
        elif needs_grad:
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
