"""NYUv2's supervised training loss on the device: the objective of NYUv2/train.py:279-327, forward and backward.

``NyuDepthLoss`` replaces the reference's chain of ``F.interpolate(("disp", s), scale_factor=2**s, mode="bilinear",
align_corners=True)``, ``nn.L1Loss`` against the (optionally DepthNorm-ed) target and the LL term against a J=4 Haar
DWT of that target.  Every term's mean absolute difference is one libwmd call (include/wmd_loss.h), summed in fp64 in
a fixed order, and its gradient is a gather over each low-resolution pixel's footprint with no atomics, so a training
step gives the same bits on every run, also under ``torch.use_deterministic_algorithms(True)``, where torch's CUDA
bilinear backward raises.  Nothing waits on the host, and the loss can be captured in a CUDA graph.

The sampling is torch's align_corners rule, except that the weight ``1 - lambda`` is exact (fp64) where torch rounds it
to float32, and the sample is evaluated in fp64 from the float32 inputs: the map of a constant is that constant.
"""
import ctypes

import torch

from . import _lib
from .ops import _dense, _launch, _on_device
from .wavelets import DWT

SCALES = (0, 1, 2, 3)          # train.py: `for scale in range(4)`
LL_KEY = ("wavelets", 3, "LL")


def _terms(preds, log2s):
    arr = (_lib.LossTerm * len(preds))()
    for d, p, k in zip(arr, preds, log2s):
        d.pred, d.h, d.w, d.log2_factor = _lib.ptr(p), int(p.shape[2]), int(p.shape[3]), int(k)
    return arr


def _loss_fwd(target, preds, log2s, means, want_signs):
    """means[:] = the terms of `preds` against `target` (N, 1, H, W); returns the int8 signs (or None)."""
    n, _, h, w = (int(v) for v in target.shape)
    dev = target.device
    signs = torch.empty((len(preds), n, h, w), dtype=torch.int8, device=dev) if want_signs else None
    ws = torch.empty(int(_lib.load().wmd_loss_nyu_ws_bytes(n, h, w, len(preds))), dtype=torch.uint8, device=dev)
    _launch("loss_nyu_fwd", lambda: dict(n=n, h=h, w=w, terms=len(preds))).wmd_loss_nyu_fwd(
        _lib.ptr(target), n, h, w, _terms(preds, log2s), len(preds), _lib.ptr(signs), _lib.ptr(ws), ws.numel(),
        _lib.ptr(means), _lib.stream_ptr())
    return signs


def _loss_bwd(signs, target_shape, preds, log2s, grad_means):
    n, _, h, w = target_shape
    grads = [torch.empty_like(p) for p in preds]
    ptrs = (ctypes.c_void_p * len(grads))(*[_lib.ptr(g) for g in grads])
    _launch("loss_nyu_bwd", lambda: dict(n=n, h=h, w=w, terms=len(preds))).wmd_loss_nyu_bwd(
        _lib.ptr(signs), n, h, w, _terms(preds, log2s), len(preds), _lib.ptr(grad_means), ptrs, _lib.stream_ptr())
    return grads


class _NyuLossFn(torch.autograd.Function):
    """(target, ll_target or None, log2 factors, want_signs, *preds) -> (K,) float32 terms: the scale terms against
    target, then the LL term (the last pred, factor 1) against ll_target.  No gradient flows to either target."""

    @staticmethod
    def forward(ctx, target, ll_target, log2s, want_signs, *preds):
        preds = tuple(_dense(p) for p in preds)
        ks = len(log2s)
        means = torch.empty(len(preds), dtype=torch.float32, device=target.device)
        signs = _loss_fwd(target, preds[:ks], log2s, means[:ks], want_signs) if ks else None
        ll_signs = _loss_fwd(ll_target, preds[ks:], (0,), means[ks:], want_signs) if ll_target is not None else None
        ctx.log2s, ctx.shapes = log2s, (tuple(target.shape), None if ll_target is None else tuple(ll_target.shape))
        ctx.save_for_backward(signs, ll_signs, *preds)
        return means

    @staticmethod
    def backward(ctx, grad_means):
        signs, ll_signs, *preds = ctx.saved_tensors
        g = _dense(grad_means)
        ks = len(ctx.log2s)
        grads = _loss_bwd(signs, ctx.shapes[0], preds[:ks], ctx.log2s, g) if ks else []
        if ll_signs is not None:
            grads += _loss_bwd(ll_signs, ctx.shapes[1], preds[ks:], (0,), g[ks:])
        return (None, None, None, None) + tuple(grads)


def _check(t, what):
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32:
        raise _lib.WmdError("%s must be a float32 CUDA tensor" % what)
    return t


class NyuDepthLoss:
    """The reference's NYUv2 training objective (train.py:279-327; argument names and defaults are train.py's).

    ``__call__(outputs, depth) -> (total, losses)``.  depth: (N, 1, H, W) float32 CUDA tensor, the loader's depth;
    outputs: the decoder's dict, whose ("disp", s) for each s in ``output_scales`` (scales 0 to 3 only) must be
    (N, 1, H / 2**s, W / 2**s) float32.  A missing key raises KeyError and a wrong shape ValueError.  The target is
    ``10.0 / depth`` with ``disparity`` (DepthNorm) and ``depth`` otherwise.  ``losses`` holds, as 0-dim CUDA tensors:

      "loss_depth/s"  the mean |upsampled ("disp", s) - target|,  "loss/s"  0.1 times it,
      "loss_LL3"      the mean |("wavelets", 3, "LL") - yl_gt| / 16, with yl_gt the J=4 Haar DWT's LL of the target,
                      present when ``use_wavelets`` is set and the key is in ``outputs`` (DecoderWave names its LL
                      ("wavelets", 2, "LL"), so, as in the reference, it has none),
      "loss"          the float32 sum over s in ascending order of "loss/s" for s in ``loss_scales``, plus "loss_LL3"
                      with ``supervise_LL``;

    ``total`` is ``losses["loss"]``.  Gradients flow to the predictions only.  Works under ``torch.no_grad`` and on
    whichever decoder path produced ``outputs``."""

    def __init__(self, output_scales=SCALES, loss_scales=SCALES, disparity=False, use_wavelets=False,
                 supervise_LL=False):
        self.scales = tuple(s for s in SCALES if s in output_scales)
        self.loss_scales = tuple(s for s in self.scales if s in loss_scales)
        self.disparity, self.use_wavelets, self.supervise_LL = bool(disparity), bool(use_wavelets), bool(supervise_LL)
        if not self.loss_scales and not (self.use_wavelets and self.supervise_LL):
            raise ValueError("no term would be trained: loss_scales %s has no scale of output_scales %s in 0..3, and the "
                             "LL term is not supervised" % (tuple(loss_scales), tuple(output_scales)))
        self.dwt = DWT(J=4, wave="haar", mode="reflect") if self.use_wavelets else None

    @_on_device
    def __call__(self, outputs, depth):
        _check(depth, "depth")
        if depth.dim() != 4 or depth.shape[1] != 1:
            raise ValueError("depth must be (N, 1, H, W), got %s" % (tuple(depth.shape),))
        n, _, h, w = (int(v) for v in depth.shape)
        preds = [_check(outputs[("disp", s)], str(("disp", s))) for s in self.scales]
        for s, p in zip(self.scales, preds):
            if p.dim() != 4 or tuple(p.shape[:2]) != (n, 1) or p.shape[2] << s != h or p.shape[3] << s != w:
                raise ValueError("(\"disp\", %d) must be (%d, 1, %d / 2**%d, %d / 2**%d), got %s"
                                 % (s, n, h, s, w, s, tuple(p.shape)))
        depth_n = 10.0 / depth if self.disparity else depth
        target = _dense(depth_n.detach())
        ll_target = None
        if self.use_wavelets and LL_KEY in outputs:
            ll = _check(outputs[LL_KEY], str(LL_KEY))
            with torch.no_grad():
                ll_target = _dense(self.dwt(target)[0])
            if tuple(ll.shape) != tuple(ll_target.shape):
                raise ValueError("%s must be %s like the target's J=4 LL, got %s"
                                 % (LL_KEY, tuple(ll_target.shape), tuple(ll.shape)))
            preds.append(ll)
        want_signs = torch.is_grad_enabled() and any(p.requires_grad for p in preds)
        terms = _NyuLossFn.apply(target, ll_target, tuple(self.scales), want_signs, *preds).unbind(0)
        losses, total = {}, None
        for s, l_depth in zip(self.scales, terms):
            loss = 0.1 * l_depth
            if s in self.loss_scales:
                total = loss if total is None else total + loss
            losses["loss/%d" % s] = loss
            losses["loss_depth/%d" % s] = l_depth
        if ll_target is not None:
            l_ll = terms[-1] / 2 ** 4
            losses["loss_LL3"] = l_ll
            if self.supervise_LL:
                total = l_ll if total is None else total + l_ll
        if total is None:
            raise KeyError("%s: the only supervised term, is missing from outputs" % (LL_KEY,))
        losses["loss"] = total
        return total, losses
