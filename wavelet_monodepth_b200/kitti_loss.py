"""KITTI's stereo depth-hints training loss on the device: ``Trainer.generate_images_pred`` + ``compute_losses_hints``
(KITTI/trainer.py:329-560) for the configuration every released KITTI model was trained with (``--use_depth_hints
--frame_ids 0 --use_stereo``), forward and backward.

``KittiDepthHintsLoss`` replaces the reference's chain of upsample, back-projection, projection, grid sample, SSIM,
automasking with depth hints, the proxy-supervised hint term and the edge-aware smoothness.  Every sum is fp64 in a
fixed order and the backward is a gather with no atomics (include/wmd_loss_kitti.h), so a training step gives the same bits
on every run, also under ``torch.use_deterministic_algorithms(True)``.

The tie-breaking noise is drawn as the reference draws it, ``torch.randn((N, 1, H, W))`` on the CPU default generator,
once per loss scale in order, then copied to the device: a seeded step sees the reference's noise.  That draw is the
one host step, so the call cannot be captured in a CUDA graph (the reference's cannot either).
"""
import ctypes

import torch

from . import _lib
from .ops import _dense, _launch, _on_device

SCALES = (0, 1, 2, 3)          # options.py: --scales default


def _desc(t, scales, loss_scales, opt):
    """wmd_loss_kitti_desc of a dict of dense tensors"""
    d = _lib.KittiLossDesc()
    d.N, _, d.H, d.W = (int(v) for v in t["target"].shape)
    for name in ("target", "source", "K", "inv_K", "stereo_T", "depth_hint", "depth_hint_mask"):
        setattr(d, name, _lib.ptr(t[name]))
    d.n_scales, d.n_loss = len(scales), len(loss_scales)
    for i, s in enumerate(loss_scales):
        d.scale[i] = s
        d.disp[i], d.color[i], d.noise[i] = _lib.ptr(t["disp"][i]), _lib.ptr(t["color"][i]), _lib.ptr(t["noise"][i])
    d.min_depth, d.max_depth, d.disparity_smoothness = opt
    return d


def _kitti_fwd(t, scales, loss_scales, opt):
    """(terms (1 + 3 L), color_depth_hint, warped (L, N, 3, H, W), identity_selection, depth_hint_pixels, state)"""
    d = _desc(t, scales, loss_scales, opt)
    n, h, w, nl = d.N, d.H, d.W, d.n_loss
    dev = t["target"].device
    ws = torch.empty(int(_lib.load().wmd_loss_kitti_ws_bytes(ctypes.byref(d))), dtype=torch.uint8, device=dev)
    terms = torch.empty(1 + 3 * nl, dtype=torch.float32, device=dev)
    chint = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    warped = torch.empty((nl, n, 3, h, w), dtype=torch.float32, device=dev)
    idsel = torch.empty((nl, n, 1, h, w), dtype=torch.float32, device=dev)
    hpix = torch.empty((nl, n, 1, h, w), dtype=torch.float32, device=dev)
    _launch("loss_kitti_fwd", lambda: dict(n=n, h=h, w=w, scales=nl)).wmd_loss_kitti_fwd(
        ctypes.byref(d), _lib.ptr(chint), _lib.ptr(warped), _lib.ptr(idsel), _lib.ptr(hpix), _lib.ptr(ws), ws.numel(),
        _lib.ptr(terms), _lib.stream_ptr())
    return terms, chint, warped, idsel, hpix, ws


def _kitti_bwd(t, scales, loss_scales, opt, warped, idsel, hpix, state, grad_terms):
    d = _desc(t, scales, loss_scales, opt)
    grads = [torch.empty_like(p) for p in t["disp"]]
    ptrs = (ctypes.c_void_p * len(grads))(*[_lib.ptr(g) for g in grads])
    ws = torch.empty(int(_lib.load().wmd_loss_kitti_bwd_ws_bytes(ctypes.byref(d))), dtype=torch.uint8, device=warped.device)
    _launch("loss_kitti_bwd", lambda: dict(n=d.N, h=d.H, w=d.W, scales=d.n_loss)).wmd_loss_kitti_bwd(
        ctypes.byref(d), _lib.ptr(warped), _lib.ptr(idsel), _lib.ptr(hpix), _lib.ptr(state), _lib.ptr(grad_terms),
        _lib.ptr(ws), ws.numel(), ptrs, _lib.stream_ptr())
    return grads


class _KittiLossFn(torch.autograd.Function):
    """(constants dict, scales, loss_scales, opt, *disps) -> (terms, color_depth_hint, warped, identity_selection,
    depth_hint_pixels); the gradient flows from the terms to the disps only."""

    @staticmethod
    def forward(ctx, const, scales, loss_scales, opt, *disps):
        t = dict(const, disp=[_dense(p) for p in disps])
        terms, chint, warped, idsel, hpix, state = _kitti_fwd(t, scales, loss_scales, opt)
        ctx.const, ctx.args = const, (scales, loss_scales, opt)
        ctx.save_for_backward(warped, idsel, hpix, state, *t["disp"])
        ctx.mark_non_differentiable(chint, warped, idsel, hpix)
        return terms, chint, warped, idsel, hpix

    @staticmethod
    def backward(ctx, grad_terms, *_):
        warped, idsel, hpix, state, *disps = ctx.saved_tensors
        if grad_terms is None:
            grad_terms = torch.zeros(1 + 3 * len(disps), dtype=torch.float32, device=warped.device)
        t = dict(ctx.const, disp=disps)
        grads = _kitti_bwd(t, *ctx.args, warped, idsel, hpix, state, _dense(grad_terms))
        return (None, None, None, None) + tuple(grads)


def _tensor(t, what, shape):
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32:
        raise _lib.WmdError("%s must be a float32 CUDA tensor" % what)
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s must be %s, got %s" % (what, tuple(shape), tuple(t.shape)))
    return _dense(t.detach())


class KittiDepthHintsLoss:
    """The reference's KITTI objective with ``--use_depth_hints --frame_ids 0 --use_stereo`` (argument names and
    defaults are options.py's).  Automasking and SSIM are on; monocular frames, ``v1_multiscale``,
    ``avg_reprojection``, ``no_ssim`` and disabled automasking are outside it and are not parameters.

    ``__call__(inputs, outputs) -> (total, losses)``.  ``inputs`` holds the reference's ("color", 0, s) for each loss
    scale, ("color", "s", 0), ("K", 0), ("inv_K", 0), "stereo_T", "depth_hint" and "depth_hint_mask"; ``outputs`` the
    decoder's ("disp", s) for each loss scale, (N, 1, H / 2**s, W / 2**s).  All float32 CUDA tensors; a missing key
    raises KeyError, a wrong shape ValueError, a wrong dtype or device WmdError.  ``losses`` holds "reproj_loss/s",
    "depth_hint_loss/s", "loss/s" and "loss" as 0-dim tensors; ``total`` is ``losses["loss"]``, divided by
    ``len(scales)`` as the reference divides it.  Into ``outputs`` go the keys ``Trainer.log()`` reads:
    ("color", "s", s), ("color_depth_hint", "s", 0), "identity_selection/s" and "depth_hint_pixels/s".
    Gradients flow to the ("disp", s) only."""

    def __init__(self, height=192, width=640, scales=SCALES, loss_scales=SCALES, min_depth=0.1, max_depth=100.0,
                 disparity_smoothness=1e-3):
        if height % 8 or width % 8 or height < 8 or width < 8:
            raise ValueError("height and width must be positive multiples of 8, got %d x %d" % (height, width))
        self.height, self.width = int(height), int(width)
        self.scales = tuple(int(s) for s in scales)
        self.loss_scales = tuple(sorted(int(s) for s in loss_scales))
        if not self.loss_scales or not set(self.loss_scales) <= set(SCALES) or len(self.scales) > 4 \
                or len(self.loss_scales) > len(self.scales):
            raise ValueError("loss_scales %s must be a non-empty subset of 0..3 no longer than scales %s"
                             % (tuple(loss_scales), tuple(scales)))
        if not 0 < min_depth < max_depth:
            raise ValueError("need 0 < min_depth < max_depth, got %s, %s" % (min_depth, max_depth))
        self.opt = (float(min_depth), float(max_depth), float(disparity_smoothness))

    @_on_device
    def __call__(self, inputs, outputs):
        tgt = inputs[("color", 0, 0)]
        n = int(tgt.shape[0]) if torch.is_tensor(tgt) and tgt.dim() == 4 else -1
        H, W = self.height, self.width
        const = {"target": _tensor(tgt, "(\"color\", 0, 0)", (n, 3, H, W)),
                 "source": _tensor(inputs[("color", "s", 0)], "(\"color\", \"s\", 0)", (n, 3, H, W)),
                 "K": _tensor(inputs[("K", 0)], "(\"K\", 0)", (n, 4, 4)),
                 "inv_K": _tensor(inputs[("inv_K", 0)], "(\"inv_K\", 0)", (n, 4, 4)),
                 "stereo_T": _tensor(inputs["stereo_T"], "stereo_T", (n, 4, 4)),
                 "depth_hint": _tensor(inputs["depth_hint"], "depth_hint", (n, 1, H, W)),
                 "depth_hint_mask": _tensor(inputs["depth_hint_mask"], "depth_hint_mask", (n, 1, H, W)),
                 "color": [_tensor(inputs[("color", 0, s)], str(("color", 0, s)), (n, 3, H >> s, W >> s))
                           for s in self.loss_scales]}
        disps = [outputs[("disp", s)] for s in self.loss_scales]
        for s, p in zip(self.loss_scales, disps):
            _tensor(p, str(("disp", s)), (n, 1, H >> s, W >> s))
        # the reference's tie-breaking draw: CPU generator, one (N, 1, H, W) per loss scale, in order
        const["noise"] = [torch.randn((n, 1, H, W)).to(tgt.device) for _ in self.loss_scales]
        terms, chint, warped, idsel, hpix = _KittiLossFn.apply(const, self.scales, self.loss_scales, self.opt, *disps)
        outputs[("color_depth_hint", "s", 0)] = chint
        losses = {}
        for i, s in enumerate(self.loss_scales):
            outputs[("color", "s", s)] = warped[i]
            outputs["identity_selection/%d" % s] = idsel[i]
            outputs["depth_hint_pixels/%d" % s] = hpix[i]
            losses["reproj_loss/%d" % s] = terms[1 + 3 * i]
            losses["depth_hint_loss/%d" % s] = terms[2 + 3 * i]
            losses["loss/%d" % s] = terms[3 + 3 * i]
        losses["loss"] = terms[0]
        return terms[0], losses
