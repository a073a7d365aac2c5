"""NYUv2 depth evaluation on the device: the reference's NYUv2/utils.py evaluate() for whole batches of predictions.

The split's ground truth is uploaded, cropped (Eigen) or resized (224 mode) and its log10 taken once
(``NyuDepthEvaluator``); each ``add`` then runs the reference's prediction chain on the decoder's disparities and sums
compute_errors_nyu's terms per frame on the device, with no host wait.  ``summary`` does the one read-back and pools the
per-frame sums with ``math.fsum``, so results do not depend on how the split is chunked into ``add`` calls.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from .ops import _dense, _on_device, _prof

_f64 = torch.float64
METRICS = ("rel", "rms", "log_10", "a1", "a2", "a3")
GT_SHAPE = (480, 640)
BORDER = 16                                              # utils.py:285
EIGEN_CROP = (20, 459, 24, 615)                          # NYUv2/evaluate.py:56, inclusive


def _cuda(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise _lib.WmdError("%s must be a CUDA tensor" % what)
    return t


@_on_device
def compute_errors_nyu(pred, gt):
    """utils.py:85-98 on two CUDA tensors of equal size -> (6,) fp64 device tensor (rel, rms, log_10, a1, a2, a3), in
    fp64 (log10 of gt too), pooled over a fixed grid of CTAs so the bits do not depend on timing."""
    _cuda(pred, "pred"), _cuda(gt, "gt")
    if pred.dtype not in (torch.float32, _f64) or gt.dtype not in (torch.float32, _f64) or pred.numel() != gt.numel():
        raise _lib.WmdError("compute_errors_nyu takes float tensors of equal size")
    pred, gt = _dense(pred.reshape(-1), _f64), _dense(gt.reshape(-1), _f64)
    n = pred.numel()
    lib = _lib.load()
    ws = torch.empty(int(lib.wmd_eval_nyu_errors_ws_bytes(n)), dtype=torch.uint8, device=pred.device)
    out = torch.empty(6, dtype=_f64, device=pred.device)
    with _prof("eval_nyu_errors", lambda: dict(n=n)):
        rc = lib.wmd_eval_nyu_errors_f64(_lib.ptr(pred), _lib.ptr(gt), n, _lib.ptr(ws), ws.numel(), _lib.ptr(out),
                                         _lib.stream_ptr())
    _lib.check(rc, "wmd_eval_nyu_errors_f64")
    return out


class NyuDepthEvaluator:
    """utils.py:275-372 (without edges, figures or wavelet dumps) for a fixed ground-truth split, on the device.

    gt_depths: (N, 480, 640) depth in metres (numpy array or tensor), cast to float32 as the reference does.  Eigen mode
    crops it to rows 20..459 and columns 24..615; 224 mode (``use_224``) crops its 16-pixel border and resizes it to
    224 x 224 with the reference's own float32 ``F.interpolate`` on the device.  Its log10 is taken once, with
    ``torch.log10`` of the float32 values, as the reference does.

    ``add(disp)`` scores the next n frames: the decoder's ("disp", 0), (n, 1, h, w) or (n, h, w) float32 (any h x w in
    Eigen mode, 224 x 224 in 224 mode).  ``disp`` is not modified, and ``add`` never waits on the device, so it can be
    captured in a CUDA graph.  With ``depth_out`` ((n, 440, 592) or (n, 224, 224) float64 CUDA tensor) it also writes the
    reference's ``predictions``.  ``sums`` (frames, 7) is a device tensor of each frame's fp64 sums: |y - x| / y,
    (y - x)^2, |log10 y - log10 x|, the three threshold counts and the pixel count.
    """

    def __init__(self, gt_depths, use_224=False, use_disparity=False, device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise _lib.WmdError("NyuDepthEvaluator runs on a CUDA device only")
        gt = gt_depths.detach() if torch.is_tensor(gt_depths) else torch.from_numpy(np.asarray(gt_depths))
        if gt.dim() != 3 or tuple(gt.shape[1:]) != GT_SHAPE or gt.shape[0] < 1:
            raise _lib.WmdError("gt_depths must be (N, 480, 640), got %s" % (tuple(gt.shape),))
        self.use_224, self.use_disparity = bool(use_224), bool(use_disparity)
        with torch.cuda.device(self.device):
            g = gt.to(self.device).float()
            if self.use_224:
                g = F.interpolate(g[:, None, BORDER:-BORDER, BORDER:-BORDER], (224, 224), mode="bilinear",
                                  align_corners=True)[:, 0]
            else:
                g = g[:, EIGEN_CROP[0]:EIGEN_CROP[1] + 1, EIGEN_CROP[2]:EIGEN_CROP[3] + 1]
            self.gt = g.contiguous()
            self.gt_log10 = torch.log10(self.gt)
            self.sums = torch.full((gt.shape[0], 7), float("nan"), dtype=_f64, device=self.device)
        self.num_frames, self.next_frame = int(gt.shape[0]), 0
        self.mode = _lib.EVAL_NYU_224 if self.use_224 else _lib.EVAL_NYU_EIGEN

    @property
    def out_shape(self):
        """(H, W) of one frame's prediction map: (440, 592) or (224, 224)."""
        return tuple(self.gt.shape[1:])

    def reset(self):
        """Start scoring the split again from its first frame (the next threshold of a sweep)."""
        self.next_frame = 0

    def add(self, disp, depth_out=None):
        """Score the next n frames of the split."""
        _cuda(disp, "disp")
        if disp.dtype != torch.float32:
            raise _lib.WmdError("disp must be float32, got %s" % disp.dtype)
        d = disp[:, 0] if disp.dim() == 4 and disp.shape[1] == 1 else disp
        if d.dim() != 3:
            raise _lib.WmdError("disp must be (n, 1, h, w) or (n, h, w), got %s" % (tuple(disp.shape),))
        if d.device != self.device:
            raise _lib.WmdError("disp is on %s, the split on %s" % (d.device, self.device))
        n, h, w = (int(v) for v in d.shape)
        if self.next_frame + n > self.num_frames:
            raise _lib.WmdError("%d more frames than the split's %d" % (self.next_frame + n - self.num_frames,
                                                                        self.num_frames))
        if self.use_224 and (h, w) != (224, 224):
            raise _lib.WmdError("224 mode takes 224 x 224 disparities, got %d x %d" % (h, w))
        if h < 1 or w < 1:
            raise _lib.WmdError("disp has no pixels")
        if depth_out is not None:
            _cuda(depth_out, "depth_out")
            if depth_out.dtype != _f64 or tuple(depth_out.shape) != (n,) + self.out_shape or \
                    not depth_out.is_contiguous():
                raise _lib.WmdError("depth_out must be a contiguous float64 %s tensor" % ((n,) + self.out_shape,))
        if n == 0:
            return
        d = d.contiguous()
        f0 = self.next_frame
        lib = _lib.load()
        with torch.cuda.device(self.device), _prof("eval_nyu_frames", lambda: dict(n=n, h=h, w=w)):
            ws = torch.empty(int(lib.wmd_eval_nyu_ws_bytes(n, self.mode)), dtype=torch.uint8, device=self.device)
            rc = lib.wmd_eval_nyu_frames(
                _lib.ptr(d), n, h, w, self.mode, int(self.use_disparity), _lib.ptr(self.gt[f0:]),
                _lib.ptr(self.gt_log10[f0:]), _lib.ptr(depth_out), _lib.ptr(ws), ws.numel(), _lib.ptr(self.sums[f0:]),
                _lib.stream_ptr())
        _lib.check(rc, "wmd_eval_nyu_frames")
        self.next_frame += n

    def summary(self):
        """compute_errors_nyu over every pixel of the frames added so far: each column of ``sums`` pooled with
        math.fsum and divided by the pooled pixel count (a_k is an exact count over it) -> dict of METRICS and
        ``frames``."""
        k = self.next_frame
        s = self.sums[:k].cpu().numpy()
        tot = [math.fsum(s[:, j]) if not np.isnan(s[:, j]).any() else math.nan for j in range(7)]
        with np.errstate(all="ignore"):
            m = np.array(tot[:6]) / np.float64(tot[6])
            m[1] = np.sqrt(m[1])
        res = dict(zip(METRICS, (float(v) for v in m)))
        res["frames"] = k
        return res
