"""NYUv2 depth evaluation on the device: the reference's NYUv2/utils.py evaluate() for whole batches of predictions.

The split's ground truth is uploaded, cropped (Eigen) or resized (224 mode) and its log10 taken once
(``NyuDepthEvaluator``); each ``add`` then runs the reference's prediction chain on the decoder's disparities and sums
compute_errors_nyu's terms per frame on the device, with no host wait.  ``summary`` does the one read-back and pools the
per-frame sums with ``math.fsum``, so results do not depend on how the split is chunked into ``add`` calls.

With ``edges_gt`` the evaluator also scores the depth boundary error (utils.py:122-169, ``--eval_edges``): each frame's
Canny edges of the prediction (scikit-image 0.16.2's canny, restated exactly), their exact distance transform and the
accuracy / completeness chamfer scores, all on the device in the same ``add``.  ``compute_depth_boundary_error`` is the
reference's function of the same name for batches of CUDA tensors.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from .ops import _dense, _launch, _on_device

_f64 = torch.float64
METRICS = ("rel", "rms", "log_10", "a1", "a2", "a3")
GT_SHAPE = (480, 640)
BORDER = 16                                              # utils.py:285
EIGEN_CROP = (20, 459, 24, 615)                          # NYUv2/evaluate.py:56, inclusive
EDGE_SIGMA = math.sqrt(2.0)                              # utils.py:137
EDGE_LOW, EDGE_HIGH = 0.15, 0.3                          # compute_depth_boundary_error's defaults
_CANNY_FILTERS = {}


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
    ws = torch.empty(int(_lib.load().wmd_eval_nyu_errors_ws_bytes(n)), dtype=torch.uint8, device=pred.device)
    out = torch.empty(6, dtype=_f64, device=pred.device)
    _launch("eval_nyu_errors", lambda: dict(n=n)).wmd_eval_nyu_errors_f64(
        _lib.ptr(pred), _lib.ptr(gt), n, _lib.ptr(ws), ws.numel(), _lib.ptr(out), _lib.stream_ptr())
    return out


def _canny_filters(h, w, device):
    """The gaussian skimage's canny smooths with, for an h x w frame on `device`, uploaded once per shape: scipy's
    13 weights for sigma sqrt(2) (w0 .. w6, read back as scipy's own impulse response, so they are its bits) and the
    bleed-over map, scipy's gaussian_filter of a map of ones (it depends only on the shape)."""
    key = (int(h), int(w), str(device))
    if key not in _CANNY_FILTERS:
        from scipy import ndimage as ndi
        delta = np.zeros(13)
        delta[6] = 1.0
        taps = ndi.gaussian_filter1d(delta, EDGE_SIGMA, mode="constant", truncate=4.0)[6:]
        bleed = ndi.gaussian_filter(np.ones((h, w)), EDGE_SIGMA, mode="constant", truncate=4.0)
        _CANNY_FILTERS[key] = (torch.from_numpy(np.ascontiguousarray(taps)).to(device),
                               torch.from_numpy(bleed).to(device))
    return _CANNY_FILTERS[key]


def _edges_f32(edges, what):
    """An OC++ edge map as the reference holds it: float32 k / 255 (evaluate.py:73-75 divides the uint8 PNG value in
    float64 and stores it in float32); a uint8 map is converted so, a float32 one taken as it is."""
    e = edges.detach() if torch.is_tensor(edges) else torch.from_numpy(np.asarray(edges))
    if e.dtype == torch.uint8:
        e = (e.double() / 255.0).float()
    elif e.dtype != torch.float32:
        raise _lib.WmdError("%s must be float32 (k / 255) or uint8, got %s" % (what, e.dtype))
    return e


def _gt_sums(edges_np):
    """(n, 2) fp64: each frame's np.sum and np.nansum, numpy's own float32 sums of the view it is given"""
    return np.array([[np.sum(e), np.nansum(e)] for e in edges_np], np.float64).reshape(-1, 2)


def _edt(features, out):
    """wmd_eval_edt of (n, h, w) byte feature masks into `out` (n, h, w) fp64"""
    n, h, w = (int(v) for v in features.shape)
    ws = torch.empty(int(_lib.load().wmd_eval_edt_ws_bytes(n, h, w)), dtype=torch.uint8, device=features.device)
    _launch("eval_edt", lambda: dict(n=n, h=h, w=w)).wmd_eval_edt(
        _lib.ptr(features), n, h, w, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    return out


def _edges_frames(pred, edges_gt, d_gt, gt_sums, scores, low, high):
    """wmd_eval_edges_frames on (n, h, w) pred (fp32 or fp64) -> (edges_est bool, d_est fp64); writes scores (n, 2)"""
    n, h, w = (int(v) for v in pred.shape)
    dev = pred.device
    taps, bleed = _canny_filters(h, w, dev)
    edges_est = torch.empty((n, h, w), dtype=torch.bool, device=dev)
    d_est = torch.empty((n, h, w), dtype=_f64, device=dev)
    ws = torch.empty(int(_lib.load().wmd_eval_edges_ws_bytes(n, h, w)), dtype=torch.uint8, device=dev)
    _launch("eval_edges_frames", lambda: dict(n=n, h=h, w=w)).wmd_eval_edges_frames(
        _lib.ptr(pred), int(pred.dtype == _f64), n, h, w, _lib.ptr(taps), _lib.ptr(bleed), float(low), float(high),
        _lib.ptr(edges_gt), _lib.ptr(d_gt), _lib.ptr(gt_sums), _lib.ptr(edges_est), _lib.ptr(d_est), _lib.ptr(scores),
        _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    return edges_est, d_est


@_on_device
def compute_depth_boundary_error(edges_gt, pred, mask=None, low_thresh=EDGE_LOW, high_thresh=EDGE_HIGH):
    """utils.py:122-169 for a batch: edges_gt and pred (n, h, w) or (h, w) CUDA tensors of one size (edges_gt float32
    k / 255 or uint8, pred float32, or float64 which is rounded to float32 as the reference's ``astype('f')`` does)
    -> (dbe_acc (n,), dbe_com (n,) fp64, edges_est (n, h, w) bool, D_est (n, h, w) fp64), all on the device.

    A frame whose edges_gt sums to 0 scores NaN, NaN (the reference's intent: its own function raises
    UnboundLocalError there, returning the D_est it never computed); its edges_est and D_est are still the
    prediction's.  The two ground-truth sums are numpy's float32 sums, so edges_gt is read back to the host once."""
    if mask is not None:
        raise _lib.WmdError("compute_depth_boundary_error takes no mask (the reference's callers pass none)")
    _cuda(edges_gt, "edges_gt"), _cuda(pred, "pred")
    if pred.dtype not in (torch.float32, _f64):
        raise _lib.WmdError("pred must be float32 or float64, got %s" % pred.dtype)
    if edges_gt.device != pred.device:
        raise _lib.WmdError("edges_gt is on %s, pred on %s" % (edges_gt.device, pred.device))
    squeeze = pred.dim() == 2
    p = pred[None] if squeeze else pred
    g = _edges_f32(edges_gt[None] if edges_gt.dim() == 2 else edges_gt, "edges_gt")
    if p.dim() != 3 or tuple(g.shape) != tuple(p.shape) or min(p.shape[1:]) < 1:
        raise _lib.WmdError("edges_gt and pred must be (n, h, w) or (h, w) of one size, got %s and %s"
                            % (tuple(edges_gt.shape), tuple(pred.shape)))
    p, g = p.contiguous(), g.contiguous()
    n = int(p.shape[0])
    sums = torch.from_numpy(_gt_sums(g.cpu().numpy())).to(p.device)
    d_gt = _edt((g == 1).to(torch.uint8), torch.empty(g.shape, dtype=_f64, device=p.device))
    scores = torch.empty((n, 2), dtype=_f64, device=p.device)
    edges_est, d_est = _edges_frames(p, g, d_gt, sums, scores, low_thresh, high_thresh)
    if squeeze:
        return scores[0, 0], scores[0, 1], edges_est[0], d_est[0]
    return scores[:, 0], scores[:, 1], edges_est, d_est


class NyuDepthEvaluator:
    """utils.py:275-372 (with edges optional; without figures or wavelet dumps) for a fixed ground-truth split, on the
    device.

    gt_depths: (N, 480, 640) depth in metres (numpy array or tensor), cast to float32 as the reference does.  Eigen mode
    crops it to rows 20..459 and columns 24..615; 224 mode (``use_224``) crops its 16-pixel border and resizes it to
    224 x 224 with the reference's own float32 ``F.interpolate`` on the device.  Its log10 is taken once, with
    ``torch.log10`` of the float32 values, as the reference does.

    ``add(disp)`` scores the next n frames: the decoder's ("disp", 0), (n, 1, h, w) or (n, h, w) float32 (any h x w in
    Eigen mode, 224 x 224 in 224 mode).  ``disp`` is not modified, and ``add`` never waits on the device, so it can be
    captured in a CUDA graph.  With ``depth_out`` ((n, 440, 592) or (n, 224, 224) float64 CUDA tensor) it also writes the
    reference's ``predictions``.  ``sums`` (frames, 7) is a device tensor of each frame's fp64 sums: |y - x| / y,
    (y - x)^2, |log10 y - log10 x|, the three threshold counts and the pixel count.

    edges_gt: (N, 480, 640) OC++ edge maps, float32 k / 255 as evaluate.py loads them (a uint8 0..255 map is
    converted the same way), Eigen mode only.  Each is cropped like the depth, and its distance map and numpy's float32
    sum are taken once.  ``add`` then also scores each frame's depth boundary error on the fp64 prediction map rounded
    to float32 (the correctly rounded value of the reference's float32 chain) into ``edges_scores`` (frames, 2) fp64,
    (dbe_acc, dbe_comp), still without a host wait; ``summary`` adds their NaN-propagating means ``e_acc``, ``e_comp``.
    """

    def __init__(self, gt_depths, use_224=False, use_disparity=False, device=None, edges_gt=None):
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
        self.edges_gt = self.edges_scores = None
        if edges_gt is not None:
            self._init_edges(edges_gt)

    def _init_edges(self, edges_gt):
        if self.use_224:
            raise _lib.WmdError("edge metrics need the Eigen crop; 224 mode has none (the reference crops the "
                                "480 x 640 edge map against a 224 x 224 prediction there and fails)")
        e = _edges_f32(edges_gt, "edges_gt")
        if tuple(e.shape) != (self.num_frames,) + GT_SHAPE:
            raise _lib.WmdError("edges_gt must be (%d, 480, 640), got %s" % (self.num_frames, tuple(e.shape)))
        crop = (slice(None), slice(EIGEN_CROP[0], EIGEN_CROP[1] + 1), slice(EIGEN_CROP[2], EIGEN_CROP[3] + 1))
        sums = _gt_sums(e.cpu().numpy()[crop])                 # the reference sums the cropped view (utils.py:124)
        with torch.cuda.device(self.device):
            g = e.to(self.device)[crop].contiguous()
            self.edges_gt = g
            self.edges_gt_sums = torch.from_numpy(sums).to(self.device)
            self.d_gt = _edt((g == 1).to(torch.uint8), torch.empty(g.shape, dtype=_f64, device=self.device))
            self.edges_scores = torch.full((self.num_frames, 2), float("nan"), dtype=_f64, device=self.device)
        _canny_filters(*self.out_shape, self.device)           # uploaded here, so that add() can be graph-captured

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
        with torch.cuda.device(self.device):
            if self.edges_gt is not None and depth_out is None:
                depth_out = torch.empty((n,) + self.out_shape, dtype=_f64, device=self.device)
            ws = torch.empty(int(_lib.load().wmd_eval_nyu_ws_bytes(n, self.mode)), dtype=torch.uint8, device=self.device)
            _launch("eval_nyu_frames", lambda: dict(n=n, h=h, w=w)).wmd_eval_nyu_frames(
                _lib.ptr(d), n, h, w, self.mode, int(self.use_disparity), _lib.ptr(self.gt[f0:]),
                _lib.ptr(self.gt_log10[f0:]), _lib.ptr(depth_out), _lib.ptr(ws), ws.numel(), _lib.ptr(self.sums[f0:]),
                _lib.stream_ptr())
            if self.edges_gt is not None:
                _edges_frames(depth_out, self.edges_gt[f0:f0 + n], self.d_gt[f0:f0 + n],
                              self.edges_gt_sums[f0:f0 + n], self.edges_scores[f0:f0 + n], EDGE_LOW, EDGE_HIGH)
        self.next_frame += n

    def summary(self):
        """compute_errors_nyu over every pixel of the frames added so far: each column of ``sums`` pooled with
        math.fsum and divided by the pooled pixel count (a_k is an exact count over it) -> dict of METRICS and
        ``frames``; with edges also ``e_acc`` and ``e_comp``, the reference's ``edges_scores.mean(0)`` (np.mean, so one
        frame without ground-truth edges makes them NaN)."""
        k = self.next_frame
        s = self.sums[:k].cpu().numpy()
        tot = [math.fsum(s[:, j]) if not np.isnan(s[:, j]).any() else math.nan for j in range(7)]
        with np.errstate(all="ignore"):
            m = np.array(tot[:6]) / np.float64(tot[6])
            m[1] = np.sqrt(m[1])
        res = dict(zip(METRICS, (float(v) for v in m)))
        res["frames"] = k
        if self.edges_scores is not None:
            e = self.edges_scores[:k].cpu().numpy().mean(0) if k else np.full(2, np.nan)
            res["e_acc"], res["e_comp"] = float(e[0]), float(e[1])
        return res
