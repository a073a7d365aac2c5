"""KITTI depth evaluation on the device: the reference's KITTI/evaluate_depth.py for whole batches of predictions.

The split's ground truth is uploaded and its valid pixels found once (``KittiDepthEvaluator``); each ``add`` then samples
the predicted disparities at those pixels, takes the per-frame medians and sums the seven metrics on the device, with
no host wait.  ``summary`` does the one read-back.  Every metric is computed in fp64 in a fixed order, so results do not
depend on how the split is chunked into ``add`` calls.
"""
import numpy as np
import torch

from . import _lib
from .ops import _dense, _launch, _on_device, compact

_f64 = torch.float64
METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")
STEREO_SCALE_FACTOR = 5.4          # evaluate_depth.py:35


def _disp_args(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise _lib.WmdError("%s must be a CUDA tensor" % what)
    if t.dtype not in (torch.float32, _f64):
        raise _lib.WmdError("%s must be float32 or float64, got %s" % (what, t.dtype))
    return _dense(t, t.dtype), int(t.dtype == _f64)


@_on_device
def compute_errors(gt, pred):
    """evaluate_depth.py:50-68 on CUDA tensors of valid pixels -> (7,) fp64 device tensor
    (abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3), summed in fp64; log(gt) is taken in fp64 too."""
    if not (torch.is_tensor(gt) and torch.is_tensor(pred) and gt.is_cuda and pred.is_cuda):
        raise _lib.WmdError("compute_errors takes CUDA tensors")
    if gt.dtype not in (torch.float32, _f64) or pred.dtype not in (torch.float32, _f64) or gt.numel() != pred.numel():
        raise _lib.WmdError("compute_errors takes float tensors of equal size")
    if gt.numel() >= 2 ** 31:
        raise _lib.WmdError("compute_errors: too many pixels")
    gt, pred = _dense(gt.reshape(-1), _f64), _dense(pred.reshape(-1), _f64)
    out = torch.empty(7, dtype=_f64, device=gt.device)
    _launch().wmd_eval_errors_f64(_lib.ptr(gt), _lib.ptr(pred), gt.numel(), _lib.ptr(out), _lib.stream_ptr())
    return out


@_on_device
def batch_post_process_disparity(l_disp, r_disp):
    """evaluate_depth.py:71-79: l_disp, r_disp (N, h, w) CUDA tensors, both float32 or both float64 (r_disp already
    flipped back, as the reference's caller passes it) -> (N, h, w) fp64."""
    lt, l64 = _disp_args(l_disp, "l_disp")
    rt, r64 = _disp_args(r_disp, "r_disp")
    if l64 != r64 or lt.dim() != 3 or lt.shape != rt.shape:
        raise _lib.WmdError("batch_post_process_disparity: l_disp and r_disp must be (N, h, w) of one dtype")
    n, h, w = lt.shape
    out = torch.empty((n, h, w), dtype=_f64, device=lt.device)
    if out.numel() == 0:
        return out
    _launch("post_process_disparity", lambda: dict(n=n, h=h, w=w)).wmd_post_process_disparity(
        _lib.ptr(lt), _lib.ptr(rt), l64, _lib.ptr(out), n, h, w, _lib.stream_ptr())
    return out


def compute_density(sparse_outputs):
    """evaluate_depth.py:37-47 per sample: active wavelet-mask pixels over all pixels of the four scales -> (N,) fp64
    device tensor (integer sums, then one division, so a batch of one gives the reference's float)."""
    num, den = None, 0
    for i in range(4):
        m = sparse_outputs.get(("wavelet_mask", i))
        if m is None:
            continue
        s = m.sum(dim=(1, 2, 3), dtype=torch.int64)
        num = s if num is None else num + s
        den += int(m.shape[2]) * int(m.shape[3])
    if num is None:
        raise _lib.WmdError("compute_density: no ('wavelet_mask', i) outputs")
    num = num.to(_f64)
    return num / torch.full_like(num, float(den))      # a true division (a Python-scalar divisor may become a reciprocal)


class KittiDepthEvaluator:
    """evaluate_depth.py:258-323 for a fixed ground-truth split, on the device.

    gt_depths: list of per-frame (H, W) depth maps (numpy arrays or tensors; KITTI's are float32 at mixed sizes).  They
    are uploaded, masked (eval_split "eigen": depth range and Eigen crop; any other split: gt > 0) and compacted once.
    Stereo evaluation is ``median_scaling=False, pred_depth_scale_factor=5.4`` (:263-267).

    ``add(pred_disp)`` scores the next frames of the split: (n, 1, h, w) or (n, h, w) float32 disparities (disp_to_depth's
    scaled disparity) or float64 (post-processed), h and w no larger than any frame's.  It never waits on the device, so
    it can be captured in a CUDA graph.  ``errors`` (frames, 7) and ``ratios`` (frames,) are device tensors.

    The reference takes rmse_log's log(gt) with numpy's float32 log of the float32 ground truth, which is not correctly
    rounded; the evaluator takes that same log once per split, on the host, so that its metrics match the reference's.
    """

    def __init__(self, gt_depths, eval_split="eigen", median_scaling=True, pred_depth_scale_factor=1.0, device=None):
        frames = [g.detach().cpu().numpy() if torch.is_tensor(g) else np.asarray(g) for g in gt_depths]
        if not frames or any(f.ndim != 2 for f in frames):
            raise _lib.WmdError("gt_depths must be a non-empty list of (H, W) depth maps")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise _lib.WmdError("KittiDepthEvaluator runs on a CUDA device only")
        self.eval_split, self.median_scaling = eval_split, bool(median_scaling)
        self.pred_depth_scale_factor = float(pred_depth_scale_factor)
        n = len(frames)
        sizes = np.array([f.shape for f in frames], dtype=np.int32)
        self.h_max, self.w_max = (int(v) for v in sizes.max(0))
        self.h_min, self.w_min = (int(v) for v in sizes.min(0))
        padded = np.zeros((n, self.h_max, self.w_max), dtype=np.float32)
        for i, f in enumerate(frames):
            padded[i, :f.shape[0], :f.shape[1]] = f
        with torch.cuda.device(self.device):
            gt = torch.from_numpy(padded).to(self.device)
            self.hw = torch.from_numpy(sizes).to(self.device)
            mask = torch.empty(gt.shape, dtype=torch.uint8, device=self.device)
            split = _lib.EVAL_EIGEN if eval_split == "eigen" else _lib.EVAL_GT_POSITIVE
            _launch().wmd_eval_gt_mask(
                _lib.ptr(gt), _lib.ptr(self.hw), _lib.ptr(mask), n, self.h_max, self.w_max, split, _lib.stream_ptr())
            _, pixels, self.offsets = compact(mask, want_idxmap=False)
            total = int(self.offsets[-1])                 # the split's one read-back: sizes the buffers below
            self.pixels = pixels[:max(total, 1)].clone()
            self.gt = torch.empty(max(total, 1), dtype=torch.float32, device=self.device)
            _launch().wmd_eval_gather_f32(
                _lib.ptr(gt), _lib.ptr(self.pixels), _lib.ptr(self.offsets[n:]), total, _lib.ptr(self.gt),
                _lib.stream_ptr())
            with np.errstate(all="ignore"):
                self.gt_log = torch.from_numpy(np.log(self.gt.cpu().numpy())).to(self.device)
            self.depth = torch.empty(max(total, 1), dtype=_f64, device=self.device)
            self.errors = torch.full((n, 7), float("nan"), dtype=_f64, device=self.device)
            self.ratios = torch.full((n,), float("nan"), dtype=_f64, device=self.device)
            self.counts = torch.zeros((n,), dtype=torch.int32, device=self.device)
        self.num_frames, self.next_frame = n, 0
        self._density, self._total_ops = [], []

    def reset(self):
        """Start scoring the split again from its first frame (the next threshold of a sweep)."""
        self.next_frame = 0
        self._density, self._total_ops = [], []

    def add(self, pred_disp, sparse_outputs=None):
        """Score the next n frames; with the sparse decoder's outputs also record their densities and op counts."""
        disp, f64 = _disp_args(pred_disp, "pred_disp")
        if disp.dim() == 4 and disp.shape[1] == 1:
            disp = disp[:, 0]
        if disp.dim() != 3:
            raise _lib.WmdError("pred_disp must be (n, 1, h, w) or (n, h, w), got %s" % (tuple(pred_disp.shape),))
        if disp.device != self.device:
            raise _lib.WmdError("pred_disp is on %s, the split on %s" % (disp.device, self.device))
        n, h, w = (int(v) for v in disp.shape)
        if self.next_frame + n > self.num_frames:
            raise _lib.WmdError("%d more frames than the split's %d" % (self.next_frame + n - self.num_frames,
                                                                        self.num_frames))
        if h > self.h_min or w > self.w_min or h < 1 or w < 1:
            raise _lib.WmdError("pred_disp %dx%d must be no larger than every ground-truth frame (%dx%d)"
                                % (h, w, self.h_min, self.w_min))
        f0 = self.next_frame
        with torch.cuda.device(self.device):
            _launch("eval_frames", lambda: dict(n=n, h=h, w=w)).wmd_eval_frames(
                _lib.ptr(disp), f64, n, h, w, f0, _lib.ptr(self.hw), _lib.ptr(self.pixels), _lib.ptr(self.offsets),
                _lib.ptr(self.gt), _lib.ptr(self.gt_log), self.h_max, self.w_max, self.pred_depth_scale_factor,
                int(self.median_scaling), _lib.ptr(self.depth), _lib.ptr(self.errors[f0:]), _lib.ptr(self.ratios[f0:]),
                _lib.ptr(self.counts[f0:]), _lib.stream_ptr())
        self.next_frame += n
        if sparse_outputs is not None:
            self._density.append(compute_density(sparse_outputs))
            ops = sparse_outputs.get("total_ops_per_sample")
            self._total_ops.append(ops if ops is not None else sparse_outputs.get("total_ops"))

    def summary(self):
        """The reference's printed results (evaluate_depth.py:309-323) for the frames added so far: the frame-order mean
        of the seven metrics; with median scaling ``med`` and ``std`` of the ratios; with sparse outputs ``density_mean``
        / ``density_std`` and ``total_ops_mean`` / ``total_ops_std``."""
        k = self.next_frame
        errors = self.errors[:k].cpu().numpy()
        res = dict(zip(METRICS, (float(v) for v in errors.mean(0))))
        if self.median_scaling:
            ratios = self.ratios[:k].cpu().numpy()
            med = np.median(ratios)
            res["med"], res["std"] = float(med), float(np.std(ratios / med))
        if self._density:
            dens = torch.cat(self._density).cpu().numpy()
            ops = []
            for v in self._total_ops:
                if hasattr(v, "result"):                       # an OpsFuture (count_ops="async")
                    r = v.result()
                    v = r.get("total_ops_per_sample", r["total_ops"])
                ops.extend(v if isinstance(v, (list, tuple)) else [v])
            ops = np.array(ops, dtype=np.float64)
            res.update(density_mean=float(np.mean(dens)), density_std=float(np.std(dens)),
                       total_ops_mean=float(np.mean(ops)), total_ops_std=float(np.std(ops)))
        res["frames"] = k
        return res
