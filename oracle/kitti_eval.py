"""numpy fp64 restatement of the KITTI depth evaluation (KITTI/evaluate_depth.py), per frame, and its synthetic split.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  ``evaluate_frame`` follows evaluate_depth.py:276-307 for one
frame, with cv2.resize's INTER_LINEAR rule restated in fp64 (``resize_linear``) so that the checker needs no OpenCV;
``oracle/pin_kitti_eval.py`` checks it against the unmodified reference and against cv2 where cv2 is importable.
"""
import warnings

import numpy as np

MIN_DEPTH, MAX_DEPTH = 1e-3, 80            # evaluate_depth.py:85-86
STEREO_SCALE_FACTOR = 5.4                  # evaluate_depth.py:35
GT_SIZES = ((375, 1242), (370, 1226), (374, 1238), (376, 1241))     # the KITTI Eigen ground-truth sizes
DISP_SIZES = ((192, 640), (320, 1024))
# the four evaluation modes the fixture pins: name -> (eval_split, median_scaling, pred_depth_scale_factor)
MODES = {
    "mono_eigen": ("eigen", True, 1.0),
    "mono_eigen_benchmark": ("eigen_benchmark", True, 1.0),
    "stereo_eigen": ("eigen", False, STEREO_SCALE_FACTOR),
    "stereo_eigen_benchmark": ("eigen_benchmark", False, STEREO_SCALE_FACTOR),
}


def compute_errors(gt, pred):
    """evaluate_depth.py:50-68, verbatim."""
    thresh = np.maximum((gt / pred), (pred / gt))
    a1 = (thresh < 1.25).mean()
    a2 = (thresh < 1.25 ** 2).mean()
    a3 = (thresh < 1.25 ** 3).mean()
    rmse = np.sqrt(((gt - pred) ** 2).mean())
    rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
    abs_rel = np.mean(np.abs(gt - pred) / gt)
    sq_rel = np.mean(((gt - pred) ** 2) / gt)
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


def batch_post_process_disparity(l_disp, r_disp):
    """evaluate_depth.py:71-79, verbatim."""
    _, h, w = l_disp.shape
    m_disp = 0.5 * (l_disp + r_disp)
    l, _ = np.meshgrid(np.linspace(0, 1, w), np.linspace(0, 1, h))
    l_mask = (1.0 - np.clip(20 * (l - 0.05), 0, 1))[None, ...]
    r_mask = l_mask[:, :, ::-1]
    return r_mask * l_disp + l_mask * r_disp + (1.0 - l_mask - r_mask) * m_disp


def _axis(dst, src):
    """cv2 INTER_LINEAR taps of one axis: f = (d + 0.5) src / dst - 0.5, s = floor(f), weight f - s; s < 0 -> s = 0 with
    weight 0; s >= src - 1 -> s = src - 1 with weight 0 (and, horizontally, a single tap)."""
    d = np.arange(dst, dtype=np.float64)
    f = (d + 0.5) * (src / dst) - 0.5
    s = np.floor(f)
    a = f - s
    s = s.astype(np.int64)
    a[s < 0] = 0.0
    s[s < 0] = 0
    last = s >= src - 1
    a[last] = 0.0
    s[last] = src - 1
    return s, np.minimum(s + 1, src - 1), a, last


def resize_linear(src, H, W):
    """cv2.resize(src, (W, H)) for a 2-D float64 image, INTER_LINEAR, in fp64: horizontal pass, then vertical."""
    src = np.asarray(src, dtype=np.float64)
    h, w = src.shape
    sx, sx1, ax, lastx = _axis(W, w)
    sy, sy1, ay, _ = _axis(H, h)
    with np.errstate(invalid="ignore"):
        rows = src[:, sx] * (1 - ax) + src[:, sx1] * ax
        rows[:, lastx] = src[:, sx[lastx]]
        return rows[sy] * (1 - ay)[:, None] + rows[sy1] * ay[:, None]


def valid_mask(gt_depth, eval_split):
    """evaluate_depth.py:283-293."""
    gt_height, gt_width = gt_depth.shape[:2]
    if eval_split == "eigen":
        mask = np.logical_and(gt_depth > MIN_DEPTH, gt_depth < MAX_DEPTH)
        crop = np.array([0.40810811 * gt_height, 0.99189189 * gt_height,
                         0.03594771 * gt_width, 0.96405229 * gt_width]).astype(np.int32)
        crop_mask = np.zeros(mask.shape)
        crop_mask[crop[0]:crop[1], crop[2]:crop[3]] = 1
        return np.logical_and(mask, crop_mask)
    return gt_depth > 0


def evaluate_frame(gt_depth, pred_disp, eval_split="eigen", median_scaling=True, pred_depth_scale_factor=1.0):
    """evaluate_depth.py:276-307 for one frame -> (errors (7,), ratio (1.0 without median scaling), valid count)."""
    gt_height, gt_width = gt_depth.shape[:2]
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        pred_depth = 1 / resize_linear(pred_disp, gt_height, gt_width)
        mask = valid_mask(gt_depth, eval_split)
        pred_depth = pred_depth[mask]
        gt = gt_depth[mask]
        pred_depth *= pred_depth_scale_factor
        ratio = 1.0
        if median_scaling:
            ratio = np.median(gt) / np.median(pred_depth)
            pred_depth *= ratio
        pred_depth[pred_depth < MIN_DEPTH] = MIN_DEPTH
        pred_depth[pred_depth > MAX_DEPTH] = MAX_DEPTH
        return np.array(compute_errors(gt, pred_depth), dtype=np.float64), float(ratio), int(mask.sum())


def evaluate(gt_depths, pred_disps, mode):
    """Every frame of a split in one of MODES -> errors (N, 7), ratios (N,), counts (N,)."""
    split, med, sf = MODES[mode]
    res = [evaluate_frame(g, d, split, med, sf) for g, d in zip(gt_depths, pred_disps)]
    return (np.stack([r[0] for r in res]), np.array([r[1] for r in res]), np.array([r[2] for r in res], np.int64))


# ------------------------------------------------------------------------------------------ synthetic split
SPECIAL = ("empty", "one_valid", "even_count", "all_equal", "zero_disp", "nan_disp", "negative_disp")


def synthetic_split(seed, n_regular=9):
    """Deterministic KITTI-like inputs: dict with
      gt:        list of float32 (H, W) ground truths cycling through GT_SIZES, ~5 % of pixels set (LiDAR-like), values
                 spread over [0, 100] including some exactly float32(1e-3) and 80;
      disp:      {(h, w): (N, h, w) float32 disparities} for DISP_SIZES, ~1 / depth of the same scene with noise;
      special:   {name: frame index} for the frames of SPECIAL, which follow the n_regular regular frames.
    """
    rng = np.random.default_rng(seed)
    n = n_regular + len(SPECIAL)
    gt, scenes = [], []
    for i in range(n):
        H, W = GT_SIZES[i % len(GT_SIZES)]
        coarse = rng.uniform(3.0, 60.0, (6, 20))
        scene = resize_linear(coarse, H, W)                  # smooth depth field of the frame
        scenes.append(coarse)
        lidar = rng.random((H, W)) < 0.05
        g = np.where(lidar, scene * rng.uniform(0.8, 1.25, (H, W)), 0.0).astype(np.float32)
        ys, xs = np.nonzero(lidar)
        pick = rng.choice(ys.size, 64, replace=False)
        g[ys[pick[:16]], xs[pick[:16]]] = np.float32(1e-3)
        g[ys[pick[16:32]], xs[pick[16:32]]] = np.float32(80.0)
        g[ys[pick[32:48]], xs[pick[32:48]]] = rng.uniform(80.0, 100.0, 16).astype(np.float32)
        g[ys[pick[48:]], xs[pick[48:]]] = rng.uniform(0.0, 1e-3, 16).astype(np.float32)
        gt.append(g)
    special = {name: n_regular + k for k, name in enumerate(SPECIAL)}

    def inner(g, count):
        """count pixels inside both the Eigen crop and the frame, the rest zero."""
        H, W = g.shape
        out = np.zeros_like(g)
        ys = rng.integers(int(0.45 * H), int(0.95 * H), count)
        xs = rng.integers(int(0.05 * W), int(0.95 * W), count)
        flat = np.unique(ys * W + xs)[:count]
        out.flat[flat] = rng.uniform(1.0, 70.0, flat.size).astype(np.float32)
        return out, flat
    gt[special["empty"]] = np.zeros_like(gt[special["empty"]])
    gt[special["one_valid"]], _ = inner(gt[special["one_valid"]], 1)
    g, flat = inner(gt[special["even_count"]], 1000)
    if flat.size % 2:
        g.flat[flat[-1]] = 0.0
    gt[special["even_count"]] = g
    g, flat = inner(gt[special["all_equal"]], 500)
    g.flat[flat] = np.float32(20.0)
    gt[special["all_equal"]] = g

    disp = {}
    for (h, w) in DISP_SIZES:
        d = np.stack([(0.3 / resize_linear(c, h, w)) * rng.uniform(0.9, 1.1, (h, w)) for c in scenes]).astype(np.float32)
        d[special["zero_disp"], : h // 3, : w // 4] = 0.0
        d[special["nan_disp"], h // 2:h // 2 + 8, w // 2:w // 2 + 8] = np.nan          # reaches ~13 valid pixels
        d[special["negative_disp"], h // 2:, w // 2:] *= -1.0
        disp[(h, w)] = d
    return dict(gt=gt, disp=disp, special=special)


def post_process_inputs(seed, n=2, h=192, w=640):
    """float32 (n, h, w) left and right-flipped disparities for batch_post_process_disparity, as the reference forms
    them from disp_to_depth's float32 output (evaluate_depth.py:195,204)."""
    rng = np.random.default_rng(seed)
    l_disp = rng.uniform(0.01, 0.3, (n, h, w)).astype(np.float32)
    r_disp = rng.uniform(0.01, 0.3, (n, h, w)).astype(np.float32)
    return l_disp, r_disp
