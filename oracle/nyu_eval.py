"""numpy restatement of the NYUv2 depth evaluation (NYUv2/utils.py: add_results, evaluate, compute_errors_nyu), and its
synthetic splits.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  ``predict`` is the reference's prediction chain (utils.py:216-229 and
the Eigen crop at :252-253) in fp64, in torch's bilinear formula and order, so that it equals the device's map bit for
bit; ``frame_sums`` and ``metrics`` are compute_errors_nyu (:85-98) pooled over every pixel of every frame.  The ground
truth's log10 is an input: the reference takes torch's float32 log10 of the float32 ground truth.
``oracle/pin_nyu_eval.py`` checks all of it against the unmodified reference.
"""
import math

import numpy as np

EIGEN_CROP = (20, 459, 24, 615)            # NYUv2/evaluate.py:56, rows 20..459 and columns 24..615 inclusive
BORDER = 16                                # utils.py:285
MIN_DEPTH, MAX_DEPTH = 0.4, 10.0           # utils.py:229
THRESHOLDS = (1.25, 1.25 ** 2, 1.25 ** 3)
GT_SHAPE = (480, 640)
DISP_SIZES = ((240, 320), (60, 80), (241, 319))      # Eigen mode; 224 mode takes (224, 224)
METRICS = ("rel", "rms", "log_10", "a1", "a2", "a3")
# the evaluation modes the fixture pins: name -> (use_224, use_disparity)
MODES = {"eigen": (False, False), "eigen_disp": (False, True), "224": (True, False), "224_disp": (True, True)}


def _axis(out, inp, dtype=np.float64):
    """torch's align_corners=True taps of one axis: scale (in - 1) / (out - 1), src = scale * d, i0 = int(src),
    lambda = src - i0, i1 = i0 + (i0 < in - 1); weights (1 - lambda, lambda)."""
    scale = dtype((inp - 1) / (out - 1) if dtype is np.float64 else np.float32(inp - 1) / np.float32(out - 1)) \
        if out > 1 else dtype(0)
    src = scale * np.arange(out).astype(dtype)
    i0 = np.minimum(src.astype(np.int64), inp - 1)
    lam = (src - i0.astype(dtype)).astype(dtype)
    i1 = i0 + (i0 < inp - 1)
    return i0, i1, (dtype(1) - lam).astype(dtype), lam


def resize_ac(a, H, W, dtype=np.float64, skip_zero_weight=False):
    """F.interpolate(a, (H, W), mode='bilinear', align_corners=True) of (..., h, w), evaluated in `dtype` as
    h0 * (w0 * x00 + w1 * x01) + h1 * (w0 * x10 + w1 * x11).  Every tap is read and multiplied, a zero weight included,
    as torch does; ``skip_zero_weight`` leaves zero-weight taps out (only to show that this matters)."""
    a = np.asarray(a, dtype)
    y0, y1, h0, h1 = _axis(H, a.shape[-2], dtype)
    x0, x1, w0, w1 = _axis(W, a.shape[-1], dtype)
    r0, r1 = a[..., y0, :], a[..., y1, :]
    with np.errstate(invalid="ignore", over="ignore"):
        def lerp(lo, hi, wl, wh):
            t = wl * lo + wh * hi
            if skip_zero_weight:
                t = np.where(wh == 0, wl * lo, np.where(wl == 0, wh * hi, t))
            return t.astype(dtype)
        t0 = lerp(r0[..., x0], r0[..., x1], w0, w1)
        t1 = lerp(r1[..., x0], r1[..., x1], w0, w1)
        return lerp(t0, t1, h0[:, None], h1[:, None])


def scale_disp(disp, use_disparity=False):
    """utils.py:216-219 in fp64: disp / 100, or DepthNorm(disp, 1000) / 10000 as torch evaluates it
    (1000 / t is reciprocal(t) * 1000)."""
    d = np.asarray(disp, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (1.0 / d) * 1000.0 / 10000.0 if use_disparity else d / 100.0


def predict(disp, use_224=False, use_disparity=False, skip_zero_weight=False):
    """(n, h, w) disparities -> the reference's ``predictions`` in fp64: (n, 440, 592) Eigen-cropped, or (n, 224, 224).
    Eigen: resize to (224, 304), ReplicationPad2d(8), resize to (480, 640), clamp [0.4, 10], crop."""
    p = scale_disp(disp, use_disparity)
    if not use_224:
        p = resize_ac(p, 224, 304, skip_zero_weight=skip_zero_weight)
        p = np.pad(p, ((0, 0), (8, 8), (8, 8)), mode="edge")
        p = resize_ac(p, 480, 640, skip_zero_weight=skip_zero_weight)
    with np.errstate(invalid="ignore"):
        p = np.where(p < MIN_DEPTH, MIN_DEPTH, p)          # comparisons: NaN stays NaN, as torch.clamp keeps it
        p = np.where(p > MAX_DEPTH, MAX_DEPTH, p)
    if not use_224:
        p = p[:, EIGEN_CROP[0]:EIGEN_CROP[1] + 1, EIGEN_CROP[2]:EIGEN_CROP[3] + 1]
    return np.ascontiguousarray(p)


def prepare_gt(gt, use_224=False):
    """The ground truth the metrics see, float32: the Eigen crop (utils.py:252), or the 16-pixel border crop resized to
    224 x 224 (utils.py:288-291) as torch's float32 CPU kernel computes it."""
    g = np.asarray(gt, np.float32)
    if not use_224:
        return np.ascontiguousarray(g[:, EIGEN_CROP[0]:EIGEN_CROP[1] + 1, EIGEN_CROP[2]:EIGEN_CROP[3] + 1])
    return resize_ac(g[:, BORDER:-BORDER, BORDER:-BORDER], 224, 224, dtype=np.float32)


def frame_sums(pred, gt, gt_log10):
    """Per-frame sums (n, 7) fp64: sum |y - x| / y, sum (y - x)^2, sum |log10 y - log10 x|, the counts of
    max(y / x, x / y) < 1.25^k for k = 1, 2, 3, and the pixel count.  y = gt (float32), x = pred (fp64); log10 y is
    the caller's gt_log10."""
    x = np.asarray(pred, np.float64)
    y = np.asarray(gt, np.float32).astype(np.float64)
    ly = np.asarray(gt_log10, np.float32).astype(np.float64)
    n = x.shape[0]
    x, y, ly = x.reshape(n, -1), y.reshape(n, -1), ly.reshape(n, -1)
    with np.errstate(all="ignore"):
        t = np.maximum(y / x, x / y)                         # NaN-propagating, as torch.max
        d = y - x
        cols = [np.abs(d) / y, d * d, np.abs(ly - np.log10(x))]
        out = np.empty((n, 7), np.float64)
        for j, c in enumerate(cols):
            out[:, j] = [math.fsum(r) if not np.isnan(r).any() else np.nan for r in c]
        for k, c in enumerate(THRESHOLDS):
            out[:, 3 + k] = (t < c).sum(1)
        out[:, 6] = x.shape[1]
    return out


def metrics(sums):
    """compute_errors_nyu's (rel, rms, log_10, a1, a2, a3) from per-frame sums: each column pooled with math.fsum, over
    the pooled pixel count."""
    s = np.atleast_2d(np.asarray(sums, np.float64))
    tot = np.array([math.fsum(s[:, j]) if not np.isnan(s[:, j]).any() else math.nan for j in range(7)])
    with np.errstate(all="ignore"):
        m = tot[:6] / tot[6]
        m[1] = np.sqrt(m[1])
    return m


def frame_metrics(sums):
    """Each frame's own compute_errors_nyu, (n, 6)."""
    return np.stack([metrics(r) for r in np.atleast_2d(sums)])


def compute_errors_nyu(pred, gt):
    """utils.py:85-98 over two equal-size arrays in fp64 (log10 y in fp64 too) -> (6,)."""
    p = np.asarray(pred, np.float64).reshape(1, -1)
    g = np.asarray(gt, np.float64).reshape(1, -1)
    x, y = p, g
    with np.errstate(all="ignore"):
        t = np.maximum(y / x, x / y)
        d = y - x
        cols = [(np.abs(d) / y)[0], (d * d)[0], np.abs(np.log10(y) - np.log10(x))[0]]
    s = [math.fsum(c) if not np.isnan(c).any() else math.nan for c in cols]
    s += [float((t < c).sum()) for c in THRESHOLDS] + [float(x.size)]
    return metrics(np.array(s))


def near_ties(pred, gt, tol):
    """pixels whose max(y / x, x / y) lies within tol (relative) of a 1.25^k threshold"""
    x = np.asarray(pred, np.float64).reshape(-1)
    y = np.asarray(gt, np.float32).astype(np.float64).reshape(-1)
    with np.errstate(all="ignore"):
        t = np.maximum(y / x, x / y)
    return sum(int((np.abs(t - c) <= tol * c).sum()) for c in THRESHOLDS)


# ------------------------------------------------------------------------------------------ synthetic splits
SPECIAL = ("nan_disp", "inf_disp", "zero_disp", "negative_disp", "all_equal", "zero_gt")
ALL_EQUAL_DEPTH = 3.0


def _scene(rng):
    """480 x 640 float32 depth in metres: a smooth field with rectangular objects (depth edges), within [0.7, 9.5]."""
    yy, xx = np.mgrid[0:GT_SHAPE[0], 0:GT_SHAPE[1]].astype(np.float64)
    yy, xx = yy / (GT_SHAPE[0] - 1), xx / (GT_SHAPE[1] - 1)
    a, b, c = rng.uniform(1.5, 4.0), rng.uniform(-1.0, 2.5), rng.uniform(-1.0, 1.0)
    f1, f2 = rng.uniform(1.0, 4.0, 2)
    g = a + b * yy + c * xx + 0.4 * np.sin(2 * np.pi * f1 * xx + 1.3) * np.cos(2 * np.pi * f2 * yy)
    for _ in range(4):
        y0, x0 = rng.integers(0, 400), rng.integers(0, 560)
        g[y0:y0 + rng.integers(40, 200), x0:x0 + rng.integers(40, 240)] += rng.uniform(-1.2, 3.5)
    return np.clip(g, 0.7, 9.5).astype(np.float32)


def _pred_depth(rng, gt, h, w, use_224):
    """a predicted depth field at (h, w): the scene resized, with smooth and per-pixel noise, one region pushed below
    0.4 and one above 10 so that both clamps act."""
    src = gt[BORDER:-BORDER, BORDER:-BORDER] if use_224 else gt
    d = resize_ac(src[None].astype(np.float64), h, w)[0]
    yy, xx = np.mgrid[0:h, 0:w] / np.array([max(h - 1, 1), max(w - 1, 1)])[:, None, None]
    d = d * (1 + 0.12 * np.sin(5.0 * xx + 3.0 * yy)) * rng.uniform(0.88, 1.12, (h, w))
    d[: h // 5, : w // 5] *= 0.15
    d[-(h // 5):, -(w // 5):] *= 4.0
    return d


def synthetic_split(seed, n=3, special=False):
    """Deterministic NYU-like inputs: dict with
      gt:    (n, 480, 640) float32 ground truth;
      disp:  {(h, w, use_disparity): (n, h, w) float32} for DISP_SIZES and (224, 224): depth * 100 without
             use_disparity, 0.1 / depth with it, so both map to the same depth in metres;
      special: {name: frame} when ``special``: one frame per SPECIAL entry (n is then len(SPECIAL))."""
    rng = np.random.default_rng(seed)
    if special:
        n = len(SPECIAL)
    gt = np.stack([_scene(rng) for _ in range(n)])
    disp = {}
    for (h, w) in DISP_SIZES + ((224, 224),):
        depth = np.stack([_pred_depth(rng, gt[i], h, w, (h, w) == (224, 224)) for i in range(n)])
        for use_disparity in (False, True):
            disp[(h, w, use_disparity)] = (0.1 / depth if use_disparity else depth * 100.0).astype(np.float32)
    out = dict(gt=gt, disp=disp)
    if not special:
        return out
    sp = {name: k for k, name in enumerate(SPECIAL)}
    gt[sp["all_equal"]] = np.float32(ALL_EQUAL_DEPTH)
    gt[sp["zero_gt"], 240, 320] = 0.0                       # inside the Eigen crop and the 224-mode region
    for (h, w, use_disparity), d in disp.items():
        # a NaN where the first resize gives it zero weight in one output column (only the 319-wide size has one
        # inside the frame: output column 101 samples column 106 exactly and reads column 107 with weight 0)
        d[sp["nan_disp"], h // 2, 107 if w == 319 else w // 2] = np.nan
        d[sp["inf_disp"], h // 3, w // 3] = np.inf
        d[sp["zero_disp"], h // 4:h // 2, w // 4:w // 2] = 0.0
        d[sp["negative_disp"], h // 2:3 * h // 4, w // 2:3 * w // 4] *= -1.0
        d[sp["all_equal"]] = np.float32(0.1 / ALL_EQUAL_DEPTH if use_disparity else ALL_EQUAL_DEPTH * 100.0)
    out["special"] = sp
    return out


def sample_indices(seed, shape, count=1024):
    """Flat indices into an (n, H, W) prediction: `count` seeded ones, plus the first frame's first and last rows and
    columns."""
    n, H, W = shape
    idx = [np.random.default_rng(seed).choice(n * H * W, count, replace=False), np.arange(W),
           (H - 1) * W + np.arange(W), np.arange(H) * W, np.arange(H) * W + W - 1]
    return np.unique(np.concatenate(idx)).astype(np.int64)
