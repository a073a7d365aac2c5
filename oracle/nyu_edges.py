"""numpy/scipy restatement of the NYUv2 depth boundary error (NYUv2/utils.py:122-169 compute_depth_boundary_error, and
its use in add_results / evaluate at :259-271, 303-343), and the synthetic edge maps the fixture uses.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

``canny`` is scikit-image 0.16.2's ``feature.canny`` (skimage/feature/_canny.py of that release, the version the
reference pins in environment.yml) written over the scipy primitives it calls: ``ndi.gaussian_filter``, ``ndi.sobel``,
``np.hypot``, ``binary_erosion``, ``label`` and ``ndi.sum``.  scikit-image itself is not importable here, so this
restatement stands in for it when ``oracle/pin_nyu_edges.py`` runs the unmodified reference, the way ``oracle.haar``
stands in for pytorch_wavelets.

``gaussian_restated``, ``sobel_restated`` and ``hypot_glibc`` spell out the arithmetic of those primitives in the order
scipy and glibc evaluate it; they are the spec the device kernels follow (csrc/eval_edges.cu), and
tests/test_oracle_nyu_edges.py checks them against the primitives bit for bit.
"""
import math

import numpy as np
from scipy import ndimage as ndi

from oracle import nyu_eval as one

SIGMA = math.sqrt(2.0)                     # utils.py:137
LOW, HIGH = 0.15, 0.3                      # compute_depth_boundary_error's defaults
MAX_DIST = 10.0                            # utils.py:144
TRUNCATE = 4.0                             # ndi.gaussian_filter's default
EPS = np.finfo(float).eps                  # smooth_with_function_and_mask's bleed-over guard
CROP_SHAPE = (440, 592)


# ------------------------------------------------------------------------------------------ scikit-image 0.16.2 canny
def _fsmooth(x, sigma):
    """skimage.filters.gaussian(x, sigma, mode='constant') in 0.16.2: img_as_float passes float32 through, so
    ndi.gaussian_filter runs (and stores each pass) in the input's own precision."""
    return ndi.gaussian_filter(x, sigma, mode="constant", cval=0.0, truncate=TRUNCATE)


def canny_parts(image, sigma=SIGMA, low_threshold=LOW, high_threshold=HIGH):
    """The steps of skimage 0.16.2 canny with mask=None -> dict of bleed, smoothed, isobel, jsobel, magnitude,
    local_maxima, low, high, edges.  image: 2-D float32 (dtype_max 1, so the thresholds are used as given)."""
    image = np.asarray(image)
    assert image.ndim == 2 and image.dtype == np.float32
    mask = np.ones(image.shape, dtype=bool)
    bleed = _fsmooth(mask.astype(float), sigma)
    masked = np.zeros(image.shape, image.dtype)
    masked[mask] = image[mask]
    sm = _fsmooth(masked, sigma)
    smoothed = sm / (bleed + EPS)
    jsobel = ndi.sobel(smoothed, axis=1)
    isobel = ndi.sobel(smoothed, axis=0)
    abs_isobel, abs_jsobel = np.abs(isobel), np.abs(jsobel)
    magnitude = np.hypot(isobel, jsobel)
    eroded = ndi.binary_erosion(mask, ndi.generate_binary_structure(2, 2), border_value=0)
    eroded = eroded & (magnitude > 0)
    lm = np.zeros(image.shape, bool)
    with np.errstate(all="ignore"):
        # 0 to 45 degrees
        pts = ((isobel >= 0) & (jsobel >= 0) & (abs_isobel >= abs_jsobel)) | \
              ((isobel <= 0) & (jsobel <= 0) & (abs_isobel >= abs_jsobel))
        pts = eroded & pts
        c1 = magnitude[1:, :][pts[:-1, :]]
        c2 = magnitude[1:, 1:][pts[:-1, :-1]]
        m = magnitude[pts]
        w = abs_jsobel[pts] / abs_isobel[pts]
        c_plus = c2 * w + c1 * (1 - w) <= m
        c1 = magnitude[:-1, :][pts[1:, :]]
        c2 = magnitude[:-1, :-1][pts[1:, 1:]]
        c_minus = c2 * w + c1 * (1 - w) <= m
        lm[pts] = c_plus & c_minus
        # 45 to 90 degrees
        pts = ((isobel >= 0) & (jsobel >= 0) & (abs_isobel <= abs_jsobel)) | \
              ((isobel <= 0) & (jsobel <= 0) & (abs_isobel <= abs_jsobel))
        pts = eroded & pts
        c1 = magnitude[:, 1:][pts[:, :-1]]
        c2 = magnitude[1:, 1:][pts[:-1, :-1]]
        m = magnitude[pts]
        w = abs_isobel[pts] / abs_jsobel[pts]
        c_plus = c2 * w + c1 * (1 - w) <= m
        c1 = magnitude[:, :-1][pts[:, 1:]]
        c2 = magnitude[:-1, :-1][pts[1:, 1:]]
        c_minus = c2 * w + c1 * (1 - w) <= m
        lm[pts] = c_plus & c_minus
        # 90 to 135 degrees
        pts = ((isobel <= 0) & (jsobel >= 0) & (abs_isobel <= abs_jsobel)) | \
              ((isobel >= 0) & (jsobel <= 0) & (abs_isobel <= abs_jsobel))
        pts = eroded & pts
        c1a = magnitude[:, 1:][pts[:, :-1]]
        c2a = magnitude[:-1, 1:][pts[1:, :-1]]
        m = magnitude[pts]
        w = abs_isobel[pts] / abs_jsobel[pts]
        c_plus = c2a * w + c1a * (1.0 - w) <= m
        c1 = magnitude[:, :-1][pts[:, 1:]]
        c2 = magnitude[1:, :-1][pts[:-1, 1:]]
        c_minus = c2 * w + c1 * (1.0 - w) <= m
        lm[pts] = c_plus & c_minus
        # 135 to 180 degrees
        pts = ((isobel <= 0) & (jsobel >= 0) & (abs_isobel >= abs_jsobel)) | \
              ((isobel >= 0) & (jsobel <= 0) & (abs_isobel >= abs_jsobel))
        pts = eroded & pts
        c1 = magnitude[:-1, :][pts[1:, :]]
        c2 = magnitude[:-1, 1:][pts[1:, :-1]]
        m = magnitude[pts]
        w = abs_jsobel[pts] / abs_isobel[pts]
        c_plus = c2 * w + c1 * (1 - w) <= m
        c1 = magnitude[1:, :][pts[:-1, :]]
        c2 = magnitude[1:, :-1][pts[:-1, 1:]]
        c_minus = c2 * w + c1 * (1 - w) <= m
        lm[pts] = c_plus & c_minus
        high = lm & (magnitude >= high_threshold)
        low = lm & (magnitude >= low_threshold)
    labels, count = ndi.label(low, np.ones((3, 3), bool))
    if count == 0:
        edges = low
    else:
        sums = np.array(ndi.sum(high, labels, np.arange(count, dtype=np.int32) + 1), copy=None, ndmin=1)
        good = np.zeros((count + 1,), bool)
        good[1:] = sums > 0
        edges = good[labels]
    return dict(bleed=bleed, smoothed=smoothed, isobel=isobel, jsobel=jsobel, magnitude=magnitude,
                local_maxima=lm, low=low, high=high, edges=edges)


def canny(image, sigma=1.0, low_threshold=None, high_threshold=None, mask=None, use_quantiles=False):
    """``skimage.feature.canny`` as the reference calls it (utils.py:137): float32 image, mask None, given thresholds."""
    assert mask is None and not use_quantiles and low_threshold is not None and high_threshold is not None
    return canny_parts(image, sigma, low_threshold, high_threshold)["edges"]


# ------------------------------------------------------------------------------------------ the device's spec
def gaussian_weights(sigma=SIGMA, truncate=TRUNCATE):
    """scipy's _gaussian_kernel1d(sigma, 0, radius) with radius int(truncate * sigma + 0.5), read back from scipy's
    own filter as the impulse response (so it is scipy's bits by construction) -> w[0..radius]."""
    radius = int(truncate * float(sigma) + 0.5)
    delta = np.zeros(2 * radius + 1)
    delta[radius] = 1.0
    return ndi.gaussian_filter1d(delta, sigma, mode="constant", truncate=truncate)[radius:].copy()


def _gauss_pass(x, w, axis):
    """scipy's symmetric correlate1d, mode constant 0: t = x[i] w0, then t += (x[i-j] + x[i+j]) wj for j = r .. 1,
    in float64, stored in x's dtype"""
    r = len(w) - 1
    a = np.moveaxis(np.asarray(x), axis, 0).astype(np.float64)
    n = a.shape[0]
    p = np.concatenate([np.zeros((r,) + a.shape[1:]), a, np.zeros((r,) + a.shape[1:])])
    with np.errstate(all="ignore"):
        t = a * w[0]
        for j in range(r, 0, -1):
            t = t + (p[r - j:r - j + n] + p[r + j:r + j + n]) * w[j]
    return np.ascontiguousarray(np.moveaxis(t.astype(x.dtype), 0, axis))


def gaussian_restated(x, sigma=SIGMA):
    """ndi.gaussian_filter(x, sigma, mode='constant') of a 2-D float32 or float64 map: axis 0, then axis 1"""
    w = gaussian_weights(sigma)
    return _gauss_pass(_gauss_pass(np.asarray(x), w, 0), w, 1)


def _shift(a, d, axis):
    """a[clamp(i + d)] along axis: scipy's 'reflect' (half-sample symmetric) extension for a radius-1 filter"""
    n = a.shape[axis]
    idx = np.clip(np.arange(n) + d, 0, n - 1)
    return np.take(a, idx, axis=axis)


def sobel_restated(x, axis):
    """ndi.sobel(x, axis) of a 2-D float64 map: t = 0 x + (x[+1] - x[-1]) along `axis`, then t = 2 t + (t[-1] + t[+1])
    along the other axis, both with the 'reflect' extension"""
    x = np.asarray(x, np.float64)
    other = 1 - axis
    with np.errstate(all="ignore"):
        d = 0.0 * x + (_shift(x, 1, axis) - _shift(x, -1, axis))
        return 2.0 * d + (_shift(d, -1, other) + _shift(d, 1, other))


def hypot_glibc(x, y):
    """glibc's e_hypot.c (the non-FMA kernel numpy's np.hypot reaches on x86-64), elementwise in float64"""
    x, y = np.broadcast_arrays(np.asarray(x, np.float64), np.asarray(y, np.float64))
    out = np.empty(x.shape)
    with np.errstate(all="ignore"):
        fin = np.isfinite(x) & np.isfinite(y)
        out[~fin] = np.where(np.isinf(x[~fin]) | np.isinf(y[~fin]), np.inf, x[~fin] + y[~fin])
        ax0, ay0 = np.abs(x[fin]), np.abs(y[fin])
        ax, ay = np.maximum(ax0, ay0), np.minimum(ax0, ay0)
        r = np.empty(ax.shape)
        large, tiny = ax > 2.0 ** 511, ay < 2.0 ** -511
        big_gap = np.where(large, ay <= ax * 2.0 ** -54,
                           np.where(tiny, ax >= ay / 2.0 ** -54, ay <= ax * 2.0 ** -54))
        r[big_gap] = ax[big_gap] + ay[big_gap]
        k = ~big_gap
        sx = np.where(large, 2.0 ** -600, np.where(tiny, 2.0 ** 600, 1.0))[k]
        h = _hypot_kernel(ax[k] * sx, ay[k] * sx)
        r[k] = h / sx
        out[fin] = r
    return out


def _hypot_kernel(ax, ay):
    h = np.sqrt(ax * ax + ay * ay)
    t1, t2 = np.empty(h.shape), np.empty(h.shape)
    c = h <= 2.0 * ay
    delta = h - ay
    t1[c] = (ax * (2.0 * delta - ax))[c]
    t2[c] = ((delta - 2.0 * (ax - ay)) * delta)[c]
    delta = h - ax
    t1[~c] = (2.0 * delta * (ax - 2.0 * ay))[~c]
    t2[~c] = ((4.0 * delta - ay) * ay + delta * delta)[~c]
    return h - (t1 + t2) / (2.0 * h)


# ------------------------------------------------------------------------------------------ depth boundary error
def normalise(pred):
    """utils.py:131-134 in float32: zeros to NaN, minus nanmin, over nanmax"""
    p = np.array(pred, dtype="f")
    p[p == 0] = np.nan
    with np.errstate(all="ignore"), _quiet():
        p = p - np.nanmin(p)
        p = p / np.nanmax(p)
    return p


class _quiet:
    """silences numpy's all-NaN RuntimeWarning (nanmin of an all-NaN map is NaN, as the reference gets)"""

    def __enter__(self):
        import warnings
        self._w = warnings.catch_warnings()
        self._w.__enter__()
        warnings.simplefilter("ignore", RuntimeWarning)

    def __exit__(self, *a):
        self._w.__exit__(*a)


def edges_est(pred, low=LOW, high=HIGH):
    """the prediction's Canny edges (utils.py:131-138), bool"""
    return canny(normalise(pred), sigma=SIGMA, low_threshold=low, high_threshold=high)


def edt(features):
    """ndi.distance_transform_edt(1 - features): the Euclidean distance of each pixel to the nearest feature pixel"""
    return ndi.distance_transform_edt(1 - np.asarray(features).astype(np.int64))


def gt_features(edges_gt):
    """the feature pixels of 1 - edges_gt: those exactly 1.0 (grey levels are not features)"""
    return np.asarray(edges_gt) == 1


def no_feature_edt(H, W):
    """what scipy returns for a map with no feature pixel: sqrt((i + 1)^2 + j^2)"""
    i, j = np.mgrid[0:H, 0:W]
    return np.sqrt(((i + 1) ** 2 + j ** 2).astype(np.float64))


def dbe(edges_gt, pred, low=LOW, high=HIGH):
    """compute_depth_boundary_error as the device computes it, for one frame -> (acc, comp, edges_est, D_est).
    An all-zero edges_gt gives NaN scores (the reference means that, but raises UnboundLocalError on its
    ``return ... D_est``); edges_est and D_est are still the prediction's."""
    g = np.asarray(edges_gt, np.float32)
    e = edges_est(pred, low, high)
    d_est = edt(e)
    if np.sum(g) == 0:
        return math.nan, math.nan, e, d_est
    d_gt = edt(gt_features(g))
    near = e & (d_gt < MAX_DIST)
    if not near.any():
        return MAX_DIST, MAX_DIST, e, d_est
    acc = math.fsum(d_gt[near]) / near.sum()
    with np.errstate(all="ignore"):
        num = math.fsum(np.minimum(d_gt[e], MAX_DIST)) + math.fsum(np.minimum(d_est * g.astype(np.float64), MAX_DIST)
                                                                   .ravel())
    comp = num / (float(e.sum()) + float(np.nansum(g)))
    return acc, comp, e, d_est


def dbe_numpy(edges_gt, pred, low=LOW, high=HIGH):
    """compute_depth_boundary_error with the reference's own numpy reductions (np.nansum, pairwise), so its scores
    equal the reference's bit for bit; ``dbe`` is the device's contract, with exact fsum sums"""
    g = np.asarray(edges_gt, np.float32)
    e = edges_est(pred, low, high)
    d_est = edt(e)
    if np.sum(g) == 0:
        return math.nan, math.nan, e, d_est
    d_gt = edt(gt_features(g))
    near = (e * (d_gt < MAX_DIST)) * np.ones(e.shape)
    if np.sum(near) == 0:
        return MAX_DIST, MAX_DIST, e, d_est
    acc = np.nansum(d_gt * near) / np.nansum(near)
    ch1 = d_gt * e
    ch1[ch1 > MAX_DIST] = MAX_DIST
    ch2 = d_est * g
    ch2[ch2 > MAX_DIST] = MAX_DIST
    comp = np.nansum(ch1 + ch2) / (np.nansum(e) + np.nansum(g))
    return float(acc), float(comp), e, d_est


# ------------------------------------------------------------------------------------------ synthetic edge maps
def step_edges(depth, step=0.25):
    """a binary OC-style edge map of a depth map: pixels whose right or lower neighbour differs by more than `step`"""
    d = np.asarray(depth, np.float64)
    e = np.zeros(d.shape, bool)
    e[:, :-1] |= np.abs(d[:, 1:] - d[:, :-1]) > step
    e[:-1, :] |= np.abs(d[1:, :] - d[:-1, :]) > step
    return e


def as_k255(k):
    """evaluate.py:73-75: float32(k / 255), k the PNG's uint8 value (the division in float64, stored in float32)"""
    return (np.asarray(k, np.uint8).astype(np.float64) / 255.0).astype(np.float32)


def spiral_mask(H, W, band=6, gap=6):
    """a square spiral band `band` pixels wide with `gap` pixels between its turns, wound inwards from the border ->
    (bool (H, W) band, bool (H, W) its last straight piece, at the centre)"""
    m = np.zeros((H, W), bool)
    last = np.zeros((H, W), bool)
    pitch = band + gap
    t, l, b, r, lstart = 0, 0, H, W, 0
    while b - t >= 2 * pitch and r - l >= 2 * pitch:
        m[t:t + band, lstart:r] = True                 # top, rightwards (joining the previous turn's left side)
        m[t:b, r - band:r] = True                      # right, downwards
        m[b - band:b, l:r] = True                      # bottom, leftwards
        m[t + pitch:b, l:l + band] = True              # left, upwards
        last[:] = False
        last[t + pitch:b, l:l + band] = True
        lstart = l
        t, l, b, r = t + pitch, l + pitch, b - pitch, r - pitch
    return m, last


EDGE_SPECIAL = ("grey", "grey_only", "edge_free", "constant", "nan_disp", "spiral")
DISP_SIZE = (240, 320)
SPIRAL_DEPTHS = (2.0, 2.35, 2.75, 4.5)     # background, band, the band's inner end, a blob setting the range (metres)


def edge_split(seed, n=3, special=False):
    """Deterministic NYU-like inputs with edge maps: dict with gt (n, 480, 640) float32 depth, disp (n, 240, 320)
    float32 (depth * 100), edges (n, 480, 640) float32 k / 255, and with ``special`` the frame index of each
    EDGE_SPECIAL case.  Edge maps mark the scene's depth steps: binary in a plain split; in the special split grey
    levels k in 60..255 ("grey"), 60..254 ("grey_only": no feature pixel), none ("edge_free"), binary elsewhere.
    The special cases: a constant prediction (Canny finds nothing), a NaN disparity, and a prediction whose edges are
    one long single-pixel spiral of low-threshold pixels with high ones only at its inner end (the hysteresis worst
    case)."""
    if special:
        n = len(EDGE_SPECIAL)
    split = one.synthetic_split(seed, n=n)
    gt, disp = split["gt"], split["disp"][DISP_SIZE + (False,)].copy()
    rng = np.random.default_rng(1000 + seed)
    edges = np.stack([step_edges(g) for g in gt]).astype(np.float32)
    out = dict(gt=gt, disp=disp, edges=edges)
    if not special:
        return out
    sp = {name: k for k, name in enumerate(EDGE_SPECIAL)}
    e = edges[sp["grey"]] > 0
    edges[sp["grey"]] = np.where(e, as_k255(rng.integers(60, 256, e.shape)), 0)
    e = edges[sp["grey_only"]] > 0
    edges[sp["grey_only"]] = np.where(e, as_k255(rng.integers(60, 255, e.shape)), 0)
    edges[sp["edge_free"]] = 0
    disp[sp["constant"]] = np.float32(300.0)
    disp[sp["nan_disp"], 120, 160] = np.nan
    disp[sp["spiral"]] = spiral_disp(*DISP_SIZE)
    out["special"] = sp
    return out


def spiral_disp(H, W):
    """(H, W) float32 disparity of the spiral case: the band 0.35 m in front of a 2 m background, a step that Canny
    finds between the two thresholds; along the band's last piece the step grows to 0.75 m, so only the spiral's inner
    end passes the high threshold and every other edge pixel is kept by hysteresis alone.  A small 4.5 m blob where the
    background is farthest from the band fixes the normalisation range."""
    band, last = spiral_mask(H, W)
    depth = np.where(band, SPIRAL_DEPTHS[1], SPIRAL_DEPTHS[0])
    rows = np.nonzero(last.any(1))[0]
    ramp = np.clip((rows.max() - np.arange(H)) / max(len(rows) - 1, 1), 0, 1)[:, None]     # 0 at the bottom, 1 top
    depth = np.where(last, SPIRAL_DEPTHS[1] + (SPIRAL_DEPTHS[2] - SPIRAL_DEPTHS[1]) * ramp, depth)
    y, x = np.unravel_index(np.argmax(ndi.distance_transform_edt(~band)), band.shape)
    depth[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2] = SPIRAL_DEPTHS[3]
    return (depth * 100.0).astype(np.float32)
