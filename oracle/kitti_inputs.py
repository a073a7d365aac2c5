"""numpy restatement of KITTI's training inputs (``KITTI/datasets/mono_dataset.py`` ``__getitem__`` / ``preprocess``
with ``kitti_dataset.KITTIRAWDataset``), every step at Pillow's and torchvision's rounding points.

- Resize: Pillow's 8-bit two-pass LANCZOS resample (``Image.resize(..., LANCZOS)``, libImaging/Resample.c).  Per
  output pixel the Lanczos-3 weights are computed in double with libm ``sin`` (``math.sin``), normalised by their sum,
  rounded away from zero to 22-bit fixed point; each pass accumulates in int from ``1 << 21`` and keeps
  ``clip(acc >> 22, 0, 255)``.  Horizontal pass first, uint8 between the passes.  An unchanged extent is a copy.
- ``ImageEnhance`` blends (libImaging/Blend.c): ``in1 + alpha * (in2 - in1)`` in float32 with alpha = float32(factor),
  truncated and clipped to [0, 255].  Brightness blends from black, contrast from ``int(mean(L) + 0.5)`` of the image
  as it is at that point of the order (an exact integer sum divided in double), saturation from the image's own L.
- RGB -> L: ``(19595 R + 38470 G + 7471 B + 0x8000) >> 16``.
- RGB <-> HSV: libImaging/Convert.c's ``rgb2hsv`` / ``hsv2rgb``, whose float and double sub-expressions are kept
  apart here exactly as C's promotion rules keep them.
- Hue: the HSV hue byte plus ``uint8(trunc(h * 255))`` modulo 256, then back to RGB.
- ToTensor: uint8 / 255 in float32.
"""
import math
import random

import numpy as np

PRECISION_BITS = 22
LANCZOS_SUPPORT = 3.0
OPS = ("brightness", "contrast", "saturation", "hue")
JITTER_RANGES = ((0.8, 1.2), (0.8, 1.2), (0.8, 1.2), (-0.1, 0.1))
MIN_DEPTH, MAX_DEPTH = 0.1, 100.0
KITTI_K = np.array([[0.58, 0, 0.5, 0], [0, 1.92, 0.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float32)


# --------------------------------------------------------------------------------------------------------- resample
def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    if -3.0 <= x < 3.0:
        return _sinc(x) * _sinc(x / 3)
    return 0.0


def lanczos_table(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for LANCZOS: (bounds (out, 2) int32 of (first tap, taps),
    coeffs (out, ksize) int32).  An unchanged extent gives the identity (Pillow copies the image)."""
    if in_size == out_size:
        bounds = np.stack([np.arange(out_size), np.ones(out_size, np.int64)], 1).astype(np.int32)
        return bounds, np.full((out_size, 1), 1 << PRECISION_BITS, np.int32)
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = LANCZOS_SUPPORT * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    coeffs = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:                                   # C's left-to-right double sum
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        for x, w in enumerate(k):
            coeffs[xx, x] = int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, coeffs


def _pass(img, table, axis):
    """one 8-bit pass along `axis` (1 horizontal, 0 vertical) of an (H, W, C) uint8 image"""
    bounds, coeffs = table
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((len(bounds),) + src.shape[1:], np.uint8)
    for o, (lo, n) in enumerate(bounds):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        acc += np.tensordot(coeffs[o, :n].astype(np.int64), src[lo:lo + n], axes=(0, 0))
        out[o] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def resize(img, width, height):
    """Image.fromarray(img).resize((width, height), LANCZOS) of an (H, W, 3) uint8 array"""
    h, w = img.shape[:2]
    if w != width:
        img = _pass(img, lanczos_table(w, width), 1)
    if h != height:
        img = _pass(img, lanczos_table(h, height), 0)
    return np.ascontiguousarray(img)


def pyramid(view, height, width, scales, flip):
    """the reference's chain: flip the decoded view, then each listed scale resized from the one before it"""
    img = view[:, ::-1] if flip else view
    out = {}
    for s in scales:
        img = resize(img, width >> s, height >> s)
        out[s] = img
    return out


# ------------------------------------------------------------------------------------------------------ colour ops
def rgb_to_l(img):
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    return ((19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16).astype(np.uint8)


def rgb_to_hsv(img):
    f32, f64 = np.float32, np.float64
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    maxc = np.maximum(r, np.maximum(g, b))
    minc = np.minimum(r, np.minimum(g, b))
    same = maxc == minc
    with np.errstate(divide="ignore", invalid="ignore"):
        cr = (maxc - minc).astype(f32)
        s = cr / maxc.astype(f32)
        rc = (maxc - r).astype(f32) / cr
        gc = (maxc - g).astype(f32) / cr
        bc = (maxc - b).astype(f32) / cr
        h = np.where(r == maxc, (bc - gc).astype(f64),
                     np.where(g == maxc, (2.0 + rc.astype(f64)) - bc.astype(f64),
                              (4.0 + gc.astype(f64)) - rc.astype(f64))).astype(f32)
        h = np.fmod(h.astype(f64) / 6.0 + 1.0, 1.0).astype(f32)
        uh = np.clip(np.trunc(h.astype(f64) * 255.0), 0, 255)
        us = np.clip(np.trunc(s.astype(f64) * 255.0), 0, 255)
    uh = np.where(same, 0, uh).astype(np.uint8)
    us = np.where(same, 0, us).astype(np.uint8)
    return np.stack([uh, us, maxc.astype(np.uint8)], -1)


def _c_round(x):
    """C round(): half away from zero (x >= 0 here)"""
    fl = np.floor(x)
    return fl + (x - fl >= 0.5)


def hsv_to_rgb(hsv):
    f32, f64 = np.float32, np.float64
    h, s, v = (hsv[..., c].astype(np.int64) for c in range(3))
    hf = h.astype(f32).astype(f64) * 6.0 / 255.0
    i = np.floor(hf).astype(np.int64)
    f = (hf - i.astype(f32).astype(f64)).astype(f32)
    fs = (s.astype(f32).astype(f64) / 255.0).astype(f32)
    vd = v.astype(f32).astype(f64)
    p = np.clip(_c_round(vd * (1.0 - fs.astype(f64))), 0, 255).astype(np.uint8)
    q = np.clip(_c_round(vd * (1.0 - (fs * f).astype(f64))), 0, 255).astype(np.uint8)
    t = np.clip(_c_round(vd * (1.0 - fs.astype(f64) * (1.0 - f.astype(f64)))), 0, 255).astype(np.uint8)
    v8 = v.astype(np.uint8)
    sel = (i % 6)[..., None]
    cases = [np.stack(c, -1) for c in ((v8, t, p), (q, v8, p), (p, v8, t), (p, q, v8), (t, p, v8), (v8, p, q))]
    out = np.choose(np.broadcast_to(sel, cases[0].shape), cases)
    return np.where((s == 0)[..., None], np.stack([v8] * 3, -1), out).astype(np.uint8)


def blend(in1, in2, factor):
    """Image.blend(in1, in2, factor) on uint8 arrays"""
    alpha = np.float32(factor)
    a = np.asarray(in1).astype(np.float32)
    t = a + alpha * (np.asarray(in2).astype(np.float32) - a)
    return np.clip(np.trunc(t), 0, 255).astype(np.uint8)


def contrast_mean(img):
    """int(ImageStat.Stat(img.convert('L')).mean[0] + 0.5)"""
    lum = rgb_to_l(img)
    return int(int(lum.astype(np.int64).sum()) / lum.size + 0.5)


def hue_shift(hue_factor):
    """the byte torchvision adds to the HSV hue: uint8(trunc(h * 255)) modulo 256"""
    return math.trunc(hue_factor * 255) % 256


def adjust(img, op, factor):
    if op == 0:
        return blend(np.zeros_like(img), img, factor)
    if op == 1:
        return blend(np.uint8(contrast_mean(img)), img, factor)
    if op == 2:
        return blend(np.repeat(rgb_to_l(img)[..., None], 3, -1), img, factor)
    hsv = rgb_to_hsv(img)
    hsv[..., 0] = (hsv[..., 0].astype(np.int64) + hue_shift(factor)) % 256
    return hsv_to_rgb(hsv)


def jitter(img, params):
    """the reference's ColorJitter Compose: params = (factors (b, c, s, h), order), or None for no augmentation"""
    if params is None:
        return img
    factors, order = params
    for op in order:
        img = adjust(img, op, factors[op])
    return img


def to_tensor(img):
    """T.ToTensor(): (3, H, W) float32, uint8 / 255"""
    return np.ascontiguousarray(img.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)


# ------------------------------------------------------------------------------------------------------ the draws
def get_params(rng=random):
    """torchvision 0.8.2's ColorJitter.get_params(brightness, contrast, saturation, hue) with the reference's ranges:
    uniform draws for b, c, s, h in that order, then a shuffle of the four transforms.  Returns (factors, order)."""
    factors = tuple(rng.uniform(lo, hi) for lo, hi in JITTER_RANGES)
    order = [0, 1, 2, 3]
    rng.shuffle(order)
    return factors, tuple(order)


def draws(is_train, rng=random):
    """__getitem__'s draws in its order: (do_color_aug, do_flip, jitter params or None)"""
    do_color_aug = is_train and rng.random() > 0.5
    do_flip = is_train and rng.random() > 0.5
    return do_color_aug, do_flip, (get_params(rng) if do_color_aug else None)


# ------------------------------------------------------------------------------------------ cameras and depth hints
def cameras(height, width, scales):
    """{("K", s), ("inv_K", s)} exactly as __getitem__ forms them"""
    out = {}
    for s in scales:
        K = KITTI_K.copy()
        K[0, :] *= width // (2 ** s)
        K[1, :] *= height // (2 ** s)
        out[("K", s)] = K
        out[("inv_K", s)] = np.linalg.pinv(K)
    return out


def stereo_T(side, flip):
    T = np.eye(4, dtype=np.float32)
    T[0, 3] = (-1 if side == "l" else 1) * (-1 if flip else 1) * 0.1
    return T


def nearest_index(in_size, out_size):
    """cv2.resize INTER_NEAREST's source index per output index: min(floor(x * in / out), in - 1)"""
    scale = 1.0 / (out_size / in_size)
    return np.minimum(np.floor(np.arange(out_size) * scale).astype(np.int64), in_size - 1)


def depth_to_disp(depth):
    """KITTI/layers.py depth_to_disp(depth, 0.1, 100) on float32"""
    min_disp, max_disp = 1 / MAX_DEPTH, 1 / MIN_DEPTH
    disp = 1 / (depth + 1e-5)
    disp = (disp - min_disp) / (max_disp - min_disp)
    disp[depth <= 0] = 0
    disp[disp <= 0] = 0
    return disp


def hints(depth, flip, height, width):
    """(depth_hint, disp_hint, depth_hint_mask), each (1, H, W) float32, from the raw (h, w) hint or None (missing)"""
    if depth is None:
        z = np.zeros((1, height, width), np.float32)
        return z, z, z
    if flip:
        depth = depth[:, ::-1]
    d = depth[nearest_index(depth.shape[0], height)][:, nearest_index(depth.shape[1], width)]
    disp = depth_to_disp(d)
    return d[None].astype(np.float32), disp[None].astype(np.float32), (d > 0)[None].astype(np.float32)


def item(views, height, width, scales, flip, params):
    """{("color", f, s), ("color_aug", f, s)} (3, H >> s, W >> s) float32 of one item's decoded uint8 views {f: view}"""
    out = {}
    for f, view in views.items():
        for s, img in pyramid(view, height, width, scales, flip).items():
            out[("color", f, s)] = to_tensor(img)
            out[("color_aug", f, s)] = to_tensor(jitter(img, params))
    return out


def expected(views, draws, side, hint, height, width, scales, use_depth_hints):
    """the reference __getitem__'s dict (numpy, minus image_path) of one item: views {frame: decoded uint8 view},
    draws (do_color_aug, do_flip, params), hint the raw (h, w) hint, or None when its file is missing"""
    do_color_aug, do_flip, params = draws
    out = item(views, height, width, scales, do_flip, params if do_color_aug else None)
    out.update(cameras(height, width, scales))
    if "s" in views:
        out["stereo_T"] = stereo_T(side, do_flip)
        if use_depth_hints:
            d, disp, mask = hints(hint, do_flip, height, width)
            out.update(depth_hint=d, depth_hint_mask=mask)
            if hint is not None:
                out["disp_hint"] = disp
    return out


# -------------------------------------------------------------------------------------------------- synthetic data
RAW_SIZES = ((375, 1242), (376, 1241), (374, 1238), (370, 1226), (370, 1224))     # (H, W) of KITTI raw recordings


def synthetic_view(seed, h, w):
    """a seeded (h, w, 3) uint8 view: coloured gradients, noise, clipped highlights and shadows, and grey bands (where
    the HSV round trip takes its saturation-0 branch)"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    phase = rng.uniform(0, 2 * np.pi, 3)
    img = np.stack([128 + 150 * np.sin(x / (23 + 7 * c) + phase[c]) * np.cos(y / (17 + 5 * c)) for c in range(3)], -1)
    img += rng.integers(-40, 41, (h, w, 3))
    img = np.clip(img, 0, 255).astype(np.uint8)
    grey = (np.arange(h) % 29) < 4
    img[grey] = img[grey].mean(-1, keepdims=True).astype(np.uint8)
    return img


def synthetic_hint(seed, h, w):
    """a seeded (h, w) float32 depth hint in [0, 80) with zeros and a few negative values"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(-2, 80, (h, w)).astype(np.float32)
    d[rng.random((h, w)) < 0.1] = 0
    return d
