"""numpy restatement of NYUv2's training inputs (``NYUv2/data.py``: ``depthDatasetMemory`` with
``getDefaultTrainTransform`` or ``getNoTransform``), every step at Pillow's and torchvision's rounding points.

- Draws (Python's ``random``, in this order): ``random() < 0.5`` flips; ``random() < 0.1`` swaps, and only then
  ``randint(0, 5)`` picks one of ``permutations(range(3))``; ``uniform(1 / 0.8, 0.8)`` is the gamma, always drawn.
  The testing transform draws nothing.
- Flip: both images mirrored over their full 640 columns.  Swap: output channel c is input channel perm[c].
- Gamma: torchvision's ``adjust_gamma``, Pillow's ``point`` with ``int((255 + 1 - 1e-3) * 1 * pow(v / 255, gamma))``,
  the same table for the three channels.
- Crop ``(16, 16, 624, 464)``, then ``resize`` to (640, 480) / (320, 240), or (224, 224) for both with ``is_224``:
  BICUBIC is Pillow's 8-bit two-pass resample (horizontal first, uint8 between the passes, 22-bit coefficients rounded
  away from zero, each pass from ``1 << 21``, ``clip(acc >> 22, 0, 255)``) with a = -0.5 and support 2 widened by the
  scale; NEAREST is Geometry.c's affine scale, source index ``int(acc)`` from ``acc = scale / 2`` in steps of
  ``scale``, in double.
- ToTensor: the image ``u / 255`` in float32; the depth ``(u / 255) * 1000`` in float32, clamped to [10, 1000].
"""
import itertools
import math

import numpy as np

from oracle.kitti_inputs import PRECISION_BITS, _pass

CROP = 16
PERMS = list(itertools.permutations(range(3), 3))


# --------------------------------------------------------------------------------------------------------- resample
def _bicubic(x):
    x = abs(x)
    if x < 1.0:
        return ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * -0.5
    return 0.0


def bicubic_table(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for BICUBIC: (bounds (out, 2) of (first, taps), coeffs)"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    coeffs = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        for x, w in enumerate(k):
            coeffs[xx, x] = int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, coeffs


def nearest_index(in_size, out_size):
    """Geometry.c's affine-scale source index per output index"""
    a = float(in_size) / out_size
    idx, acc = [], a * 0.5
    for _ in range(out_size):
        idx.append(int(acc))
        acc += a
    return np.array(idx, np.int64)


def resize(img, width, height, resample):
    """Image.fromarray(img).resize((width, height), BICUBIC or NEAREST) of an (H, W, 3) or (H, W) uint8 array"""
    h, w = img.shape[:2]
    if resample == "nearest":
        return np.ascontiguousarray(img[nearest_index(h, height)][:, nearest_index(w, width)])
    img = _pass(img, bicubic_table(w, width), 1)
    return np.ascontiguousarray(_pass(img, bicubic_table(h, height), 0))


# ------------------------------------------------------------------------------------------------------ the chain
def gamma_lut(gamma):
    if gamma is None:
        return np.arange(256, dtype=np.uint8)
    return np.array([int((255 + 1 - 1e-3) * 1 * math.pow(v / 255.0, gamma)) for v in range(256)], np.uint8)


def sizes(is_224):
    """((image w, h), (depth w, h)) of ToTensor's resizes"""
    return ((224, 224), (224, 224)) if is_224 else ((640, 480), (320, 240))


def expected(image, depth, flip, perm, gamma, is_224, resample="bicubic"):
    """the reference transform's {"image": (3, H, W), "depth": (1, h, w)} float32 of one decoded item; perm an index
    into PERMS or -1, gamma None for no gamma"""
    if flip:
        image, depth = image[:, ::-1], depth[:, ::-1]
    if perm >= 0:
        image = image[..., list(PERMS[perm])]
    image = gamma_lut(gamma)[image]
    image = image[CROP:-CROP, CROP:-CROP]
    depth = depth[CROP:-CROP, CROP:-CROP]
    (iw, ih), (dw, dh) = sizes(is_224)
    image = resize(image, iw, ih, resample)
    depth = resize(depth, dw, dh, resample)
    img = np.ascontiguousarray(image.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)
    d = (depth[None].astype(np.float32) / np.float32(255)) * np.float32(1000)
    return {"image": img, "depth": np.clip(d, np.float32(10), np.float32(1000))}


def draws(is_train, rng):
    """the training transform's draws in its order: (flip, perm index or -1, gamma); none for the testing one"""
    if not is_train:
        return False, -1, None
    flip = rng.random() < 0.5
    perm = rng.randint(0, 5) if rng.random() < 0.1 else -1
    return flip, perm, rng.uniform(1 / 0.8, 0.8)


# -------------------------------------------------------------------------------------------------- synthetic data
def synthetic_image(seed):
    """a seeded (480, 640, 3) uint8 RGB view: coloured gradients, noise, clipped highlights and shadows, and channels
    that differ, so that every permutation moves values"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:480, 0:640].astype(np.float64)
    phase = rng.uniform(0, 2 * np.pi, 3)
    img = np.stack([128 + 160 * np.sin(x / (19 + 9 * c) + phase[c]) * np.cos(y / (13 + 6 * c)) + 40 * (c - 1)
                    for c in range(3)], -1)
    img += rng.integers(-30, 31, (480, 640, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def synthetic_depth(seed):
    """a seeded (480, 640) uint8 depth: a slanted plane with steps and noise, reaching 0 .. 2 (clamped to 10 by the
    reference) and 255"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:480, 0:640].astype(np.float64)
    d = 20 + 0.3 * x + 0.2 * y + 30 * ((x // 80 + y // 60) % 3) + rng.normal(0, 4, (480, 640))
    d[rng.random((480, 640)) < 0.03] = 0
    d[:40, 500:] = 300
    d[440:, :90] = rng.integers(0, 3, (40, 90))
    return np.clip(d, 0, 255).astype(np.uint8)
