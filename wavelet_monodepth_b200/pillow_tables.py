"""Pillow's 8-bit resample tables, computed on the host for libwmd's integer-only resample kernels.

``Image.resize`` with a convolution filter runs libImaging/Resample.c: per output pixel the filter's weights are
computed in double (``precompute_coeffs``), normalised by their left-to-right sum and rounded away from zero to 22-bit
fixed point (``normalize_coeffs_8bpc``).  A table here is (out_size, 2 + k) int32 rows of (first tap, taps, k
coefficients).  ``offset`` is added to each row's first tap, so that a kernel can read a cropped image in its uncropped
coordinates.  The weights need libm (``sin`` for LANCZOS), so they are made here with ``math`` and uploaded.

NEAREST is not a convolution in Pillow: ``resize`` runs Geometry.c's affine scale, whose source index is ``int(acc)``
with ``acc`` starting at ``scale / 2`` and ``scale`` added per output pixel, in double.  ``nearest_table`` states it as
a one-tap table of coefficient ``1 << 22``, so it runs through the same kernels.
"""
import math

import numpy as np

PRECISION_BITS = 22


def lanczos(x):
    """Pillow's lanczos_filter (support 3)"""
    def sinc(t):
        if t == 0.0:
            return 1.0
        t = t * math.pi
        return math.sin(t) / t
    return sinc(x) * sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def bicubic(x):
    """Pillow's bicubic_filter (a = -0.5, support 2)"""
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def table(in_size, out_size, filt, support, offset=0):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc of filt for in_size -> out_size: (out_size, 2 + k) int32"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = support * filterscale
    k = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    tab = np.zeros((out_size, 2 + k), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [filt((x + xmin - center + 0.5) * ss) for x in range(n)]
        total = 0.0
        for v in w:
            total += v
        if total != 0.0:
            w = [v / total for v in w]
        tab[xx, 0], tab[xx, 1] = xmin + offset, n
        tab[xx, 2:2 + n] = [int(v * (1 << PRECISION_BITS) + (-0.5 if v < 0 else 0.5)) for v in w]
    return tab


def nearest_table(in_size, out_size, offset=0):
    """Pillow's NEAREST resize as (out_size, 3) int32 one-tap rows (first, 1, 1 << 22)"""
    scale = float(in_size) / out_size
    first = np.empty(out_size, np.int64)
    acc = scale * 0.5
    for xx in range(out_size):
        first[xx] = int(acc)
        acc += scale
    return np.stack([first + offset, np.ones(out_size, np.int64), np.full(out_size, 1 << PRECISION_BITS)],
                    1).astype(np.int32)
