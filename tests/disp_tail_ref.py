"""fp64 reference of the fused baseline tail (wmd_disp_tail16_f32, include/wmd.h), built on conv_ref.

    u    = ELU(b1 + conv3x3(up2(x); W1))     zero padding at full resolution (the gather's shift0 = 1 source)
    disp = sigmoid(b2 + conv3x3(u; W2))      reflection padding

Returns (disp64 (N, cout, 2H, 2W), S) with S the error scale carried through both stages: S = S2 + sum |W2| S1, where
S1 = |b1| + sum |x w1| is the scale of each u element and S2 = |b2| + sum |u w2| that of the second stage's own sums.  An
fp32-faithful kernel's error is a small multiple of 2^-22 S whatever the signs of the operands (ELU and the sigmoid have
slopes <= 1, so an error in u reaches disp at most through |W2|).
"""
import torch

import conv_ref as cr

BAR = 3e-8          # err / S: ~3x the worst measured on an H100 (1.09e-8, mixed signs at 48x160; tests/test_gpu_disp_tail.py)


def disp_tail_ref(x_rows, w1, b1, w2, b2, n, h, w, floor=False):
    """x_rows: (N*h*w, ld >= 16) half-resolution rows; weights (16,16,3,3), (16,), (cout,16,3,3), (cout,).

    floor: also return F of the bound BAR S + F: the tf32x3 floor of the first stage (conv_ref.tf32_floor, plus 2^-149
    for ELU's rounding) carried through |W2|, plus the FMA floor of the second (conv_ref.fma_floor, every u counted as
    nonzero)."""
    h2, w2_ = 2 * h, 2 * w
    cout = int(w2.shape[0])
    u, s1, *f1 = cr.conv_ref(x_rows, 16, w1, b1, n, h2, w2_, pad=cr.PAD_ZERO, act=cr.ACT_ELU, shift0=1,
                             floor="tf32x3" if floor else None)
    z, s2 = cr.conv_ref(u, 16, w2, b2, n, h2, w2_, pad=cr.PAD_REFLECT, act=cr.ACT_SIGMOID)
    carried, _ = cr.conv_ref(s1, 16, w2.abs(), None, n, h2, w2_, pad=cr.PAD_REFLECT)

    def nchw(rows):
        return rows.reshape(n, h2, w2_, cout).permute(0, 3, 1, 2)
    if not floor:
        return nchw(z), nchw(s2 + carried)
    f1 = f1[0] + 2.0 ** -149
    fc, _ = cr.conv_ref(f1, 16, w2.abs(), None, n, h2, w2_, pad=cr.PAD_REFLECT)
    f2 = cr.FMA_FLOOR * (144 + 8)
    return nchw(z), nchw(s2 + carried), nchw(fc + f2)
