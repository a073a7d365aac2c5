"""fp64 adjoint of the gather-GEMM convolution contract: torch autograd through tests/conv_ref.py.

For the linear part z = A W + b of a dense layer (A the implicit im2col rows gathered by conv_ref.gather_rows) and a given
pre-activation gradient dz, returns the fp64 gradients of x0, x1 (rows), W and b, and the per-element scale S of each,
the magnitude sum of the element's terms: the same adjoint applied to |x0|, |x1|, |W| and |dz| (for dW: |A|^T |dz|).
Work is cut into row blocks; it runs on whatever device the inputs live on.
"""
import torch

import conv_ref

_f64 = torch.float64

# err / S bars of the backward kernels (measurements: tests/test_gpu_native_training.py)
BARS = {"dW": 2.5e-6, "db": 3e-6, "dx0": 2e-5, "dx1": 1e-5}


def _adjoint(x0, c0, x1, c1, weight, dz, n, h, w, taps, pad, shift0, block_rows):
    x0 = x0.detach().to(_f64).requires_grad_(True)
    x1 = x1.detach().to(_f64).requires_grad_(True) if x1 is not None else None
    cout = weight.shape[0]
    wk = weight.detach().to(_f64).requires_grad_(True)
    wm = wk.permute(2, 3, 1, 0).reshape(-1, cout)
    rows = n * h * w
    for r in range(0, rows, block_rows):
        m = torch.arange(r, min(rows, r + block_rows), device=dz.device)
        a = conv_ref.gather_rows(m, x0, c0, n, h, w, taps, pad, shift0=shift0, x1=x1, c1=c1).reshape(len(m), -1)
        (a @ wm).backward(dz[r:r + len(m)].to(_f64))
    return x0.grad, (x1.grad if x1 is not None else None), wk.grad


def conv_grads(x0, c0, x1, c1, weight, dz, n, h, w, taps=9, pad=conv_ref.PAD_REFLECT, shift0=0, block_elems=1 << 24):
    """dict name -> (fp64 gradient, S) for 'x0', 'x1' (rows; None without x1), 'w' (weight layout) and 'b'."""
    block_rows = max(1, block_elems // max(taps * (c0 + c1), 1))
    g = _adjoint(x0, c0, x1, c1, weight, dz, n, h, w, taps, pad, shift0, block_rows)
    s = _adjoint(x0.abs(), c0, x1.abs() if x1 is not None else None, c1, weight.abs(), dz.abs(), n, h, w, taps, pad,
                 shift0, block_rows)
    dz64 = dz.to(_f64)
    out = {"x0": (g[0], s[0]), "w": (g[2], s[2]), "b": (dz64.sum(0), dz64.abs().sum(0))}
    out["x1"] = (g[1], s[1]) if x1 is not None else None
    return out


def wgrad_floor(x0, c0, x1, c1, weight, dz, n, h, w, taps=9, pad=conv_ref.PAD_REFLECT, shift0=0, block_elems=1 << 24):
    """F of the tf32x3 weight gradient's bound BAR S + F, per element of dW (weight layout): A and dz are both split to
    nearest into tf32 hi + lo (conv_bwd.cu), so conv_ref.tf32_floor applies with A in the role of x and dz in that of
    w - 2^-126 (sum |dz| over A != 0 + sum |A| over dz != 0 + 6 K') - plus 2^-149 for each 32-pixel chunk's
    round-to-nearest add and each partial slab (at most rows / 32 + 8 of them)."""
    block_rows = max(1, block_elems // max(taps * (c0 + c1), 1))
    nz = lambda t: (t != 0).to(_f64) if t is not None else None      # noqa: E731
    ab = lambda t: t.abs() if t is not None else None                # noqa: E731
    a = _adjoint(nz(x0), c0, nz(x1), c1, weight, dz.abs(), n, h, w, taps, pad, shift0, block_rows)[2]
    b = _adjoint(ab(x0), c0, ab(x1), c1, weight, nz(dz), n, h, w, taps, pad, shift0, block_rows)[2]
    k = _adjoint(nz(x0), c0, nz(x1), c1, weight, nz(dz), n, h, w, taps, pad, shift0, block_rows)[2]
    return conv_ref.TF32_FLOOR * (a + b + 6 * k) + conv_ref.FMA_FLOOR * (n * h * w / 32 + 24)


def act_bwd_floor(dy, rows_summed=None):
    """F of act_backward's dz = dy act'(y), per element: |dz - exact| <= 4 x 2^-24 |exact| + F, F = 2^-149 (1 + |dy|) for
    the two roundings (act'(y) = y (1 - y) and the product) that may land among the subnormals.  rows_summed: also the
    floor of db = sum over rows of dz, the rows' F plus 2^-149 per add of the fixed-order sum."""
    f = conv_ref.FMA_FLOOR * (1 + dy.to(_f64).abs())
    if rows_summed is None:
        return f
    return f, f.sum(0) + conv_ref.FMA_FLOOR * (rows_summed + 1100)


def dgrad_floor(c0, c1, weight, dz, n, h, w, amax_dz, taps=9, pad=conv_ref.PAD_REFLECT, shift0=0, block_elems=1 << 24):
    """The absolute floor F of the f16x3 data gradient (conv_ref, the f16x3 bound), per element of dx0 and dx1 (rows).

    The data gradient is the forward contract run on dz (scaled by amax_dz) with the flipped, transposed weights, whose
    scale comes from the same max |W|; a folded element is a sum of up to four such outputs.  So F is the adjoint
    applied to the floor's terms: 2^-25 (|W| over dz != 0 / s_dz + |dz| over W != 0 / s_w) + 2^-50 (count) / (s_dz s_w),
    plus 2^-149 for each of the up to four fp32 outputs the fold adds.  Returns {'x0': F0, 'x1': F1 or None}."""
    block_rows = max(1, block_elems // max(taps * (c0 + c1), 1))
    s_x, s_w = conv_ref.f16_scale(amax_dz), conv_ref.f16_scale(conv_ref.finite_max(weight))
    rows0 = n * (h >> shift0) * (w >> shift0)
    x0 = torch.zeros(rows0, c0, dtype=_f64, device=dz.device)
    x1 = torch.zeros(n * h * w, c1, dtype=_f64, device=dz.device) if c1 else None
    nz_w, nz_dz = (weight != 0).to(_f64), (dz != 0).to(_f64)

    def adj(wt, d):
        with torch.enable_grad():               # also from a backward pass, where autograd records nothing
            return _adjoint(x0, c0, x1, c1, wt, d, n, h, w, taps, pad, shift0, block_rows)[:2]

    a, b, c = adj(weight.abs(), nz_dz), adj(nz_w, dz.abs()), adj(nz_w, nz_dz)
    floor = conv_ref.F16_FLOOR
    out = [floor * (a[i] / s_x + b[i] / s_w) + floor ** 2 * c[i] / (s_x * s_w) + 4 * 2.0 ** -149 if a[i] is not None
           else None for i in range(2)]
    return {"x0": out[0], "x1": out[1]}
