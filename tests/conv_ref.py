"""fp64 reference of the gather-GEMM convolution contract (wmd_conv_desc, include/wmd.h), in plain torch.

A direct restatement of the comment above wmd_conv_desc: for output row m (pixel p = pixels[m], or m itself) and tap
(dy, dx) the input pixel q = p + (dy, dx) is mapped into the image by the pad mode (reflect / replicate), or reads zeros
(zero padding); the gate zeros both sources at q; source 0 is x0[map0[n, qy >> shift0, qx >> shift0]] (map0 None: that
pixel's linear index; taps == 1 and map0 None: row m itself, zeros past rows0), source 1 is x1[map1[q]] (map1 None: row q);
a row index of -1 reads zeros.  Returns y64 = act(bias + A @ W) in float64 and the per-element scale
S = |bias| + |A| @ |W|, the sum of the magnitudes of every term of the dot product: an fp32-faithful kernel's error is a
small multiple of 2^-22 S whatever the signs of the operands.

Independent of libwmd and ops.*: index maps are applied with torch indexing, the work is cut into row blocks so that
K = 9 x 2048 fits in memory, and it runs on whatever device the inputs live on.
"""
import math

import torch

PAD_ZERO, PAD_REFLECT, PAD_REPLICATE = 0, 1, 2
ACT_NONE, ACT_ELU, ACT_LRELU, ACT_SIGMOID = 0, 1, 2, 3
_f64 = torch.float64

# err / S bars of the three engines (the error model and the measurements behind them: tests/test_gpu_conv_contract.py)
BAR = {"tf32x3": 4e-5, "f16x3": 2.5e-5, "simt": 1.5e-5}
ACT_ALLOW = 5e-7                  # absolute error of the kernels' expf-based ELU / sigmoid epilogues


# f16x3 bound: |y - y64| <= BAR["f16x3"] S + F per element.  Derivation (conv_tc.cu, load_frag / pack_weight_tc16_kernel):
# an operand v of a launch is scaled by s = 2^e (f16_scale_exp of its maximum: the larger of amax0 / amax1 for the
# activations, max |w| for the weights), v' = v s with |v'| < 2^14, and split h1 = fp16(v'), h2 = fp16(v' - h1) (the
# remainder is exact in fp32).  fp16 has 11 significant bits down to 2^-14 and a fixed spacing of 2^-24 below, so each
# rounding is off by at most 2^-11 of its operand or 2^-25, whichever is larger; h2's error is then at most
# max(2^-22 |v'|, 2^-25):  |dv| <= 2^-22 |v| + 2^-25 / s, and dv = 0 for v = 0.  The kernel forms
# h1x h1w + h1x h2w + h2x h1w = (x + dx)(w + dw) - h2x h2w, off from x w by
#   dx w + x dw + dx dw - h2x h2w.
# The relative parts (2^-22 |x w| each, and |h2x h2w| <= 2^-22 |x w|) and the fp32 accumulation of the products in scaled
# units are what the relative bar covers; what is left is the absolute part
#   F = 2^-25 (sum_{x != 0} |w| / s_x + sum_{w != 0} |x| / s_w) + 2^-50 K' / (s_x s_w)
# (K' = terms with x != 0 and w != 0; the mixed products 2^-22 |x| 2^-25 / s_w are 2^-22 of F), plus 2^-149 for the
# one rounding of y = acc 2^-(e + e_w) + bias where y is an fp32 subnormal.  Within 2^-11 of both maxima, F is below
# 2^-22 S and the pair carries tf32x3's 22 bits; at 2^-m of a maximum F is ~2^(m - 25) of that operand's terms in S.
F16_FLOOR = 2.0 ** -25


# tf32x3 and fp32 FMA bounds: |y - y64| <= BAR[engine] S + F per element, F an absolute floor for the bottom of the fp32
# range (the relative bars alone hold only while every piece, product and partial sum is a normal number).
#
# tf32x3 (conv_tc.cu load_frag / pack_weight_tc_kernel; head_mlp.cu, disp_tail.cu and conv_bwd.cu split the same way):
# each operand v is split into hi + lo (activations: hi truncated, lo the exact remainder, which the MMA reads truncated
# to tf32; weights: both pieces rounded to tf32), the MMA forms hi_x hi_w + hi_x lo_w + lo_x hi_w with fp32
# accumulation.  The worst case assumed is a tensor core that flushes every subnormal input piece, every subnormal
# product and every subnormal accumulator to zero (what H100 does is measured by tests/test_gpu_conv_range.py; keeping
# them is only more accurate).  Then:
#   * a piece is lost only if it is below 2^-126, so the represented operand is off by |dv| < 2^-126 beyond the
#     relative part (tf32 rounding of the pieces and the dropped lo lo: the relative bar);
#   * x' w' - x w = dx w + x dw + dx dw: 2^-126 (|w| for x != 0 + |x| for w != 0), and |dx dw| < 2^-252;
#   * each of the three products of a term is lost only if below 2^-126: 3 x 2^-126 per term with x != 0 and w != 0;
#   * an accumulator is flushed only if below 2^-126, once per MMA instruction that adds a nonzero product: at most
#     3 x 2^-126 per such term (the round-to-nearest epoch and split-K adds on the CUDA cores keep subnormals: 2^-150
#     each, far below);
#   * the bias add, the split-K / stream-K partial sums and the epilogue: a few fp32 roundings of 2^-150 each.
#   F = 2^-126 (sum_{x != 0} |w| + sum_{w != 0} |x| + 6 K') + 16 x 2^-149,  K' = terms with x != 0 and w != 0.
# Where every nonzero operand is >= 2^-102 and every nonzero product >= 2^-99, F < 2^-22 S + 2^-145: the normal range
# keeps its relative bar.  The tightest case is a subnormal operand against a large one: x in [2^-127, 2^-126) flushed
# against w = 2^20 is off by |x w| ~ F / 2.
# fp32 FMA (conv.cu, head.cu, the second stage of disp_tail.cu): acc = fma(x, w, acc) with denormals kept (no -ftz); a
# rounding is off by at most 2^-24 of its result or 2^-150, whichever is larger.  The relative parts are the bar's; the
# absolute parts add up to 2^-150 per rounding: one per term with x w != 0 (a zero product leaves acc exactly), plus the
# bias, the reduction tree and the epilogue.  Each is counted as 2^-149 to cover their (1 + 2^-24)^K growth:
#   F = 2^-149 (K' + extra).
TF32_FLOOR = 2.0 ** -126
FMA_FLOOR = 2.0 ** -149


def tf32_floor(a, wk):
    """F of the tf32x3 bound for gathered rows a (rows, K) and weights wk (K, cout), float64 (derivation above)."""
    nza, nzw = (a != 0).to(_f64), (wk != 0).to(_f64)
    return TF32_FLOOR * (nza @ wk.abs() + a.abs() @ nzw + 6 * (nza @ nzw)) + 16 * 2.0 ** -149


def fma_floor(a, wk, extra=8):
    """F of the fp32 FMA bound: 2^-149 per rounding, K' terms with a w != 0 plus `extra` (bias, reduction, epilogue)."""
    return FMA_FLOOR * (((a != 0).to(_f64) @ (wk != 0).to(_f64)) + extra)


def f16_scale(m):
    """The power-of-two operand scale of an fp16-pair launch whose maximum is m (f16_scale_exp in csrc/conv_tc.cu):
    m s in [2^13, 2^14), the exponent clamped to [-126, 127]; m = 0 or non-finite: 1."""
    m = float(m)
    e = 0
    if 0.0 < m < float("inf"):
        e = 14 - math.frexp(m)[1]
    return 2.0 ** max(-126, min(127, e))


def f16_floor(a, wk, s_x, s_w):
    """F of the f16x3 bound (derivation above) for gathered rows a (rows, K) and weights wk (K, cout), float64."""
    nza, nzw = (a != 0).to(_f64), (wk != 0).to(_f64)
    return (F16_FLOOR * (nza @ wk.abs() / s_x + a.abs() @ nzw / s_w) + F16_FLOOR ** 2 * (nza @ nzw) / (s_x * s_w)
            + 2.0 ** -149)


def finite_max(t):
    """max |t| over the finite values (0 if none): what every libwmd maximum producer reports."""
    a = t.detach().abs()
    a = a[torch.isfinite(a)]
    return float(a.max()) if a.numel() else 0.0


def _pad_coord(q, n, pad):
    """(mapped q, inside) under pad mode `pad`, as pad_coord in csrc/common.cuh."""
    if pad == PAD_REFLECT:
        q = q.abs()
        return torch.where(q >= n, 2 * (n - 1) - q, q), torch.ones_like(q, dtype=torch.bool)
    if pad == PAD_REPLICATE:
        return q.clamp(0, n - 1), torch.ones_like(q, dtype=torch.bool)
    return q.clamp(0, n - 1), (q >= 0) & (q < n)


def activate(y, act, act_param=0.0):
    if act == ACT_ELU:
        return torch.where(y > 0, y, torch.expm1(y.clamp(max=0)))
    if act == ACT_LRELU:
        return torch.where(y > 0, y, y * act_param)
    if act == ACT_SIGMOID:
        return torch.sigmoid(y)
    return y


def _take(x, rows, c):
    """x[rows, :c] in float64 with rows < 0 reading zeros (not 0 * x[0]: that row may hold a NaN or an Inf)."""
    ok = rows >= 0
    v = x[rows.clamp(min=0), :c].to(_f64)
    return torch.where(ok.unsqueeze(-1), v, torch.zeros((), dtype=_f64, device=v.device))


def gather_rows(m, x0, c0, n, h, w, taps=9, pad=PAD_REFLECT, map0=None, shift0=0, x1=None, c1=0, map1=None, gate=None,
                pixels=None, rows0=None):
    """The implicit im2col rows A[m] of output rows `m` (int64 tensor): (len(m), taps, c0 + c1) float64."""
    dev = m.device
    p = pixels.to(dev).long()[m] if pixels is not None else m
    hw = h * w
    nn, rem = p // hw, p % hw
    y, x = rem // w, rem % w
    if taps == 9:
        dy = torch.arange(9, device=dev) // 3 - 1
        dx = torch.arange(9, device=dev) % 3 - 1
    else:
        dy = dx = torch.zeros(1, dtype=torch.long, device=dev)
    qy, oky = _pad_coord(y[:, None] + dy[None], h, pad)
    qx, okx = _pad_coord(x[:, None] + dx[None], w, pad)
    nn = nn[:, None].expand_as(qy)
    ok = oky & okx
    q = (nn * h + qy) * w + qx
    if gate is not None:
        ok = ok & (gate.to(dev).reshape(-1)[q] != 0)
    if taps == 1 and map0 is None:
        r0 = m[:, None].expand_as(q)
        if rows0 is not None:
            r0 = torch.where(r0 < rows0, r0, torch.full_like(r0, -1))
    else:
        hs, ws = h >> shift0, w >> shift0
        qs = (nn * hs + (qy >> shift0)) * ws + (qx >> shift0)
        r0 = map0.to(dev).reshape(-1).long()[qs] if map0 is not None else qs
    r0 = torch.where(ok, r0, torch.full_like(r0, -1))
    a = _take(x0, r0, c0)
    if c1:
        r1 = map1.to(dev).reshape(-1).long()[q] if map1 is not None else q
        r1 = torch.where(ok, r1, torch.full_like(r1, -1))
        a = torch.cat([a, _take(x1, r1, c1)], -1)
    return a


def conv_ref(x0, c0, weight, bias, n, h, w, taps=9, pad=PAD_REFLECT, act=ACT_NONE, act_param=0.0, map0=None, shift0=0,
             x1=None, c1=0, map1=None, gate=None, pixels=None, count=None, max_rows=None, rows0=None, block_elems=1 << 24,
             read_max=False, f16_amax=None, floor=None):
    """(y64, S) for rows [0, min(count, max_rows)): the arguments of ops.conv_rows, with a plain (cout, c0 + c1, k, k)
    weight and an optional bias (cout,).  count: int or 1-element tensor (with pixels); rows0 (taps == 1, map0 None
    only): rows x0 holds, rows past it read zeros (default: x0.shape[0]).
    read_max: also return the largest |value| the launch reads from source 0 and from source 1 (the maxima its fp16-pair
    operand scales must cover): (y64, S, max0, max1).  Non-finite values count as 0 there, as in the kernels.
    f16_amax: the activation maximum an f16x3 launch scales by (the larger of its amax0 / amax1 scalars): also return F,
    the absolute floor of the f16x3 bound (f16_floor; the weight scale follows from the finite max |weight|), last.
    floor: 'tf32x3' or 'simt': also return that engine's F (tf32_floor / fma_floor), last."""
    if f16_amax is not None:
        floor = "f16x3"
    dev = x0.device
    cout = weight.shape[0]
    rows = int(count) if pixels is not None else n * h * w
    if max_rows is not None:
        rows = min(rows, int(max_rows))
    if rows0 is None and taps == 1 and map0 is None:
        rows0 = x0.shape[0]
    k = taps * (c0 + c1)
    wk = weight.to(dev, _f64).permute(2, 3, 1, 0).reshape(k, cout)      # [tap][channel] x cout, the order of A
    wa = wk.abs()
    b = bias.to(dev, _f64) if bias is not None else torch.zeros(cout, dtype=_f64, device=dev)
    y64 = torch.empty(rows, cout, dtype=_f64, device=dev)
    s = torch.empty(rows, cout, dtype=_f64, device=dev)
    if floor == "f16x3":
        s_x, s_w = f16_scale(f16_amax), f16_scale(finite_max(weight))
    if floor is not None:
        fl = torch.empty(rows, cout, dtype=_f64, device=dev)
    step = max(1, block_elems // max(k, 1))
    max0 = max1 = 0.0
    for r in range(0, rows, step):
        m = torch.arange(r, min(rows, r + step), device=dev)
        a = gather_rows(m, x0, c0, n, h, w, taps, pad, map0, shift0, x1, c1, map1, gate, pixels, rows0)
        if read_max:
            max0 = max(max0, finite_max(a[..., :c0]) if c0 else 0.0)
            max1 = max(max1, finite_max(a[..., c0:]) if c1 else 0.0)
        a = a.reshape(len(m), k)
        y64[r:r + len(m)] = a @ wk + b
        s[r:r + len(m)] = a.abs() @ wa + b.abs()
        if floor == "f16x3":
            fl[r:r + len(m)] = f16_floor(a, wk, s_x, s_w)
        elif floor == "tf32x3":
            fl[r:r + len(m)] = tf32_floor(a, wk)
        elif floor == "simt":
            fl[r:r + len(m)] = fma_floor(a, wk)
    out = (activate(y64, act, act_param), s)
    if read_max:
        out += (max0, max1)
    if floor is not None:
        out += (fl,)
    return out


def index_map(mask):
    """(N, H, W) 0/1 mask -> int32 map: running row index over the batch in (n, y, x) order, -1 where inactive."""
    flat = mask.reshape(-1) != 0
    run = torch.cumsum(flat.to(torch.int64), 0) - 1
    return torch.where(flat, run, torch.full_like(run, -1)).reshape(mask.shape).to(torch.int32)


def pixel_list(mask):
    """(N, H, W) 0/1 mask -> int32 linear indices (n*H + y)*W + x of the active pixels, in order."""
    return torch.nonzero(mask.reshape(-1) != 0).reshape(-1).to(torch.int32)
