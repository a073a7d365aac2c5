"""CPU: the fp64 conv-contract reference (tests/conv_ref.py) against torch's conv2d and the sparse-op oracle.

The GPU contract tests (test_gpu_conv_contract.py) measure the kernels' error against this reference, so it has to be
right on its own: every gather path it restates is checked here against an independent formulation, exactly (fp64
sums of the same products in a different order: <= 1e-12 relative).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sparse_ops as osp

import conv_ref as cr
from helpers import close, rnd, rows_of


def nchw_of(rows, n, h, w):
    return rows.reshape(n, h, w, -1).permute(0, 3, 1, 2)


_MODE = {cr.PAD_ZERO: "constant", cr.PAD_REFLECT: "reflect", cr.PAD_REPLICATE: "replicate"}


@pytest.mark.parametrize("pad", [cr.PAD_ZERO, cr.PAD_REFLECT, cr.PAD_REPLICATE])
@pytest.mark.parametrize("n,cin,cout,h,w", [(2, 5, 7, 6, 9), (1, 40, 33, 2, 5), (1, 3, 4, 5, 2)])
def test_dense_3x3_matches_conv2d(pad, n, cin, cout, h, w):
    x, wt, b = rnd(n, cin, h, w, seed=1), rnd(cout, cin, 3, 3, seed=2), rnd(cout, seed=3)
    y64, s = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w, pad=pad)
    xp = F.pad(x.double(), (1, 1, 1, 1), mode=_MODE[pad])
    assert close(nchw_of(y64, n, h, w), F.conv2d(xp, wt.double(), b.double()))
    assert close(nchw_of(s, n, h, w), F.conv2d(xp.abs(), wt.double().abs(), b.double().abs()))


@pytest.mark.parametrize("act", [cr.ACT_ELU, cr.ACT_LRELU, cr.ACT_SIGMOID])
def test_activations_and_1x1(act):
    n, cin, cout, h, w = 2, 12, 9, 3, 7
    x, wt, b = rnd(n, cin, h, w, seed=4), rnd(cout, cin, 1, 1, seed=5), rnd(cout, seed=6)
    y64, _ = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w, taps=1, act=act, act_param=0.2)
    z = F.conv2d(x.double(), wt.double(), b.double())
    want = {cr.ACT_ELU: F.elu, cr.ACT_LRELU: lambda t: F.leaky_relu(t, 0.2), cr.ACT_SIGMOID: torch.sigmoid}[act](z)
    assert close(nchw_of(y64, n, h, w), want)


def test_bias_none_and_row_blocks():
    n, cin, cout, h, w = 1, 7, 5, 9, 11
    x, wt = rnd(n, cin, h, w, seed=7), rnd(cout, cin, 3, 3, seed=8)
    y64, s = cr.conv_ref(rows_of(x), cin, wt, None, n, h, w, pad=cr.PAD_REFLECT, block_elems=100)   # two rows per block
    xp = F.pad(x.double(), (1, 1, 1, 1), mode="reflect")
    assert close(nchw_of(y64, n, h, w), F.conv2d(xp, wt.double()))
    assert bool((s >= y64.abs()).all())


@pytest.mark.parametrize("pad", [cr.PAD_ZERO, cr.PAD_REFLECT, cr.PAD_REPLICATE])
@pytest.mark.parametrize("p_in,p_out", [(0.6, 0.5), (0.1, 0.9), (0.0, 0.5)])
def test_sparse_3x3_matches_oracle(pad, p_in, p_out):
    """Compact input rows through an index map, outputs at a pixel list (the reference's sparse_conv3x3)."""
    cin, cout, h, w = 6, 5, 9, 13
    rs = np.random.RandomState(9)
    im = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < p_in).astype(np.float32))
    om = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < p_out).astype(np.float32))
    wt, b = rnd(cout, cin, 3, 3, seed=10), rnd(cout, seed=11)
    m_in = int(im.sum())
    xv = rnd(cin * m_in, seed=12)
    idx, _ = osp.index_map(im)
    want, _, _ = osp.conv3x3(wt.double(), b.double(), xv.double(), idx, om, padding=_MODE[pad], make_result=False)
    rows = xv.reshape(cin, m_in).t().contiguous() if m_in else torch.zeros(1, cin)
    pix = cr.pixel_list(om[0])
    y64, _ = cr.conv_ref(rows, cin, wt, b, 1, h, w, pad=pad, map0=cr.index_map(im[0]), pixels=pix, count=len(pix))
    assert y64.shape == (len(pix), cout)
    assert close(y64.t().reshape(-1), want)


def test_upsample_concat_gate_matches_oracle():
    """Half-resolution compact source 0 (shift0 = 1), dense skip source 1, gate: sparse_upsample + sparse_conv3x3."""
    c0, cs, cout, h, w = 5, 3, 4, 7, 9
    rs = np.random.RandomState(13)
    s0 = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < 0.3).astype(np.float32))
    u = F.interpolate(s0, scale_factor=2, mode="nearest")
    s2, s3, s4 = F.max_pool2d(s0, 5, 1, 2), F.max_pool2d(u, 5, 1, 2), F.max_pool2d(u, 3, 1, 1)
    m2 = int(s2.sum())
    xv, skip = rnd(c0 * m2, seed=14), rnd(1, cs, 2 * h, 2 * w, seed=15)
    wt, b = rnd(cout, c0 + cs, 3, 3, seed=16), rnd(cout, seed=17)
    map2, _ = osp.index_map(s2)
    map3, _ = osp.index_map(s3)
    up, _ = osp.upsample_concat(xv.double(), c0, map2, skip.double(), s3, make_result=False)
    want, _, _ = osp.conv3x3(wt.double(), b.double(), up, map3, s4, padding="reflect", make_result=False)
    pix = cr.pixel_list(s4[0])
    y64, _ = cr.conv_ref(xv.reshape(c0, m2).t().contiguous(), c0, wt, b, 1, 2 * h, 2 * w, map0=cr.index_map(s2[0]),
                         shift0=1, x1=rows_of(skip), c1=cs, gate=s3[0], pixels=pix, count=len(pix))
    assert close(y64.t().reshape(-1), want)


def test_compact_skip_map1_matches_dense_skip():
    """x1 holding only the rows of listed pixels (map1) is the same convolution as the dense skip map."""
    n, c0, c1, cout, h, w = 2, 4, 6, 5, 6, 8
    rs = np.random.RandomState(18)
    sel = torch.from_numpy((rs.uniform(size=(n, h, w)) < 0.5).astype(np.uint8))
    x0, skip = rnd(n, c0, h, w, seed=19), rnd(n, c1, h, w, seed=20)
    skip = skip * sel[:, None].float()                           # the dense map is zero where the compact one has no row
    wt, b = rnd(cout, c0 + c1, 3, 3, seed=21), rnd(cout, seed=22)
    dense, _ = cr.conv_ref(rows_of(x0), c0, wt, b, n, h, w, x1=rows_of(skip), c1=c1)
    compact = rows_of(skip)[cr.pixel_list(sel).long()]
    got, _ = cr.conv_ref(rows_of(x0), c0, wt, b, n, h, w, x1=compact, c1=c1, map1=cr.index_map(sel))
    assert close(got, dense)


def test_rows0_reads_zeros_past_the_source_rows():
    """1x1 form over a source's own rows: output rows past rows0 see only source 1 (here: nothing but the bias)."""
    n, cin, cout, h, w = 1, 8, 6, 5, 7
    rows0 = 20
    x, wt, b = rnd(n, cin, h, w, seed=23), rnd(cout, cin, 1, 1, seed=24), rnd(cout, seed=25)
    y64, s = cr.conv_ref(rows_of(x)[:rows0], cin, wt, b, n, h, w, taps=1)
    full = rows_of(F.conv2d(x.double(), wt.double(), b.double()))
    assert close(y64[:rows0], full[:rows0])
    assert torch.equal(y64[rows0:], b.double().expand(n * h * w - rows0, cout))
    assert torch.equal(s[rows0:], b.double().abs().expand(n * h * w - rows0, cout))


def test_count_and_max_rows():
    n, cin, cout, h, w = 1, 3, 2, 4, 4
    x, wt, b = rnd(n, cin, h, w, seed=26), rnd(cout, cin, 3, 3, seed=27), rnd(cout, seed=28)
    pix = torch.arange(0, 16, 2, dtype=torch.int32)
    y8, _ = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w, pixels=pix, count=8)
    y5, _ = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w, pixels=pix, count=8, max_rows=5)
    y0, _ = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w, pixels=pix, count=0)
    assert y8.shape == (8, cout) and torch.equal(y5, y8[:5]) and y0.shape == (0, cout)
    dense, _ = cr.conv_ref(rows_of(x), cin, wt, b, n, h, w)
    assert torch.equal(y8, dense[pix.long()])


# ------------------------------------------------------------------------------------------ the f16x3 bound
def _emulate_f16x3(x, w, amax, wmax):
    """x (R, K) @ w (K, cout) as the f16x3 engine forms it, in fp64: each operand scaled by its launch's power of two,
    split into h1 = fp16(v s) and h2 = fp16(v s - h1) (torch float16 casts: round to nearest even, with subnormals), the
    three products h1 h1 + h1 h2 + h2 h1 summed exactly, the scales undone.  No tensor-core accumulation: this checks the
    split part of the bound only."""
    s_x, s_w = cr.f16_scale(amax), cr.f16_scale(wmax)

    def split(v, s):
        v = (v.double() * s).float()                  # a power of two: exact
        h1 = v.half().float()
        h2 = (v - h1).half().float()                  # the remainder is exact in fp32
        return h1.double(), h2.double()

    x1, x2 = split(x, s_x)
    w1, w2 = split(w, s_w)
    return (x1 @ w1 + x1 @ w2 + x2 @ w1) / (s_x * s_w)


def _split_err(x, w, amax, wmax):
    """(|emulated - exact|, S, F) per element."""
    want = x.double() @ w.double()
    err = (_emulate_f16x3(x, w, amax, wmax) - want).abs()
    return err, x.double().abs() @ w.double().abs(), cr.f16_floor(x.double(), w.double(), cr.f16_scale(amax),
                                                                   cr.f16_scale(wmax))


REL_SPLIT = 2.0 ** -20            # the split's relative part: 2^-22 for dx, dw and h2x h2w each, with room


@pytest.mark.parametrize("top", [-140, -126, -60, 0, 60, 116, 127])
@pytest.mark.parametrize("side", ["x", "w"])
def test_f16x3_floor_bounds_the_emulated_split(top, side):
    """Rows (or output channels) at 2^-m of the launch maximum 2^top, m = 0 .. 45, mixed signs, K = 64: the emulated
    split never leaves 2^-20 S + F, and F is what lets it - a plain relative bar fails from m ~ 22 on."""
    g = torch.Generator().manual_seed(top + 200)
    ms = torch.arange(46, dtype=torch.float64)
    x = torch.rand(46, 64, generator=g, dtype=torch.float64) * 2 - 1
    w = torch.rand(64, 46, generator=g, dtype=torch.float64) * 2 - 1
    if side == "x":
        x = x * torch.exp2(top - ms)[:, None]
        x[0, 0] = 2.0 ** top                          # the maximum sits in row 0
        w[0, 0] = 1.0
    else:
        w = w * torch.exp2(top - ms)[None, :]
        w[0, 0] = 2.0 ** top
        x[0, 0] = 1.0
    x, w = x.float(), w.float()
    err, s, f = _split_err(x, w, cr.finite_max(x), cr.finite_max(w))
    assert bool((err <= REL_SPLIT * s + f).all()), float((err / (REL_SPLIT * s + f)).max())
    if top >= -60:                                    # the deep rows are normal fp32 numbers: the relative bar alone fails
        assert float((err / s)[s > 0].max()) > cr.BAR["f16x3"]


def test_f16x3_floor_is_tight():
    """One term per element (K = 1), x at 2^-m of its maximum with m = 24 .. 36: there the low piece is an fp16
    subnormal and the split's error reaches F within a factor of 2 (4096 samples per m); past m ~ 38 x s drops under
    fp16's smallest subnormal and the error is |x w| itself, below F."""
    g = torch.Generator().manual_seed(7)
    w = (torch.rand(1, 32, generator=g) * 0.5 + 0.5)
    for m in range(24, 37):
        x = (torch.rand(4096, 1, generator=g, dtype=torch.float64) * 0.5 + 0.5) * 2.0 ** -m
        x[0, 0] = 1.0
        err, s, f = _split_err(x.float(), w, 1.0, cr.finite_max(w))
        ratio = (err / (REL_SPLIT * s + f))[1:]
        assert float(ratio.max()) <= 1.0 and float(ratio.max()) >= 0.5, (m, float(ratio.max()))


def test_f16_scale_matches_the_kernel_rule():
    """m s in [2^13, 2^14) for every finite m > 0, the exponent clamped to [-126, 127]; 0 and non-finite maxima: 1."""
    for m in [2.0 ** -149, 2.0 ** -126, 1e-30, 0.3, 1.0, 8191.9, 2.0 ** 116, 3.4e38]:
        s = cr.f16_scale(m)
        e = math.log2(s)
        assert e == int(e) and -126 <= e <= 127
        assert m * s < 2.0 ** 14 and (m * s >= 2.0 ** 13 or e == 127)
    assert cr.f16_scale(0.0) == cr.f16_scale(float("inf")) == cr.f16_scale(float("nan")) == 1.0


# ------------------------------------------------------------------------------------------ the tf32x3 and FMA floors
TINY = 2.0 ** -126                 # the smallest normal fp32


def _tf32(v, rna):
    """float32 array -> tf32 values (13 low mantissa bits cleared): truncated, or rounded to nearest with ties away
    (cvt.rna) except where that overflows a finite v, which is truncated (tf32_rna_finite in csrc/common.cuh)."""
    bits = v.view(np.uint32)
    t = (bits & np.uint32(0xFFFFE000)).view(np.float32)
    if not rna:
        return t
    r = ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return np.where(np.isinf(r) & np.isfinite(v), t, r)


def _flush(v, on):
    return np.where(np.abs(v) < TINY, 0.0, v) if on else v


def _emulate_tf32x3(x, w, flush):
    """x (R, K) @ w (K, C) as the tf32x3 engine forms it: activations split by truncation (the MMA reads the exact
    remainder truncated to tf32), weights split to nearest (both pieces), products lo_x hi_w, hi_x lo_w, hi_x hi_w exact,
    one accumulator rounding to fp32 per MMA of 8 k (in the kernel's order: small terms first).  flush: every subnormal
    piece, product and accumulator becomes 0 (the worst case the floor assumes); else subnormals are kept."""
    x, w = x.numpy(), w.numpy()
    xh = _tf32(x, False)
    xl = _tf32((x - xh).astype(np.float32), False)
    wh = _tf32(w, True)
    wl = _tf32((w - wh).astype(np.float32), True)
    xh, xl, wh, wl = (_flush(v.astype(np.float64), flush) for v in (xh, xl, wh, wl))
    acc = np.zeros((x.shape[0], w.shape[1]), dtype=np.float32)
    for k0 in range(0, x.shape[1], 8):
        ks = slice(k0, k0 + 8)
        for a, b in ((xl, wh), (xh, wl), (xh, wh)):
            p = _flush(a[:, ks, None] * b[None, ks, :], flush).sum(1)
            acc = _flush((acc.astype(np.float64) + p).astype(np.float32), flush).astype(np.float32)
    return torch.from_numpy(acc.astype(np.float64))


def _emulate_fma(x, w):
    """x (R, K) @ w (K, C) as an fp32 FMA chain: acc = fp32(acc + x w) in k order (x w is exact in fp64), subnormals kept."""
    x, w = x.numpy().astype(np.float64), w.numpy().astype(np.float64)
    acc = np.zeros((x.shape[0], w.shape[1]), dtype=np.float32)
    for k in range(x.shape[1]):
        acc = (acc.astype(np.float64) + x[:, k, None] * w[None, k, :]).astype(np.float32)
    return torch.from_numpy(acc.astype(np.float64))


def _engine_err(engine, x, w, flush=True):
    """(|emulated - exact|, S, F) per element of x @ w for 'tf32x3' or 'simt'."""
    got = _emulate_tf32x3(x, w, flush) if engine == "tf32x3" else _emulate_fma(x, w)
    x64, w64 = x.double(), w.double()
    floor = cr.tf32_floor(x64, w64) if engine == "tf32x3" else cr.fma_floor(x64, w64)
    return (got - x64 @ w64).abs(), x64.abs() @ w64.abs(), floor


def _spread(top, side, seed):
    """x (46, 64) and w (64, 46), mixed signs; the rows of x (side 'x'), the columns of w ('w') or both at 2^-m of
    2^top, m = 0 .. 45; the other operand at most 2^-7, so that no sum overflows."""
    g = torch.Generator().manual_seed(seed)
    ms = torch.arange(46, dtype=torch.float64)
    x = torch.rand(46, 64, generator=g, dtype=torch.float64) * 2 - 1
    w = torch.rand(64, 46, generator=g, dtype=torch.float64) * 2 - 1
    if side in ("x", "both"):
        x = x * torch.exp2(top - ms)[:, None]
    else:
        x = x * 2.0 ** -7
    if side in ("w", "both"):
        w = w * torch.exp2(top - ms)[None, :]
    else:
        w = w * 2.0 ** -7
    return x.float(), w.float()


FLOOR_CASES = ([(side, top) for side in ("x", "w") for top in (-149, -140, -126, -100, -60, 0, 60, 116, 127)]
               + [("both", top) for top in (-75, -70, -63, -40, 0, 60)])


@pytest.mark.parametrize("side,top", FLOOR_CASES)
@pytest.mark.parametrize("engine,flush", [("tf32x3", True), ("tf32x3", False), ("simt", False)],
                         ids=["tf32x3-flush", "tf32x3-keep", "simt"])
def test_floor_bounds_the_emulated_engine(engine, flush, side, top):
    """From 2^-149 to 2^127 the emulated engine never leaves BAR S + F, with subnormals flushed or kept; where pieces,
    products or sums are subnormal the plain relative bar fails, so F is what lets it."""
    x, w = _spread(top, side, seed=top + 300 + len(side))
    err, s, f = _engine_err(engine, x, w, flush)
    bound = cr.BAR[engine] * s + f
    assert bool((err <= bound).all()), float((err / bound).max())
    if side == "both" and top <= -63 or side != "both" and top - 7 <= -140:
        assert float((err / s)[s > 0].max()) > cr.BAR[engine]


def test_floor_is_negligible_in_the_normal_range():
    """Operands >= 2^-102 and products >= 2^-99: F < 2^-22 S + 2^-145, so the relative bar is unchanged there."""
    x, w = _spread(-40, "both", seed=5)
    x = torch.where(x.abs() < 2.0 ** -50, torch.full_like(x, 2.0 ** -50), x)
    w = torch.where(w.abs() < 2.0 ** -49, torch.full_like(w, 2.0 ** -49), w)
    x64, w64 = x.double(), w.double()
    s = x64.abs() @ w64.abs()
    for f in (cr.tf32_floor(x64, w64), cr.fma_floor(x64, w64)):
        assert bool((f < 2.0 ** -22 * s + 2.0 ** -145).all())


def test_tf32_floor_is_tight():
    """x in [2^-127, 2^-126) against w = +-2^20, K = 1: a tensor core that flushes subnormal pieces loses x whole, an
    error of |x w|, which reaches F within a factor of 2 (4096 samples)."""
    g = torch.Generator().manual_seed(9)
    x = ((torch.rand(4096, 1, generator=g, dtype=torch.float64) * 0.5 + 0.5) * TINY).float()
    w = torch.tensor([[2.0 ** 20, -2.0 ** 20]])
    err, s, f = _engine_err("tf32x3", x, w, flush=True)
    ratio = err / (cr.BAR["tf32x3"] * s + f)
    assert 0.5 <= float(ratio.max()) <= 1.0, float(ratio.max())


def test_fma_floor_is_tight():
    """64 products of 2^-150 (1 + 2^-10) each, all in the subnormal range: every rounding of the chain goes up by
    nearly 2^-150, and the chain's error reaches F (2^-149 per rounding, plus 8 for the epilogue) within a factor of 2.5."""
    x = torch.full((1, 64), 2.0 ** -75 * (1 + 2.0 ** -10))
    w = torch.full((64, 1), 2.0 ** -75)
    err, s, f = _engine_err("simt", x, w)
    ratio = float((err / (cr.BAR["simt"] * s + f)).max())
    assert 0.4 <= ratio <= 1.0, ratio


def test_round_to_nearest_split_keeps_the_top_binade_finite():
    """cvt.rna rounds a finite |w| >= (2 - 2^-11) 2^127 up to Inf; the split truncates there instead, so hi + lo is
    finite and FLT_MAX weights against tiny activations stay within the bound.  Below the threshold the split is the
    plain round to nearest."""
    fmax = np.float32(np.finfo(np.float32).max)
    edge = np.float32(np.ldexp(2 - 2.0 ** -11, 127))
    below = np.nextafter(edge, np.float32(0))
    v = np.array([fmax, -fmax, edge, below, np.float32(1.5)], dtype=np.float32)
    hi = _tf32(v, True)
    assert np.isfinite(hi).all() and np.isfinite(v - hi).all()
    assert hi[2] == (v[2].view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)      # the tie: truncated
    assert hi[3] == np.float32(np.ldexp(2 - 2.0 ** -10, 127))                          # below it: to nearest
    x = torch.full((3, 16), 2.0 ** -100)
    x[1] *= -1
    w = torch.full((16, 2), float(fmax))
    w[:, 1] = -float(fmax)
    err, s, f = _engine_err("tf32x3", x, w, flush=True)
    assert bool((err <= cr.BAR["tf32x3"] * s + f).all())
