"""fp64 reference of the coefficient-head contracts (include/wmd.h), in plain torch, built on conv_ref.

Each function restates the comment above its entry point and returns (value64, S), S the sum of the magnitudes of every
term of the element, carried through whatever follows the sums (the activations used here, none / ELU / sigmoid /
LeakyReLU, have slope <= 1, so an error in a sum reaches the output at most scaled by the weights after it):
  head_conv3x3_ref  wmd_head_conv3x3_f32:  scale (act(a) - act(b)) or scale act(a), a / b 3x3 convolutions of row slices
  head_gather_ref   wmd_head_gather_f32:   s_g = bias[g] + sum_tap z[map(p + tap), col0 + tap G + g], the same epilogue
  head_idwt_ref     wmd_head_idwt_f32:     yh of the dual sigmoid heads (zero outside the mask) -> one-level Haar synthesis
                                           -> disp = [clamp01](out disp_scale)
  head_mlp_ref      wmd_head_mlp_f32:      z = Wz lrelu(W1 x + b1)
Values are per output row (pixel p = pixels[m], or m itself, for m < min(count, max_rows)), shape (rows, cout), except
head_idwt_ref's dense planes.  Independent of libwmd and ops.*; runs on whatever device the inputs live on.
"""
import torch
import torch.nn.functional as F

import conv_ref as cr

_f64 = torch.float64

# err / S bars of the head kernels and idwt_bilinear's bound (measurements and error model: tests/test_gpu_head_contract.py)
BAR = {"head_conv3x3": 4e-7, "head_gather": 4.5e-7, "head_idwt": 4.5e-7, "head_mlp": 4e-6}
BILINEAR_ULP = 2.5                # units of 2^-23 x the largest |disp| around the four neighbours
# idwt_bilinear's absolute floor: |err| <= BILINEAR_ULP 2^-23 max|disp| + BILINEAR_FLOOR.  The blend is six products; one
# that lands among the subnormals may lose up to 2^-150 beyond its relative error (sums of subnormals are exact):
# 6 x 2^-150 = 3 x 2^-149
BILINEAR_FLOOR = 3 * 2.0 ** -149


def _rows(n, h, w, pixels, count, max_rows):
    rows = int(count) if pixels is not None else n * h * w
    return rows if max_rows is None else min(rows, int(max_rows))


def _epilogue(s, sabs, cout, scale, act, dual):
    """scale (act(s_j) - act(s_{cout+j})) or scale act(s_j) of the sums s (rows, G) and their scales."""
    if dual:
        v = scale * (cr.activate(s[:, :cout], act) - cr.activate(s[:, cout:2 * cout], act))
        return v, abs(scale) * (sabs[:, :cout] + sabs[:, cout:2 * cout])
    return scale * cr.activate(s[:, :cout], act), abs(scale) * sabs[:, :cout]


def head_conv3x3_ref(t, ld, c, off_a, off_b, wa, ba, wb, bb, cout, scale, act, pad, map, pixels, count, max_rows, n, h,
                     w):
    """t: rows (R, ld); wa / wb plain (cout, c, 3, 3) weights, ba / bb (cout,) or None; off_b < 0: single head.
    map: (N, H, W) row of each pixel in t (-1 inactive) or None (the pixel's linear index)."""
    assert t.shape[1] == ld and off_a + c <= ld and (off_b < 0 or off_b + c <= ld)
    rows = _rows(n, h, w, pixels, count, max_rows)
    kw = dict(pad=pad, map0=map, pixels=pixels, count=count, max_rows=rows)
    a, sa = cr.conv_ref(t[:, off_a:], c, wa, ba, n, h, w, **kw)
    if off_b < 0:
        return scale * cr.activate(a, act), abs(scale) * sa
    b, sb = cr.conv_ref(t[:, off_b:], c, wb, bb, n, h, w, **kw)
    return scale * (cr.activate(a, act) - cr.activate(b, act)), abs(scale) * (sa + sb)


def gather_sums(z, col0, groups, map, bias, pad, pixels, count, max_rows, n, h, w, block=1 << 16):
    """(s, S) (rows, groups): s_g = bias[g] + sum over the nine taps of z[map(p + tap), col0 + tap groups + g]."""
    dev = z.device
    rows = _rows(n, h, w, pixels, count, max_rows)
    b = bias.to(dev, _f64) if bias is not None else torch.zeros(groups, dtype=_f64, device=dev)
    s = b.expand(rows, groups).clone()
    sabs = b.abs().expand(rows, groups).clone()
    for r in range(0, rows, block):
        m = torch.arange(r, min(rows, r + block), device=dev)
        for tap in range(9):
            a = cr.gather_rows(m, z[:, col0 + tap * groups:], groups, n, h, w, pad=pad, map0=map, pixels=pixels)[:, tap]
            s[r:r + len(m)] += a
            sabs[r:r + len(m)] += a.abs()
    return s, sabs


def head_gather_ref(z, ldz, col0, groups, map, bias, scale, act, dual, pad, pixels, count, max_rows, cout, n, h, w):
    """z: rows (R, ldz) of tap products; the value and scale of out[n, j, y, x] at each listed pixel, (rows, cout)."""
    assert z.shape[1] == ldz and col0 + 9 * groups <= ldz
    assert groups == (2 * cout if dual else cout)
    s, sabs = gather_sums(z, col0, groups, map, bias, pad, pixels, count, max_rows, n, h, w)
    return _epilogue(s, sabs, cout, scale, act, dual)


def synth(ll, lh, hl, hh):
    """One-level Haar synthesis (N, C, H, W) x 4 -> (N, C, 2H, 2W): out[2i+a, 2j+b] = 1/2 (ll + (-1)^a lh + (-1)^b hl +
    (-1)^(a+b) hh)."""
    n, c, h, w = ll.shape
    out = ll.new_empty(n, c, 2 * h, 2 * w)
    for a in (0, 1):
        for b in (0, 1):
            out[:, :, a::2, b::2] = 0.5 * (ll + (-1) ** a * lh + (-1) ** b * hl + (-1) ** (a + b) * hh)
    return out


def head_idwt_ref(z, col0, map, mask, bias, scale, pad, ll, disp_scale, clamp01, n, h, w):
    """The whole level tail in fp64.  z rows (R, ldz), ll (N, 1, H, W), mask (N, H, W) or None.

    Returns dict(yh, s_yh (N, 3, H, W); out, s_out, disp, s_disp (N, 1, 2H, 2W)): yh = scale (sigmoid(s+) - sigmoid(s-))
    of the dual heads (groups 6 from col0), exactly zero where mask == 0; out the synthesis of (ll, yh); the error scale of
    out is 1/2 (|ll| + |lh| + |hl| + |hh|) + 1/2 sum over the bands of S_yh (an error in a coefficient reaches each of its
    four outputs with weight 1/2)."""
    dev = z.device
    y, sy = head_gather_ref(z, z.shape[1], col0, 6, map, bias, scale, cr.ACT_SIGMOID, True, pad, None, None, None, 3, n,
                            h, w)
    yh = y.reshape(n, h, w, 3).permute(0, 3, 1, 2).contiguous()
    s_yh = sy.reshape(n, h, w, 3).permute(0, 3, 1, 2).contiguous()
    if mask is not None:
        on = (mask.to(dev).reshape(n, 1, h, w) != 0)
        yh = torch.where(on, yh, torch.zeros_like(yh))
        s_yh = torch.where(on, s_yh, torch.zeros_like(s_yh))
    l64 = ll.to(dev, _f64).reshape(n, 1, h, w)
    bands = [yh[:, k:k + 1] for k in range(3)]
    out = synth(l64, *bands)
    s_bands = 0.5 * (l64.abs() + sum(b.abs() for b in bands) + s_yh.sum(1, keepdim=True))
    s_out = torch.repeat_interleave(torch.repeat_interleave(s_bands, 2, 2), 2, 3)
    disp = out * float(disp_scale)
    if clamp01:
        disp = disp.clamp(0.0, 1.0)
    return dict(yh=yh, s_yh=s_yh, out=out, s_out=s_out, disp=disp, s_disp=s_out * abs(float(disp_scale)))


def head_mlp_ref(x, c, w1, b1, wz, slope, count, max_rows, floor=False):
    """x rows (R, ldx >= c), w1 (n1, c[, 1, 1]), b1 (n1,) or None, wz (nz, n1[, 1, 1]) -> (z (rows, nz), S).

    rows = min(count, max_rows) (count None: max_rows).  S = |Wz| S1 + |Wz| |t| with S1 = |b1| + |W1| |x| the scale of
    t's pre-activation sums and t = lrelu(W1 x + b1).
    floor: also return F of the bound BAR S + F, both stages being tf32x3 (conv_ref.tf32_floor): F1 of the first stage
    plus 2 x 2^-149 for its bias add and LeakyReLU product, carried through |Wz| (slope <= 1), plus the second stage's
    own floor, with every t counted as nonzero (the kernel's t may be nonzero where the exact one is 0)."""
    dev = x.device
    rows = int(max_rows) if count is None else min(int(count), int(max_rows))
    w1 = w1.to(dev, _f64).reshape(w1.shape[0], c)
    wz = wz.to(dev, _f64).reshape(wz.shape[0], w1.shape[0])
    b = b1.to(dev, _f64) if b1 is not None else torch.zeros(w1.shape[0], dtype=_f64, device=dev)
    xs = x[:rows, :c].to(_f64)
    pre = xs @ w1.T + b
    s1 = xs.abs() @ w1.abs().T + b.abs()
    t = cr.activate(pre, cr.ACT_LRELU, slope)
    if floor:
        f1 = cr.tf32_floor(xs, w1.T) + 2 * 2.0 ** -149
        return t @ wz.T, (s1 + t.abs()) @ wz.abs().T, f1 @ wz.abs().T + cr.tf32_floor(t.abs() + f1, wz.T)
    return t @ wz.T, (s1 + t.abs()) @ wz.abs().T


def bilinear_ulps(got, disp, size, align_corners):
    """Worst |got - F.interpolate(disp)| of a bilinear resize in units of 2^-23 x the largest finite |disp| of the 3 x 3
    window around each output's top-left neighbour (a bound of the four neighbours it mixes), plus BILINEAR_FLOOR /
    BILINEAR_ULP: at most BILINEAR_ULP exactly when |err| <= BILINEAR_ULP 2^-23 max|disp| + BILINEAR_FLOOR.  disp
    (N, C, h, w) on got's device; the interpolation runs in disp's dtype.  got must be NaN, +Inf and -Inf exactly where torch's resize is: a
    non-finite neighbour reaches even the outputs that give it zero weight (0 x NaN, 0 x Inf)."""
    dev = got.device
    want = F.interpolate(disp, size=size, mode="bilinear", align_corners=align_corners)
    assert got.shape == want.shape
    g = got.to(want.dtype)
    for what, f in (("NaN", torch.isnan), ("+Inf", lambda t: t == float("inf")), ("-Inf", lambda t: t == -float("inf"))):
        assert torch.equal(f(g), f(want)), "bilinear: %d %s outputs where torch's resize has %d" % (
            int(f(g).sum()), what, int(f(want).sum()))
    hs, ws = disp.shape[-2:]
    m = F.max_pool2d(torch.where(torch.isfinite(disp), disp.abs(), torch.zeros_like(disp)), 3, stride=1, padding=1)
    ys, xs = torch.arange(size[0], device=dev, dtype=_f64), torch.arange(size[1], device=dev, dtype=_f64)
    if align_corners:
        fy = ys * ((hs - 1) / max(size[0] - 1, 1))
        fx = xs * ((ws - 1) / max(size[1] - 1, 1))
    else:
        fy = ((ys + 0.5) * (hs / size[0]) - 0.5).clamp(min=0)
        fx = ((xs + 0.5) * (ws / size[1]) - 0.5).clamp(min=0)
    y0, x0 = fy.floor().long().clamp(max=hs - 1), fx.floor().long().clamp(max=ws - 1)
    mag = m[:, :, y0][:, :, :, x0]
    ok = torch.isfinite(want)
    if not bool(ok.any()):
        return 0.0
    return float(((g - want).abs() / (mag * 2.0 ** -23 + BILINEAR_FLOOR / BILINEAR_ULP))[ok].max())
