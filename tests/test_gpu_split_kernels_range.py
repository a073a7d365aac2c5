"""GPU: the tf32-split and fp32 kernels that are not convolutions, across the exponent range and on non-finite inputs,
element by element against their fp64 contracts at BAR S + F (F: the tf32x3 and FMA floors of tests/conv_ref.py,
carried through each reference).

  * head_mlp (both supported (c, n1)), disp_tail16, conv_wgrad (3x3 with a skip source, 1x1, and a cout-1 layer long
    enough to split its pixel reduction across CTAs), head_gather and head_conv3x3: one operand at a time with its maximum
    from 2^-126 to FLT_MAX (the others small enough that nothing overflows), and all-zero sources;
  * a NaN, +Inf or -Inf at one pixel of one frame: the non-finite outputs are exactly where the operation puts them (a
    head_mlp row; disp_tail16's up2 -> 3x3 (zero pad) -> 3x3 (reflect) footprint; conv_wgrad's dW[:, c] for a bad x at
    channel c, dW[o] for a bad dz at output o), and every other output keeps the clean run's bits;
  * act_backward with y and dy at both ends, where dz and the bias-gradient sums are fp32 subnormals.
The module prints, per kernel and case group, the worst err / S and the worst err / (BAR S + F).
"""
import pytest
import torch

from wavelet_monodepth_b200 import ops
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_ZERO

import conv_grad_ref
import conv_ref as cr
import disp_tail_ref
import head_ref as hr
from contract import Worst, errors

pytestmark = pytest.mark.gpu
DEV = "cuda"
_f64 = torch.float64
FLT_MAX = torch.finfo(torch.float32).max
EXPS = [-126, -100, -60, 0, 60, 100, 128]      # 128: maxima up to FLT_MAX = (1 - 2^-24) 2^128

WORST = Worst("kernel, group, case")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def check(kernel, group, key, got, want, s, f, bar, allow=0.0):
    """Non-finite exactly where want is; |got - want| <= bar S + F + allow elsewhere."""
    what = "%s %s %s" % (kernel, group, key)
    e_s, e_b = errors(got, want, s, allow, floor=f, bar=bar, what=what)
    WORST.note((kernel, group, str(key)), e_s, e_b)
    assert e_b <= 1.0, "%s: err / (BAR S + F) = %.3g (err / S = %.3g)" % (what, e_b, e_s)


def _rand(shape, gen, e):
    """uniform in (-2^e, 2^e) with the first element at the top of the binade (e = 128: FLT_MAX)"""
    t = ((torch.rand(shape, generator=gen, device=DEV, dtype=_f64) * 2 - 1) * 2.0 ** (e - 1) * 2)
    t = t.clamp(-FLT_MAX, FLT_MAX).float()
    t.view(-1)[0] = 2.0 ** (e - 1) * 2 * (1 - 2.0 ** -24)
    return t


def _exps(names, side, e, budget=100):
    """Exponents of a kernel's operands: `side` at e, the others 0, or lower so that the product chain stays below
    2^budget.  side 'zero': the first operand all zero."""
    if side == "zero":
        return {n: 0 for n in names}
    other = min(0, (budget - e) // max(len(names) - 1, 1))
    return {n: (e if n == side else other) for n in names}


def _cases(names):
    return [(n, e) for n in names for e in EXPS] + [("zero", 0)]


# ------------------------------------------------------------------------------------------ head_mlp
MLP_SHAPES = [(32, 64), (64, 128)]


def _mlp_operands(c, n1, ex, seed, rows=300):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = _rand((rows, c), gen, ex["x"])
    w1 = _rand((n1, c, 1, 1), gen, ex["w1"])
    b1 = _rand((n1,), gen, ex["x"] + ex["w1"] - 2)
    wz = _rand((54, n1, 1, 1), gen, ex["wz"])
    return x, w1, b1, wz


@pytest.mark.parametrize("side,e", _cases(["x", "w1", "wz"]))
@pytest.mark.parametrize("c,n1", MLP_SHAPES)
def test_head_mlp_range(c, n1, side, e):
    """z = Wz lrelu(W1 x + b1) within head_ref.BAR S + F, both GEMMs tf32x3; weights up to FLT_MAX round to Inf under
    a plain round-to-nearest split, the pack truncates those instead."""
    ex = _exps(["x", "w1", "wz"], side, e)
    x, w1, b1, wz = _mlp_operands(c, n1, ex, seed=e * 7 + len(side) + c)
    if side == "zero":
        x.zero_()
    z = ops.head_mlp(x, c, ops.pack_head_mlp(w1, b1, wz), n1, slope=0.1)
    torch.cuda.synchronize()
    want, s, f = hr.head_mlp_ref(x, c, w1, b1, wz, 0.1, None, x.shape[0], floor=True)
    assert bool((want.abs() < FLT_MAX).all())
    check("head_mlp%d" % c, side, e, z[:, :54], want, s, f, hr.BAR["head_mlp"])


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("c,n1", MLP_SHAPES)
def test_head_mlp_non_finite_row(c, n1, value):
    """One non-finite value in row 137: only that row's outputs may be non-finite (at least one is), every other row
    keeps the clean run's bits."""
    x, w1, b1, wz = _mlp_operands(c, n1, {"x": 0, "w1": 0, "wz": 0}, seed=3)
    packed = ops.pack_head_mlp(w1, b1, wz)
    clean = ops.head_mlp(x, c, packed, n1)
    bad = x.clone()
    bad[137, 5] = float(value)
    hit = ops.head_mlp(bad, c, packed, n1)
    torch.cuda.synchronize()
    rows = ~torch.isfinite(hit[:, :54]).all(1)
    assert rows.nonzero().reshape(-1).tolist() == [137]
    keep = torch.arange(x.shape[0], device=DEV) != 137
    assert torch.equal(clean[keep], hit[keep])


# ------------------------------------------------------------------------------------------ disp_tail16
def _tail_operands(ex, seed, n=2, h=7, w=9, cout=2):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = _rand((n * h * w, 16), gen, ex["x"])
    w1 = _rand((16, 16, 3, 3), gen, ex["w1"])
    b1 = _rand((16,), gen, ex["x"] + ex["w1"] - 2)
    w2 = _rand((cout, 16, 3, 3), gen, ex["w2"])
    b2 = _rand((cout,), gen, ex["w2"] - 2)
    return x, w1, b1, w2, b2, n, h, w, cout


@pytest.mark.parametrize("side,e", _cases(["x", "w1", "w2"]))
def test_disp_tail16_range(side, e):
    """sigmoid(W2 ELU(W1 up2(x) + b1) + b2) within disp_tail_ref.BAR S + F (+ the ELU and sigmoid's own absolute error,
    the ELU's carried through |W2|)."""
    ex = _exps(["x", "w1", "w2"], side, e)
    x, w1, b1, w2, b2, n, h, w, cout = _tail_operands(ex, seed=e * 5 + len(side))
    if side == "zero":
        x.zero_()
    out = ops.disp_tail16(x, ops.pack_disp_tail16(w1, b1, w2, b2), cout, n, h, w)
    torch.cuda.synchronize()
    want, s, f = disp_tail_ref.disp_tail_ref(x, w1, b1, w2, b2, n, h, w, floor=True)
    allow = cr.ACT_ALLOW * (1 + w2.double().abs().sum((1, 2, 3))).reshape(1, cout, 1, 1)
    check("disp_tail16", side, e, out, want, s, f, disp_tail_ref.BAR, allow=allow.expand_as(want))


def _footprint(n, h, w, pix):
    """The full-resolution pixels disp_tail16 reads half-resolution pixel `pix` through: up2, a zero-padded 3x3, then a
    reflect-padded 3x3 (with its mirrors), as a (N, 2H, 2W) bool."""
    ind = torch.zeros(n * h * w, 1, dtype=_f64, device=DEV)
    ind[pix] = 1
    ones = torch.ones(1, 1, 3, 3, dtype=_f64)
    u, _ = cr.conv_ref(ind, 1, ones, None, n, 2 * h, 2 * w, pad=PAD_ZERO, shift0=1)
    d, _ = cr.conv_ref((u > 0).to(_f64), 1, ones, None, n, 2 * h, 2 * w, pad=PAD_REFLECT)
    return (d > 0).reshape(n, 2 * h, 2 * w)


@pytest.mark.parametrize("where", ["corner", "inner"])
@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
def test_disp_tail16_non_finite_footprint(value, where):
    """A non-finite x at one half-resolution pixel of frame 1 (of 3): the non-finite outputs are exactly its footprint in
    every channel (the tf32 split of an Inf gives NaN, so sigmoid(-Inf) = 0 is not kept), frames 0 and 2 keep their
    bits and the rest of frame 1 meets its bound."""
    x, w1, b1, w2, b2, n, h, w, cout = _tail_operands({"x": 0, "w1": 0, "w2": 0}, seed=4, n=3)
    packed = ops.pack_disp_tail16(w1, b1, w2, b2)
    pix = h * w + (0 if where == "corner" else 3 * w + 4)
    clean = ops.disp_tail16(x, packed, cout, n, h, w)
    bad = x.clone()
    bad[pix, 6] = float(value)
    hit = ops.disp_tail16(bad, packed, cout, n, h, w)
    torch.cuda.synchronize()
    fp = _footprint(n, h, w, pix)
    assert torch.equal(~torch.isfinite(hit), fp[:, None].expand_as(hit))
    assert torch.equal(clean[[0, 2]], hit[[0, 2]])
    want, s, f = disp_tail_ref.disp_tail_ref(x, w1, b1, w2, b2, n, h, w, floor=True)
    keep = ~fp[1][None].expand(cout, -1, -1)
    check("disp_tail16", "non-finite", value, hit[1][keep], want[1][keep], s[1][keep], f[1][keep], disp_tail_ref.BAR,
          allow=cr.ACT_ALLOW * (1 + float(w2.abs().sum())))


# ------------------------------------------------------------------------------------------ conv_wgrad
# (name, c0, c1, cout, n, h, w, taps, pad): the last has 9 output tiles over 61 440 rows, so its pixel reduction is
# split across CTAs (the split-pixel path of DepthDecoder's dispconv(0))
WG_LAYERS = [
    ("3x3_skip", 24, 8, 40, 2, 9, 11, 9, PAD_REFLECT),
    ("1x1", 64, 0, 48, 2, 8, 8, 1, PAD_REFLECT),
    ("cout1_split_rows", 16, 0, 1, 2, 96, 320, 9, PAD_REFLECT),
]


def _wg_operands(layer, ex, seed):
    name, c0, c1, cout, n, h, w, taps, pad = layer
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rows = n * h * w
    x0 = torch.zeros(rows, ops.pad4(c0), device=DEV)
    x0[:, :c0] = _rand((rows, c0), gen, ex["x"])
    x1 = _rand((rows, c1), gen, ex["x"] - 2) if c1 else None
    dz = torch.zeros(rows, ops.pad4(cout), device=DEV)
    dz[:, :cout] = _rand((rows, cout), gen, ex["dz"])
    return x0, x1, dz


def _wgrad(layer, x0, x1, dz):
    name, c0, c1, cout, n, h, w, taps, pad = layer
    dw = ops.conv_wgrad(x0, c0, dz, cout, n, h, w, taps=taps, pad=pad, x1=x1, c1=c1)
    torch.cuda.synchronize()
    return dw


@pytest.mark.parametrize("side,e", _cases(["x", "dz"]))
@pytest.mark.parametrize("layer", WG_LAYERS, ids=[c[0] for c in WG_LAYERS])
def test_conv_wgrad_range(layer, side, e):
    """dW = sum_p A(p) dz(p) within conv_grad_ref.BARS['dW'] S + F (conv_grad_ref.wgrad_floor), A and dz both split to
    nearest: operands up to FLT_MAX take the truncated high piece instead of an infinite one."""
    name, c0, c1, cout, n, h, w, taps, pad = layer
    ex = _exps(["x", "dz"], side, e, budget=110)
    x0, x1, dz = _wg_operands(layer, ex, seed=e * 3 + len(side) + c0)
    if side == "zero":
        x0.zero_()
        if x1 is not None:
            x1.zero_()
    dw = _wgrad(layer, x0, x1, dz)
    k = 3 if taps == 9 else 1
    wzero = torch.zeros(cout, c0 + c1, k, k, device=DEV)
    ref = conv_grad_ref.conv_grads(x0[:, :c0], c0, x1, c1, wzero, dz[:, :cout], n, h, w, taps=taps, pad=pad)
    f = conv_grad_ref.wgrad_floor(x0[:, :c0], c0, x1, c1, wzero, dz[:, :cout], n, h, w, taps=taps, pad=pad)
    want, s = ref["w"]
    assert bool((want.abs() < FLT_MAX).all())
    check("conv_wgrad", name + "/" + side, e, dw, want, s, f, conv_grad_ref.BARS["dW"])


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("operand", ["x0", "x1", "dz"])
@pytest.mark.parametrize("layer", [WG_LAYERS[0], WG_LAYERS[2]], ids=[WG_LAYERS[0][0], WG_LAYERS[2][0]])
def test_conv_wgrad_non_finite(layer, operand, value):
    """A bad x at channel c reaches only dW[:, c]; a bad dz at output o only dW[o].  Every other element keeps the clean
    run's bits, and the bad slice has a non-finite element."""
    name, c0, c1, cout, n, h, w, taps, pad = layer
    if operand == "x1" and not c1:
        pytest.skip("no skip source")
    x0, x1, dz = _wg_operands(layer, {"x": 0, "dz": 0}, seed=8)
    clean = _wgrad(layer, x0, x1, dz)
    pix = n * h * w - w - 3                          # last frame, next-to-last row
    x0b, x1b, dzb = x0.clone(), (x1.clone() if x1 is not None else None), dz.clone()
    sl = torch.zeros_like(clean, dtype=torch.bool)
    if operand == "x0":
        x0b[pix, 5] = float(value)
        sl[:, 5] = True
    elif operand == "x1":
        x1b[pix, 3] = float(value)
        sl[:, c0 + 3] = True
    else:
        o = cout - 1
        dzb[pix, o] = float(value)
        sl[o] = True
    hit = _wgrad(layer, x0b, x1b, dzb)
    bad = ~torch.isfinite(hit)
    assert bool(bad.any()) and not bool((bad & ~sl).any())
    assert torch.equal(clean[~sl], hit[~sl])


# ------------------------------------------------------------------------------------------ fp32 head kernels
HEAD_N, HEAD_H, HEAD_W = 2, 6, 10


@pytest.mark.parametrize("e", EXPS[:-1] + [123, "zero"])
@pytest.mark.parametrize("dual", [False, True], ids=["single", "dual-sigmoid"])
def test_head_gather_range(dual, e):
    """s_g = bias + sum of nine tap products in fp32 FMAs, z at 2^e (123: nine terms of 2^123 stay finite): within
    head_ref.BAR S + F, F = 2^-149 per rounding of the sums and the epilogue."""
    n, h, w = HEAD_N, HEAD_H, HEAD_W
    cout = 3
    groups = 2 * cout if dual else cout
    ez = 0 if e == "zero" else e
    gen = torch.Generator(device=DEV).manual_seed(ez + 200 + dual)
    z = _rand((n * h * w, 9 * groups + 2), gen, ez)
    if e == "zero":
        z.zero_()
    bias = _rand((groups,), gen, ez - 2)
    act, scale = (ACT_SIGMOID, 0.75) if dual else (ACT_NONE, 1.0)
    out = ops.head_gather(z, groups, bias, n, h, w, cout, scale=scale, act=act, dual=dual)
    torch.cuda.synchronize()
    want, s = hr.head_gather_ref(z, z.shape[1], 0, groups, None, bias, scale, act, dual, PAD_REFLECT, None, None, None,
                                 cout, n, h, w)
    got = out.permute(0, 2, 3, 1).reshape(-1, cout)
    f = torch.tensor(cr.FMA_FLOOR * ((9 + 8) * scale * (2 if dual else 1) + 1), dtype=_f64, device=DEV)
    allow = cr.ACT_ALLOW * scale * 2 if dual else 0.0
    check("head_gather", "dual" if dual else "single", e, got, want, s, f, hr.BAR["head_gather"], allow=allow)


@pytest.mark.parametrize("side,e", [(sd, x) for sd in ("t", "w") for x in EXPS[:-1] + [123]] + [("zero", 0)])
def test_head_conv3x3_range(side, e):
    """One 3x3 stage (c = 16, cout = 2) in fp32 FMAs, the rows t or the weights at 2^e: within head_ref.BAR S + F,
    F = 2^-149 per rounding (9c products, the warp's reduction tree and the epilogue)."""
    n, h, w = HEAD_N, HEAD_H, HEAD_W
    c, cout = 16, 2
    ex = _exps(["t", "w"], side, e, budget=110)
    gen = torch.Generator(device=DEV).manual_seed(e + len(side) + 400)
    t = _rand((n * h * w, c), gen, ex["t"])
    if side == "zero":
        t.zero_()
    wa = _rand((cout, c, 3, 3), gen, ex["w"])
    ba = _rand((cout,), gen, ex["t"] + ex["w"] - 2)
    out = ops.head_conv3x3(t, c, 0, ops.pack_head_weight(wa), ba, n, h, w, cout)
    torch.cuda.synchronize()
    want, s = hr.head_conv3x3_ref(t, c, c, 0, -1, wa, ba, None, None, cout, 1.0, ACT_NONE, PAD_REFLECT, None, None, None,
                                  None, n, h, w)
    got = out.permute(0, 2, 3, 1).reshape(-1, cout)
    f = torch.tensor(cr.FMA_FLOOR * (9 * c + 48), dtype=_f64, device=DEV)
    assert bool((want.abs() < FLT_MAX).all())
    check("head_conv3x3", side, e, got, want, s, f, hr.BAR["head_conv3x3"])


# ------------------------------------------------------------------------------------------ act_backward
ACT_BWD_REL = 4 * 2.0 ** -24          # dz's relative part (tests/launch_check.py, ACT_BWD_ULP)


@pytest.mark.parametrize("ey", [-126, -100, 0])
@pytest.mark.parametrize("edy", [-149, -126, -100, -40, 0, 100, 118])   # 700 rows of 2^118: db stays finite
@pytest.mark.parametrize("act", [ACT_NONE, ACT_ELU, ACT_LRELU, ACT_SIGMOID], ids=["none", "elu", "lrelu", "sigmoid"])
def test_act_backward_range(act, edy, ey):
    """dz = dy act'(y) with dy at 2^edy and y at 2^ey (sigmoid: y (1 - y) ~ 2^ey, so dz reaches 2^(edy + ey), deep in
    the subnormals): dz within 4 x 2^-24 |dz| + F, db = sum dz within BARS['db'] S + F (conv_grad_ref.act_bwd_floor)."""
    gen = torch.Generator(device=DEV).manual_seed(edy * 11 + ey + act)
    rows, cout = 700, 5
    y = _rand((rows, cout), gen, ey)
    if act == ACT_SIGMOID:
        y = y.abs()
    elif act == ACT_ELU:
        y = torch.where(torch.arange(rows, device=DEV)[:, None] % 2 == 0, y, -1 + y.abs().clamp(max=0.5))
    dy = _rand((rows, cout), gen, edy)
    dz, db = ops.act_backward(y, dy, cout, act, act_param=0.1)
    torch.cuda.synchronize()
    y64, dy64 = y.double(), dy.double()
    d = {ACT_NONE: torch.ones_like(y64), ACT_ELU: torch.where(y64 > 0, 1.0, y64 + 1),
         ACT_LRELU: torch.where(y64 > 0, 1.0, float(torch.tensor(0.1, dtype=torch.float32))),
         ACT_SIGMOID: y64 * (1 - y64)}[act]
    want = dy64 * d
    f, fb = conv_grad_ref.act_bwd_floor(dy, rows_summed=rows)
    check("act_backward", "dz/%d" % act, "%d/%d" % (edy, ey), dz[:, :cout], want, want.abs(), f, ACT_BWD_REL)
    check("act_backward", "db/%d" % act, "%d/%d" % (edy, ey), db, want.sum(0), want.abs().sum(0), fb,
          conv_grad_ref.BARS["db"])
