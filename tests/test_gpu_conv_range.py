"""GPU: the gather-GEMM convolutions across the exponent range and on non-finite inputs, element by element against the
fp64 contract (tests/conv_ref.py).

The fp16-pair engine (f16x3) scales a launch's activations by one power of two taken from the larger source maximum
(shared by every frame and both sources) and its weights by one taken from max |w|.  An operand far below its maximum
has its low fp16 piece in the subnormal range, so f16x3 is held to BAR S + F (conv_ref, the f16x3 bound), not to the
plain relative bar.  tf32x3 and the fp32 FMA engine are held to BAR S + F with their own floors (conv_ref, the tf32x3
and FMA bounds), which matter only where pieces, products or sums are fp32 subnormals.  The cases:
  * spread within one launch: frames, the skip source or output channels at 2^-m of the maximum, m = 0 .. 45, through
    the window kernel, the gather path and the 1x1 form, whole and balanced (stream-K); maxima up to 2^20 loose;
  * exponent edges, every engine: source maxima from 2^-126 to 2^127 against weight maxima from 2^-126 to FLT_MAX,
    products and partial sums down in the subnormal range; tf32x3 also split-K (2 and 4 splits);
  * all-zero sources (maximum 0): y = act(bias) exactly;
  * a NaN, +Inf or -Inf at one pixel of one frame, under no activation, ELU and sigmoid: the non-finite outputs are
    exactly the fp64 reference's (the pixel's 3x3 halo and its pad-mode mirrors), except that the tensor-core engines may
    give NaN wherever the reference's pre-activation is non-finite (ELU(-Inf) = -1 and sigmoid(+-Inf) are finite); every
    other output meets its bar;
  * backward: f16x3 data gradients whose dz spans decades (saturated sigmoid, deep ELU rows), at conv_grad_ref.BARS S
    + F; a non-finite upstream gradient in one frame leaves the other frame's data gradients bit-identical;
  * a decoder batch with one corrupted frame: the other frames' outputs (dense) and input-feature gradients (native
    training step) keep their bits, the sparse decoder's keep their masks and stay within the parity bar.
The module prints, per engine, case group and ratio, the worst err / S and the worst err / (BAR S + F).
"""
import numpy as np
import pytest
import torch

from oracle import parity
from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import ops, synth, train_native
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_grad_ref
import conv_ref as cr
from contract import Worst, errors
from conv_launch import pack

pytestmark = pytest.mark.gpu
DEV = "cuda"
BAR = cr.BAR
ENGINES = ["f16x3", "tf32x3", "simt"]
FLT_MAX = torch.finfo(torch.float32).max
PARITY_TOL = 1e-4                 # oracle/parity.py: the float bar of the parity statement

WORST = Worst("engine, group, ratio")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def _amax(x):
    """the library's own maximum of a source (finite values only), as a 1-element device tensor"""
    out = torch.zeros(1, device=DEV)
    ops.amax_rows(x, out)
    return out


class Geo:
    """One launch's geometry: layout 'window' (dense 3x3), 'gather' (pixel list), '1x1'; '-balanced': stream-K,
    '-splitK' (tf32x3 only): the reduction cut into K equal ranges."""

    def __init__(self, layout, n, h, w, c0, c1, cout):
        self.layout, self.n, self.h, self.w, self.c0, self.c1, self.cout = layout, n, h, w, c0, c1, cout
        self.taps = 1 if layout.startswith("1x1") else 9
        self.splits = 0 if layout.endswith("-balanced") else None
        if "-split" in layout:
            self.splits = int(layout.rsplit("-split", 1)[1])
        total = n * h * w
        self.pixels = None
        if layout.startswith("gather"):
            p = torch.arange(total, device=DEV)
            self.pixels = p[p % 5 != 3].to(torch.int32)         # holes: the tap table, not the window
        self.rows = total if self.pixels is None else len(self.pixels)


def run(engine, g, x0, x1, wt, b, amax0=None, amax1=None, pad=PAD_REFLECT, act=ACT_NONE):
    """y rows (rows, cout) of one launch; f16x3 takes the given maxima, or the library's own of each source."""
    wp = pack(wt, g.c1, engine)
    kw = {}
    if engine == "f16x3":
        kw["amax0"] = amax0 if amax0 is not None else _amax(x0)
        if x1 is not None:
            kw["amax1"] = amax1 if amax1 is not None else _amax(x1)
    if engine != "simt" and g.splits is not None:
        kw["splits"] = g.splits
    count = torch.tensor([g.rows], dtype=torch.int32, device=DEV) if g.pixels is not None else None
    y = ops.conv_rows(x0, g.c0, wp, b, g.cout, g.n, g.h, g.w, taps=g.taps, pad=pad, act=act, x1=x1, c1=g.c1,
                      pixels=g.pixels, count=count, **kw)
    torch.cuda.synchronize()
    return y[:g.rows, :g.cout], (kw.get("amax0"), kw.get("amax1"))


def reference(engine, g, x0, x1, wt, b, maxima, pad=PAD_REFLECT, act=ACT_NONE):
    """(y64, S, F, pre64): F the engine's floor (f16x3: from the scalars the launch scaled by), pre64 the fp64
    pre-activation."""
    amax16 = None
    if engine == "f16x3":
        amax16 = max(float(maxima[0]), float(maxima[1]) if maxima[1] is not None else 0.0)
    ref = cr.conv_ref(x0, g.c0, wt, b, g.n, g.h, g.w, taps=g.taps, pad=pad, x1=x1, c1=g.c1, pixels=g.pixels,
                      count=g.rows, f16_amax=amax16, floor=engine)
    return cr.activate(ref[0], act), ref[1], ref[2], ref[0]


def check(engine, y, y64, s, f, group, key, act=ACT_NONE, pre64=None):
    """Non-finite exactly where y64 is; elsewhere |y - y64| <= BAR S + F (+ the activation's own error).  The tensor-core
    engines may also give NaN where pre64 (the fp64 pre-activation) is non-finite (contract.errors)."""
    what = "%s %s %s" % (engine, group, key)
    allow = 0.0 if act in (ACT_NONE, ACT_LRELU) else cr.ACT_ALLOW
    e_s, e_b = errors(y, y64, s, allow, floor=f, bar=BAR[engine], pre=pre64 if engine != "simt" else None, what=what)
    WORST.note((engine, group, str(key)), e_s, e_b)
    assert e_b <= 1.0, "%s: err / (BAR S + F) = %.3g (err / S = %.3g)" % (what, e_b, e_s)


def _rand(shape, gen, lo=-1.0, hi=1.0):
    return torch.rand(shape, generator=gen, device=DEV) * (hi - lo) + lo


# ------------------------------------------------------------------------------------------ spread within one launch
RATIOS = [0, 11, 16, 20, 22, 24, 30, 38, 45]
LAYOUTS = ["window", "window-balanced", "gather", "gather-balanced", "1x1", "1x1-balanced"]


def _spread_operands(g, kind, m, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    n, hw = g.n, g.h * g.w
    x0 = _rand((n * hw, g.c0), gen)
    x1 = _rand((n * hw, g.c1), gen)
    wt = _rand((g.cout, g.c0 + g.c1, 3 if g.taps == 9 else 1, 3 if g.taps == 9 else 1), gen)
    b = _rand((g.cout,), gen)
    if kind == "frames":             # frame j at 2^-(m j / 3): one scale for the batch
        sc = torch.exp2(-torch.round(torch.arange(n, device=DEV) * m / (n - 1))).repeat_interleave(hw)[:, None]
        x0, x1 = x0 * sc, x1 * sc
    elif kind == "x1":               # the skip source far below x0
        x1 = x1 * 2.0 ** -m
    else:                            # the second half of the output channels: weights at 2^-m of max |w|
        wt[g.cout // 2:] *= 2.0 ** -m
        b[g.cout // 2:] *= 2.0 ** -m
    return x0.contiguous(), x1.contiguous(), wt, b


@pytest.mark.parametrize("m", RATIOS)
@pytest.mark.parametrize("kind", ["frames", "x1", "cout"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_spread_within_one_launch(layout, kind, m):
    """f16x3 within BAR S + F at every ratio; tf32x3 and SIMT within their plain bars on the same inputs."""
    g = Geo(layout, 4, 6, 10, 40, 24, 48)
    x0, x1, wt, b = _spread_operands(g, kind, m, seed=m * 31 + len(kind) + len(layout))
    for engine in ENGINES:
        y, maxima = run(engine, g, x0, x1, wt, b)
        y64, s, f, _ = reference(engine, g, x0, x1, wt, b, maxima)
        check(engine, y, y64, s, f, "spread/" + kind, m)


@pytest.mark.parametrize("m", [0, 11, 22])
@pytest.mark.parametrize("loose", [1, 10, 20])
@pytest.mark.parametrize("layout", ["window", "gather-balanced", "1x1"])
def test_loose_maxima(layout, loose, m):
    """amax0 up to 2^20 above the largest |x0| (the header allows upper bounds): the scale, and with it F, follow."""
    g = Geo(layout, 4, 6, 10, 40, 24, 48)
    x0, x1, wt, b = _spread_operands(g, "frames", m, seed=m + 7 * loose)
    amax0 = _amax(x0) * 2.0 ** loose
    y, maxima = run("f16x3", g, x0, x1, wt, b, amax0=amax0)
    y64, s, f, _ = reference("f16x3", g, x0, x1, wt, b, maxima)
    check("f16x3", y, y64, s, f, "loose", "%d/%d" % (loose, m))


# ------------------------------------------------------------------------------------------ exponent edges
EDGES = [-126, -110, -87, 100, 115, 116, 120, 127]


# K = 9 x 16 terms of 2^(xexp + wexp): past xexp + wexp = 118 the exact result itself leaves fp32
EDGE_PAIRS = [(x, wx) for x in EDGES for wx in (-40, 0, 40) if x + wx <= 118]

# weights at both ends too (128: up to FLT_MAX = (1 - 2^-24) 2^128); pairs such as (-87, -40) and (-70, -70) put every
# product and partial sum among the fp32 subnormals
WIDE_EDGES = [-126, -110, -87, -70, 100, 115, 120, 127]
W_EDGES = [-126, -100, -70, -40, 0, 40, 100, 128]
WIDE_PAIRS = [(x, wx) for x in WIDE_EDGES for wx in W_EDGES if x + wx <= 118 and (x, wx) not in EDGE_PAIRS]
WIDE_RUNS = ([("f16x3", lay) for lay in ("window", "window-balanced", "gather", "gather-balanced")]
             + [("tf32x3", lay) for lay in ("window", "window-balanced", "gather", "gather-balanced", "window-split2",
                                            "gather-split4")]
             + [("simt", lay) for lay in ("window", "gather")])


def _edge_case(engine, layout, xexp, wexp):
    """One launch with source maxima 2^xexp and weight maxima 2^wexp, the largest value of each at the top of its binade:
    the fp64 result is a finite fp32 number, and the output must be finite and within BAR S + F."""
    g = Geo(layout, 2, 5, 12, 8, 8, 40)
    gen = torch.Generator(device=DEV).manual_seed(xexp * 3 + wexp)
    x0 = (_rand((g.n * g.h * g.w, g.c0), gen).double() * 2.0 ** xexp).float()
    x1 = (_rand((g.n * g.h * g.w, g.c1), gen).double() * 2.0 ** (xexp - 3)).float()
    x0[0, 0] = 2.0 ** xexp * (1 - 2.0 ** -24)       # the top of the binade: the largest scaled value the exponent allows
    wt = (_rand((g.cout, g.c0 + g.c1, 3, 3), gen).double() * 2.0 ** (wexp - 1) * 2).float()
    wt[0, 0, 1, 1] = 2.0 ** (wexp - 1) * 2 * (1 - 2.0 ** -24)
    wt[1, 3, 0, 2] = -wt[0, 0, 1, 1]
    b = (_rand((g.cout,), gen).double() * 2.0 ** (xexp + wexp)).float()
    y, maxima = run(engine, g, x0, x1, wt, b)
    y64, s, f, _ = reference(engine, g, x0, x1, wt, b, maxima)
    assert bool((y64.abs() < FLT_MAX).all())
    check(engine, y, y64, s, f, "edges", "%d/%d" % (xexp, wexp))


@pytest.mark.parametrize("xexp,wexp", EDGE_PAIRS)
@pytest.mark.parametrize("layout", ["window", "window-balanced", "gather", "gather-balanced"])
def test_exponent_edges(layout, xexp, wexp):
    """Source maxima near both ends of fp32 (2^-126: most values subnormal) against weight maxima far from 1, on all
    three engines: wherever the fp64 result is a finite fp32 number, the output is finite and within BAR S + F.  The
    small pairs (2^-126 / 2^-110 against 2^-40) put f16x3's 2^-(e + e_w) below the float range: the whole-tile epilogue
    and the stream-K fix-up (balanced) then rescale the sums first."""
    for engine in ENGINES:
        _edge_case(engine, layout, xexp, wexp)


@pytest.mark.parametrize("xexp,wexp", WIDE_PAIRS)
@pytest.mark.parametrize("engine,layout", WIDE_RUNS, ids=["%s-%s" % r for r in WIDE_RUNS])
def test_exponent_edges_of_the_weights(engine, layout, xexp, wexp):
    """The same with weight maxima from 2^-126 to FLT_MAX and subnormal products, tf32x3 also split-K (2 and 4 splits).
    FLT_MAX weights round to Inf under a plain round-to-nearest tf32 split; the weight pack truncates those instead."""
    _edge_case(engine, layout, xexp, wexp)


@pytest.mark.parametrize("act", [ACT_NONE, ACT_LRELU])
@pytest.mark.parametrize("layout", ["window", "gather-balanced", "1x1"])
@pytest.mark.parametrize("engine", ENGINES)
def test_all_zero_sources_give_the_bias(engine, layout, act):
    """Maximum 0 (no scale to take): y = act(bias) exactly, with weights far from 1."""
    g = Geo(layout, 2, 5, 12, 40, 8, 40)
    gen = torch.Generator(device=DEV).manual_seed(5)
    x0 = torch.zeros(g.n * g.h * g.w, g.c0, device=DEV)
    x1 = torch.zeros(g.n * g.h * g.w, g.c1, device=DEV)
    wt = _rand((g.cout, g.c0 + g.c1, 3 if g.taps == 9 else 1, 3 if g.taps == 9 else 1), gen) * 2.0 ** -40
    b = _rand((g.cout,), gen)
    y, maxima = run(engine, g, x0, x1, wt, b, act=act)
    if engine == "f16x3":
        assert float(maxima[0]) == 0.0 and float(maxima[1]) == 0.0
    want = torch.where(b > 0, b, b * 0.0) if act == ACT_LRELU else b
    assert torch.equal(y, want.expand_as(y))


# ------------------------------------------------------------------------------------------ non-finite inputs
@pytest.mark.parametrize("layout", ["window", "window-balanced", "gather", "gather-balanced"])
@pytest.mark.parametrize("pad", [PAD_ZERO, PAD_REFLECT, PAD_REPLICATE])
@pytest.mark.parametrize("source", ["x0", "x1"])
@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
def test_non_finite_input_stays_in_its_halo(value, source, pad, layout):
    """One non-finite value at a corner pixel of frame 2 (63-pixel frames: tiles span two frames; balanced: stream-K cut
    tiles), under no activation, ELU and sigmoid: the non-finite outputs are the reference's (tensor cores: NaN also
    allowed where the pre-activation is non-finite), the rest of the batch meets its bar."""
    g = Geo(layout, 4, 7, 9, 40, 24, 48)
    gen = torch.Generator(device=DEV).manual_seed(11)
    hw = g.h * g.w
    x0 = _rand((g.n * hw, g.c0), gen)
    x1 = _rand((g.n * hw, g.c1), gen)
    wt = _rand((g.cout, g.c0 + g.c1, 3, 3), gen)
    b = _rand((g.cout,), gen)
    pix = 2 * hw + 0 * g.w + (g.w - 1)               # frame 2, y = 0, x = W - 1
    (x0 if source == "x0" else x1)[pix, 5] = float(value)
    for act, engine in ((act, engine) for act in (ACT_NONE, ACT_ELU, ACT_SIGMOID) for engine in ENGINES):
        y, maxima = run(engine, g, x0, x1, wt, b, pad=pad, act=act)
        if engine == "f16x3":                       # the library's maxima skip the non-finite value
            assert float(maxima[0]) == cr.finite_max(x0) and float(maxima[1]) == cr.finite_max(x1)
        y64, s, f, pre64 = reference(engine, g, x0, x1, wt, b, maxima, pad=pad, act=act)
        assert 0 < int((~torch.isfinite(pre64)).any(1).sum()) <= 9
        check(engine, y, y64, s, f, "non-finite/%d" % act, value, act=act, pre64=pre64)


# ------------------------------------------------------------------------------------------ decoder batch isolation
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_decoder_frames_are_isolated_from_a_corrupted_frame(value):
    """DepthWaveProgressiveDecoder, batch 4: one NaN or +Inf in frame 2's features leaves frames 0, 1 and 3 bit-identical
    to the clean batch (the dense row counts and so the schedules do not change; every operand scale skips the value)."""
    ch = synth.RESNET18_CH
    dense = kd.DepthWaveProgressiveDecoder(np.array(ch))
    synth.load_random(dense, seed=3)
    dense = dense.to(DEV).eval()
    feats = [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(20 + i))
             for i, s in enumerate(synth.kitti_feature_shapes(4, 96, 320, ch))]
    with torch.no_grad():
        clean = dense(feats)
        bad = [f.clone() for f in feats]
        bad[-1][2, 7, 1, 3] = float(value)
        hit = dense(bad)
    keep = torch.tensor([0, 1, 3], device=DEV)
    for s in range(4):
        a, c = clean[("disp", s)], hit[("disp", s)]
        assert torch.equal(a[keep], c[keep]), "disp %d: the clean frames changed" % s


# ------------------------------------------------------------------------------------------ backward
@pytest.fixture
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


# (name, c0, c1, cout, n, h, w, pad, taps, shift0); every data gradient has cin >= 32 and a reduction of >= 128 terms,
# so it runs on the tensor cores in f16x3
BWD_LAYERS = [
    ("reflect3x3", 32, 0, 48, 2, 9, 11, PAD_REFLECT, 9, 0),
    ("zero3x3_skip", 24, 16, 40, 2, 8, 12, PAD_ZERO, 9, 1),
    ("replicate3x3", 40, 0, 32, 2, 7, 10, PAD_REPLICATE, 9, 0),
    ("1x1", 64, 0, 128, 2, 8, 8, PAD_REFLECT, 1, 0),
]
ROW_PUSH = [1.0, 8.0, 12.0, 16.0, 20.0]      # per-pixel gain of x0: pre-activations of up to ~ +-20 sigma


def _backward_layer(layer, act, seed, gy_hook=None):
    """One train_native.conv layer, forward and backward, with x0 rows pushed by ROW_PUSH gains (one per pixel, in
    turn): saturated sigmoid rows and deep negative ELU rows make dz = dy y (1 - y) or dy (y + 1) span many decades.
    Returns the operands, the layer's y and the gradients."""
    name, c0, c1, cout, n, h, w, pad, taps, shift0 = layer
    gen = torch.Generator(device="cpu").manual_seed(seed)
    hs, ws = h >> shift0, w >> shift0
    x0 = torch.zeros(n * hs * ws, ops.pad4(c0))
    x0[:, :c0] = torch.randn(n * hs * ws, c0, generator=gen)
    x0[:, :c0] *= torch.tensor(ROW_PUSH)[torch.arange(n * hs * ws) % len(ROW_PUSH)][:, None]
    x1 = torch.randn(n, c1, h, w, generator=gen) if c1 else None
    k = 3 if taps == 9 else 1
    weight = torch.randn(cout, c0 + c1, k, k, generator=gen) / (k * k * (c0 + c1)) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1
    gy = torch.zeros(n * h * w, ops.pad4(cout))
    gy[:, :cout] = torch.randn(n * h * w, cout, generator=gen)
    if gy_hook is not None:
        gy_hook(gy, n, h, w)
    x0d = x0.to(DEV).requires_grad_(True)
    x1d = x1.to(DEV).requires_grad_(True) if x1 is not None else None
    wd, bd = weight.to(DEV).requires_grad_(True), bias.to(DEV).requires_grad_(True)
    amax0 = _amax(x0d.detach())
    y, _ = train_native.conv(x0d, amax0, x1d, wd, bd, n, h, w, taps=taps, pad=pad, act=act, shift0=shift0)
    y.backward(gy.to(DEV))
    return x0d, x1d, wd, bd, gy.to(DEV), y.detach()


@pytest.mark.parametrize("act", [ACT_SIGMOID, ACT_ELU], ids=["sigmoid", "elu"])
@pytest.mark.parametrize("layer", BWD_LAYERS, ids=[c[0] for c in BWD_LAYERS])
def test_backward_data_gradient_with_dz_over_decades(layer, act, _fp32_convs):
    """f16x3 data gradients (dx0, dx1: forward engine on dz, scaled by max |dz|) within conv_grad_ref.BARS S + F when
    dz spans decades; dW (3xTF32) and db stay within their plain bars."""
    name, c0, c1, cout, n, h, w, pad, taps, shift0 = layer
    x0d, x1d, wd, bd, gy, y = _backward_layer(layer, act, seed=len(name) + act)
    y64 = y[:, :cout].double()
    dact = y64 * (1 - y64) if act == ACT_SIGMOID else torch.where(y64 > 0, 1.0, y64 + 1)
    dz = gy[:, :cout].double() * dact
    nz = dz[dz != 0].abs()
    assert float(nz.max() / nz.min()) > 1e6                        # dz spans decades
    x1rows = x1d.detach().permute(0, 2, 3, 1).reshape(n * h * w, c1) if c1 else None
    ref = conv_grad_ref.conv_grads(x0d.detach()[:, :c0], c0, x1rows, c1, wd.detach(), dz, n, h, w, taps=taps, pad=pad,
                                   shift0=shift0)
    floor = conv_grad_ref.dgrad_floor(c0, c1, wd.detach(), dz.float(), n, h, w, cr.finite_max(dz.float()), taps=taps,
                                      pad=pad, shift0=shift0)
    bars = conv_grad_ref.BARS

    def held(what, got, want, s, f, bar):
        e_s, e_b = errors(got, want, s, floor=f, bar=bar, what=name + ":" + what)
        WORST.note(("f16x3" if what.startswith("dx") else what, "bwd/" + ("sigmoid" if act == ACT_SIGMOID else "elu"),
                    name + ":" + what), e_s, e_b)
        assert e_b <= 1.0, "%s %s: err / (BAR S + F) = %.3g (err / S = %.3g)" % (name, what, e_b, e_s)

    held("dx0", x0d.grad[:, :c0], *ref["x0"], floor["x0"], bars["dx0"])
    if c1:
        want, s = ref["x1"]
        held("dx1", x1d.grad.permute(0, 2, 3, 1).reshape(n * h * w, c1), want, s, floor["x1"], bars["dx1"])
    held("dW", wd.grad, *ref["w"], 0.0, bars["dW"])
    held("db", bd.grad, *ref["b"], 0.0, bars["db"])


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("layer", BWD_LAYERS[:2], ids=[c[0] for c in BWD_LAYERS[:2]])
def test_backward_frames_are_isolated_from_a_non_finite_gradient(layer, value, _fp32_convs):
    """A NaN or +-Inf in the upstream gradient at one pixel of frame 1: max |dz| skips it, so the data gradients of
    frame 0 keep their bits; frame 1's are non-finite only in that pixel's halo (3x3: at most 9 pixels of dx)."""
    name, c0, c1, cout, n, h, w, pad, taps, shift0 = layer
    pix = 1 * h * w + (h // 2) * w + w // 2

    def corrupt(gy, n, h, w):
        gy[pix, 3] = float(value)

    clean = _backward_layer(layer, ACT_ELU, seed=3)
    hit = _backward_layer(layer, ACT_ELU, seed=3, gy_hook=corrupt)
    r0 = (h >> shift0) * (w >> shift0)                 # rows of frame 0 in x0
    assert torch.equal(clean[0].grad[:r0], hit[0].grad[:r0])
    bad = ~torch.isfinite(hit[0].grad[r0:, :c0]).all(1)
    assert 0 < int(bad.sum()) <= 9
    if c1:
        assert torch.equal(clean[1].grad[0], hit[1].grad[0])
        assert 0 < int((~torch.isfinite(hit[1].grad[1])).any(0).sum()) <= 9


# ------------------------------------------------------------------------------------------ decoder batch isolation
def _kitti_pair(seed=3):
    ch = np.array(synth.RESNET18_CH)
    sparse = kd.SparseDepthWaveProgressiveDecoder(ch)
    synth.load_random(sparse, seed=seed, gains={".2.conv.": 4.0})
    dense = kd.DepthWaveProgressiveDecoder(ch)
    dense.load_state_dict(sparse.state_dict())
    feats = [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(20 + i))
             for i, s in enumerate(synth.kitti_feature_shapes(4, 96, 320, synth.RESNET18_CH))]
    return sparse.to(DEV).eval(), dense.to(DEV), feats


def _corrupt(feats, value):
    bad = [f.clone() for f in feats]
    bad[-1][2, 7, 1, 3] = float(value)
    return bad


KEEP = [0, 1, 3]


@pytest.mark.parametrize("value", ["nan", "inf"])
def test_training_step_feature_gradients_are_isolated_from_a_corrupted_frame(value, _fp32_convs):
    """One native training step of DepthWaveProgressiveDecoder (batch 4) with one NaN or +Inf in frame 2's features: the
    input-feature gradients of frames 0, 1 and 3 are bit-identical to the clean step's."""
    _, dense, feats = _kitti_pair()
    dense.train()

    def grads(fs):
        fd = [f.detach().clone().requires_grad_(True) for f in fs]
        out = dense(fd)
        g = torch.Generator(device="cpu").manual_seed(5)
        loss = 0
        for k in sorted(out, key=str):
            wgt = torch.randn(tuple(out[k].shape), generator=g).to(DEV)
            loss = loss + (out[k] * wgt).sum()
        loss.backward()
        return [f.grad for f in fd]

    clean, hit = grads(feats), grads(_corrupt(feats, value))
    for j, (a, b) in enumerate(zip(clean, hit)):
        assert a is not None and torch.equal(a[KEEP], b[KEEP]), "feature %d: the clean frames' gradients changed" % j


@pytest.mark.parametrize("value", ["nan", "inf"])
def test_sparse_decoder_frames_are_isolated_from_a_corrupted_frame(value):
    """SparseDepthWaveProgressiveDecoder (batch 4, thr 0.05) with one NaN or +Inf in frame 2's features: frames 0, 1 and
    3 keep their masks exactly and their outputs within the parity bar (their bits may move: balanced cuts follow the
    batch's total row count)."""
    sparse, _, feats = _kitti_pair()
    with torch.no_grad():
        clean = sparse(feats, 0.05)
        hit = sparse(_corrupt(feats, value), 0.05)
    checked = 0
    for k, a in clean.items():
        if not torch.is_tensor(a) or a.dim() == 0 or a.shape[0] != 4:
            continue
        b = hit[k]
        if a.dtype == torch.bool:
            assert torch.equal(a[KEEP], b[KEEP]), "%s: the clean frames' mask changed" % (k,)
        else:
            assert parity.rel_err(b[KEEP], a[KEEP]) <= PARITY_TOL, (k, parity.rel_err(b[KEEP], a[KEEP]))
        checked += 1
    assert checked >= 20
    assert [clean["total_ops_per_sample"][j] for j in KEEP] == [hit["total_ops_per_sample"][j] for j in KEEP]
