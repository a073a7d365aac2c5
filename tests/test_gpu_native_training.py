"""GPU: the native training step of the dense wavelet decoders (train_native.py, csrc/conv_bwd.cu).

Per layer, the backward kernels are checked element by element against the fp64 adjoint of the conv contract
(tests/conv_grad_ref.py, torch autograd through tests/conv_ref.py) given the layer's own saved output y: dz = dy act'(y)
is formed in fp64 from the kernel's y, and |got - want| <= bar x S for dx0, dx1, dW and db, S the magnitude sum of the
element's terms.  Operands are mixed-sign, or same-sign (x, W, dy >= 0), which exposes a one-signed rounding bias.

Measured worst err / S over all cases, mixed- and same-sign, on one H100 80GB HBM3 (132 SMs, 700 W power limit):
    dW  (wgrad, 3xTF32 mma.sync, 32-pixel epochs)   9.5e-7
    dx0 (forward engine f16x3 + fold)               8.5e-6
    dx1 (skip columns of the fold)                  3.9e-6
    db  (fixed-order fp64 column sums)              1.2e-6 (measured with the earlier fp32 sums)
Each quantity's bar (BARS) is 2.3-2.6x its worst.

The whole decoders' parameter and input-feature gradients (allow_tf32 False) are compared with an fp64 CPU run of the
oracle: the tiny fixtures directly, KITTI R18 640x192 and NYU DenseNet161 640x480 (2 frames each) taking the native
forward's LeakyReLU sides (see "full size" below; measured worst 6.4e-6 of each tensor's largest element, bar 2e-5); the native step is deterministic, launches no cuDNN / cuBLAS kernel, and with TF32 allowed the cuDNN path runs.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_grad_ref
from oracle import kitti as okitti
from oracle import nyu as onyu
from wavelet_monodepth_b200 import _lib, kitti_decoders as kd, nyu_decoders as nd, ops, synth, train_native

from helpers import kitti_features, load_golden, nyu_features, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
BARS = conv_grad_ref.BARS

ACTS = {"none": _lib.ACT_NONE, "elu": _lib.ACT_ELU, "lrelu": _lib.ACT_LRELU, "sigmoid": _lib.ACT_SIGMOID}
PADS = {"zero": _lib.PAD_ZERO, "reflect": _lib.PAD_REFLECT, "replicate": _lib.PAD_REPLICATE}

# (name, c0, c1, cout, n, h, w, taps, pad, act, shift0)
CASES = [
    ("pad_zero", 32, 0, 32, 2, 9, 11, 9, "zero", "elu", 0),
    ("pad_reflect", 32, 0, 32, 2, 9, 11, 9, "reflect", "elu", 0),
    ("pad_replicate", 32, 0, 32, 2, 9, 11, 9, "replicate", "lrelu", 0),
    ("thin_h1", 16, 0, 32, 2, 1, 7, 9, "replicate", "elu", 0),
    ("thin_w1_zero", 16, 0, 32, 1, 5, 1, 9, "zero", "none", 0),
    ("thin_2x2_reflect", 16, 0, 32, 3, 2, 2, 9, "reflect", "elu", 0),
    ("odd_width", 24, 0, 40, 2, 6, 13, 9, "reflect", "lrelu", 0),
    ("shift_skip", 32, 20, 32, 2, 10, 14, 9, "reflect", "elu", 1),
    ("shift_skip_thin", 8, 12, 16, 2, 2, 6, 9, "reflect", "elu", 1),
    ("taps1", 64, 0, 64, 2, 8, 8, 1, "reflect", "lrelu", 0),
    ("taps1_cout3", 33, 0, 3, 2, 7, 9, 1, "zero", "sigmoid", 0),
    ("cin13", 13, 0, 20, 2, 7, 9, 9, "reflect", "elu", 0),
    ("cin33_cout70", 33, 0, 70, 2, 6, 7, 9, "reflect", "none", 0),
    ("cin65_cout130", 65, 0, 130, 1, 6, 6, 9, "replicate", "elu", 0),
    ("cin129_skip", 129, 7, 64, 1, 4, 6, 9, "reflect", "lrelu", 1),
    ("cout1", 32, 0, 1, 2, 8, 10, 9, "replicate", "none", 0),
    ("cout3", 32, 0, 3, 2, 8, 10, 9, "zero", "none", 0),
    ("cout6_sigmoid", 64, 0, 6, 2, 8, 10, 9, "reflect", "sigmoid", 0),
    # few output tiles over many rows: the weight gradient splits its pixel reduction across CTAs (DepthDecoder's
    # dispconv(0) at full resolution reaches that path only at production sizes otherwise)
    ("cout1_split_rows", 16, 0, 1, 2, 96, 320, 9, "reflect", "none", 0),
    ("cout6_split_rows", 16, 0, 6, 2, 96, 320, 9, "zero", "elu", 0),
    ("cout1_sigmoid_split_rows", 16, 0, 1, 2, 96, 320, 9, "reflect", "sigmoid", 0),
    ("below_one_chunk", 16, 0, 32, 1, 3, 5, 9, "reflect", "elu", 0),
    ("long_reduction", 64, 0, 64, 4, 96, 100, 9, "reflect", "elu", 0),
    ("kitti_r50_level1_upconv1", 32, 64, 32, 8, 160, 512, 9, "reflect", "elu", 1),
    ("nyu_conv2", 2208, 0, 1104, 8, 15, 20, 9, "replicate", "none", 0),
    # NYU Decoder's up3 convA at 640x480 x8: a whole-tile reduction of 1200 32-pixel chunks, whose fp32 chunk sums
    # drifted past the dW bar in the launch check of the Decoder's training step
    ("nyu_decoder_up3_conva", 552, 192, 276, 8, 60, 80, 9, "zero", "lrelu", 1),
]


def _operands(c0, c1, cout, n, h, w, shift0, same_sign, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)

    def r(*shape):
        t = torch.randn(*shape, generator=g)
        return t.abs() if same_sign else t

    hs, ws = h >> shift0, w >> shift0
    x0 = torch.zeros(n * hs * ws, ops.pad4(c0))
    x0[:, :c0] = r(n * hs * ws, c0)
    x1 = r(n, c1, h, w) if c1 else None
    taps_k = 3
    weight = r(cout, c0 + c1, taps_k, taps_k) / (taps_k * (c0 + c1)) ** 0.5
    bias = r(cout) * 0.1
    gy = torch.zeros(n * h * w, ops.pad4(cout))
    gy[:, :cout] = r(n * h * w, cout)
    return x0, x1, weight, bias, gy


def _check(name, got, want, s, bar):
    got = got.double().cpu()
    want, s = want.cpu(), s.cpu()
    excess = ((got - want).abs() - bar * s).max().item()
    worst = ((got - want).abs() / s.clamp_min(1e-300)).max().item()
    print("worst err/S", name, "%.3g" % worst)
    assert excess <= 0.0, "%s: worst err/S %.3g over bar %.1g" % (name, worst, bar)
    return worst


@pytest.mark.parametrize("same_sign", [False, True], ids=["mixed", "same"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_layer_gradients_vs_fp64(case, same_sign):
    name, c0, c1, cout, n, h, w, taps, pad, act, shift0 = case
    x0, x1, weight, bias, gy = _operands(c0, c1, cout, n, h, w, shift0, same_sign, seed=len(name) * 7 + same_sign)
    if taps == 1:
        weight = weight[:, :, 1:2, 1:2].contiguous()
    x0d, gyd = x0.to(DEV).requires_grad_(True), gy.to(DEV)
    x1d = x1.to(DEV).requires_grad_(True) if x1 is not None else None
    wd, bd = weight.to(DEV).requires_grad_(True), bias.to(DEV).requires_grad_(True)
    amax0 = torch.zeros(1, device=DEV)
    ops.amax_rows(x0d.detach(), amax0)
    y, _ = train_native.conv(x0d, amax0, x1d, wd, bd, n, h, w, taps=taps, pad=PADS[pad], act=ACTS[act],
                             act_param=0.1, shift0=shift0)
    y.backward(gyd)
    # fp64 reference, given the layer's own y
    y64 = y.detach()[:, :cout].double()
    dact = {"none": torch.ones_like(y64), "elu": torch.where(y64 > 0, 1.0, y64 + 1), "lrelu": torch.where(y64 > 0, 1.0, 0.1),
            "sigmoid": y64 * (1 - y64)}[act]
    dz = gyd[:, :cout].double() * dact
    x1rows = x1d.detach().permute(0, 2, 3, 1).reshape(n * h * w, c1) if x1 is not None else None
    ref = conv_grad_ref.conv_grads(x0d.detach()[:, :c0], c0, x1rows, c1, wd.detach(), dz, n, h, w, taps=taps,
                                   pad=PADS[pad], shift0=shift0)
    _check("dW", wd.grad, *ref["w"], BARS["dW"])
    _check("db", bd.grad, *ref["b"], BARS["db"])
    _check("dx0", x0d.grad[:, :c0], *ref["x0"], BARS["dx0"])
    assert torch.all(x0d.grad[:, c0:] == 0)
    if x1 is not None:
        want, s = ref["x1"]
        _check("dx1", x1d.grad, want.reshape(n, h, w, c1).permute(0, 3, 1, 2), s.reshape(n, h, w, c1).permute(0, 3, 1, 2), BARS["dx1"])


@pytest.mark.parametrize("rows,cout,spread", [(8 * 240 * 320, 1, 0.0), (8 * 240 * 320, 3, 1.0), (1000, 1, 1.0),
                                              (64 * 1024 + 7, 40, 1.0)])
def test_bias_gradient_of_many_same_sign_rows(rows, cout, spread):
    """db over the rows of NYU's Decoder's last convolution (cout 1, 8 frames of 240 x 320) under a mean loss, where
    every dz is the same 1 / rows, and over same-sign rows of several sizes.  Summed in fp32 (a per-thread chain, then
    up to 1024 block partials in block order) db drifted by 1.0e-5 of the sum, 3.4x BARS['db'] (the launch check of
    the Decoder's training step found it); summed in fp64 and rounded once it is within one fp32 rounding of the sum."""
    g = torch.Generator(device="cpu").manual_seed(rows + cout)
    y = torch.randn((rows, cout), generator=g).to(DEV)
    dy = ((1.0 + spread * torch.rand((rows, cout), generator=g)) / rows).to(DEV)
    dz, db = ops.act_backward(y, dy, cout, _lib.ACT_NONE)
    assert torch.equal(dz[:, :cout], dy)
    want = dy.double().sum(0)
    err = float(((db.double() - want).abs() / want).max())
    assert err <= 2.0 ** -23, (rows, cout, err)
    assert err <= BARS["db"]


# ------------------------------------------------------------------------------------------ whole decoders
def _kitti_module(meta, sd):
    mod = kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]))
    mod.load_state_dict(sd, strict=False)
    return mod.to(DEV).train()


def _nyu_module(meta, sd):
    mod = nd.DecoderWave(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    mod.load_state_dict(sd, strict=False)
    return mod.to(DEV).train()


def _loss(out, seed=5):
    """A sum over every output with fixed random weights, so that every element has its own gradient."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    total = 0
    for k in sorted(out, key=str):
        wgt = torch.randn(tuple(out[k].shape), generator=g, dtype=torch.float64)
        total = total + (out[k].double() * wgt.to(out[k].device)).sum()
    return total


def _native_grads(mod, feats):
    fd = [f.to(DEV).requires_grad_(True) for f in feats]
    mod.zero_grad(set_to_none=True)
    _loss(mod(fd)).backward()
    return {k: p.grad for k, p in mod.named_parameters()}, [f.grad for f in fd]


def _oracle_grads(forward, sd, feats):
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double().clone().requires_grad_(True) for f in feats]
    _loss(forward(params, f64)).backward()
    return {k: p.grad for k, p in params.items()}, [f.grad for f in f64]


def _compare(got, want, tol):
    gp, gf = got
    wp, wf = want
    checked = 0
    for k, g in wp.items():
        if g is None or k not in gp:
            continue
        err = (gp[k].double().cpu() - g).abs().max().item() / max(g.abs().max().item(), 1e-30)
        print("grad rel err", k, "%.3g" % err)
        assert err <= tol, (k, err)
        checked += 1
    for j, (a, b) in enumerate(zip(gf, wf)):
        if b is None:
            continue
        assert a is not None, j
        err = (a.double().cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
        assert err <= tol, ("feature", j, err)
    return checked


@pytest.fixture(autouse=True)
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


GRAD_TOL = 1e-4


def test_kitti_decoder_gradients_vs_fp64_oracle():
    _, meta = load_golden("kitti_tiny_dense")
    sd = seeded_params(kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"])), meta)
    feats = kitti_features(meta)
    got = _native_grads(_kitti_module(meta, sd), feats)
    assert _compare(got, _oracle_grads(okitti.dense_forward, sd, feats), GRAD_TOL) >= 30


def test_nyu_decoder_gradients_vs_fp64_oracle():
    _, meta = load_golden("nyu_tiny_dense")
    sd = seeded_params(nd.DecoderWave(enc_features=list(meta["enc_features"]), decoder_width=0.5), meta)
    feats = nyu_features(meta)
    got = _native_grads(_nyu_module(meta, sd), feats)
    assert _compare(got, _oracle_grads(onyu.dense_forward, sd, feats), GRAD_TOL) >= 14


def _errors(got, want):
    gp, gf = got
    wp, wf = want
    res = {k: (gp[k].double().cpu() - g).abs().max().item() / max(g.abs().max().item(), 1e-30)
           for k, g in wp.items() if g is not None}
    res.update({("feature", j): (a.double().cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
                for j, (a, b) in enumerate(zip(gf, wf)) if b is not None})
    return res


# ------------------------------------------------------------------------------------------ full size
# The fp64 function's gradient jumps where a LeakyReLU input changes sign.  An fp32 forward within its rounding bound can
# leave a handful of elements of millions on the other side of that kink from fp64: each such element changes its pixel's dz
# by 0.9 dy, an error of the size of one element's whole contribution (measured on the R18 step below: 4 flipped of 7.4
# million LeakyReLU inputs move the level-3 head's weight gradient by 7e-3 of its largest element, while every layer's
# backward on that step's real operands is within 1e-5 of fp64; cuDNN's fp32 forward, with a smaller rounding bound,
# flips fewer).  So at full size the fp64 reference takes the kink sides the native forward
# took, which checks the whole backward; the number of flipped elements is checked on its own.
def _capture_lrelu_sides(monkeypatch):
    """Record, for every LeakyReLU convolution of the native forward, the (N, C, H, W) mask of positive outputs."""
    sides = []
    conv = train_native.conv

    def spy(x0, amax0, x1, weight, bias, n, h, w, **kw):
        y, am = conv(x0, amax0, x1, weight, bias, n, h, w, **kw)
        if kw.get("act") == _lib.ACT_LRELU:
            c = int(weight.shape[0])
            sides.append((y.detach()[:, :c] > 0).reshape(n, h, w, c).permute(0, 3, 1, 2).cpu())
        return y, am

    monkeypatch.setattr(train_native, "conv", spy)
    return sides


def _lrelu(x, slope, side):
    return torch.where(side, x, slope * x)


def _kitti_fp64(p, feats, sides):
    """oracle.kitti.dense_forward with the LeakyReLU sides given (one [ll |] pos | neg mask per level)."""
    out, x, yl = {}, feats[-1], None
    for lvl, i in enumerate(range(4, 0, -1)):
        x = okitti._conv_block(x, *okitti._block(p, okitti.slot(i, "upconv0")))
        x = okitti._conv_block(torch.cat([okitti._up2(x), feats[i - 1]], 1), *okitti._block(p, okitti.slot(i, "upconv1")))
        off, res = 0, {}
        for name in (["ll"] if i == 4 else []) + ["pos", "neg"]:
            w1, b1, w2, b2 = okitti._head(p, okitti.slot(i, name))
            c = w1.shape[0]
            t = _lrelu(F.conv2d(x, w1, b1), 0.1, sides[lvl][:, off:off + c])
            res[name] = torch.sigmoid(okitti._conv3_reflect(t, w2, b2))
            off += c
        if i == 4:
            yl = 2 ** i * res["ll"]
        yh = 2 ** (i - 1) * res["pos"].unsqueeze(1) - 2 ** (i - 1) * res["neg"].unsqueeze(1)
        out[("wavelets", i - 1, "LL")] = yl
        for k, band in enumerate(("LH", "HL", "HH")):
            out[("wavelets", i - 1, band)] = yh[:, :, k]
        yl = okitti._idwt(yl, yh)
        out[("disp", i - 1)] = torch.clamp(yl / 2 ** (i - 1), 0, 1)
    return out


def _nyu_fp64(p, blocks, sides):
    """oracle.nyu.dense_forward with the LeakyReLU sides of up1..up3 given."""
    out = {}

    def up(name, x, skip, side):
        x = torch.cat([F.interpolate(x, scale_factor=2, mode="nearest"), skip], 1)
        return _lrelu(onyu._conv3(x, *onyu._p(p, name + ".convA"), "reflection"), 0.2, side)

    d = up("up1", onyu._conv3(blocks[-1], *onyu._p(p, "conv2"), "replicate"), blocks[-2], sides[0])
    ll = 2 ** 3 * onyu._conv3(d, *onyu._p(p, "wave1_ll"), "replicate")
    out[("disp", 3)] = ll / 2 ** 3
    out[("wavelets", 2, "LL")] = ll
    for s, scale in enumerate((2, 1, 0)):
        if s:
            d = up("up%d" % (s + 1), d, blocks[-2 - s], sides[s])
        hc = 2 ** scale * onyu._conv3(d, *onyu._p(p, "wave%d" % (s + 1)), "zero").unsqueeze(1)
        for k, band in enumerate(("LH", "HL", "HH")):
            out[("wavelets", scale, band)] = hc[:, :, k]
        ll = onyu._idwt(ll, hc)
        out[("disp", scale)] = ll / 2 ** scale
    return out


FULL_SIZE_TOL = 2e-5
MAX_FLIPS = 32          # measured 4 (KITTI R18) and 10 (NYU D161) of 7.4 and 9.3 million


def _full_size_check(monkeypatch, mod, sd, feats, forward64):
    """Native gradients against fp64 taking the native forward's kink sides; returns those sides."""
    sides = _capture_lrelu_sides(monkeypatch)
    got = _native_grads(mod.to(DEV).train(), feats)
    monkeypatch.undo()
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double().clone().requires_grad_(True) for f in feats]
    _loss(forward64(params, f64, sides)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items()}, [f.grad for f in f64]))
    assert len(errs) >= 14
    for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:5]:
        print("full-size grad rel err", k, "%.3g" % e)
    for k, e in errs.items():
        assert e <= FULL_SIZE_TOL, (k, e)
    return sides


def test_kitti_r18_full_size_gradients_vs_fp64(monkeypatch):
    ch = [64, 64, 128, 256, 512]
    mod = kd.DepthWaveProgressiveDecoder(np.array(ch))
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.kitti_feature_shapes(2, 192, 640, ch), seed=12)
    sides = _full_size_check(monkeypatch, mod, sd, feats, _kitti_fp64)
    p, x, flips = {k: v.double() for k, v in sd.items()}, feats[-1].double(), 0
    for lvl, i in enumerate(range(4, 0, -1)):
        x = okitti._conv_block(x, *okitti._block(p, okitti.slot(i, "upconv0")))
        x = okitti._conv_block(torch.cat([okitti._up2(x), feats[i - 1].double()], 1), *okitti._block(p, okitti.slot(i, "upconv1")))
        heads = [okitti._head(p, okitti.slot(i, nm)) for nm in (["ll"] if i == 4 else []) + ["pos", "neg"]]
        pre = F.conv2d(x, torch.cat([hd[0] for hd in heads]), torch.cat([hd[1] for hd in heads]))
        flips += int(((pre > 0) != sides[lvl]).sum())
    print("LeakyReLU inputs on the other side of the kink from fp64:", flips)
    assert flips <= MAX_FLIPS


def test_nyu_d161_full_size_gradients_vs_fp64(monkeypatch):
    ch = [96, 96, 192, 384, 2208]
    mod = nd.DecoderWave(enc_features=ch, decoder_width=0.5)
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.nyu_feature_shapes(2, 480, 640, ch), seed=12)
    sides = _full_size_check(monkeypatch, mod, sd, feats, _nyu_fp64)
    p, blocks, flips = {k: v.double() for k, v in sd.items()}, [f.double() for f in feats], 0
    d = onyu._conv3(blocks[-1], *onyu._p(p, "conv2"), "replicate")
    for s in range(3):
        x = torch.cat([F.interpolate(d, scale_factor=2, mode="nearest"), blocks[-2 - s]], 1)
        pre = onyu._conv3(x, *onyu._p(p, "up%d.convA" % (s + 1)), "reflection")
        flips += int(((pre > 0) != sides[s]).sum())
        d = F.leaky_relu(pre, 0.2)
    print("LeakyReLU inputs on the other side of the kink from fp64:", flips)
    assert flips <= MAX_FLIPS


def test_kitti_decoder_without_skips_matches_the_cudnn_path():
    _, meta = load_golden("kitti_tiny_dense")
    mod = kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]), use_skips=False)
    synth.load_random(mod, seed=4)
    mod = mod.to(DEV).train()
    feats = kitti_features(meta)
    native = _native_grads(mod, feats)
    fd = [f.to(DEV).requires_grad_(True) for f in feats]
    mod.zero_grad(set_to_none=True)
    _loss(mod._autograd_forward(fd)).backward()
    for k, p in mod.named_parameters():
        err = (native[0][k] - p.grad).abs().max().item() / p.grad.abs().max().item()
        assert err <= 1e-4, (k, err)
    assert all(g is None for g in native[1][:4]) and native[1][4] is not None


def test_backward_is_deterministic():
    _, meta = load_golden("kitti_tiny_dense")
    sd = seeded_params(kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"])), meta)
    mod = _kitti_module(meta, sd)
    feats = synth.blocky_features(synth.kitti_feature_shapes(4, 96, 320, meta["num_ch_enc"]), seed=3)
    a = _native_grads(mod, feats)
    b = _native_grads(mod, feats)
    for k in a[0]:
        assert torch.equal(a[0][k], b[0][k]), k
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------ selection
_VENDOR = ("cudnn", "cublas", "xmma", "cutlass", "gemm", "convolve", "sm90_", "sm80_")


def _kernel_names(step):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _step(mod, feats):
    def run():
        mod.zero_grad(set_to_none=True)
        out = mod([f.to(DEV).requires_grad_(True) for f in feats])
        sum(out[("disp", s)].mean() for s in range(4)).backward()
    return run


def test_native_step_launches_no_vendor_kernel():
    _, meta = load_golden("kitti_tiny_dense")
    sd = seeded_params(kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"])), meta)
    names = _kernel_names(_step(_kitti_module(meta, sd), kitti_features(meta)))
    assert any("conv_wgrad_kernel" in k for k in names)
    vendor = [k for k in names if "wmd::" not in k and any(v in k.lower() for v in _VENDOR)]
    assert not vendor, vendor[:5]
    _, meta = load_golden("nyu_tiny_dense")
    sd = seeded_params(nd.DecoderWave(enc_features=list(meta["enc_features"]), decoder_width=0.5), meta)
    names = _kernel_names(_step(_nyu_module(meta, sd), nyu_features(meta)))
    assert any("conv_wgrad_kernel" in k for k in names)
    vendor = [k for k in names if "wmd::" not in k and any(v in k.lower() for v in _VENDOR)]
    assert not vendor, vendor[:5]


def test_tf32_allowed_keeps_the_cudnn_path():
    _, meta = load_golden("kitti_tiny_dense")
    sd = seeded_params(kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"])), meta)
    mod = _kitti_module(meta, sd)
    torch.backends.cudnn.allow_tf32 = True
    names = _kernel_names(_step(mod, kitti_features(meta)))
    assert not any(k in n for n in names for k in ("conv_wgrad_kernel", "act_bwd_kernel", "fold_src0_kernel"))
    # the convolutions ran on the vendor library; the only libwmd kernels are the IDWT and its adjoint (DWT)
    assert any("wmd::" not in n and any(v in n.lower() for v in _VENDOR) for n in names)
    assert {n for n in names if "wmd::" in n} <= {n for n in names if "idwt" in n.lower() or "dwt" in n.lower()}


def test_depthwise_nyu_decoder_keeps_the_autograd_path():
    mod = nd.DecoderWave(dw_waveconv=True, dw_upconv=True).to(DEV).train()
    feats = synth.blocky_features(synth.nyu_feature_shapes(1, 64, 64, [96, 96, 192, 384, 2208]), seed=1)
    names = _kernel_names(_step(mod, feats))
    assert not any("conv_wgrad_kernel" in k for k in names)


# ------------------------------------------------------------------------------------------ training
def test_sgd_steps_track_the_fp64_trajectory():
    _, meta = load_golden("kitti_tiny_dense")
    sd = seeded_params(kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"])), meta)
    mod = _kitti_module(meta, sd)
    feats = kitti_features(meta)
    fd = [f.to(DEV) for f in feats]
    g = torch.Generator(device="cpu").manual_seed(9)
    with torch.no_grad():
        shapes = {s: tuple(v.shape) for (_, s), v in ((k, v) for k, v in mod(fd).items() if k[0] == "disp")}
    targets = {s: 0.5 * torch.rand(shapes[s], generator=g) for s in range(4)}

    def loss_of(out):
        return sum(((out[("disp", s)].double() - targets[s].to(out[("disp", s)].device).double()) ** 2).mean()
                   for s in range(4))

    lr = 0.005
    opt = torch.optim.SGD(mod.parameters(), lr=lr)
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double() for f in feats]
    got, want = [], []
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        loss = loss_of(mod(fd))
        loss.backward()
        opt.step()
        got.append(loss.item())
        ref = loss_of(okitti.dense_forward(params, f64))
        grads = torch.autograd.grad(ref, list(params.values()), allow_unused=True)
        with torch.no_grad():
            for p, gr in zip(params.values(), grads):
                if gr is not None:
                    p -= lr * gr
        want.append(ref.item())
    assert want[-1] < want[0]
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-4 * abs(b), (got, want)
    print("loss trajectory", got, want)
