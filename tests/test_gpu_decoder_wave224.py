"""GPU: DecoderWave224 (NYUv2's 224-pixel wavelet decoder) on libwmd, and the KITTI dense decoder without skips.

Inference (no_grad) runs the native level engine; every float output is checked against the reference's outputs
(tests/golden/nyu224_tiny_dense.npz) or the CPU oracle (full size) at the 1e-4 relative bar.  ("disp", 1) is the
reference's floor division ll // 2: it may differ from the oracle by exactly 1.0 where the oracle's ll / 2 lies within
the bar of an integer - such floor ties are counted, printed and bounded.

Training with fp32 convolutions (allow_tf32 False) runs every convolution forward and backward on libwmd; the
gradients are checked against an fp64 run of the oracle as in test_gpu_native_training.py (tiny fixture directly,
DenseNet161 224x224 on the native forward's LeakyReLU kink sides).  ("disp", 1) has a zero gradient and is left out of
the comparison losses (torch itself has no derivative for floor division).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import haar
from oracle import nyu as onyu
from oracle import wave224
from wavelet_monodepth_b200 import _lib, kitti_decoders as kd, nyu_decoders as nd, synth, train_native

from helpers import REL_TOL, compare_outputs, key_str, kitti_features, load_golden, nyu_features, rel_err, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
MNV2_LIGHT_CH = [32, 24, 32, 64, 160]
GRAD_TOL = 1e-4
FULL_SIZE_TOL = 2e-5
MAX_FLIPS = 32


@pytest.fixture(autouse=True)
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _tiny(cls=nd.DecoderWave224, name="nyu224_tiny_dense"):
    want, meta = load_golden(name)
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    sd = seeded_params(mod, meta)
    mod.load_state_dict(sd, strict=False)
    return mod.to(DEV), sd, want, meta


def _full(ch, n, seed=11):
    mod = nd.DecoderWave224(enc_features=ch, decoder_width=0.5)
    sd = synth.load_random(mod, seed=seed)
    feats = synth.blocky_features(synth.nyu_feature_shapes(n, 224, 224, ch), seed=seed + 1)
    return mod.to(DEV), sd, feats


# ------------------------------------------------------------------------------------------ inference parity
def _ll1(want):
    """The oracle's LL at scale 1 (the input of ("disp", 1) = ll // 2), from its ("disp", 2) = ll2 / 4 and level-1 details."""
    ll2 = 4 * want["disp_2"]
    yh = torch.stack([want["wavelets_1_%s" % b] for b in ("LH", "HL", "HH")], 2)
    return haar.DWTInverse("haar", "zero")((ll2, [yh]))


def _check_parity(got, want, what):
    """want: key_str -> CPU tensor.  Returns (worst rel err of the float outputs, number of floor ties in ("disp", 1))."""
    got = {key_str(k): v.detach().cpu() for k, v in got.items()}
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    worst = 0.0
    for k, wv in want.items():
        assert tuple(got[k].shape) == tuple(wv.shape), (what, k)
        if k == "disp_1":
            continue
        e = rel_err(got[k], wv)
        worst = max(worst, e)
        assert e <= REL_TOL, (what, k, e)
    diff = got["disp_1"] - want["disp_1"]
    moved = diff != 0
    half = _ll1(want) / 2
    near = (half - half.round()).abs() <= REL_TOL * half.abs().max()
    assert torch.all(diff[moved].abs() == 1.0), (what, diff[moved].unique())
    assert torch.all(near[moved]), (what, "a ('disp', 1) element moved away from a floor tie")
    ties = int(moved.sum())
    print("%s: worst rel err %.3g, floor ties in ('disp', 1): %d of %d" % (what, worst, ties, moved.numel()))
    assert ties <= max(8, moved.numel() // 10000), (what, ties)
    return worst, ties


def test_tiny_no_grad_matches_reference_golden():
    mod, _, want, meta = _tiny()
    with torch.no_grad():
        got = mod.eval()(nyu_features(meta, DEV))
    _check_parity(got, {k: torch.from_numpy(v) for k, v in want.items()}, "nyu224 tiny")


def test_tiny_no_grad_runs_native_kernels_only():
    mod, _, _, meta = _tiny()
    feats = nyu_features(meta, DEV)
    before = _lib.launch_count()
    names = _kernel_names(lambda: mod.eval()(feats), grad=False)
    assert _lib.launch_count() - before >= 12
    assert any("conv_rows" in k for k in names) and any("head_conv3x3" in k for k in names)
    vendor = [k for k in names if "wmd::" not in k and any(v in k.lower() for v in _VENDOR)]
    assert not vendor, vendor[:5]


@pytest.mark.parametrize("ch", [synth.DENSENET161_CH, MNV2_LIGHT_CH], ids=["densenet161", "mobilenetv2_light"])
def test_full_size_224_batch8_vs_oracle(ch):
    mod, sd, feats = _full(list(ch), 8)
    with torch.no_grad():
        got = mod.eval()([f.to(DEV) for f in feats])
        want = {key_str(k): v for k, v in wave224.nyu224_dense_forward(sd, feats).items()}
    assert got[("disp", 0)].shape == (8, 1, 224, 224)
    _check_parity(got, want, "nyu224 %s 224x224 bs8" % ("d161" if ch[-1] == 2208 else "mnv2-light"))


def test_mobilenetv2_light_fine_levels_take_the_fma_engine():
    """up2 / up3 / up4 (cout 20, 10, 5) are below the tensor-core tiles: the fp32 FMA engine runs them."""
    mod, _, feats = _full(MNV2_LIGHT_CH, 1)
    names = _kernel_names(lambda: mod.eval()([f.to(DEV) for f in feats]), grad=False)
    assert sum("conv_rows_kernel" in k for k in names) >= 3
    assert any("conv_rows_tc_kernel" in k for k in names)


def test_depth_epilogue_is_the_clamped_division_of_disp0():
    """NYUv2/utils.py:215-229 at 224 (no resize): clamp(("disp", 0) / 100, 0.4, 10), fused into the last IDWT."""
    mod, _, _, meta = _tiny()
    feats = nyu_features(meta, DEV)
    mod.depth_epilogue = (100, 0.4, 10)
    with torch.no_grad():
        got = mod.eval()(feats)
    mod.depth_epilogue = None
    with torch.no_grad():
        plain = mod(feats)
    assert torch.equal(got[("depth", 0)], torch.clamp(got[("disp", 0)] / 100, 0.4, 10))
    assert ("depth", 0) not in plain
    for k, v in plain.items():
        assert torch.equal(got[k], v), k


# ------------------------------------------------------------------------------------------ training
def _loss(out, seed=5):
    """Fixed random weights on every output but ("disp", 1), whose gradient is zero by construction."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    total = 0
    for k in sorted(out, key=str):
        wgt = torch.randn(tuple(out[k].shape), generator=g, dtype=torch.float64)
        if k != ("disp", 1):
            total = total + (out[k].double() * wgt.to(out[k].device)).sum()
    return total


def _native_grads(mod, feats):
    fd = [f.to(DEV).requires_grad_(True) for f in feats]
    mod.zero_grad(set_to_none=True)
    _loss(mod(fd)).backward()
    return {k: p.grad for k, p in mod.named_parameters()}, [f.grad for f in fd]


def _errors(got, want):
    gp, gf = got
    wp, wf = want
    res = {k: (gp[k].double().cpu() - g).abs().max().item() / max(g.abs().max().item(), 1e-30)
           for k, g in wp.items() if g is not None}
    res.update({("feature", j): (a.double().cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
                for j, (a, b) in enumerate(zip(gf, wf)) if b is not None})
    return res


def test_tiny_gradients_vs_fp64_oracle():
    mod, sd, _, meta = _tiny()
    feats = nyu_features(meta)
    got = _native_grads(mod.train(), feats)
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double().clone().requires_grad_(True) for f in feats]
    _loss(wave224.nyu224_dense_forward(params, f64)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items()}, [f.grad for f in f64]))
    assert len(errs) == 20 + 5
    for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:5]:
        print("grad rel err", k, "%.3g" % e)
    for k, e in errs.items():
        assert e <= GRAD_TOL, (k, e)


def test_disp1_alone_has_zero_gradients():
    mod, _, _, meta = _tiny()
    fd = [f.to(DEV).requires_grad_(True) for f in nyu_features(meta)]
    out = mod.train()(fd)
    (out[("disp", 1)].double() * torch.randn_like(out[("disp", 1)].double())).sum().backward()
    for k, p in mod.named_parameters():
        if k.startswith(("up4.", "wave4.")):
            assert p.grad is None, k              # level 4 comes after ("disp", 1)
        else:
            assert p.grad is not None and not bool(p.grad.any()), k
    assert fd[0].grad is None
    for f in fd[1:]:
        assert f.grad is not None and not bool(f.grad.any())


def _capture_lrelu_sides(monkeypatch):
    """(N, C, H, W) masks of the positive outputs of every LeakyReLU convolution (up1..up4) of the native forward."""
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


def _up_pre(p, j, d, skip):
    x = torch.cat([F.interpolate(d, scale_factor=2, mode="nearest"), skip], 1)
    return onyu._conv3(x, *onyu._p(p, "up%d.convA" % j), "reflection")


def _lrelu(x, side):
    return torch.where(side, x, 0.2 * x)


def _nyu224_fp64(p, blocks, sides):
    """oracle.wave224.nyu224_dense_forward with the LeakyReLU sides of up1..up4 given."""
    out = {}
    d = onyu._conv3(blocks[-1], *onyu._p(p, "conv2"), "replicate")
    d = _lrelu(_up_pre(p, 1, d, blocks[-2]), sides[0])
    ll = 2 ** 4 * onyu._conv3(d, *onyu._p(p, "wave1_ll"), "replicate")
    out[("wavelets", 3, "LL")] = ll
    for j in range(1, 5):
        s = 4 - j
        if j > 1:
            d = _lrelu(_up_pre(p, j, d, blocks[-1 - j]), sides[j - 1])
        hc = 2 ** s * onyu._conv3(d, *onyu._p(p, "wave%d" % j), "zero").unsqueeze(1)
        for k, band in enumerate(("LH", "HL", "HH")):
            out[("wavelets", s, band)] = hc[:, :, k]
        ll = onyu._idwt(ll, hc)
        out[("disp", s)] = ll.detach() // 2 if s == 1 else ll / 2 ** s
    return out


def test_densenet161_224_full_size_gradients_vs_fp64(monkeypatch):
    ch = list(synth.DENSENET161_CH)
    mod, sd, feats = _full(ch, 2)
    sides = _capture_lrelu_sides(monkeypatch)
    got = _native_grads(mod.train(), feats)
    monkeypatch.undo()
    assert len(sides) == 4
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double().clone().requires_grad_(True) for f in feats]
    _loss(_nyu224_fp64(params, f64, sides)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items()}, [f.grad for f in f64]))
    assert len(errs) == 20 + 5
    for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:5]:
        print("full-size grad rel err", k, "%.3g" % e)
    for k, e in errs.items():
        assert e <= FULL_SIZE_TOL, (k, e)
    p, blocks, flips, total = {k: v.double() for k, v in sd.items()}, [f.double() for f in feats], 0, 0
    d = onyu._conv3(blocks[-1], *onyu._p(p, "conv2"), "replicate")
    for j in range(1, 5):
        pre = _up_pre(p, j, d, blocks[-1 - j])
        flips += int(((pre > 0) != sides[j - 1]).sum())
        total += pre.numel()
        d = F.leaky_relu(pre, 0.2)
    print("LeakyReLU inputs on the other side of the kink from fp64: %d of %d" % (flips, total))
    assert flips <= MAX_FLIPS


def test_backward_is_deterministic():
    mod, _, feats = _full(MNV2_LIGHT_CH, 2)
    mod.train()
    a = _native_grads(mod, feats)
    b = _native_grads(mod, feats)
    for k in a[0]:
        assert torch.equal(a[0][k], b[0][k]), k
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------ selection
_VENDOR = ("cudnn", "cublas", "xmma", "cutlass", "gemm", "convolve", "sm90_", "sm80_")
_WMD_CONV = ("conv_rows", "conv_wgrad", "act_bwd", "fold_src", "head_conv3x3")


def _kernel_names(step, grad=True):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.set_grad_enabled(grad):
            step()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _step(mod, feats):
    # ("disp", 1) stays out of the loss: the cuDNN path's floor division has no derivative in torch
    def run():
        mod.zero_grad(set_to_none=True)
        out = mod([f.to(DEV).requires_grad_(True) for f in feats])
        sum(out[("disp", s)].mean() for s in (0, 2, 3)).backward()
    return run


def test_native_step_launches_no_vendor_kernel():
    mod, _, _, meta = _tiny()
    names = _kernel_names(_step(mod.train(), nyu_features(meta)))
    assert any("conv_wgrad_kernel" in k for k in names)
    vendor = [k for k in names if "wmd::" not in k and any(v in k.lower() for v in _VENDOR)]
    assert not vendor, vendor[:5]


def test_tf32_allowed_keeps_the_cudnn_path():
    mod, _, _, meta = _tiny()
    torch.backends.cudnn.allow_tf32 = True
    names = _kernel_names(_step(mod.train(), nyu_features(meta)))
    assert not any(k in n for n in names for k in _WMD_CONV), [n for n in names if "wmd::" in n][:5]
    assert any("wmd::" not in n and any(v in n.lower() for v in _VENDOR) for n in names)


def test_depthwise_224_decoder_keeps_the_autograd_path():
    mod = nd.DecoderWave224(dw_waveconv=True, dw_upconv=True).to(DEV)
    feats = synth.blocky_features(synth.nyu_feature_shapes(1, 64, 64, [96, 96, 192, 384, 2208]), seed=1)
    names = _kernel_names(_step(mod.train(), feats))
    assert not any("conv_wgrad_kernel" in k for k in names)
    names = _kernel_names(lambda: mod.eval()([f.to(DEV) for f in feats]), grad=False)
    assert not any(k in n for n in names for k in _WMD_CONV)


# ------------------------------------------------------------------------------------------ KITTI without skips
def _kitti_noskip():
    want, meta = load_golden("kitti_tiny_dense_noskip")
    mod = kd.DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]), use_skips=False)
    mod.load_state_dict(seeded_params(mod, meta), strict=False)
    return mod.to(DEV).eval(), want, meta


def test_kitti_without_skips_no_grad_matches_reference_golden():
    mod, want, meta = _kitti_noskip()
    with torch.no_grad():
        got = mod(kitti_features(meta, DEV))
    worst = compare_outputs(got, want, "kitti dense without skips native")
    print("kitti without skips: worst rel err %.3g" % worst)


def test_kitti_without_skips_reads_no_skip_map():
    mod, _, meta = _kitti_noskip()
    feats = kitti_features(meta, DEV)
    nan = [torch.full_like(f, float("nan")) for f in feats[:4]] + [feats[4]]
    with torch.no_grad():
        a = mod(feats)
        b = mod(nan)
    for k in a:
        assert torch.equal(a[k], b[k]), k
