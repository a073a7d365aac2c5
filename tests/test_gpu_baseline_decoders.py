"""GPU: the baseline decoders on libwmd - monodepth2's DepthDecoder and DenseDepth's Decoder / Decoder224.

Inference (no_grad) runs the native engines; outputs are checked against the reference's (tests/golden/*_baseline.npz)
and, at full size, against an fp64 run of the oracle, at the 1e-4 relative bar.  Training with fp32 convolutions
(allow_tf32 False) runs every convolution forward and backward on libwmd; gradients are checked against an fp64 run of
the oracle as in test_gpu_native_training.py (DepthDecoder directly: ELU and sigmoid have no kink; Decoder on the
native forward's LeakyReLU kink sides).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import baseline
from oracle import nyu as onyu
from wavelet_monodepth_b200 import _lib, kitti_decoders as kd, nyu_decoders as nd, synth, train_native
from wavelet_monodepth_b200._lib import WmdError

from helpers import (REL_TOL, compare_outputs, key_str, kitti_features, kitti_variant, load_golden, nyu_features, rel_err,
                     seeded_params)

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAD_TOL = 1e-4
FULL_SIZE_TOL = 2e-5
MAX_FLIPS = 32
MNV2_CH = [32, 24, 32, 64, 1280]
MNV2_LIGHT_CH = [32, 24, 32, 64, 160]
_VENDOR = ("cudnn", "cublas", "xmma", "cutlass", "gemm", "convolve", "sm90_", "sm80_")
_WMD_CONV = ("conv_rows", "conv_wgrad", "act_bwd", "fold_src", "head_conv3x3", "disp_tail16")
NYU = {"Decoder": (nd.Decoder, "nyu_tiny_baseline", False), "Decoder224": (nd.Decoder224, "nyu224_tiny_baseline", True)}


@pytest.fixture(autouse=True)
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _kitti_tiny(variant="default"):
    want, meta = load_golden("kitti_tiny_baseline")
    kw, arrays = kitti_variant(want, meta, variant)
    mod = kd.DepthDecoder(np.array(meta["num_ch_enc"]), **kw)
    sd = seeded_params(mod, meta)
    mod.load_state_dict(sd)
    return mod.to(DEV), sd, arrays, meta, kw


def _nyu_tiny(name):
    cls, fixture, _ = NYU[name]
    want, meta = load_golden(fixture)
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    sd = seeded_params(mod, meta)
    mod.load_state_dict(sd)
    return mod.to(DEV), sd, want, meta


def _kernel_names(step, grad=True):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.set_grad_enabled(grad):
            step()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _vendor(names):
    return [k for k in names if "wmd::" not in k and any(v in k.lower() for v in _VENDOR)]


# ------------------------------------------------------------------------------------------ inference parity
@pytest.mark.parametrize("variant", ["default", "scales13", "noskip", "ch3"])
def test_kitti_tiny_no_grad_matches_reference_golden(variant):
    mod, _, want, meta, _ = _kitti_tiny(variant)
    with torch.no_grad():
        got = mod.eval()(kitti_features(meta, DEV))
    assert set(map(key_str, got)) == set(want)
    print("DepthDecoder %s tiny: worst rel err %.3g" % (variant, compare_outputs(got, want, variant)))
    assert mod.outputs is got


@pytest.mark.parametrize("name", sorted(NYU))
def test_nyu_tiny_no_grad_matches_reference_golden(name):
    mod, _, want, meta = _nyu_tiny(name)
    with torch.no_grad():
        got = mod.eval()(nyu_features(meta, DEV))
    print("%s tiny: worst rel err %.3g" % (name, compare_outputs(got, want, name)))


def _vs_fp64_oracle(got, want, what):
    assert set(got) == set(want), what
    worst = 0.0
    for k, v in want.items():
        assert tuple(got[k].shape) == tuple(v.shape), (what, k)
        e = rel_err(got[k], v)
        worst = max(worst, e)
        assert e <= REL_TOL, (what, k, e)
    print("%s: worst rel err vs fp64 oracle %.3g" % (what, worst))


@pytest.mark.parametrize("ch,n,height,width", [(synth.RESNET18_CH, 16, 192, 640), (synth.RESNET50_CH, 4, 320, 1024)],
                         ids=["r18_640x192_b16", "r50_1024x320_b4"])
def test_kitti_full_size_vs_oracle(ch, n, height, width):
    mod = kd.DepthDecoder(np.array(ch))
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.kitti_feature_shapes(n, height, width, ch), seed=12)
    with torch.no_grad():
        got = mod.to(DEV).eval()([f.to(DEV) for f in feats])
        p64 = {k: v.to(DEV, torch.float64) for k, v in sd.items()}
        want = baseline.kitti_baseline_forward(p64, [f.to(DEV, torch.float64) for f in feats])
    _vs_fp64_oracle(got, want, "DepthDecoder %dx%d x%d" % (width, height, n))


@pytest.mark.parametrize("name,ch,size", [
    ("Decoder", synth.DENSENET161_CH, (480, 640)), ("Decoder", MNV2_CH, (480, 640)),
    ("Decoder224", synth.DENSENET161_CH, (224, 224)), ("Decoder224", MNV2_LIGHT_CH, (224, 224))],
    ids=["decoder_d161_640x480", "decoder_mnv2_640x480", "decoder224_d161", "decoder224_mnv2light"])
def test_nyu_full_size_batch8_vs_oracle(name, ch, size):
    cls, _, extra = NYU[name]
    mod = cls(enc_features=list(ch), decoder_width=0.5)
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.nyu_feature_shapes(8, size[0], size[1], ch), seed=12)
    with torch.no_grad():
        got = mod.to(DEV).eval()([f.to(DEV) for f in feats])
        p64 = {k: v.to(DEV, torch.float64) for k, v in sd.items()}
        want = baseline.nyu_baseline_forward(p64, [f.to(DEV, torch.float64) for f in feats], extra_stage=extra)
    _vs_fp64_oracle(got, want, "%s %s %dx%d x8" % (name, ch[-1], size[1], size[0]))


# ------------------------------------------------------------------------------------------ native path properties
def test_no_grad_native_path_launches_no_vendor_kernel():
    mod, _, _, meta, _ = _kitti_tiny()
    feats = kitti_features(meta, DEV)
    names = _kernel_names(lambda: mod.eval()(feats), grad=False)
    assert any("disp_tail16_kernel" in k for k in names) and any("head_conv3x3" in k for k in names)
    assert not _vendor(names), _vendor(names)[:5]
    for name in NYU:
        mod, _, _, meta = _nyu_tiny(name)
        feats = nyu_features(meta, DEV)
        names = _kernel_names(lambda: mod.eval()(feats), grad=False)
        assert any("conv_rows" in k for k in names) and any("head_conv3x3" in k for k in names)
        assert not _vendor(names), (name, _vendor(names)[:5])


def test_finest_scale_bounds_the_levels_run():
    """scales=[1, 3]: level 0 feeds no output, so neither its convolutions nor the fused tail run."""
    mod, _, _, meta, _ = _kitti_tiny("scales13")
    names = _kernel_names(lambda: mod.eval()(kitti_features(meta, DEV)), grad=False)
    assert not any("disp_tail16" in k for k in names)
    assert sum("head_conv3x3" in k for k in names) == 2


def test_native_outputs_are_bit_identical_across_launches():
    mods = [_kitti_tiny()[0]] + [_nyu_tiny(name)[0] for name in sorted(NYU)]
    feats = [kitti_features(_kitti_tiny()[3], DEV)] + [nyu_features(_nyu_tiny(name)[3], DEV) for name in sorted(NYU)]
    with torch.no_grad():
        for mod, f in zip(mods, feats):
            a, b = mod.eval()(f), mod(f)
            for k in a:
                assert torch.equal(a[k], b[k]), (type(mod).__name__, k)


def test_empty_batch_returns_empty_outputs_with_the_right_keys():
    mod, _, want, meta, kw = _kitti_tiny("ch3")
    with torch.no_grad():
        out = mod.eval()([f[:0] for f in kitti_features(meta, DEV)])
    assert set(map(key_str, out)) == set(want)
    for k, v in out.items():
        assert v.shape == (0,) + want[key_str(k)].shape[1:] and v.is_cuda, k
    for name in sorted(NYU):
        mod, _, want, meta = _nyu_tiny(name)
        with torch.no_grad():
            out = mod.eval()([f[:0] for f in nyu_features(meta, DEV)])
        assert list(out) == [("disp", 0)] and out[("disp", 0)].shape == (0,) + want["disp_0"].shape[1:], name


def test_cpu_tensors_raise():
    mod, _, _, meta, _ = _kitti_tiny()
    with torch.no_grad(), pytest.raises(WmdError):
        mod.eval()(kitti_features(meta))
    for name in sorted(NYU):
        mod, _, _, meta = _nyu_tiny(name)
        with torch.no_grad(), pytest.raises(WmdError):
            mod.eval()(nyu_features(meta))


def test_weight_updates_repack():
    mod, _, _, meta, _ = _kitti_tiny()
    feats = kitti_features(meta, DEV)
    with torch.no_grad():
        a = mod.eval()(feats)[("disp", 0)].clone()
        mod.convs[("upconv", 0, 1)].conv.conv.weight.data.mul_(0.5)     # invisible to the version counter
        mod.invalidate_packs()
        b = mod(feats)[("disp", 0)]
    assert not torch.equal(a, b)


def test_more_than_four_output_channels_keep_the_cudnn_graph():
    mod = kd.DepthDecoder(np.array((8, 8, 16, 32, 64)), num_output_channels=5).to(DEV)
    feats = synth.blocky_features(synth.kitti_feature_shapes(1, 64, 96, (8, 8, 16, 32, 64)), seed=1)
    names = _kernel_names(lambda: mod.eval()([f.to(DEV) for f in feats]), grad=False)
    assert not any(k in n for n in names for k in _WMD_CONV)


# ------------------------------------------------------------------------------------------ training
def _loss(out, seed=5):
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


def _errors(got, want):
    gp, gf = got
    wp, wf = want
    res = {k: (gp[k].double().cpu() - g.cpu()).abs().max().item() / max(g.abs().max().item(), 1e-30)
           for k, g in wp.items() if g is not None}
    res.update({("feature", j): (a.double().cpu() - b.cpu()).abs().max().item() / max(b.abs().max().item(), 1e-30)
                for j, (a, b) in enumerate(zip(gf, wf)) if b is not None})
    return res


def _check_grads(mod, sd, feats, forward64, n_params, tol, what, device="cpu"):
    got = _native_grads(mod.train(), feats)
    params = {k: v.to(device, torch.float64).clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.to(device, torch.float64).clone().requires_grad_(True) for f in feats]
    _loss(forward64(params, f64)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items()}, [f.grad for f in f64]))
    assert len(errs) == n_params + 5, sorted(errs, key=str)
    for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:3]:
        print("%s grad rel err %s %.3g" % (what, k, e))
    for k, e in errs.items():
        assert e <= tol, (what, k, e)


@pytest.mark.parametrize("variant", ["default", "scales13", "noskip", "ch3"])
def test_kitti_tiny_gradients_vs_fp64_oracle(variant):
    mod, sd, _, meta, kw = _kitti_tiny(variant)
    scales, skips = kw.get("scales", range(4)), kw.get("use_skips", True)
    finest = min(scales)
    # levels finer than the finest scale feed no output: their parameters get no gradient
    used = {k: v for k, v in sd.items() if not any(k.startswith("decoder.%d." % s) for s in range(2 * (4 - finest) + 2, 10))}
    got = _native_grads(mod.train(), kitti_features(meta))
    for k, p in mod.named_parameters():
        assert (p.grad is None) == (k not in used), k
    params = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.double().clone().requires_grad_(True) for f in kitti_features(meta)]
    _loss(baseline.kitti_baseline_forward(params, f64, scales=scales, use_skips=skips)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items() if k in used}, [f.grad for f in f64]))
    for k, e in errs.items():
        assert e <= GRAD_TOL, (variant, k, e)
    print("DepthDecoder %s tiny: worst grad rel err %.3g" % (variant, max(errs.values())))


@pytest.mark.parametrize("name", sorted(NYU))
def test_nyu_tiny_gradients_vs_fp64_oracle(name):
    mod, sd, _, meta = _nyu_tiny(name)
    extra = NYU[name][2]
    _check_grads(mod, sd, nyu_features(meta), lambda p, f: baseline.nyu_baseline_forward(p, f, extra_stage=extra),
                 len(sd), GRAD_TOL, name + " tiny")


def test_kitti_r18_full_size_gradients_vs_fp64():
    ch = synth.RESNET18_CH
    mod = kd.DepthDecoder(np.array(ch))
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.kitti_feature_shapes(2, 192, 640, ch), seed=12)
    _check_grads(mod.to(DEV), sd, feats, baseline.kitti_baseline_forward, len(sd), FULL_SIZE_TOL, "DepthDecoder R18",
                 device=DEV)


def _capture_lrelu_sides(monkeypatch):
    sides = []
    conv = train_native.conv

    def spy(x0, amax0, x1, weight, bias, n, h, w, **kw):
        y, am = conv(x0, amax0, x1, weight, bias, n, h, w, **kw)
        if kw.get("act") == _lib.ACT_LRELU:
            c = int(weight.shape[0])
            sides.append((y.detach()[:, :c] > 0).reshape(n, h, w, c).permute(0, 3, 1, 2))
        return y, am

    monkeypatch.setattr(train_native, "conv", spy)
    return sides


def _pre(p, k, d, skip):
    x = torch.cat([F.interpolate(d, scale_factor=2, mode="nearest"), skip], 1)
    return F.conv2d(F.pad(x, (1, 1, 1, 1)), *onyu._p(p, "up%d.convA" % k))


def _decoder_fp64(p, blocks, sides):
    """oracle.baseline.nyu_baseline_forward (Decoder) with the LeakyReLU sides of up1..up4 given."""
    d = F.conv2d(F.pad(blocks[4], (1, 1, 1, 1)), *onyu._p(p, "conv2"))
    for k in range(1, 5):
        pre = _pre(p, k, d, blocks[4 - k])
        d = torch.where(sides[k - 1], pre, 0.2 * pre)
    return {("disp", 0): F.conv2d(F.pad(d, (1, 1, 1, 1)), p["conv3.weight"], p["conv3.bias"])}


def test_decoder_d161_full_size_gradients_vs_fp64(monkeypatch):
    ch = list(synth.DENSENET161_CH)
    mod = nd.Decoder(enc_features=ch, decoder_width=0.5)
    sd = synth.load_random(mod, seed=11)
    feats = synth.blocky_features(synth.nyu_feature_shapes(2, 480, 640, ch), seed=12)
    sides = _capture_lrelu_sides(monkeypatch)
    got = _native_grads(mod.to(DEV).train(), feats)
    monkeypatch.undo()
    assert len(sides) == 4
    params = {k: v.to(DEV, torch.float64).clone().requires_grad_(True) for k, v in sd.items()}
    f64 = [f.to(DEV, torch.float64).clone().requires_grad_(True) for f in feats]
    _loss(_decoder_fp64(params, f64, sides)).backward()
    errs = _errors(got, ({k: p.grad for k, p in params.items()}, [f.grad for f in f64]))
    assert len(errs) == len(sd) + 5
    for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:3]:
        print("Decoder D161 640x480 grad rel err %s %.3g" % (k, e))
    for k, e in errs.items():
        assert e <= FULL_SIZE_TOL, (k, e)
    with torch.no_grad():
        p = {k: v.detach() for k, v in params.items()}
        blocks = [f.detach() for f in f64]
        d = F.conv2d(F.pad(blocks[4], (1, 1, 1, 1)), *onyu._p(p, "conv2"))
        flips = total = 0
        for k in range(1, 5):
            pre = _pre(p, k, d, blocks[4 - k])
            flips += int(((pre > 0) != sides[k - 1]).sum())
            total += pre.numel()
            d = F.leaky_relu(pre, 0.2)
    print("LeakyReLU inputs on the other side of the kink from fp64: %d of %d" % (flips, total))
    assert flips <= MAX_FLIPS


def test_backward_is_deterministic_and_launches_no_vendor_kernel():
    cases = [_kitti_tiny()[:4:3]] + [_nyu_tiny(name)[:4:3] for name in sorted(NYU)]
    for mod, meta in cases:
        feats = kitti_features(meta) if isinstance(mod, kd.DepthDecoder) else nyu_features(meta)
        a = _native_grads(mod.train(), feats)
        b = _native_grads(mod, feats)
        for k in a[0]:
            assert torch.equal(a[0][k], b[0][k]), (type(mod).__name__, k)
        for x, y in zip(a[1], b[1]):
            assert torch.equal(x, y)
        names = _kernel_names(lambda: _native_grads(mod, feats))
        assert any("conv_wgrad_kernel" in k for k in names)
        assert not _vendor(names), (type(mod).__name__, _vendor(names)[:5])


def test_tf32_allowed_and_depthwise_keep_the_cudnn_path():
    torch.backends.cudnn.allow_tf32 = True
    cases = [_kitti_tiny()[:4:3]] + [_nyu_tiny(name)[:4:3] for name in sorted(NYU)]
    for mod, meta in cases:
        feats = kitti_features(meta) if isinstance(mod, kd.DepthDecoder) else nyu_features(meta)
        names = _kernel_names(lambda: _native_grads(mod.train(), feats))
        assert not any(k in n for n in names for k in _WMD_CONV), type(mod).__name__
        assert _vendor(names)
    torch.backends.cudnn.allow_tf32 = False
    for cls in (nd.Decoder, nd.Decoder224):
        mod = cls(is_depthwise=True).to(DEV)
        feats = synth.blocky_features(synth.nyu_feature_shapes(1, 64, 64, synth.DENSENET161_CH), seed=1)
        for grad in (True, False):
            step = (lambda: _native_grads(mod.train(), feats)) if grad else (lambda: mod.eval()([f.to(DEV) for f in feats]))
            names = _kernel_names(step, grad=grad)
            assert not any(k in n for n in names for k in _WMD_CONV), (cls.__name__, grad)
