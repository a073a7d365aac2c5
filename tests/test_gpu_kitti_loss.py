"""GPU: KITTI's depth-hints training loss on libwmd (kitti_loss.KittiDepthHintsLoss, csrc/loss_kitti.cu).

* Fixture parity: on the cases of tests/golden/kitti_hints_loss*.npz, each with the loss built from its own options
  (depth range, smoothness weight, loss scales) and cameras, the warped colours, color_depth_hint and both masks equal
  the contract-mode oracle's, the terms are within one float32 ulp (NaN where the oracle's is NaN: the one-pixel-thick
  scales' smoothness) and every gradient element within one float32 ulp of its scale's largest (the fp64 sums differ
  from the oracle's in order only).
* Per term: the case's weighted sum of every term back-propagated through ``losses``, against the oracle's gradient
  with the same grad_terms, at the same bars.
* Full size: R18 640x192 with 12 frames, the same bars; the mask pixels that differ from the fp64-mode oracle are
  counted and printed.
* Edge cases: N = 0, a missing key, wrong shapes and dtypes, a size not divisible by 8, a NaN disparity.
* Reproducibility: repeated calls give the same bits; the noise is the reference's draw after torch.manual_seed.
* End to end: native DepthWaveProgressiveDecoder and DepthDecoder steps with the loss run under
  torch.use_deterministic_algorithms(True) and give the same parameter gradients twice.  At the decoders' own
  disparities the native gradient is no farther from a float64 torch restatement of the reference's chain than the
  float32 restatement is (both on the contract's masks; the float32 chain's own mask flips are counted and printed).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import kitti_loss as okl
from wavelet_monodepth_b200 import _lib, kitti_decoders as kd, synth
from wavelet_monodepth_b200.kitti_loss import KittiDepthHintsLoss

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIX = okl.load_fixture(os.path.join(os.path.dirname(__file__), "golden"))
R18 = (64, 64, 128, 256, 512)


def ulps(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def to_dev(inp, disps, case, grad=True):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)          # noqa: E731
    inputs = {("color", 0, 0): t(inp["target"]), ("color", "s", 0): t(inp["source"]), ("K", 0): t(inp["K"]),
              ("inv_K", 0): t(inp["inv_K"]), "stereo_T": t(inp["stereo_T"]), "depth_hint": t(inp["depth_hint"]),
              "depth_hint_mask": t(inp["depth_hint_mask"])}
    for s in case["scales"]:
        if s:
            inputs[("color", 0, s)] = t(inp["colors"][s])
    outputs = {("disp", s): t(disps[s]).requires_grad_(grad) for s in case["scales"]}
    return inputs, outputs


def native(case, inp, disps, seed, weights=None):
    """the loss built from the case's options; the gradient of the total, or of sum_k weights[k] losses[k] (the keys in
    okl.term_keys order)"""
    inputs, outputs = to_dev(inp, disps, case)
    loss = KittiDepthHintsLoss(case["H"], case["W"], case["scales"], case["loss_scales"], **okl.options(case))
    torch.manual_seed(seed)
    total, losses = loss(inputs, outputs)
    if weights is None:
        total.backward()
    else:
        sum(float(w) * losses[k] for w, k in zip(weights, okl.term_keys(case["loss_scales"]))).backward()
    grads = {s: outputs[("disp", s)].grad.cpu().numpy().astype(np.float64) for s in case["loss_scales"]}
    return losses, outputs, grads


def check_against_oracle(case, inp, disps, seed, weights=None):
    """the bars above; returns the oracle's result and the worst (term ulp, gradient ulp of the scale's largest)"""
    noise = okl.draw_noise(seed, inp, case["loss_scales"])
    o = okl.run(inp, disps, noise, case["scales"], case["loss_scales"], mode="contract", grad_terms=weights,
                **okl.options(case))
    losses, outputs, grads = native(case, inp, disps, seed, weights)
    worst = [0.0, 0.0]
    for k, v in losses.items():
        got, want = float(v.detach()), float(o[k])
        assert np.isnan(got) == np.isnan(want), (k, got, want)
        if not np.isnan(want):
            worst[0] = max(worst[0], float(ulps(got, want)))
            assert ulps(got, want) <= 1, (k, got, want)
    assert np.array_equal(outputs[("color_depth_hint", "s", 0)].cpu().numpy(), o["color_depth_hint"].astype(np.float32))
    for s in case["loss_scales"]:
        assert np.array_equal(outputs[("color", "s", s)].cpu().numpy(), o["warped"][s].astype(np.float32), equal_nan=True)
        for key in ("identity_selection", "depth_hint_pixels"):
            got = outputs["%s/%d" % (key, s)].cpu().numpy()[:, 0]
            assert np.array_equal(got, o[key][s]), (key, s, int((got != o[key][s]).sum()))
        want = o["grad"][s]
        assert np.isfinite(want).all() and np.isfinite(grads[s]).all(), (s, int((~np.isfinite(grads[s])).sum()))
        scale = np.float32(np.abs(want).max())
        err = np.abs(grads[s] - want).max() / (float(scale) * 2.0 ** -24)
        worst[1] = max(worst[1], float(err))
        assert err <= 1, (s, err)
    return o, worst


def _case(name):
    case = okl.CASES[name]
    seed = int(FIX["%s/seed" % name])
    return case, seed, okl.make_inputs(case, seed)


@pytest.mark.parametrize("name", [str(c) for c in FIX["cases"]])
def test_fixture_parity(name):
    case, seed, (inp, disps) = _case(name)
    _, worst = check_against_oracle(case, inp, disps, seed)
    print("\n%s: worst term %.3g ulp, worst gradient %.3g ulp of its scale's largest" % (name, *worst))


@pytest.mark.parametrize("name", [str(c) for c in FIX["cases"]])
def test_weighted_terms(name):
    """every term with its own weight (FIX's weights: distinct per term and scale, some negative): the backward reads
    each reproj_loss/s, depth_hint_loss/s and loss/s coefficient of grad_terms where the oracle does"""
    case, seed, (inp, disps) = _case(name)
    w = FIX["%s/weights" % name]
    _, worst = check_against_oracle(case, inp, disps, seed, weights=w)
    print("\n%s weighted: worst term %.3g ulp, worst gradient %.3g ulp of its scale's largest" % (name, *worst))


def test_full_size_r18_640x192_x12():
    case = dict(N=12, H=192, W=640, scales=okl.SCALES, loss_scales=okl.SCALES)
    inp, disps = okl.make_inputs(case, 77)
    o, _ = check_against_oracle(case, inp, disps, 77)
    o64 = okl.run(inp, disps, okl.draw_noise(77, inp, case["loss_scales"]), mode="fp64", grads=False)
    flips = {s: int((o["identity_selection"][s] != o64["identity_selection"][s]).sum()
                    + (o["depth_hint_pixels"][s] != o64["depth_hint_pixels"][s]).sum()) for s in case["loss_scales"]}
    print("\nmask pixels that differ from the fp64-mode oracle, per scale (of %d): %s" % (12 * 192 * 640, flips))


def test_nan_disparity_follows_the_contract():
    case = dict(okl.CASES["special"])
    inp, disps = okl.make_inputs(case, 5)
    disps[2][0, 0, 3, 4] = np.nan
    noise = okl.draw_noise(5, inp, case["loss_scales"])
    o = okl.run(inp, disps, noise, mode="contract")
    losses, outputs, grads = native(case, inp, disps, 5)
    for k, v in losses.items():
        assert np.isnan(float(v)) == np.isnan(float(o[k])), k
        if not np.isnan(float(o[k])):
            assert ulps(float(v), float(o[k])) <= 1, k
    for key in ("identity_selection", "depth_hint_pixels"):
        assert np.array_equal(outputs["%s/2" % key].cpu().numpy()[:, 0], o[key][2])
    assert np.array_equal(np.isnan(grads[2]), np.isnan(o["grad"][2]))


def test_edge_cases():
    case = dict(N=2, H=64, W=96, scales=okl.SCALES, loss_scales=okl.SCALES)
    inp, disps = okl.make_inputs(case, 3)
    loss = KittiDepthHintsLoss(64, 96)
    inputs, outputs = to_dev(inp, disps, case)
    # N = 0: runs, the reprojection and hint terms are 0, the smoothness means are NaN as torch's are
    z_in = {k: v[:0] for k, v in inputs.items()}
    z_out = {k: v[:0].detach().requires_grad_() for k, v in outputs.items()}
    total, losses = loss(z_in, z_out)
    total.backward()
    assert float(losses["reproj_loss/0"]) == 0.0 and np.isnan(float(total))
    assert z_out[("disp", 0)].grad.shape == (0, 1, 64, 96)
    for key in (("color", "s", 0), "depth_hint", ("K", 0), ("color", 0, 3)):
        bad = dict(inputs)
        del bad[key]
        with pytest.raises(KeyError):
            loss(bad, dict(outputs))
    bad_out = dict(outputs)
    del bad_out[("disp", 1)]
    with pytest.raises(KeyError):
        loss(inputs, bad_out)
    with pytest.raises(ValueError):
        loss(inputs, {**outputs, ("disp", 1): outputs[("disp", 2)]})
    with pytest.raises(ValueError):
        loss(dict(inputs, depth_hint=inputs["depth_hint"][:, :, :-1]), dict(outputs))
    with pytest.raises(_lib.WmdError):
        loss(dict(inputs, stereo_T=inputs["stereo_T"].double()), dict(outputs))
    with pytest.raises(_lib.WmdError):
        loss(dict(inputs, depth_hint=inputs["depth_hint"].cpu()), dict(outputs))
    with pytest.raises(ValueError):
        KittiDepthHintsLoss(100, 96)
    with pytest.raises(ValueError):
        KittiDepthHintsLoss(64, 92)


def test_repeatable_and_the_reference_noise():
    case = okl.CASES["r96x320"]
    inp, disps = okl.make_inputs(case, 11)
    runs = [native(case, inp, disps, 11) for _ in range(2)]
    for k in runs[0][0]:
        assert float(runs[0][0][k]) == float(runs[1][0][k]), k
    for s in case["loss_scales"]:
        assert np.array_equal(runs[0][2][s], runs[1][2][s])
    # the loss draws torch.randn((N, 1, H, W)) per loss scale from the CPU generator: the same stream as the reference
    torch.manual_seed(11)
    KittiDepthHintsLoss(96, 320)(*to_dev(inp, disps, case, grad=False))
    after = torch.randn(3)
    torch.manual_seed(11)
    for _ in case["loss_scales"]:
        torch.randn((2, 1, 96, 320))
    assert torch.equal(after, torch.randn(3))


# ------------------------------------------------------------------------------------------ end to end
def torch_chain(inputs, outputs, scales, loss_scales, H, W, min_depth=0.1, max_depth=100.0, smooth_w=1e-3,
                contract_masks=False):
    """the reference's generate_images_pred + compute_losses_hints for the stereo depth-hints configuration, restated
    with torch ops in the inputs' dtype.  Where outputs also holds the native loss's masks ("identity_selection/s",
    "depth_hint_pixels/s"), the pixels where the chain's own argmin differs from them are counted, and with
    contract_masks the chain uses them,
    so that a comparison measures the float32 arithmetic and not the decisions it flips."""
    def ssim(x, y):
        x, y = F.pad(x, (1, 1, 1, 1), mode="reflect"), F.pad(y, (1, 1, 1, 1), mode="reflect")
        mx, my = F.avg_pool2d(x, 3, 1), F.avg_pool2d(y, 3, 1)
        sx, sy = F.avg_pool2d(x * x, 3, 1) - mx ** 2, F.avg_pool2d(y * y, 3, 1) - my ** 2
        sxy = F.avg_pool2d(x * y, 3, 1) - mx * my
        n = (2 * mx * my + 0.01 ** 2) * (2 * sxy + 0.03 ** 2)
        d = (mx ** 2 + my ** 2 + 0.01 ** 2) * (sx + sy + 0.03 ** 2)
        return torch.clamp((1 - n / d) / 2, 0, 1)

    def reproj(p, t):
        return 0.85 * ssim(p, t).mean(1, True) + 0.15 * (t - p).abs().mean(1, True)

    N, dt = inputs[("color", 0, 0)].shape[0], inputs[("color", 0, 0)].dtype
    ys, xs = torch.meshgrid(torch.arange(H, device=DEV, dtype=dt), torch.arange(W, device=DEV, dtype=dt), indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(H * W, device=DEV, dtype=dt)], 0)[None].repeat(N, 1, 1)
    ones = torch.ones(N, 1, H * W, device=DEV, dtype=dt)
    P = torch.matmul(inputs[("K", 0)], inputs["stereo_T"])[:, :3, :]

    def warp(depth):
        cam = depth.view(N, 1, -1) * torch.matmul(inputs[("inv_K", 0)][:, :3, :3], pix)
        q = torch.matmul(P, torch.cat([cam, ones], 1))
        g = (q[:, :2] / (q[:, 2:3] + 1e-7)).view(N, 2, H, W).permute(0, 2, 3, 1).clone()
        g[..., 0] /= W - 1
        g[..., 1] /= H - 1
        return F.grid_sample(inputs[("color", "s", 0)], (g - 0.5) * 2, padding_mode="border", align_corners=False)

    tgt = inputs[("color", 0, 0)]
    hl = reproj(warp(inputs["depth_hint"]), tgt) + 1000 * (1 - inputs["depth_hint_mask"])
    total, flips = 0, []
    for s in loss_scales:
        disp = outputs[("disp", s)]
        up = F.interpolate(disp, [H, W], mode="bilinear", align_corners=False)
        depth = 1 / (1 / max_depth + (1 / min_depth - 1 / max_depth) * up)
        r = reproj(warp(depth), tgt)
        ident = reproj(inputs[("color", "s", 0)], tgt) + torch.randn(N, 1, H, W).to(DEV) * 0.00001
        k = torch.argmin(torch.cat([r, ident, hl], 1), 1, keepdim=True)
        rm, hm = (k != 1).float(), (k == 2).float()
        if "identity_selection/%d" % s in outputs:
            rm_c, hm_c = 1 - outputs["identity_selection/%d" % s], outputs["depth_hint_pixels/%d" % s]
            flips.append(int((rm != rm_c).sum() + (hm != hm_c).sum()))
            if contract_masks:
                rm, hm = rm_c, hm_c
        loss = (r * rm).sum() / (rm.sum() + 1e-7)
        loss = loss + (torch.log((inputs["depth_hint"] - depth).abs() + 1) * inputs["depth_hint_mask"] * hm).sum() \
            / (hm.sum() + 1e-7)
        nd = disp / (disp.mean(2, True).mean(3, True) + 1e-7)
        img = inputs[("color", 0, s)]
        gx = (nd[:, :, :, :-1] - nd[:, :, :, 1:]).abs() * torch.exp(-2 * (img[:, :, :, :-1] - img[:, :, :, 1:]).abs().mean(1, True))
        gy = (nd[:, :, :-1] - nd[:, :, 1:]).abs() * torch.exp(-2 * (img[:, :, :-1] - img[:, :, 1:]).abs().mean(1, True))
        total = total + loss + smooth_w * (gx.mean() + gy.mean()) / 2 ** s
    return total / len(scales), flips


def _decoder(make, n, H, W):
    torch.backends.cudnn.allow_tf32 = False
    mod = make()
    synth.load_random(mod, seed=1)
    mod = mod.to(DEV).train()
    feats = [f.to(DEV) for f in synth.blocky_features(synth.kitti_feature_shapes(n, H, W, R18), seed=2)]
    return mod, feats


def _inputs(n, H, W, seed=5, dtype=torch.float32):
    case = dict(N=n, H=H, W=W, scales=okl.SCALES, loss_scales=okl.SCALES)
    inp, _ = okl.make_inputs(case, seed)
    inputs, _ = to_dev(inp, {s: np.zeros((n, 1, H >> s, W >> s), np.float32) for s in okl.SCALES}, case, grad=False)
    return {k: v.to(dtype) for k, v in inputs.items()}


def _native_step(make, n=4, H=192, W=640, seed=5):
    mod, feats = _decoder(make, n, H, W)
    out = mod(feats)
    torch.manual_seed(seed)
    total, _ = KittiDepthHintsLoss(H, W)(_inputs(n, H, W, seed), out)
    mod.zero_grad()
    total.backward()
    return {k: p.grad.detach().clone() for k, p in mod.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("make", [lambda: kd.DepthWaveProgressiveDecoder(np.array(R18)),
                                  lambda: kd.DepthDecoder(np.array(R18))], ids=["wave", "baseline"])
def test_end_to_end_step(make):
    """a native decoder step with the loss is deterministic; at the decoder's own disparities, the native gradient is
    no farther from the float64 chain's than the float32 torch chain's is (both use the contract's masks, so that the
    comparison measures arithmetic; the float32 chain's own mask flips are counted and printed)"""
    torch.use_deterministic_algorithms(True)
    try:
        a = _native_step(make)
        b = _native_step(make)
    finally:
        torch.use_deterministic_algorithms(False)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    n, H, W, seed = 4, 192, 640, 5
    mod, feats = _decoder(make, n, H, W)
    with torch.no_grad():
        out = {k: v.detach() for k, v in mod(feats).items() if k[0] == "disp"}
    grads = {}
    for tag, dt in (("native", torch.float32), ("f32", torch.float32), ("f64", torch.float64)):
        disps = {k: v.to(dt).clone().requires_grad_() for k, v in out.items()}
        torch.manual_seed(seed)
        if tag == "native":
            total, _ = KittiDepthHintsLoss(H, W)(_inputs(n, H, W, seed), disps)
            masks = {k: v for k, v in disps.items() if isinstance(k, str)}
        else:
            total, flips = torch_chain(_inputs(n, H, W, seed, dt), dict(disps, **{k: v.to(dt) for k, v in masks.items()}),
                                       okl.SCALES, okl.SCALES, H, W, contract_masks=True)
            if tag == "f32":
                print("\nfloat32 torch chain's mask pixels that differ from the contract's, per scale: %s" % flips)
        total.backward()
        assert all(disps[("disp", s)].grad is not None for s in okl.SCALES), (tag, [s for s in okl.SCALES if disps[("disp", s)].grad is None], sorted(map(str, disps)))
        grads[tag] = {s: disps[("disp", s)].grad.double() for s in okl.SCALES}
    for s in okl.SCALES:
        ref = grads["f64"][s]
        scale = float(ref.abs().max())
        e_nat = float((grads["native"][s] - ref).abs().max()) / scale
        e_32 = float((grads["f32"][s] - ref).abs().max()) / scale
        print("scale %d: native %.3g, float32 chain %.3g of the largest float64 gradient" % (s, e_nat, e_32))
        assert e_nat <= max(e_32, 2.0 ** -22), (s, e_nat, e_32)
