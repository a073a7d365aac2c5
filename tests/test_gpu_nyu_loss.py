"""GPU: NYUv2's training loss on libwmd (nyu_loss.NyuDepthLoss, csrc/loss_nyu.cu).

* Fixture parity: on the cases of tests/golden/nyu_loss.npz the terms are within one float32 ulp of the oracle's (the
  fp64 sums differ only in order) and within 1e-6 of the reference's own float32 run, and the gradients equal the
  oracle's within 1 ulp, ties and NaN frames included.
* Edge shapes: 1 x k and k x 1 predictions, factors 1 to 8, a mismatched shape, a missing key, N = 0.
* Reproducibility: repeated calls and a CUDA-graph replay of the forward and backward give the same bits.
* End to end: a native DecoderWave step with NyuDepthLoss(disparity=True) and a DecoderWave224 step with the LL term
  supervised run under torch.use_deterministic_algorithms(True), give the same parameter gradients twice, and match
  the same step with torch's float32 loss chain (deterministic mode off) within 1e-5 of each tensor's largest element.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nyu_loss as onl
from wavelet_monodepth_b200 import nyu_decoders as nd, wavelets
from wavelet_monodepth_b200.nyu_loss import NyuDepthLoss

from helpers import load_golden, nyu_features, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
LL_KEY = ("wavelets", 3, "LL")


def ulps(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def run(loss, depth, preds, ll=None, grad=True):
    """-> (losses as floats, grads {key: numpy} of the leaf predictions, the device's yl_gt or None)"""
    outputs = {("disp", s): torch.from_numpy(p).to(DEV).requires_grad_(grad) for s, p in preds.items()}
    if ll is not None:
        outputs[LL_KEY] = torch.from_numpy(ll).to(DEV).requires_grad_(grad)
    d = torch.from_numpy(depth).to(DEV)
    total, losses = loss(outputs, d)
    if grad:
        total.backward()
    grads = {k: v.grad.cpu().numpy() for k, v in outputs.items() if v.grad is not None}
    yl = None
    if ll is not None:
        yl = wavelets.DWT(J=4)(10.0 / d if loss.disparity else d)[0].cpu().numpy()
    return {k: float(v.detach()) for k, v in losses.items()}, grads, yl


@pytest.mark.parametrize("name", list(onl.CASES))
def test_fixture_parity(name):
    fx, meta = load_golden("nyu_loss")
    n, H, W, disparity, use_wavelets, supervise_ll, kind = onl.CASES[name]
    depth, preds, ll = onl.case_inputs(name, meta["seeds"][name])
    loss = NyuDepthLoss(disparity=disparity, use_wavelets=use_wavelets, supervise_LL=supervise_ll)
    got, grads, yl = run(loss, depth, preds, ll)
    target = (10.0 / torch.from_numpy(depth)).numpy()[:, 0] if disparity else depth[:, 0]
    p = {s: v[:, 0] for s, v in preds.items()}
    want = onl.losses(p, target, None if ll is None else ll[:, 0], None if yl is None else yl[:, 0],
                      supervise_ll=supervise_ll)
    ref32 = dict(zip(meta["scalar_keys"][name], fx[name + "__f32_scalars"]))
    assert sorted(got) == sorted(want) == sorted(ref32)
    for k in want:
        assert np.isnan(got[k]) == np.isnan(want[k]) == np.isnan(ref32[k]), k
        if not np.isnan(want[k]):
            assert ulps(got[k], want[k]) <= 1.0, (k, got[k], want[k])
            assert abs(got[k] - ref32[k]) <= 1e-6 * abs(ref32[k]), (k, got[k], ref32[k])
    g = np.float32(0.1)
    for s in onl.SCALES:
        w = onl.grad(p[s], target, g)
        assert ulps(grads[("disp", s)][:, 0], w).max() <= 1.0, s
    if ll is not None:
        w = onl.grad(ll[:, 0], yl[:, 0], 1.0 / 16 if supervise_ll else 0.0)
        assert np.array_equal(grads[LL_KEY][:, 0], w)


def test_torch_sign_of_nan_is_zero_on_the_gpu():
    """The contract's sgn(NaN) = 0 is torch's: its CUDA L1 backward gives a NaN input a zero gradient."""
    x = torch.tensor([float("nan"), 2.0, -1.0], device=DEV, requires_grad=True)
    F.l1_loss(x, torch.zeros(3, device=DEV)).backward()
    assert torch.equal(x.grad, torch.tensor([0.0, 1.0 / 3, -1.0 / 3], device=DEV))


@pytest.mark.parametrize("H,W", [(1, 24), (24, 1), (8, 8), (16, 40), (40, 16)])
def test_edge_shapes_and_factors(H, W):
    rng = np.random.default_rng(H * 100 + W)
    depth = rng.uniform(10, 1000, (2, 1, H, W)).astype(np.float32)
    for s in onl.SCALES:
        if H % (1 << s) or W % (1 << s):
            continue
        pred = rng.uniform(10, 1000, (2, 1, H >> s, W >> s)).astype(np.float32)
        got, grads, _ = run(NyuDepthLoss(output_scales=(s,), loss_scales=(s,)), depth, {s: pred})
        want = onl.term(pred[:, 0], depth[:, 0])
        assert ulps(got["loss_depth/%d" % s], want) <= 1.0, (H, W, s)
        assert np.array_equal(grads[("disp", s)][:, 0], onl.grad(pred[:, 0], depth[:, 0], np.float32(0.1))), (H, W, s)


def test_argument_errors_and_empty_batches():
    loss = NyuDepthLoss()
    depth = torch.full((2, 1, 16, 24), 100.0, device=DEV)
    outs = {("disp", s): torch.full((2, 1, 16 >> s, 24 >> s), 90.0, device=DEV) for s in onl.SCALES}
    bad = dict(outs)
    bad[("disp", 2)] = torch.zeros(2, 1, 4, 5, device=DEV)
    with pytest.raises(ValueError):
        loss(bad, depth)
    missing = dict(outs)
    del missing[("disp", 3)]
    with pytest.raises(KeyError):
        loss(missing, depth)
    with pytest.raises(ValueError):
        NyuDepthLoss(loss_scales=(4,))
    empty = {k: v[:0].clone().requires_grad_(True) for k, v in outs.items()}
    total, losses = loss(empty, depth[:0])
    assert all(torch.isnan(v) for v in losses.values())
    total.backward()
    assert all(v.grad is not None and v.grad.shape == v.shape and v.grad.numel() == 0 for v in empty.values())
    with torch.no_grad():                                       # train.py's val()
        total, losses = loss(outs, depth)
    assert abs(float(losses["loss_depth/0"]) - 10.0) == 0.0 and float(total) == pytest.approx(4.0)


def _graph_case():
    depth, preds, ll = onl.case_inputs("w224_sLL", 7)
    outs = {("disp", s): torch.from_numpy(p).to(DEV).requires_grad_(True) for s, p in preds.items()}
    outs[LL_KEY] = torch.from_numpy(ll).to(DEV).requires_grad_(True)
    return NyuDepthLoss(use_wavelets=True, supervise_LL=True, disparity=True), outs, torch.from_numpy(depth).to(DEV)


def test_repeats_and_graph_replay_give_the_same_bits():
    loss, outs, depth = _graph_case()
    keys = sorted(outs, key=str)

    def step(o, d):
        total, losses = loss(o, d)
        grads = torch.autograd.grad(total, [o[k] for k in keys])
        return [losses[k] for k in sorted(losses)], grads

    first = step(outs, depth)
    for _ in range(3):
        again = step(outs, depth)
        assert all(torch.equal(a, b) for a, b in zip(first[0], again[0]))
        assert all(torch.equal(a, b) for a, b in zip(first[1], again[1]))
    # the graph's leaves are made, warmed up and captured on one side stream, so that no autograd node of theirs
    # belongs to the legacy stream, which a capture may not wait on
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in outs.items()}
        d = depth.clone()
        for _ in range(2):
            step(leaves, d)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        captured = step(leaves, d)
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(first[0], captured[0]))
        assert all(torch.equal(a, b) for a, b in zip(first[1], captured[1]))


# ------------------------------------------------------------------------------------------ end to end
def _torch_loss(outputs, depth, disparity, use_wavelets, supervise_ll):
    """train.py:279-327 in torch float32, the reference's chain"""
    depth_n = 10.0 / depth if disparity else depth
    total = 0
    for s in range(4):
        pred = F.interpolate(outputs[("disp", s)], scale_factor=2 ** s, mode="bilinear", align_corners=True)
        loss = 0.1 * F.l1_loss(pred, depth_n)
        total = total + loss
    if use_wavelets and LL_KEY in outputs:
        yl_gt = wavelets.DWT(J=4, wave="haar", mode="reflect")(depth_n)[0]
        l_ll = F.l1_loss(outputs[LL_KEY], yl_gt) / 2 ** 4
        if supervise_ll:
            total = total + l_ll
    return total


def _decoder(cls, golden):
    _, meta = load_golden(golden)
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    mod.load_state_dict(seeded_params(mod, meta), strict=False)
    return mod.to(DEV).train(), [f.to(DEV) for f in nyu_features(meta)]


def _step(mod, feats, depth, loss_fn):
    mod.zero_grad(set_to_none=True)
    out = mod(feats)
    loss_fn(out, depth).backward()
    return {k: p.grad.clone() for k, p in mod.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("cls,golden,opts", [
    (nd.DecoderWave, "nyu_tiny_dense", dict(disparity=True)),
    (nd.DecoderWave224, "nyu224_tiny_dense", dict(use_wavelets=True, supervise_LL=True)),
])
def test_native_decoder_step_is_deterministic_and_matches_torch_loss(cls, golden, opts):
    assert not torch.backends.cudnn.allow_tf32          # the native training step
    mod, feats = _decoder(cls, golden)
    # a target within 30 % of the decoder's own ("disp", 0), so that the signs of the differences vary: with a target
    # far from every prediction the loss's gradient is one constant per scale, whose detail coefficients cancel
    # exactly, and the detail heads' bias gradients are rounding noise of either loss
    with torch.no_grad():
        disp = mod(feats)[("disp", 0)].abs() + 0.05
    gen = torch.Generator(device="cpu").manual_seed(1)
    near = disp * (0.7 + 0.6 * torch.rand(disp.shape, generator=gen)).to(DEV)
    depth = 10.0 / near if opts.get("disparity") else near
    loss = NyuDepthLoss(**opts)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = _step(mod, feats, depth, lambda o, d: loss(o, d)[0])
        b = _step(mod, feats, depth, lambda o, d: loss(o, d)[0])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.are_deterministic_algorithms_enabled() == prev
    assert sorted(a) == sorted(b) and len(a) > 0
    for k in a:
        assert torch.equal(a[k], b[k]), k
    ref = _step(mod, feats, depth, lambda o, d: _torch_loss(o, d, opts.get("disparity", False),
                                                            opts.get("use_wavelets", False),
                                                            opts.get("supervise_LL", False)))
    assert sorted(ref) == sorted(a)
    for k in a:
        err = (a[k] - ref[k]).abs().max().item() / max(ref[k].abs().max().item(), 1e-30)
        assert err <= 1e-5, (k, err)
