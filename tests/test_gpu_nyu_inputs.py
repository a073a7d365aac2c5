"""GPU: NYUv2's training inputs on libwmd.  NyuInputs' {"image", "depth"} equals the reference's transform (the digests
of tests/golden/nyu_inputs_*.npz) in two launches per call, and oracle.nyu_inputs on every permutation x flip x gamma
at both sizes and both filters.  One item alone gives the bits it gets in a batch, the same batch gives the same bits
twice, an empty batch launches nothing, and the batch drives a native decoder step with NyuDepthLoss."""
import numpy as np
import pytest
import torch

from oracle import nyu_inputs as oni
from wavelet_monodepth_b200 import _lib, synth
from wavelet_monodepth_b200 import nyu_inputs as ni

import nyu_inputs_cases as nic

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MODES = [(False, "bicubic"), (True, "bicubic"), (False, "nearest"), (True, "nearest")]
MODE_IDS = ["640-bicubic", "224-bicubic", "640-nearest", "224-nearest"]


def run(items, is_224=False, resample="bicubic"):
    out = ni.NyuInputs(is_224, resample)(ni.collate(items), DEV)
    torch.cuda.synchronize()
    return out


def host(out, n):
    return {k: v[n].cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("name", nic.CASES)
def test_reference_digests_in_two_launches(name):
    fx = nic.load(name)
    cfg = fx["config"]
    fn = ni.NyuInputs(cfg["is_224"], cfg["resample"])
    batch = ni.collate(nic.items(fx))
    fn(batch, DEV)                                            # tables uploaded once, outside the count
    torch.cuda.synchronize()
    before = _lib.launch_count()
    out = fn(batch, DEV)
    torch.cuda.synchronize()
    assert _lib.launch_count() - before == 2
    assert nic.mismatches(fx, lambda n: host(out, n)) == []
    (ih, iw), (dh, dw) = ni.sizes(cfg["is_224"])
    assert out["image"].shape == (len(fx["view"]), 3, ih, iw) and out["depth"].shape == (len(fx["view"]), 1, dh, dw)


@pytest.mark.parametrize("is_224,resample", MODES, ids=MODE_IDS)
def test_every_permutation_flip_and_gamma(is_224, resample):
    """36 items: the six permutations x flip x gamma 0.8 / 1.0 / 1.25, plus two without swap or gamma"""
    its = []
    for p in range(6):
        for flip in (False, True):
            for gamma in (0.8, 1.0, 1.25):
                seed = 7 + len(its) % 5
                its.append({"image": oni.synthetic_image(seed), "depth": oni.synthetic_depth(seed), "flip": flip,
                            "perm": p, "gamma": gamma})
    for flip in (False, True):
        its.append({"image": oni.synthetic_image(3), "depth": oni.synthetic_depth(3), "flip": flip, "perm": -1,
                    "gamma": None})
    out = run(its, is_224, resample)
    for n, it in enumerate(its):
        exp = oni.expected(it["image"], it["depth"], it["flip"], it["perm"], it["gamma"], is_224, resample)
        got = host(out, n)
        for k in ("image", "depth"):
            assert got[k].dtype == np.float32 and np.array_equal(got[k], exp[k]), (n, k, it["flip"], it["perm"],
                                                                                   it["gamma"])


def test_one_item_alone_and_repeated_batches():
    fx = nic.load("640_bicubic")
    its = nic.items(fx)
    a, b = run(its), run(its)
    for k in ("image", "depth"):
        assert torch.equal(a[k], b[k]), k
    for n in (0, 3, len(its) - 1):
        alone = run(its[n:n + 1])
        for k in ("image", "depth"):
            assert torch.equal(a[k][n:n + 1], alone[k]), (n, k)


def test_empty_batch_launches_nothing():
    for is_224 in (False, True):
        before = _lib.launch_count()
        out = ni.NyuInputs(is_224)(ni.collate([]), DEV)
        assert _lib.launch_count() == before
        (ih, iw), (dh, dw) = ni.sizes(is_224)
        assert out["image"].shape == (0, 3, ih, iw) and out["depth"].shape == (0, 1, dh, dw)
        assert out["image"].is_cuda and out["depth"].is_cuda


@pytest.mark.parametrize("is_224", [False, True], ids=["DecoderWave-640", "DecoderWave224"])
def test_drives_a_native_decoder_step_and_the_loss(is_224):
    from wavelet_monodepth_b200 import nyu_decoders as nd
    from wavelet_monodepth_b200.nyu_loss import NyuDepthLoss
    assert not torch.backends.cudnn.allow_tf32                 # the native training step
    fx = nic.load("224_bicubic" if is_224 else "640_bicubic")
    inputs = run(nic.items(fx)[:4], is_224)
    n, _, h, w = inputs["image"].shape
    ch = [32, 24, 32, 64, 160]
    cls = nd.DecoderWave224 if is_224 else nd.DecoderWave
    dec = cls(enc_features=ch, decoder_width=0.5)
    synth.load_random(dec, seed=1)
    dec = dec.to(DEV).train()
    feats = [f.to(DEV) for f in synth.blocky_features(synth.nyu_feature_shapes(n, h, w, ch), seed=2)]
    out = dec(feats)
    assert out[("disp", 0)].shape == inputs["depth"].shape          # as train.py pairs them
    total, losses = NyuDepthLoss()(out, inputs["depth"])
    total.backward()
    assert torch.isfinite(total)
    grads = [p.grad for p in dec.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)
