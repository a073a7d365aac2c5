"""GPU: KITTI's training inputs on libwmd.  KittiInputs' dict equals the reference's __getitem__ (the digests of
tests/golden/kitti_inputs_*.npz) and oracle.kitti_inputs on every key: batches mixing the five raw sizes, flips and
augmentation, all 24 jitter orders, 640x192 and 1024x320, one item, missing and mixed hints.  The same batch gives the
same bits twice and item by item, and the dict drives a native decoder step with KittiDepthHintsLoss."""
import itertools

import numpy as np
import pytest
import torch

from oracle import kitti_inputs as oki
from wavelet_monodepth_b200 import _lib
from wavelet_monodepth_b200 import kitti_inputs as ki

import kitti_inputs_cases as kic

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def run(items, height, width, frame_idxs, scales=(0, 1, 2, 3), hints=False):
    fn = ki.KittiInputs(height, width, frame_idxs, scales, use_depth_hints=hints)
    out = fn(ki.collate(items), DEV)
    torch.cuda.synchronize()
    return out


def host(out, n):
    return {k: v[n].cpu().numpy() for k, v in out.items() if k != "image_path"}


@pytest.mark.parametrize("name", kic.CASES)
def test_reference_digests(name):
    fx = kic.load(name)
    cfg = fx["config"]
    its = kic.items(fx)
    before = _lib.launch_count()
    out = run(its, cfg["height"], cfg["width"], cfg["frame_idxs"], cfg["scales"], cfg["use_depth_hints"])
    assert _lib.launch_count() - before == 2 * len(cfg["scales"]) + 2
    assert kic.mismatches(fx, lambda n: host(out, n)) == []
    assert out["image_path"] == [str(p) for p in fx["image_path"]]
    for n, found in enumerate(fx.get("hint_found", [])):
        if cfg["use_depth_hints"] and not found:                 # the reference has no disp_hint: zeros here
            assert not out["disp_hint"][n].any() and not out["depth_hint"][n].any()


def _pyramids(sizes, height, width, seed):
    """{(size index, flip): oracle pyramid} of one seeded view per raw size"""
    views = [oki.synthetic_view(seed + k, *hw) for k, hw in enumerate(sizes)]
    return views, {(k, f): oki.pyramid(v, height, width, (0, 1, 2, 3), f) for k, v in enumerate(views) for f in (0, 1)}


@pytest.mark.parametrize("height,width", [(192, 640), (320, 1024)])
def test_every_jitter_order_on_mixed_sizes(height, width):
    """24 items, one per jitter order, over the five raw sizes, flipped and not, factors 0.8 / 1.0 / 1.2, hue +-0.1,
    plus two items without augmentation"""
    views, pyr = _pyramids(oki.RAW_SIZES, height, width, 40)
    its, exp = [], []
    levels = (0.8, 1.0, 1.2)
    for i, order in enumerate(list(itertools.permutations(range(4))) + [None, None]):
        k, flip = i % 5, (i // 5) % 2
        params = None
        if order is not None:
            params = ((levels[i % 3], levels[(i + 1) % 3], levels[(i + 2) % 3], 0.1 if i % 2 else -0.1), order)
        its.append({"views": {0: views[k]}, "do_color_aug": params is not None, "do_flip": bool(flip),
                    "jitter": params, "side": "l", "image_path": str(i)})
        exp.append({s: (oki.to_tensor(img), oki.to_tensor(oki.jitter(img, params))) for s, img in pyr[k, flip].items()})
    out = run(its, height, width, [0])
    for n, e in enumerate(exp):
        for s, (plain, aug) in e.items():
            assert np.array_equal(out[("color", 0, s)][n].cpu().numpy(), plain), (n, s)
            assert np.array_equal(out[("color_aug", 0, s)][n].cpu().numpy(), aug), (n, s, its[n]["jitter"])


def test_one_item_with_hints_and_scale_subsets():
    """N = 1 at 1024x320 with a hint, flipped and jittered; and target scales (0, 2) and (1,) chain from the source"""
    view = oki.synthetic_view(3, 370, 1226)
    hint = oki.synthetic_hint(4, 320, 1024)
    params = ((1.2, 0.8, 1.1, -0.07), (3, 1, 0, 2))
    it = {"views": {0: view, "s": view[:, ::-1].copy()}, "do_color_aug": True, "do_flip": True, "jitter": params,
          "side": "r", "image_path": "x", "hint": hint}
    for scales in ((0, 1, 2, 3), (0, 2), (1,)):
        out = run([it], 320, 1024, [0, "s"], scales, hints=True)
        exp = oki.expected(it["views"], (True, True, params), "r", hint, 320, 1024, scales, True)
        got = host(out, 0)
        assert set(got) == set(exp)
        for k in exp:
            assert np.array_equal(got[k], exp[k]) and got[k].dtype == exp[k].dtype, (scales, k)


def test_missing_and_mixed_hints():
    view = oki.synthetic_view(5, 375, 1242)
    base = {"views": {0: view, "s": view}, "do_color_aug": False, "do_flip": False, "jitter": None, "side": "l",
            "image_path": "x"}
    missing = dict(base, hint=None)
    out = run([missing, dict(missing, do_flip=True)], 192, 640, [0, "s"], hints=True)
    assert "disp_hint" not in out
    assert not out["depth_hint"].any() and not out["depth_hint_mask"].any()
    assert out["depth_hint"].shape == (2, 1, 192, 640)
    hint = oki.synthetic_hint(6, 188, 621)
    out = run([dict(base, hint=hint), missing, dict(base, hint=hint, do_flip=True)], 192, 640, [0, "s"], hints=True)
    for n, (h, flip) in enumerate(((hint, False), (None, False), (hint, True))):
        d, disp, mask = oki.hints(h, flip, 192, 640)
        assert np.array_equal(out["depth_hint"][n].cpu().numpy(), d)
        assert np.array_equal(out["disp_hint"][n].cpu().numpy(), disp)
        assert np.array_equal(out["depth_hint_mask"][n].cpu().numpy(), mask)


def test_repeatable_and_independent_of_the_batch():
    fx = kic.load("train640")
    cfg = fx["config"]
    its = kic.items(fx)
    args = (cfg["height"], cfg["width"], cfg["frame_idxs"], cfg["scales"], True)
    a, b = run(its, *args), run(its, *args)
    alone = run(its[3:4], *args)
    for k, v in a.items():
        if k != "image_path":
            assert torch.equal(v, b[k]), k
            if k in alone:                      # item 3's disp_hint is absent alone when its hint is missing
                assert torch.equal(v[3:4], alone[k]), k


def test_drives_a_native_decoder_step_and_the_loss():
    from wavelet_monodepth_b200 import kitti_decoders as kd, synth
    from wavelet_monodepth_b200.kitti_loss import KittiDepthHintsLoss
    fx = kic.load("train640")
    its = kic.items(fx)[:4]
    inputs = run(its, 192, 640, [0, "s"], hints=True)
    r18 = (64, 64, 128, 256, 512)
    dec = kd.DepthWaveProgressiveDecoder(np.array(r18))
    synth.load_random(dec, seed=1)
    dec = dec.to(DEV).train()
    feats = [f.to(DEV) for f in synth.blocky_features(synth.kitti_feature_shapes(4, 192, 640, r18), seed=2)]
    out = dec(feats)
    total, losses = KittiDepthHintsLoss(192, 640)(inputs, out)
    total.backward()
    assert torch.isfinite(total)
    grads = [p.grad for p in dec.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)
