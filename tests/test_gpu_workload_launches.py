"""GPU: every libwmd launch of the decoders, training steps, evaluations and losses the package ships beyond the
benchmarked decoders, against the fp64 contract of its kernel (tests/launch_check.py).

tests/test_gpu_production_launches.py checks the benchmarked decoders; this file checks the rest at production batch and
image sizes, where the size-dependent parts of their kernels are: the 224-pixel wavelet decoder (its MobileNetV2-light
pyramid's fine levels take the FMA engine) and the 224-pixel baseline decoder; native training of those two, of NYU's
baseline Decoder, of DecoderWave with NyuDepthLoss (the loss's CTA partials and its backward's footprint gather), of
the KITTI R50 1024x320 wave decoder, and of KITTI's wave (R50 1024x320) and baseline (R18 640x192, 12 frames) decoders
with KittiDepthHintsLoss (its warps, CTA partials and gathers at production sizes); the KITTI dense decoder without
skips; the sparse NYU decoder at its threshold extremes; NYU evaluation with depth boundary errors on 440x592 frames (fixed CTA grids, union-find hysteresis, the
exact distance transform) and in 224 mode; KITTI evaluation of post-processed disparities, whose medians are taken by
radix select over full LiDAR frames.  The data pipelines run where their outputs are used: depth hints of one 1024x320
pair with both views in one batch (all twelve matchers and the fusion); KittiInputs on twelve items of KITTI's five raw
sizes, flipped, jittered and with hints, driving an R18 wave decoder step with KittiDepthHintsLoss; NyuInputs' depths as
the NyuDepthLoss target of a DecoderWave step; the ground truth of eight full velodyne scans, over the calibration
dates' image sizes, both cameras and both depth conventions, scored by KittiDepthEvaluator.  Inputs are synthetic
(synth, oracle.nyu_edges.edge_split, oracle.kitti_eval.synthetic_split, oracle.depth_hints.make_pair,
oracle.kitti_inputs.synthetic_view, oracle.nyu_inputs.synthetic_image, oracle.kitti_gt.synthetic_scan).  The entry
points are called through their modules, as the package's users do: a name imported from a module would bypass the
harness's wrapper, and the completeness check would name its symbol.

Each workload runs once plainly and once under the harness, which checks each launch at its kernel's bar and that every
kernel launched ran inside a checked call, with every buffer guarded and poisoned, exactly sized workspaces and inputs
compared bit for bit after each call; the two runs must agree bit for bit, so no result depends on what was in memory.
The launch symbols launch_check.REACH attributes to a workload must be called by it.  Each prints its per-entry-point call
counts and wall times; the module prints the worst error of every (entry point, engine, mode) at the end.
"""
import gc
import os
import random
import time

import numpy as np
import pytest
import torch

from oracle import depth_hints as odh
from oracle import kitti_eval as oke
from oracle import kitti_gt as okg
from oracle import kitti_inputs as oki
from oracle import kitti_loss as okl
from oracle import nyu_edges as ne
from oracle import nyu_inputs as oni
from wavelet_monodepth_b200 import (kitti_decoders as kd, kitti_eval, kitti_gt, kitti_hints, kitti_inputs,
                                    nyu_decoders as nd, nyu_eval, nyu_inputs, synth)
from wavelet_monodepth_b200.kitti_loss import KittiDepthHintsLoss
from wavelet_monodepth_b200.nyu_loss import NyuDepthLoss

import launch_check as lc
from workloads import D161, DEV, R18, R50, kitti_feats, nyu, same

pytestmark = pytest.mark.gpu
MNV2_LIGHT_CH = (32, 24, 32, 64, 160)
D161_224 = (synth.DENSENET161_CH, 224, 224)
MNV2_224 = (MNV2_LIGHT_CH, 224, 224)
EVAL_FRAMES = 16
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from lc.REPORT.module_report()


@pytest.fixture(autouse=True)
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _raw(t):
    """a float tensor's bits (NaN rows compare equal), any other tensor as it is"""
    if t.is_floating_point():
        return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])
    return t


def _feats(shapes, seed, grad=False):
    return [f.to(DEV).requires_grad_(grad) for f in synth.blocky_features(shapes, seed=seed)]


def _nyu_module(cls, ch):
    dec = cls(enc_features=list(ch), decoder_width=0.5)
    synth.load_random(dec, seed=11)
    return dec.to(DEV)


# ------------------------------------------------------------------------------------------ inference
def nyu224(cls, n, spec):
    def run():
        ch, h, w = spec
        dec = _nyu_module(cls, ch).eval()
        with torch.no_grad():
            return dec(_feats(synth.nyu_feature_shapes(n, h, w, ch), seed=3))
    return run


def kitti_no_skips(n, spec):
    def run():
        ch, h, w = spec
        dec = kd.DepthWaveProgressiveDecoder(np.array(ch), use_skips=False)
        synth.bench_kitti_params(dec)
        with torch.no_grad():
            return dec.to(DEV).eval()(kitti_feats(n, *spec))
    return run


# ------------------------------------------------------------------------------------------ training
def train(make, n, spec, shapes, loss=None, inputs=None):
    """One native training step with fp32 convolutions: outputs, parameter and input-feature gradients.  With `loss`
    (a NyuDepthLoss) the objective is that loss against the "depth" of inputs(n) (a NyuInputs batch), or without
    `inputs` against a target within 30 % of the decoder's own ("disp", 0) (so the signs of the differences vary);
    otherwise the sum of the ("disp", s) means."""
    def run():
        ch, h, w = spec
        mod = make(ch)
        synth.load_random(mod, seed=1)
        mod = mod.to(DEV).train()
        feats = _feats(shapes(n, h, w, ch), seed=2, grad=True)
        out = mod(feats)
        res = {("out",) + tuple(k): v.detach() for k, v in out.items()}
        if loss is None:
            total = sum(v.mean() for k, v in out.items() if k[0] == "disp")
        else:
            if inputs is None:
                d0 = out[("disp", 0)].detach()
                gen = torch.Generator(device="cpu").manual_seed(5)
                target = (d0.abs() + 0.05) * (0.7 + 0.6 * torch.rand(d0.shape, generator=gen)).to(DEV)
            else:
                batch = inputs(n)
                res.update({("input", k): v for k, v in batch.items()})
                target = batch["depth"]
            total, losses = loss(out, target)
            res.update({("loss", k): v.detach() for k, v in losses.items()})
        total.backward()
        res.update({("grad", k): p.grad for k, p in mod.named_parameters() if p.grad is not None})
        res.update({("feature_grad", j): f.grad for j, f in enumerate(feats) if f.grad is not None})
        return res
    return run


def kitti_loss_inputs(n, h, w):
    """oracle.kitti_loss's synthetic stereo frames (images, KITTI's intrinsics, hints) as a loss's inputs dict"""
    inp, _ = okl.make_inputs(dict(N=n, H=h, W=w, scales=okl.SCALES), 5)
    inputs = {("color", 0, 0): inp["target"], ("color", "s", 0): inp["source"], ("K", 0): inp["K"],
              ("inv_K", 0): inp["inv_K"], "stereo_T": inp["stereo_T"], "depth_hint": inp["depth_hint"],
              "depth_hint_mask": inp["depth_hint_mask"]}
    inputs.update({("color", 0, s): inp["colors"][s] for s in okl.SCALES if s})
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in inputs.items()}


def kitti_inputs_batch(n, h, w):
    """KittiInputs on n items (frames 0 and "s") over KITTI's five raw image sizes: left and right sides, flipped and
    not, two in three jittered, depth hints at two raw sizes and one missing"""
    items = []
    for i in range(n):
        view = oki.synthetic_view(60 + i, *oki.RAW_SIZES[i % len(oki.RAW_SIZES)])
        side = "lr"[(i // 2) % 2]
        hint = None if i == 5 else oki.synthetic_hint(90 + i, *((320, 1024) if i % 3 else (188, 621)))
        items.append({"views": {0: view, "s": np.ascontiguousarray(np.roll(view, 12 if side == "l" else -12, 1))},
                      "do_color_aug": i % 3 != 0, "do_flip": i % 2 == 1,
                      "jitter": oki.get_params(random.Random(i)) if i % 3 != 0 else None, "side": side,
                      "image_path": "frame_%d" % i, "hint": hint})
    return kitti_inputs.KittiInputs(h, w, [0, "s"], use_depth_hints=True)(kitti_inputs.collate(items))


def nyu_inputs_batch(n):
    """NyuInputs (640x480 image, 320x240 depth, bicubic) on n items: flipped and not, every channel order, gammas 0.8,
    1.0 and 1.25, and items without a swap or gamma"""
    items = [{"image": oni.synthetic_image(20 + i), "depth": oni.synthetic_depth(20 + i), "flip": i % 2 == 1,
              "perm": i % 7 - 1, "gamma": None if i % 7 == 0 else (0.8, 1.0, 1.25)[i % 3]} for i in range(n)]
    return nyu_inputs.NyuInputs(False, "bicubic")(nyu_inputs.collate(items))


def train_kitti_loss(make, n, spec, inputs=kitti_loss_inputs):
    """One native training step of a KITTI decoder with KittiDepthHintsLoss on inputs(n, h, w), by default
    oracle.kitti_loss's synthetic stereo frames; the tie-breaking noise from a seeded CPU generator, so both runs draw
    the same.  Inputs, outputs, terms, masks, warps, parameter and input-feature gradients."""
    def run():
        ch, h, w = spec
        mod = make(ch)
        synth.load_random(mod, seed=1)
        mod = mod.to(DEV).train()
        feats = _feats(synth.kitti_feature_shapes(n, h, w, ch), seed=2, grad=True)
        inputs_ = inputs(n, h, w)
        out = mod(feats)
        torch.manual_seed(5)
        total, losses = KittiDepthHintsLoss(h, w)(inputs_, out)
        res = {("out",) + tuple(k if isinstance(k, tuple) else (k,)): v.detach() for k, v in out.items()
               if torch.is_tensor(v)}
        res.update({("input", k): v for k, v in inputs_.items()})
        res.update({("loss", k): v.detach() for k, v in losses.items()})
        total.backward()
        res.update({("grad", k): p.grad for k, p in mod.named_parameters() if p.grad is not None})
        res.update({("feature_grad", j): f.grad for j, f in enumerate(feats) if f.grad is not None})
        return res
    return run


def _nyu(cls):
    return lambda ch: cls(enc_features=list(ch), decoder_width=0.5)


# ------------------------------------------------------------------------------------------ evaluation
def _to_depth_range(disp, lo, hi):
    """the decoder's disparities mapped affinely onto [lo, hi] (its structure, at the scale a split's depths have)"""
    d = disp.detach()
    return lo + (hi - lo) * (d - d.amin()) / (d.amax() - d.amin())


def nyu_eval_edges(n, spec, batch=8):
    """SparseDecoderWave outputs, mapped onto 1..5 m, into NyuDepthEvaluator with edges_gt (Eigen mode) in batches of
    `batch`; then compute_errors_nyu over the whole split's prediction maps."""
    def run():
        ch, h, w = spec
        split = ne.edge_split(5, n=n)
        dec = _nyu_module(nd.SparseDecoderWave, ch).eval()
        ev = nyu_eval.NyuDepthEvaluator(split["gt"], edges_gt=split["edges"])
        depth = torch.empty((n,) + ev.out_shape, dtype=torch.float64, device=DEV)
        for b in range(0, n, batch):
            with torch.no_grad():
                disp = dec(_feats(synth.nyu_feature_shapes(batch, h, w, ch), seed=40 + b), 0.1)[("disp", 0)]
            ev.add(100.0 * _to_depth_range(disp, 1.0, 5.0), depth_out=depth[b:b + batch])
        errors = nyu_eval.compute_errors_nyu(depth, ev.gt)
        return {"sums": ev.sums, "edges_scores": ev.edges_scores, "depth": depth, "errors": errors}
    return run


def nyu_eval_224(n, spec):
    def run():
        ch, h, w = spec
        gt = ne.edge_split(6, n=n)["gt"]
        dec = _nyu_module(nd.DecoderWave224, ch).eval()
        with torch.no_grad():
            disp = dec(_feats(synth.nyu_feature_shapes(n, h, w, ch), seed=50))[("disp", 0)]
        ev = nyu_eval.NyuDepthEvaluator(gt, use_224=True)
        depth = torch.empty((n,) + ev.out_shape, dtype=torch.float64, device=DEV)
        ev.add(100.0 * _to_depth_range(disp, 1.0, 5.0), depth_out=depth)
        return {"sums": ev.sums, "depth": depth}
    return run


def kitti_eval_pp(n, spec):
    """Sparse R18 decoder on the frames and their flips, disp_to_depth's scaled disparity (min 0.1, max 100 m),
    batch_post_process_disparity, KittiDepthEvaluator with median scaling on a synthetic split at KITTI's ground-truth
    sizes (its empty, one-valid, even-count and all-equal frames included); then compute_errors over the split's valid
    ground truth and the depths the evaluator sampled there."""
    def run():
        ch, h, w = spec
        split = oke.synthetic_split(7, n_regular=n - len(oke.SPECIAL))
        dec = kd.SparseDepthWaveProgressiveDecoder(np.array(ch))
        synth.bench_kitti_params(dec)
        dec = dec.to(DEV).eval()
        feats = kitti_feats(n, *spec)
        with torch.no_grad():
            left = dec(feats, 0.05)[("disp", 0)][:, 0]
            right = dec([torch.flip(f, [3]) for f in feats], 0.05)[("disp", 0)][:, 0]
        lo, hi = 1 / 100.0, 1 / 0.1
        pp = kitti_eval.batch_post_process_disparity(lo + (hi - lo) * left, torch.flip(lo + (hi - lo) * right, [2]))
        ev = kitti_eval.KittiDepthEvaluator(split["gt"])
        ev.add(pp)
        total = int(ev.offsets[-1])
        errors = kitti_eval.compute_errors(ev.gt[:total], ev.depth[:total])
        return {"pp": pp, "errors": ev.errors, "ratios": ev.ratios, "counts": ev.counts, "pooled": errors}
    return run


# ------------------------------------------------------------------------------------------ data pipelines
def hints_pair(seed, h, w):
    """DepthHintGenerator on one synthetic pair, its left and right views in one batch (the right one mirrored around
    the matchers): all twelve matchers and the fusion"""
    def run():
        left, right = odh.make_pair(seed, h, w)
        base = torch.from_numpy(np.stack([left, right])).to(DEV)
        lookup = torch.from_numpy(np.stack([right, left])).to(DEV)
        depth, index = kitti_hints.DepthHintGenerator(h, w)(base, lookup, [False, True], return_index=True)
        return {"depth": depth, "index": index}
    return run


def gt_export_then_eval(n):
    """generate_depth_maps on n full synthetic scans, one call per depth convention (vel_depth off, on), the frames
    mixing the calibration dates' image sizes and both cameras; the maps then score seeded 640x192 disparities in
    KittiDepthEvaluator"""
    def run():
        with np.load(os.path.join(GOLDEN, "kitti_gt_calib.npz")) as f:
            calib = {k: f[k] for k in f.files}
        dates = sorted(okg.DATES)
        res, gts = {}, []
        for vd in (False, True):
            frames = [(dates[(2 * i + vd) % len(dates)], 2 + (i + vd) % 2) for i in range(n // 2)]
            scans = [okg.synthetic_scan(300 + 10 * vd + i) for i in range(n // 2)]
            offsets = np.concatenate([[0], np.cumsum([s.shape[0] for s in scans])])
            P = np.stack([calib["%s/P%d" % fr] for fr in frames])
            sizes = np.array([calib["%s/size" % d] for d, _ in frames], np.int32)
            depth = kitti_gt.generate_depth_maps(torch.from_numpy(np.concatenate(scans)).to(DEV), offsets, P, sizes, vd)
            res["depth", vd] = depth
            gts += [depth[k, :h, :w] for k, (h, w) in enumerate(sizes.tolist())]
        ev = kitti_eval.KittiDepthEvaluator(gts)
        gen = torch.Generator(device="cpu").manual_seed(9)
        ev.add((0.01 + 0.3 * torch.rand((n, 1, 192, 640), generator=gen)).to(DEV))
        res.update(errors=ev.errors, ratios=ev.ratios, counts=ev.counts)
        return res
    return run


WORKLOADS = {
    "wave224_d161_x8": nyu224(nd.DecoderWave224, 8, D161_224),
    "wave224_mnv2light_x8": nyu224(nd.DecoderWave224, 8, MNV2_224),
    "baseline_decoder224_d161_x8": nyu224(nd.Decoder224, 8, D161_224),
    "train_wave224_mnv2light_x8_nyuloss_ll": train(_nyu(nd.DecoderWave224), 8, MNV2_224, synth.nyu_feature_shapes,
                                                   NyuDepthLoss(use_wavelets=True, supervise_LL=True)),
    "train_nyu_wave_d161_640x480_x8_nyuloss": train(_nyu(nd.DecoderWave), 8, D161, synth.nyu_feature_shapes,
                                                    NyuDepthLoss()),
    "train_decoder_d161_640x480_x8": train(_nyu(nd.Decoder), 8, D161, synth.nyu_feature_shapes),
    "train_decoder224_mnv2light_x8": train(_nyu(nd.Decoder224), 8, MNV2_224, synth.nyu_feature_shapes),
    "train_wave_r50_1024x320_x8": train(lambda ch: kd.DepthWaveProgressiveDecoder(np.array(ch)), 8, R50,
                                        synth.kitti_feature_shapes),
    "train_wave_r50_1024x320_x8_kittiloss": train_kitti_loss(lambda ch: kd.DepthWaveProgressiveDecoder(np.array(ch)),
                                                              8, R50),
    "train_baseline_r18_640x192_x12_kittiloss": train_kitti_loss(lambda ch: kd.DepthDecoder(np.array(ch)), 12, R18),
    "dense_no_skips_r18_640x192_x16": kitti_no_skips(16, R18),
    "nyu_sparse_d161_640x480_x8_thr0": nyu(nd.SparseDecoderWave, 8, D161, 0.0),
    "nyu_sparse_d161_640x480_x8_thr0.5": nyu(nd.SparseDecoderWave, 8, D161, 0.5),
    "eval_nyu_sparse_d161_x%d_edges" % EVAL_FRAMES: nyu_eval_edges(EVAL_FRAMES, D161),
    "eval_nyu_wave224_mnv2light_x8": nyu_eval_224(8, MNV2_224),
    "eval_kitti_sparse_r18_x%d_postprocess" % EVAL_FRAMES: kitti_eval_pp(EVAL_FRAMES, R18),
    "hints_320x1024_pair_both_sides": hints_pair(odh.FULL["full0"][0], 320, 1024),
    "train_wave_r18_640x192_x12_from_kitti_inputs": train_kitti_loss(
        lambda ch: kd.DepthWaveProgressiveDecoder(np.array(ch)), 12, R18, kitti_inputs_batch),
    "train_nyu_wave_d161_640x480_x8_from_nyu_inputs": train(_nyu(nd.DecoderWave), 8, D161, synth.nyu_feature_shapes,
                                                            NyuDepthLoss(), nyu_inputs_batch),
    "gt_export_full_scans_then_eval": gt_export_then_eval(8),
}


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_every_launch_meets_its_contract(name, monkeypatch):
    run = WORKLOADS[name]
    t0 = time.perf_counter()
    plain = {k: _raw(v) if torch.is_tensor(v) else v for k, v in run().items()}
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    harness = lc.Harness(monkeypatch)
    with harness.workload(name):
        checked = {k: _raw(v) if torch.is_tensor(v) else v for k, v in run().items()}
    monkeypatch.undo()
    t2 = time.perf_counter()
    same(plain, checked, name)
    assert not harness.reached(name), (name, "never called", harness.reached(name))
    print("%s (%.1f s plain, %.1f s checked; %s): %s" % (name, t1 - t0, t2 - t1, harness.report(),
                                                         ", ".join("%s x%d" % kv for kv in sorted(harness.calls.items()))))
    del plain, checked, harness
    gc.collect()
    torch.cuda.empty_cache()
