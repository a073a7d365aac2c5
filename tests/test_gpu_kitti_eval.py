"""GPU: KITTI depth evaluation on libwmd against the reference's per-frame results (tests/golden/kitti_eval.npz, written
by oracle/pin_kitti_eval.py from the unmodified evaluate_depth.py) and against the numpy oracle.

Per-frame metrics and ratios: 1e-12 relative, NaN where the reference is NaN; valid counts and a1..a3 exact (the only
allowed exception, a pixel within 1e-12 of a 1.25^k threshold, is counted and must not occur on the seeded data)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import kitti_eval as oke
from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200.kitti_eval import (METRICS, KittiDepthEvaluator, batch_post_process_disparity,
                                               compute_density, compute_errors)
from wavelet_monodepth_b200._lib import WmdError

from helpers import GOLDEN, kitti_features, load_golden, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"


def load_fixture():
    with np.load(os.path.join(GOLDEN, "kitti_eval.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def assert_rel(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern differs", got, want)
    f = ~np.isnan(want)
    err = np.abs(got[f] - want[f]) / np.maximum(np.abs(want[f]), 1e-300)
    assert err.size == 0 or err.max() <= tol, (what, float(err.max()))


def evaluator(gt, mode):
    split, med, sf = oke.MODES[mode]
    return KittiDepthEvaluator(gt, eval_split=split, median_scaling=med, pred_depth_scale_factor=sf)


def run(gt, disp, mode, chunk=None):
    ev = evaluator(gt, mode)
    d = torch.as_tensor(disp).to(DEV)
    step = chunk or d.shape[0]
    for i in range(0, d.shape[0], step):
        ev.add(d[i:i + step])
    return ev


def near_ties(gt, disp, mode, tol=1e-12):
    """pixels whose max(gt/pred, pred/gt) lies within tol of 1.25, 1.25^2 or 1.25^3 (the oracle's values)"""
    split, med, sf = oke.MODES[mode]
    n = 0
    with np.errstate(all="ignore"):
        for g, d in zip(gt, disp):
            m = oke.valid_mask(g, split)
            p = (1 / oke.resize_linear(d, *g.shape))[m] * sf
            t = g[m]
            if med:
                p = p * (np.median(t) / np.median(p))
            p = np.clip(p, oke.MIN_DEPTH, oke.MAX_DEPTH)
            th = np.maximum(t / p, p / t)
            n += sum(int((np.abs(th - c) <= tol * c).sum()) for c in (1.25, 1.25 ** 2, 1.25 ** 3))
    return n


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int64)


@pytest.mark.parametrize("seed", [0, 1])
def test_every_mode_matches_the_reference_fixture(seed):
    fx, meta = load_fixture()
    split = oke.synthetic_split(seed)
    for h, w in meta["disp_sizes"]:
        disp = split["disp"][(h, w)]
        for mode in meta["modes"]:
            key = "s%d_%dx%d_%s" % (seed, w, h, mode)
            ev = run(split["gt"], disp, mode)
            errors, ratios = ev.errors.cpu().numpy(), ev.ratios.cpu().numpy()
            want = fx[key + "__errors"]
            assert np.array_equal(ev.counts.cpu().numpy(), fx[key + "__counts"]), key
            assert_rel(errors[:, :4], want[:, :4], 1e-12, key)
            ties = near_ties(split["gt"], disp, mode)
            assert ties == 0, (key, "pixels within 1e-12 of a threshold", ties)
            assert np.array_equal(errors[:, 4:], want[:, 4:], equal_nan=True), key
            if oke.MODES[mode][1]:
                assert_rel(ratios, fx[key + "__ratios"], 1e-12, key)
            s = ev.summary()
            for j, name in enumerate(METRICS):
                assert_rel(s[name], want[:, j].mean(), 1e-12, (key, name))
            if oke.MODES[mode][1]:
                r = fx[key + "__ratios"]
                assert_rel([s["med"], s["std"]], [np.median(r), np.std(r / np.median(r))], 1e-12, (key, "ratios"))


@pytest.mark.parametrize("size", [(192, 640), (320, 1024)])
def test_medians_equal_numpy_on_the_special_frames(size):
    """ratio = median(gt) / median(depth); the depth the device samples is the oracle's, so each ratio is exact."""
    split = oke.synthetic_split(0)
    ev = run(split["gt"], split["disp"][size], "mono_eigen")
    ratios = ev.ratios.cpu().numpy()
    for name, i in split["special"].items():
        _, want, count = oke.evaluate_frame(split["gt"][i], split["disp"][size][i])
        assert int(ev.counts[i]) == count, name
        assert (np.isnan(want) and np.isnan(ratios[i])) or ratios[i] == want, (name, ratios[i], want)


def test_chunking_repeats_and_graph_replay_are_bit_identical():
    split = oke.synthetic_split(1)
    disp = split["disp"][(192, 640)]
    whole = run(split["gt"], disp, "mono_eigen")
    for chunk in (1, 7):
        ev = run(split["gt"], disp, "mono_eigen", chunk)
        assert torch.equal(bits(ev.errors), bits(whole.errors)), chunk
        assert torch.equal(bits(ev.ratios), bits(whole.ratios)), chunk
    again = run(split["gt"], disp, "mono_eigen")
    assert torch.equal(bits(again.errors), bits(whole.errors))
    ev = evaluator(split["gt"], "mono_eigen")
    d = torch.from_numpy(disp).to(DEV)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ev.add(d)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(ev.errors), bits(whole.errors))
    assert torch.equal(bits(ev.ratios), bits(whole.ratios))


def test_post_processing_matches_the_reference_samples():
    fx, meta = load_fixture()
    l_disp, r_disp = oke.post_process_inputs(meta["post_seed"])
    l, r = torch.from_numpy(l_disp).to(DEV), torch.from_numpy(r_disp).to(DEV)
    out = batch_post_process_disparity(l, torch.flip(r, [2]))
    assert out.dtype == torch.float64
    got = out.reshape(-1)[torch.from_numpy(fx["post__idx"]).to(DEV)].cpu().numpy()
    assert_rel(got, fx["post__values"], 1e-15, "post-processing")
    want64 = oke.batch_post_process_disparity(l_disp.astype(np.float64), r_disp[:, :, ::-1].astype(np.float64))
    got64 = batch_post_process_disparity(l.double(), torch.flip(r, [2]).double()).cpu().numpy()
    assert_rel(got64, want64, 1e-15, "post-processing fp64")


def test_compute_errors_matches_the_reference_formula():
    rng = np.random.default_rng(3)
    gt = rng.uniform(1.0, 80.0, 5000)
    pred = gt * rng.uniform(0.6, 1.6, 5000)
    got = compute_errors(torch.from_numpy(gt).to(DEV), torch.from_numpy(pred).to(DEV)).cpu().numpy()
    assert_rel(got, oke.compute_errors(gt, pred), 1e-12, "compute_errors")


def test_sparse_decoder_to_metrics_end_to_end():
    _, meta = load_golden("kitti_tiny_dense")
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]))
    mod.load_state_dict(seeded_params(mod, meta), strict=False)
    mod = mod.to(DEV).eval()
    feats = kitti_features(meta, DEV)
    split = oke.synthetic_split(0)
    gt = split["gt"][:2]
    min_disp, max_disp = 1 / 100.0, 1 / 0.1                # disp_to_depth(disp, 0.1, 100) (KITTI/layers.py:16-25)
    ev = evaluator(gt, "mono_eigen")
    for thr in (0.1, 0.2, 0.3):
        ev.reset()
        with torch.no_grad():
            out = mod(feats, thr)
        scaled = min_disp + (max_disp - min_disp) * out[("disp", 0)]
        ev.add(scaled, sparse_outputs=out)
        want = [oke.evaluate_frame(g, d) for g, d in zip(gt, scaled[:, 0].cpu().numpy())]
        assert_rel(ev.errors[:, :4].cpu().numpy(), np.stack([w[0][:4] for w in want]), 1e-12, thr)
        assert np.array_equal(ev.errors[:, 4:].cpu().numpy(), np.stack([w[0][4:] for w in want])), thr
        assert np.array_equal(ev.counts.cpu().numpy(), [w[2] for w in want]), thr
        dens = compute_density(out).cpu().numpy()
        for b in range(2):
            num, den = 0, 0
            for i in range(4):
                m = out[("wavelet_mask", i)][b:b + 1]
                num += int(m.sum())
                den += m.shape[2] * m.shape[3]
            assert dens[b] == float(num) / float(den), (thr, b)
        s = ev.summary()
        assert s["frames"] == 2 and s["density_mean"] == float(np.mean(dens))
        assert s["total_ops_mean"] == float(np.mean(out["total_ops_per_sample"]))


def test_bad_inputs_raise():
    split = oke.synthetic_split(0)
    ev = evaluator(split["gt"][:3], "mono_eigen")
    disp = torch.from_numpy(split["disp"][(192, 640)][:3])
    with pytest.raises(WmdError):
        ev.add(disp)                                       # CPU tensor
    with pytest.raises(WmdError):
        ev.add(disp.to(DEV).half())                        # wrong dtype
    with pytest.raises(WmdError):
        ev.add(torch.cat([disp, disp]).to(DEV))            # more frames than the split holds
    ev.add(disp[:2].to(DEV))
    with pytest.raises(WmdError):
        ev.add(disp[:2].to(DEV))                           # only one frame left
    with pytest.raises(WmdError):
        compute_errors(torch.ones(4), torch.ones(4))
    with pytest.raises(WmdError):
        batch_post_process_disparity(disp.to(DEV), disp.to(DEV).double())
