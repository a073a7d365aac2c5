"""GPU: NYUv2 depth evaluation on libwmd against the reference's results (tests/golden/nyu_eval.npz, written by
oracle/pin_nyu_eval.py from the unmodified NYUv2/utils.py) and against the numpy oracle.

Against the reference's fp64 run: rel and rms to 1e-12 relative, log_10 to 1e-7 (torch's CPU and CUDA float32 log10 of
the ground truth may differ by an ulp) and to 1e-12 against the oracle fed the evaluator's own log10; a_k counts exact,
with no pixel within 1e-12 of a threshold.  The prediction map is bit-identical to the oracle's."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import nyu_eval as one
from wavelet_monodepth_b200 import nyu_decoders as nd, synth
from wavelet_monodepth_b200._lib import WmdError
from wavelet_monodepth_b200.nyu_eval import METRICS, NyuDepthEvaluator, compute_errors_nyu

from helpers import GOLDEN, load_golden, nyu_features, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
MNV2_LIGHT_CH = [32, 24, 32, 64, 160]


def load_fixture():
    with np.load(os.path.join(GOLDEN, "nyu_eval.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def assert_rel(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern differs", got, want)
    f = ~np.isnan(want) & ~(np.isinf(want) & (got == want))
    err = np.abs(got[f] - want[f]) / np.maximum(np.abs(want[f]), 1e-300)
    assert err.size == 0 or err.max() <= tol, (what, float(err.max()))


def assert_log10(got, want, what):
    """log_10 to 1e-12 relative plus 1e-15 absolute: each pixel's |log10 y - log10 x| carries the fp64 log10's ulp,
    which is all an all-equal frame's log_10 (a cancellation of log10 3 against itself) is made of"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern differs")
    f = np.isfinite(want)
    assert np.array_equal(got[~f & ~np.isnan(want)], want[~f & ~np.isnan(want)]), what
    assert np.all(np.abs(got[f] - want[f]) <= 1e-12 * np.abs(want[f]) + 1e-15), (what, got, want)


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int64)


def splits(meta):
    for s in meta["seeds"]:
        yield "s%d" % s, s, one.synthetic_split(s)
    yield "special", meta["special_seed"], one.synthetic_split(meta["special_seed"], special=True)


def run(gt, disp, use_224, use_disparity, chunk=None, depth=False):
    ev = NyuDepthEvaluator(gt, use_224=use_224, use_disparity=use_disparity)
    d = torch.as_tensor(disp).to(DEV)
    out = torch.empty((d.shape[0],) + ev.out_shape, dtype=torch.float64, device=DEV) if depth else None
    step = chunk or d.shape[0]
    for i in range(0, d.shape[0], step):
        ev.add(d[i:i + step], depth_out=None if out is None else out[i:i + step])
    return ev, out


def frame_metrics(sums):
    return one.frame_metrics(sums.cpu().numpy())


@pytest.mark.parametrize("split_name", ["s0", "s1", "special"])
def test_every_mode_matches_the_reference_fixture(split_name):
    fx, meta = load_fixture()
    for name, seed, split in splits(meta):
        if name != split_name:
            continue
        for mode, (use_224, use_disparity) in meta["modes"].items():
            for h, w in [(224, 224)] if use_224 else meta["disp_sizes"]:
                key = "%s_%s_%dx%d" % (name, mode, w, h)
                disp = split["disp"][(h, w, use_disparity)]
                ev, depth = run(split["gt"], disp, use_224, use_disparity, depth=True)
                sums = ev.sums.cpu().numpy()
                got = one.frame_metrics(sums)
                # the prediction map is the oracle's, bit for bit, NaN pattern included
                want_map = one.predict(disp, use_224, use_disparity)
                dm = depth.cpu().numpy()
                assert np.array_equal(np.isnan(dm), np.isnan(want_map)), key
                assert np.array_equal(dm[~np.isnan(dm)], want_map[~np.isnan(want_map)]), key
                # against the fp64 reference run
                for tag in ("frames", "pooled"):
                    want = fx["%s__f64_%s" % (key, tag)]
                    g = got if tag == "frames" else np.array(list(ev.summary().values())[:6])
                    assert_rel(g[..., :2], want[..., :2], 1e-12, (key, tag))
                    assert_rel(g[..., 2], want[..., 2], 1e-7, (key, tag, "log_10"))
                assert np.array_equal(sums[:, 3:6].astype(np.int64), fx[key + "__f64_counts"]), key
                ties = sum(one.near_ties(dm[i], ev.gt[i].cpu().numpy(), 1e-12) for i in range(dm.shape[0]))
                assert ties == 0, (key, "pixels within 1e-12 of a threshold", ties)
                # against the oracle fed the evaluator's own ground truth and log10
                want = one.frame_sums(want_map, ev.gt.cpu().numpy(), ev.gt_log10.cpu().numpy())
                assert_rel(got[:, :2], one.frame_metrics(want)[:, :2], 1e-12, (key, "oracle"))
                assert_log10(got[:, 2], one.frame_metrics(want)[:, 2], (key, "oracle log_10"))
                assert np.array_equal(sums[:, 3:], want[:, 3:]), key
                # the reference's own float32 numbers
                w32, ok = fx[key + "__f32_frames"][:, :3], ~np.isnan(got[:, :3]).any(1)
                small = np.abs(w32) < 1e-4
                assert np.all(np.abs(got[:, :3] - w32)[ok[:, None] & small] <= 1e-6), key
                assert_rel(np.where(small, 1.0, got[:, :3])[ok], np.where(small, 1.0, w32)[ok], 1e-6, (key, "f32"))
                for i in range(dm.shape[0]):
                    if np.isfinite(disp[i]).all() and not (disp[i] == 0).any():
                        diff = int(np.abs(sums[i, 3:6] - fx[key + "__f32_counts"][i]).sum())
                        assert diff <= one.near_ties(dm[i], ev.gt[i].cpu().numpy(), 2.0 ** -20), (key, i, diff)


def test_gt224_is_the_devices_interpolate_and_within_an_ulp_of_the_cpu_fixture():
    fx, meta = load_fixture()
    worst = {}
    for name, seed, split in splits(meta):
        ev = NyuDepthEvaluator(split["gt"], use_224=True)
        g = torch.from_numpy(split["gt"]).to(DEV)[:, None, 16:-16, 16:-16]
        want = torch.nn.functional.interpolate(g, (224, 224), mode="bilinear", align_corners=True)[:, 0]
        assert torch.equal(bits(ev.gt.double()), bits(want.double())), name
        assert torch.equal(ev.gt_log10, torch.log10(want)), name
        got = ev.gt.cpu().numpy().reshape(-1)[fx[name + "__gt224_idx"]]
        ulps = np.abs(got.view(np.int32).astype(np.int64) - fx[name + "__gt224_values"].view(np.int32))
        worst[name] = (int(ulps.max()), int((ulps > 0).sum()), ulps.size)
    print("device gt224 vs CPU fixture (max ulp, values differing, values):", worst)
    assert all(v[0] <= 1 for v in worst.values()), worst


def test_chunking_repeats_and_graph_replay_are_bit_identical():
    split = one.synthetic_split(1, n=11)
    for use_224, (h, w) in ((False, (241, 319)), (True, (224, 224))):
        disp = split["disp"][(h, w, False)]
        whole, _ = run(split["gt"], disp, use_224, False)
        for chunk in (1, 5):
            ev, _ = run(split["gt"], disp, use_224, False, chunk)
            assert torch.equal(bits(ev.sums), bits(whole.sums)), (use_224, chunk)
            assert ev.summary() == whole.summary()
        again, _ = run(split["gt"], disp, use_224, False)
        assert torch.equal(bits(again.sums), bits(whole.sums))
        ev = NyuDepthEvaluator(split["gt"], use_224=use_224)
        d = torch.from_numpy(disp).to(DEV)
        before = d.clone()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ev.add(d[:6])
            ev.add(d[6:])
        ev.sums.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(ev.sums), bits(whole.sums)), use_224
        assert torch.equal(d, before)                       # add() leaves disp as it was


def test_compute_errors_nyu_against_the_oracle_and_reproducible():
    rng = np.random.default_rng(4)
    for n in (1, 1023, 5_000_000):
        gt = rng.uniform(0.5, 10.0, n)
        pred = gt * rng.uniform(0.6, 1.6, n)
        p, g = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
        got = compute_errors_nyu(p, g)
        assert_rel(got.cpu().numpy(), one.compute_errors_nyu(pred, gt), 1e-12, n)
        assert torch.equal(bits(compute_errors_nyu(p, g)), bits(got)), n
    got = compute_errors_nyu(p.float(), g.float()).cpu().numpy()       # float32 inputs are widened
    assert_rel(got, one.compute_errors_nyu(pred.astype(np.float32), gt.astype(np.float32)), 1e-12, "f32")


def _nyu(cls, meta):
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    mod.load_state_dict(seeded_params(mod, meta), strict=False)
    return mod.to(DEV).eval()


def test_sparse_decoder_threshold_sweep_end_to_end():
    _, meta = load_golden("nyu_tiny_dense")
    mod = _nyu(nd.SparseDecoderWave, meta)
    feats = nyu_features(meta, DEV)
    gt = one.synthetic_split(2, n=2)["gt"]
    ev = NyuDepthEvaluator(gt)
    for thr in (0.1, 0.2, 0.3):
        ev.reset()
        with torch.no_grad():
            disp = mod(feats, thr)[("disp", 0)]
        ev.add(disp)
        d = disp[:, 0].cpu().numpy()
        g = one.prepare_gt(gt)
        want = one.frame_sums(one.predict(d), g, ev.gt_log10.cpu().numpy())
        sums = ev.sums.cpu().numpy()
        assert_rel(one.frame_metrics(sums)[:, :2], one.frame_metrics(want)[:, :2], 1e-12, thr)
        assert_log10(one.frame_metrics(sums)[:, 2], one.frame_metrics(want)[:, 2], thr)
        assert np.array_equal(sums[:, 3:], want[:, 3:]), thr
        s = ev.summary()
        assert s["frames"] == 2
        assert_rel([s[m] for m in METRICS], one.metrics(want), 1e-12, thr)


@pytest.mark.parametrize("name", ["DecoderWave224", "Decoder224", "Decoder"])
def test_decoders_end_to_end(name):
    cls = getattr(nd, name)
    use_224 = name.endswith("224")
    ch = MNV2_LIGHT_CH if use_224 else [16, 16, 32, 64, 128]
    size = (224, 224) if use_224 else (480, 640)
    mod = cls(enc_features=ch, decoder_width=0.5)
    synth.load_random(mod, seed=5)
    mod = mod.to(DEV).eval()
    feats = [f.to(DEV) for f in synth.blocky_features(synth.nyu_feature_shapes(2, size[0], size[1], ch), seed=6)]
    with torch.no_grad():
        disp = mod(feats)[("disp", 0)]
    gt = one.synthetic_split(3, n=2)["gt"]
    for use_disparity in (False, True):
        ev = NyuDepthEvaluator(gt, use_224=use_224, use_disparity=use_disparity)
        before = disp.clone()
        depth = torch.empty((2,) + ev.out_shape, dtype=torch.float64, device=DEV)
        ev.add(disp, depth_out=depth)
        assert torch.equal(disp, before)
        d = disp[:, 0].cpu().numpy()
        want_map = one.predict(d, use_224, use_disparity)
        assert np.array_equal(depth.cpu().numpy(), want_map, equal_nan=True), (name, use_disparity)
        want = one.frame_sums(want_map, ev.gt.cpu().numpy(), ev.gt_log10.cpu().numpy())
        sums = ev.sums.cpu().numpy()
        assert_rel(one.frame_metrics(sums)[:, :2], one.frame_metrics(want)[:, :2], 1e-12, (name, use_disparity))
        assert_log10(one.frame_metrics(sums)[:, 2], one.frame_metrics(want)[:, 2], (name, use_disparity))
        assert np.array_equal(sums[:, 3:], want[:, 3:]), (name, use_disparity)


def test_bad_inputs_raise():
    split = one.synthetic_split(0)
    gt = split["gt"]
    ev = NyuDepthEvaluator(gt)
    disp = torch.from_numpy(split["disp"][(240, 320, False)])
    with pytest.raises(WmdError):
        ev.add(disp)                                       # CPU tensor
    with pytest.raises(WmdError):
        ev.add(disp.to(DEV).double())                      # not float32
    with pytest.raises(WmdError):
        ev.add(torch.cat([disp, disp]).to(DEV))            # more frames than the split holds
    ev.add(disp[:2].to(DEV))
    with pytest.raises(WmdError):
        ev.add(disp[:2].to(DEV))                           # only one frame left
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt[:, :240])                     # ground truth not (N, 480, 640)
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt[0])
    ev224 = NyuDepthEvaluator(gt, use_224=True)
    with pytest.raises(WmdError):
        ev224.add(disp.to(DEV))                            # 224 mode takes 224 x 224
    with pytest.raises(WmdError):
        ev.add(disp[:1].to(DEV), depth_out=torch.empty((1, 224, 224), dtype=torch.float64, device=DEV))
    with pytest.raises(WmdError):
        compute_errors_nyu(torch.ones(4), torch.ones(4))
    with pytest.raises(WmdError):
        compute_errors_nyu(torch.ones(4, device=DEV), torch.ones(5, device=DEV))
