"""GPU: the NYUv2 depth boundary error on libwmd against the numpy/scipy oracle (oracle/nyu_edges.py) and the
reference's results (tests/golden/nyu_edges.npz, written by oracle/pin_nyu_edges.py from the unmodified NYUv2/utils.py).

Canny edges are bit-identical to the oracle's, distance maps to scipy's, scores within 1e-12 relative (the device sums
in a fixed order, numpy pairwise), with NaN and 10 exact."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import nyu_edges as ne
from oracle import nyu_eval as one
from wavelet_monodepth_b200 import nyu_decoders as nd
from wavelet_monodepth_b200._lib import WmdError
from wavelet_monodepth_b200.nyu_eval import NyuDepthEvaluator, compute_depth_boundary_error

from helpers import GOLDEN, load_golden, nyu_features, seeded_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
CROP = (slice(20, 460), slice(24, 616))


def load_fixture():
    with np.load(os.path.join(GOLDEN, "nyu_edges.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def fixture_splits(meta):
    yield "s%d" % meta["seed"], ne.edge_split(meta["seed"])
    yield "special", ne.edge_split(meta["special_seed"], special=True)


def unpack(packed, n, shape=(440, 592)):
    return np.unpackbits(packed)[:n * shape[0] * shape[1]].reshape((n,) + shape).astype(bool)


def assert_scores(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, got, want)
    exact = np.isnan(want) | (want == 10.0)
    assert np.array_equal(got[exact & ~np.isnan(want)], want[exact & ~np.isnan(want)]), (what, got, want)
    f = ~np.isnan(want)
    assert np.all(np.abs(got[f] - want[f]) <= 1e-12 * np.abs(want[f])), (what, got, want)


def check_against_oracle(edges_gt, pred, what):
    """compute_depth_boundary_error on the device vs the oracle, frame by frame"""
    acc, comp, est, d_est = compute_depth_boundary_error(torch.from_numpy(edges_gt).to(DEV),
                                                         torch.from_numpy(pred).to(DEV))
    est, d_est = est.cpu().numpy(), d_est.cpu().numpy()
    for i in range(pred.shape[0]):
        o_acc, o_comp, o_est, o_d = ne.dbe(edges_gt[i], pred[i])
        assert np.array_equal(est[i], o_est), (what, i, int((est[i] != o_est).sum()))
        assert np.array_equal(d_est[i].view(np.int64), ne.edt(est[i]).view(np.int64)), (what, i)
        assert_scores([float(acc[i]), float(comp[i])], [o_acc, o_comp], (what, i))
    return acc.cpu().numpy(), comp.cpu().numpy(), est


def test_functional_matches_the_oracle_and_the_reference_fixture():
    fx, meta = load_fixture()
    for name, split in fixture_splits(meta):
        pred = one.predict(split["disp"]).astype(np.float32)
        g = np.ascontiguousarray(split["edges"][(slice(None),) + CROP])
        acc, comp, est = check_against_oracle(g, pred, name)
        keep = meta["frames"][name]
        assert np.array_equal(est[keep], unpack(fx[name + "__f64_edges"], len(keep))), name
        assert_scores(np.stack([acc[keep], comp[keep]], 1), fx[name + "__f64_scores"], name)
        if name == "special":
            sp = split["special"]
            assert np.isnan(acc[sp["edge_free"]]) and np.isnan(comp[sp["edge_free"]])
            assert acc[sp["constant"]] == 10.0 and comp[sp["constant"]] == 10.0
            assert est[sp["spiral"]].sum() > 20000


def _scene_pred(rng, h, w):
    yy, xx = np.mgrid[0:h, 0:w] / np.array([max(h - 1, 1), max(w - 1, 1)])[:, None, None]
    d = 2.0 + yy + 0.5 * np.sin(6 * xx)
    d[h // 4:h // 2 + 1, w // 3:2 * w // 3 + 1] += 2.0
    return (d * rng.uniform(0.97, 1.03, (h, w))).astype(np.float32)


@pytest.mark.parametrize("h,w", [(1, 1), (2, 5), (13, 7), (440, 592), (480, 640)])
def test_functional_sizes(h, w):
    rng = np.random.default_rng(h * 1000 + w)
    pred = np.stack([_scene_pred(rng, h, w), _scene_pred(rng, h, w), np.full((h, w), 3.0, np.float32)])
    pred[1, h // 2, w // 2] = 0.0                                  # a zero is a NaN to the normalisation
    g = np.stack([ne.step_edges(p, 0.5) for p in pred]).astype(np.float32)
    g[1] = np.where(g[1] > 0, ne.as_k255(rng.integers(100, 256, (h, w))), 0)
    check_against_oracle(np.ascontiguousarray(g), pred, (h, w))
    # one frame as (h, w), and fp64 input rounded to float32
    acc, comp, est, d = compute_depth_boundary_error(torch.from_numpy(g[0]).to(DEV),
                                                     torch.from_numpy(pred[0].astype(np.float64)).to(DEV))
    o = ne.dbe(g[0], pred[0])
    assert est.shape == (h, w) and np.array_equal(est.cpu().numpy(), o[2])
    assert_scores([float(acc), float(comp)], o[:2], (h, w, "2-D"))


def evaluator_run(split, chunk=None, edges=True, depth=False):
    ev = NyuDepthEvaluator(split["gt"], edges_gt=split["edges"] if edges else None)
    d = torch.from_numpy(split["disp"]).to(DEV)
    n = d.shape[0]
    out = torch.empty((n, 440, 592), dtype=torch.float64, device=DEV) if depth else None
    step = chunk or n
    for i in range(0, n, step):
        ev.add(d[i:i + step], depth_out=None if out is None else out[i:i + step])
    return ev, out


def test_evaluator_against_the_reference_runs():
    fx, meta = load_fixture()
    for name, split in fixture_splits(meta):
        keep = meta["frames"][name]
        sub = {k: split[k][keep] for k in ("gt", "disp", "edges")}
        ev, depth = evaluator_run(sub, depth=True)
        scores = ev.edges_scores.cpu().numpy()
        assert_scores(scores, fx[name + "__f64_scores"], name)
        s = ev.summary()
        assert_scores([s["e_acc"], s["e_comp"]], fx[name + "__f64_e_edges"], name)
        # the reference's own float32 run: edge pixels that flip because the input is the rounded fp64 map
        _, _, est, _ = compute_depth_boundary_error(ev.edges_gt, depth.float())
        flips = int((est.cpu().numpy() != unpack(fx[name + "__f32_edges"], len(keep))).sum())
        print("%s: %d edge pixels differ from the reference's float32 run (CPU float32 vs float64 chain: %d)"
              % (name, flips, meta["flips_f32_vs_f64"][name]))
        assert flips <= 3 * meta["flips_f32_vs_f64"][name], (name, flips)
        if flips == 0:
            assert_scores(scores, fx[name + "__f32_scores"], (name, "f32"))


def test_evaluator_edge_free_frame_makes_the_mean_nan():
    split = ne.edge_split(7, special=True)
    ev, _ = evaluator_run(split)
    s = ev.summary()
    k = split["special"]["edge_free"]
    assert np.isnan(ev.edges_scores[k].cpu().numpy()).all()
    assert np.isnan(s["e_acc"]) and np.isnan(s["e_comp"])


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int64)


def test_chunking_repeats_graph_replay_and_depth_sums_are_bit_identical():
    split = ne.edge_split(3, n=11)
    whole, _ = evaluator_run(split)
    plain, _ = evaluator_run(split, edges=False)
    assert torch.equal(bits(whole.sums), bits(plain.sums))          # the depth metrics do not change with edges
    for chunk in (1, 5):
        ev, _ = evaluator_run(split, chunk)
        assert torch.equal(bits(ev.edges_scores), bits(whole.edges_scores)), chunk
        assert ev.summary() == whole.summary()
    again, _ = evaluator_run(split)
    assert torch.equal(bits(again.edges_scores), bits(whole.edges_scores))
    ev = NyuDepthEvaluator(split["gt"], edges_gt=split["edges"])
    d = torch.from_numpy(split["disp"]).to(DEV)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ev.add(d[:6])
        ev.add(d[6:])
    ev.edges_scores.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(ev.edges_scores), bits(whole.edges_scores))
    assert torch.equal(bits(ev.sums), bits(whole.sums))


def test_uint8_edge_maps_are_converted_like_evaluate_py():
    split = ne.edge_split(4, n=2)
    k = np.random.default_rng(4).integers(0, 256, split["edges"].shape).astype(np.uint8) * (split["edges"] > 0)
    a = NyuDepthEvaluator(split["gt"], edges_gt=k.astype(np.uint8))
    b = NyuDepthEvaluator(split["gt"], edges_gt=ne.as_k255(k))
    assert torch.equal(a.edges_gt, b.edges_gt)


def test_sparse_decoder_threshold_sweep_with_edges():
    _, meta = load_golden("nyu_tiny_dense")
    mod = nd.SparseDecoderWave(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    mod.load_state_dict(seeded_params(mod, meta), strict=False)
    mod = mod.to(DEV).eval()
    feats = nyu_features(meta, DEV)
    split = ne.edge_split(2, n=2)
    ev = NyuDepthEvaluator(split["gt"], edges_gt=split["edges"])
    for thr in (0.1, 0.2, 0.3):
        ev.reset()
        with torch.no_grad():
            disp = mod(feats, thr)[("disp", 0)]
        ev.add(disp)
        pred = one.predict(disp[:, 0].cpu().numpy()).astype(np.float32)
        want = np.array([ne.dbe(split["edges"][i][CROP], pred[i])[:2] for i in range(2)])
        assert_scores(ev.edges_scores.cpu().numpy(), want, thr)
        s = ev.summary()
        assert_scores([s["e_acc"], s["e_comp"]], want.mean(0), thr)


def test_bad_inputs_raise():
    split = ne.edge_split(0, n=2)
    gt, e = split["gt"], split["edges"]
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt, use_224=True, edges_gt=e)            # 224 mode has no Eigen crop for the edges
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt, edges_gt=e[:, :240])                 # wrong shape
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt, edges_gt=e[:1])                      # not one map per frame
    with pytest.raises(WmdError):
        NyuDepthEvaluator(gt, edges_gt=e.astype(np.float64))       # wrong dtype
    g = torch.from_numpy(e[:, 20:460, 24:616].copy())
    p = torch.full((2, 440, 592), 3.0)
    with pytest.raises(WmdError):
        compute_depth_boundary_error(g, p)                         # CPU tensors
    with pytest.raises(WmdError):
        compute_depth_boundary_error(g.to(DEV), p.to(DEV), mask=torch.ones(440, 592, device=DEV))
    with pytest.raises(WmdError):
        compute_depth_boundary_error(g.to(DEV), p[:, :100].to(DEV))
    with pytest.raises(WmdError):
        compute_depth_boundary_error(g.to(DEV), p.to(DEV).half())
