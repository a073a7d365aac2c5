"""GPU: decoder-level parity through the reference-facing API.

 * against the golden vectors the unmodified reference produced (tests/golden, small configs),
 * against the CPU oracle on the same seeded inputs, batched (oracle = per-sample reference semantics),
 * at BASELINE.json's full sizes through size-independent properties (sparse(thr<0) == dense, known-answer
   op counts, zero outside the wavelet mask, IDWT(DWT(x)) == x).
Float bar: 1e-4 relative (north_star).  Masks / counts / total_ops: exact.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import kitti as okitti
from oracle import nyu as onyu
from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import kitti_layers as kl
from wavelet_monodepth_b200 import nyu_decoders as nd
from wavelet_monodepth_b200 import ops, synth, wavelets

import footprint
from helpers import (REL_TOL, compare_outputs, golden_names, key_str, kitti_features, load_golden, nyu_features,
                     rel_err, seeded_params)

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _kitti(cls, meta):
    mod = cls(np.array(meta["num_ch_enc"]))
    sd = seeded_params(mod, meta)
    mod.load_state_dict(sd, strict=False)
    return mod.to(DEV).eval(), sd


def _nyu(cls, meta):
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    sd = seeded_params(mod, meta)
    mod.load_state_dict(sd, strict=False)
    return mod.to(DEV).eval(), sd


# ------------------------------------------------------------------------------------------ golden (reference outputs)
def test_kitti_dense_vs_reference_golden():
    want, meta = load_golden("kitti_tiny_dense")
    mod, _ = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    with torch.no_grad():
        got = mod(kitti_features(meta, DEV))
    compare_outputs(got, want, "kitti dense native")


@pytest.mark.parametrize("name", golden_names("kitti_tiny_sparse"))
def test_kitti_sparse_vs_reference_golden(name):
    want, meta = load_golden(name)
    mod, _ = _kitti(kd.SparseDepthWaveProgressiveDecoder, meta)
    got = mod(kitti_features(meta, DEV), meta["thresh_ratio"])
    compare_outputs(got, want, name)


def test_nyu_dense_vs_reference_golden():
    want, meta = load_golden("nyu_tiny_dense")
    mod, _ = _nyu(nd.DecoderWave, meta)
    with torch.no_grad():
        got = mod(nyu_features(meta, DEV))
    compare_outputs(got, want, "nyu dense native")


@pytest.mark.parametrize("name", golden_names("nyu_tiny_sparse"))
def test_nyu_sparse_vs_reference_golden(name):
    want, meta = load_golden(name)
    mod, _ = _nyu(nd.SparseDecoderWave, meta)
    got = mod(nyu_features(meta, DEV), meta["thresh_ratio"])
    compare_outputs(got, want, name)


# ------------------------------------------------------------------------------------------ batched vs per-sample oracle
@pytest.mark.parametrize("thr", [0.2, 0.25, 0.42])
def test_kitti_sparse_batched_equals_per_sample_oracle(thr):
    _, meta = load_golden("kitti_tiny_dense")
    mod, sd = _kitti(kd.SparseDepthWaveProgressiveDecoder, meta)
    feats = kitti_features(meta)                       # N = 2
    got = mod([f.to(DEV) for f in feats], thr)
    per = [okitti.sparse_forward(sd, [f[b:b + 1] for f in feats], thr) for b in range(2)]
    for k in per[0]:
        if k == "total_ops" or (isinstance(k, tuple) and k[0] == "total_ops"):
            assert got[k] == per[0][k] + per[1][k], k
            continue
        want = torch.cat([p[k] for p in per])
        if "mask" in key_str(k):
            assert torch.equal(got[k].cpu().bool(), want.bool()), k
        else:
            assert rel_err(got[k], want) <= REL_TOL, k
    assert got["total_ops_per_sample"] == [p["total_ops"] for p in per]


def test_nyu_sparse_batched_equals_per_sample_oracle():
    _, meta = load_golden("nyu_tiny_dense")
    mod, sd = _nyu(nd.SparseDecoderWave, meta)
    feats = nyu_features(meta)
    got = mod([f.to(DEV) for f in feats], 0.2)
    per = [onyu.sparse_forward(sd, [f[b:b + 1] for f in feats], 0.2) for b in range(2)]
    assert got["total_ops"] == per[0]["total_ops"] + per[1]["total_ops"]
    for k in per[0]:
        if k == "total_ops":
            continue
        want = torch.cat([p[k] for p in per])
        if "mask" in key_str(k):
            assert torch.equal(got[k].cpu().bool(), want.bool()), k
        else:
            assert rel_err(got[k], want) <= REL_TOL, k


# ------------------------------------------------------------------------------------------ training path
def test_dense_decoder_trains_through_native_idwt():
    """KITTI/trainer.py:208-212: gradients flow through inverse_wt.  Compare grads with the CPU oracle graph."""
    _, meta = load_golden("kitti_tiny_dense")
    mod, sd = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    mod.train()
    feats = kitti_features(meta)
    out = mod([f.to(DEV) for f in feats])
    loss = sum(out[("disp", s)].mean() for s in range(4))
    loss.backward()
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    with torch.enable_grad():
        o = okitti.dense_forward(params, feats)
        sum(o[("disp", s)].mean() for s in range(4)).backward()
    named = dict(mod.named_parameters())
    checked = 0
    for k, p in params.items():
        if p.grad is None:
            continue
        g = named[k].grad
        assert g is not None, k
        assert rel_err(g, p.grad) <= 1e-3, k
        checked += 1
    assert checked >= 30
    # and the native inference path agrees with the differentiable one
    mod.eval()
    with torch.no_grad():
        nat = mod([f.to(DEV) for f in feats])
    for s in range(4):
        assert rel_err(nat[("disp", s)], out[("disp", s)].detach()) <= REL_TOL


def test_weight_update_invalidates_packed_cache():
    _, meta = load_golden("kitti_tiny_dense")
    mod, _ = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    feats = kitti_features(meta, DEV)
    with torch.no_grad():
        a = mod(feats)[("disp", 0)].clone()
        for p in mod.parameters():
            p.mul_(1.05)
        b = mod(feats)[("disp", 0)]
    assert float((a - b).abs().max()) > 1e-4


# ------------------------------------------------------------------------------------------ functional API (reference wire format)
def test_functional_sparse_ops_vs_reference_golden():
    want, meta = load_golden("sparse_ops")
    cin, cout = meta["cin"], meta["cout"]
    conv = kl.Conv3x3(cin, cout)
    block = kl.ConvBlock(cin, cout, use_refl=True)
    seq = nn.Sequential(kl.Conv1x1(cin, cin), nn.LeakyReLU(0.1, inplace=True), kl.Conv3x3(cin, 3))
    for m in (conv, block, seq):
        m.load_state_dict(synth.random_state_dict(synth.module_shapes(m), seed=meta["param_seed"]), strict=False)
        m.to(DEV)
    for a in ("dense", "half", "few", "empty"):
        in_mask = torch.from_numpy(want["in_%s_mask" % a]).to(DEV)
        xvals = torch.from_numpy(want["in_%s_xvals" % a]).to(DEV)
        idxmap, n_ops = kl.mask2idxmap(in_mask)
        assert n_ops == meta["h"] * meta["w"] and idxmap.dtype == torch.int64
        for b in ("dense", "half", "few", "empty"):
            out_mask = torch.from_numpy(want["in_%s_mask" % b]).to(DEV)
            for pad in ("reflect", "constant", "replicate"):
                flat, c, n_ops = kl.sparse_conv3x3(conv, xvals, idxmap, out_mask, padding=pad, make_result=False)
                assert c == cout and n_ops == int(want["conv_%s_%s_%s_ops" % (a, b, pad)])
                assert rel_err(flat, want["conv_%s_%s_%s" % (a, b, pad)]) <= REL_TOL, (a, b, pad)
            dense, _ = kl.sparse_conv3x3(block, xvals, idxmap, out_mask)
            assert rel_err(dense, want["block_%s_%s" % (a, b)]) <= REL_TOL
            dense, n_ops = kl.sparse_conv3x3(seq, xvals, idxmap, out_mask, nonlin=torch.sigmoid)
            assert n_ops == int(want["head_%s_%s_ops" % (a, b)])
            assert rel_err(dense, want["head_%s_%s" % (a, b)]) <= REL_TOL
            sel = kl.sparse_select(xvals, cin, idxmap, out_mask, pad=True)
            assert torch.equal(sel.cpu(), torch.from_numpy(want["select_%s_%s" % (a, b)]))
    lo_mask = torch.from_numpy(want["in_half_mask"]).to(DEV)
    lo_idx, _ = kl.mask2idxmap(lo_mask)
    vals, ochn = kl.sparse_upsample(torch.from_numpy(want["up_lo_vals"]).to(DEV), cin, lo_idx,
                                    torch.from_numpy(want["up_skip"]).to(DEV),
                                    torch.from_numpy(want["up_hi_mask"]).to(DEV), make_result=False)
    assert ochn == cin + meta["cskip"] and torch.equal(vals.cpu(), torch.from_numpy(want["up_out"]))
    yx = kl.mask2yx(lo_mask)
    assert torch.equal(yx.cpu(), torch.nonzero(lo_mask[0, 0].cpu() > 0.5).t())


def test_reference_module_runs_on_native_wavelets():
    """sys.modules['pytorch_wavelets'] = wavelets is the documented drop-in: exercise that call convention."""
    idwt = wavelets.IDWT(wave="haar", mode="zero").to(DEV)
    yl = torch.rand(2, 1, 12, 40, device=DEV)
    yh = torch.rand(2, 1, 3, 12, 40, device=DEV)
    out = idwt((yl, list([yh])))
    assert out.shape == (2, 1, 24, 80)
    assert torch.equal(out, kd.SparseDepthWaveProgressiveDecoder.my_iwt_once((yl, [yh])))


# ------------------------------------------------------------------------------------------ BASELINE sizes: properties
def _full_kitti(ch, n, height, width, seed=1):
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(ch))
    synth.load_random(mod, seed=seed, gains={".2.conv.": 4.0})
    dense = kd.DepthWaveProgressiveDecoder(np.array(ch))
    dense.load_state_dict(mod.state_dict())
    feats = [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(3 + i))
             for i, s in enumerate(synth.kitti_feature_shapes(n, height, width, ch))]
    return mod.to(DEV).eval(), dense.to(DEV).eval(), feats


def test_full_size_r50_1024x320_known_answer_and_dense_equivalence():
    mod, dense, feats = _full_kitti(synth.RESNET50_CH, 2, 320, 1024)
    out = mod(feats, -1.0)
    assert out["total_ops_per_sample"] == [17473692295, 17473692295]     # KITTI/sparsity_test_notebook.ipynb:1345
    with torch.no_grad():
        d = dense(feats)
    for s in range(4):
        assert out[("disp", s)].shape == (2, 1, 320 >> s, 1024 >> s)
        assert rel_err(out[("disp", s)], d[("disp", s)]) <= REL_TOL
        assert bool(out[("wavelet_mask", s)].all())


def test_full_size_r18_640x192_bs16_sparse_properties():
    mod, dense, feats = _full_kitti(synth.RESNET18_CH, 16, 192, 640)
    out = mod(feats, 0.05)
    with torch.no_grad():
        d = dense(feats)
    # level 4 is dense in both: identical coarsest outputs
    assert rel_err(out[("disp", 3)], d[("disp", 3)]) <= REL_TOL
    for s in (2, 1, 0):
        m = out[("wavelet_mask", s)]
        for band in ("LH", "HL", "HH"):
            assert bool((out[("wavelets", s, band)][~m] == 0).all())
        # nesting of the dilated sets (SURVEY A.3)
        assert bool((out[("upconv1_mask", s)] | ~m).all()) and bool((out[("upsample_mask", s)] | ~out[("upconv1_mask", s)]).all())
        assert bool((out[("upconv0_mask", s)] | ~out[("lowres_mask", s)]).all())
    assert len(out["total_ops_per_sample"]) == 16 and out["total_ops"] == sum(out["total_ops_per_sample"])
    # determinism: same inputs, same bits
    out2 = mod(feats, 0.05)
    assert torch.equal(out[("disp", 0)], out2[("disp", 0)])


def test_full_size_nyu_densenet161_known_answer():
    mod = nd.SparseDecoderWave(enc_features=list(synth.DENSENET161_CH), decoder_width=0.5)
    synth.load_random(mod, seed=2)
    mod = mod.to(DEV).eval()
    dense = nd.DecoderWave(enc_features=list(synth.DENSENET161_CH), decoder_width=0.5)
    dense.load_state_dict(mod.state_dict())
    dense = dense.to(DEV).eval()
    feats = [torch.rand(s, device=DEV) for s in synth.nyu_feature_shapes(1, 480, 640, synth.DENSENET161_CH)]
    out = mod(feats, -10)
    assert out["total_ops"] == 33463546800                                 # NYUv2/sparsity_test_notebook.ipynb:1344
    with torch.no_grad():
        d = dense(feats)
    for s in range(4):
        assert rel_err(out[("disp", s)], d[("disp", s)]) <= REL_TOL
    assert out[("disp", 0)].shape == (1, 1, 240, 320)


def test_full_size_haar_round_trip_1024x320_bs32():
    x = torch.rand(32, 1, 320, 1024, device=DEV) * 80
    ll, hf = ops.dwt_haar(x)
    rec = ops.idwt_haar(ll, hf)
    assert rel_err(rec, x) <= 1e-6
    # linearity: IDWT(a) + IDWT(b) == IDWT(a + b) up to rounding
    ll2, hf2 = torch.rand_like(ll), torch.rand_like(hf)
    lhs = ops.idwt_haar(ll + ll2, hf + hf2)
    assert rel_err(lhs, rec + ops.idwt_haar(ll2, hf2)) <= 1e-6


def test_full_res_consumer_epilogue_matches_trainer_interpolate():
    """decoder.full_res_size -> ("disp_full", s) == F.interpolate(("disp", s), size, bilinear, align_corners=False)
    (KITTI/trainer.py:338-339), produced by the fused IDWT+bilinear kernel."""
    import torch.nn.functional as F
    _, meta = load_golden("kitti_tiny_dense")
    mod, _ = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    mod.full_res_size = (meta["height"], meta["width"])
    with torch.no_grad():
        out = mod(kitti_features(meta, DEV))
    for s in (1, 2, 3):
        want = F.interpolate(out[("disp", s)], mod.full_res_size, mode="bilinear", align_corners=False)
        assert float((out[("disp_full", s)] - want).abs().max()) <= 2e-6
    assert ("disp_full", 0) not in out


def test_cuda_graph_replay_matches_eager_and_follows_input_updates():
    """graphs.GraphedSparseDecoder: same kernels captured once; replay == eager bit for bit, also after the bound
    input tensors are overwritten in place (what a graphed encoder does).  Captured under the guarded, poisoning
    allocator (tests/footprint.py) and replayed on features A, B, then A again: the third replay equals the first and
    the eager run on A bit for bit, so no replay reads what an earlier one left behind or a buffer no kernel wrote, and
    no replay writes past a buffer."""
    from wavelet_monodepth_b200 import graphs
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 4, 192, 640)
    feats_a = [f.clone() for f in feats]
    torch.manual_seed(7)
    feats_b = [0.5 * f + 0.1 * torch.rand_like(f) for f in feats_a]

    def copy(out):
        return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in out.items()}

    def equal(got, want, what):
        assert set(got) == set(want), what
        for k, v in want.items():
            assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), (what, key_str(k))
    eager_a = copy(mod(feats_a, 0.05))
    eager_b = copy(mod(feats_b, 0.05))
    assert not torch.equal(eager_a[("disp", 0)], eager_b[("disp", 0)])
    feats = [f.clone() for f in feats_a]
    with footprint.Footprint() as fp:
        g = graphs.GraphedSparseDecoder(mod, feats, 0.05)
        assert g.launches > 40 and g.bound_to(feats) and not g.bound_to([f.clone() for f in feats])
        first = copy(g.replay())
        equal(first, eager_a, "replay on A")
        for f, b in zip(feats, feats_b):                     # new content in the same tensors
            f.copy_(b)
        equal(copy(g.replay()), eager_b, "replay on B")
        for f, a in zip(feats, feats_a):
            f.copy_(a)
        third = copy(g.replay())
        torch.cuda.synchronize()
    equal(third, first, "third replay against the first")
    equal(third, eager_a, "third replay on A")
    assert fp.checked >= fp.allocated > 0


def test_layout_move_options_are_bit_identical_eager_and_graphed():
    """gated_layout: a sparse level's skip map is transposed only under its upsample mask (the only rows upconv(i,1)
    reads).  That does not change what is computed: every output must equal the plain run bit for bit, launch by launch
    and inside a captured CUDA graph."""
    from wavelet_monodepth_b200 import graphs
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 3, 192, 640)
    mod.gated_layout = False
    mod.compact_skip = False                                 # gated_layout concerns the dense-row layout of the skip maps
    for thr in (0.05, 0.2, 0.4, 0.6, 0.8):                   # first threshold at which the gate really removes rows
        want = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in mod(feats, thr).items()}
        dens = float(want[("upsample_mask", 0)].float().mean())
        if 0.0 < dens < 0.9:
            break
    assert 0.0 < dens < 0.9, dens
    for gated in (False, True):
        mod.gated_layout = gated
        for _ in range(3):                                   # repeated: allocator reuse across the side streams
            got = mod(feats, thr)
            torch.cuda.synchronize()
            for k, v in want.items():
                assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), (gated, key_str(k))
        g = graphs.GraphedSparseDecoder(mod, feats, thr)
        for _ in range(2):
            got = g.replay()
            for k, v in want.items():
                assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), (gated, key_str(k))
        del g
    # gated move reading the two finest skip maps in place from pinned host memory (zero-copy over PCIe)
    on_host = [feats[0].cpu().pin_memory(), feats[1].cpu().pin_memory()] + list(feats[2:])
    got = mod(on_host, thr)
    torch.cuda.synchronize()
    for k, v in want.items():
        assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), ("host", key_str(k))
    g = graphs.GraphedSparseDecoder(mod, on_host, thr)
    got = g.replay()
    for k, v in want.items():
        assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), ("host graph", key_str(k))
    del g
    with pytest.raises(kd.WmdError):                         # pageable host memory is refused
        mod([feats[0].cpu()] + list(feats[1:]), thr)
    with pytest.raises(kd.WmdError):                         # a dense level's skip map must be on the device
        mod(list(feats[:3]) + [feats[3].cpu().pin_memory(), feats[4]], thr)
    mod.gated_layout = False
    with pytest.raises(kd.WmdError):                         # without the gated move nothing reads host memory
        mod(on_host, thr)


def test_fused_head_stages_match_the_two_launch_path():
    """fused_heads: levels 2 and 1 run their 1x1 head stages as one kernel (wmd_head_mlp_f32).  Both paths are
    fp32-faithful but sum in different orders: coefficients agree to 1e-5, masks to a handful of threshold ties."""
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 3, 192, 640)
    mod.fused_heads = False
    want = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in mod(feats, 0.05).items()}
    mod.fused_heads = True
    try:
        l0 = _lib_launches()
        got = mod(feats, 0.05)
        torch.cuda.synchronize()
        assert _lib_launches() - l0 < 75
    finally:
        mod.fused_heads = False
    for s in range(4):
        assert rel_err(got[("disp", s)], want[("disp", s)]) <= 1e-5, s
        for b in ("LH", "HL", "HH"):
            assert rel_err(got[("wavelets", s, b)], want[("wavelets", s, b)]) <= 1e-5, (s, b)
        flips = float((got[("wavelet_mask", s)] != want[("wavelet_mask", s)]).float().mean())
        assert flips <= 1e-4, (s, flips)


def _lib_launches():
    from wavelet_monodepth_b200 import _lib
    return _lib.launch_count()


# ------------------------------------------------------------------------------------------ host-side behaviour added in round 2
def test_async_op_count_future_equals_the_synchronous_ints_eager_and_graphed():
    """count_ops = "async": out["total_ops"] is an OpsFuture (no host wait in forward / replay); its result() carries
    exactly the keys and values the synchronous mode stores in the output dict."""
    from wavelet_monodepth_b200 import graphs
    from wavelet_monodepth_b200.opsfuture import OpsFuture
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 3, 192, 640)
    sync = mod(feats, 0.05)
    mod.count_ops = "async"
    try:
        out = mod(feats, 0.05)
        assert isinstance(out["total_ops"], OpsFuture) and ("total_ops", 0) not in out
        res = out["total_ops"].result()
        for k in ("total_ops", "total_ops_per_sample", ("total_ops", 0), ("total_ops", 1), ("total_ops", 2), ("total_ops", 3)):
            assert res[k] == sync[k], k
        assert int(out["total_ops"]) == sync["total_ops"]
        g = graphs.GraphedSparseDecoder(mod, feats, 0.05)
        futs = [g.replay()["total_ops"] for _ in range(7)]           # more replays in flight than pinned ring slots
        assert all(f.result()["total_ops"] == sync["total_ops"] for f in futs)
    finally:
        mod.count_ops = True
    nmod = nd.SparseDecoderWave(enc_features=[16, 16, 32, 64, 128], decoder_width=0.5)
    synth.load_random(nmod, seed=5, gains={"wave": 4.0})
    nmod = nmod.to(DEV).eval()
    nfeats = [torch.rand(s, device=DEV) for s in synth.nyu_feature_shapes(2, 96, 128, [16, 16, 32, 64, 128])]
    want = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in nmod(nfeats, 0.1).items()}
    g = graphs.GraphedSparseDecoder(nmod, nfeats, 0.1)                # NYU decoder under a CUDA graph
    got = g.replay()
    for k, v in want.items():
        assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), key_str(k)


def test_invalidate_packs_after_a_data_write_the_version_counter_cannot_see():
    _, meta = load_golden("kitti_tiny_dense")
    mod, _ = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    feats = kitti_features(meta, DEV)
    with torch.no_grad():
        a = mod(feats)[("disp", 0)].clone()
        for p in mod.parameters():
            p.data.mul_(1.05)                                         # invisible to p._version
        mod.invalidate_packs()
        b = mod(feats)[("disp", 0)].clone()
        assert float((a - b).abs().max()) > 1e-4
        sd = {k: v * 0.5 for k, v in mod.state_dict().items() if k.endswith("weight")}
        mod.load_state_dict(sd, strict=False)                         # post-hook invalidates
        c = mod(feats)[("disp", 0)]
        assert float((b - c).abs().max()) > 1e-4


def test_empty_batch_returns_empty_outputs_with_the_right_keys():
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 2, 192, 640)
    out = mod([f[:0] for f in feats], 0.05)
    assert out[("disp", 0)].shape == (0, 1, 192, 640) and out[("wavelet_mask", 1)].shape == (0, 1, 48, 160)
    assert out["total_ops"] == 0
    _, pix, off = ops.compact(torch.zeros((0, 1, 8, 8), dtype=torch.uint8, device=DEV))
    assert off.tolist() == [0] and pix.numel() == 0


def test_nan_coefficients_never_set_the_mask_like_torch_max():
    """torch.abs(yh).max(2)[0] > thresh is False where a band is NaN, and a NaN in yl makes every test False."""
    yh = torch.rand(2, 3, 16, 24, device=DEV) + 1.0
    yh[0, 1, 3, 4] = float("nan")
    yl = torch.rand(2, 1, 32, 48, device=DEV)
    yl[1, 0, 5, 5] = float("nan")
    thresh = ops.range_thresh(yl, 0.05)
    assert bool(torch.isnan(thresh[1])) and not bool(torch.isnan(thresh[0]))
    m = ops.level_masks(yh, thresh)
    want0 = (yh[0].abs().max(0)[0] > thresh[0])
    assert torch.equal(m["S0"][0, 0].bool(), want0) and not bool(m["S0"][0, 0, 3, 4])
    assert not bool(m["S0"][1].any())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_decoder_on_a_non_current_device():
    """ADVICE r1: model.to('cuda:1') while cuda:0 is current - kernels must launch on the tensors' device."""
    mod, _, feats = _full_kitti(synth.RESNET18_CH, 2, 192, 640)
    want = mod(feats, 0.05)
    mod1 = mod.to("cuda:1")
    feats1 = [f.to("cuda:1") for f in feats]
    assert torch.cuda.current_device() == 0
    got = mod1(feats1, 0.05)
    assert got[("disp", 0)].device.index == 1
    for s in range(4):
        assert torch.equal(got[("disp", s)].cpu(), want[("disp", s)].cpu())
    assert got["total_ops"] == want["total_ops"]


def test_npy_coefficient_dumps_as_test_simple_writes_them(tmp_path):
    """KITTI/test_simple.py:154-164 dumps, per scale, an (H_s, W_s, 4) float64 array [LL, LH, HL, HH] with np.save
    (evaluate_depth.py:231-235 does the same for the sparse decoder).  Same procedure on the native outputs and on the
    reference's golden outputs; the files must agree."""
    want, meta = load_golden("kitti_tiny_dense")
    mod, _ = _kitti(kd.DepthWaveProgressiveDecoder, meta)
    with torch.no_grad():
        outputs = mod(kitti_features(meta, DEV))
    coeffs = ["LL", "LH", "HL", "HH"]
    fh, fw = meta["height"], meta["width"]
    for scale in range(4):
        mine = np.zeros((fh // (2 ** (scale + 1)), fw // (2 ** (scale + 1)), 4))
        ref = np.zeros_like(mine)
        for j in range(4):
            mine[..., j] = outputs[("wavelets", scale, coeffs[j])].cpu()[0, 0].numpy()
            ref[..., j] = want["wavelets_%d_%s" % (scale, coeffs[j])][0, 0]
        np.save(tmp_path / ("x_scale_%d_wavelets.npy" % scale), mine)
        back = np.load(tmp_path / ("x_scale_%d_wavelets.npy" % scale))
        assert back.dtype == np.float64 and back.shape == ref.shape
        assert rel_err(back, ref) <= REL_TOL
    np.save(tmp_path / "x_disp.npy", outputs[("disp", 0)].cpu().numpy())
    assert rel_err(np.load(tmp_path / "x_disp.npy"), want["disp_0"]) <= REL_TOL


def test_fused_level_tail_is_bit_identical_to_the_three_kernel_chain_and_epilogue_matches_disp_to_depth(monkeypatch):
    """The fused level tail: head gather-sum -> yh -> IDWT -> disp -> next threshold in one kernel (wmd_head_idwt_f32) must
    equal the head_gather + idwt_haar + range_thresh chain bit for bit (same summation order), on sparse, masked-dense and
    dense levels, TMA-staged (W % 16 == 0) and plain staging; depth_range adds disp_to_depth(("disp", 0))
    (KITTI/layers.py:16-25)."""
    for ch, hw in ((synth.RESNET18_CH, (192, 640)), (synth.RESNET18_CH, (128, 256))):      # widths 40.. (plain) / 16.. (TMA)
        mod, dense, feats = _full_kitti(ch, 3, *hw)
        for scales in ([1, 2, 3], [1]):
            with monkeypatch.context() as m:
                m.setattr(kd, "_fused_tail_fits", lambda width: False)          # every level on the chain
                want = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in mod(feats, 0.05, scales).items()}
            got = mod(feats, 0.05, scales)
            assert set(got) == set(want)
            for k, v in want.items():
                assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), (hw, scales, key_str(k))
        with torch.no_grad(), monkeypatch.context() as m:
            m.setattr(kd, "_fused_tail_fits", lambda width: False)
            want = {k: v.clone() for k, v in dense(feats).items()}
        with torch.no_grad():
            got = dense(feats)
        for k, v in want.items():
            assert torch.equal(got[k], v), (hw, "dense", key_str(k))
        mod.depth_range = (0.1, 100.0)
        got = mod(feats, 0.05)
        disp = got[("disp", 0)]
        min_disp, max_disp = 1 / 100.0, 1 / 0.1                      # the reference's arithmetic, on the GPU by torch
        scaled = min_disp + (max_disp - min_disp) * disp
        assert torch.equal(got[("scaled_disp", 0)], scaled)
        assert rel_err(got[("depth", 0)], 1 / scaled) <= 1e-6
        mod.depth_range = None


def test_nyu_consumer_epilogue_depth_div_clamp():
    """NYUv2/utils.py:219,229: pred = clamp(outputs[("disp", 0)] / 100, 0.4, 10) - fused into the last IDWT."""
    yl = torch.rand(2, 1, 24, 32, device=DEV) * 800
    yh = (torch.rand(2, 1, 3, 24, 32, device=DEV) - 0.5) * 100
    out, depth = ops.idwt_haar(yl, yh, epilogue=("div_clamp", 100.0, 0.4, 10.0))
    assert torch.equal(out, ops.idwt_haar(yl, yh))
    assert torch.equal(depth, torch.clamp(out / 100, min=0.4, max=10))
    _, depth2 = ops.idwt_haar(yl, yh, epilogue=("div_clamp", 100.0, None, None))
    assert torch.equal(depth2, out / 100)


def test_cold_first_launch_equals_warm_launches_in_a_fresh_process():
    """Regression for two timing-dependent races that only showed on the COLD first launch of a kernel instantiation
    (registers of an asynchronous tcgen05.ld read before its wait; a raw stage handed back to the TMA before the row's
    shared-memory loads had landed): a fresh process runs the sparse decoder three times and every libwmd op's outputs
    of forward 0 must equal those of forwards 1 and 2 bit for bit (scripts/probe_determinism.py)."""
    import os
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(repo, "scripts", "probe_determinism.py"), "r18"], capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "done" in res.stdout and "DIFF" not in res.stdout and "shape" not in res.stdout, res.stdout[-3000:]


def test_compact_skip_rows_bit_identical_to_dense_skip_rows_device_and_pinned_host():
    """compact_skip: a sparse level moves only the rows of its upsample mask out of the NCHW skip map (list-based
    gather, wmd_gather_rows_list_f32) and upconv(i,1) reads them through S3's index map (wmd_conv_desc.map1) - same
    values in the same MMAs as the dense row layout: every output must be bit-identical, eager and graphed, with the skip
    maps on the device or in pinned host memory (read in place)."""
    from wavelet_monodepth_b200 import graphs
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(synth.RESNET18_CH))
    synth.bench_kitti_params(mod)                            # the bench workload: clustered masks, 7-30 % dense
    mod = mod.to(DEV).eval()
    feats = [f.to(DEV) for f in synth.bench_kitti_features(3, 192, 640, synth.RESNET18_CH)]
    mod.compact_skip = False
    want = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in mod(feats, 0.05).items()}
    assert 0.0 < float(want[("upsample_mask", 0)].float().mean()) < 0.9
    mod.compact_skip = True
    mod.compact_skip_levels = (1, 2, 3)
    on_host = [f.cpu().pin_memory() for f in feats[:3]] + list(feats[3:])
    for inputs in (feats, on_host):
        got = mod(inputs, 0.05)
        torch.cuda.synchronize()
        for k, v in want.items():
            assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), (inputs is on_host, key_str(k))
        g = graphs.GraphedSparseDecoder(mod, inputs, 0.05)
        got = g.replay()
        for k, v in want.items():
            assert (torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v), ("graph", inputs is on_host, key_str(k))
        del g
    with pytest.raises(kd.WmdError):                       # the dense level's skip map must be on the device
        mod(list(feats[:3]) + [feats[3].cpu().pin_memory(), feats[4]], 0.05)


def test_f16x3_operand_form_meets_the_same_parity_bars(monkeypatch):
    """f16x3: fp16-pair operands with per-tensor power-of-two scaling - the tiny sparse golden (reference outputs) and the
    batched-vs-per-sample oracle comparison hold at the tolerance of the default form, masks and total_ops exact; every
    tensor-core launch that has its sources' maxima really runs the f16 form."""
    seen = []
    real = ops.conv_rows

    def spy(*a, **kw):
        seen.append((kw.get("amax0") is not None, a[2].kind, a[2].data16 is not None))
        return real(*a, **kw)
    monkeypatch.setattr(kd.ops, "conv_rows", spy)
    for name in ("kitti_tiny_sparse_thr-1_s0", "kitti_tiny_sparse_thr0.2_s1"):
        want, meta = load_golden(name)
        mod, _ = _kitti(kd.SparseDepthWaveProgressiveDecoder, meta)
        got = mod(kitti_features(meta, DEV), meta["thresh_ratio"])
        compare_outputs(got, want, name + " f16x3")
    tc = [s for s in seen if s[1] == "tc"]
    assert tc and all(has_amax and has16 for has_amax, _, has16 in tc), tc
