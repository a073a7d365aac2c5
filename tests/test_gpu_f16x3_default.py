"""GPU: the fp16-pair operand form (f16x3) as the KITTI decoders' default.

- Every layout move of a sparse level's skip map reports the max |x| of exactly the pixels upconv(i,1) reads (the level's
  upsample mask S3), whether it is plain, gated, list-based or a channels_last view used in place.  The operand scale is a
  power of two taken from that maximum, so the layout options pick the same scale and give the same bits.
- The flagship decoder (ResNet50 pyramid, 1024x320) runs every tensor-core launch in f16x3.
- The shared-memory ring is 6 stages deep for f16 N = 128 tiles and 8 for N = 64 / 32.  Contract cases whose chunk counts
  per tile are not multiples of the ring depth put the tile boundaries at changing ring offsets, with several tiles per CTA
  (whole tiles) and stream-K segments (balanced); each is checked against the fp64 reference of tests/conv_ref.py.
"""
import numpy as np
import pytest
import torch

from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import _lib, ops, synth

from conv_launch import DEV, WORST, Layer, run, sm_count

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def _map_and_gate(n, c, h, w, p, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c, h, w), generator=g) * 37.0
    gate = (torch.rand((n, 1, h, w), generator=g) < p).to(torch.uint8)
    # the largest value of the map lies on an unmarked pixel of a 32-pixel group that holds a marked one: the gated move
    # reads that group, but the pixel's row is never read by the consumer
    m0 = gate[0].reshape(-1).bool()
    off = next(j for j in range(h * w) if not m0[j] and bool(m0[32 * (j // 32):32 * (j // 32) + 32].any()))
    x.view(n, c, h * w)[0, 0, off] = 1.0e4
    return x.to(DEV), gate.to(DEV)


@pytest.mark.parametrize("n,c,h,w,p", [(2, 70, 12, 40, 0.3), (1, 33, 9, 130, 0.6), (2, 64, 16, 48, 0.05)])
def test_skip_map_moves_report_the_maximum_over_the_mask(n, c, h, w, p):
    x, gate = _map_and_gate(n, c, h, w, p, seed=80 + c)
    marked = gate.reshape(-1).bool()
    want = float(x.permute(0, 2, 3, 1).reshape(-1, c)[marked].abs().max())
    assert want < 1.0e4
    got = {}

    def amax(name):
        got[name] = torch.zeros(1, device=DEV)
        return got[name]
    rows_g = ops.nchw_to_rows(x, gate=gate, amax=amax("gated"))
    rows_p = ops.nchw_to_rows(x, amax=amax("plain"), amax_mask=gate)           # the mask restricts only the maximum
    _, pixels, offsets = ops.compact(gate, want_idxmap=False)
    ops.gather_rows_list(x, pixels, offsets[n:], amax=amax("list"))
    if c % 4 == 0:                                                              # channels_last views, used in place
        xcl = x.contiguous(memory_format=torch.channels_last)
        ops.nchw_to_rows(xcl, gate=gate, amax=amax("view gated"))
        ops.nchw_to_rows(xcl, amax=amax("view masked"), amax_mask=gate)
    assert {k: float(v) for k, v in got.items()} == {k: want for k in got}, want
    whole = torch.zeros(1, device=DEV)
    ops.nchw_to_rows(x, amax=whole)                                            # without a mask: the whole map
    assert float(whole) == 1.0e4
    assert torch.equal(rows_p[:, :c], x.permute(0, 2, 3, 1).reshape(-1, c))
    assert torch.equal(rows_g[marked][:, :c], x.permute(0, 2, 3, 1).reshape(-1, c)[marked])


def test_masked_row_maximum_of_a_view():
    g = torch.Generator().manual_seed(3)
    rows = torch.randn((1000, 52), generator=g).to(DEV)
    mask = (torch.rand(1000, generator=g) < 0.1).to(torch.uint8).to(DEV)
    rows[~mask.bool()] *= 100.0
    out = torch.zeros(1, device=DEV)
    ops.amax_rows(rows, out, mask=mask)
    assert float(out) == float(rows[mask.bool()].abs().max())
    none = torch.zeros(1, device=DEV)
    ops.amax_rows(rows, none, mask=torch.zeros(1000, dtype=torch.uint8, device=DEV))
    assert float(none) == 0.0


def test_flagship_decoder_runs_every_tensor_core_launch_in_f16x3_without_configuration():
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(synth.RESNET50_CH))
    synth.bench_kitti_params(mod)
    mod = mod.to(DEV).eval()
    feats = [f.to(DEV) for f in synth.bench_kitti_features(2, 320, 1024, synth.RESNET50_CH)]
    mod(feats, 0.05)
    prof = ops.Profiler()
    torch.cuda.synchronize()
    ops.set_profiler(prof)
    try:
        mod(feats, 0.05)
        torch.cuda.synchronize()
    finally:
        ops.set_profiler(None)
    tc = [info for name, _, info in prof.results() if name == "conv_rows_tc"]
    assert len(tc) >= 8, len(tc)
    assert all(info["f16"] for info in tc), [(info["taps"], info["c0"], info["c1"], info["cout"]) for info in tc
                                             if not info["f16"]]


# (cout, c0, c1, taps): tile width N, chunks per tile, ring depth S; tile boundaries fall at chunk g = k * chunks of a CTA,
# i.e. at ring offsets (k * chunks) % S
RING = [
    (128, 224, 0, 1),     # N = 128, 7 chunks, S = 6: offsets 1, 2, 3, 4, 5, 0
    (96, 40, 20, 9),      # N = 128, 27 chunks, S = 6: offsets 3, 0, 3
    (64, 416, 0, 1),      # N = 64, 13 chunks, S = 8: offsets 5, 2, 7
    (48, 32, 0, 9),       # N = 64, 9 chunks, S = 8: offsets 1, 2, 3
    (40, 64, 36, 9),      # N = 32, two N tiles (8-column tail), 36 chunks (an epoch boundary inside), S = 8: offsets 4, 0
    (32, 160, 0, 1),      # N = 32, 5 chunks, S = 8: offsets 5, 2, 7
]


@pytest.mark.parametrize("dist", ["mixed", "same"])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("cout,c0,c1,taps", RING)
def test_f16x3_ring_wraps_across_tile_boundaries(cout, c0, c1, taps, splits, dist):
    n_tiles = -(-cout // _lib.load().wmd_conv_tc_tile_n(cout))
    h = (7 * sm_count()) // (2 * n_tiles) + 1                       # ~3.5 tiles per CTA, rows of 128 pixels
    run(Layer(1, h, 128, c0, cout, c1=c1, taps=taps), "f16x3", dist, "ring", splits=splits, seed=cout + c0)
