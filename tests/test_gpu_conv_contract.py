"""GPU: the gather-GEMM convolutions against the fp64 reference of the whole wmd_conv_desc contract (tests/conv_ref.py).

Metric: err = max over the written elements of |y - y64| / S, with S = |bias| + sum |a| |w| (the magnitudes of every term
of the element's dot product).  An fp32-faithful kernel's error is a small multiple of 2^-22 S whatever the data; a kernel
that drops a correction term, a slab or the bias, or lets the tensor core's truncating accumulation run too long, is off
by 1e-4 S or more on some element.  With an activation the slope is <= 1 and the activation's own error (ELU / sigmoid
< 5e-7 absolute, test_conv_epilogue_elu_matches_expm1_over_the_whole_range) is allowed on top.

Operands are mixed-sign (x, w, b uniform in [-1, 1]) or same-sign (x, b in [0, 1], w in [0, 2/K]): the second does not
cancel a one-signed bias, which is what the tensor core's truncating accumulation has.  Every launch also checks that
nothing outside [0, min(count, max_rows)) x [0, cout) of `out` changes (the buffer is prefilled with a sentinel, and the
source rows carry huge values in their padding columns, which must not be read), and that amax_out is exactly max |y|.

Model of the bars: a tf32x3 / f16x3 product carries ~22 mantissa bits (~2^-20 of |a w|); on top of that each accumulation
epoch (K <= 1024) carries the tensor core's truncation bias, which grows with the number of MMAs that add into the
accumulators.  tf32x3 issues 3 MMAs of K = 8 per 8 channels, f16x3 3 MMAs of K = 16 per 16, so tf32x3's bias is twice
f16x3's.  SIMT: fp32 FMA chains with round-to-nearest (no bias, error ~ sqrt(K) 2^-24).

Worst observed err on one H100 80GB HBM3 (132 SMs, 700 W power limit), per case group, mixed-sign | same-sign
(- = not run):
    group       tf32x3              f16x3               simt
    tails       1.5e-6 | 1.4e-5     8.6e-7 | 7.4e-6     2.7e-7 | 1.6e-6
    epochs      1.6e-6 | 1.7e-5     8.7e-7 | 8.6e-6     2.6e-7 | 2.0e-6
    K18432           - | 1.6e-5          - | 8.1e-6          - | 6.5e-6
    schedules   1.6e-6 | 1.0e-5     8.1e-7 | 3.2e-6          - | -
    splits      8.2e-7 | 4.8e-6          - | -               - | -
    gather      1.6e-6 | 9.3e-6     9.7e-7 | 5.3e-6     2.3e-7 | 1.3e-6
    rows0       4.3e-7 | 1.1e-6     2.4e-7 | 5.6e-7          - | -
    epilogue    1.3e-6 | -          5.8e-7 | -          2.5e-7 | -
    grid        1.8e-6 | -               - | -               - | -
    workspace   1.8e-6 | -               - | -               - | -
The same-sign worst is the truncation bias of one full epoch: ~1.6e-8 x K of S for tf32x3, ~8.5e-9 x K for f16x3 (K <= 1024
per epoch), so it does not grow past one epoch.  Bars: 2.4x (tf32x3), 2.9x (f16x3) and 2.3x (simt) the worst observed;
kernels with a correction term, a slab, the bias or the epochs removed were off by 1.0e-4 S or more on some element.
"""
import pytest
import torch

from wavelet_monodepth_b200 import _lib, ops
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr
from conv_launch import DEV, WORST, Layer, gather_layer, mask, operands, run, sm_count

pytestmark = pytest.mark.gpu
ENGINES = ["tf32x3", "f16x3", "simt"]
DISTS = ["mixed", "same"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


# ------------------------------------------------------------------------------------------ N tiles and channel tails
# (cout, c0, c1, n, h, w, pad): cout straddles tc_tile_n's 48 / 96 switches (1-3 N tiles with tails), c0 % 32 in {0, 8, 20},
# c1 in {0, 20, 64}, cin % 4 != 0, rows % 128 in {0, 1, 127}
TAILS = [
    (5, 6, 0, 1, 8, 16, PAD_REFLECT),
    (31, 20, 0, 1, 3, 43, PAD_ZERO),
    (32, 64, 20, 1, 5, 51, PAD_REPLICATE),
    (47, 40, 0, 2, 8, 8, PAD_REFLECT),
    (48, 32, 64, 1, 3, 43, PAD_REFLECT),
    (63, 52, 20, 1, 5, 51, PAD_ZERO),
    (64, 8, 0, 2, 4, 16, PAD_REPLICATE),
    (95, 72, 64, 1, 3, 43, PAD_REFLECT),
    (96, 96, 0, 1, 5, 51, PAD_REFLECT),
    (128, 40, 20, 2, 8, 8, PAD_ZERO),
    (129, 64, 0, 1, 3, 43, PAD_REPLICATE),
    (138, 84, 20, 1, 5, 51, PAD_REFLECT),
    (257, 33, 0, 1, 8, 16, PAD_REFLECT),
]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("cout,c0,c1,n,h,w,pad", TAILS)
def test_tails(cout, c0, c1, n, h, w, pad, engine, dist):
    run(Layer(n, h, w, c0, cout, c1=c1, pad=pad), engine, dist, "tails", seed=cout)


# ------------------------------------------------------------------------------------------ reduction length and epochs
@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
@pytest.mark.parametrize("cin", [992, 1024, 1056, 2080])          # 31, 32, 33 and 65 chunks of one tap
def test_epoch_edges_1x1(cin, engine, splits, dist):
    run(Layer(1, 4, 128, cin, 96, taps=1), engine, dist, "epochs", splits=splits, seed=cin)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
def test_longest_decoder_reduction_same_sign(engine, splits):
    """upconv(4, 0)'s K = 9 x 2048 = 18 432 on post-ELU-like (non-negative) inputs: 18 epochs per whole tile."""
    run(Layer(1, 8, 40, 2048, 256), engine, "same", "K18432", splits=splits, seed=40)


# ------------------------------------------------------------------------------------------ schedules
SCHEDULES = ["3", "sm-1", "sm", "sm+1", "1.5sm", "2sm", "2.3sm", "5.3sm"]


def _tiles(label):
    sm = sm_count()
    return {"3": 3, "sm-1": sm - 1, "sm": sm, "sm+1": sm + 1, "1.5sm": (3 * sm) // 2, "2sm": 2 * sm,
            "2.3sm": (23 * sm) // 10, "5.3sm": (53 * sm) // 10}[label]


@pytest.mark.parametrize("engine,splits,dist", [("tf32x3", 1, "mixed"), ("tf32x3", 0, "mixed"), ("tf32x3", 0, "same"),
                                                ("f16x3", 0, "mixed")])
@pytest.mark.parametrize("label", SCHEDULES)
def test_schedules_by_tile_count(label, engine, splits, dist):
    """One N tile (cout 96 in a 128-wide tile), 18 chunks; the tile count relative to the SM count picks stream-K with up
    to 7 segments (few tiles), 3-slab stream-K (one round and a part), data-parallel rounds + remainder, or none."""
    run(Layer(1, _tiles(label), 128, 64, 96), engine, dist, "schedules", splits=splits, seed=7)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("splits", [0, 1, 2, 5, 9, 12])             # 9 chunks: nchunks and nchunks + 3 (clamped)
def test_splits(splits, dist):
    run(Layer(1, 3, 128, 32, 64), "tf32x3", dist, "splits", splits=splits, seed=8)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ["tf32x3", "f16x3"])
def test_balanced_cut_tiles_with_cout_tail(engine, dist):
    """cout 138: two N tiles, the second with a 10-column tail; 18 tiles on all SMs: every tile is cut."""
    run(Layer(1, 9, 128, 256, 138, c1=0), engine, dist, "schedules", splits=0, seed=9)


# ------------------------------------------------------------------------------------------ gather paths
GATHER = ["shift0_compact_map0", "compact_map1", "gate", "count_lt_max_rows", "max_rows_lt_count", "decoder_level",
          "pad_zero", "pad_reflect", "pad_replicate", "thin_1_37_z", "thin_1_37_r", "thin_2_33_f", "thin_40_1_r",
          "thin_35_2_f", "thin_1_1_z"]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", GATHER)
def test_gather_paths(case, engine, dist):
    run(gather_layer(case), engine, dist, "gather", seed=11)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 2), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
def test_count_zero_writes_nothing(engine, splits):
    pix = cr.pixel_list(mask((1, 16, 24), 0.5, 12))
    run(Layer(1, 16, 24, 64, 96, pixels=pix, count=0), engine, "mixed", "gather", splits=splits, seed=12)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1)])
def test_1x1_rows_past_rows0_read_zeros(engine, splits, dist):
    """The tensor-core engine's 1x1 form over x0's own rows: x0 holds 300 of the 384 rows (the cut falls inside a tile);
    the rest read zeros from source 0 and still read source 1."""
    run(Layer(1, 6, 64, 40, 64, c1=16, taps=1, x0_rows=300), engine, dist, "rows0", splits=splits, seed=13)


# ------------------------------------------------------------------------------------------ epilogue
def _epi_layer():
    return Layer(1, 9, 128, 64, 138)                 # 2 N tiles (10-column tail), 18 tiles: balanced cuts every tile


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0)])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_ELU, ACT_LRELU, ACT_SIGMOID])
def test_activations(act, engine, splits):
    run(_epi_layer(), engine, "mixed", "epilogue", splits=splits, act=act, seed=14)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
@pytest.mark.parametrize("bias", ["none", "off1", "off2", "off3"])
def test_bias_none_and_unaligned_views(bias, engine, splits):
    """bias may be any 4-byte aligned pointer: 1, 2 and 3 floats into an allocation, on whole tiles and on cut tiles."""
    run(_epi_layer(), engine, "mixed", "epilogue", splits=splits, act=ACT_ELU, bias=bias, seed=15)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 2), ("tf32x3", 3), ("f16x3", 0),
                                           ("simt", None)])
def test_dense_capacity_past_the_image(engine, splits):
    """pixels == NULL with a capacity (max_rows) larger than the image: only the image's rows are written, in every mode."""
    run(Layer(1, 5, 51, 64, 96, max_rows=255 + 130), engine, "mixed", "epilogue", splits=splits, seed=16)


# ------------------------------------------------------------------------------------------ grid independence
def test_results_do_not_depend_on_the_grid():
    """wmd_conv_tc_set_reserved_sms shrinks the persistent grid.  Whole tiles: bit-identical for every grid (a tile's
    arithmetic does not depend on which CTA runs it or where it falls in the ring).  Balanced: within the bar and
    reproducible for every grid."""
    sm = sm_count()
    lib = _lib.load()
    L = Layer(1, 40, 128, 64, 138, c1=32)            # 80 tiles, 27 chunks
    ins = operands(L, "mixed", 17)
    was = lib.wmd_conv_tc_set_reserved_sms(-1)
    whole = []
    try:
        for k in [0, 1, sm // 2, sm - 2, sm - 1]:
            lib.wmd_conv_tc_set_reserved_sms(k)
            whole.append(run(L, "tf32x3", "mixed", "grid", splits=1, ops_in=ins))
            a = run(L, "tf32x3", "mixed", "grid", splits=0, ops_in=ins)
            b = run(L, "tf32x3", "mixed", "grid", splits=0, ops_in=ins)
            assert torch.equal(a, b), k
    finally:
        lib.wmd_conv_tc_set_reserved_sms(was)
    for k, o in enumerate(whole[1:]):
        assert torch.equal(o, whole[0]), k


# ------------------------------------------------------------------------------------------ workspace hygiene
def test_balanced_launches_leave_the_workspace_counters_zero():
    """Back-to-back balanced launches of different tile counts share one scratch buffer; each stays within the bar, and
    the arrival counters at its head are zero afterwards."""
    sm = sm_count()
    for i, tiles in enumerate([3, sm + 1, 2 * sm + 7, 5, sm - 1]):
        run(Layer(1, tiles, 128, 96, 64), "tf32x3", "mixed", "workspace", splits=0, seed=20 + i)
    torch.cuda.synchronize()
    ws = ops._scratch.splitk(torch.device(DEV), 4096)
    assert bool((ws[:1024] == 0).all())
