"""GPU: the row-set form of the tensor-core convolution (conv_rows_tc_kernel_rowset, csrc/conv_tc.cu).

A 3x3 launch through a pixel list, an index map or a gate, on whole tiles or balanced, runs in the row-set kernel (tf32
launches with N = 128 tiles keep the gather kernel, so the contract cases with cout >= 96 check that one in tf32x3): per
tile and source the producer stages the distinct source rows once per channel chunk (TC_SET_ROWS = 480 of them at
most, within a row range of TC_SET_SPAN = 4096), and a source past either limit stages one slot per tap instead.  Which
of the two a tile takes must not change its bits: on whole tiles a row's sum does not depend on its tile, so the same
pixel list in raster order (distinct rows staged) and randomly permuted (most tiles past the limits) must give the
same rows.  Every launch is also checked against the fp64 contract reference (tests/conv_ref.py) at the bars of
test_gpu_conv_contract.py, with amax_out == max |y| and no writes outside [0, rows) x [0, cout).
"""
import pytest
import torch

from wavelet_monodepth_b200._lib import PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr
from conv_launch import (DEV, FLAGSHIP_DENSE, GATHER, SET, SET_ROWS, WIN, WORST, Layer, decoder_like, distinct_rows,
                         flagship_tc_kernels, gather_layer, mask, operands, run, tc_kernels)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def _pixels(cells, w, h):
    """Flat pixel indices of (image, y, x) cells, ascending."""
    return torch.tensor(sorted(n * h * w + y * w + x for n, y, x in cells), dtype=torch.int32, device=DEV)


def capacity_layer(extra):
    """Two images of 52 x 24, one 128-pixel tile each.  Image 0: 16 interior runs of 8 pixels, 3 rows apart, whose 3x3
    neighbourhoods do not touch: 16 x 3 x 10 = 480 distinct rows, exactly a slot.  Image 1 (extra = 1): runs of
    8 x 13 + 7 x 3 = 125 pixels on the same rows plus a run of 3 in the top row (2 x 5 rows): 375 + 96 + 10 = 481."""
    h, w = 52, 24
    runs0 = [(0, 3 + 3 * i, 2 + k) for i in range(16) for k in range(8)]
    lens = [8] * 13 + [7] * 3
    runs1 = [(1, 3 + 3 * i, 2 + k) for i, L in enumerate(lens) for k in range(L)] + [(1, 0, 5 + k) for k in range(3)]
    pix = _pixels(runs0 + (runs1 if extra else []), w, h)
    return Layer(2, h, w, 36, 64, c1=20, pad=PAD_ZERO, pixels=pix, count=len(pix))


def straddle_layer():
    """A pixel list over two images whose second tile holds the end of image 0 and the start of image 1."""
    m = mask((2, 16, 24), 0.5, 21)
    pix = cr.pixel_list(m)
    assert int(m[0].sum()) % 128 != 0
    return Layer(2, 16, 24, 40, 96, c1=12, pixels=pix, count=len(pix))


def gated_pad_layer(pad):
    """A dense grid through an all-ones gate: every tap row is read, with this padding."""
    return Layer(2, 13, 17, 24, 40, c1=8, pad=pad, gate=torch.ones(2 * 13 * 17, dtype=torch.uint8, device=DEV))


def scattered_layer():
    """A sparse list over a large image: a tile's rows span more than the bitmap (4096 rows), every tap is staged."""
    pix = cr.pixel_list(mask((1, 160, 160), 0.01, 22))
    return Layer(1, 160, 160, 32, 48, pixels=pix, count=len(pix))


def rowset_layer(case):
    if case == "capacity_480":
        return capacity_layer(0)
    if case == "capacity_481":
        return capacity_layer(1)
    if case == "straddle":
        return straddle_layer()
    if case == "scattered":
        return scattered_layer()
    if case == "count_zero":
        return Layer(1, 16, 24, 64, 96, pixels=cr.pixel_list(mask((1, 16, 24), 0.5, 12)), count=0)
    if case.startswith("gated_"):
        return gated_pad_layer({"gated_zero": PAD_ZERO, "gated_reflect": PAD_REFLECT,
                                "gated_replicate": PAD_REPLICATE}[case])
    return gather_layer(case)


CASES = ["shift0_compact_map0", "compact_map1", "gate", "count_lt_max_rows", "max_rows_lt_count", "decoder_level",
         "gated_zero", "gated_reflect", "gated_replicate", "count_zero", "straddle", "capacity_480", "capacity_481",
         "scattered"]


def test_capacity_tiles_are_what_they_say():
    """The capacity cases' first tiles hold exactly a slot's rows and one past it (host-side count of the tap rows)."""
    for extra, want in ((0, SET_ROWS), (1, SET_ROWS + 1)):
        L = capacity_layer(extra)
        tile = L.pixels[128 * extra:128 * (extra + 1)]
        assert len(tile) == 128
        assert distinct_rows(tile.cpu(), L.h, L.w, L.pad) == want


@pytest.mark.parametrize("dist", ["mixed", "same"])
@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("case", CASES)
def test_rowset_balanced_meets_the_contract(case, engine, dist):
    run(rowset_layer(case), engine, dist, "gather", splits=0, seed=31)


@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("layer", ["decoder_level", "compact_map1", "plain_list"])
def test_permuted_pixel_list_gives_the_same_rows(layer, engine):
    if layer == "decoder_level":
        L = decoder_like(2, 40, 64, 23)
    elif layer == "compact_map1":
        sel = mask((2, 40, 64), 0.5, 24)
        pix = cr.pixel_list(mask((2, 40, 64), 0.4, 25))
        L = Layer(2, 40, 64, 32, 48, c1=20, map1=cr.index_map(sel), pixels=pix, count=len(pix))
    else:
        pix = cr.pixel_list(mask((2, 40, 64), 0.3, 26))
        L = Layer(2, 40, 64, 36, 80, pad=PAD_REPLICATE, pixels=pix, count=len(pix))
    g = torch.Generator().manual_seed(27)
    perm = torch.randperm(L.count, generator=g).to(DEV)
    P = Layer(L.n, L.h, L.w, L.c0, L.cout, c1=L.c1, pad=L.pad, shift0=L.shift0, map0=L.map0, map1=L.map1, gate=L.gate,
              pixels=L.pixels[perm].contiguous(), count=L.count)
    ops_in = operands(L, "mixed", 28)
    want = run(L, engine, "mixed", "gather", splits=1, ops_in=ops_in)[:L.count]
    got = run(P, engine, "mixed", "gather", splits=1, ops_in=ops_in)[:L.count]
    back = torch.empty_like(got)
    back[perm] = got
    assert torch.equal(back, want)


def test_sparse_3x3_launches_run_the_rowset_kernel():
    """Not split (whole tiles, balanced): row set, except tf32 N = 128 tiles; split-K and 1x1: gather; dense windows
    that fit: window."""
    dense = Layer(2, 10, 32, 40, 64)
    one = Layer(2, 10, 32, 40, 64, taps=1)
    wide = rowset_layer("count_lt_max_rows")                  # cout 96: N = 128 tiles
    launches = [(rowset_layer(c), 0, "f16x3", SET) for c in ("decoder_level", "gate", "compact_map1")]
    launches += [(rowset_layer("decoder_level"), 1, "tf32x3", SET), (rowset_layer("decoder_level"), 3, "tf32x3", GATHER),
                 (wide, 0, "f16x3", SET), (wide, 0, "tf32x3", GATHER), (one, 0, "f16x3", GATHER), (dense, 0, "f16x3", WIN)]
    inputs = [operands(L, "mixed", 1) for L, _, _, _ in launches]
    names = tc_kernels(lambda: [run(L, e, "mixed", "gather", splits=s, ops_in=x)
                                for (L, s, e, _), x in zip(launches, inputs)], len(launches))
    assert names == [k for _, _, _, k in launches], names


def test_flagship_decoder_runs_its_sparse_3x3_launches_in_the_rowset_kernel():
    shapes, names = flagship_tc_kernels()
    want = [WIN if s in FLAGSHIP_DENSE else (SET if s[0] == 9 else GATHER) for s in shapes]
    assert want.count(SET) == 6, shapes
    assert names == want, list(zip(shapes, names))
