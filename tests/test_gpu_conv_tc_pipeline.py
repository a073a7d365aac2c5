"""GPU: the warp-specialised tensor-core convolution when every CTA runs many tiles.

The layers here have two N tiles and several tiles per SM, so the producer warpgroup runs ahead across tile boundaries:
it builds the next tile's tap table and fills the ring with that tile's first chunks while the consumer warpgroups still
multiply the current tile and write its epilogue.  Whole tiles, split-K and balanced (stream-K) scheduling, and a 1x1
layer whose tiles are only four chunks long.
"""
import pytest
import torch
import torch.nn.functional as F

from wavelet_monodepth_b200 import ops
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, PAD_REFLECT

from helpers import REL_TOL, rel_err, rnd, torch_conv

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _tiles_per_sm(rows, cout):
    return (-(-rows // 128)) * (-(-cout // 128)) / torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("splits", [0, 1, 3])
def test_tc_many_tiles_per_cta_two_sources_vs_torch(splits):
    n, h, w, c0, c1, cout = 4, 96, 128, 64, 96, 256
    assert _tiles_per_sm(n * h * w, cout) > 4
    lo, skip = rnd(n, c0, h // 2, w // 2, seed=120), rnd(n, c1, h, w, seed=121)
    wt, b = rnd(cout, c0 + c1, 3, 3, seed=122, lo=-0.05, hi=0.05), rnd(cout, seed=123)
    x = torch.cat([F.interpolate(lo, scale_factor=2, mode="nearest"), skip], 1)
    want = torch_conv(x.to(DEV).double(), wt.to(DEV).double(), b.to(DEV).double(), PAD_REFLECT, ACT_ELU)
    lo_rows, skip_rows = ops.nchw_to_rows(lo.to(DEV)), ops.nchw_to_rows(skip.to(DEV))
    wp = ops.pack_weight(wt.to(DEV), c1, kind="tc")
    outs = [ops.conv_rows(lo_rows, c0, wp, b.to(DEV), cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, shift0=1,
                          x1=skip_rows, c1=c1, splits=splits).clone() for _ in range(2)]
    assert rel_err(ops.rows_to_nchw(outs[0], n, cout, h, w), want) <= REL_TOL
    assert torch.equal(outs[0], outs[1])


def test_tc_many_short_tiles_1x1_vs_torch():
    n, h, w, cin, cout = 4, 96, 128, 128, 256                # 4 chunks per tile
    assert _tiles_per_sm(n * h * w, cout) > 4
    x, wt, b = rnd(n, cin, h, w, seed=124), rnd(cout, cin, 1, 1, seed=125, lo=-0.1, hi=0.1), rnd(cout, seed=126)
    want = F.leaky_relu(F.conv2d(x.to(DEV).double(), wt.to(DEV).double(), b.to(DEV).double()), 0.1)
    rows, wp = ops.nchw_to_rows(x.to(DEV)), ops.pack_weight(wt.to(DEV), kind="tc")
    outs = [ops.conv_rows(rows, cin, wp, b.to(DEV), cout, n, h, w, taps=1, act=ACT_LRELU, act_param=0.1).clone()
            for _ in range(2)]
    assert rel_err(ops.rows_to_nchw(outs[0], n, cout, h, w), want) <= REL_TOL
    assert torch.equal(outs[0], outs[1])
