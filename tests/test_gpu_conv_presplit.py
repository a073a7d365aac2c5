"""GPU: the window and row-set kernels' fp16-pair operands split once per slot (csrc/conv_tc.cu, split_slot_rows).

In the f16x3 form the window and row-set kernels split a slot's fp32 rows into fp16 pairs in shared memory, once per
channel chunk, and read the fragments with ldmatrix; the gather kernel still splits every fragment element in
registers.  Both go through the same split, so they must give the same bits.  A dense 3x3 layer one row too wide for a
window runs in the gather kernel; the same layer through identity index maps and an all-ones gate runs in the row-set
kernel, which stages each tile's distinct rows once per channel chunk.  The two are compared bit for bit (int32 views:
NaN outputs included) on whole tiles and balanced, with mixed-sign and same-sign operands, cin % 32 != 0, N = 32 / 64 /
128 tiles, and operands holding NaN and +-Inf or spread over 2^-12 .. 2^-30 of their maximum (where the low piece h2
is an fp16 subnormal).  A permuted pixel list sends most row-set tiles to the per-tap fallback (128 gathered rows per
slot); a row's bits must not depend on which of the two staging forms its tile took.
"""
import pytest
import torch

from wavelet_monodepth_b200 import ops
from wavelet_monodepth_b200._lib import PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr
from conv_launch import (DEV, GATHER, SENTINEL, SET, SET_ROWS, Layer, decoder_like, dense_layer, distinct_rows, mask,
                         operands, pack, tc_kernels, twin)

pytestmark = pytest.mark.gpu

# (n, h, w, c0, c1, cout, pad, shift0): one past the widest window of each kind (the gather kernel runs them), and an
# N = 32 tile
TOO_WIDE = [
    (1, 3, 80, 32, 8, 64, PAD_ZERO, 0),
    (1, 4, 80, 20, 36, 48, PAD_REPLICATE, 1),
    (1, 2, 194, 40, 0, 128, PAD_REFLECT, 1),
    (2, 3, 81, 44, 0, 32, PAD_REFLECT, 0),
]


def _shape(x, c, values, seed):
    """Operand columns [0, c) of x in place: as drawn, with NaN / +Inf / -Inf at about 0.1 % of the elements each, or
    with element (r, k) scaled by 2^-(11 + e), e = (r + 3 k) % 20 (e = 0 keeps the maximum's scale, the rest span
    2^-12 .. 2^-30)."""
    v = x[:, :c]
    if values == "nonfinite":
        g = torch.Generator(device=DEV)
        g.manual_seed(seed)
        pick = torch.randint(0, 3000, v.shape, generator=g, device=DEV)
        v[pick == 0] = float("nan")
        v[pick == 1] = float("inf")
        v[pick == 2] = float("-inf")
    elif values == "tiny":
        r = torch.arange(v.shape[0], device=DEV).unsqueeze(1)
        k = torch.arange(c, device=DEV).unsqueeze(0)
        e = (r + 3 * k) % 20
        v.mul_(torch.where(e == 0, torch.ones_like(v), torch.exp2(-(11 + e).float())))


def _operands(L, dist, values, seed):
    x0, x1, wt, b = operands(L, dist, seed)
    _shape(x0, L.c0, values, seed + 1)
    if x1 is not None:
        _shape(x1, L.c1, values, seed + 2)
    return x0, x1, wt, b


def _amax(x, c):
    """max |x| over the finite operand columns, as the layers' producers report it"""
    v = x[:, :c].abs()
    return v[torch.isfinite(v)].max().reshape(1)


def launch(L, splits, ops_in):
    """One f16x3 launch; returns the output buffer and amax_out, bit patterns as int32."""
    x0, x1, wt, b = ops_in
    out = torch.full((L.max_rows + 5, ops.pad4(L.cout) + 4), SENTINEL, device=DEV)
    amax_out = torch.zeros(1, device=DEV)
    count = torch.tensor([L.count], dtype=torch.int32, device=DEV) if L.pixels is not None else None
    ops.conv_rows(x0, L.c0, pack(wt, L.c1, "f16x3"), b, L.cout, L.n, L.h, L.w, taps=9, pad=L.pad, map0=L.map0,
                  shift0=L.shift0, x1=x1, c1=L.c1, gate=L.gate, pixels=L.pixels, count=count, max_rows=L.max_rows,
                  out=out, splits=splits, map1=L.map1, amax0=_amax(x0, L.c0),
                  amax1=_amax(x1, L.c1) if L.c1 else None, amax_out=amax_out)
    return out.view(torch.int32), amax_out.view(torch.int32)


def test_too_wide_layers_run_the_gather_kernel_and_their_twins_the_rowset_kernel():
    launches = []
    for case in TOO_WIDE:
        L = dense_layer(case)
        launches += [(L, GATHER), (twin(L), SET)]
    inputs = [_operands(L, "mixed", "uniform", 1) for L, _ in launches]
    names = tc_kernels(lambda: [launch(L, 1, x) for (L, _), x in zip(launches, inputs)], len(launches))
    assert names == [k for _, k in launches], names


@pytest.mark.parametrize("values", ["uniform", "nonfinite", "tiny"])
@pytest.mark.parametrize("dist", ["mixed", "same"])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("case", TOO_WIDE)
def test_rowset_slot_split_gives_the_register_splits_bits(case, splits, dist, values):
    L = dense_layer(case)
    ops_in = _operands(L, dist, values, 5 * L.w + L.c0 + L.cout)
    y_reg, am_reg = launch(L, splits, ops_in)
    y_set, am_set = launch(twin(L), splits, ops_in)
    if values == "nonfinite":
        y = y_reg.view(torch.float32)[:L.rows, :L.cout]
        assert not bool(torch.isfinite(y).all()) and bool(torch.isfinite(y).any())
    assert torch.equal(y_set, y_reg)
    assert torch.equal(am_set, am_reg)


@pytest.mark.parametrize("values", ["uniform", "nonfinite", "tiny"])
@pytest.mark.parametrize("cout", [32, 80, 128])
@pytest.mark.parametrize("layer", ["plain_list", "decoder_level"])
def test_per_tap_fallback_gives_the_staged_forms_bits(layer, cout, values):
    """Raster order: tiles stage their distinct rows; permuted: the tiles' rows exceed a slot and are staged per tap
    (checked on the host for the plain list).  Whole tiles: a row's sum does not depend on its tile."""
    if layer == "plain_list":
        pix = cr.pixel_list(mask((2, 40, 64), 0.6, 26))
        L = Layer(2, 40, 64, 36, cout, pad=PAD_REPLICATE, pixels=pix, count=len(pix))
    else:
        D = decoder_like(2, 40, 64, 23)
        L = Layer(D.n, D.h, D.w, D.c0, cout, c1=D.c1, shift0=D.shift0, map0=D.map0, gate=D.gate, pixels=D.pixels,
                  count=D.count)
    g = torch.Generator().manual_seed(27)
    perm = torch.randperm(L.count, generator=g).to(DEV)
    P = Layer(L.n, L.h, L.w, L.c0, L.cout, c1=L.c1, pad=L.pad, shift0=L.shift0, map0=L.map0, map1=L.map1, gate=L.gate,
              pixels=L.pixels[perm].contiguous(), count=L.count)
    if layer == "plain_list":
        full = (L.count // 128) * 128
        raster = [distinct_rows(L.pixels[t:t + 128].cpu(), L.h, L.w, L.pad) for t in range(0, full, 128)]
        permuted = [distinct_rows(P.pixels[t:t + 128].cpu(), L.h, L.w, L.pad) for t in range(0, full, 128)]
        assert max(raster) <= SET_ROWS < min(permuted), (raster, permuted)
    ops_in = _operands(L, "mixed", values, 28)
    want, am_want = launch(L, 1, ops_in)
    got, am_got = launch(P, 1, ops_in)
    back = torch.empty_like(got[:L.count])
    back[perm] = got[:L.count]
    assert torch.equal(back, want[:L.count])
    assert torch.equal(got[L.count:], want[L.count:])
    assert torch.equal(am_got, am_want)
