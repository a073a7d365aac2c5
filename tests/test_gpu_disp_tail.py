"""GPU: the fused baseline tail (wmd_disp_tail16_f32) against its fp64 contract reference (tests/disp_tail_ref.py).

Element by element |disp - disp64| <= BAR * S, S the error scale carried through both stages (see disp_tail_ref).  The
shapes put every border and corner of the reflected halo against the zero-padded upsampled source, include outputs 2
and 4 pixels thin, sizes that are not multiples of the 16 x 32 tile, several samples in one grid, cout 1..4 and ld > 16;
mixed-sign and same-sign operands.  Nothing outside ``disp`` may be written.
"""
import numpy as np
import pytest
import torch

from wavelet_monodepth_b200 import _lib, ops
from wavelet_monodepth_b200._lib import WmdError

from disp_tail_ref import BAR, disp_tail_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = 12345.0
GUARD = 4096


def _operands(n, h, w, cout, ld, seed, same_sign):
    rs = np.random.RandomState(seed)
    lo = 0.0 if same_sign else -1.0

    def u(*shape, scale=1.0):
        return torch.from_numpy((scale * rs.uniform(lo, 1.0, size=shape)).astype(np.float32)).to(DEV)
    x = u(n * h * w, ld, scale=2.0)
    return x, u(16, 16, 3, 3, scale=1 / 12), u(16, scale=0.1), u(cout, 16, 3, 3, scale=1 / 12), u(cout, scale=0.1)


def _run(x, w1, b1, w2, b2, n, h, w):
    """disp from the kernel, written into a view of a larger sentinel-filled buffer; returns (disp, guards intact)."""
    cout = int(w2.shape[0])
    numel = n * cout * 4 * h * w
    buf = torch.full((numel + 2 * GUARD,), SENTINEL, dtype=torch.float32, device=DEV)
    out = buf[GUARD:GUARD + numel].view(n, cout, 2 * h, 2 * w)
    ops.disp_tail16(x, ops.pack_disp_tail16(w1, b1, w2, b2), cout, n, h, w, out=out)
    torch.cuda.synchronize()
    intact = bool((buf[:GUARD] == SENTINEL).all() and (buf[GUARD + numel:] == SENTINEL).all())
    return out, intact


# (n, h, w) at half resolution: the output is (2h, 2w)
SHAPES = [
    (1, 1, 1), (2, 1, 3), (1, 2, 37), (3, 9, 21), (2, 8, 16), (1, 19, 2), (4, 13, 30), (2, 24, 80),
]


@pytest.mark.parametrize("same_sign", [False, True], ids=["mixed", "same_sign"])
@pytest.mark.parametrize("n,h,w", SHAPES)
def test_tail_matches_fp64_contract(n, h, w, same_sign):
    worst = 0.0
    for cout in (1, 2, 3, 4):
        ld = 16 if (n + cout) % 2 else 16 + 4 * cout
        x, w1, b1, w2, b2 = _operands(n, h, w, cout, ld, seed=100 * n + 10 * h + w + cout, same_sign=same_sign)
        got, intact = _run(x, w1, b1, w2, b2, n, h, w)
        assert intact, "the kernel wrote outside disp"
        want, s = disp_tail_ref(x, w1, b1, w2, b2, n, h, w)
        ratio = ((got.double() - want).abs() / s.clamp(min=1e-30)).max().item()
        worst = max(worst, ratio)
        assert ratio <= BAR, (cout, ld, ratio)
    print("disp_tail16 %s n=%d %dx%d: worst |err| / S = %.3g" % ("same-sign" if same_sign else "mixed", n, 2 * h, 2 * w,
                                                                  worst))


def test_full_size_level0_matches_fp64_contract():
    """ResNet18 640x192 level 0 (upconv(0,0) at 320x96), two samples."""
    n, h, w = 2, 96, 320
    x, w1, b1, w2, b2 = _operands(n, h, w, 1, 16, seed=7, same_sign=False)
    got, intact = _run(x, w1, b1, w2, b2, n, h, w)
    assert intact
    want, s = disp_tail_ref(x, w1, b1, w2, b2, n, h, w)
    ratio = ((got.double() - want).abs() / s).max().item()
    print("disp_tail16 640x192 x2: worst |err| / S = %.3g" % ratio)
    assert ratio <= BAR


def test_tail_is_bit_identical_across_launches():
    x, w1, b1, w2, b2 = _operands(3, 9, 21, 3, 16, seed=3, same_sign=False)
    packed = ops.pack_disp_tail16(w1, b1, w2, b2)
    a = ops.disp_tail16(x, packed, 3, 3, 9, 21)
    b = ops.disp_tail16(x, packed, 3, 3, 9, 21)
    assert torch.equal(a, b)


def test_empty_batch_launches_nothing():
    x, w1, b1, w2, b2 = _operands(1, 4, 4, 2, 16, seed=4, same_sign=False)
    packed = ops.pack_disp_tail16(w1, b1, w2, b2)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    out = ops.disp_tail16(x[:0], packed, 2, 0, 4, 4)
    assert _lib.launch_count() == before
    assert out.shape == (0, 2, 8, 8)


def test_bad_arguments_are_refused():
    x, w1, b1, w2, b2 = _operands(1, 4, 4, 2, 16, seed=5, same_sign=False)
    packed = ops.pack_disp_tail16(w1, b1, w2, b2)
    with pytest.raises(WmdError):
        ops.disp_tail16(x.cpu(), packed, 2, 1, 4, 4)                          # host rows
    with pytest.raises(WmdError):
        ops.disp_tail16(x[:, :12].contiguous(), packed, 2, 1, 4, 4)         # ld < 16
    with pytest.raises(WmdError):
        ops.pack_disp_tail16(w1, b1, torch.zeros(5, 16, 3, 3, device=DEV), None)   # cout > 4
