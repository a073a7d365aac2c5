"""CPU: the fp64 reference of the fused baseline tail (tests/disp_tail_ref.py) against an independent F.conv2d composition
of upconv(0,1) -> dispconv(0) -> sigmoid, value and error scale, exactly (fp64 sums in another order: <= 1e-12)."""
import pytest
import torch
import torch.nn.functional as F

from disp_tail_ref import disp_tail_ref
from helpers import close, rnd, rows_of


def _composition(x, w1, b1, w2, b2):
    up = F.interpolate(x.double(), scale_factor=2, mode="nearest")
    pre1 = F.conv2d(F.pad(up, (1, 1, 1, 1)), w1.double(), b1.double())
    s1 = F.conv2d(F.pad(up.abs(), (1, 1, 1, 1)), w1.double().abs(), b1.double().abs())
    u = F.elu(pre1)
    ur = F.pad(u, (1, 1, 1, 1), mode="reflect")
    disp = torch.sigmoid(F.conv2d(ur, w2.double(), b2.double()))
    s = F.conv2d(ur.abs(), w2.double().abs(), b2.double().abs()) + \
        F.conv2d(F.pad(s1, (1, 1, 1, 1), mode="reflect"), w2.double().abs())
    return disp, s


@pytest.mark.parametrize("n,h,w,cout,ld", [(2, 3, 5, 1, 16), (1, 1, 1, 4, 20), (1, 4, 2, 3, 16), (3, 2, 7, 2, 24)])
def test_matches_conv2d_composition(n, h, w, cout, ld):
    x = rnd(n, 16, h, w, seed=1)
    w1, b1, w2, b2 = rnd(16, 16, 3, 3, seed=2), rnd(16, seed=3), rnd(cout, 16, 3, 3, seed=4), rnd(cout, seed=5)
    rows = torch.cat([rows_of(x), rnd(n * h * w, ld - 16, seed=6)], 1)      # columns past 16 are not read
    got, s = disp_tail_ref(rows, w1, b1, w2, b2, n, h, w)
    want, want_s = _composition(x, w1, b1, w2, b2)
    assert got.shape == (n, cout, 2 * h, 2 * w)
    assert close(got, want) and close(s, want_s)
