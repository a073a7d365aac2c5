"""CPU: the fp64 adjoint reference of the conv contract (tests/conv_grad_ref.py) against F.conv2d gradients.

The GPU training tests compare libwmd's backward kernels with conv_grad_ref; this pins that reference to torch's own
convolution adjoint for the three pad modes, the nearest x2 upsample + skip concat (shift0 = 1) and 1x1 layers.
"""
import pytest
import torch
import torch.nn.functional as F

import conv_grad_ref
import conv_ref

_MODE = {conv_ref.PAD_REFLECT: "reflect", conv_ref.PAD_REPLICATE: "replicate", conv_ref.PAD_ZERO: "constant"}


def _torch_grads(x0, x1, weight, dz, taps, pad, shift0):
    x0 = x0.clone().requires_grad_(True)
    x1 = x1.clone().requires_grad_(True) if x1 is not None else None
    w = weight.clone().requires_grad_(True)
    x = F.interpolate(x0, scale_factor=2, mode="nearest") if shift0 else x0
    if x1 is not None:
        x = torch.cat([x, x1], 1)
    if taps == 9:
        x = F.pad(x, (1, 1, 1, 1), mode=_MODE[pad])
    y = F.conv2d(x, w)
    y.backward(dz)
    return x0.grad, (x1.grad if x1 is not None else None), w.grad


def _rows(x):
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n * h * w, c)


@pytest.mark.parametrize("taps,pad,shift0,c1", [(9, conv_ref.PAD_REFLECT, 0, 0), (9, conv_ref.PAD_REPLICATE, 0, 0),
                                                (9, conv_ref.PAD_ZERO, 0, 0), (9, conv_ref.PAD_REFLECT, 1, 3),
                                                (1, conv_ref.PAD_REFLECT, 0, 0)])
def test_adjoint_matches_conv2d(taps, pad, shift0, c1):
    g = torch.Generator().manual_seed(taps + pad + 7 * shift0)
    n, c0, cout, h, w = 2, 5, 4, 6, 8
    k = 3 if taps == 9 else 1
    x0 = torch.randn(n, c0, h >> shift0, w >> shift0, generator=g, dtype=torch.float64)
    x1 = torch.randn(n, c1, h, w, generator=g, dtype=torch.float64) if c1 else None
    weight = torch.randn(cout, c0 + c1, k, k, generator=g, dtype=torch.float64)
    dz = torch.randn(n, cout, h, w, generator=g, dtype=torch.float64)
    want = _torch_grads(x0, x1, weight, dz, taps, pad, shift0)
    got = conv_grad_ref.conv_grads(_rows(x0), c0, _rows(x1) if c1 else None, c1, weight, _rows(dz), n, h, w, taps=taps,
                                   pad=pad, shift0=shift0)
    assert torch.allclose(got["x0"][0], _rows(want[0]), rtol=1e-12, atol=1e-12)
    assert torch.allclose(got["w"][0], want[2], rtol=1e-12, atol=1e-12)
    assert torch.allclose(got["b"][0], dz.sum((0, 2, 3)), rtol=1e-12, atol=1e-12)
    if c1:
        assert torch.allclose(got["x1"][0], _rows(want[1]), rtol=1e-12, atol=1e-12)
    for name in ("x0", "w"):
        assert torch.all(got[name][1] >= got[name][0].abs() - 1e-12)
