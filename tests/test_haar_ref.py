"""CPU: the float32 and fp64 Haar restatements (tests/haar_ref.py) against oracle.haar and against each other.

The GPU range tests hold the Haar kernels bit for bit to these restatements, so they have to be right on their own: the
synthesis is the oracle's DWTInverse bit for bit across the exponent range (subnormals included), the analysis meets its
own fp64 bound there, the clamp keeps a NaN, and the comparisons reject what they must.
"""
import numpy as np
import pytest
import torch

from oracle import haar as ohaar

import haar_ref as har

FLT_MAX = float(np.finfo(np.float32).max)


def _coeffs(shape, e, seed):
    """float32 values of both signs with magnitudes in [1, 2) 2^e (down to the subnormal grid for small e)."""
    rs = np.random.RandomState(seed)
    v = rs.uniform(1.0, 2.0, size=shape) * rs.choice([-1.0, 1.0], size=shape)
    return torch.from_numpy(np.ldexp(v, e).astype(np.float32))


@pytest.mark.parametrize("e", [0, 120, -126, -140, -149, 127])
def test_idwt32_is_the_oracles_synthesis_bit_for_bit(e):
    ll, hf = _coeffs((2, 3, 5, 6), e, 1), _coeffs((2, 3, 3, 5, 6), e, 2)
    want = ohaar.DWTInverse("haar", "zero")((ll, [hf]))
    assert har.same_bits(har.idwt32(ll, hf), want)
    if e < 127:
        assert bool(torch.isfinite(want).all())


def test_idwt32_keeps_a_non_finite_coefficient_in_its_block():
    ll, hf = _coeffs((1, 1, 4, 4), 0, 3), _coeffs((1, 1, 3, 4, 4), 0, 4)
    hf[0, 0, 1, 2, 3] = float("nan")
    out = har.idwt32(ll, hf)
    bad = ~torch.isfinite(out[0, 0])
    assert bool(bad[4:6, 6:8].all()) and int(bad.sum()) == 4


@pytest.mark.parametrize("e", [0, 100, -100, -126, -140, -149, 126])
def test_dwt32_meets_the_fp64_bound(e):
    x = _coeffs((2, 2, 6, 8), e, 5)
    ll, hf = har.dwt32(x)
    rl, rh, s = har.dwt64(x)
    bound = har.DWT_ULP * 2.0 ** -24 * s + har.DWT_FLOOR
    assert bool(((ll.double() - rl).abs() <= bound).all())
    assert bool(((hf.double() - rh).abs() <= bound.unsqueeze(2)).all())


def test_dwt32_needs_its_floor_on_subnormals():
    """On the subnormal grid the relative part alone cannot hold: products round to multiples of 2^-149."""
    x = _coeffs((1, 1, 8, 8), -148, 6)
    ll, hf = har.dwt32(x)
    rl, rh, s = har.dwt64(x)
    rel = har.DWT_ULP * 2.0 ** -24 * s
    assert bool(((ll.double() - rl).abs() > rel).any() or ((hf.double() - rh).abs() > rel.unsqueeze(2)).any())


def test_dwt32_inverts_idwt32_on_exact_values():
    x = torch.arange(-32, 32, dtype=torch.float32).reshape(1, 1, 8, 8)
    ll, hf = har.dwt32(x)
    back = har.idwt32(ll, hf)
    assert float((back - x).abs().max()) <= 2 ** -18


def test_disp_is_torch_clamp_and_keeps_nan():
    out = torch.tensor([float("nan"), -1.0, 0.5, 3.0, float("inf"), -float("inf"), -0.0])
    d = har.disp(out, 0.5, True)
    assert torch.isnan(d[0]) and d[1:].tolist() == [0.0, 0.25, 1.0, 1.0, 0.0, 0.0]
    assert torch.equal(har.disp(out, 0.5, False)[1:], out[1:] * 0.5)


def test_comparisons_reject_what_they_must():
    a = torch.tensor([1.0, float("nan"), float("inf"), 0.0])
    assert har.same_bits(a, a.clone()) and har.same_values(a, a.clone())
    b = a.clone()
    b[0] = float(np.nextafter(np.float32(1.0), np.float32(2.0)))
    assert not har.same_bits(b, a) and not har.same_values(b, a)
    c = a.clone()
    c[1] = 0.0
    assert not har.same_bits(c, a) and not har.same_values(c, a)
    d = a.clone()
    d[3] = float("nan")
    assert not har.same_bits(d, a) and not har.same_values(d, a)
    z = a.clone()
    z[3] = -0.0
    assert not har.same_bits(z, a) and har.same_values(z, a)
    i = a.clone()
    i[2] = FLT_MAX
    assert not har.same_bits(i, a) and not har.same_values(i, a)
