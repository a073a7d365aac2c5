"""GPU: the exact kernels of the decoder's hot path across the fp32 range, at their tile edges and on non-finite inputs.

Each output is held to a plain restatement of its operation (tests/haar_ref.py, head_ref, conv_ref and torch), not to
libwmd itself:
  * idwt_haar / idwt_haar_epi: bit-identical to the float32 restatement of the separable order for coefficients at 2^e,
    e = -149 .. 127 and at the top of the binade below FLT_MAX, scalar (odd W) and vector (even W) paths, 1 x 1 planes,
    C > 1 and a grid-stride loop that runs several times; the disparity is torch.clamp(out * scale, 0, 1) and the
    epilogue planes the torch expressions on it, NaN included; a NaN or +-Inf coefficient in any band spoils only its
    2 x 2 block;
  * head_idwt (the fused level tail): ll across the same exponents, a NaN / Inf in ll and in one row of tap products,
    against head_ref.head_idwt_ref and the torch clamp; the threshold is NaN only for the frame that holds the NaN;
  * dwt_haar: bit-identical to its stated order, within DWT_ULP 2^-24 S + DWT_FLOOR of fp64, non-finite values kept in
    their 2 x 2 block;
  * idwt_bilinear: F.interpolate of the reference disparity (head_ref.bilinear_ulps, which also holds the NaN / +-Inf
    pattern to torch's), output sizes off the 32 x 128 tile, anisotropic factors, both align_corners settings, the
    largest factors the shared-patch bound accepts and the smallest it refuses;
  * range_thresh, level_masks, compact, gate_map and the layout moves: bit-identical to the torch expressions at their
    size limits, block and tile edges, and on NaN payloads, +-Inf, -0.0 and subnormals;
  * a decoder frame with a NaN: ("disp", s) and the epilogue planes are NaN exactly where torch.clamp of the library's
    own reconstruction is, and the other frames keep their bits.
The module prints the worst error per kernel and case group (0 for the exact kernels).
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import parity
from wavelet_monodepth_b200 import _lib
from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import nyu_decoders as nd
from wavelet_monodepth_b200 import ops, synth
from wavelet_monodepth_b200._lib import PAD_REFLECT

import conv_ref as cr
import haar_ref as har
import head_ref as hr
from contract import Worst, errors
from launch_check import epilogue_ref, level_masks_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
FLT_MAX = float(np.finfo(np.float32).max)
EXPS = [-149, -140, -126, -100, 0, 100, 126, 127, "max"]
NONFINITE = ["nan", "inf", "-inf"]
PARITY_TOL = 1e-4                 # oracle/parity.py: the float bar of the parity statement

WORST = Worst("kernel, group, case")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def vals(shape, e, seed):
    """float32 values of magnitude [1, 2) 2^e (e = "max": the top binade's last 1/1024, up to FLT_MAX), both signs."""
    rs = np.random.RandomState(seed)
    if e == "max":
        v = rs.uniform(1.0 - 2.0 ** -11, 1.0, size=shape) * FLT_MAX
    else:
        v = np.minimum(np.ldexp(rs.uniform(1.0, 2.0, size=shape), e), FLT_MAX)
    v = v * rs.choice([-1.0, 1.0], size=shape)
    return torch.from_numpy(v.astype(np.float32)).to(DEV)


def _poison(t, idx, value):
    t = t.clone()
    t[idx] = float(value)
    return t


def _status(code):
    return "status %d," % code


# ============================================================================================ idwt_haar
# (N, C, H, W): odd W (scalar path), even W (float2 / float4 path), 1 x 1 and 1 x 2 planes, C > 1
IDWT_SHAPES = [(2, 3, 5, 7), (2, 3, 4, 6), (1, 1, 1, 1), (3, 2, 1, 2)]
EPILOGUES = [("disp_to_depth", 0.1, 100.0), ("div_clamp", 100.0, 0.4, 10.0), ("div_clamp", 100.0, None, None)]


def _check_idwt(res, ll, hf, disp_scale, clamp01, epi, group):
    """out bit for bit, disp and the epilogue planes by value, against the float32 restatement and torch."""
    want = har.idwt32(ll, hf).to(DEV)
    assert har.same_bits(res[0], want), (group, "reconstruction")
    disp = har.disp(want, 1.0 if disp_scale is None else disp_scale, clamp01)
    k = 1
    if disp_scale is not None:
        assert har.same_values(res[1], disp), (group, "disparity")
        k = 2
    if epi is not None:
        planes = epilogue_ref(epi, want, disp)
        assert len(res) - k == len(planes)
        for got, p in zip(res[k:], planes):
            assert har.same_values(got, p), (group, epi[0])
    WORST.note(("idwt_haar", group, "exact"), 0.0, bar=0)


def _idwt(ll, hf, disp_scale, clamp01, epi=None):
    res = ops.idwt_haar(ll, hf, disp_scale=disp_scale, clamp01=clamp01, epilogue=epi)
    return res if isinstance(res, tuple) else (res,)


@pytest.mark.parametrize("shape", IDWT_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("e", EXPS)
def test_idwt_haar_exponents(e, shape):
    n, c, h, w = shape
    ll, hf = vals((n, c, h, w), e, 1), vals((n, c, 3, h, w), e, 2)
    for scale, clamp01 in ((None, False), (0.25, False), (0.25, True), (2.0 ** -100, True)):
        _check_idwt(_idwt(ll, hf, scale, clamp01), ll, hf, scale, clamp01, None, "e=%s" % e)
    for epi in EPILOGUES:
        for clamp01 in (False, True):
            _check_idwt(_idwt(ll, hf, 0.5, clamp01, epi), ll, hf, 0.5, clamp01, epi, "epilogue e=%s" % e)


@pytest.mark.parametrize("w", [127, 128])
def test_idwt_haar_grid_stride_loop(w):
    """4 x 32 planes of 80 x w: several passes of the grid-stride loop on both paths."""
    ll, hf = vals((4, 32, 80, w), 0, 3), vals((4, 32, 3, 80, w), -3, 4)
    _check_idwt(_idwt(ll, hf, 0.5, True), ll, hf, 0.5, True, None, "grid stride")
    epi = ("div_clamp", 100.0, 0.4, 10.0)
    _check_idwt(_idwt(ll, hf, None, False, epi), ll, hf, None, False, epi, "grid stride")


def _epi_raw(ll, hf, disp_scale, clamp01, epi, want_depth):
    """wmd_idwt_haar_epi_f32 with or without the DISP_TO_DEPTH depth plane (ops always asks for it)."""
    mode, a, b, lo, hi, e0, e1, _ = ops._epilogue_args(epi, torch.empty((1,), device=DEV))
    n, c, h, w = ll.shape
    out = torch.empty((n, c, 2 * h, 2 * w), device=DEV)
    disp, e0 = torch.empty_like(out), torch.empty_like(out)
    e1 = torch.empty_like(out) if want_depth else None
    rc = _lib.load().wmd_idwt_haar_epi_f32(_lib.ptr(ll), _lib.ptr(hf), _lib.ptr(out), _lib.ptr(disp), float(disp_scale),
                                            int(clamp01), mode, a, b, lo, hi, _lib.ptr(e0), _lib.ptr(e1), n, c, h, w,
                                            _lib.stream_ptr())
    _lib.check(rc, "wmd_idwt_haar_epi_f32")
    return (out, disp, e0) + ((e1,) if want_depth else ())


@pytest.mark.parametrize("e", [-140, 0, 127])
@pytest.mark.parametrize("w", [5, 6])
def test_idwt_haar_disp_to_depth_without_the_depth_plane(w, e):
    ll, hf = vals((2, 1, 3, w), e, 5), vals((2, 1, 3, 3, w), e, 6)
    epi = ("disp_to_depth", 0.1, 100.0)
    for clamp01 in (False, True):
        full = _epi_raw(ll, hf, 0.5, clamp01, epi, True)
        part = _epi_raw(ll, hf, 0.5, clamp01, epi, False)
        want = har.idwt32(ll, hf).to(DEV)
        planes = epilogue_ref(epi, want, har.disp(want, 0.5, clamp01))
        assert har.same_values(part[2], planes[0]) and har.same_values(full[3], planes[1])
        for a, b in zip(full[:3], part):
            assert har.same_bits(a, b)
    WORST.note(("idwt_haar", "epilogue no depth plane", "exact"), 0.0, bar=0)


@pytest.mark.parametrize("w", [6, 7])
@pytest.mark.parametrize("value", NONFINITE)
@pytest.mark.parametrize("band", ["ll", "lh", "hl", "hh"])
def test_idwt_haar_non_finite_coefficient_stays_in_its_block(band, value, w):
    ll, hf = vals((2, 2, 4, w), 0, 7), vals((2, 2, 3, 4, w), -1, 8)
    i, j = 2, 3
    if band == "ll":
        ll_b, hf_b = _poison(ll, (1, 1, i, j), value), hf
    else:
        ll_b, hf_b = ll, _poison(hf, (1, 1, ("lh", "hl", "hh").index(band), i, j), value)
    block = torch.zeros((2, 2, 8, 2 * w), dtype=torch.bool, device=DEV)
    block[1, 1, 2 * i:2 * i + 2, 2 * j:2 * j + 2] = True
    for epi in (("div_clamp", 100.0, 0.4, 10.0), ("disp_to_depth", 0.1, 100.0)):
        for clamp01 in (False, True):
            clean = _idwt(ll, hf, 0.5, clamp01, epi)
            hit = _idwt(ll_b, hf_b, 0.5, clamp01, epi)
            _check_idwt(hit, ll_b, hf_b, 0.5, clamp01, epi, "non-finite")
            assert torch.equal(~torch.isfinite(hit[0]), block), "the reconstruction's non-finite outputs leave the block"
            for a, b in zip(clean, hit):
                assert har.same_bits(b[~block], a[~block]), "outputs outside the block changed"
            if value == "nan":
                for t in hit[1:]:
                    assert bool(torch.isnan(t[block]).all()), "a NaN reconstruction must stay NaN through the clamp"


# ============================================================================================ head_idwt
def _tail_operands(n, h, w, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = (torch.rand(n * h * w, 56, generator=g) * 6 - 3).to(DEV)
    bias = (torch.rand(6, generator=g) * 2 - 1).to(DEV)
    return z, bias


def _tail(z, bias, ll, clamp01, epi):
    return ops.head_idwt(z, bias, ll, 2.0, 0.25, pad=PAD_REFLECT, clamp01=clamp01, thresh_ratio=0.15, epilogue=epi)


def _check_tail(res, z, bias, ll, clamp01, epi, group):
    n, _, h, w = ll.shape
    ref = hr.head_idwt_ref(z, 0, None, None, bias, 2.0, PAD_REFLECT, ll, 0.25, clamp01, n, h, w)
    a = cr.ACT_ALLOW * 2.0
    err = max(errors(res["yh"], ref["yh"], ref["s_yh"], 2 * a, what="yh")[0],
              errors(res["out"], ref["out"], ref["s_out"], 3 * a, what="out")[0],
              errors(res["disp"], ref["disp"], ref["s_disp"], 3 * a * 0.25, what="disp")[0])
    WORST.note(("head_idwt", group, "err / S"), err, bar=hr.BAR["head_idwt"])
    assert err <= hr.BAR["head_idwt"], (group, err)
    # the exact parts: the synthesis of the kernel's own coefficients, the torch clamp, the epilogue and the threshold
    out = har.idwt32(ll, res["yh"].reshape(n, 1, 3, h, w)).to(DEV)
    assert har.same_bits(res["out"], out), (group, "reconstruction")
    disp = har.disp(out, 0.25, clamp01)
    assert har.same_values(res["disp"], disp), (group, "disparity")
    if epi is not None:
        names = ("scaled_disp", "depth") if epi[0] == "disp_to_depth" else ("depth",)
        for k, p in zip(names, epilogue_ref(epi, out, disp)):
            assert har.same_values(res[k], p), (group, k)
    o = out.reshape(n, -1)
    assert har.same_bits(res["thresh"], (o.amax(1) - o.amin(1)) * torch.tensor(0.15, device=DEV)), (group, "threshold")


@pytest.mark.parametrize("e", EXPS)
def test_head_idwt_ll_exponents(e):
    n, h, w = 2, 8, 32
    z, bias = _tail_operands(n, h, w, 11)
    ll = vals((n, 1, h, w), e, 12)
    for clamp01, epi in ((True, None), (False, None), (True, ("disp_to_depth", 0.1, 100.0)),
                         (False, ("div_clamp", 100.0, 0.4, 10.0))):
        _check_tail(_tail(z, bias, ll, clamp01, epi), z, bias, ll, clamp01, epi, "ll e=%s" % e)


@pytest.mark.parametrize("where", ["ll", "z"])
@pytest.mark.parametrize("value", NONFINITE)
def test_head_idwt_non_finite_frame(where, value):
    """A NaN / Inf in frame 1's ll or in one row of its tap products: every plane follows the references, frame 1's
    threshold is NaN when its reconstruction holds a NaN, and frames 0 and 2 keep their bits."""
    n, h, w = 3, 8, 16
    z, bias = _tail_operands(n, h, w, 13)
    ll = vals((n, 1, h, w), 0, 14)
    if where == "ll":
        z_b, ll_b = z, _poison(ll, (1, 0, 3, 5), value)
    else:
        z_b, ll_b = _poison(z, ((1 * h + 3) * w + 5, slice(None)), value), ll
    for clamp01, epi in ((True, ("disp_to_depth", 0.1, 100.0)), (True, None), (False, ("div_clamp", 100.0, 0.4, 10.0))):
        clean = _tail(z, bias, ll, clamp01, epi)
        hit = _tail(z_b, bias, ll_b, clamp01, epi)
        _check_tail(hit, z_b, bias, ll_b, clamp01, epi, "non-finite " + where)
        if bool(torch.isnan(hit["out"][1]).any()):
            assert torch.isnan(hit["thresh"][1]), "a frame with a NaN reconstruction must get a NaN threshold"
            assert bool(torch.isnan(hit["disp"][1]).any()), "the NaN must reach the clamped disparity"
        keep = [0, 2]
        for k, v in clean.items():
            assert har.same_bits(hit[k][keep], v[keep]), ("the other frames changed", k)
    if value == "nan":
        assert torch.isnan(hit["thresh"][1])


# ============================================================================================ dwt_haar
DWT_SHAPES = [(2, 3, 6, 10), (1, 1, 2, 2), (3, 2, 4, 2)]


def _check_dwt(x, group):
    ll, hf = ops.dwt_haar(x)
    l32, h32 = har.dwt32(x)
    assert har.same_bits(ll, l32) and har.same_bits(hf, h32), (group, "not the stated order's bits")
    l64, h64, s = har.dwt64(x)
    if bool(torch.isfinite(l32).all()) and bool(torch.isfinite(h32).all()):
        bar = har.DWT_ULP * 2.0 ** -24
        e_l, f_l = errors(ll, l64.to(DEV), s.to(DEV), floor=har.DWT_FLOOR, bar=bar)
        e_h, f_h = errors(hf, h64.to(DEV), s.unsqueeze(2).to(DEV), floor=har.DWT_FLOOR, bar=bar)
        WORST.note(("dwt_haar", group, "err / (BAR S + F)"), max(e_l, e_h), max(f_l, f_h), bar=bar)
        assert max(f_l, f_h) <= 1, (group, f_l, f_h)
    else:
        WORST.note(("dwt_haar", group, "exact"), 0.0, bar=0)
    return ll, hf


@pytest.mark.parametrize("shape", DWT_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("e", EXPS)
def test_dwt_haar_exponents(e, shape):
    _check_dwt(vals(shape, e, 21), "e=%s" % e)


def test_dwt_haar_grid_stride_loop():
    _check_dwt(vals((4, 32, 160, 256), -130, 22), "grid stride")


@pytest.mark.parametrize("value", NONFINITE)
def test_dwt_haar_non_finite_input_stays_in_its_block(value):
    x = vals((2, 2, 8, 10), 0, 23)
    ll, hf = _check_dwt(x, "non-finite")
    ll_b, hf_b = _check_dwt(_poison(x, (1, 0, 5, 6), value), "non-finite")
    bad = torch.zeros((2, 2, 4, 5), dtype=torch.bool, device=DEV)
    bad[1, 0, 2, 3] = True
    assert torch.equal(~torch.isfinite(ll_b), bad)
    assert torch.equal(~torch.isfinite(hf_b), bad.unsqueeze(2).expand_as(hf_b))
    assert har.same_bits(ll_b[~bad], ll[~bad])
    keep = ~bad.unsqueeze(2).expand_as(hf_b)
    assert har.same_bits(hf_b[keep], hf[keep])


# ============================================================================================ idwt_bilinear
def _smooth(n, c, h, w, e, seed, spread=2.0 ** -12):
    """(ll, hf) of a disparity-like plane: ll = 1.5 x 2^e (e = "max": 0.7 FLT_MAX) within `spread`, details of `spread`
    times that.

    The kernel and torch take the source index in float32, the fp64 resize of the reference a finer one; neighbours
    within 2^-11 of each other keep what that index difference can cost below 0.01 of bilinear_ulps' unit, so the bar
    measures the blend itself.  Where the factors are powers of two both indices are exact and any spread may be used."""
    base = 0.7 * FLT_MAX if e == "max" else 1.5 * 2.0 ** e
    rs = np.random.RandomState(seed)
    ll = base * (1 + spread * rs.uniform(-1, 1, (n, c, h, w)))
    hf = base * spread * rs.uniform(-1, 1, (n, c, 3, h, w))
    return torch.from_numpy(ll.astype(np.float32)).to(DEV), torch.from_numpy(hf.astype(np.float32)).to(DEV)


def _bilinear(ll, hf, size, scale, clamp01, ac, group):
    n, c, h, w = ll.shape
    got = ops.idwt_bilinear(ll, hf, size, disp_scale=scale, clamp01=clamp01, align_corners=ac)
    disp = har.disp(har.idwt32(ll, hf), scale, clamp01).to(DEV).double()
    ulps = hr.bilinear_ulps(got, disp, size, ac)
    WORST.note(("idwt_bilinear", group, "ac" if ac else "-"), ulps, bar=hr.BILINEAR_ULP)
    assert ulps <= hr.BILINEAR_ULP, (group, size, ac, ulps)
    return got


# (coefficient H, W, full size): off the 32 x 128 tile, anisotropic factors, one row / one column under align_corners
BILINEAR_SIZES = [(6, 10, (37, 150)), (6, 10, (33, 129)), (5, 7, (161, 300)), (8, 16, (40, 257)), (4, 9, (97, 40)),
                  (6, 10, (1, 150)), (6, 10, (64, 1))]


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("h,w,size", BILINEAR_SIZES)
def test_idwt_bilinear_sizes(h, w, size, ac):
    if 1 in size and not ac:
        # without align_corners a 1-pixel axis is a downsampling: refused, whatever the other axis
        with pytest.raises(_lib.WmdError, match=_status(-5)):
            ops.idwt_bilinear(*_smooth(2, 1, h, w, 0, 31), size, 0.5, True, ac)
        return
    ll, hf = _smooth(2, 3, h, w, 0, 31)
    for clamp01 in (False, True):
        _bilinear(ll, hf, size, 0.5, clamp01, ac, "sizes")


def _need(hs, ws, fh, fw, ac):
    """The launch's shared-patch estimate, in the kernel's float32 arithmetic."""
    f32 = np.float32
    if ac:
        sy = f32(hs - 1) / f32(fh - 1) if fh > 1 else f32(0)
        sx = f32(ws - 1) / f32(fw - 1) if fw > 1 else f32(0)
    else:
        sy, sx = f32(hs) / f32(fh), f32(ws) / f32(fw)
    return (int(f32(32) * sy) + 4) * (int(f32(128) * sx) + 4)


def _smallest_accepted(hs, ws, ac, axis):
    """(accepted, refused) full sizes along `axis` at the shared-patch bound, the other axis 4x upsampled."""
    other = 4 * (ws if axis == 0 else hs)
    for f in range(2, 64 * max(hs, ws)):
        fh, fw = (f, other) if axis == 0 else (other, f)
        if _need(hs, ws, fh, fw, ac) <= 2048:
            prev = (f - 1, other) if axis == 0 else (other, f - 1)
            assert _need(hs, ws, *prev, ac) > 2048
            return (fh, fw), prev
    raise AssertionError("no accepted size")


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("axis", [0, 1])
def test_idwt_bilinear_largest_factor_accepted_and_smallest_refused(axis, ac):
    h, w = 24, 40
    ll, hf = _smooth(1, 2, h, w, 0, 33)
    ok, refused = _smallest_accepted(2 * h, 2 * w, ac, axis)
    _bilinear(ll, hf, ok, 0.5, True, ac, "patch bound")
    with pytest.raises(_lib.WmdError, match=_status(-5)):
        ops.idwt_bilinear(ll, hf, refused, disp_scale=0.5, clamp01=True, align_corners=ac)


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("value", NONFINITE)
@pytest.mark.parametrize("band", ["ll", "hh"])
def test_idwt_bilinear_non_finite_coefficient(band, value, ac):
    """The non-finite outputs are exactly torch's footprint of the spoiled 2 x 2 block, zero-weight neighbours included;
    under the clamp a NaN stays NaN (an Inf clamps to a finite disparity)."""
    h, w = 6, 10
    ll, hf = _smooth(2, 1, h, w, 0, 35)
    if band == "ll":
        ll = _poison(ll, (1, 0, 2, 4), value)
    else:
        hf = _poison(hf, (1, 0, 2, 2, 4), value)
    # factors of 1/2, 1/4 and 1/8 in both index rules: the clamped Inf puts 0 or 1 beside ~0.75, so the index must be exact
    for size in (((45, 77), (23, 153)) if ac else ((48, 80), (24, 160))):
        for clamp01 in (False, True):
            got = _bilinear(ll, hf, size, 1.0, clamp01, ac, "non-finite")
            if value == "nan" or not clamp01:
                assert not bool(torch.isfinite(got[1]).all())
            assert bool(torch.isfinite(got[0]).all())


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("e", [126, "max"])
def test_idwt_bilinear_largest_disparities(e, ac):
    """Disparities near 2^126 and near 0.35 FLT_MAX (ll near 0.7 FLT_MAX; the blend cannot overflow)."""
    ll, hf = _smooth(2, 1, 6, 10, e, 37)
    for size in ((48, 80), (37, 150)):
        _bilinear(ll, hf, size, 1.0, False, ac, "e=%s" % e)


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("e", [-146, -140, -130, -127])
def test_idwt_bilinear_subnormal_disparities(e, ac):
    """Disparities among the subnormals (from 1 to 11 x 2^-149 at e = -146), ll and details varying by a quarter:
    held to BILINEAR_ULP 2^-23 max|disp| + BILINEAR_FLOOR (3 x 2^-149), which a flushed (zero) or doubled output fails
    (tests/test_head_ref.py).  Factors of 1/4 and 1/8, where the float32 and fp64 source indices agree."""
    ll, hf = _smooth(2, 1, 6, 10, e, 38, spread=0.25)
    disp = har.idwt32(ll, hf)
    assert 8 * 2.0 ** -149 <= float(disp.abs().max()) < 2.0 ** -126
    for size in (((45, 77), (23, 153)) if ac else ((48, 80), (24, 160))):
        _bilinear(ll, hf, size, 1.0, False, ac, "subnormal e=%s" % e)


# ============================================================================================ range_thresh
def _thresh_ref(x, ratio):
    xs = x.reshape(x.shape[0], -1)
    mn, mx = xs.amin(1), xs.amax(1)
    return (mx - mn) * torch.tensor(ratio, dtype=torch.float32, device=x.device), torch.stack([mn, mx], 1)


def _check_thresh(x, ratio, group):
    t, mm = ops.range_thresh(x, ratio, return_minmax=True)
    wt, wmm = _thresh_ref(x, ratio)
    assert har.same_bits(t, wt) and har.same_bits(mm, wmm), (group, ratio)
    WORST.note(("range_thresh", group, "exact"), 0.0, bar=0)
    return t, mm


@pytest.mark.parametrize("n,per", [(16384, 3), (16384, 4), (7, 1), (5, 7), (3, 4099), (2, 64 * 4096 + 3), (1, 64 * 4096 * 2)])
def test_range_thresh_sizes(n, per):
    """N up to 16384; per_sample % 4 != 0 (every sample after the first misaligned: the scalar path), 1, one block and
    the 64-block cap."""
    x = vals((n, per), 0, 41)
    for ratio in (0.15, 1.0, 0.0, -0.5):
        _check_thresh(x, ratio, "sizes")


def test_range_thresh_refuses_n_past_16384():
    with pytest.raises(_lib.WmdError, match=_status(-2)):
        ops.range_thresh(torch.zeros((16385, 2), device=DEV), 0.1)


@pytest.mark.parametrize("per", [8, 9])
def test_range_thresh_value_range(per):
    """Constant samples, subnormal ranges, ranges past FLT_MAX (max - min = Inf), and ratios of 0, < 0 and 1."""
    rows = [torch.full((per,), 3.0), torch.zeros(per), vals((per,), -149, 42).cpu(), vals((per,), -140, 43).cpu(),
            vals((per,), "max", 44).cpu(), vals((per,), 127, 45).cpu(), torch.full((per,), -FLT_MAX)]
    x = torch.stack(rows).to(DEV)
    for ratio in (0.15, 0.0, -0.3, 1.0, 2.0 ** -140):
        t, _ = _check_thresh(x, ratio, "value range")
        assert float(t[0]) == 0.0 and float(t[1]) == 0.0


@pytest.mark.parametrize("per", [4, 6, 4099])
@pytest.mark.parametrize("value", NONFINITE)
def test_range_thresh_non_finite_sample(value, per):
    x = vals((4, per), 0, 46)
    clean, cmm = _check_thresh(x, 0.2, "non-finite")
    t, mm = _check_thresh(_poison(x, (2, per // 2), value), 0.2, "non-finite")
    if value == "nan":
        assert torch.isnan(t[2]) and bool(torch.isnan(mm[2]).all())
    keep = [0, 1, 3]
    assert har.same_bits(t[keep], clean[keep]) and har.same_bits(mm[keep], cmm[keep])


def test_range_thresh_scratch_reused_across_batch_sizes():
    """One scratch buffer, N = 16384, then 3, then 16384 again: the self-resetting tickets leave it ready each time."""
    for k, (n, per) in enumerate(((16384, 5), (3, 70000), (16384, 5), (16384, 8))):
        _check_thresh(vals((n, per), 0, 50 + k), 0.1, "scratch reuse")


# ============================================================================================ level_masks
MASK_HW = [1, 2, 31, 32, 33, 64, 65]
SETS = ("S0", "S1", "S2", "S3", "S4", "S5")
SUBSETS = [sub for k in range(len(SETS) + 1) for sub in itertools.combinations(SETS, k)]    # every choice of NULLs


def _bands(n, h, w, seed):
    """|yh| in [0, 1) with NaN, +-Inf, subnormals and exact zeros sprinkled in."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    yh = torch.rand((n, 3, h, w), generator=g) * 2 - 1
    pick = torch.rand((n, 3, h, w), generator=g)
    specials = torch.tensor([float("nan"), float("inf"), -float("inf"), 2.0 ** -140, -2.0 ** -149, 0.0])
    idx = torch.randint(0, len(specials), (n, 3, h, w), generator=g)
    yh = torch.where(pick < 0.06, specials[idx], yh)
    return yh.to(DEV)


@pytest.mark.parametrize("w", MASK_HW)
@pytest.mark.parametrize("h", MASK_HW)
def test_level_masks_tile_edges_and_values(h, w):
    n = 3
    yh = _bands(n, h, w, 100 * h + w)
    threshes = [(0.5, 0.0, 0.9), (float("nan"), float("inf"), -1.0), (2.0 ** -140, -0.0, 2.0 ** -149)]
    for k, th in enumerate(threshes):
        t = torch.tensor(th, dtype=torch.float32, device=DEV)
        want = level_masks_ref(yh, t, n, h, w, DEV)
        for sub in (SUBSETS if k == 0 else [SETS]):            # the first threshold set under every subset of outputs
            got = ops.level_masks(yh, t, want=sub)
            assert sorted(got) == sorted(sub)
            for key, m in got.items():
                assert torch.equal(m, want[key]), (th, sub, key)
    if h in (1, 33, 65):
        want = level_masks_ref(None, None, n, h, w, DEV)
        for sub in (SETS, ("S1", "S2", "S4", "S5"), ("S3",)):
            got = ops.level_masks(None, None, n=n, h=h, w=w, device=torch.device(DEV), want=sub)
            for key, m in got.items():
                assert torch.equal(m, want[key]), ("all ones", sub, key)
    WORST.note(("level_masks", "tile edges", "exact"), 0.0, bar=0)


def test_level_masks_nan_threshold_sets_no_bit():
    yh = _bands(2, 33, 65, 7)
    t = torch.tensor([float("nan"), 0.1], device=DEV)
    got = ops.level_masks(yh, t)
    for key in got:
        assert not bool(got[key][0].any()), key


# ============================================================================================ compact / gate_map
# N x H x W around the 8-pixel vector load and the 2048-pixel block
COMPACT_SHAPES = [(1, 1, 7), (1, 3, 3), (1, 23, 89), (2, 32, 32), (3, 1, 683), (1, 1, 2399), (1, 49, 49), (1, 1, 8191),
                  (3, 1, 2731)]


def _mask_bytes(shape, kind, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if kind == "zeros":
        return torch.zeros(shape, dtype=torch.uint8, device=DEV)
    if kind == "ones":
        return torch.ones(shape, dtype=torch.uint8, device=DEV)
    if kind == "255":
        return torch.full(shape, 255, dtype=torch.uint8, device=DEV)
    v = torch.tensor([0, 0, 1, 2, 255], dtype=torch.uint8)[torch.randint(0, 5, shape, generator=g)]
    return v.to(DEV)


@pytest.mark.parametrize("kind", ["random", "zeros", "ones", "255"])
@pytest.mark.parametrize("n,h,w", COMPACT_SHAPES)
def test_compact_block_edges_and_mask_bytes(n, h, w, kind):
    m = _mask_bytes((n, 1, h, w), kind, n * h * w)
    idxmap, pixels, offsets = ops.compact(m)
    mm = m.reshape(n, h, w)
    per = (mm != 0).reshape(n, -1).sum(1)
    assert torch.equal(offsets, torch.cat([per.new_zeros(1), per.cumsum(0)]).to(torch.int32))
    assert torch.equal(idxmap, cr.index_map(mm))
    lst = cr.pixel_list(mm)
    assert torch.equal(pixels[:len(lst)], lst)
    WORST.note(("compact", "block edges", "exact"), 0.0, bar=0)


@pytest.mark.parametrize("with_map", [False, True])
@pytest.mark.parametrize("n,h,w", [(1, 1, 7), (2, 32, 32), (3, 1, 2731), (5, 37, 67)])
def test_gate_map(n, h, w, with_map):
    gate = _mask_bytes((n, 1, h, w), "random", 3 * n * h * w)
    g = torch.Generator(device="cpu").manual_seed(9)
    idx = torch.randint(-1, 1 << 30, (n, h, w), generator=g, dtype=torch.int32).to(DEV) if with_map else None
    out = ops.gate_map(gate, idx)
    src = idx if with_map else torch.arange(n * h * w, dtype=torch.int32, device=DEV).reshape(n, h, w)
    assert torch.equal(out, torch.where(gate.reshape(n, h, w) != 0, src, torch.full_like(src, -1)))
    WORST.note(("gate_map", "map" if with_map else "linear", "exact"), 0.0, bar=0)


# ============================================================================================ layout moves
SPECIAL_BITS = [0x7FC00000, 0x7FC12345, 0xFFC00001, 0x7F800001, 0x7F800000, 0xFF800000, 0x80000000, 0x00000001,
                0x807FFFFF, 0x7F7FFFFF, 0x00800000]
AMAX_BITS = [b for b in SPECIAL_BITS if b != 0x7F7FFFFF]        # FLT_MAX goes only where a mask must exclude it
LAYOUT_SHAPES = [(2, 5, 7, 9), (2, 40, 13, 21), (1, 33, 12, 25)]


def _i32(bits):
    return torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in bits], dtype=torch.int32)


def _special_map(shape, seed, frac=0.1, bits=SPECIAL_BITS):
    """A float32 map whose bits include non-canonical NaN payloads, a signalling NaN, +-Inf, -0.0 and subnormals."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(shape, generator=g)
    pick = torch.rand(shape, generator=g) < frac
    sp = _i32(bits)[torch.randint(0, len(bits), shape, generator=g)].view(torch.float32)
    return torch.where(pick, sp, x).to(DEV)


def _amax_map(shape, seed, mask):
    """_special_map without FLT_MAX, then FLT_MAX in one channel of the first pixel `mask` leaves out: a maximum that
    ignored its mask would report it."""
    x = _special_map(shape, seed, bits=AMAX_BITS)
    n, c, h, w = shape
    off = torch.nonzero(mask.reshape(-1) == 0)
    assert len(off), "the mask leaves no pixel out"
    p = int(off[0])
    x[p // (h * w), c // 2, (p % (h * w)) // w, p % w] = FLT_MAX
    return x


def _masked_max(x, sel):
    """max |x| over the finite values of the selected pixels, which must stay below the planted FLT_MAX"""
    want = cr.finite_max(x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])[sel])
    assert want < FLT_MAX
    return want


def _nhwc_bits(x):
    n, c = x.shape[:2]
    return x.view(torch.int32).permute(0, 2, 3, 1).reshape(-1, c)


@pytest.mark.parametrize("n,c,h,w", LAYOUT_SHAPES)
def test_nchw_to_rows_forms_are_bit_copies(n, c, h, w):
    gate = _mask_bytes((n, 1, h, w), "random", c)
    sel = gate.reshape(-1) != 0
    x = _amax_map((n, c, h, w), c * h, gate)
    xr = _nhwc_bits(x)
    rows = ops.nchw_to_rows(x)
    assert torch.equal(rows.view(torch.int32)[:, :c], xr) and bool((rows.view(torch.int32)[:, c:] == 0).all())
    amax = torch.zeros(1, device=DEV)
    rows = ops.nchw_to_rows(x, amax=amax)
    assert torch.equal(rows.view(torch.int32)[:, :c], xr) and float(amax) == FLT_MAX == cr.finite_max(x)
    rows = ops.nchw_to_rows(x, gate=gate)
    assert torch.equal(rows.view(torch.int32)[sel, :c], xr[sel])
    amax = torch.zeros(1, device=DEV)
    rows = ops.nchw_to_rows(x, gate=gate, amax=amax)
    assert torch.equal(rows.view(torch.int32)[sel, :c], xr[sel])
    assert float(amax) == _masked_max(x, sel)
    amax = torch.zeros(1, device=DEV)
    rows = ops.nchw_to_rows(x, amax=amax, amax_mask=gate)
    assert torch.equal(rows.view(torch.int32)[:, :c], xr)
    assert float(amax) == _masked_max(x, sel)
    WORST.note(("nchw_to_rows", "special bits", "exact"), 0.0, bar=0)


@pytest.mark.parametrize("n,c,h,w", LAYOUT_SHAPES)
def test_gather_scatter_and_rows_to_nchw_are_bit_copies(n, c, h, w):
    m = _mask_bytes((n, 1, h, w), "random", w)
    x = _amax_map((n, c, h, w), c * w, m)
    xr = _nhwc_bits(x)
    _, pixels, offsets = ops.compact(m)
    cnt = int(offsets[n])
    amax = torch.zeros(1, device=DEV)
    rows = ops.gather_rows_list(x, pixels, offsets[n:], amax=amax)
    p = pixels[:cnt].long()
    assert torch.equal(rows.view(torch.int32)[:cnt, :c], xr[p])
    assert float(amax) == _masked_max(x, p)
    ld = ops.pad4(c)
    src = _special_map((n * h * w, ld), ld + c)
    out = ops.rows_to_nchw(src, n, c, h, w)
    want = src.view(torch.int32)[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2)
    assert torch.equal(out.view(torch.int32), want)
    out = ops.scatter_rows(src, c, pixels, offsets[n:], n, h, w)
    want = torch.zeros((n * h * w, c), dtype=torch.int32, device=DEV)
    want[p] = src.view(torch.int32)[:cnt, :c]
    assert torch.equal(out.view(torch.int32), want.reshape(n, h, w, c).permute(0, 3, 1, 2))
    WORST.note(("gather / scatter / rows_to_nchw", "special bits", "exact"), 0.0, bar=0)


@pytest.mark.parametrize("kind", ["non-finite", "subnormal"])
def test_amax_skips_non_finite_values(kind):
    """Every amax form: a map of only NaN / +-Inf reports 0, a map of subnormals its subnormal maximum."""
    n, c, h, w = 2, 12, 9, 15
    if kind == "non-finite":
        bits = _i32([0x7FC00000, 0xFF800000, 0x7F800000, 0x7F800001, 0xFFC12345])
        g = torch.Generator(device="cpu").manual_seed(3)
        x = bits[torch.randint(0, len(bits), (n, c, h, w), generator=g)].view(torch.float32).to(DEV)
        want = 0.0
    else:
        x = vals((n, c, h, w), -140, 61)
        want = float(x.abs().max())
        assert 0 < want < 2.0 ** -126
    gate = torch.ones((n, 1, h, w), dtype=torch.uint8, device=DEV)
    forms = [dict(), dict(gate=gate), dict(amax_mask=gate)]
    for kw in forms:
        amax = torch.zeros(1, device=DEV)
        ops.nchw_to_rows(x, amax=amax, **kw)
        assert float(amax) == want, (kind, sorted(kw))
    _, pixels, offsets = ops.compact(gate)
    amax = torch.zeros(1, device=DEV)
    ops.gather_rows_list(x, pixels, offsets[n:], amax=amax)
    assert float(amax) == want, (kind, "gather_rows_list")
    WORST.note(("amax", kind, "exact"), 0.0, bar=0)


# ============================================================================================ a decoder frame with a NaN
KEEP = [0, 1, 3]


def _kitti_feats():
    return [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(20 + i))
            for i, s in enumerate(synth.kitti_feature_shapes(4, 96, 320, synth.RESNET18_CH))]


def _nan_frame(feats):
    bad = [f.clone() for f in feats]
    bad[-1][2, 7, 1, 3] = float("nan")
    return bad


def _recon(out, s, ll=None):
    """The float32 restatement of scale s's reconstruction from the library's own coefficients (ll: its LL band, if the
    decoder does not return it)."""
    ll = out[("wavelets", s, "LL")] if ll is None else ll
    hf = torch.cat([out[("wavelets", s, b)] for b in ("LH", "HL", "HH")], 1).unsqueeze(1)
    return har.idwt32(ll, hf).to(DEV)


def _check_nan_disp(out, s, recon, clamp01):
    """("disp", s) = [torch.clamp](recon / 2^s, 0, 1) by value, NaN where it is NaN; whether frame 2's holds a NaN."""
    want = har.disp(recon, 1.0 / 2 ** s, clamp01)
    assert har.same_values(out[("disp", s)], want), ("disp", s)
    return bool(torch.isnan(want[2]).any())


@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_kitti_decoder_nan_frame_keeps_nan_disparity(kind):
    """A NaN in frame 2's deepest features: ("disp", s) = clamp(yl / 2^s, 0, 1) is NaN exactly where the torch clamp of
    the library's reconstruction is, scaled_disp / depth follow it; frames 0, 1, 3 keep their bits on the dense decoder
    and their masks (values within the parity bar: balanced cuts follow the batch's row count) on the sparse one."""
    ch = synth.RESNET18_CH
    mod = (kd.DepthWaveProgressiveDecoder if kind == "dense" else kd.SparseDepthWaveProgressiveDecoder)(np.array(ch))
    synth.load_random(mod, seed=3)
    mod = mod.to(DEV).eval()
    mod.depth_range = (0.1, 100.0)
    feats = _kitti_feats()
    with torch.no_grad():
        args = () if kind == "dense" else (0.05,)
        clean = mod(feats, *args)
        out = mod(_nan_frame(feats), *args)
    assert all([_check_nan_disp(out, s, _recon(out, s), True) for s in range(4)]), "the NaN did not reach every scale"
    for k, p in zip(("scaled_disp", "depth"), epilogue_ref(("disp_to_depth", 0.1, 100.0), None, out[("disp", 0)])):
        assert har.same_values(out[(k, 0)], p), k
    for k, a in clean.items():
        if not torch.is_tensor(a) or a.dim() == 0 or a.shape[0] != 4:
            continue
        b = out[k]
        if kind == "dense" or a.dtype == torch.bool:
            assert har.same_bits(b[KEEP].float(), a[KEEP].float()), ("the clean frames changed", k)
        else:
            assert parity.rel_err(b[KEEP], a[KEEP]) <= PARITY_TOL, (k, parity.rel_err(b[KEEP], a[KEEP]))


def test_nyu_decoder_nan_frame_keeps_nan_depth():
    """DecoderWave with the reference's depth epilogue clamp(("disp", 0) / 100, 0.4, 10) (NYUv2/utils.py:219,229): a NaN
    in frame 2's features gives NaN depth exactly where the torch clamp of the reconstruction does; frames 0, 1, 3 keep
    their bits."""
    enc = [16, 16, 32, 64, 128]
    mod = nd.DecoderWave(enc_features=enc, decoder_width=0.5)
    synth.load_random(mod, seed=5, gains={"wave": 4.0})
    mod = mod.to(DEV).eval()
    mod.depth_epilogue = (100, 0.4, 10)
    feats = [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(30 + i))
             for i, s in enumerate(synth.nyu_feature_shapes(4, 96, 128, enc))]
    with torch.no_grad():
        clean = mod(feats)
        out = mod(_nan_frame(feats))
    recon = _recon(out, 2)                            # the coarsest level's LL is returned, the finer ones are its chain
    assert _check_nan_disp(out, 2, recon, False)
    recon = _recon(out, 1, recon)
    assert _check_nan_disp(out, 1, recon, False)
    recon = _recon(out, 0, recon)
    assert har.same_bits(out[("disp", 0)], recon)
    (want,) = epilogue_ref(("div_clamp", 100, 0.4, 10), recon, None)
    assert bool(torch.isnan(want[2]).any()), "the NaN never reached the depth"
    assert har.same_values(out[("depth", 0)], want)
    for k, a in clean.items():
        if torch.is_tensor(a) and a.dim() and a.shape[0] == 4:
            assert har.same_bits(out[k][KEEP], a[KEEP]), ("the clean frames changed", k)
