"""CPU: the fp64 references of the coefficient-head contracts (tests/head_ref.py) against independent compositions:
F.conv2d on F.pad for every pad mode, the sparse-op oracle for the index-map form, the oracle's DWTInverse for the
synthesis and explicit matmuls for the 1x1 stages, value and error scale, exactly (fp64 sums in another order: <= 1e-12).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import haar as ohaar
from oracle import sparse_ops as osp

import conv_ref as cr
import head_ref as hr
from helpers import close, rnd, rows_of

_MODE = {cr.PAD_ZERO: "constant", cr.PAD_REFLECT: "reflect", cr.PAD_REPLICATE: "replicate"}
_ACT = {cr.ACT_NONE: lambda v: v, cr.ACT_ELU: F.elu, cr.ACT_SIGMOID: torch.sigmoid}
PADS = [cr.PAD_ZERO, cr.PAD_REFLECT, cr.PAD_REPLICATE]


def _conv(x, wt, b, pad):
    """(value, S) of a 3x3 conv of x (N, C, H, W) in fp64, by F.conv2d on the padded input."""
    xp = F.pad(x.double(), (1, 1, 1, 1), mode=_MODE[pad])
    bb = b.double() if b is not None else None
    return F.conv2d(xp, wt.double(), bb), F.conv2d(xp.abs(), wt.double().abs(), bb.abs() if bb is not None else None)


def _rows_nchw(v, n, h, w):
    return v.reshape(n, h, w, -1).permute(0, 3, 1, 2)


def _tap_products(t_rows, w_list, offsets):
    """z rows (R, 9 G): z[r, tap G + g] = t[r] . w_g[:, tap], w_g the heads' output channels concatenated in order."""
    ws = torch.cat([F.pad(wk.double(), (0, 0, 0, 0, off, t_rows.shape[1] - off - wk.shape[1]))
                    for wk, off in zip(w_list, offsets)], 0)                 # (G, ld, 3, 3)
    g = ws.shape[0]
    return (t_rows.double() @ ws.permute(1, 2, 3, 0).reshape(t_rows.shape[1], 9 * g)).float()


@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("act,cout,dual", [(cr.ACT_NONE, 1, False), (cr.ACT_ELU, 2, True), (cr.ACT_SIGMOID, 3, True),
                                           (cr.ACT_SIGMOID, 4, False)])
def test_head_conv3x3_matches_conv2d(pad, act, cout, dual):
    n, c, h, w, ld, off_a, off_b = 2, 5, 4, 6, 17, 3, 11
    x = rnd(n, ld, h, w, seed=1)
    wa, ba, wb, bb = rnd(cout, c, 3, 3, seed=2), rnd(cout, seed=3), rnd(cout, c, 3, 3, seed=4), rnd(cout, seed=5)
    v, s = hr.head_conv3x3_ref(rows_of(x), ld, c, off_a, off_b if dual else -1, wa, ba, wb, bb, cout, -1.5, act, pad,
                               None, None, None, None, n, h, w)
    a, sa = _conv(x[:, off_a:off_a + c], wa, ba, pad)
    want, want_s = -1.5 * _ACT[act](a), 1.5 * sa
    if dual:
        b, sb = _conv(x[:, off_b:off_b + c], wb, bb, pad)
        want, want_s = want + 1.5 * _ACT[act](b), want_s + 1.5 * sb
    assert close(_rows_nchw(v, n, h, w), want) and close(_rows_nchw(s, n, h, w), want_s)


def _sparse_case(h, w, seed):
    """A batch-1 input set (index map with holes) and an output list."""
    rs = np.random.RandomState(seed)
    m_in = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < 0.6).astype(np.uint8))
    m_out = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < 0.5).astype(np.uint8))
    return m_in, m_out, cr.index_map(m_in.reshape(1, h, w)), cr.pixel_list(m_out.reshape(1, h, w))


@pytest.mark.parametrize("pad", PADS)
def test_head_conv3x3_index_map_matches_sparse_oracle(pad):
    h, w, c, ld, cout = 7, 9, 6, 10, 3
    m_in, m_out, idx, pix = _sparse_case(h, w, 11)
    rows = int(m_in.sum())
    t = rnd(rows, ld, seed=12)
    wa, ba, wb, bb = rnd(cout, c, 3, 3, seed=13), rnd(cout, seed=14), rnd(cout, c, 3, 3, seed=15), rnd(cout, seed=16)
    v, s = hr.head_conv3x3_ref(t, ld, c, 0, 4, wa, ba, wb, bb, cout, 2.0, cr.ACT_SIGMOID, pad, idx, pix, len(pix) + 3,
                               len(pix), 1, h, w)
    xidx = idx.reshape(1, 1, h, w).long()

    def one(off, wt, b):
        xv = t[:, off:off + c].double().T.reshape(-1)
        val, _ = osp.conv3x3(wt.double(), b.double(), xv, xidx, m_out.bool(), torch.sigmoid, _MODE[pad])
        sv, _ = osp.conv3x3(wt.double().abs(), b.double().abs(), xv.abs(), xidx, m_out.bool(), None, _MODE[pad])
        return val, sv
    a, sa = one(0, wa, ba)
    b, sb = one(4, wb, bb)
    p = pix.long()
    assert close(v, (2.0 * (a - b)).reshape(cout, -1)[:, p].T)
    assert close(s, (2.0 * (sa + sb)).reshape(cout, -1)[:, p].T)


@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("groups,dual,act", [(1, False, cr.ACT_NONE), (2, True, cr.ACT_ELU), (3, False, cr.ACT_SIGMOID),
                                             (4, True, cr.ACT_NONE), (6, True, cr.ACT_SIGMOID), (8, False, cr.ACT_ELU)])
def test_head_gather_matches_conv2d(pad, groups, dual, act):
    n, h, w, c, col0 = 2, 5, 3, 4, 3
    cout = groups // 2 if dual else groups
    x = rnd(n, 2 * c, h, w, seed=groups)
    heads = [rnd(cout, c, 3, 3, seed=20 + groups)] + ([rnd(cout, c, 3, 3, seed=30 + groups)] if dual else [])
    z = _tap_products(rows_of(x), heads, [0, c][:len(heads)])
    zz = torch.cat([rnd(z.shape[0], col0, seed=7), z, rnd(z.shape[0], 2, seed=8)], 1)      # ldz = col0 + 9 G + 2
    bias = rnd(groups, seed=9)
    v, s = hr.head_gather_ref(zz, zz.shape[1], col0, groups, None, bias, 0.5, act, dual, pad, None, None, None, cout, n,
                              h, w)
    # the same sums as two convolutions of the rows (up to the fp32 rounding of z: compare against z's own values)
    a, sa = _conv(x[:, :c], heads[0], bias[:cout], pad)
    want, want_s = 0.5 * _ACT[act](a), 0.5 * sa
    if dual:
        b, sb = _conv(x[:, c:], heads[1], bias[cout:], pad)
        want, want_s = want - 0.5 * _ACT[act](b), want_s + 0.5 * sb
    got = _rows_nchw(v, n, h, w)
    assert float((got - want).abs().max()) <= 1e-5                  # z is fp32: the sums agree to its rounding
    # exactly: the gather-sum of the fp32 tap products against F.conv2d of a one-hot "tap" weight over z's columns
    zt = _rows_nchw(zz[:, col0:col0 + 9 * groups].double(), n, h, w)           # (N, 9 G, H, W), channel tap G + g
    onehot = torch.zeros(groups, 9 * groups, 3, 3, dtype=torch.float64)
    for tap in range(9):
        onehot[torch.arange(groups), tap * groups + torch.arange(groups), tap // 3, tap % 3] = 1.0
    zp = F.pad(zt, (1, 1, 1, 1), mode=_MODE[pad])
    sums = F.conv2d(zp, onehot, bias.double())
    sabs = F.conv2d(zp.abs(), onehot, bias.double().abs())
    if dual:
        ex = 0.5 * (_ACT[act](sums[:, :cout]) - _ACT[act](sums[:, cout:]))
        ex_s = 0.5 * (sabs[:, :cout] + sabs[:, cout:])
    else:
        ex, ex_s = 0.5 * _ACT[act](sums), 0.5 * sabs
    assert close(got, ex) and close(_rows_nchw(s, n, h, w), ex_s)


@pytest.mark.parametrize("pad", PADS)
def test_head_gather_index_map_matches_sparse_oracle(pad):
    h, w, groups, cout = 6, 8, 6, 3
    m_in, m_out, idx, pix = _sparse_case(h, w, 21)
    rows = int(m_in.sum())
    z = rnd(rows, 9 * groups + 1, seed=22)
    bias = rnd(groups, seed=23)
    v, s = hr.head_gather_ref(z, z.shape[1], 1, groups, idx, bias, 3.0, cr.ACT_SIGMOID, True, pad, pix, len(pix), 1000,
                              cout, 1, h, w)
    # the sparse oracle on z's columns with one-hot tap weights: sum_tap z[row(tap), 1 + tap G + g]
    onehot = torch.zeros(groups, 9 * groups, 3, 3, dtype=torch.float64)
    for tap in range(9):
        onehot[torch.arange(groups), tap * groups + torch.arange(groups), tap // 3, tap % 3] = 1.0
    xv = z[:, 1:1 + 9 * groups].double().T.reshape(-1)
    xidx = idx.reshape(1, 1, h, w).long()
    sums, _ = osp.conv3x3(onehot, bias.double(), xv, xidx, m_out.bool(), None, _MODE[pad])
    sabs, _ = osp.conv3x3(onehot, bias.double().abs(), xv.abs(), xidx, m_out.bool(), None, _MODE[pad])
    p = pix.long()
    sums, sabs = sums.reshape(groups, -1)[:, p].T, sabs.reshape(groups, -1)[:, p].T
    assert close(v, 3.0 * (torch.sigmoid(sums[:, :3]) - torch.sigmoid(sums[:, 3:])))
    assert close(s, 3.0 * (sabs[:, :3] + sabs[:, 3:]))


def test_head_gather_rows_follow_count_and_max_rows():
    h, w = 4, 5
    _, _, idx, pix = _sparse_case(h, w, 31)
    z = rnd(20, 9, seed=32)
    full, _ = hr.head_gather_ref(z, 9, 0, 1, None, None, 1.0, cr.ACT_NONE, False, cr.PAD_ZERO, pix, len(pix), None, 1, 1,
                                 h, w)
    part, _ = hr.head_gather_ref(z, 9, 0, 1, None, None, 1.0, cr.ACT_NONE, False, cr.PAD_ZERO, pix, len(pix), 3, 1, 1, h,
                                 w)
    assert full.shape == (len(pix), 1) and part.shape == (3, 1) and torch.equal(part, full[:3])


@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("clamp01", [False, True])
def test_head_idwt_matches_dwt_inverse(pad, masked, clamp01):
    n, h, w, c, col0 = 2, 3, 4, 5, 2
    x = rnd(n, 2 * c, h, w, seed=41)
    wp, wm = rnd(3, c, 3, 3, seed=42), rnd(3, c, 3, 3, seed=43)
    z = _tap_products(rows_of(x), [wp, wm], [0, c])
    zz = torch.cat([rnd(z.shape[0], col0, seed=44), z], 1)
    bias = rnd(6, seed=45)
    ll = rnd(n, 1, h, w, seed=46, lo=0.0, hi=4.0)
    mask = (torch.from_numpy(np.random.RandomState(47).uniform(size=(n, h, w))) < 0.5).to(torch.uint8) if masked else None
    r = hr.head_idwt_ref(zz, col0, None, mask, bias, 2.0, pad, ll, 0.3, clamp01, n, h, w)
    # independent: the one-hot tap-sum conv of the six groups, the sigmoid difference, the oracle's synthesis
    zt = _rows_nchw(z.double(), n, h, w)
    onehot = torch.zeros(6, 54, 3, 3, dtype=torch.float64)
    for tap in range(9):
        onehot[torch.arange(6), tap * 6 + torch.arange(6), tap // 3, tap % 3] = 1.0
    zp = F.pad(zt, (1, 1, 1, 1), mode=_MODE[pad])
    sums = F.conv2d(zp, onehot, bias.double())
    sabs = F.conv2d(zp.abs(), onehot, bias.double().abs())
    yh = 2.0 * (torch.sigmoid(sums[:, :3]) - torch.sigmoid(sums[:, 3:]))
    s_yh = 2.0 * (sabs[:, :3] + sabs[:, 3:])
    if masked:
        yh, s_yh = yh * mask[:, None].double(), s_yh * mask[:, None].double()
    assert close(r["yh"], yh) and close(r["s_yh"], s_yh)
    if masked:
        assert bool((r["yh"][(mask[:, None] == 0).expand(-1, 3, -1, -1)] == 0).all())
    inv = ohaar.DWTInverse("haar", "zero")
    for name, buf in list(inv.named_buffers()):                      # its fp32 taps +-1/sqrt2, in fp64
        setattr(inv, name, torch.sign(buf).double() * 0.5 ** 0.5)
    out = inv((ll.double(), [yh[:, None]]))
    assert close(r["out"], out)
    disp = out * 0.3
    assert close(r["disp"], disp.clamp(0, 1) if clamp01 else disp)
    # the error scale: every output of a 2 x 2 block carries half of its four coefficients' magnitudes and scales
    blk = 0.5 * (ll.double().abs() + yh.abs().sum(1, keepdim=True) + s_yh.sum(1, keepdim=True))
    assert close(r["s_out"], F.interpolate(blk, scale_factor=2, mode="nearest"))
    assert close(r["s_disp"], 0.3 * r["s_out"])


@pytest.mark.parametrize("c,nz,count", [(32, 54, None), (64, 9, 5), (32, 56, 100)])
def test_head_mlp_matches_matmuls(c, nz, count):
    n1, rows, ldx = 2 * c, 40, c + 4
    x = rnd(rows, ldx, seed=51)
    w1, b1, wz = rnd(n1, c, 1, 1, seed=52), rnd(n1, seed=53), rnd(nz, n1, 1, 1, seed=54)
    z, s = hr.head_mlp_ref(x, c, w1, b1, wz, 0.2, count, 30)
    m = 30 if count is None else min(count, 30)
    xs = x[:m, :c].double()
    pre = torch.einsum("rc,kc->rk", xs, w1.double()[:, :, 0, 0]) + b1.double()
    t = torch.where(pre > 0, pre, 0.2 * pre)
    want = torch.einsum("rk,zk->rz", t, wz.double()[:, :, 0, 0])
    s1 = torch.einsum("rc,kc->rk", xs.abs(), w1.double()[:, :, 0, 0].abs()) + b1.double().abs()
    want_s = torch.einsum("rk,zk->rz", s1 + t.abs(), wz.double()[:, :, 0, 0].abs())
    assert z.shape == (m, nz) and close(z, want) and close(s, want_s)
    z0, _ = hr.head_mlp_ref(x, c, w1, None, wz, 0.2, None, rows)
    pre0 = x[:, :c].double() @ w1.double()[:, :, 0, 0].T
    assert close(z0, torch.where(pre0 > 0, pre0, 0.2 * pre0) @ wz.double()[:, :, 0, 0].T)


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("e", [-146, -140, -130, -127, 0])
def test_bilinear_ulps_floor_rejects_flushed_and_doubled_outputs(e, ac):
    """bilinear_ulps' bound BILINEAR_ULP 2^-23 max|disp| + BILINEAR_FLOOR: torch's own float32 resize of a plane of
    subnormal (or normal) disparities, 6 x 2^-149 and up, meets it; the same output flushed to zero or doubled does not."""
    rs = np.random.RandomState(61)
    disp = torch.from_numpy((np.ldexp(rs.uniform(1.0, 1.5, (2, 1, 12, 20)), e) * 6).astype(np.float32))
    size = (45, 77) if ac else (48, 80)
    got = F.interpolate(disp, size=size, mode="bilinear", align_corners=ac)
    d64 = disp.double()
    assert hr.bilinear_ulps(got, d64, size, ac) <= hr.BILINEAR_ULP
    assert hr.bilinear_ulps(torch.zeros_like(got), d64, size, ac) > hr.BILINEAR_ULP
    assert hr.bilinear_ulps(2 * got, d64, size, ac) > hr.BILINEAR_ULP


def test_bilinear_ulps_requires_torchs_non_finite_pattern():
    disp = torch.rand(1, 1, 6, 8, dtype=torch.float64)
    disp[0, 0, 2, 3] = float("nan")
    disp[0, 0, 4, 6] = float("inf")
    got = F.interpolate(disp, size=(24, 32), mode="bilinear", align_corners=False).float()
    assert hr.bilinear_ulps(got, disp, (24, 32), False) <= hr.BILINEAR_ULP
    spoiled = []
    for v in (float("nan"), float("inf"), -float("inf")):          # a non-finite output where torch's is finite
        g = got.clone()
        g[0, 0, 20, 2] = v
        spoiled.append(g)
    for v in (0.5, -float("inf")):                                  # torch's NaN footprint made finite, or -Inf
        g = got.clone()
        g[torch.isnan(g)] = v
        spoiled.append(g)
    for g in spoiled:
        with pytest.raises(AssertionError):
            hr.bilinear_ulps(g, disp, (24, 32), False)
