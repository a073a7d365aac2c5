"""GPU: every libwmd kernel against the CPU oracle, through the C ABI (ops.* are thin ctypes wrappers).

Bars: bit-exact for integer / byte / index work (masks, index maps, compaction, layout moves) and for the
Haar synthesis (explicit roundings in the dependency's order); <= 1e-4 relative (north_star) for the
floating-point convolutions, whose summation order differs from the CPU matmul.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import haar as ohaar
from oracle import kitti as okitti
from oracle import sparse_ops as osp
from wavelet_monodepth_b200 import _lib, ops, wavelets
from wavelet_monodepth_b200._lib import (ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE,
                                         PAD_ZERO)

from helpers import REL_TOL, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rnd(*shape, seed=0, lo=-1.0, hi=1.0):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(lo, hi, size=shape).astype(np.float32))


# ------------------------------------------------------------------------------------------ Haar
@pytest.mark.parametrize("shape", [(1, 1, 4, 6), (2, 1, 20, 64), (3, 2, 7, 5), (2, 1, 160, 512)])
def test_idwt_bit_exact_vs_oracle(shape):
    n, c, h, w = shape
    ll, hf = rnd(n, c, h, w, seed=1, lo=0, hi=16), rnd(n, c, 3, h, w, seed=2, lo=-8, hi=8)
    want = ohaar.DWTInverse("haar", "zero")((ll, [hf]))
    got = ops.idwt_haar(ll.to(DEV), hf.to(DEV))
    assert torch.equal(got.cpu(), want)
    out, disp = ops.idwt_haar(ll.to(DEV), hf.to(DEV), disp_scale=0.25, clamp01=True)
    assert torch.equal(out.cpu(), want)
    assert torch.equal(disp.cpu(), torch.clamp(want / 4, 0, 1))
    # the reference's own closed form (depth_decoder.py:225-239) agrees to rounding
    if c == 1:
        assert float((got.cpu() - ohaar.closed_form_idwt(ll, hf)).abs().max()) < 4e-6


def test_idwt_empty_batch_and_module_api():
    idwt = wavelets.IDWT(wave="haar", mode="zero").to(DEV)
    ll, hf = rnd(2, 1, 8, 10, seed=3).to(DEV), rnd(2, 1, 3, 8, 10, seed=4).to(DEV)
    y = idwt((ll, [hf]))
    assert y.shape == (2, 1, 16, 20)
    assert ops.idwt_haar(ll[:0], hf[:0]).shape == (0, 1, 16, 20)
    # non-contiguous band views (the decoders pass yh[:, :, k] style slices around)
    big = rnd(2, 1, 3, 8, 20, seed=5).to(DEV)
    y2 = idwt((ll, [big[..., ::2]]))
    assert torch.equal(y2, idwt((ll, [big[..., ::2].contiguous()])))


@pytest.mark.parametrize("shape", [(2, 1, 240, 320), (1, 3, 6, 10)])
def test_dwt_vs_oracle_and_perfect_reconstruction(shape):
    x = rnd(*shape, seed=6, lo=0, hi=10)
    j = 4 if shape[2] % 16 == 0 else 1
    yl, yh = ohaar.DWTForward(J=j, wave="haar", mode="reflect")(x)
    dwt = wavelets.DWT(J=j, wave="haar", mode="reflect").to(DEV)
    gl, gh = dwt(x.to(DEV))
    assert rel_err(gl, yl) < 1e-6
    for a, b in zip(gh, yh):
        assert a.shape == b.shape and rel_err(a, b) < 2e-6
    rec = wavelets.IDWT(wave="haar").to(DEV)((gl, gh))
    assert rel_err(rec, x) < 2e-6


def test_idwt_autograd_matches_oracle():
    ll = rnd(2, 1, 6, 8, seed=7).requires_grad_(True)
    hf = rnd(2, 1, 3, 6, 8, seed=8).requires_grad_(True)
    wgt = rnd(2, 1, 12, 16, seed=9)
    (ohaar.DWTInverse("haar")((ll, [hf])) * wgt).sum().backward()
    ll_g, hf_g = ll.detach().to(DEV).requires_grad_(True), hf.detach().to(DEV).requires_grad_(True)
    (wavelets.IDWT("haar").to(DEV)((ll_g, [hf_g])) * wgt.to(DEV)).sum().backward()
    assert float((ll_g.grad.cpu() - ll.grad).abs().max()) < 1e-6
    assert float((hf_g.grad.cpu() - hf.grad).abs().max()) < 1e-6
    x = rnd(1, 2, 8, 8, seed=10).requires_grad_(True)
    yl, yh = ohaar.DWTForward(J=2, wave="haar")(x)
    (yl.sum() + sum((h * h).sum() for h in yh)).backward()
    xg = x.detach().to(DEV).requires_grad_(True)
    gl, gh = wavelets.DWT(J=2, wave="haar").to(DEV)(xg)
    (gl.sum() + sum((h * h).sum() for h in gh)).backward()
    assert float((xg.grad.cpu() - x.grad).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------ masks
@pytest.mark.parametrize("n,per", [(1, 7), (3, 4096), (2, 320 * 1024), (5, 40 * 128 + 3)])
def test_range_thresh_bit_exact(n, per):
    x = rnd(n, per, seed=11, lo=-3, hi=9)
    for ratio in (0.05, -1.0, 0.0):
        want = torch.stack([(x[i].max() - x[i].min()) * ratio for i in range(n)])
        got, mm = ops.range_thresh(x.to(DEV), ratio, return_minmax=True)
        assert torch.equal(got.cpu(), want)
        assert torch.equal(mm.cpu()[:, 0], x.min(1)[0]) and torch.equal(mm.cpu()[:, 1], x.max(1)[0])
    # scratch is left clean: a second pass over different data is still right
    y = rnd(n, per, seed=12)
    assert torch.equal(ops.range_thresh(y.to(DEV), 0.1).cpu(), torch.stack([(y[i].max() - y[i].min()) * 0.1
                                                                          for i in range(n)]))


@pytest.mark.parametrize("n,h,w", [(1, 5, 7), (2, 40, 128), (3, 33, 65), (1, 1, 1), (2, 64, 32)])
def test_level_masks_bit_exact(n, h, w):
    yh = rnd(n, 1, 3, h, w, seed=13)
    yh[yh.abs() < 0.3] = 0                              # exact zeros: ratio 0 must drop them (strict >)
    yl = rnd(n, 1, 2 * h, 2 * w, seed=14, lo=0, hi=4)
    for ratio in (0.2, 0.0, -1.0, 0.5):
        thresh = ops.range_thresh(yl.to(DEV), ratio)
        got = ops.level_masks(yh.to(DEV), thresh)
        for b in range(n):
            want = okitti.level_masks(yl[b:b + 1], yh[b:b + 1], ratio)
            for k in ("S0", "S1", "S2", "S3", "S4", "S5"):
                assert torch.equal(got[k][b:b + 1].cpu().bool(), want[k].bool()), (ratio, b, k)
    ones = ops.level_masks(None, None, n=n, h=h, w=w, device=torch.device(DEV))
    assert all(bool(v.all()) for v in ones.values())


@pytest.mark.parametrize("n,h,w,p", [(1, 10, 14, 0.5), (3, 40, 128, 0.2), (2, 31, 67, 0.9), (2, 8, 8, 0.0),
                                     (4, 160, 512, 0.1), (1, 3, 5, 1.0), (7, 1, 3, 0.6), (5, 2, 1, 0.5), (33, 3, 3, 0.4)])
def test_compaction_bit_exact(n, h, w, p):
    rs = np.random.RandomState(15)
    mask = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < p).astype(np.uint8))
    idxmap, pixels, offsets = ops.compact(mask.to(DEV))
    flat = mask.reshape(-1).bool()
    want_idx = torch.where(flat, torch.cumsum(flat.long(), 0) - 1, torch.full((flat.numel(),), -1)).to(torch.int32)
    assert torch.equal(idxmap.reshape(-1).cpu(), want_idx)
    m = int(flat.sum())
    assert torch.equal(pixels[:m].cpu().long(), torch.nonzero(flat).reshape(-1))
    per = mask.reshape(n, -1).sum(1).long()
    assert torch.equal(offsets.cpu().long(), torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(per, 0)]))
    # batch-1 agrees with the reference's mask2idxmap (oracle restatement)
    oi, _ = osp.index_map(mask[:1].float())
    assert torch.equal(idxmap[0].cpu().long(), oi[0, 0])
    gm = ops.gate_map(mask.to(DEV), idxmap)
    assert torch.equal(gm.cpu(), idxmap.cpu())
    lin = ops.gate_map(mask.to(DEV))
    assert torch.equal(lin.reshape(-1).cpu().long(), torch.where(flat, torch.arange(flat.numel()), torch.tensor(-1)))


# ------------------------------------------------------------------------------------------ layout
@pytest.mark.parametrize("n,c,h,w", [(2, 64, 6, 20), (1, 3, 5, 7), (2, 138, 9, 4), (1, 2208, 15, 20)])
def test_layout_round_trips(n, c, h, w):
    x = rnd(n, c, h, w, seed=16)
    rows = ops.nchw_to_rows(x.to(DEV))
    ld = rows.shape[1]
    assert ld == (c + 3) // 4 * 4
    want = x.permute(0, 2, 3, 1).reshape(n * h * w, c)
    assert torch.equal(rows[:, :c].cpu(), want)
    assert ld == c or bool((rows[:, c:] == 0).all())
    assert torch.equal(ops.rows_to_nchw(rows, n, c, h, w).cpu(), x)
    if c % 4 == 0:   # channels_last input is used in place
        cl = x.to(DEV).contiguous(memory_format=torch.channels_last)
        r2 = ops.nchw_to_rows(cl)
        assert r2.data_ptr() == cl.data_ptr() and torch.equal(r2.cpu(), want)
    rs = np.random.RandomState(17)
    mask = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < 0.4).astype(np.uint8)).to(DEV)
    _, pixels, offsets = ops.compact(mask, want_idxmap=False)
    m = int(offsets[n])
    g = ops.gather_rows(x.to(DEV), pixels, offsets[n:])
    assert torch.equal(g[:m, :c].cpu(), want[mask.reshape(-1).bool().cpu()])
    dense = ops.scatter_rows(g, c, pixels, offsets[n:], n, h, w)
    assert torch.equal(dense.cpu(), x * mask.cpu().float())


def test_pack_weight_layout():
    wt = rnd(5, 6, 3, 3, seed=18)
    p = ops.pack_weight(wt.to(DEV), kind="simt").data.cpu()
    assert p.shape == (54, 8)
    want = wt.permute(2, 3, 1, 0).reshape(54, 5)
    assert torch.equal(p[:, :5], want) and bool((p[:, 5:] == 0).all())
    ph = ops.pack_head_weight(wt[:3].to(DEV)).cpu()
    assert torch.equal(ph, wt[:3].permute(2, 3, 1, 0).reshape(54, 3))


# ------------------------------------------------------------------------------------------ conv
@pytest.fixture(params=["simt", "tc"])
def kind(request):
    """Both gather-GEMM engines answer to the same contract: fp32 FMA tiles and wgmma 3xTF32."""
    return request.param


def _torch_conv(x, wt, b, pad, act):
    mode = {PAD_REFLECT: "reflect", PAD_REPLICATE: "replicate", PAD_ZERO: "constant"}[pad]
    y = F.conv2d(F.pad(x, (1, 1, 1, 1), mode=mode), wt, b)
    return {ACT_NONE: lambda t: t, ACT_ELU: F.elu, ACT_LRELU: lambda t: F.leaky_relu(t, 0.2),
            ACT_SIGMOID: torch.sigmoid}[act](y)


@pytest.mark.parametrize("n,cin,cout,h,w,pad,act", [
    (2, 64, 32, 12, 20, PAD_REFLECT, ACT_ELU),          # thin tile config
    (1, 96, 64, 9, 11, PAD_ZERO, ACT_LRELU),            # mid
    (2, 40, 128, 6, 10, PAD_REPLICATE, ACT_NONE),       # wide, channel tail (40 % 32 != 0)
    (1, 372, 138, 5, 7, PAD_REFLECT, ACT_LRELU),        # NYU up3 shapes: cout % 4 != 0
    (1, 6, 5, 10, 14, PAD_REFLECT, ACT_SIGMOID),        # tiny, cin % 4 != 0
    (3, 256, 256, 4, 6, PAD_REFLECT, ACT_ELU),
])
def test_dense_conv_rows_vs_torch(n, cin, cout, h, w, pad, act, kind):
    x, wt, b = rnd(n, cin, h, w, seed=19), rnd(cout, cin, 3, 3, seed=20, lo=-0.1, hi=0.1), rnd(cout, seed=21)
    want = _torch_conv(x, wt, b, pad, act)
    y = ops.conv_rows(ops.nchw_to_rows(x.to(DEV)), cin, ops.pack_weight(wt.to(DEV), kind=kind), b.to(DEV), cout, n, h, w,
                      pad=pad, act=act, act_param=0.2)
    got = ops.rows_to_nchw(y, n, cout, h, w)
    assert rel_err(got, want) <= REL_TOL


def test_conv1x1_rows_vs_torch(kind):
    n, cin, cout, h, w = 2, 32, 64, 7, 9
    x, wt, b = rnd(n, cin, h, w, seed=22), rnd(cout, cin, 1, 1, seed=23), rnd(cout, seed=24)
    want = F.leaky_relu(F.conv2d(x, wt, b), 0.1)
    y = ops.conv_rows(ops.nchw_to_rows(x.to(DEV)), cin, ops.pack_weight(wt.to(DEV), kind=kind), b.to(DEV), cout, n, h, w,
                      taps=1, act=ACT_LRELU, act_param=0.1)
    assert rel_err(ops.rows_to_nchw(y, n, cout, h, w), want) <= REL_TOL


def test_upsample_skip_fused_conv_vs_torch(kind):
    n, c0, c1, cout, h, w = 2, 16, 8, 32, 5, 6       # output grid 2h x 2w
    lo, skip = rnd(n, c0, h, w, seed=25), rnd(n, c1, 2 * h, 2 * w, seed=26)
    wt, b = rnd(cout, c0 + c1, 3, 3, seed=27, lo=-0.2, hi=0.2), rnd(cout, seed=28)
    want = F.elu(F.conv2d(F.pad(torch.cat([F.interpolate(lo, scale_factor=2, mode="nearest"), skip], 1),
                                (1, 1, 1, 1), mode="reflect"), wt, b))
    y = ops.conv_rows(ops.nchw_to_rows(lo.to(DEV)), c0, ops.pack_weight(wt.to(DEV), c1, kind=kind), b.to(DEV), cout, n, 2 * h,
                      2 * w, pad=PAD_REFLECT, act=ACT_ELU, shift0=1, x1=ops.nchw_to_rows(skip.to(DEV)), c1=c1)
    assert rel_err(ops.rows_to_nchw(y, n, cout, 2 * h, 2 * w), want) <= REL_TOL


def _sparse_case(seed, h, w, p_in, p_out):
    rs = np.random.RandomState(seed)
    in_mask = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < p_in).astype(np.float32))
    out_mask = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < p_out).astype(np.float32))
    return in_mask, out_mask


@pytest.mark.parametrize("pad_name,pad", [("reflect", PAD_REFLECT), ("constant", PAD_ZERO), ("replicate", PAD_REPLICATE)])
@pytest.mark.parametrize("p_in,p_out", [(0.6, 0.5), (0.1, 0.9), (1.0, 1.0), (0.5, 0.0), (0.0, 0.5)])
def test_sparse_conv_vs_oracle(pad_name, pad, p_in, p_out, kind):
    """Per-sample oracle (batch-1 reference semantics) vs one batched launch over 2 samples."""
    cin, cout, h, w = 24, 40, 13, 17
    wt, b = rnd(cout, cin, 3, 3, seed=29, lo=-0.2, hi=0.2), rnd(cout, seed=30)
    masks = [_sparse_case(31 + k, h, w, p_in, p_out) for k in range(2)]
    xs = [rnd(cin * int(m[0].sum()), seed=40 + k) for k, m in enumerate(masks)]
    wants = []
    for (im, om), xv in zip(masks, xs):
        idx, _ = osp.index_map(im)
        dense, _ = osp.conv3x3(wt, b, xv, idx, om, nonlin=F.elu, padding=pad_name, make_result=True)
        wants.append(dense)
    in_mask = torch.cat([m[0] for m in masks]).to(torch.uint8).to(DEV)
    out_mask = torch.cat([m[1] for m in masks]).to(torch.uint8).to(DEV)
    rows = torch.cat([xv.reshape(cin, -1).t() for xv in xs] + [torch.zeros(1, cin)]).contiguous().to(DEV)
    idxmap, _, _ = ops.compact(in_mask, want_pixels=False)
    _, pixels, offsets = ops.compact(out_mask, want_idxmap=False)
    y = ops.conv_rows(rows, cin, ops.pack_weight(wt.to(DEV), kind=kind), b.to(DEV), cout, 2, h, w, pad=pad, act=ACT_ELU,
                      map0=idxmap, pixels=pixels, count=offsets[2:])
    got = ops.scatter_rows(y, cout, pixels, offsets[2:], 2, h, w)
    assert rel_err(got, torch.cat(wants)) <= REL_TOL
    assert bool((got.cpu()[out_mask.cpu().expand(-1, cout, -1, -1) == 0] == 0).all())


def test_sparse_upsample_concat_gate_vs_oracle(kind):
    """The fused sparse_upsample + sparse_conv3x3 chain of one decoder level (depth_decoder.py:355-357)."""
    c0, cs, cout, h, w = 16, 8, 32, 9, 11
    rs = np.random.RandomState(50)
    s0 = torch.from_numpy((rs.uniform(size=(1, 1, h, w)) < 0.25).astype(np.float32))
    u = F.interpolate(s0, scale_factor=2, mode="nearest")
    s2, s3, s4 = F.max_pool2d(s0, 5, 1, 2), F.max_pool2d(u, 5, 1, 2), F.max_pool2d(u, 3, 1, 1)
    m2 = int(s2.sum())
    xv = rnd(c0 * m2, seed=51)
    skip = rnd(1, cs, 2 * h, 2 * w, seed=52)
    wt, b = rnd(cout, c0 + cs, 3, 3, seed=53, lo=-0.2, hi=0.2), rnd(cout, seed=54)
    map2, _ = osp.index_map(s2)
    map3, _ = osp.index_map(s3)
    up, uc = osp.upsample_concat(xv, c0, map2, skip, s3, make_result=False)
    want, _ = osp.conv3x3(wt, b, up, map3, s4, nonlin=F.elu, padding="reflect", make_result=True)

    rows = torch.cat([xv.reshape(c0, -1).t(), torch.zeros(1, c0)]).contiguous().to(DEV)
    idx2, _, _ = ops.compact(s2.to(torch.uint8).to(DEV), want_pixels=False)
    _, pix4, off4 = ops.compact(s4.to(torch.uint8).to(DEV), want_idxmap=False)
    y = ops.conv_rows(rows, c0, ops.pack_weight(wt.to(DEV), cs, kind=kind), b.to(DEV), cout, 1, 2 * h, 2 * w, pad=PAD_REFLECT,
                      act=ACT_ELU, map0=idx2, shift0=1, x1=ops.nchw_to_rows(skip.to(DEV)), c1=cs,
                      gate=s3.to(torch.uint8).to(DEV), pixels=pix4, count=off4[1:])
    got = ops.scatter_rows(y, cout, pix4, off4[1:], 1, 2 * h, 2 * w)
    assert rel_err(got, want) <= REL_TOL


@pytest.mark.parametrize("c,cout,dual", [(32, 3, True), (64, 1, False), (138, 3, False), (256, 3, True)])
def test_head_conv_vs_oracle(c, cout, dual):
    n, h, w = 2, 10, 12
    t = rnd(n, 2 * c, h, w, seed=55)
    wa, ba = rnd(cout, c, 3, 3, seed=56, lo=-0.3, hi=0.3), rnd(cout, seed=57)
    wb, bb = rnd(cout, c, 3, 3, seed=58, lo=-0.3, hi=0.3), rnd(cout, seed=59)
    a = torch.sigmoid(F.conv2d(F.pad(t[:, :c], (1, 1, 1, 1), mode="reflect"), wa, ba))
    want = 4.0 * (a - torch.sigmoid(F.conv2d(F.pad(t[:, c:], (1, 1, 1, 1), mode="reflect"), wb, bb))) if dual else 4.0 * a
    rows = ops.nchw_to_rows(t.to(DEV))
    kw = dict(off_b=c, wb=ops.pack_head_weight(wb.to(DEV)), bb=bb.to(DEV)) if dual else {}
    got = ops.head_conv3x3(rows, c, 0, ops.pack_head_weight(wa.to(DEV)), ba.to(DEV), n, h, w, cout, scale=4.0,
                           act=ACT_SIGMOID, pad=PAD_REFLECT, **kw)
    assert rel_err(got, want) <= REL_TOL
    # sparse variant: outputs only at a pixel list, zero elsewhere (make_result semantics)
    rs = np.random.RandomState(60)
    mask = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < 0.3).astype(np.uint8)).to(DEV)
    _, pix, off = ops.compact(mask, want_idxmap=False)
    got_s = ops.head_conv3x3(rows, c, 0, ops.pack_head_weight(wa.to(DEV)), ba.to(DEV), n, h, w, cout, scale=4.0,
                             act=ACT_SIGMOID, pad=PAD_REFLECT, pixels=pix, count=off[n:], **kw)
    assert rel_err(got_s, want * mask.cpu().float()) <= REL_TOL
    assert bool((got_s.cpu()[mask.cpu().expand(-1, cout, -1, -1) == 0] == 0).all())


@pytest.mark.parametrize("c", [32, 128])
def test_factored_head_vs_torch(c, kind):
    """Tap-product GEMM + gather-sum == conv3x3(reflect) -> sigmoid difference of the +/- heads."""
    n, h, w = 2, 9, 14
    t = rnd(n, 2 * c, h, w, seed=70)
    wa, ba = rnd(3, c, 3, 3, seed=71, lo=-0.3, hi=0.3), rnd(3, seed=72)
    wb, bb = rnd(3, c, 3, 3, seed=73, lo=-0.3, hi=0.3), rnd(3, seed=74)
    want = 2.0 * (torch.sigmoid(F.conv2d(F.pad(t[:, :c], (1, 1, 1, 1), mode="reflect"), wa, ba)) -
                  torch.sigmoid(F.conv2d(F.pad(t[:, c:], (1, 1, 1, 1), mode="reflect"), wb, bb)))
    rows = ops.nchw_to_rows(t.to(DEV))
    wz = ops.pack_weight(ops.head_tap_weight([wa.to(DEV), wb.to(DEV)], [0, c], 2 * c), kind=kind)
    z = ops.conv_rows(rows, 2 * c, wz, None, 54, n, h, w, taps=1)
    bias = torch.cat([ba, bb]).to(DEV)
    got = ops.head_gather(z, 6, bias, n, h, w, 3, scale=2.0, act=ACT_SIGMOID, dual=True, pad=PAD_REFLECT)
    assert rel_err(got, want) <= REL_TOL
    rs = np.random.RandomState(75)
    mask = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < 0.3).astype(np.uint8)).to(DEV)
    _, pix, off = ops.compact(mask, want_idxmap=False)
    got_s = ops.head_gather(z, 6, bias, n, h, w, 3, scale=2.0, act=ACT_SIGMOID, dual=True, pad=PAD_REFLECT,
                            pixels=pix, count=off[n:])
    assert rel_err(got_s, want * mask.cpu().float()) <= REL_TOL


@pytest.mark.parametrize("splits", [0, 2, 3, 4])
def test_tc_split_k_vs_torch(splits):
    """Split-K work items + fixed-order reduce pass give the same convolution (and are deterministic)."""
    n, cin, cout, h, w = 2, 160, 128, 9, 13
    x, wt, b = rnd(n, cin, h, w, seed=80), rnd(cout, cin, 3, 3, seed=81, lo=-0.1, hi=0.1), rnd(cout, seed=82)
    want = _torch_conv(x, wt, b, PAD_REFLECT, ACT_ELU)
    rows, wp = ops.nchw_to_rows(x.to(DEV)), ops.pack_weight(wt.to(DEV), kind="tc")
    y = ops.conv_rows(rows, cin, wp, b.to(DEV), cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, splits=splits)
    assert rel_err(ops.rows_to_nchw(y, n, cout, h, w), want) <= REL_TOL
    y2 = ops.conv_rows(rows, cin, wp, b.to(DEV), cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, splits=splits)
    assert torch.equal(y, y2)
    # sparse list + split-K
    rs = np.random.RandomState(83)
    mask = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < 0.4).astype(np.uint8)).to(DEV)
    _, pix, off = ops.compact(mask, want_idxmap=False)
    ys = ops.conv_rows(rows, cin, wp, b.to(DEV), cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, pixels=pix, count=off[n:],
                       splits=splits)
    got = ops.scatter_rows(ys, cout, pix, off[n:], n, h, w)
    assert rel_err(got, want * mask.cpu().float()) <= REL_TOL


@pytest.mark.parametrize("h,w,size,ac", [(12, 40, (192, 640), False), (24, 80, (192, 640), False), (48, 160, (192, 640), False),
                                          (30, 40, (240, 320), True), (7, 9, (50, 31), False), (60, 80, (240, 320), True)])
def test_fused_idwt_bilinear_vs_torch(h, w, size, ac):
    """disp -> full-resolution bilinear plane straight from the coefficients (trainer.py:338-339, NYUv2/utils.py:223-227)."""
    n = 2
    ll, hf = rnd(n, 1, h, w, seed=90, lo=0, hi=8), rnd(n, 1, 3, h, w, seed=91, lo=-2, hi=2)
    disp = torch.clamp(ohaar.DWTInverse("haar", "zero")((ll, [hf])) / 4, 0, 1)
    want = F.interpolate(disp, size, mode="bilinear", align_corners=ac)
    got = ops.idwt_bilinear(ll.to(DEV), hf.to(DEV), size, disp_scale=0.25, clamp01=True, align_corners=ac)
    assert got.shape == want.shape
    assert float((got.cpu() - want).abs().max()) <= 2e-6


@pytest.mark.parametrize("n,c,h,w,p", [(2, 64, 12, 40, 0.3), (1, 5, 7, 9, 0.5), (3, 96, 16, 128, 0.02), (2, 32, 8, 64, 0.0),
                                       (1, 130, 5, 131, 1.0)])
def test_gated_layout_move_writes_exactly_the_marked_rows(n, c, h, w, p):
    """wmd_nchw_to_rows_gated_f32: marked pixels get the same row the plain transpose writes (bit-exact),
    unmarked rows keep whatever the buffer held."""
    g = torch.Generator().manual_seed(n * 1000 + c)
    x = torch.randn(n, c, h, w, generator=g).to(DEV)
    gate = (torch.rand(n, 1, h, w, generator=g) < p).to(torch.uint8).to(DEV)
    want = ops.nchw_to_rows(x)
    ld = want.shape[1]
    lib = _lib.load()
    rows = torch.full((n * h * w, ld), -7.0, device=DEV)
    rc = lib.wmd_nchw_to_rows_gated_f32(_lib.ptr(x), _lib.ptr(rows), _lib.ptr(gate), n, c, h * w, ld, _lib.stream_ptr())
    assert rc == 0
    on = gate.reshape(-1).bool()
    assert torch.equal(rows[on], want[on])
    assert bool((rows[~on] == -7.0).all())
    got = ops.nchw_to_rows(x, gate=gate)                     # wrapper (fresh buffer): marked rows only are defined
    assert torch.equal(got[on], want[on])


@pytest.mark.parametrize("c,rows,count", [(32, 1000, None), (64, 777, None), (32, 4096, 3001), (64, 300, 0), (64, 20000, 19999),
                                          (32, 15, 15)])
def test_fused_head_mlp_vs_torch(c, rows, count):
    """wmd_head_mlp_f32: z = Wz . lrelu(W1 . x + b1) (the 1x1 stages of the +/- heads chained with the tap products)
    against fp64 torch; rows past `count` are not produced."""
    n1, nz = 2 * c, 54
    x = rnd(rows, c, seed=c + rows)
    w1 = rnd(n1, c, 1, 1, seed=1, lo=-0.3, hi=0.3)
    b1 = rnd(n1, seed=2, lo=-0.2, hi=0.2)
    wz = rnd(nz, n1, 1, 1, seed=3, lo=-0.3, hi=0.3)
    assert ops.head_mlp_supported(c, n1) and not ops.head_mlp_supported(128, 256)
    packed = ops.pack_head_mlp(w1.to(DEV), b1.to(DEV), wz.to(DEV))
    cnt = torch.tensor([count], dtype=torch.int32, device=DEV) if count is not None else None
    z = ops.head_mlp(x.to(DEV), c, packed, n1, 0.1, count=cnt, max_rows=rows)
    m = rows if count is None else count
    t = F.leaky_relu(x.double() @ w1.double().reshape(n1, c).T + b1.double(), 0.1)
    want = (t @ wz.double().reshape(nz, n1).T).float()
    assert z.shape == (rows, 56)
    if m:
        assert rel_err(z[:m, :nz].cpu(), want[:m]) <= 1e-5
        assert bool((z[:m, nz:] == 0).all())
    # same numbers as the two-launch path it replaces (both engines are fp32-faithful)
    if m:
        wp = ops.pack_weight(w1.to(DEV), kind="simt")
        t2 = ops.conv_rows(x.to(DEV), c, wp, b1.to(DEV), n1, 1, 1, rows, taps=1, act=ACT_LRELU, act_param=0.1)
        z2 = ops.conv_rows(t2, n1, ops.pack_weight(wz.to(DEV), kind="simt"), None, nz, 1, 1, rows, taps=1)
        assert rel_err(z[:m, :nz], z2[:m, :nz]) <= 1e-5


def _blob_mask(n, h, w, p, seed, grow):
    """uint8 (n,1,h,w): random seeds dilated `grow` times by a 3x3 window - clustered like the decoder's dilated sets."""
    rs = np.random.RandomState(seed)
    m = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < p).astype(np.float32))
    for _ in range(grow):
        m = F.max_pool2d(m, 3, 1, 1)
    return m.to(torch.uint8)


@pytest.mark.parametrize("case", ["dense_two_sources", "blobs_two_sources_balanced", "blobs_one_source", "isolated_pixels_fallback",
                                  "thin_n32", "wide_n128"])
def test_shared_tap_gather_is_bit_identical_to_per_tap_gather(case):
    """conv_rows_tc<N, SH>: one raw-stage fill per (chunk, dy) feeding the three dx taps through the slot table must give
    the bits of the one-gather-per-tap form (same MMAs, same order) - dense grids, clustered active lists (extras at
    run ends), isolated pixels (extras overflow -> per-chunk fills), stream-K cuts that start mid-group, all N tiles."""
    from wavelet_monodepth_b200 import _lib
    lib = _lib.load()
    cfg = {
        "dense_two_sources": dict(n=2, h=40, w=64, c0=64, c1=96, cout=64, p=None, grow=0, pad=PAD_REFLECT),
        "blobs_two_sources_balanced": dict(n=3, h=48, w=96, c0=256, c1=64, cout=64, p=0.02, grow=2, pad=PAD_REFLECT),
        "blobs_one_source": dict(n=4, h=64, w=80, c0=128, c1=0, cout=64, p=0.03, grow=2, pad=PAD_ZERO),
        "isolated_pixels_fallback": dict(n=2, h=48, w=64, c0=64, c1=32, cout=48, p=0.35, grow=0, pad=PAD_REPLICATE),
        "thin_n32": dict(n=2, h=64, w=128, c0=32, c1=64, cout=32, p=0.04, grow=1, pad=PAD_REFLECT),
        "wide_n128": dict(n=2, h=24, w=40, c0=160, c1=96, cout=128, p=0.05, grow=2, pad=PAD_REFLECT),
    }[case]
    n, h, w, c0, c1, cout = (cfg[k] for k in ("n", "h", "w", "c0", "c1", "cout"))
    wt, b = rnd(cout, c0 + c1, 3, 3, seed=70, lo=-0.1, hi=0.1), rnd(cout, seed=71)
    wp = ops.pack_weight(wt.to(DEV), c1, kind="tc")
    kw = dict(pad=cfg["pad"], act=ACT_ELU)
    if c1:                                               # upconv(i,1) form: low-res source through map + shift, skip source gated
        lo_rows = rnd(n * (h // 2) * (w // 2), c0, seed=72).to(DEV)
        skip = rnd(n * h * w, c1, seed=73).to(DEV)
        kw.update(shift0=1, x1=skip, c1=c1)
    else:
        lo_rows = rnd(n * h * w, c0, seed=72).to(DEV)
    if cfg["p"] is not None:
        out_mask = _blob_mask(n, h, w, cfg["p"], 74, cfg["grow"]).to(DEV)
        _, pixels, offsets = ops.compact(out_mask, want_idxmap=False)
        kw.update(pixels=pixels, count=offsets[n:])
        if c1:
            gate = _blob_mask(n, h, w, cfg["p"], 74, cfg["grow"] + 1).to(DEV)          # superset of the outputs
            lo_mask = _blob_mask(n, h // 2, w // 2, 0.5, 75, 1).to(DEV)
            map0, _, _ = ops.compact(lo_mask, want_pixels=False)
            kw.update(gate=gate, map0=map0)
        else:
            in_mask = _blob_mask(n, h, w, cfg["p"], 74, max(cfg["grow"] - 1, 0)).to(DEV)
            map0, _, _ = ops.compact(in_mask, want_pixels=False)
            kw.update(map0=map0)
        assert int(offsets[n]) > 3 * 256                # several tiles
    outs = []
    was = lib.wmd_conv_tc_set_shared_taps(-1)
    try:
        for sh in (0, 1):
            lib.wmd_conv_tc_set_shared_taps(sh)
            for _ in range(2):                           # twice: deterministic
                outs.append(ops.conv_rows(lo_rows, c0, wp, b.to(DEV), cout, n, h, w, **kw).clone())
            torch.cuda.synchronize()
    finally:
        lib.wmd_conv_tc_set_shared_taps(was)
    rows = int(kw["count"][0]) if "count" in kw else n * h * w
    for o in outs[1:]:
        assert torch.equal(o[:rows, :cout], outs[0][:rows, :cout])
    assert float(outs[0][:rows].abs().max()) > 0


@pytest.mark.parametrize("n,c,h,w,p", [(2, 64, 12, 40, 0.3), (1, 5, 7, 9, 0.5), (3, 96, 16, 128, 0.02), (2, 32, 8, 64, 0.0), (2, 130, 9, 33, 1.0)])
def test_gather_rows_list_matches_indexing(n, c, h, w, p):
    x = rnd(n, c, h, w, seed=90)
    mask = _blob_mask(n, h, w, p, 91, 1).to(DEV) if 0 < p < 1 else torch.full((n, 1, h, w), int(p), dtype=torch.uint8, device=DEV)
    _, pixels, offsets = ops.compact(mask, want_idxmap=False)
    m = int(offsets[n])
    want = x.permute(0, 2, 3, 1).reshape(n * h * w, c)[mask.reshape(-1).bool().cpu()]
    for src in (x.to(DEV), x.pin_memory()):
        rows = ops.gather_rows_list(src, pixels, offsets[n:])
        assert torch.equal(rows[:m, :c].cpu(), want)
        assert rows.shape[1] == ops.pad4(c) and bool((rows[:m, c:] == 0).all())


@pytest.mark.parametrize("scale", [1.0, 1e-3, 3e4])
@pytest.mark.parametrize("n,cin,c1,cout,h,w", [(2, 64, 0, 32, 12, 20), (1, 96, 32, 64, 9, 11), (2, 40, 0, 128, 6, 10), (2, 256, 64, 256, 8, 12)])
def test_f16x3_conv_matches_fp64_reference_across_magnitudes(n, cin, c1, cout, h, w, scale):
    """precision = f16x3: operands fed as fp16 pairs of power-of-two scaled values (scale from the sources' max |x|, weights'
    scale in the packed header), fp32 accumulation - as accurate as the tf32 hi/lo form whatever the magnitude of the
    activations (1e-3 .. 3e4: far outside fp16's own range without the scaling)."""
    c0 = cin - c1
    x0 = rnd(n, c0, h, w, seed=80) * scale
    x1 = rnd(n, c1, h, w, seed=81) * scale * 0.25 if c1 else None
    wt, b = rnd(cout, cin, 3, 3, seed=82, lo=-0.1, hi=0.1), rnd(cout, seed=83) * scale
    xin = torch.cat([x0, x1], 1) if c1 else x0
    want = F.elu(F.conv2d(F.pad(xin.double(), (1, 1, 1, 1), mode="reflect"), wt.double(), b.double())).float()
    wp = ops.pack_weight(wt.to(DEV), c1, kind="tc", precision="f16x3")
    assert wp.data16 is not None
    am = torch.zeros(3, device=DEV)
    r0 = ops.nchw_to_rows(x0.to(DEV), amax=am[0:1])
    r1 = ops.nchw_to_rows(x1.to(DEV), amax=am[1:2]) if c1 else None
    assert float(am[0]) == float(x0.abs().max())
    kw = dict(pad=PAD_REFLECT, act=ACT_ELU, x1=r1, c1=c1)
    y16 = ops.conv_rows(r0, c0, wp, b.to(DEV), cout, n, h, w, amax0=am[0:1], amax1=am[1:2] if c1 else None, amax_out=am[2:3], **kw)
    y32 = ops.conv_rows(r0, c0, wp, b.to(DEV), cout, n, h, w, **kw)
    got16, got32 = ops.rows_to_nchw(y16, n, cout, h, w), ops.rows_to_nchw(y32, n, cout, h, w)
    e16, e32 = rel_err(got16, want), rel_err(got32, want)
    assert e16 <= 1e-5 and e16 <= 2 * e32 + 1e-6, (e16, e32)        # both carry the truncating accumulation's bias
    assert abs(float(am[2]) - float(got16.abs().max())) <= 1e-6 * float(got16.abs().max())


def test_conv_epilogue_elu_matches_expm1_over_the_whole_range():
    """The tensor-core engine's ELU uses a short branch-free e^v - 1 (Taylor above -0.25, 2^(v log2 e) - 1 on the SFU below):
    an identity 1x1 convolution passes x through to 22 bits (hi + tf32(lo)), so y - ELU(x) is the activation's own error
    plus that: < 5e-7 absolute for x <= 0, including both sides of the -0.25 switch and large negatives."""
    c = 128
    n, h, w = 1, 8, 64
    x = torch.empty(n, c, h, w)
    flat = x.view(-1)
    g = torch.Generator().manual_seed(5)
    flat.copy_(torch.cat([torch.linspace(-30.0, 4.0, flat.numel() // 2),
                          -torch.rand(flat.numel() // 4, generator=g) * 0.6,                 # dense around the switch
                          torch.rand(flat.numel() - flat.numel() // 2 - flat.numel() // 4, generator=g) * 2e-3 - 1e-3]))
    flat[:4] = torch.tensor([-0.25, -0.2500001, -0.2499999, -88.0])
    wt = torch.eye(c).reshape(c, c, 1, 1)
    wp = ops.pack_weight(wt.to(DEV), 0, kind="tc")
    assert wp.kind == "tc"
    y = ops.conv_rows(ops.nchw_to_rows(x.to(DEV)), c, wp, None, c, n, h, w, taps=1, act=ACT_ELU)
    got = ops.rows_to_nchw(y, n, c, h, w).cpu().double()
    want = torch.where(x > 0, x.double(), torch.expm1(x.double()))
    err = (got - want).abs()
    neg = x <= 0
    # the operands carry 22 mantissa bits (hi + tf32(lo)): 2.4e-7 relative on the input, on top of the activation's own error
    assert float(err[neg].max()) < 5e-7, float(err[neg].max())
    assert float((err[~neg] / want[~neg]).max()) < 5e-7
    near0 = neg & (x.abs() < 0.2) & (x != 0)
    assert float((err[near0] / want[near0].abs()).max()) < 6e-7                       # relative where the result is small


@pytest.mark.parametrize("n,c,h,w,p", [(2, 70, 12, 40, 0.3), (1, 33, 9, 130, 0.6)])
def test_layout_moves_report_the_maximum_of_what_they_move(n, c, h, w, p):
    """amax side channel of the layout moves (operand scaling of the f16x3 form): plain = max |x| of the map, gated = at
    least the maximum over the marked rows (it covers whole 32-pixel groups), list gather = exactly the listed rows."""
    x = rnd(n, c, h, w, seed=70) * 37.0
    rs = np.random.RandomState(71)
    gate = torch.from_numpy((rs.uniform(size=(n, 1, h, w)) < p).astype(np.uint8)).to(DEV)
    am = torch.zeros(3, device=DEV)
    ops.nchw_to_rows(x.to(DEV), amax=am[0:1])
    rows_g = ops.nchw_to_rows(x.to(DEV), gate=gate, amax=am[1:2])
    _, pixels, offsets = ops.compact(gate, want_idxmap=False)
    ops.gather_rows_list(x.to(DEV), pixels, offsets[n:], amax=am[2:3])
    marked = gate.reshape(-1).bool().cpu()
    want_rows = x.permute(0, 2, 3, 1).reshape(-1, c)[marked]
    assert float(am[0]) == float(x.abs().max())
    assert float(am[2]) == float(want_rows.abs().max())
    assert float(want_rows.abs().max()) <= float(am[1]) <= float(x.abs().max())
    assert torch.equal(rows_g[marked.to(DEV)][:, :c].cpu(), want_rows)
