"""GPU: the launch symbols no benchmarked or shipped workload calls (launch_check.REACH), each in a small direct case under
the launch-checking harness: every buffer guarded and poisoned, exactly sized workspaces, inputs compared bit for bit,
the result checked against its kernel's contract, and the regions the contract leaves unwritten checked against a
sentinel.

Two symbols have no caller in the package at all (wmd_conv_rows_tc_f32, the whole-tile form of the split-K entry;
wmd_gather_rows_list_f32, the list gather without a maximum): their cases call them through the C ABI under the
guarded allocator and require the same bits as the wrapped form they stand for.
"""
import ctypes

import numpy as np
import pytest
import torch

from wavelet_monodepth_b200 import _lib, ops

import conv_launch as cl
import footprint
import launch_check as lc

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = cl.SENTINEL


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from lc.REPORT.module_report()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _list(n, h, w, p, seed):
    """a sorted pixel list of about p n h w pixels, its device count, and its mask"""
    m = cl.mask((n, h, w), p, seed)
    pix = m.reshape(-1).nonzero()[:, 0].to(torch.int32)
    return pix, torch.tensor([pix.numel()], dtype=torch.int32, device=DEV), m


def _sentinel(shape):
    out = torch.empty(shape, dtype=torch.float32, device=DEV)
    return out.fill_(SENTINEL)


def _untouched(t):
    return bool((t == SENTINEL).all())


def _run(monkeypatch, case, fn):
    h = lc.Harness(monkeypatch)
    with h.workload(case):
        fn()
    monkeypatch.undo()
    assert not h.reached(case), (case, "never called", h.reached(case))
    print("%s: %s" % (case, h.report()))


def test_conv_rows_split_k(monkeypatch):
    """tensor-core conv_rows with splits = 3 (partial sums in an exactly sized workspace, summed by the reduce pass) on
    a pixel list shorter than max_rows: rows past the count and columns past cout keep the sentinel"""
    def run():
        n, h, w, c0, cout = 2, 24, 40, 96, 40
        pix, count, _ = _list(n, h, w, 0.4, 1)
        g = _gen(2)
        x0 = cl.uniform((n * h * w, c0), -1.0, 1.0, g)
        wt = cl.uniform((cout, c0, 3, 3), -1.0, 1.0, g)
        b = cl.uniform((cout,), -1.0, 1.0, g)
        wp = ops.pack_weight(wt, kind="tc", precision="tf32x3")
        max_rows = pix.numel() + 37
        out = _sentinel((max_rows, ops.pad4(cout) + 4))
        ops.conv_rows(x0, c0, wp, b, cout, n, h, w, pixels=pix, count=count, max_rows=max_rows, out=out, splits=3)
        rows = pix.numel()
        assert _untouched(out[rows:]) and _untouched(out[:rows, cout:]), "conv_rows split-K wrote past its rows"
    _run(monkeypatch, "direct:conv_rows_split_k", run)


def test_gather_and_scatter_rows(monkeypatch):
    """gather_rows of a listed subset of an NCHW map into rows, scatter_rows of them back into a sentinel map: the
    gather's rows past the count and pad columns stay zero, the scatter's unlisted pixels keep the sentinel"""
    def run():
        n, c, h, w = 2, 6, 20, 36
        pix, count, m = _list(n, h, w, 0.3, 3)
        x = cl.uniform((n, c, h, w), -2.0, 2.0, _gen(4))
        rows = ops.gather_rows(x, pix, count, max_rows=pix.numel() + 9)
        r = pix.numel()
        assert bool((rows[r:] == 0).all()) and bool((rows[:r, c:] == 0).all()), "gather_rows wrote past its rows"
        out = _sentinel((n, c, h, w))
        ops.scatter_rows(rows, c, pix, count, n, h, w, out=out)
        keep = (m.reshape(n, 1, h, w) == 0).expand(-1, c, -1, -1)
        assert _untouched(out[keep]), "scatter_rows wrote an unlisted pixel"
    _run(monkeypatch, "direct:gather_scatter_rows", run)


def test_idwt_forms(monkeypatch):
    """the fused IDWT -> disparity -> bilinear resize, both corner conventions; the IDWT with each consumer epilogue.
    The 48 x 160 disparity is resized by source steps of exactly 1/4 (align_corners: (48 - 1) / (189 - 1)), so the
    float32 source index is exact and the checker's fp64 resize measures the blend alone on this rough plane."""
    def run():
        g = _gen(5)
        ll = cl.uniform((2, 1, 24, 80), 0.0, 1.0, g)
        hf = cl.uniform((2, 1, 3, 24, 80), -0.2, 0.2, g)
        for ac, size in ((False, (192, 640)), (True, (189, 637))):
            ops.idwt_bilinear(ll, hf, size, disp_scale=0.5, clamp01=True, align_corners=ac)
        ops.idwt_haar(ll, hf, disp_scale=1.0, clamp01=True, epilogue=("disp_to_depth", 0.1, 100.0))
        ops.idwt_haar(ll, hf, epilogue=("div_clamp", 1000.0, 10.0, 1000.0))
    _run(monkeypatch, "direct:idwt_forms", run)


def test_gated_layout_moves(monkeypatch):
    """nchw_to_rows under a gate, with and without the maximum, from device and pinned host maps: the rows of unmarked
    pixels are left untouched, so they keep the allocator's poison bytes; and the full move with a masked maximum"""
    def run():
        n, c, h, w = 2, 12, 16, 28
        _, _, gate = _list(n, h, w, 0.35, 6)
        x = cl.uniform((n, c, h, w), -3.0, 3.0, _gen(7))
        off = gate.reshape(-1) == 0
        for src in (x, x.cpu().pin_memory()):
            for amax in (None, torch.zeros(1, device=DEV)):
                rows = ops.nchw_to_rows(src, gate=gate.reshape(n, 1, h, w), amax=amax)
                torch.cuda.synchronize()
                poison = rows[off].view(torch.int32)
                assert bool((poison == -1).all()), "a gated move wrote the row of an unmarked pixel"
        ops.nchw_to_rows(x, amax=torch.zeros(1, device=DEV), amax_mask=gate)     # every row, the maximum masked
    _run(monkeypatch, "direct:gated_layout_moves", run)


def _abi_case(monkeypatch, case, symbol, fn):
    """fn() under the guarded allocator and the harness's spy: its one libwmd call outside a wrapped entry point is
    `symbol`"""
    h = lc.Harness(monkeypatch)
    with footprint.Footprint() as fp:
        fn()
        torch.cuda.synchronize()
    monkeypatch.undo()
    assert h.outside == [symbol], h.outside
    assert not h.reached(case), (case, "never called", h.reached(case))
    print("%s: %d arenas checked" % (case, fp.checked))


def test_conv_rows_tc_whole_tiles_abi(monkeypatch):
    """wmd_conv_rows_tc_f32 gives the bits of the wrapped conv_rows with splits = 1, and writes nothing past its rows"""
    def run():
        n, h, w, c0, cout = 2, 16, 24, 64, 48
        pix, count, _ = _list(n, h, w, 0.5, 8)
        g = _gen(9)
        x0 = cl.uniform((n * h * w, c0), -1.0, 1.0, g)
        wt = cl.uniform((cout, c0, 3, 3), -1.0, 1.0, g)
        wp = ops.pack_weight(wt, kind="tc", precision="tf32x3")
        max_rows = pix.numel() + 11
        want = ops.conv_rows(x0, c0, wp, None, cout, n, h, w, pixels=pix, count=count, max_rows=max_rows, splits=1)
        out = _sentinel((max_rows, ops.pad4(cout)))
        d = _lib.ConvDesc()
        d.N, d.H, d.W = n, h, w
        d.x0, d.c0, d.ld0, d.rows0 = _lib.ptr(x0), c0, x0.shape[1], x0.shape[0]
        d.w, d.cout, d.taps, d.pad_mode = _lib.ptr(wp.data), cout, 9, ops.PAD_REFLECT
        d.pixels, d.count, d.max_rows = _lib.ptr(pix), _lib.ptr(count), max_rows
        d.y, d.ldy, d.precision = _lib.ptr(out), out.shape[1], _lib.PREC_TF32X3
        ops._launch().wmd_conv_rows_tc_f32(ctypes.byref(d), _lib.stream_ptr())
        r = pix.numel()
        assert _untouched(out[r:]), "wmd_conv_rows_tc_f32 wrote past its rows"
        assert torch.equal(out[:r, :cout], want[:r, :cout])
    _abi_case(monkeypatch, "direct:conv_rows_tc_abi", "wmd_conv_rows_tc_f32", run)


def test_gather_rows_list_abi(monkeypatch):
    """wmd_gather_rows_list_f32 gives the bits of the wrapped gather_rows_list (its amax form with no maximum), and
    writes nothing past the listed rows"""
    def run():
        n, c, h, w = 2, 10, 18, 30
        pix, count, _ = _list(n, h, w, 0.3, 10)
        x = cl.uniform((n, c, h, w), -2.0, 2.0, _gen(11))
        want = ops.gather_rows_list(x, pix, count)
        ld = ops.pad4(c)
        rows = _sentinel((n * h * w, ld))
        ops._launch().wmd_gather_rows_list_f32(_lib.ptr(x), _lib.ptr(rows), ld, c, _lib.ptr(pix), _lib.ptr(count),
                                              n * h * w, n, h, w, _lib.stream_ptr())
        r = pix.numel()
        assert _untouched(rows[r:]), "wmd_gather_rows_list_f32 wrote past its rows"
        assert torch.equal(rows[:r], want[:r])
        assert np.isfinite(rows[:r].cpu().numpy()).all()
    _abi_case(monkeypatch, "direct:gather_rows_list_abi", "wmd_gather_rows_list_f32", run)
