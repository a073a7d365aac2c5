"""One gather-GEMM convolution launch checked against the fp64 reference of the whole wmd_conv_desc contract
(tests/conv_ref.py), and what the tensor-core form tests share: which kernel a launch ran in, and the layers that pick it.

`run` fills `out` with a sentinel and the source rows' padding columns with huge values, so it also checks that nothing
outside [0, min(count, max_rows)) x [0, cout) of `out` changes and that the padding is not read, and that amax_out is
exactly max |y|.  Each launch's err / S goes to WORST under (engine, group, operands); a module that runs launches
prints its own with `yield from WORST.module_report()` in an autouse module fixture.
"""
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import ops, synth
from wavelet_monodepth_b200._lib import ACT_LRELU, ACT_NONE, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr
from contract import Worst, errors

DEV = "cuda"
SENTINEL = -3.0e38                # never produced by these layers
PAD_GARBAGE = 1.0e6               # padding columns of the source rows (must not be read)
WORST = Worst("engine, group, operands")

WIN, SET, GATHER = "conv_rows_tc_kernel_window", "conv_rows_tc_kernel_rowset", "conv_rows_tc_kernel"
SET_ROWS = 480                    # TC_SET_ROWS: distinct source rows a row-set slot holds


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def mask(shape, p, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) < p).to(torch.uint8).to(DEV)


def uniform(shape, lo, hi, g):
    return torch.rand(shape, generator=g, device=DEV, dtype=torch.float32) * (hi - lo) + lo


class Layer:
    """Geometry and index maps of one launch (index tensors on the device)."""

    def __init__(self, n, h, w, c0, cout, c1=0, taps=9, pad=PAD_REFLECT, shift0=0, map0=None, map1=None, gate=None,
                 pixels=None, count=None, max_rows=None, x0_rows=None):
        self.n, self.h, self.w, self.c0, self.c1, self.cout, self.taps, self.pad = n, h, w, c0, c1, cout, taps, pad
        self.shift0, self.map0, self.map1, self.gate = shift0, map0, map1, gate
        self.pixels, self.count = pixels, count
        total = n * h * w
        self.max_rows = max_rows if max_rows is not None else (len(pixels) if pixels is not None else total)
        if x0_rows is None:
            if map0 is not None:
                x0_rows = max(int(map0.max()) + 1, 1)
            elif taps == 1:
                x0_rows = total
            else:
                x0_rows = n * (h >> shift0) * (w >> shift0)
        self.x0_rows = x0_rows
        self.x1_rows = (max(int(map1.max()) + 1, 1) if map1 is not None else total) if c1 else 0

    @property
    def k(self):
        return self.taps * (self.c0 + self.c1)

    @property
    def rows(self):
        r = self.count if self.pixels is not None else self.n * self.h * self.w
        return min(r, self.max_rows)


def _source(rows, c, lo, hi, g):
    """rows x c operand in a row buffer whose 4..7 padding columns hold PAD_GARBAGE."""
    x = torch.full((rows, ops.pad4(c) + 4), PAD_GARBAGE, device=DEV)
    x[:, :c] = uniform((rows, c), lo, hi, g)
    return x


def operands(L, dist, seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    lo = 0.0 if dist == "same" else -1.0
    x0 = _source(L.x0_rows, L.c0, lo, 1.0, g)
    x1 = _source(L.x1_rows, L.c1, lo, 1.0, g) if L.c1 else None
    k = 3 if L.taps == 9 else 1
    wlo, whi = (0.0, 2.0 / L.k) if dist == "same" else (-1.0, 1.0)
    wt = uniform((L.cout, L.c0 + L.c1, k, k), wlo, whi, g)
    b = uniform((L.cout,), lo, 1.0, g)
    return x0, x1, wt, b


def _bias(b, mode):
    """None, the plain tensor, or a view `mode` floats into a fresh (256-byte aligned) allocation."""
    if mode == "none":
        return None
    off = 0 if mode == "aligned" else int(mode[-1])
    base = torch.zeros(b.numel() + 4, device=DEV)
    base[off:off + b.numel()] = b
    v = base[off:off + b.numel()]
    assert v.data_ptr() % 16 == 4 * off
    return v


def pack(wt, c1, engine):
    if engine == "simt":
        return ops.pack_weight(wt, c1, kind="simt")
    wp = ops.pack_weight(wt, c1, kind="tc", precision=engine)
    assert wp.kind == "tc" and (engine == "tf32x3" or wp.data16 is not None)
    return wp


def run(L, engine, dist, group, splits=None, act=ACT_NONE, act_param=0.2, bias="aligned", seed=0, ops_in=None):
    """One launch, checked against the reference at cr.BAR[engine]; returns the whole output buffer."""
    if engine == "f16x3":
        assert splits in (None, 0, 1), "f16x3 runs whole tiles or balanced only"
    x0, x1, wt, b = ops_in if ops_in is not None else operands(L, dist, seed)
    bv = _bias(b, bias)
    wp = pack(wt, L.c1, engine)
    tc = engine != "simt"
    out = torch.full((L.max_rows + 5, ops.pad4(L.cout) + 4), SENTINEL, device=DEV)
    amax_out = torch.zeros(1, device=DEV) if tc else None
    am0 = x0[:, :L.c0].abs().max().reshape(1) if engine == "f16x3" else None
    am1 = x1[:, :L.c1].abs().max().reshape(1) if engine == "f16x3" and L.c1 else None
    count = torch.tensor([L.count], dtype=torch.int32, device=DEV) if L.pixels is not None else None
    ops.conv_rows(x0, L.c0, wp, bv, L.cout, L.n, L.h, L.w, taps=L.taps, pad=L.pad, act=act, act_param=act_param,
                  map0=L.map0, shift0=L.shift0, x1=x1, c1=L.c1, gate=L.gate, pixels=L.pixels, count=count,
                  max_rows=L.max_rows, out=out, splits=splits if tc else None, map1=L.map1, amax0=am0, amax1=am1,
                  amax_out=amax_out)
    rows = L.rows
    sent = torch.tensor(SENTINEL, device=DEV)
    assert bool((out[rows:] == sent).all()), "rows past min(count, max_rows) were written"
    assert bool((out[:rows, L.cout:] == sent).all()), "columns past cout were written"
    y = out[:rows, :L.cout]
    y64, s = cr.conv_ref(x0, L.c0, wt, bv, L.n, L.h, L.w, taps=L.taps, pad=L.pad, act=act, act_param=act_param,
                         map0=L.map0, shift0=L.shift0, x1=x1, c1=L.c1, map1=L.map1, gate=L.gate, pixels=L.pixels,
                         count=L.count, max_rows=L.max_rows)
    allow = 0.0 if act in (ACT_NONE, ACT_LRELU) else cr.ACT_ALLOW
    what = (engine, group, dist, splits)
    err = errors(y, y64, s, allow, what=what)[0]
    WORST.note((engine, group, dist), err, bar=cr.BAR[engine])
    assert err <= cr.BAR[engine], (what, err)
    if tc:
        want = float(y.abs().max()) if rows else 0.0
        assert float(amax_out) == want, ("amax_out", float(amax_out), want)
    return out


def gather_layer(case):
    if case == "shift0_compact_map0":
        lo = mask((2, 6, 10), 0.6, 1)
        return Layer(2, 12, 20, 40, 64, c1=24, shift0=1, map0=cr.index_map(lo))
    if case == "compact_map1":
        sel = mask((2, 10, 14), 0.5, 2)
        return Layer(2, 10, 14, 32, 48, c1=20, map1=cr.index_map(sel))
    if case == "gate":
        return Layer(2, 10, 14, 36, 33, c1=8, gate=mask((2, 10, 14), 0.5, 3))
    if case in ("count_lt_max_rows", "max_rows_lt_count"):
        m_in, m_out = mask((2, 16, 24), 0.7, 4), mask((2, 16, 24), 0.4, 5)
        pix = cr.pixel_list(m_out)
        p = len(pix)
        return Layer(2, 16, 24, 48, 96, map0=cr.index_map(m_in), pixels=pix, count=p,
                     max_rows=p + 37 if case == "count_lt_max_rows" else p - 45)
    if case == "decoder_level":                 # sparse_upsample + sparse_conv3x3: compact half-res x0, skip, gate, list
        s0 = mask((1, 8, 12), 0.5, 6)
        up = s0.repeat_interleave(2, 1).repeat_interleave(2, 2)
        pix = cr.pixel_list(mask((1, 16, 24), 0.5, 7) * up)
        return Layer(1, 16, 24, 40, 64, c1=20, shift0=1, map0=cr.index_map(s0), gate=up, pixels=pix, count=len(pix))
    if case.startswith("pad_"):
        pad = {"pad_zero": PAD_ZERO, "pad_reflect": PAD_REFLECT, "pad_replicate": PAD_REPLICATE}[case]
        return Layer(1, 13, 17, 24, 40, pad=pad)
    if case.startswith("thin_"):
        _, h, w, pad = case.split("_")
        return Layer(2, int(h), int(w), 20, 36, c1=12, pad={"z": PAD_ZERO, "f": PAD_REFLECT, "r": PAD_REPLICATE}[pad])
    raise KeyError(case)


def decoder_like(n, h, w, seed):
    """sparse_upsample + sparse_conv3x3 of a decoder level: compact half-resolution x0, full-resolution skip x1, the
    upsample mask as gate, the level's pixel list."""
    s0 = mask((n, h // 2, w // 2), 0.5, seed)
    up = s0.repeat_interleave(2, 1).repeat_interleave(2, 2)
    pix = cr.pixel_list(mask((n, h, w), 0.6, seed + 1) * up)
    return Layer(n, h, w, 40, 64, c1=24, shift0=1, map0=cr.index_map(s0), gate=up, pixels=pix, count=len(pix))


def dense_layer(case):
    """A dense 3x3 layer from (n, h, w, c0, c1, cout, pad, shift0)."""
    n, h, w, c0, c1, cout, pad, shift0 = case
    return Layer(n, h, w, c0, cout, c1=c1, pad=pad, shift0=shift0)


def twin(L):
    """The same launch through index maps and a gate that select every pixel.  Its tiles are not dense, so it runs in the
    row-set kernel where tc_rowset_takes (conv_tc.cu) picks that: 3x3, not split, and not a tf32x3 launch of N = 128
    tiles (cout >= 96); otherwise in the gather kernel."""
    total = L.n * L.h * L.w
    src0 = L.n * (L.h >> L.shift0) * (L.w >> L.shift0)
    return Layer(L.n, L.h, L.w, L.c0, L.cout, c1=L.c1, pad=L.pad, shift0=L.shift0,
                 map0=torch.arange(src0, dtype=torch.int32, device=DEV),
                 map1=torch.arange(total, dtype=torch.int32, device=DEV) if L.c1 else None,
                 gate=torch.ones(total, dtype=torch.uint8, device=DEV))


def distinct_rows(pix, h, w, pad):
    """Distinct source rows (shift 0, no map) that the nine taps of these pixels read: the row-set size of their tile."""
    rows = set()
    for p in pix.tolist():
        n, y, x = p // (h * w), (p // w) % h, p % w
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                qy, qx = y + dy, x + dx
                if pad == PAD_ZERO and not (0 <= qy < h and 0 <= qx < w):
                    continue
                if pad == PAD_REFLECT:
                    qy, qx = abs(qy) if qy < h else 2 * h - 2 - qy, abs(qx) if qx < w else 2 * w - 2 - qx
                qy, qx = min(max(qy, 0), h - 1), min(max(qx, 0), w - 1)
                rows.add((n * h + qy) * w + qx)
    return len(rows)


def tc_kernels(fn, launches):
    """Names (WIN, SET or GATHER) of the tensor-core conv kernels fn launches, in launch order.  A short profiling
    session can come back without some kernel records; it is taken again until it holds all `launches`."""
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        evs = sorted((e for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and GATHER in e.name),
                     key=lambda e: e.time_range.start)
        if len(evs) >= launches:
            break
    return [WIN if WIN in e.name else (SET if SET in e.name else GATHER) for e in evs]


FLAGSHIP_DENSE = ((9, 2048, 0, 256), (9, 256, 1024, 256))     # (taps, c0, c1, cout) of its dense 3x3 launches


def flagship_tc_kernels():
    """(taps, c0, c1, cout) and kernel name of every tensor-core conv launch of the flagship sparse decoder (ResNet50
    pyramid, 1024x320, 2 frames, threshold 0.05), in launch order."""
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(synth.RESNET50_CH))
    synth.bench_kitti_params(mod)
    mod = mod.to(DEV).eval()
    feats = [f.to(DEV) for f in synth.bench_kitti_features(2, 320, 1024, synth.RESNET50_CH)]
    mod(feats, 0.05)
    prof = ops.Profiler()
    ops.set_profiler(prof)
    try:
        mod(feats, 0.05)
        torch.cuda.synchronize()
    finally:
        ops.set_profiler(None)
    tc = [info for name, _, info in prof.results() if name == "conv_rows_tc"]
    names = tc_kernels(lambda: mod(feats, 0.05), len(tc))
    return [(info["taps"], info["c0"], info["c1"], info["cout"]) for info in tc], names
