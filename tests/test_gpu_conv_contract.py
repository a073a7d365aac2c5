"""GPU: the gather-GEMM convolutions against the fp64 reference of the whole wmd_conv_desc contract (tests/conv_ref.py).

Metric: err = max over the written elements of |y - y64| / S, with S = |bias| + sum |a| |w| (the magnitudes of every term
of the element's dot product).  An fp32-faithful kernel's error is a small multiple of 2^-22 S whatever the data; a kernel
that drops a correction term, a slab or the bias, or lets the tensor core's truncating accumulation run too long, is off
by 1e-4 S or more on some element.  With an activation the slope is <= 1 and the activation's own error (ELU / sigmoid
< 5e-7 absolute, test_conv_epilogue_elu_matches_expm1_over_the_whole_range) is allowed on top.

Operands are mixed-sign (x, w, b uniform in [-1, 1]) or same-sign (x, b in [0, 1], w in [0, 2/K]): the second does not
cancel a one-signed bias, which is what the tensor core's truncating accumulation has.  Every launch also checks that
nothing outside [0, min(count, max_rows)) x [0, cout) of `out` changes (the buffer is prefilled with a sentinel, and the
source rows carry huge values in their padding columns, which must not be read), and that amax_out is exactly max |y|.

Model of the bars: a tf32x3 / f16x3 product carries ~22 mantissa bits (~2^-20 of |a w|); on top of that each accumulation
epoch (K <= 1024) carries the tensor core's truncation bias, which grows with the number of MMAs that add into the
accumulators.  tf32x3 issues 3 MMAs of K = 8 per 8 channels, f16x3 3 MMAs of K = 16 per 16, so tf32x3's bias is twice
f16x3's.  SIMT: fp32 FMA chains with round-to-nearest (no bias, error ~ sqrt(K) 2^-24).

Worst observed err on one H100 80GB HBM3 (132 SMs, 700 W power limit), per case group, mixed-sign | same-sign
(- = not run):
    group       tf32x3              f16x3               simt
    tails       1.5e-6 | 1.4e-5     8.6e-7 | 7.4e-6     2.7e-7 | 1.6e-6
    epochs      1.6e-6 | 1.7e-5     8.7e-7 | 8.6e-6     2.6e-7 | 2.0e-6
    K18432           - | 1.6e-5          - | 8.1e-6          - | 6.5e-6
    schedules   1.6e-6 | 1.0e-5     8.1e-7 | 3.2e-6          - | -
    splits      8.2e-7 | 4.8e-6          - | -               - | -
    gather      1.6e-6 | 9.3e-6     9.7e-7 | 5.3e-6     2.3e-7 | 1.3e-6
    rows0       4.3e-7 | 1.1e-6     2.4e-7 | 5.6e-7          - | -
    epilogue    1.3e-6 | -          5.8e-7 | -          2.5e-7 | -
    grid        1.8e-6 | -               - | -               - | -
    workspace   1.8e-6 | -               - | -               - | -
The same-sign worst is the truncation bias of one full epoch: ~1.6e-8 x K of S for tf32x3, ~8.5e-9 x K for f16x3 (K <= 1024
per epoch), so it does not grow past one epoch.  Bars: 2.4x (tf32x3), 2.9x (f16x3) and 2.3x (simt) the worst observed;
kernels with a correction term, a slab, the bias or the epochs removed were off by 1.0e-4 S or more on some element.
"""
import numpy as np
import pytest
import torch

from wavelet_monodepth_b200 import _lib, ops
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr

pytestmark = pytest.mark.gpu
DEV = "cuda"

BAR, ACT_ALLOW = cr.BAR, cr.ACT_ALLOW
SENTINEL = -3.0e38                # never produced by these layers
PAD_GARBAGE = 1.0e6               # padding columns of the source rows (must not be read)
ENGINES = ["tf32x3", "f16x3", "simt"]
DISTS = ["mixed", "same"]

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst err per (engine, group, operands):")
        for k in sorted(_WORST):
            print("  %-7s %-10s %-6s %.2e  (bar %.1e, %d launches)" % (k + (_WORST[k][0], BAR[k[0]], _WORST[k][1])))


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


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


def _uniform(shape, lo, hi, g):
    return torch.rand(shape, generator=g, device=DEV, dtype=torch.float32) * (hi - lo) + lo


def _source(rows, c, lo, hi, g):
    """rows x c operand in a row buffer whose 4..7 padding columns hold PAD_GARBAGE."""
    x = torch.full((rows, ops.pad4(c) + 4), PAD_GARBAGE, device=DEV)
    x[:, :c] = _uniform((rows, c), lo, hi, g)
    return x


def operands(L, dist, seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    lo = 0.0 if dist == "same" else -1.0
    x0 = _source(L.x0_rows, L.c0, lo, 1.0, g)
    x1 = _source(L.x1_rows, L.c1, lo, 1.0, g) if L.c1 else None
    k = 3 if L.taps == 9 else 1
    wlo, whi = (0.0, 2.0 / L.k) if dist == "same" else (-1.0, 1.0)
    wt = _uniform((L.cout, L.c0 + L.c1, k, k), wlo, whi, g)
    b = _uniform((L.cout,), lo, 1.0, g)
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
    """One launch, checked against the reference; returns the whole output buffer."""
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
    allow = 0.0 if act in (ACT_NONE, ACT_LRELU) else ACT_ALLOW
    err = float(((y.double() - y64).abs() - allow).clamp(min=0).div(s.clamp(min=1e-300)).max()) if rows else 0.0
    key = (engine, group, dist)
    was = _WORST.get(key, (0.0, 0))
    _WORST[key] = (max(was[0], err), was[1] + 1)
    assert err <= BAR[engine], (engine, group, dist, splits, err)
    if tc:
        want = float(y.abs().max()) if rows else 0.0
        assert float(amax_out) == want, ("amax_out", float(amax_out), want)
    return out


# ------------------------------------------------------------------------------------------ N tiles and channel tails
# (cout, c0, c1, n, h, w, pad): cout straddles tc_tile_n's 48 / 96 switches (1-3 N tiles with tails), c0 % 32 in {0, 8, 20},
# c1 in {0, 20, 64}, cin % 4 != 0, rows % 128 in {0, 1, 127}
TAILS = [
    (5, 6, 0, 1, 8, 16, PAD_REFLECT),
    (31, 20, 0, 1, 3, 43, PAD_ZERO),
    (32, 64, 20, 1, 5, 51, PAD_REPLICATE),
    (47, 40, 0, 2, 8, 8, PAD_REFLECT),
    (48, 32, 64, 1, 3, 43, PAD_REFLECT),
    (63, 52, 20, 1, 5, 51, PAD_ZERO),
    (64, 8, 0, 2, 4, 16, PAD_REPLICATE),
    (95, 72, 64, 1, 3, 43, PAD_REFLECT),
    (96, 96, 0, 1, 5, 51, PAD_REFLECT),
    (128, 40, 20, 2, 8, 8, PAD_ZERO),
    (129, 64, 0, 1, 3, 43, PAD_REPLICATE),
    (138, 84, 20, 1, 5, 51, PAD_REFLECT),
    (257, 33, 0, 1, 8, 16, PAD_REFLECT),
]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("cout,c0,c1,n,h,w,pad", TAILS)
def test_tails(cout, c0, c1, n, h, w, pad, engine, dist):
    run(Layer(n, h, w, c0, cout, c1=c1, pad=pad), engine, dist, "tails", seed=cout)


# ------------------------------------------------------------------------------------------ reduction length and epochs
@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
@pytest.mark.parametrize("cin", [992, 1024, 1056, 2080])          # 31, 32, 33 and 65 chunks of one tap
def test_epoch_edges_1x1(cin, engine, splits, dist):
    run(Layer(1, 4, 128, cin, 96, taps=1), engine, dist, "epochs", splits=splits, seed=cin)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
def test_longest_decoder_reduction_same_sign(engine, splits):
    """upconv(4, 0)'s K = 9 x 2048 = 18 432 on post-ELU-like (non-negative) inputs: 18 epochs per whole tile."""
    run(Layer(1, 8, 40, 2048, 256), engine, "same", "K18432", splits=splits, seed=40)


# ------------------------------------------------------------------------------------------ schedules
SCHEDULES = ["3", "sm-1", "sm", "sm+1", "1.5sm", "2sm", "2.3sm", "5.3sm"]


def _tiles(label):
    sm = sm_count()
    return {"3": 3, "sm-1": sm - 1, "sm": sm, "sm+1": sm + 1, "1.5sm": (3 * sm) // 2, "2sm": 2 * sm,
            "2.3sm": (23 * sm) // 10, "5.3sm": (53 * sm) // 10}[label]


@pytest.mark.parametrize("engine,splits,dist", [("tf32x3", 1, "mixed"), ("tf32x3", 0, "mixed"), ("tf32x3", 0, "same"),
                                                ("f16x3", 0, "mixed")])
@pytest.mark.parametrize("label", SCHEDULES)
def test_schedules_by_tile_count(label, engine, splits, dist):
    """One N tile (cout 96 in a 128-wide tile), 18 chunks; the tile count relative to the SM count picks stream-K with up
    to 7 segments (few tiles), 3-slab stream-K (one round and a part), data-parallel rounds + remainder, or none."""
    run(Layer(1, _tiles(label), 128, 64, 96), engine, dist, "schedules", splits=splits, seed=7)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("splits", [0, 1, 2, 5, 9, 12])             # 9 chunks: nchunks and nchunks + 3 (clamped)
def test_splits(splits, dist):
    run(Layer(1, 3, 128, 32, 64), "tf32x3", dist, "splits", splits=splits, seed=8)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ["tf32x3", "f16x3"])
def test_balanced_cut_tiles_with_cout_tail(engine, dist):
    """cout 138: two N tiles, the second with a 10-column tail; 18 tiles on all SMs: every tile is cut."""
    run(Layer(1, 9, 128, 256, 138, c1=0), engine, dist, "schedules", splits=0, seed=9)


# ------------------------------------------------------------------------------------------ gather paths
def _mask(shape, p, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) < p).to(torch.uint8).to(DEV)


def gather_layer(case):
    if case == "shift0_compact_map0":
        lo = _mask((2, 6, 10), 0.6, 1)
        return Layer(2, 12, 20, 40, 64, c1=24, shift0=1, map0=cr.index_map(lo))
    if case == "compact_map1":
        sel = _mask((2, 10, 14), 0.5, 2)
        return Layer(2, 10, 14, 32, 48, c1=20, map1=cr.index_map(sel))
    if case == "gate":
        return Layer(2, 10, 14, 36, 33, c1=8, gate=_mask((2, 10, 14), 0.5, 3))
    if case in ("count_lt_max_rows", "max_rows_lt_count"):
        m_in, m_out = _mask((2, 16, 24), 0.7, 4), _mask((2, 16, 24), 0.4, 5)
        pix = cr.pixel_list(m_out)
        p = len(pix)
        return Layer(2, 16, 24, 48, 96, map0=cr.index_map(m_in), pixels=pix, count=p,
                     max_rows=p + 37 if case == "count_lt_max_rows" else p - 45)
    if case == "decoder_level":                 # sparse_upsample + sparse_conv3x3: compact half-res x0, skip, gate, list
        s0 = _mask((1, 8, 12), 0.5, 6)
        up = s0.repeat_interleave(2, 1).repeat_interleave(2, 2)
        pix = cr.pixel_list(_mask((1, 16, 24), 0.5, 7) * up)
        return Layer(1, 16, 24, 40, 64, c1=20, shift0=1, map0=cr.index_map(s0), gate=up, pixels=pix, count=len(pix))
    if case.startswith("pad_"):
        pad = {"pad_zero": PAD_ZERO, "pad_reflect": PAD_REFLECT, "pad_replicate": PAD_REPLICATE}[case]
        return Layer(1, 13, 17, 24, 40, pad=pad)
    if case.startswith("thin_"):
        _, h, w, pad = case.split("_")
        return Layer(2, int(h), int(w), 20, 36, c1=12, pad={"z": PAD_ZERO, "f": PAD_REFLECT, "r": PAD_REPLICATE}[pad])
    raise KeyError(case)


GATHER = ["shift0_compact_map0", "compact_map1", "gate", "count_lt_max_rows", "max_rows_lt_count", "decoder_level",
          "pad_zero", "pad_reflect", "pad_replicate", "thin_1_37_z", "thin_1_37_r", "thin_2_33_f", "thin_40_1_r",
          "thin_35_2_f", "thin_1_1_z"]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", GATHER)
def test_gather_paths(case, engine, dist):
    run(gather_layer(case), engine, dist, "gather", seed=11)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 2), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
def test_count_zero_writes_nothing(engine, splits):
    pix = cr.pixel_list(_mask((1, 16, 24), 0.5, 12))
    run(Layer(1, 16, 24, 64, 96, pixels=pix, count=0), engine, "mixed", "gather", splits=splits, seed=12)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1)])
def test_1x1_rows_past_rows0_read_zeros(engine, splits, dist):
    """The tensor-core engine's 1x1 form over x0's own rows: x0 holds 300 of the 384 rows (the cut falls inside a tile);
    the rest read zeros from source 0 and still read source 1."""
    run(Layer(1, 6, 64, 40, 64, c1=16, taps=1, x0_rows=300), engine, dist, "rows0", splits=splits, seed=13)


# ------------------------------------------------------------------------------------------ epilogue
def _epi_layer():
    return Layer(1, 9, 128, 64, 138)                 # 2 N tiles (10-column tail), 18 tiles: balanced cuts every tile


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0)])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_ELU, ACT_LRELU, ACT_SIGMOID])
def test_activations(act, engine, splits):
    run(_epi_layer(), engine, "mixed", "epilogue", splits=splits, act=act, seed=14)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 3), ("f16x3", 1), ("f16x3", 0),
                                           ("simt", None)])
@pytest.mark.parametrize("bias", ["none", "off1", "off2", "off3"])
def test_bias_none_and_unaligned_views(bias, engine, splits):
    """bias may be any 4-byte aligned pointer: 1, 2 and 3 floats into an allocation, on whole tiles and on cut tiles."""
    run(_epi_layer(), engine, "mixed", "epilogue", splits=splits, act=ACT_ELU, bias=bias, seed=15)


@pytest.mark.parametrize("engine,splits", [("tf32x3", 1), ("tf32x3", 0), ("tf32x3", 2), ("tf32x3", 3), ("f16x3", 0),
                                           ("simt", None)])
def test_dense_capacity_past_the_image(engine, splits):
    """pixels == NULL with a capacity (max_rows) larger than the image: only the image's rows are written, in every mode."""
    run(Layer(1, 5, 51, 64, 96, max_rows=255 + 130), engine, "mixed", "epilogue", splits=splits, seed=16)


# ------------------------------------------------------------------------------------------ grid independence
def test_results_do_not_depend_on_the_grid():
    """wmd_conv_tc_set_reserved_sms shrinks the persistent grid.  Whole tiles: bit-identical for every grid (a tile's
    arithmetic does not depend on which CTA runs it or where it falls in the ring).  Balanced: within the bar and
    reproducible for every grid."""
    sm = sm_count()
    lib = _lib.load()
    L = Layer(1, 40, 128, 64, 138, c1=32)            # 80 tiles, 27 chunks
    ins = operands(L, "mixed", 17)
    was = lib.wmd_conv_tc_set_reserved_sms(-1)
    whole = []
    try:
        for k in [0, 1, sm // 2, sm - 2, sm - 1]:
            lib.wmd_conv_tc_set_reserved_sms(k)
            whole.append(run(L, "tf32x3", "mixed", "grid", splits=1, ops_in=ins))
            a = run(L, "tf32x3", "mixed", "grid", splits=0, ops_in=ins)
            b = run(L, "tf32x3", "mixed", "grid", splits=0, ops_in=ins)
            assert torch.equal(a, b), k
    finally:
        lib.wmd_conv_tc_set_reserved_sms(was)
    for k, o in enumerate(whole[1:]):
        assert torch.equal(o, whole[0]), k


# ------------------------------------------------------------------------------------------ workspace hygiene
def test_balanced_launches_leave_the_workspace_counters_zero():
    """Back-to-back balanced launches of different tile counts share one scratch buffer; each stays within the bar, and
    the arrival counters at its head are zero afterwards."""
    sm = sm_count()
    for i, tiles in enumerate([3, sm + 1, 2 * sm + 7, 5, sm - 1]):
        run(Layer(1, tiles, 128, 96, 64), "tf32x3", "mixed", "workspace", splits=0, seed=20 + i)
    torch.cuda.synchronize()
    ws = ops._scratch.splitk(torch.device(DEV), 4096)
    assert bool((ws[:1024] == 0).all())
