"""GPU: the coefficient-head kernels and the fused level tail against the fp64 reference of their contracts (tests/head_ref.py).

Metric: err = max over the written elements of (|got - want| - allow) / S, with S the sum of the magnitudes of every term of
the element (head_ref.py) and `allow` the absolute error of the epilogue's expf-based sigmoid / ELU (5e-7) times |scale|,
once per activation that reaches the element.  Operands are mixed-sign (uniform in [-1, 1]) or same-sign (x, b in [0, 1],
w in [0, 2/K]); the second exposes a one-signed bias of an accumulation, which cancellation would hide.  Every launch also
checks what must NOT change: output buffers are prefilled with a sentinel that unlisted pixels, rows past
min(count, max_rows) and z columns past 56 keep; source padding columns and z columns outside [col0, col0 + 9 G) hold 1e6
and must not be read.  The fused level tail is held to more than the fp64 bar: it claims the chain's summation order, so
its yh, reconstruction, disparity, threshold and consumer epilogues are compared bit for bit with head_gather +
idwt_haar + the torch expressions.

Worst observed err (S units) on one H100 80GB HBM3 (132 SMs, 400 W power limit), per kernel and case group,
mixed-sign | same-sign (- = not run):
    kernel         group       err / S
    head_conv3x3   cout-act    3.7e-8  | 1.5e-7       fp32 FMA chains per lane + a butterfly: no bias, ~sqrt(K) 2^-24
                   channels    7.3e-8  | 1.1e-7
                   largest     8.0e-10 | 0            (sigmoid: within the activation allowance)
                   offsets     0       | 0            (sigmoid)
                   sparse      2.2e-8  | 9.9e-8
                   thin        3.7e-9  | -
    head_gather    groups      1.4e-7  | 1.8e-7       nine fp32 adds in tap order
                   sparse      1.1e-7  | 1.8e-7
                   layouts     1.2e-8  | -
    head_idwt      tail        0       | 0            sigmoid-difference coefficients: within the activation allowance;
                   thresh      0       | -            the exact synthesis adds nothing
    head_mlp       rows        1.2e-7  | 1.5e-6       3xTF32 mma.sync, K <= 128: the same-sign worst is the tensor core's
                   strides     1.0e-7  | 1.4e-6       truncating accumulation
                   magnitude   9.6e-8  | 1.7e-6
    idwt_bilinear  0.99 ulp of the largest of the four neighbours, against F.interpolate of the bit-exact disp plane
Bars: about 2.5x the worst observed (head_idwt: head_gather's bar, whose sums it shares bit for bit).  Kernels with the
reflect and replicate rules swapped in head_conv3x3, the bias dropped from head_gather, the lo x hi MMA dropped from
head_mlp, or two outputs of the fused tail's synthesis swapped were off by 4.2e-1 S, 8.8e-1 S, 4.5e-4 S (mixed-sign:
8.0e-5 S) and 1.6e-1 S on some element.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from wavelet_monodepth_b200 import _lib, ops
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

import conv_ref as cr
import head_ref as hr
from contract import Worst, errors
from conv_launch import DEV, mask, sm_count, uniform

pytestmark = pytest.mark.gpu

BAR, BILINEAR_ULP = hr.BAR, hr.BILINEAR_ULP
ACT_ALLOW = cr.ACT_ALLOW          # absolute error of the kernels' expf-based sigmoid / ELU
SENTINEL = -3.0e38                # never produced by these kernels
PAD_GARBAGE = 1.0e6               # source columns a launch must not read
DISTS = ["mixed", "same"]
PADS = [PAD_ZERO, PAD_REFLECT, PAD_REPLICATE]
ERR_SHAPE, ERR_UNSUPPORTED = -2, -5

WORST = Worst("kernel, group, operands")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def _status(excinfo):
    return "status %d," % excinfo


class Geometry:
    """Output grid, the input rows' index map and the output pixel list of one launch.

    form: "dense" (no map, every pixel), "list" (pixel list), "map" (pixel list + an index map with -1 holes inside the
    image; the rows hold only the mapped pixels).  counts: "all", "lt" (count < max_rows), "gt" (count > max_rows), "zero"."""

    def __init__(self, n, h, w, form="dense", counts="all", seed=0):
        self.n, self.h, self.w, self.form = n, h, w, form
        total = n * h * w
        self.map = None
        self.in_rows = total
        if form == "map":
            self.map = cr.index_map(mask((n, h, w), 0.7, seed + 1))
            self.in_rows = max(int(self.map.max()) + 1, 1)
        if form == "dense":
            self.pixels, self.count, self.max_rows = None, None, total
            self.rows = total
            self.written = torch.arange(total, device=DEV)
            return
        self.pixels = cr.pixel_list(mask((n, h, w), 0.5, seed + 2))
        n_list = len(self.pixels)
        count, max_rows = {"all": (n_list, n_list), "lt": (max(n_list - 3, 0), n_list),
                           "gt": (n_list + 5, max(n_list - 2, 0)), "zero": (0, n_list)}[counts]
        self.count, self.max_rows = count, max_rows
        self.rows = min(count, max_rows)
        self.written = self.pixels[:self.rows].long()
        if len(self.pixels) == 0:                           # the kernels read pixels[m] only for m < rows
            self.pixels = torch.zeros(1, dtype=torch.int32, device=DEV)

    def count_t(self):
        return torch.tensor([self.count], dtype=torch.int32, device=DEV) if self.pixels is not None else None


def _check_written(out, geo, cout):
    """out (N, cout, H, W): the pixels outside geo.written keep the sentinel; returns the written rows (rows, cout)."""
    flat = out.permute(0, 2, 3, 1).reshape(-1, cout)
    keep = torch.ones(flat.shape[0], dtype=torch.bool, device=DEV)
    keep[geo.written] = False
    assert bool((flat[keep] == SENTINEL).all()), "pixels outside the list / past min(count, max_rows) were written"
    return flat[geo.written]


# ============================================================================================ head_conv3x3
def run_conv(geo, c, cout, dual, act, pad, dist, group, ld=None, off_a=0, off_b=None, scale=-2.0, bias=True, seed=0):
    g = _gen(seed)
    n, h, w = geo.n, geo.h, geo.w
    if off_b is None:
        off_b = off_a + c
    ld = ld if ld is not None else max(off_a + c, off_b + c if dual else 0) + 3
    lo = 0.0 if dist == "same" else -1.0
    t = torch.full((geo.in_rows, ld), PAD_GARBAGE, device=DEV)
    t[:, off_a:off_a + c] = uniform((geo.in_rows, c), lo, 1.0, g)
    if dual:
        t[:, off_b:off_b + c] = uniform((geo.in_rows, c), lo, 1.0, g)
    wlo, whi = (0.0, 2.0 / (9 * c)) if dist == "same" else (-1.0, 1.0)
    wa, wb = uniform((cout, c, 3, 3), wlo, whi, g), uniform((cout, c, 3, 3), wlo, whi, g)
    ba = uniform((cout,), lo, 1.0, g) if bias else None
    bb = uniform((cout,), lo, 1.0, g) if bias else None
    out = torch.full((n, cout, h, w), SENTINEL, device=DEV)
    kw = dict(off_b=off_b, wb=ops.pack_head_weight(wb), bb=bb) if dual else {}
    ops.head_conv3x3(t, c, off_a, ops.pack_head_weight(wa), ba, n, h, w, cout, scale=scale, act=act, pad=pad,
                     idxmap=geo.map, pixels=geo.pixels, count=geo.count_t(), max_rows=geo.max_rows, out=out, **kw)
    got = _check_written(out, geo, cout)
    want, s = hr.head_conv3x3_ref(t, ld, c, off_a, off_b if dual else -1, wa, ba, wb, bb, cout, scale, act, pad, geo.map,
                                  geo.pixels, geo.count, geo.max_rows, n, h, w)
    allow = 0.0 if act == ACT_NONE else ACT_ALLOW * abs(scale) * (2 if dual else 1)
    err = errors(got, want, s, allow)[0]
    WORST.note(("head_conv3x3", group, dist), err, bar=BAR["head_conv3x3"])
    assert err <= BAR["head_conv3x3"], (group, dist, err)
    return out


ACTS = [ACT_NONE, ACT_ELU, ACT_SIGMOID]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("cout,dual", [(1, False), (2, True), (3, True), (4, False), (1, True), (4, True)])
def test_head_conv3x3_cout_act_pad(cout, dual, act, pad, dist):
    run_conv(Geometry(2, 5, 7), 13, cout, dual, act, pad, dist, "cout-act", seed=cout)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("c,cout,dual,pad", [(1, 1, False, PAD_ZERO), (13, 3, True, PAD_REPLICATE), (32, 2, True, PAD_REFLECT),
                                             (33, 4, False, PAD_ZERO), (138, 3, True, PAD_REPLICATE),
                                             (552, 1, False, PAD_ZERO), (552, 3, True, PAD_REPLICATE)])
def test_head_conv3x3_channels(c, cout, dual, pad, dist):
    """c = 552 dual cout 3 stages 119 KB of weights: the one-CTA-per-SM launch (the NYU DenseDepth-161 heads)."""
    run_conv(Geometry(2, 6, 9, "map", seed=c), c, cout, dual, ACT_NONE, pad, dist, "channels", seed=c)


@pytest.mark.parametrize("dist", DISTS)
def test_head_conv3x3_largest_weights(dist):
    """c = 782 dual cout 4: 225 216 B of staged weights, the most the launch accepts; c = 783 is refused."""
    run_conv(Geometry(1, 5, 11), 782, 4, True, ACT_SIGMOID, PAD_REFLECT, dist, "largest", seed=782)
    t = torch.zeros(55, 2 * 783, device=DEV)
    wp = torch.zeros(9 * 783, 4, device=DEV)
    with pytest.raises(_lib.WmdError, match=_status(ERR_UNSUPPORTED)):
        ops.head_conv3x3(t, 783, 0, wp, None, 1, 5, 11, 4, off_b=783, wb=wp)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("off_a,off_b,ld", [(5, 40, 77), (37, 0, 70), (2, 3, 36)])
def test_head_conv3x3_row_offsets(off_a, off_b, ld, dist):
    """off_a > 0, off_b before / overlapping off_a's slice, ld wider than what is read (the rest holds 1e6)."""
    run_conv(Geometry(1, 7, 6, "list"), 33, 3, True, ACT_SIGMOID, PAD_REFLECT, dist, "offsets", ld=ld, off_a=off_a,
             off_b=off_b, seed=off_a)


@pytest.mark.parametrize("pad", [PAD_ZERO, PAD_REPLICATE])
@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (6, 1), (2, 2), (1, 2), (2, 9), (9, 2)])
def test_head_conv3x3_thin_images(h, w, pad):
    run_conv(Geometry(3, h, w), 13, 3, True, ACT_ELU, pad, "mixed", "thin", seed=h * 10 + w)


@pytest.mark.parametrize("h,w", [(1, 7), (6, 1), (1, 1)])
def test_head_conv3x3_reflect_needs_two_pixels(h, w):
    t = torch.zeros(h * w, 8, device=DEV)
    with pytest.raises(_lib.WmdError, match=_status(ERR_SHAPE)):
        ops.head_conv3x3(t, 8, 0, torch.zeros(72, 1, device=DEV), None, 1, h, w, 1, pad=PAD_REFLECT)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("form,counts", [("dense", "all"), ("list", "all"), ("list", "lt"), ("list", "gt"),
                                         ("list", "zero"), ("map", "all"), ("map", "gt"), ("map", "lt")])
@pytest.mark.parametrize("pad", PADS)
def test_head_conv3x3_pixel_lists_and_index_maps(pad, form, counts, dist):
    """N = 3; the NYU sparse form is a pixel list plus an index map with holes; unlisted pixels keep the sentinel."""
    run_conv(Geometry(3, 9, 13, form, counts, seed=pad), 32, 3, True, ACT_NONE, pad, dist, "sparse", seed=pad + 7,
             bias=counts != "lt")


# ============================================================================================ head_gather
def _z_rows(rows, ldz, col0, ncols, lo, g, storage_offset=0):
    """rows x ldz buffer (optionally starting `storage_offset` floats into its allocation), operand in columns
    [col0, col0 + ncols), PAD_GARBAGE elsewhere."""
    base = torch.full((rows * ldz + storage_offset,), PAD_GARBAGE, device=DEV)
    z = base[storage_offset:].view(rows, ldz)
    z[:, col0:col0 + ncols] = uniform((rows, ncols), lo, 1.0, g)
    return z


def run_gather(geo, groups, dual, act, pad, dist, group, col0=0, ldz=None, storage_offset=0, scale=1.5, bias=True,
               seed=0, z=None):
    g = _gen(seed)
    cout = groups // 2 if dual else groups
    ldz = ldz if ldz is not None else col0 + 9 * groups + 2
    lo = 0.0 if dist == "same" else -1.0
    b = uniform((groups,), lo, 1.0, g) if bias else None
    if z is None:
        z = _z_rows(geo.in_rows, ldz, col0, 9 * groups, lo, g, storage_offset)
    out = torch.full((geo.n, cout, geo.h, geo.w), SENTINEL, device=DEV)
    ops.head_gather(z, groups, b, geo.n, geo.h, geo.w, cout, scale=scale, act=act, dual=dual, pad=pad, idxmap=geo.map,
                    pixels=geo.pixels, count=geo.count_t(), max_rows=geo.max_rows, out=out, col0=col0)
    got = _check_written(out, geo, cout)
    want, s = hr.head_gather_ref(z, z.shape[1], col0, groups, geo.map, b, scale, act, dual, pad, geo.pixels, geo.count,
                                 geo.max_rows, cout, geo.n, geo.h, geo.w)
    allow = 0.0 if act == ACT_NONE else ACT_ALLOW * abs(scale) * (2 if dual else 1)
    err = errors(got, want, s, allow)[0]
    WORST.note(("head_gather", group, dist), err, bar=BAR["head_gather"])
    assert err <= BAR["head_gather"], (group, dist, err)
    return out, z


GROUPS = [(1, False), (2, False), (2, True), (3, False), (4, False), (4, True), (6, False), (6, True), (8, False),
          (8, True)]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("groups,dual", GROUPS)
def test_head_gather_groups(groups, dual, pad, dist):
    act = [ACT_NONE, ACT_ELU, ACT_SIGMOID][groups % 3]
    run_gather(Geometry(2, 7, 10), groups, dual, act, pad, dist, "groups", seed=groups)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("form,counts", [("list", "all"), ("list", "gt"), ("map", "all"), ("map", "lt"), ("map", "zero")])
@pytest.mark.parametrize("groups,dual,act", [(6, True, ACT_SIGMOID), (1, False, ACT_NONE), (4, True, ACT_ELU)])
@pytest.mark.parametrize("pad", PADS)
def test_head_gather_index_maps_and_lists(pad, groups, dual, act, form, counts, dist):
    run_gather(Geometry(3, 9, 11, form, counts, seed=groups), groups, dual, act, pad, dist, "sparse", seed=groups + 3,
               bias=counts != "lt")


@pytest.mark.parametrize("groups,dual", [(2, True), (4, False), (6, True), (8, True), (3, False), (1, False)])
@pytest.mark.parametrize("pad", [PAD_REFLECT, PAD_ZERO])
def test_head_gather_column_offsets_and_strides(groups, dual, pad):
    """Even and odd col0, even and odd ldz, and a z view at an odd storage offset: every layout gives the bits of the
    8-byte aligned launch (float2 loads) on the same values, and meets the fp64 bar."""
    geo = Geometry(2, 6, 9, "map", seed=groups)
    act = ACT_SIGMOID if dual else ACT_ELU
    ref_out, ref_z = run_gather(geo, groups, dual, act, pad, "mixed", "layouts", col0=2, ldz=9 * groups + 4, seed=groups)
    vals = ref_z[:, 2:2 + 9 * groups]
    for col0, ldz, offset in [(1, 9 * groups + 4, 0), (3, 9 * groups + 5, 0), (0, 9 * groups + 1, 0),
                              (0, 9 * groups, 1), (2, 9 * groups + 4, 1), (55, 9 * groups + 56, 0)]:
        z = torch.full((geo.in_rows * ldz + offset,), PAD_GARBAGE, device=DEV)[offset:].view(geo.in_rows, ldz)
        z[:, col0:col0 + 9 * groups] = vals
        out, _ = run_gather(geo, groups, dual, act, pad, "mixed", "layouts", col0=col0, seed=groups, z=z)
        assert torch.equal(out, ref_out), (col0, ldz, offset)


# ============================================================================================ head_idwt
def _idwt_operands(n, h, w, form, col0, ldz, seed, dist="mixed"):
    g = _gen(seed)
    geo_map = cr.index_map(mask((n, h, w), 0.7, seed + 1)) if form == "map" else None
    rows = max(int(geo_map.max()) + 1, 1) if geo_map is not None else n * h * w
    lo = 0.0 if dist == "same" else -1.0
    z = _z_rows(rows, ldz, col0, 54, lo, g)
    z[:, col0:col0 + 54] *= 3.0
    bias = uniform((6,), -1.0, 1.0, g)
    ll = uniform((n, 1, h, w), 0.0, 8.0, g)
    return z, geo_map, bias, ll


def _masks(kind, n, h, w, seed):
    if kind == "none":
        return None
    if kind == "random":
        return mask((n, h, w), 0.4, seed)
    return torch.full((n, h, w), 1 if kind == "ones" else 0, dtype=torch.uint8, device=DEV)


def _range_thresh(out, ratio):
    """(max - min)(out_n) * ratio of each sample, in fp32."""
    o = out.reshape(out.shape[0], -1).cpu().numpy()
    return (o.max(1) - o.min(1)).astype(np.float32) * np.float32(ratio)


def _head_idwt_raw(z, col0, bias, ll, scale, disp_scale, idxmap, mask, pad, clamp01, epi=None):
    """wmd_head_idwt_f32 on ll exactly as given (ops.head_idwt copies an unaligned ll to an aligned one):
    epi = (mode, a, b, lo, hi, want_out1)."""
    lib = _lib.load()
    n, _, h, w = ll.shape
    res = {k: torch.full(s, SENTINEL, device=DEV) for k, s in
           (("yh", (n, 3, h, w)), ("out", (n, 1, 2 * h, 2 * w)), ("disp", (n, 1, 2 * h, 2 * w)))}
    d = _lib.HeadIdwtDesc()
    d.N, d.H, d.W = n, h, w
    d.z, d.ldz = z.data_ptr() + 4 * col0, z.shape[1]
    d.map, d.mask, d.bias = _lib.ptr(idxmap), _lib.ptr(mask), _lib.ptr(bias)
    d.scale, d.pad_mode = float(scale), pad
    d.ll, d.yh, d.out, d.disp = ll.data_ptr(), _lib.ptr(res["yh"]), _lib.ptr(res["out"]), _lib.ptr(res["disp"])
    d.disp_scale, d.clamp01 = float(disp_scale), int(bool(clamp01))
    if epi is not None:
        mode, a, b, elo, ehi, want1 = epi
        res["e0"] = torch.full_like(res["out"], SENTINEL)
        res["e1"] = torch.full_like(res["out"], SENTINEL) if want1 else None
        d.epi_mode, d.epi_a, d.epi_b, d.epi_lo, d.epi_hi = mode, a, b, elo, ehi
        d.epi_out0, d.epi_out1 = _lib.ptr(res["e0"]), _lib.ptr(res["e1"])
    rc = lib.wmd_head_idwt_f32(ctypes.byref(d), None, 0, _lib.stream_ptr())
    _lib.check(rc, "wmd_head_idwt_f32")
    return res


def _check_idwt(res, z, col0, idxmap, mask, bias, scale, pad, ll, disp_scale, clamp01, group, dist, ratio=None):
    n, _, h, w = ll.shape
    ref = hr.head_idwt_ref(z, col0, idxmap, mask, bias, scale, pad, ll, disp_scale, clamp01, n, h, w)
    a = ACT_ALLOW * abs(scale)
    err = max(errors(res["yh"], ref["yh"], ref["s_yh"], 2 * a)[0], errors(res["out"], ref["out"], ref["s_out"], 3 * a)[0],
              errors(res["disp"], ref["disp"], ref["s_disp"], 3 * a * abs(disp_scale))[0])
    WORST.note(("head_idwt", group, dist), err, bar=BAR["head_idwt"])
    if mask is not None:
        off = (mask == 0)[:, None].expand(-1, 3, -1, -1)
        assert bool((res["yh"][off] == 0).all()), "coefficients outside the wavelet mask are not exactly zero"
    assert err <= BAR["head_idwt"], (group, dist, err)
    # the chain the kernel claims bit-identity with: head_gather (groups 6, dual) -> idwt_haar, and the range threshold
    pix, cnt = None, None
    if mask is not None:
        pix = cr.pixel_list(mask)
        cnt = torch.tensor([len(pix)], dtype=torch.int32, device=DEV)
        if len(pix) == 0:
            pix = torch.zeros(1, dtype=torch.int32, device=DEV)
    yh = ops.head_gather(z, 6, bias, n, h, w, 3, scale=scale, act=ACT_SIGMOID, dual=True, pad=pad, idxmap=idxmap,
                         pixels=pix, count=cnt, max_rows=n * h * w, col0=col0)
    assert torch.equal(res["yh"], yh), "yh differs from head_gather(groups=6, dual)"
    out, disp = ops.idwt_haar(ll, yh.reshape(n, 1, 3, h, w), disp_scale=disp_scale, clamp01=clamp01)
    assert torch.equal(res["out"], out), "reconstruction differs from idwt_haar"
    assert torch.equal(res["disp"], disp), "disparity differs from idwt_haar's"
    if ratio is not None:
        assert np.array_equal(res["thresh"].cpu().numpy(), _range_thresh(res["out"], ratio)), "threshold"


# (n, h, w, pad, mask, form, clamp01, bias, col0, ldz): W < 16, plain staging (W % 16 != 0), TMA staging, several x-tiles
# and a partial last x-tile; H of 1, 2, one and two row-tiles and a partial one
IDWT_CASES = [
    (2, 1, 4, PAD_ZERO, "none", "dense", True, True, 0, 56),
    (2, 2, 12, PAD_REFLECT, "random", "map", False, True, 2, 58),
    (3, 7, 16, PAD_REPLICATE, "random", "dense", True, False, 0, 54),
    (1, 8, 20, PAD_REFLECT, "ones", "map", True, True, 4, 64),
    (2, 9, 128, PAD_ZERO, "random", "map", False, True, 0, 56),
    (1, 17, 132, PAD_REFLECT, "none", "dense", True, True, 10, 70),
    (2, 17, 272, PAD_REPLICATE, "random", "map", True, True, 0, 56),
    (1, 8, 272, PAD_REFLECT, "zeros", "dense", False, True, 0, 56),
    (2, 2, 16, PAD_ZERO, "zeros", "map", True, False, 2, 58),
    (1, 1, 132, PAD_REPLICATE, "ones", "map", False, True, 0, 56),
]


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("n,h,w,pad,mask,form,clamp01,bias,col0,ldz", IDWT_CASES)
def test_head_idwt(n, h, w, pad, mask, form, clamp01, bias, col0, ldz, dist):
    seed = 100 * h + w
    z, idxmap, b, ll = _idwt_operands(n, h, w, form, col0, ldz, seed, dist)
    b = b if bias else None
    m = _masks(mask, n, h, w, seed + 5)
    res = ops.head_idwt(z, b, ll, 2.0, 0.3, idxmap=idxmap, mask=m, pad=pad, clamp01=clamp01, col0=col0,
                        thresh_ratio=0.15)
    _check_idwt(res, z, col0, idxmap, m, b, 2.0, pad, ll, 0.3, clamp01, "tail", dist, ratio=0.15)
    if w % 16 == 0:
        # ll as a view one float into its allocation: not 16-byte aligned, so the launch stages it without the TMA
        base = torch.empty(ll.numel() + 4, device=DEV)
        llv = base[1:1 + ll.numel()].view_as(ll)
        llv.copy_(ll)
        assert llv.data_ptr() % 16 != 0
        plain = _head_idwt_raw(z, col0, b, llv, 2.0, 0.3, idxmap, m, pad, clamp01)
        for k in ("yh", "out", "disp"):
            assert torch.equal(plain[k], res[k]), ("plain staging", k)


@pytest.mark.parametrize("n,h,w", [(1, 8, 16), (3, 7, 20), (300, 2, 4)])
def test_head_idwt_threshold_and_counters(n, h, w):
    """The per-sample range threshold is bit-exact for N = 1, 3, 300, and a second call on other data is still right:
    the tickets were left at zero."""
    for rep in range(2):
        z, idxmap, b, ll = _idwt_operands(n, h, w, "dense", 0, 56, 7 + rep)
        m = _masks("random", n, h, w, 9 + rep)
        res = ops.head_idwt(z, b, ll * (1 + rep), 1.0, 0.5, mask=m, pad=PAD_REPLICATE, clamp01=False, thresh_ratio=0.3)
        _check_idwt(res, z, 0, None, m, b, 1.0, PAD_REPLICATE, ll * (1 + rep), 0.5, False, "thresh", "mixed", ratio=0.3)


@pytest.mark.parametrize("w", [16, 20])
def test_head_idwt_epilogues(w):
    """disp_to_depth (with and without the depth plane) and div_clamp (with and without the clamp) equal the torch
    expressions on the kernel's own disparity and reconstruction planes, bit for bit."""
    n, h = 2, 5
    z, idxmap, b, ll = _idwt_operands(n, h, w, "map", 0, 56, 31)
    ll = ll * 100.0
    m = _masks("random", n, h, w, 32)
    kw = dict(idxmap=idxmap, mask=m, pad=PAD_REFLECT)
    r = ops.head_idwt(z, b, ll, 4.0, 0.01, clamp01=True, epilogue=("disp_to_depth", 0.1, 100.0), **kw)
    min_disp, max_disp = 1 / 100.0, 1 / 0.1
    scaled = min_disp + (max_disp - min_disp) * r["disp"]
    assert torch.equal(r["scaled_disp"], scaled)
    assert torch.equal(r["depth"], 1 / scaled)
    raw = _head_idwt_raw(z, 0, b, ll, 4.0, 0.01, idxmap, m, PAD_REFLECT, True,
                         epi=(_lib.EPI_DISP_TO_DEPTH, min_disp, max_disp - min_disp, 0.0, 0.0, False))
    assert torch.equal(raw["disp"], r["disp"]) and torch.equal(raw["e0"], scaled)
    r = ops.head_idwt(z, b, ll, 4.0, 0.01, clamp01=False, epilogue=("div_clamp", 100.0, 0.4, 10.0), **kw)
    assert torch.equal(r["depth"], torch.clamp(r["out"] / 100, min=0.4, max=10))
    r = ops.head_idwt(z, b, ll, 4.0, 0.01, clamp01=False, epilogue=("div_clamp", 100.0, None, None), **kw)
    assert torch.equal(r["depth"], r["out"] / 100)


@pytest.mark.parametrize("w", [8, 9])
def test_idwt_haar_epilogues(w):
    """The same two epilogues on the plain IDWT (both the float2 and the scalar kernel)."""
    g = _gen(41)
    ll = uniform((2, 1, 6, w), 0.0, 800.0, g)
    hf = uniform((2, 1, 3, 6, w), -50.0, 50.0, g)
    out, disp, sd, depth = ops.idwt_haar(ll, hf, disp_scale=1e-3, clamp01=True, epilogue=("disp_to_depth", 0.1, 100.0))
    o2, d2 = ops.idwt_haar(ll, hf, disp_scale=1e-3, clamp01=True)
    assert torch.equal(out, o2) and torch.equal(disp, d2)
    min_disp, max_disp = 1 / 100.0, 1 / 0.1
    scaled = min_disp + (max_disp - min_disp) * disp
    assert torch.equal(sd, scaled) and torch.equal(depth, 1 / scaled)
    lib = _lib.load()
    e0 = torch.full_like(out, SENTINEL)
    rc = lib.wmd_idwt_haar_epi_f32(_lib.ptr(ll), _lib.ptr(hf), _lib.ptr(torch.empty_like(out)), None, 1e-3, 1,
                                   _lib.EPI_DISP_TO_DEPTH, min_disp, max_disp - min_disp, 0.0, 0.0, _lib.ptr(e0), None,
                                   2, 1, 6, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_idwt_haar_epi_f32")
    assert torch.equal(e0, scaled)
    _, depth = ops.idwt_haar(ll, hf, epilogue=("div_clamp", 100.0, 0.4, 10.0))
    assert torch.equal(depth, torch.clamp(out / 100, min=0.4, max=10))
    _, depth = ops.idwt_haar(ll, hf, epilogue=("div_clamp", 100.0, None, None))
    assert torch.equal(depth, out / 100)


# ============================================================================================ head_mlp
def run_mlp(c, max_rows, count, ldx, ldz, nz, bias, slope, mag, dist, group, seed=0):
    g = _gen(seed)
    n1 = 2 * c
    lo = 0.0 if dist == "same" else -1.0
    x = torch.full((max(max_rows, 1), ldx), PAD_GARBAGE, device=DEV)
    x[:, :c] = uniform((x.shape[0], c), lo, 1.0, g) * mag
    w1 = uniform((n1, c, 1, 1), lo, 1.0, g) * (2.0 / c if dist == "same" else 1.0)
    b1 = uniform((n1,), lo, 1.0, g) * mag if bias else None
    wz = uniform((nz, n1, 1, 1), lo, 1.0, g) * (2.0 / n1 if dist == "same" else 1.0)
    packed = ops.pack_head_mlp(w1, b1, wz)
    z = torch.full((max_rows + 3, ldz), SENTINEL, device=DEV)
    cnt = torch.tensor([count], dtype=torch.int32, device=DEV) if count is not None else None
    lib = _lib.load()
    rc = lib.wmd_head_mlp_f32(_lib.ptr(x), ldx, c, _lib.ptr(packed), n1, float(slope), _lib.ptr(cnt), max_rows,
                              _lib.ptr(z), ldz, _lib.stream_ptr())
    _lib.check(rc, "wmd_head_mlp_f32")
    rows = max_rows if count is None else min(count, max_rows)
    assert bool((z[rows:] == SENTINEL).all()), "rows past min(count, max_rows) were written"
    assert bool((z[:rows, 56:] == SENTINEL).all()), "columns past 56 were written"
    assert bool((z[:rows, nz:56] == 0).all()), "columns nz..55 are not zero"
    want, s = hr.head_mlp_ref(x, c, w1, b1, wz, slope, count, max_rows)
    err = errors(z[:rows, :nz], want, s)[0]
    WORST.note(("head_mlp", group, dist), err, bar=BAR["head_mlp"])
    assert err <= BAR["head_mlp"], (group, dist, err)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("rows,count", [(77, None), (1000, None), (300, 0), (4096, 3001), (250, 1000), ("sm", None),
                                        ("sm", "sm-1")])
def test_head_mlp_rows_and_counts(c, rows, count, dist):
    """Rows not a multiple of 16 / 128; count none / 0 / < max_rows / > max_rows; more rows than SMs x 128, so every
    persistent CTA runs several tiles."""
    big = 2 * sm_count() * 128 + 77
    rows = big if rows == "sm" else rows
    count = big - 200 if count == "sm-1" else count
    run_mlp(c, rows, count, c, 56, 54, True, 0.1, 1.0, dist, "rows", seed=c + rows)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("ldx_pad,ldz,nz", [(4, 56, 54), (36, 58, 9), (0, 64, 56), (4, 64, 54)])
def test_head_mlp_strides_and_widths(c, ldx_pad, ldz, nz, dist):
    """ldx in {c, c + 4, c + 36} with 1e6 in the padding; ldz in {56, 58, 64}: columns 56.. keep the sentinel;
    nz in {9, 54, 56}: columns nz..55 are exactly zero."""
    run_mlp(c, 333, None, c + ldx_pad, ldz, nz, True, 0.2, 1.0, dist, "strides", seed=c + ldz)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("mag,bias,slope", [(1e-3, True, 0.1), (3e4, True, 0.2), (1.0, False, 0.1), (3e4, False, 0.1)])
def test_head_mlp_magnitudes(c, mag, bias, slope, dist):
    run_mlp(c, 515, 500, c + 4, 56, 54, bias, slope, mag, dist, "magnitude", seed=c)


# ============================================================================================ idwt_bilinear
def _bilinear_case(n, c, h, w, size, ac, clamp01, scale, seed):
    g = _gen(seed)
    ll = uniform((n, c, h, w), 0.0, 8.0, g)
    hf = uniform((n, c, 3, h, w), -2.0, 2.0, g)
    got = ops.idwt_bilinear(ll, hf, size, disp_scale=scale, clamp01=clamp01, align_corners=ac)
    _, disp = ops.idwt_haar(ll, hf, disp_scale=scale, clamp01=clamp01)
    ulps = hr.bilinear_ulps(got, disp, size, ac)
    WORST.note(("idwt_bilinear", "ulp", "mixed"), ulps, bar=BILINEAR_ULP)
    assert ulps <= BILINEAR_ULP, ulps


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("f", [2, 4, 8])
def test_idwt_bilinear_integer_factors(f, ac):
    h, w = 9, 21
    _bilinear_case(2, 3, h, w, (2 * h * f, 2 * w * f), ac, False, 12.5, seed=f)


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("size", [(100, 100), (100, 103), (131, 257)])
def test_idwt_bilinear_smallest_accepted_factor_and_partial_tiles(size, ac):
    """64 x 64 disparity planes to 100 (1.5625x: (floor(32 s) + 4)(floor(128 s) + 4) = 2040 <= 2048 floats of patch)
    and to sizes that leave partial 32 x 128 tiles; clamp01 off with values of order 100."""
    _bilinear_case(2, 2, 32, 32, size, ac, False, 12.5, seed=size[1])


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("size", [(99, 99), (64, 64), (96, 96)])
def test_idwt_bilinear_rejects_smaller_factors(size, ac):
    """Just below the smallest accepted factor, equal sizes and 1.5x are refused with WMD_ERR_UNSUPPORTED."""
    ll, hf = torch.zeros(1, 1, 32, 32, device=DEV), torch.zeros(1, 1, 3, 32, 32, device=DEV)
    with pytest.raises(_lib.WmdError, match=_status(ERR_UNSUPPORTED)):
        ops.idwt_bilinear(ll, hf, size, align_corners=ac)
