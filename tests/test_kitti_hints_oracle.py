"""CPU: KITTI's depth hints.  oracle.sgbm reproduces OpenCV's StereoSGBM maps stored in tests/golden/kitti_depth_hints*.npz
bit for bit, oracle.depth_hints agrees with the reference script's fused depths, include/wmd_hints.h matches its
binding and the library, and the entry points refuse bad arguments before any CUDA call."""
import ctypes
import hashlib
import os
import re

import numpy as np
import pytest

from oracle import depth_hints as odh
from oracle import sgbm
from wavelet_monodepth_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
SIDES = ("l", "r")

# every symbol of _lib.HINTS_SIGNATURES: a size query, or a launch and the Python entry point that makes it
HINT_SYMBOLS = {
    "wmd_sgbm_ws_bytes": "query",
    "wmd_sgbm_u8": ("launch", "stereo_sgbm"),
    "wmd_depth_hints_ws_bytes": "query",
    "wmd_depth_hints_f32": ("launch", "_fuse"),
}


def load(name):
    with np.load(os.path.join(GOLDEN, "kitti_depth_hints_%s.npz" % name)) as f:
        return {k: f[k] for k in f.files}


@pytest.mark.parametrize("case", sorted(odh.SMALL))
def test_oracle_reproduces_cv2_on_the_small_cases(case):
    fx = load(case)
    assert str(fx["cv2_version"]) == odh.CV2_VERSION
    left, right = fx["%s/left" % case], fx["%s/right" % case]
    seed, H, W = odh.SMALL[case]
    regen = odh.make_pair(seed, H, W)
    assert np.array_equal(regen[0], left) and np.array_equal(regen[1], right)
    for side in SIDES:
        base, lookup, rev = odh.views(left, right, side)
        maps = fx["%s/%s/maps" % (case, side)]
        assert np.array_equal(odh.matcher_maps(base[None], lookup[None], [rev], **sgbm.HINT_PARAMS)[:, 0], maps)
        assert np.array_equal(maps[4:8], maps[8:12])                   # blockSize 2 and 3: one matcher
        assert (maps != -16).mean() > 0.3 and (maps == -16).any()


def test_oracle_reproduces_cv2_stage_variants_min_widths_and_one_row():
    fx = load("stages")
    left, right = fx["stages/left"], fx["stages/right"]
    from oracle.pin_depth_hints import VARIANTS
    for name, kw in VARIANTS.items():
        got = odh.matcher_maps(left[None], right[None], [False], **dict(sgbm.HINT_PARAMS, **kw))[:, 0]
        assert np.array_equal(got, fx["stages/%s" % name]), name
    for nd in sgbm.NUM_DISPARITIES:
        for bs in sgbm.BLOCK_SIZES:
            k = "minw/%d/%d/" % (nd, bs)
            l2, r2 = fx[k + "left"], fx[k + "right"]
            assert l2.shape[1] == sgbm.min_width(nd, bs)
            assert np.array_equal(sgbm.compute(l2, r2, nd, bs, **sgbm.HINT_PARAMS), fx[k + "disp"]), (nd, bs)
            with pytest.raises(ValueError):
                sgbm.compute(l2[:, :-1], r2[:, :-1], nd, bs)
    got = odh.matcher_maps(fx["row/left"][None], fx["row/right"][None], [False], **sgbm.HINT_PARAMS)[:, 0]
    assert np.array_equal(got, fx["row/maps"])


def test_oracle_reproduces_cv2_on_the_photo_pair():
    fx = load("stages")
    left, right = fx["sample/left"], fx["sample/right"]
    for side in SIDES:
        base, lookup, rev = odh.views(left, right, side)
        got = odh.matcher_maps(base[None], lookup[None], [rev], **sgbm.HINT_PARAMS)[:, 0]
        assert np.array_equal(got, fx["sample/%s/maps" % side]), side


def test_one_full_size_matcher_against_its_digest():
    fx = load("full")
    left, right = odh.make_pair(odh.FULL["full0"][0], 320, 1024)
    got = sgbm.compute(left, right, 64, 1, **sgbm.HINT_PARAMS)
    assert hashlib.sha256(got.tobytes()).hexdigest() == str(fx["full0/l/maps_sha256"][0])


def _fusion_cases():
    for case in sorted(odh.SMALL):
        for side in SIDES:
            yield case, case, side
    for side in SIDES:
        yield "stages", "sample", side


@pytest.mark.parametrize("fixture,key,side", list(_fusion_cases()))
def test_fusion_oracle_against_the_reference(fixture, key, side):
    """fp64 mode: the float64 reference's choice is a near-minimum and its depth that matcher's, on every pixel, with
    the recorded count of near-ties decided otherwise; contract mode: the stored fused depth and the recorded flips
    against the float32 reference"""
    fx = load(fixture)
    left, right = fx["%s/left" % key], fx["%s/right" % key]
    base, lookup, rev = odh.views(left, right, side)
    maps = fx["%s/%s/maps" % (key, side)]
    p = "%s/%s/" % (key, side)
    _, i64, errs = odh.fuse(base[None], lookup[None], maps[:, None], [rev], mode="fp64")
    D = odh.depths(maps, odh.cameras(*base.shape[:2], [rev])[0][0, 0, 0])
    ties = odh.check_fp64(errs[:, 0], D, i64[0, 0], fx[p + "ref_f64_index"][0].astype(np.int64),
                          fx[p + "ref_f64_depth"][0])
    assert ties == int(fx[p + "ties_f64"])
    dc, ic, _ = odh.fuse(base[None], lookup[None], maps[:, None], [rev], mode="contract")
    assert np.array_equal(dc[0].view(np.uint32), fx[p + "contract_depth"].view(np.uint32))
    assert int((ic[0] != fx[p + "ref_f32_index"]).sum()) == int(fx[p + "flips_f32"])


def test_depth_rounding_points():
    """depth = fp32(fp32(K00 0.1) / fp32(disp + 1e-7)) (disp > 0): -0.0 for an invalid pixel, +0.0 for disparity 0"""
    k00 = odh.cameras(320, 1024, [False])[0][0, 0, 0]
    assert k00 == np.float32(np.float32(0.58) * np.float32(1024))
    d = odh.depths(np.array([-16, 0, 1, 16, 2559], np.int16), k00)
    assert d.dtype == np.float32 and np.signbit(d[0]) and d[0] == 0 and not np.signbit(d[1]) and d[1] == 0
    assert d[3] == np.float32(k00 * np.float32(0.1)) / np.float32(np.float32(1) + np.float32(1e-7))


def test_fixtures_are_small():
    for name in ("a", "b", "c", "stages", "full"):
        assert os.path.getsize(os.path.join(GOLDEN, "kitti_depth_hints_%s.npz" % name)) < 1 << 20


def header_symbols():
    text = open(os.path.join(REPO, "include", "wmd_hints.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", text))


def test_header_binding_and_library_agree():
    declared = header_symbols()
    assert declared == set(_lib.HINTS_SIGNATURES), declared ^ set(_lib.HINTS_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.LOSS_SIGNATURES, _lib.KITTI_LOSS_SIGNATURES):
        assert not declared & set(other)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    text = open(os.path.join(REPO, "include", "wmd_hints.h")).read()
    assert int(re.search(r"#define WMD_HINTS_MATCHERS (\d+)", text).group(1)) == _lib.HINTS_MATCHERS == 12


def test_every_hint_symbol_is_classified():
    import inspect
    from wavelet_monodepth_b200 import kitti_hints
    assert set(HINT_SYMBOLS) == set(_lib.HINTS_SIGNATURES)
    launches = {s: k[1] for s, k in HINT_SYMBOLS.items() if k != "query"}
    for sym, entry in launches.items():
        owner, _, attr = entry.rpartition(".")
        fn = getattr(getattr(kitti_hints, owner) if owner else kitti_hints, attr)
        assert ".%s(" % sym in inspect.getsource(fn), (sym, entry)
    # no other function of the module calls a launch symbol
    src = inspect.getsource(kitti_hints)
    for sym in launches:
        assert src.count(".%s(" % sym) == 1, sym


BIG = 1 << 20


def test_argument_errors_before_any_cuda_call():
    lib = _lib.load()
    fake = ctypes.c_void_p(0x1000)
    ok = lib.wmd_sgbm_ws_bytes(2, 64, 256, 64, 3)
    assert ok > 0
    for N, H, W, D, bs in ((2, 64, 256, 80, 3), (2, 64, 256, 64, 4), (2, 64, 256, 64, 0), (2, 64, 65, 64, 3),
                           (2, 64, 64, 64, 1), (2, 0, 256, 64, 1), (2, 64, 40000, 64, 1), (-1, 64, 256, 64, 1),
                           (4096, 1024, 1024, 64, 1)):
        assert lib.wmd_sgbm_ws_bytes(N, H, W, D, bs) == 0, (N, H, W, D, bs)
        assert lib.wmd_sgbm_u8(fake, fake, None, N, H, W, D, bs, fake, BIG, fake, None) == -2, (N, H, W, D, bs)
    for W, bs in ((66, 3), (66, 2), (65, 1)):                       # the smallest widths cv2 accepts at D = 64
        assert lib.wmd_sgbm_ws_bytes(1, 8, W, 64, bs) > 0
    assert lib.wmd_sgbm_u8(None, fake, None, 2, 64, 256, 64, 3, fake, ok, fake, None) == -1
    assert lib.wmd_sgbm_u8(fake, fake, None, 2, 64, 256, 64, 3, fake, ok, None, None) == -1
    assert lib.wmd_sgbm_u8(fake, fake, None, 2, 64, 256, 64, 3, fake, ok - 1, fake, None) == -4
    assert lib.wmd_sgbm_u8(None, None, None, 0, 64, 256, 64, 3, None, 0, None, None) == 0
    hb = lib.wmd_depth_hints_ws_bytes(2, 64, 256)
    assert hb > 0 and lib.wmd_depth_hints_ws_bytes(2, 1, 256) == 0 and lib.wmd_depth_hints_ws_bytes(1024, 1024, 1024) == 0
    args = [fake] * 6
    assert lib.wmd_depth_hints_f32(*args, 2, 1, 256, fake, BIG, fake, None, None) == -2
    assert lib.wmd_depth_hints_f32(None, *args[1:], 2, 64, 256, fake, hb, fake, None, None) == -1
    assert lib.wmd_depth_hints_f32(*args, 2, 64, 256, fake, hb, None, None, None) == -1
    assert lib.wmd_depth_hints_f32(*args, 2, 64, 256, fake, hb - 1, fake, None, None) == -4
    assert lib.wmd_depth_hints_f32(*[None] * 6, 0, 64, 256, None, 0, None, None, None) == 0
