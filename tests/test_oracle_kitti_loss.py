"""oracle.kitti_loss against tests/golden/kitti_hints_loss.npz, pinned on the unmodified reference trainer
(oracle/pin_kitti_loss.py), and the header / binding / library agreement of the KITTI loss entry points.  CPU only.

Bars, as measured when the fixture was pinned:
  * fp64 mode against the reference's float64 run: masks equal on every case; terms within 1e-10 relative and gradient
    samples within 1e-10 of each scale's largest gradient (both runs sum in fp64 in different orders, over up to 2.5e5
    pixels, and the SSIM variance cancels: measured up to 6e-11);
  * contract mode against the reference's float32 run: terms within 1e-3 relative on the random cases, where a few
    float32 mask decisions flip (torch's float32 chain rounds the warp and the SSIM statistics; each flipped hint pixel
    moves a term by about 1e-5 relative); the designed-tie case is compared in fp64 only.
"""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import kitti_loss as okl
from wavelet_monodepth_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "kitti_hints_loss.npz")
FIX = np.load(GOLDEN)
CASES = [str(c) for c in FIX["cases"]]
F64_REL = 1e-10
F32_REL = 1e-3


def _run(name, mode, grads=True):
    case = okl.CASES[name]
    seed = int(FIX["%s/seed" % name])
    inp, disps = okl.make_inputs(case, seed)
    noise = okl.draw_noise(seed, inp, case["loss_scales"])
    return case, okl.run(inp, disps, noise, case["scales"], case["loss_scales"], mode=mode, grads=grads)


def _scalars(name, tag):
    return dict(zip([str(k) for k in FIX["%s/scalar_keys" % name]], FIX["%s/%s/scalars" % (name, tag)]))


def _mask(name, tag, key, s, shape):
    bits = np.unpackbits(FIX["%s/%s/%s/%d" % (name, tag, key, s)])[:int(np.prod(shape))]
    return bits.reshape(shape).astype(np.float64)


@pytest.mark.parametrize("name", CASES)
def test_fp64_oracle_matches_reference_float64(name):
    case, o = _run(name, "fp64")
    for k, v in _scalars(name, "f64").items():
        assert abs(float(o[k]) - v) <= F64_REL * abs(v), (k, float(o[k]), v)
    for s in case["loss_scales"]:
        for key in ("identity_selection", "depth_hint_pixels"):
            want = _mask(name, "f64", key, s, o[key][s].shape)
            assert np.array_equal(o[key][s], want), (key, s, int((o[key][s] != want).sum()))
    for s in case["loss_scales"]:
        idx = FIX["%s/grad_idx/%d" % (name, s)]
        want = FIX["%s/f64/grad/%d" % (name, s)]
        got = o["grad"][s].reshape(-1)[idx]
        scale = np.abs(want).max()
        assert np.abs(got - want).max() <= F64_REL * scale, (s, np.abs(got - want).max() / scale)


@pytest.mark.parametrize("name", [c for c in CASES if okl.CASES[c].get("random", True)])
def test_contract_oracle_near_reference_float32(name):
    case, o = _run(name, "contract", grads=False)
    for k, v in _scalars(name, "f32").items():
        assert abs(float(o[k]) - v) <= F32_REL * abs(v), (k, float(o[k]), v)
    flips = 0
    for s in case["loss_scales"]:
        for key in ("identity_selection", "depth_hint_pixels"):
            flips += int((o[key][s] != _mask(name, "f32", key, s, o[key][s].shape)).sum())
    assert flips <= 1e-3 * sum(o["identity_selection"][s].size for s in case["loss_scales"]), flips


def test_special_case_covers_its_decisions():
    """the designed case has frames with no hint and hints everywhere, clamped warps on both sides and exact ties"""
    case, o = _run("special", "fp64", grads=False)
    inp, disps = okl.make_inputs(case, int(FIX["special/seed"]))
    assert inp["depth_hint_mask"][0].max() == 0 and inp["depth_hint_mask"][1].min() == 1
    assert 0.0 in disps[0] and 1.0 in disps[0]
    D = okl.depth_from_disp(okl.upsample(disps[0], case["H"], case["W"]), 0.1, 100.0)[1]
    ix = okl.project(D, inp["K"], inp["inv_K"], inp["stereo_T"])[0]
    assert (ix < 0).any() and (ix > case["W"] - 1).any()
    assert o["depth_hint_pixels"][1][1].sum() > 0


def test_fixture_is_small():
    assert os.path.getsize(GOLDEN) < 4 << 20


def test_header_declares_the_kitti_entry_points():
    """include/wmd_loss_kitti.h declares exactly the symbols _lib.KITTI_LOSS_SIGNATURES binds, shares none with the other
    tables, lays out wmd_loss_kitti_desc as _lib.KittiLossDesc does, and libwmd.so exports them"""
    text = open(os.path.join(os.path.dirname(GOLDEN), os.pardir, os.pardir, "include", "wmd_loss_kitti.h")).read()
    declared = set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", text, flags=re.S)))
    assert declared == set(_lib.KITTI_LOSS_SIGNATURES), declared ^ set(_lib.KITTI_LOSS_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.LOSS_SIGNATURES):
        assert not declared & set(other)
    fields = re.search(r"typedef struct wmd_loss_kitti_desc \{(.*?)\} wmd_loss_kitti_desc;", text, re.S).group(1)
    names = re.findall(r"\*?(\w+)(?:\[4\])?[,;]", re.sub(r"/\*.*?\*/", "", fields))
    assert names == [f for f, _ in _lib.KittiLossDesc._fields_], names
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libwmd.so is not built")
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name


def test_launch_symbols_are_called_from_the_two_entry_points_only():
    """kitti_loss reaches each launch symbol from one function, _kitti_fwd or _kitti_bwd, the two calls
    tests/test_gpu_kitti_loss.py holds to the oracle; the size queries may be called anywhere"""
    import inspect
    from wavelet_monodepth_b200 import kitti_loss
    src = {name: inspect.getsource(fn) for name, fn in inspect.getmembers(kitti_loss, inspect.isfunction)
           if fn.__module__ == kitti_loss.__name__}
    for cls in (kitti_loss._KittiLossFn, kitti_loss.KittiDepthHintsLoss):
        for name, fn in vars(cls).items():
            fn = getattr(fn, "__func__", fn)
            if inspect.isfunction(fn):
                src["%s.%s" % (cls.__name__, name)] = inspect.getsource(fn)
    for sym, want in (("wmd_loss_kitti_fwd", "_kitti_fwd"), ("wmd_loss_kitti_bwd", "_kitti_bwd")):
        callers = sorted(n for n, text in src.items() if ".%s(" % sym in text)
        assert callers == [want], (sym, callers)


def test_argument_errors_before_any_cuda_call():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libwmd.so is not built")
    lib = _lib.load()
    d = _lib.KittiLossDesc(N=2, H=96, W=320, n_scales=4, n_loss=1, min_depth=0.1, max_depth=100.0)
    assert lib.wmd_loss_kitti_ws_bytes(ctypes.byref(d)) == 0          # null input pointers
    d.N = 0
    assert lib.wmd_loss_kitti_ws_bytes(ctypes.byref(d)) > 0
    for field, bad in (("H", 100), ("W", 12), ("n_loss", 5), ("n_loss", 0), ("max_depth", 0.05)):
        e = _lib.KittiLossDesc.from_buffer_copy(d)
        setattr(e, field, bad)
        assert lib.wmd_loss_kitti_ws_bytes(ctypes.byref(e)) == 0, field
        terms = (ctypes.c_float * 4)()
        rc = lib.wmd_loss_kitti_fwd(ctypes.byref(e), None, None, None, None, ctypes.addressof(terms), 1 << 20,
                                    ctypes.addressof(terms), None)
        assert rc != 0, field
    assert lib.wmd_loss_kitti_fwd(None, None, None, None, None, None, 0, None, None) != 0
    assert lib.wmd_loss_kitti_bwd(None, None, None, None, None, None, None, 0, None, None) != 0
