"""oracle.kitti_loss against tests/golden/kitti_hints_loss*.npz (oracle.kitti_loss.FIXTURES), pinned on the unmodified
reference trainer (oracle/pin_kitti_loss.py), and the header / binding / library agreement of the KITTI loss entry
points.  CPU only.

Bars, as measured when the fixture was pinned:
  * fp64 mode against the reference's float64 run: masks equal on every case; terms within 1e-10 relative (NaN exactly
    where the reference's is NaN) and gradient samples, of the total and of the case's weighted sum of every term,
    within 1e-10 of each scale's largest gradient (both runs sum in fp64 in different orders, over up to 2.5e5 pixels,
    and the SSIM variance cancels: measured up to 6e-11);
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

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIX = okl.load_fixture(GOLDEN)
CASES = [str(c) for c in FIX["cases"]]
F64_REL = 1e-10
F32_REL = 1e-3


def _run(name, mode, grads=True, grad_terms=None):
    case = okl.CASES[name]
    seed = int(FIX["%s/seed" % name])
    inp, disps = okl.make_inputs(case, seed)
    noise = okl.draw_noise(seed, inp, case["loss_scales"])
    return case, okl.run(inp, disps, noise, case["scales"], case["loss_scales"], mode=mode, grads=grads,
                         grad_terms=grad_terms, **okl.options(case))


def _close(got, want, rel):
    """within rel of want, or both NaN"""
    return (np.isnan(got) and np.isnan(want)) or abs(got - want) <= rel * abs(want)


def _scalars(name, tag):
    return dict(zip([str(k) for k in FIX["%s/scalar_keys" % name]], FIX["%s/%s/scalars" % (name, tag)]))


def _mask(name, tag, key, s, shape):
    bits = np.unpackbits(FIX["%s/%s/%s/%d" % (name, tag, key, s)])[:int(np.prod(shape))]
    return bits.reshape(shape).astype(np.float64)


def _grad_parity(name, o, key):
    for s in okl.CASES[name]["loss_scales"]:
        idx = FIX["%s/grad_idx/%d" % (name, s)]
        want = FIX["%s/f64/%s/%d" % (name, key, s)]
        got = o["grad"][s].reshape(-1)[idx]
        assert np.isfinite(want).all() and np.isfinite(got).all(), (key, s)
        scale = np.abs(want).max()
        assert np.abs(got - want).max() <= F64_REL * scale, (key, s, np.abs(got - want).max() / scale)


@pytest.mark.parametrize("name", CASES)
def test_fp64_oracle_matches_reference_float64(name):
    case, o = _run(name, "fp64")
    for k, v in _scalars(name, "f64").items():
        assert _close(float(o[k]), v, F64_REL), (k, float(o[k]), v)
    for s in case["loss_scales"]:
        for key in ("identity_selection", "depth_hint_pixels"):
            want = _mask(name, "f64", key, s, o[key][s].shape)
            assert np.array_equal(o[key][s], want), (key, s, int((o[key][s] != want).sum()))
    _grad_parity(name, o, "grad")


@pytest.mark.parametrize("name", CASES)
def test_fp64_oracle_weighted_terms_match_reference_float64(name):
    """the gradient of sum_k w_k terms[k], each term with its own weight (some negative): an adjoint that took one
    term's coefficient for another's, or dropped one, would miss the reference's"""
    case = okl.CASES[name]
    w = FIX["%s/weights" % name]
    assert np.array_equal(w, case["weights"]) and len(w) == len(okl.term_keys(case["loss_scales"]))
    assert len(set(np.abs(w[1:]))) == len(w) - 1 and (w < 0).any()
    _, o = _run(name, "fp64", grad_terms=w)
    _grad_parity(name, o, "wgrad")


@pytest.mark.parametrize("name", [c for c in CASES if okl.CASES[c].get("random", True)])
def test_contract_oracle_near_reference_float32(name):
    case, o = _run(name, "contract", grads=False)
    for k, v in _scalars(name, "f32").items():
        assert _close(float(o[k]), v, F32_REL), (k, float(o[k]), v)
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


@pytest.mark.parametrize("name", ["camera", "odd"])
def test_camera_cases_cover_their_geometry(name):
    """a different K per frame; stereo transforms whose P[1, 3], P[2, 3] and varying a[2] reach the projection, with
    every z > 0; warps off all four sides of the image; d iy / dD of the size of d ix / dD"""
    case = okl.CASES[name]
    inp, disps = okl.make_inputs(case, int(FIX["%s/seed" % name]))
    K, iK, T = (inp[k].astype(np.float64) for k in ("K", "inv_K", "stereo_T"))
    assert len({K[n].tobytes() for n in range(case["N"])}) == case["N"]
    assert np.abs(np.einsum("nij,njk->nik", K, iK) - np.eye(4)).max() < 1e-4
    P = np.einsum("nij,njk->nik", K, T)[:, :3]
    assert (np.abs(P[:, 1, 3]) > 0).all() and (np.abs(P[:, 2, 3]) > 0).all() and len(set(np.sign(P[:, 2, 3]))) == 2
    H, W = case["H"], case["W"]
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    ray = np.einsum("nij,jhw->nihw", iK[:, :3, :3], np.stack([xs, ys, np.ones_like(xs)]))
    a2 = np.einsum("nj,njhw->nhw", P[:, 2, :3], ray)
    assert a2.max() - a2.min() > 0.05
    hint = inp["depth_hint"][:, 0].astype(np.float64)
    for D in [hint] + [okl.depth_from_disp(okl.upsample(disps[s], H, W), 0.1, 100.0)[1] for s in case["loss_scales"]]:
        assert (D * a2 + P[:, 2, 3, None, None] > 0).all()
        ix, iy, dix, diy = okl.project(D, inp["K"], inp["inv_K"], inp["stereo_T"])
        assert (ix < -1).any() and (ix > W).any() and (iy < -1).any() and (iy > H).any()
        assert np.abs(diy).max() > 0.2 * np.abs(dix).max()


@pytest.mark.parametrize("name", ["thin_row", "thin_col"])
def test_thin_cases_nan_terms_and_finite_gradients(name):
    """scale 3 is one row or one column: its smoothness is a mean over no edges, so loss/3 and loss are NaN in the
    reference and the oracle, while the reference's gradients, of the total and of every term, stay finite"""
    case = okl.CASES[name]
    assert min(case["H"], case["W"]) >> 3 == 1
    ref = _scalars(name, "f64")
    assert np.isnan(ref["loss/3"]) and np.isnan(ref["loss"]) and np.isfinite(ref["reproj_loss/3"])
    _, o = _run(name, "contract")
    for k, v in ref.items():
        assert np.isnan(float(o[k])) == np.isnan(v), k
    for s in case["loss_scales"]:
        assert np.isfinite(o["grad"][s]).all(), s
        for key in ("grad", "wgrad"):
            assert np.isfinite(FIX["%s/f64/%s/%d" % (name, key, s)]).all(), (key, s)


def test_fixture_is_small():
    for name in okl.FIXTURES:
        assert os.path.getsize(os.path.join(GOLDEN, name)) < 1 << 20, name


def test_header_declares_the_kitti_entry_points():
    """include/wmd_loss_kitti.h declares exactly the symbols _lib.KITTI_LOSS_SIGNATURES binds, shares none with the other
    tables, lays out wmd_loss_kitti_desc as _lib.KittiLossDesc does, and libwmd.so exports them"""
    text = open(os.path.join(GOLDEN, os.pardir, os.pardir, "include", "wmd_loss_kitti.h")).read()
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
