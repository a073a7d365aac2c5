"""CPU: the numpy NYUv2-loss oracle (oracle/nyu_loss.py) reproduces the reference's training loss and its gradients
(tests/golden/nyu_loss.npz, written by oracle/pin_nyu_loss.py from the unmodified NYUv2/train.py main()), its samples
are torch's bilinear upsample, its gather adjoint is the adjoint, and the loss entry points of libwmd are declared,
bound and reject bad arguments without touching a GPU.

The reference's float64 run takes the interpolation weights in fp64 (torch's rule for a float64 tensor), where the
contract keeps torch's fp32 lambda.  The oracle restates both: with fp64 weights its terms are within one float32 ulp
of the float64 run and its gradients within 2 ulp of each element; with the contract's weights its terms are within
1e-6 of the reference's own float32 run."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nyu_loss as onl
from wavelet_monodepth_b200 import _lib

from helpers import GOLDEN, load_golden

TERMS = ["loss_depth/%d" % s for s in onl.SCALES] + ["loss_LL3"]


def ulps(got, want):
    """|got - want| in float32 ulps of want"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def case(name, meta):
    n, H, W, disparity, use_wavelets, supervise_ll, kind = onl.CASES[name]
    depth, preds, ll = onl.case_inputs(name, meta["seeds"][name])
    t64 = 10.0 / depth[:, 0].astype(np.float64) if disparity else depth[:, 0].astype(np.float64)
    return depth, {s: p[:, 0] for s, p in preds.items()}, (None if ll is None else ll[:, 0]), t64, supervise_ll


def reference(fx, meta, name, tag):
    return dict(zip(meta["scalar_keys"][name], fx["%s__%s_scalars" % (name, tag)]))


@pytest.mark.parametrize("name", list(onl.CASES))
def test_oracle_terms_match_the_reference(name):
    fx, meta = load_golden("nyu_loss")
    depth, preds, ll, t64, sll = case(name, meta)
    yl = fx[name + "__yl_gt_f64"][:, 0] if ll is not None else None
    ref64, ref32 = reference(fx, meta, name, "f64"), reference(fx, meta, name, "f32")
    got64 = onl.losses(preds, t64, ll, yl, supervise_ll=sll, weights="fp64")
    got = onl.losses(preds, t64, ll, yl, supervise_ll=sll)
    assert sorted(got) == sorted(ref64), (sorted(got), sorted(ref64))
    for k in ref64:
        assert np.isnan(got64[k]) == np.isnan(ref64[k]) == np.isnan(got[k]) == np.isnan(ref32[k]), k
        if np.isnan(ref64[k]):
            continue
        if k in TERMS:
            assert ulps(got64[k], ref64[k]) <= 1.0, (k, got64[k], ref64[k])
        else:                      # 0.1 * l and the float32 sum, which the float64 run rounds differently
            assert abs(got64[k] - ref64[k]) <= 1e-6 * abs(ref64[k]), (k, got64[k], ref64[k])
        assert abs(got[k] - ref32[k]) <= 1e-6 * abs(ref32[k]), (k, got[k], ref32[k])


def tie_footprint(sg, pred_shape):
    """low-resolution pixels whose footprint holds a target pixel with sign 0 (a designed tie)"""
    a = onl.adjoint((sg == 0).astype(np.float64), *pred_shape)
    return a != 0


@pytest.mark.parametrize("name", list(onl.CASES))
def test_oracle_gradients_match_the_fp64_reference(name):
    """Within 2 float32 ulp of each element (with a floor of 2^-40 of the per-sign coefficient, for elements that
    cancel to ~1e-21), except at the designed ties of the "ties" case: there the float64 run samples the constant
    c as l0 c + l1 c with its own rounded 1 - l1, so its sample is c plus or minus an ulp and its sign is not 0.  Those
    elements are listed and each lies in a footprint of a tie."""
    fx, meta = load_golden("nyu_loss")
    depth, preds, ll, t64, _ = case(name, meta)
    items = [("disp_%d" % s, preds[s], t64, 0.1) for s in onl.SCALES]
    if name + "__grad_LL_idx" in fx:
        items.append(("LL", ll, fx[name + "__yl_gt_f64"][:, 0], 1.0 / 16))
    for key, pred, target, g in items:
        idx, want = fx["%s__grad_%s_idx" % (name, key)], fx["%s__grad_%s_f64" % (name, key)]
        got = onl.grad(pred, target, g, weights="fp64").reshape(-1)[idx]
        floor = g / target.size * 2.0 ** -40
        bad = (np.abs(got - want) > 2 * np.spacing(np.abs(want).astype(np.float32))) & (np.abs(got - want) > floor)
        if name == "ties":
            sg = onl.signs(onl.upsample(pred, *target.shape[1:], weights="fp64"), target)
            at_tie = tie_footprint(sg, pred.shape[1:]).reshape(-1)[idx]
            print("%s: %d of %d sampled elements differ, all in a tie's footprint" % (key, bad.sum(), bad.size))
            assert not (bad & ~at_tie).any(), key
        else:
            assert not bad.any(), (key, got[bad][:4], want[bad][:4])
        assert np.array_equal(np.isnan(got), np.isnan(want)), key


def test_ties_and_nan_cases_cover_their_cases():
    fx, meta = load_golden("nyu_loss")
    _, preds, _, t64, _ = case("ties", meta)
    for s in onl.SCALES:
        sg = onl.signs(onl.upsample(preds[s], *t64.shape[1:]), t64)
        assert (sg == 0).mean() == 0.5                          # the contract keeps every designed tie a tie
    ref = reference(fx, meta, "nan", "f64")
    assert np.isnan(ref["loss_depth/1"]) and np.isnan(ref["loss_LL3"]) and not np.isnan(ref["loss_depth/2"])
    _, preds, ll, _, _ = case("thin", meta)
    assert preds[3].shape[2] == 1


def test_contract_keeps_constants_exact():
    """l0 = 1 - l1 in fp64: the map of a constant is the constant at every factor, and l0 + l1 == 1."""
    for h, w in ((30, 40), (28, 28), (3, 1), (1, 5), (2, 2)):
        for k in (1, 2, 3):
            up = onl.upsample(np.full((1, h, w), 0.1, np.float32), h << k, w << k)
            assert (up == np.float64(np.float32(0.1))).all(), (h, w, k)
            for n_in, n_out in ((h, h << k), (w, w << k)):
                _, _, l0, l1 = onl.axis_taps(n_in, n_out)
                assert (l0 + l1 == 1.0).all()
                assert (l1 * 2.0 ** 27 == np.round(l1 * 2.0 ** 27)).all()       # multiples of 2^-27


@pytest.mark.parametrize("factor", [2, 4, 8, 16])
def test_samples_match_torch_cpu_upsample(factor):
    """Within 3 float32 ulp of torch's CPU float32 F.interpolate on positive inputs."""
    rng = np.random.default_rng(factor)
    for h, w in ((30, 40), (14, 14), (7, 3), (1, 6)):
        x = rng.uniform(0.01, 10.0, (2, h, w)).astype(np.float32)
        want = F.interpolate(torch.from_numpy(x)[:, None], scale_factor=factor, mode="bilinear",
                             align_corners=True)[:, 0].numpy()
        got = onl.upsample(x, h * factor, w * factor)
        assert ulps(got.astype(np.float32), want).max() <= 3, (h, w, factor, ulps(got.astype(np.float32), want).max())


def test_adjoint_is_the_adjoint():
    """<A x, y> == <x, A^T y> in fp64, A the contract's upsample and A^T the gather adjoint."""
    rng = np.random.default_rng(3)
    for h, w, k in ((30, 40, 3), (7, 1, 2), (1, 5, 1), (5, 6, 0)):
        x = rng.standard_normal((2, h, w)).astype(np.float32)
        y = rng.integers(-1, 2, (2, h << k, w << k)).astype(np.int8)
        lhs = float((onl.upsample(x, h << k, w << k) * y).sum())
        rhs = float((x.astype(np.float64) * onl.adjoint(y, h, w)).sum())
        assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1.0), (h, w, k, lhs, rhs)


def test_gradient_is_the_signed_adjoint_of_torch_fp64_at_factor_one():
    rng = np.random.default_rng(4)
    p = rng.standard_normal((2, 5, 7)).astype(np.float32)
    t = rng.standard_normal((2, 5, 7)).astype(np.float32)
    pt = torch.from_numpy(p).double().requires_grad_(True)
    F.l1_loss(pt, torch.from_numpy(t).double()).backward()
    assert np.array_equal(onl.grad(p, t, 1.0), pt.grad.float().numpy())


# ------------------------------------------------------------------------------------------ the C ABI
def test_loss_header_and_binding_agree():
    """include/wmd_loss.h declares exactly the symbols _lib.LOSS_SIGNATURES binds, shares none with the other two
    tables, and libwmd.so exports them."""
    text = open(os.path.join(os.path.dirname(GOLDEN), os.pardir, "include", "wmd_loss.h")).read()
    declared = set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", text, flags=re.S)))
    assert declared == set(_lib.LOSS_SIGNATURES), declared ^ set(_lib.LOSS_SIGNATURES)
    assert not declared & set(_lib.SIGNATURES) and not declared & set(_lib.EVAL_SIGNATURES)
    assert ctypes.sizeof(_lib.LossTerm) == 24 and _lib.LossTerm.log2_factor.offset == 16
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name


def _terms(*specs):
    arr = (_lib.LossTerm * len(specs))()
    for d, (pred, h, w, k) in zip(arr, specs):
        d.pred, d.h, d.w, d.log2_factor = pred, h, w, k
    return arr


def test_loss_entry_points_validate_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.wmd_loss_nyu_ws_bytes(8, 240, 320, 4) == 300 * 4 * 8
    assert lib.wmd_loss_nyu_ws_bytes(1, 1, 2049, 1) == 2 * 8
    assert lib.wmd_loss_nyu_ws_bytes(0, 240, 320, 4) == 0
    assert lib.wmd_loss_nyu_ws_bytes(8, 240, 320, 5) == 0 and lib.wmd_loss_nyu_ws_bytes(-1, 240, 320, 1) == 0
    big = 1 << 30
    good = _terms((1, 30, 40, 3), (1, 240, 320, 0))
    ptrs = (ctypes.c_void_p * 2)(1, 1)
    f, b = lib.wmd_loss_nyu_fwd, lib.wmd_loss_nyu_bwd
    assert f(None, 2, 240, 320, good, 2, None, 1, big, 1, None) == -1                     # NULL target
    assert f(1, 2, 240, 320, good, 2, None, None, big, 1, None) == -1                     # NULL workspace
    assert f(1, 2, 240, 320, good, 2, None, 1, big, None, None) == -1                     # NULL means
    assert f(1, 2, 240, 320, None, 2, None, 1, big, 1, None) == -1                        # NULL terms
    assert f(1, 2, 240, 320, _terms((None, 30, 40, 3)), 1, None, 1, big, 1, None) == -1   # NULL pred
    assert f(1, 2, 240, 320, good, 2, None, 1, 8, 1, None) == -4                          # workspace too small
    assert f(1, 2, 240, 320, _terms((1, 30, 41, 3)), 1, None, 1, big, 1, None) == -2      # w << 3 != W
    assert f(1, 2, 240, 320, _terms((1, 60, 80, 3)), 1, None, 1, big, 1, None) == -2      # h << 3 != H
    assert f(1, 2, 240, 320, _terms((1, 15, 20, 4)), 1, None, 1, big, 1, None) == -2      # factor 16
    assert f(1, 2, 240, 320, _terms((1, 240, 320, -1)), 1, None, 1, big, 1, None) == -2   # negative factor
    assert f(1, 2, 240, 320, good, 0, None, 1, big, 1, None) == -2                        # no term
    assert f(1, 2, 240, 320, good, 5, None, 1, big, 1, None) == -2                        # too many terms
    assert f(1, -1, 240, 320, good, 2, None, 1, big, 1, None) == -2                       # negative N
    assert f(1, 2, 0, 320, _terms((1, 0, 320, 0)), 1, None, 1, big, 1, None) == -2        # empty frame
    assert b(None, 2, 240, 320, good, 2, 1, ptrs, None) == -1                             # NULL signs
    assert b(1, 2, 240, 320, good, 2, None, ptrs, None) == -1                             # NULL upstream gradient
    assert b(1, 2, 240, 320, good, 2, 1, None, None) == -1                                # NULL grads
    assert b(1, 2, 240, 320, good, 2, 1, (ctypes.c_void_p * 2)(1, None), None) == -1      # NULL grads[1]
    assert b(1, 2, 240, 320, _terms((1, 30, 41, 3)), 1, 1, ptrs, None) == -2              # inconsistent shape
    assert b(None, 0, 240, 320, _terms((None, 30, 40, 3)), 1, 1, (ctypes.c_void_p * 1)(None), None) == 0   # N = 0
