"""CPU: the numpy NYUv2-evaluation oracle reproduces the reference's results (tests/golden/nyu_eval.npz, written by
oracle/pin_nyu_eval.py from the unmodified NYUv2/utils.py), and the NYU evaluation entry points of libwmd reject bad
arguments without touching a GPU."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import nyu_eval as one
from wavelet_monodepth_b200 import _lib

from helpers import GOLDEN


def load_fixture():
    with np.load(os.path.join(GOLDEN, "nyu_eval.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def assert_rel(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern differs")
    f = ~np.isnan(want) & ~(np.isinf(want) & (got == want))
    err = np.abs(got[f] - want[f]) / np.maximum(np.abs(want[f]), 1e-300)
    assert err.size == 0 or err.max() <= tol, (what, float(err.max()))


def splits(meta):
    for s in meta["seeds"]:
        yield "s%d" % s, s, one.synthetic_split(s)
    yield "special", meta["special_seed"], one.synthetic_split(meta["special_seed"], special=True)


def configs(meta, split):
    for mode, (use_224, use_disparity) in meta["modes"].items():
        for h, w in [(224, 224)] if use_224 else meta["disp_sizes"]:
            yield mode, use_224, use_disparity, h, w, split["disp"][(h, w, use_disparity)]


def oracle_run(gt, disp, use_224, use_disparity):
    g = one.prepare_gt(gt, use_224) if not use_224 else torch.nn.functional.interpolate(
        torch.from_numpy(gt[:, 16:-16, 16:-16]).unsqueeze(1), (224, 224), mode="bilinear",
        align_corners=True)[:, 0].numpy()
    gl = torch.log10(torch.from_numpy(g)).numpy()            # the reference's float32 log10, on the CPU
    pred = one.predict(disp, use_224, use_disparity)
    return pred, g, one.frame_sums(pred, g, gl)


def all_configs():
    fx, meta = load_fixture()
    for name, seed, split in splits(meta):
        for mode, use_224, use_disparity, h, w, disp in configs(meta, split):
            yield fx, "%s_%s_%dx%d" % (name, mode, w, h), seed, split, use_224, use_disparity, disp


@pytest.mark.parametrize("split_name", ["s0", "s1", "special"])
def test_oracle_reproduces_the_fp64_reference(split_name):
    for fx, key, seed, split, use_224, use_disparity, disp in all_configs():
        if not key.startswith(split_name + "_"):
            continue
        pred, _, sums = oracle_run(split["gt"], disp, use_224, use_disparity)
        assert_rel(one.metrics(sums)[:3], fx[key + "__f64_pooled"][:3], 1e-12, key)
        assert_rel(one.frame_metrics(sums)[:, :3], fx[key + "__f64_frames"][:, :3], 1e-12, key)
        assert np.array_equal(sums[:, 3:6].astype(np.int64), fx[key + "__f64_counts"]), key
        assert (sums[:, 6] == fx[key + "__pixels"]).all()
        assert_rel(pred.reshape(-1)[fx[key + "__pred_idx"]], fx[key + "__pred_values"], 1e-12, key)
        if key + "__nan_map" in fx:
            want = np.unpackbits(fx[key + "__nan_map"])[:pred.size].astype(bool)
            assert np.array_equal(np.isnan(pred).reshape(-1), want), key


def test_oracle_is_within_1e_6_of_the_fp32_reference():
    """The reference's own float32 numbers: rel, rms and log_10 to 1e-6; an a_k count may differ only at pixels
    within 2^-20 of a threshold.  Frames with a non-finite or zero disparity are left out of the a_k rule: next to an
    Inf (or, under DepthNorm, a zero) the float32 and fp64 chains differ by more than rounding, e.g. NaN against 10
    where torch's float32 weight of the Inf tap is 0 and the fp64 one is not."""
    for fx, key, seed, split, use_224, use_disparity, disp in all_configs():
        pred, g, sums = oracle_run(split["gt"], disp, use_224, use_disparity)
        frames, want = one.frame_metrics(sums)[:, :3], fx[key + "__f32_frames"][:, :3]
        ok = ~np.isnan(frames).any(1)
        small = np.abs(want) < 1e-4                  # all-equal frames: metrics that are zero up to rounding
        assert np.all(np.abs(frames - want)[ok[:, None] & small] <= 1e-6), key
        assert_rel(np.where(small, 1.0, frames)[ok], np.where(small, 1.0, want)[ok], 1e-6, key)
        if ok.all():
            assert_rel(one.metrics(sums)[:3], fx[key + "__f32_pooled"][:3], 1e-6, key)
        for i in range(pred.shape[0]):
            if not np.isfinite(disp[i]).all() or (disp[i] == 0).any():
                continue
            diff = int(np.abs(sums[i, 3:6] - fx[key + "__f32_counts"][i]).sum())
            assert diff <= one.near_ties(pred[i], g[i], 2.0 ** -20), (key, i, diff)


def test_fixture_covers_the_special_frames():
    fx, meta = load_fixture()
    split = one.synthetic_split(meta["special_seed"], special=True)
    sp = split["special"]
    for key in [k[:-len("__f64_frames")] for k in fx if k.startswith("special_") and k.endswith("__f64_frames")]:
        frames = fx[key + "__f64_frames"]
        assert np.isnan(frames[sp["nan_disp"], :3]).all(), key    # NaN reaches the metrics of its own frame only
        assert np.isfinite(frames[sp["inf_disp"]]).all(), key     # Inf clamps to 10; under DepthNorm it is 0 -> 0.4
        for name in ("negative_disp", "all_equal"):
            assert np.isfinite(frames[sp[name]]).all(), (key, name)
        # zero disparity under DepthNorm is Inf; at 241 x 319 output column 101 reads it with weight 0: 0 * Inf = NaN
        assert np.isnan(frames[sp["zero_disp"], 0]) == (key == "special_eigen_disp_319x241"), key
        if "_224" not in key:                                     # a zero ground-truth pixel: rel and log_10 are Inf
            assert np.isinf(frames[sp["zero_gt"], 0]) and np.isinf(frames[sp["zero_gt"], 2]), key
            assert np.isfinite(frames[sp["zero_gt"], 1]), key
    assert fx["special_eigen_320x240__f64_frames"][sp["all_equal"], 3] == 1.0
    # zero disparity under DepthNorm is Inf, clamped to 10 inside the zero block
    for h, w in meta["disp_sizes"]:
        d = split["disp"][(h, w, True)][sp["zero_disp"]]
        pred = one.predict(d[None], False, True)[0]
        y, x = (3 * h // 8) * 480 // h - 20, (3 * w // 8) * 640 // w - 24
        assert pred[y, x] == 10.0, (h, w, pred[y, x])


def test_nan_spreads_through_zero_weight_taps():
    """At 241 x 319 the first resize samples column 106 exactly in output column 101 and reads column 107 with weight
    0; the reference's NaN map includes what that zero-weight read spreads."""
    fx, meta = load_fixture()
    split = one.synthetic_split(meta["special_seed"], special=True)
    i = split["special"]["nan_disp"]
    for use_disparity, mode in ((False, "eigen"), (True, "eigen_disp")):
        key = "special_%s_319x241" % mode
        d = split["disp"][(241, 319, use_disparity)]
        want = np.unpackbits(fx[key + "__nan_map"]).astype(bool)[:d.shape[0] * 440 * 592].reshape(-1, 440, 592)[i]
        read = np.isnan(one.predict(d[i:i + 1], False, use_disparity)[0])
        skipped = np.isnan(one.predict(d[i:i + 1], False, use_disparity, skip_zero_weight=True)[0])
        assert np.array_equal(read, want), key
        assert skipped.sum() < read.sum() and not (skipped & ~read).any(), (key, skipped.sum(), read.sum())


def test_gt224_oracle_matches_torch_cpu_samples():
    fx, meta = load_fixture()
    for name, seed, split in splits(meta):
        g = one.prepare_gt(split["gt"], use_224=True).reshape(-1)[fx[name + "__gt224_idx"]]
        want = fx[name + "__gt224_values"]
        ulps = np.abs(g.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert ulps.max() <= meta["gt224_oracle_vs_cpu_max_ulp"][name], (name, int(ulps.max()))


def test_compute_errors_nyu_oracle_equals_the_pooled_sums():
    split = one.synthetic_split(0)
    pred = one.predict(split["disp"][(240, 320, False)])
    y, x = one.prepare_gt(split["gt"]).astype(np.float64), pred
    t = np.maximum(y / x, x / y)
    want = [np.mean(np.abs(y - x) / y), np.sqrt(np.mean((y - x) ** 2)), np.mean(np.abs(np.log10(y) - np.log10(x)))]
    want += [np.mean(t < c) for c in one.THRESHOLDS]
    assert_rel(one.compute_errors_nyu(x, y), want, 1e-13, "compute_errors_nyu")


def test_nyu_eval_entry_points_validate_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.wmd_eval_nyu_ws_bytes(4, 0) == 4 * (224 * 304 + 55 * 7) * 8
    assert lib.wmd_eval_nyu_ws_bytes(4, 1) == 4 * 28 * 7 * 8
    assert lib.wmd_eval_nyu_ws_bytes(4, 2) == 0 and lib.wmd_eval_nyu_ws_bytes(-1, 0) == 0
    big = 1 << 30
    assert lib.wmd_eval_nyu_frames(None, 1, 240, 320, 0, 0, 1, 1, None, 1, big, 1, None) == -1       # NULL disp
    assert lib.wmd_eval_nyu_frames(1, 1, 240, 320, 0, 0, 1, 1, None, None, big, 1, None) == -1      # NULL ws
    assert lib.wmd_eval_nyu_frames(1, 1, 240, 320, 0, 0, 1, 1, None, 1, 16, 1, None) == -1          # ws too small
    assert lib.wmd_eval_nyu_frames(1, 1, 240, 320, 5, 0, 1, 1, None, 1, big, 1, None) == -1         # unknown mode
    assert lib.wmd_eval_nyu_frames(1, 1, 0, 320, 0, 0, 1, 1, None, 1, big, 1, None) == -2           # empty frame
    assert lib.wmd_eval_nyu_frames(1, 1, 240, 320, 1, 0, 1, 1, None, 1, big, 1, None) == -2         # 224 mode
    assert lib.wmd_eval_nyu_frames(1, 1 << 16, 240, 320, 0, 0, 1, 1, None, 1, big, 1, None) == -2   # too many frames
    assert lib.wmd_eval_nyu_frames(None, 0, 240, 320, 0, 0, None, None, None, None, 0, None, None) == 0  # nothing to do
    assert lib.wmd_eval_nyu_errors_ws_bytes(4096) == 2 * 7 * 8 and lib.wmd_eval_nyu_errors_ws_bytes(4097) == 3 * 7 * 8
    assert lib.wmd_eval_nyu_errors_f64(None, None, 4, 1, big, 1, None) == -1
    assert lib.wmd_eval_nyu_errors_f64(1, 1, 4, 1, 8, 1, None) == -1
    assert lib.wmd_eval_nyu_errors_f64(1, 1, -1, 1, big, 1, None) == -2
