"""CPU: the numpy KITTI-evaluation oracle reproduces the reference's per-frame results (tests/golden/kitti_eval.npz), and
the evaluation entry points of libwmd reject bad arguments without touching a GPU."""
import json
import os
import re

import numpy as np
import pytest

from oracle import kitti_eval as oke
from wavelet_monodepth_b200 import _lib

from helpers import GOLDEN


def load_fixture():
    with np.load(os.path.join(GOLDEN, "kitti_eval.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def assert_rel(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN pattern differs")
    f = ~np.isnan(want)
    err = np.abs(got[f] - want[f]) / np.maximum(np.abs(want[f]), 1e-300)
    assert err.size == 0 or err.max() <= tol, (what, float(err.max()))


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_reproduces_reference_per_frame(seed):
    fx, meta = load_fixture()
    split = oke.synthetic_split(seed)
    for h, w in meta["disp_sizes"]:
        for mode in meta["modes"]:
            key = "s%d_%dx%d_%s" % (seed, w, h, mode)
            errors, ratios, counts = oke.evaluate(split["gt"], split["disp"][(h, w)], mode)
            assert np.array_equal(counts, fx[key + "__counts"]), key
            assert_rel(errors, fx[key + "__errors"], 1e-12, key)
            assert_rel(ratios, fx[key + "__ratios"], 1e-12, key)


def test_fixture_covers_the_special_frames():
    fx, _ = load_fixture()
    sp = oke.synthetic_split(0)["special"]
    mono = fx["s0_640x192_mono_eigen__errors"]
    counts = fx["s0_640x192_mono_eigen__counts"]
    assert counts[sp["empty"]] == 0 and np.isnan(mono[sp["empty"]]).all()
    assert counts[sp["one_valid"]] == 1 and counts[sp["even_count"]] % 2 == 0 and counts[sp["even_count"]] > 0
    assert np.isnan(mono[sp["nan_disp"], :4]).all() and (mono[sp["nan_disp"], 4:] == 0).all()
    assert not np.isnan(mono[:sp["empty"]]).any()                # regular frames are finite
    stereo = fx["s0_640x192_stereo_eigen__errors"]
    assert np.isfinite(stereo[sp["negative_disp"]]).all()        # negative depth is clamped to MIN_DEPTH


def test_post_process_oracle_matches_reference_samples():
    fx, meta = load_fixture()
    l_disp, r_disp = oke.post_process_inputs(meta["post_seed"])
    got = oke.batch_post_process_disparity(l_disp, r_disp[:, :, ::-1]).reshape(-1)[fx["post__idx"]]
    assert np.array_equal(got, fx["post__values"])


def test_eval_header_and_binding_agree():
    """include/wmd_eval.h declares exactly the symbols _lib.EVAL_SIGNATURES binds, and libwmd.so exports them."""
    text = open(os.path.join(os.path.dirname(GOLDEN), os.pardir, "include", "wmd_eval.h")).read()
    declared = set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", text, flags=re.S)))
    assert declared == set(_lib.EVAL_SIGNATURES), declared ^ set(_lib.EVAL_SIGNATURES)
    assert not declared & set(_lib.SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name


def test_eval_entry_points_validate_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.wmd_eval_gt_mask(None, None, None, 1, 4, 4, 0, None) == -1
    assert lib.wmd_eval_gt_mask(1, 1, 1, 1, 4, 4, 7, None) == -1                  # unknown split
    assert lib.wmd_eval_gt_mask(1, 1, 1, 1, 0, 4, 0, None) == -2
    assert lib.wmd_eval_gather_f32(None, 1, 1, 4, 1, None) == -1
    assert lib.wmd_eval_frames(None, 0, 1, 4, 4, 0, 1, 1, 1, 1, None, 8, 8, 1.0, 1, 1, 1, 1, 1, None) == -1
    assert lib.wmd_eval_frames(1, 0, 1, 0, 4, 0, 1, 1, 1, 1, None, 8, 8, 1.0, 1, 1, 1, 1, 1, None) == -2
    assert lib.wmd_eval_frames(1, 0, 1, 4, 4, 0, 1, 1, 1, 1, None, 1 << 16, 1 << 16, 1.0, 1, 1, 1, 1, 1, None) == -2
    assert lib.wmd_eval_frames(None, 0, 0, 4, 4, 0, None, None, None, None, None, 8, 8, 1.0, 1, None, None, None, None,
                               None) == 0                                          # nothing to do
    assert lib.wmd_eval_errors_f64(None, None, 4, None, None) == -1
    assert lib.wmd_eval_errors_f64(1, 1, -1, 1, None) == -2
    assert lib.wmd_post_process_disparity(None, None, 0, None, 1, 4, 4, None) == -1
    assert lib.wmd_post_process_disparity(1, 1, 0, 1, 1, 0, 4, None) == -2
