"""CPU: the NYUv2 depth-boundary-error oracle (oracle/nyu_edges.py) against scipy, numpy and the reference's results
(tests/golden/nyu_edges.npz, written by oracle/pin_nyu_edges.py from the unmodified NYUv2/utils.py), and the edge
entry points' binding table against include/wmd_eval.h."""
import json
import os
import re

import numpy as np
import pytest
from scipy import ndimage as ndi

from oracle import nyu_edges as ne
from oracle import nyu_eval as one
from wavelet_monodepth_b200 import _lib

from helpers import GOLDEN

EDGE_SYMBOLS = ("wmd_eval_edges_ws_bytes", "wmd_eval_edges_frames", "wmd_eval_edt_ws_bytes", "wmd_eval_edt")


def load_fixture():
    with np.load(os.path.join(GOLDEN, "nyu_edges.npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def fixture_splits(meta):
    yield "s%d" % meta["seed"], ne.edge_split(meta["seed"])
    yield "special", ne.edge_split(meta["special_seed"], special=True)


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def maps(dtype):
    rng = np.random.default_rng(11)
    out = [rng.random(s).astype(dtype) for s in ((440, 592), (13, 7), (2, 5), (1, 1), (1, 9))]
    special = rng.random((40, 50)).astype(dtype)
    special[3, 4], special[20, 30], special[35, 2], special[10, 45] = np.nan, np.inf, -np.inf, np.nan
    return out + [special]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_filter_restatement_is_scipy_bit_for_bit(dtype):
    for x in maps(dtype):
        assert bits_equal(ne.gaussian_restated(x), ndi.gaussian_filter(x, ne.SIGMA, mode="constant")), x.shape
        s = x.astype(np.float64)
        for axis in (0, 1):
            assert bits_equal(ne.sobel_restated(s, axis), ndi.sobel(s, axis)), (x.shape, axis)
    assert bits_equal(ne.gaussian_restated(np.ones((440, 592))), ne.canny_parts(np.zeros((440, 592), np.float32))
                      ["bleed"])


def test_glibc_hypot_kernel_is_np_hypot():
    rng = np.random.default_rng(5)
    n = 0
    for k in range(10):
        scale = np.array([8.0, 1.0, 1e-3, 1e-9])[rng.integers(0, 4, (2, 10 ** 6))]
        x, y = rng.normal(size=(2, 10 ** 6)) * scale
        assert bits_equal(ne.hypot_glibc(x, y), np.hypot(x, y)), k
        n += x.size
    assert n >= 10 ** 7
    odd = np.array([0.0, -0.0, 3.0, np.inf, -np.inf, np.nan, 1e-320, 1e300, 5e-300, 2.0 ** -520])
    x, y = np.meshgrid(odd, odd)
    assert np.array_equal(ne.hypot_glibc(x, y), np.hypot(x, y), equal_nan=True)


def test_edt_of_a_map_without_features():
    for shape in ((3, 4), (7, 2), (440, 592)):
        assert bits_equal(ne.edt(np.zeros(shape, bool)), ne.no_feature_edt(*shape)), shape


def test_oracle_reproduces_the_reference_fixture():
    fx, meta = load_fixture()
    assert meta["edge_free_reference"].startswith("UnboundLocalError")
    for name, split in fixture_splits(meta):
        keep = meta["frames"][name]
        pred = one.predict(split["disp"][keep]).astype(np.float32)
        ours = [ne.dbe_numpy(split["edges"][i][20:460, 24:616], pred[j]) for j, i in enumerate(keep)]
        scores = np.array([o[:2] for o in ours])
        edges = np.stack([o[2] for o in ours])
        assert np.array_equal(np.packbits(edges.reshape(-1)), fx[name + "__f64_edges"]), name
        assert np.array_equal(scores, fx[name + "__f64_scores"], equal_nan=True), name
        assert np.array_equal(scores.mean(0), fx[name + "__f64_e_edges"], equal_nan=True), name
        fs = np.array([ne.dbe(split["edges"][i][20:460, 24:616], pred[j])[:2] for j, i in enumerate(keep)])
        assert np.allclose(fs, scores, rtol=1e-12, atol=0), name


def test_special_frames_cover_their_cases():
    fx, meta = load_fixture()
    split = ne.edge_split(meta["special_seed"], special=True)
    sp = split["special"]
    keep = meta["frames"]["special"]
    scores = fx["special__f64_scores"]
    edges = np.unpackbits(fx["special__f64_edges"])[:len(keep) * 440 * 592].reshape(len(keep), 440, 592)
    row = {i: j for j, i in enumerate(keep)}
    e = split["edges"]
    assert ((e[sp["grey"]] > 0) & (e[sp["grey"]] < 1)).any() and (e[sp["grey"]] == 1).any()
    assert (e[sp["grey_only"]] > 0).any() and not (e[sp["grey_only"]] == 1).any()
    assert not e[sp["edge_free"]].any() and sp["edge_free"] not in row
    assert np.array_equal(scores[row[sp["constant"]]], [10.0, 10.0]) and not edges[row[sp["constant"]]].any()
    assert np.isnan(split["disp"][sp["nan_disp"]]).any() and np.isfinite(scores[row[sp["nan_disp"]]]).all()
    spiral = edges[row[sp["spiral"]]]
    labels, count = ndi.label(spiral, np.ones((3, 3), bool))
    assert np.bincount(labels.ravel())[1:].max() > 20000
    # the edge-free frame scores NaN in the contract, and one such frame makes the split's mean NaN
    acc, comp, _, _ = ne.dbe(e[sp["edge_free"]][20:460, 24:616],
                             one.predict(split["disp"][sp["edge_free"]][None])[0].astype(np.float32))
    assert np.isnan(acc) and np.isnan(comp)


def test_edge_entry_points_are_declared_and_bound():
    text = open(os.path.join(os.path.dirname(GOLDEN), os.pardir, "include", "wmd_eval.h")).read()
    declared = set(re.findall(r"\b(wmd_\w+)\(", text))
    for name in EDGE_SYMBOLS:
        assert name in declared and name in _lib.EVAL_SIGNATURES, name
