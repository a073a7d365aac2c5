"""Pin oracle.nyu_edges against the UNMODIFIED reference depth boundary error and write tests/golden/nyu_edges.npz.

Runs only where the reference checkout exists, like the other pin scripts.  It imports NYUv2/utils.py with the stubs
oracle/pin_nyu_eval.py uses, binds ``skimage.feature.canny`` to ``oracle.nyu_edges.canny`` (scikit-image 0.16.2's canny
restated over scipy, the way oracle.haar stands in for pytorch_wavelets) and restores numpy's removed ``np.float``
alias, which evaluate() still names.  Then, for the plain split (seed SEED) and the special split (SPECIAL_SEED, every
EDGE_SPECIAL case but "edge_free"), it runs ``utils.evaluate(..., edges=...)`` in Eigen mode with a stub model, once
with float32 disparities (the reference's own numbers) and once with float64 ones (whose ``pred.astype('f')`` is the
fp64 map rounded to float32, the device's input).  ``utils.compute_depth_boundary_error`` is wrapped to capture each
frame's prediction, edges and scores.

Checks: the float64 run's predictions are oracle.nyu_eval.predict's map; the oracle's edges equal the reference's bit
for bit and its scores (numpy sums) equal them exactly, e_edges too.  An all-zero ground-truth edge map makes the
reference raise UnboundLocalError (it returns a D_est it never computed); that is recorded, and the contract scores
such a frame NaN, NaN.

The fixture holds per-frame scores, e_edges and the packed Canny edges of both runs, and the number of edge pixels the
float32 chain flips against the float64 one; tests regenerate the inputs from the seeds.

Usage:  python -m oracle.pin_nyu_edges
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import nyu_edges as ne                                          # noqa: E402
from oracle import nyu_eval as one                                          # noqa: E402
from oracle import pin_nyu_eval as pne                                      # noqa: E402

GOLDEN = os.path.join(REPO, "tests", "golden")
SEED = 0
SPECIAL_SEED = 7


def import_utils():
    utils = pne.import_utils()
    sys.modules["skimage.feature"].canny = ne.canny
    if not hasattr(np, "float"):
        np.float = float                   # the alias numpy 1.19 still had; evaluate() allocates edges_scores with it
    return utils


def eval_frames(split):
    """the frames evaluate() can score: all but an all-zero edge map"""
    sp = split.get("special", {})
    return [i for i in range(split["gt"].shape[0]) if i != sp.get("edge_free", -1)]


def run_reference(utils, split, dtype):
    """utils.evaluate(..., edges=...) on the CPU -> (e_edges (2,), scores (n, 2), edges (n, 440, 592), preds)"""
    keep = eval_frames(split)
    gt, disp, edges = split["gt"][keep], split["disp"][keep], split["edges"][keep]
    n = gt.shape[0]
    captured = []
    plain = utils.compute_depth_boundary_error

    def capture(edges_gt, pred, *a, **k):
        r = plain(edges_gt, pred, *a, **k)
        captured.append((pred.copy(), r[0], r[1], np.asarray(r[2], bool)))
        return r
    utils.compute_depth_boundary_error = capture
    model = pne.StubModel(torch.from_numpy(disp).to(dtype))
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            _, e_edges = utils.evaluate(model, np.zeros((n, 480, 640, 3), np.uint8), gt, list(one.EIGEN_CROP),
                                        edges=edges)
    finally:
        utils.compute_depth_boundary_error = plain
    assert model.i == n and len(captured) == n
    preds = np.stack([c[0] for c in captured])
    scores = np.array([[c[1], c[2]] for c in captured], np.float64)
    return np.asarray(e_edges, np.float64), scores, np.stack([c[3] for c in captured]), preds


def main():
    utils = import_utils()
    torch.Tensor.cuda = lambda self, *a, **k: self
    arrays = {}
    meta = dict(seed=SEED, special_seed=SPECIAL_SEED, special=list(ne.EDGE_SPECIAL), flips_f32_vs_f64={})
    # the reference on an edge-free ground truth
    split = ne.edge_split(SPECIAL_SEED, special=True)
    k = split["special"]["edge_free"]
    pred = one.predict(split["disp"][k:k + 1])[0].astype(np.float32)
    try:
        utils.compute_depth_boundary_error(split["edges"][k][20:460, 24:616], pred)
        meta["edge_free_reference"] = "returned"
    except UnboundLocalError as exc:
        meta["edge_free_reference"] = "UnboundLocalError: %s" % exc
    print("edge-free ground truth, reference:", meta["edge_free_reference"])
    for name, split in (("s%d" % SEED, ne.edge_split(SEED)), ("special", ne.edge_split(SPECIAL_SEED, special=True))):
        keep = eval_frames(split)
        runs = {tag: run_reference(utils, split, dtype) for tag, dtype in (("f32", torch.float32),
                                                                            ("f64", torch.float64))}
        e64, s64, edges64, preds64 = runs["f64"]
        want_map = one.predict(split["disp"][keep])
        d = np.abs(preds64 - want_map)[np.isfinite(want_map)] / want_map[np.isfinite(want_map)]
        same32 = np.array_equal(preds64.astype(np.float32), want_map.astype(np.float32), equal_nan=True)
        print("%s: float64 run vs oracle map: max rel %.1e, equal after rounding to float32: %s" % (name, d.max(), same32))
        assert np.array_equal(np.isnan(preds64), np.isnan(want_map)) and d.max() <= 1e-12 and same32, name
        ours = [ne.dbe_numpy(split["edges"][i][20:460, 24:616], want_map[j].astype(np.float32))
                for j, i in enumerate(keep)]
        o_scores = np.array([o[:2] for o in ours])
        o_edges = np.stack([o[2] for o in ours])
        assert np.array_equal(o_edges, edges64), name
        assert np.array_equal(o_scores, s64, equal_nan=True), (name, o_scores, s64)
        assert np.array_equal(o_scores.mean(0), e64, equal_nan=True), name
        fs = np.array([ne.dbe(split["edges"][i][20:460, 24:616], want_map[j].astype(np.float32))[:2]
                       for j, i in enumerate(keep)])
        with np.errstate(invalid="ignore"):
            rel = np.nanmax(np.abs(fs - s64) / np.abs(s64))
        flips = int((runs["f32"][2] != edges64).sum())
        meta["flips_f32_vs_f64"][name] = flips
        print("%s: e_edges f64 %s f32 %s | oracle numpy sums exact, fsum %.1e rel | edge pixels %d, flipped by the "
              "float32 chain %d" % (name, e64, runs["f32"][0], rel, int(edges64.sum()), flips))
        assert rel <= 1e-12
        meta.setdefault("frames", {})[name] = keep
        for tag, (e, s, edges, _) in runs.items():
            arrays["%s__%s_e_edges" % (name, tag)] = e
            arrays["%s__%s_scores" % (name, tag)] = s
            arrays["%s__%s_edges" % (name, tag)] = np.packbits(edges.reshape(-1))
    path = os.path.join(GOLDEN, "nyu_edges.npz")
    np.savez_compressed(path, __meta__=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
