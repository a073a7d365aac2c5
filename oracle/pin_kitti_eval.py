"""Pin oracle.kitti_eval against the UNMODIFIED reference evaluation and write tests/golden/kitti_eval.npz.

Runs only where the reference checkout exists, like the other pin scripts.  For each synthetic split (seeds SEEDS) and
each disparity size it runs the reference's ``evaluate(opt)`` (KITTI/evaluate_depth.py:82-323) on its
``ext_disp_to_eval`` path in the four modes of ``oracle.kitti_eval.MODES``:
  * stub modules stand in for ``datasets`` and ``networks`` (that path never uses them);
  * ``evaluate_depth.splits_dir`` points at a temporary directory holding the synthetic ``gt_depths.npz`` (an object
    array: the frame sizes are mixed);
  * the disparities are saved as a float64 .npy, the dtype ``pred_disps`` has on the model path (:134), so cv2.resize
    runs in fp64 as it does there;
  * ``compute_errors`` is wrapped to record each frame's inputs and outputs;
  * the UnboundLocalError evaluate() raises at :320 (``sparse_decoding`` is unset on this path) is caught: every frame
    has been scored by then.
The recorded per-frame metrics must match ``oracle.kitti_eval.evaluate`` to 1e-12 relative (NaN where the reference is
NaN), the valid counts exactly; the oracle's fp64 resize must match cv2.resize to 1e-11 relative.  It then calls the
reference's ``batch_post_process_disparity`` directly on ``post_process_inputs`` and stores samples of its output.

The fixture holds only seeds, per-frame metrics, ratios, counts and post-processing samples; tests regenerate the
inputs from the seeds.

Usage:  python -m oracle.pin_kitti_eval
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types
import warnings

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_eval as oke                                        # noqa: E402

REF_KITTI = "/root/reference/KITTI"
GOLDEN = os.path.join(REPO, "tests", "golden")
SEEDS = (0, 1)
POST_SEED = 7
POST_SAMPLES = 4096


def import_evaluate_depth():
    for name in ("datasets", "networks", "networks.network_constructors"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["networks"].network_constructors = sys.modules["networks.network_constructors"]
    sys.modules["networks.network_constructors"].__all__ = []
    if REF_KITTI not in sys.path:
        sys.path.insert(0, REF_KITTI)
    import evaluate_depth
    return evaluate_depth


def run_reference(ed, workdir, gt, disp, mode):
    split, median_scaling, _ = oke.MODES[mode]
    os.makedirs(os.path.join(workdir, split), exist_ok=True)
    data = np.empty(len(gt), dtype=object)
    for i, g in enumerate(gt):
        data[i] = g
    np.savez(os.path.join(workdir, split, "gt_depths.npz"), data=data)
    disp_path = os.path.join(workdir, "disps.npy")
    np.save(disp_path, disp.astype(np.float64))
    ed.splits_dir = workdir
    opt = types.SimpleNamespace(eval_mono=median_scaling, eval_stereo=not median_scaling, ext_disp_to_eval=disp_path,
                                eval_eigen_to_benchmark=False, save_pred_disps=False, no_eval=False, eval_split=split,
                                disable_median_scaling=False, pred_depth_scale_factor=1)
    recorded = []
    plain = ed.compute_errors

    def recording(gt_depth, pred_depth):
        out = plain(gt_depth, pred_depth)
        recorded.append((gt_depth.copy(), pred_depth.copy(), np.array(out, dtype=np.float64)))
        return out
    ed.compute_errors = recording
    try:
        with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ed.evaluate(opt)
    except UnboundLocalError:
        pass
    finally:
        ed.compute_errors = plain
    assert len(recorded) == len(gt), (mode, len(recorded))
    return recorded


def rel_close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    f = ~np.isnan(a)
    return bool(np.all(np.abs(a[f] - b[f]) <= tol * np.maximum(np.abs(b[f]), 1e-300)))


def check_resize(split):
    try:
        import cv2
    except ImportError:
        print("cv2 not importable: resize check skipped")
        return
    worst = 0.0
    for (h, w), d in split["disp"].items():
        for i, g in enumerate(split["gt"]):
            if i in (split["special"]["nan_disp"],):
                continue
            ref = cv2.resize(d[i].astype(np.float64), (g.shape[1], g.shape[0]))
            got = oke.resize_linear(d[i], *g.shape)
            f = ref != 0
            worst = max(worst, float(np.max(np.abs(got[f] / ref[f] - 1))))
            assert np.array_equal(got == 0, ref == 0)
    print("oracle resize vs cv2.resize: max rel %.3g" % worst)
    assert worst <= 1e-11


def main():
    ed = import_evaluate_depth()
    arrays, meta = {}, dict(seeds=list(SEEDS), modes=oke.MODES, disp_sizes=oke.DISP_SIZES, post_seed=POST_SEED)
    with tempfile.TemporaryDirectory() as workdir:
        for seed in SEEDS:
            split = oke.synthetic_split(seed)
            check_resize(split)
            for (h, w), disp in split["disp"].items():
                for mode in oke.MODES:
                    rec = run_reference(ed, workdir, split["gt"], disp, mode)
                    ref_err = np.stack([r[2] for r in rec])
                    ref_cnt = np.array([r[0].size for r in rec], np.int64)
                    ours, ratios, counts = oke.evaluate(split["gt"], disp, mode)
                    assert np.array_equal(counts, ref_cnt), (seed, h, mode)
                    assert rel_close(ours, ref_err, 1e-12), (seed, h, mode, np.nanmax(np.abs(ours / ref_err - 1)))
                    key = "s%d_%dx%d_%s" % (seed, w, h, mode)
                    arrays[key + "__errors"] = ref_err
                    arrays[key + "__ratios"] = ratios
                    arrays[key + "__counts"] = ref_cnt
                    print("%s: %d frames, abs_rel mean %.4f" % (key, len(rec), np.nanmean(ref_err[:, 0])))
    l_disp, r_disp = oke.post_process_inputs(POST_SEED)
    pp = ed.batch_post_process_disparity(l_disp, r_disp[:, :, ::-1])
    assert pp.dtype == np.float64
    idx = np.random.default_rng(POST_SEED).choice(pp.size, POST_SAMPLES, replace=False)
    idx = np.concatenate([idx, np.arange(pp.shape[2]), pp.size - 1 - np.arange(pp.shape[2])])     # first, last rows
    arrays["post__idx"] = idx.astype(np.int64)
    arrays["post__values"] = pp.reshape(-1)[idx]
    path = os.path.join(GOLDEN, "kitti_eval.npz")
    np.savez_compressed(path, __meta__=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", path)


if __name__ == "__main__":
    main()
