"""Pin oracle.nyu_eval against the UNMODIFIED reference evaluation and write tests/golden/nyu_eval.npz.

Runs only where the reference checkout exists, like the other pin scripts.  For each synthetic split (seeds SEEDS, and
the special split SPECIAL_SEED) it runs the reference's ``utils.evaluate()`` (NYUv2/utils.py:275-372) on the CPU in the
four modes of ``oracle.nyu_eval.MODES`` and at every disparity size:
  * stub modules stand in for matplotlib, imageio and skimage (the evaluation path never calls them), and
    ``torch.Tensor.cuda`` returns the tensor itself;
  * the model is a stub that returns the split's next disparity frame as ``("disp", 0)``, a fresh copy each call (the
    reference divides it in place);
  * ``utils.compute_errors_nyu`` is wrapped to capture the concatenated predictions and ground truth; per-frame
    metrics come from the reference's own ``compute_errors_nyu`` on each frame's slice, and the exact a_k counts from
    its threshold expression on the captured tensors.
Each configuration runs twice: with float32 disparities (the reference's own numbers) and with float64 ones (the
contract's precision).  The oracle must match the float64 run to 1e-12 relative, with a_k counts exact and the same NaN
pattern; its float32 gt224 is compared with torch's CPU ``F.interpolate`` and the ulp count printed.

The fixture holds seeds, pooled and per-frame metrics and counts of both runs, sampled prediction values of the float64
run (``oracle.nyu_eval.sample_indices``), the NaN maps of the special split and samples of the CPU gt224; tests
regenerate the inputs from the seeds.

Usage:  python -m oracle.pin_nyu_eval
"""
import contextlib
import io
import json
import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import nyu_eval as one                                          # noqa: E402

REF_NYU = "/root/reference/NYUv2"
GOLDEN = os.path.join(REPO, "tests", "golden")
SEEDS = (0, 1)
SPECIAL_SEED = 5


def import_utils():
    for name in ("matplotlib", "matplotlib.cm", "imageio", "skimage", "skimage.feature"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
    sys.modules["imageio"].imsave = sys.modules["imageio"].imread = None
    sys.modules["skimage"].feature = sys.modules["skimage.feature"]
    if REF_NYU not in sys.path:
        sys.path.insert(0, REF_NYU)
    import utils
    return utils


class StubModel:
    """Returns frame i of `disp` as the decoder's ("disp", 0) on its i-th call."""

    def __init__(self, disp):
        self.disp, self.i = disp, 0

    def eval(self):
        return self

    def __call__(self, x, *args):
        d = self.disp[self.i:self.i + 1, None].clone()
        self.i += 1
        return {("disp", 0): d}


def run_reference(utils, gt, disp, use_224, use_disparity, dtype):
    """utils.evaluate() on the CPU -> (pooled (6,), per-frame (n, 6), per-frame counts (n, 3), predictions, gt seen)"""
    n = gt.shape[0]
    captured = []
    plain = utils.compute_errors_nyu

    def capture(pred, g):
        captured.append((pred.clone(), g.clone()))
        return plain(pred, g)
    utils.compute_errors_nyu = capture
    rgb = np.zeros((n, 480, 640, 3), np.uint8)
    crop = list(one.EIGEN_CROP)
    model = StubModel(torch.from_numpy(disp).to(dtype))
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            e, _ = utils.evaluate(model, rgb, gt, crop, use_disparity=use_disparity, use_224=use_224)
    finally:
        utils.compute_errors_nyu = plain
    assert model.i == n and len(captured) == 1
    pred, g = captured[0]
    pred, g = pred.reshape(n, -1), g.reshape(n, -1)
    per_frame = np.array([[float(v) for v in plain(pred[i], g[i])] for i in range(n)], np.float64)
    counts = np.zeros((n, 3), np.int64)
    for i in range(n):
        y, x = g[i], pred[i]
        thresh = torch.max((y / x), (x / y))
        for k, c in enumerate(one.THRESHOLDS):
            counts[i, k] = int((thresh < c).sum())
    shape = (n, 224, 224) if use_224 else (n, 440, 592)
    return (np.array([float(v) for v in e], np.float64), per_frame, counts, pred.reshape(shape).numpy(),
            g.reshape(shape).numpy())


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), "NaN pattern differs"
    f = ~np.isnan(b) & ~(np.isinf(a) & (a == b))
    return float(np.max(np.abs(a[f] - b[f]) / np.maximum(np.abs(b[f]), 1e-300), initial=0.0))


def ulps_f32(a, b):
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


def configs(split):
    for mode, (use_224, use_disparity) in one.MODES.items():
        for (h, w) in ((224, 224),) if use_224 else one.DISP_SIZES:
            yield mode, use_224, use_disparity, h, w, split["disp"][(h, w, use_disparity)]


def main():
    utils = import_utils()
    torch.Tensor.cuda = lambda self, *a, **k: self
    arrays = {}
    meta = dict(seeds=list(SEEDS), special_seed=SPECIAL_SEED, modes=one.MODES, disp_sizes=one.DISP_SIZES,
                special=list(one.SPECIAL))
    splits = [("s%d" % s, s, one.synthetic_split(s)) for s in SEEDS]
    splits.append(("special", SPECIAL_SEED, one.synthetic_split(SPECIAL_SEED, special=True)))
    for name, seed, split in splits:
        gt = split["gt"]
        g224_cpu = torch.nn.functional.interpolate(torch.from_numpy(gt[:, 16:-16, 16:-16]).unsqueeze(1), (224, 224),
                                                   mode="bilinear", align_corners=True)[:, 0].numpy()
        g224_ours = one.prepare_gt(gt, use_224=True)
        u = ulps_f32(g224_ours, g224_cpu)
        print("%s gt224: oracle float32 vs torch CPU F.interpolate: max %d ulp, %d of %d values differ"
              % (name, u.max(), int((u > 0).sum()), u.size))
        assert u.max() <= 2
        meta.setdefault("gt224_oracle_vs_cpu_max_ulp", {})[name] = int(u.max())
        idx224 = one.sample_indices(seed, g224_cpu.shape)
        arrays["%s__gt224_idx" % name] = idx224
        arrays["%s__gt224_values" % name] = g224_cpu.reshape(-1)[idx224]
        for mode, use_224, use_disparity, h, w, disp in configs(split):
            key = "%s_%s_%dx%d" % (name, mode, w, h)
            g_seen = one.prepare_gt(gt, use_224)
            runs = {}
            for tag, dtype in (("f32", torch.float32), ("f64", torch.float64)):
                runs[tag] = run_reference(utils, gt, disp, use_224, use_disparity, dtype)
            pooled64, frame64, counts64, pred64, gseen64 = runs["f64"]
            # the reference's ground truth is the float32 crop, or its 224-pixel resize by torch's CPU kernel
            assert np.array_equal(gseen64.astype(np.float32), g_seen if not use_224 else g224_cpu), key
            gl = torch.log10(torch.from_numpy(gseen64.astype(np.float32))).numpy()
            ours_pred = one.predict(disp, use_224, use_disparity)
            sums = one.frame_sums(ours_pred, gseen64, gl)
            e_pred = rel_err(ours_pred, pred64)
            e_frame = rel_err(one.frame_metrics(sums)[:, :3], frame64[:, :3])
            e_pool = rel_err(one.metrics(sums)[:3], pooled64[:3])
            assert e_pred <= 1e-12 and e_frame <= 1e-12 and e_pool <= 1e-12, (key, e_pred, e_frame, e_pool)
            assert np.array_equal(sums[:, 3:6].astype(np.int64), counts64), key
            pooled32, frame32, counts32, pred32, _ = runs["f32"]
            d32 = rel_err(pooled32[:3], pooled64[:3]) if not np.isnan(pooled64[:3]).any() else float("nan")
            print("%s: rel %.6f rms %.6f log_10 %.6f a1 %.6f | oracle vs f64 run: map %.1e frames %.1e pooled %.1e | "
                  "f32 vs f64 run %.1e, a_k counts differ by %d" % (key, *pooled64[:4], e_pred, e_frame, e_pool, d32,
                                                                   int(np.abs(counts32 - counts64).sum())))
            for tag, (pooled, frame, counts, _, _) in runs.items():
                arrays["%s__%s_pooled" % (key, tag)] = pooled
                arrays["%s__%s_frames" % (key, tag)] = frame
                arrays["%s__%s_counts" % (key, tag)] = counts
            idx = one.sample_indices(seed, pred64.shape)
            arrays[key + "__pred_idx"] = idx
            arrays[key + "__pred_values"] = pred64.reshape(-1)[idx]
            arrays[key + "__pixels"] = np.int64(pred64[0].size)
            if name == "special":
                arrays[key + "__nan_map"] = np.packbits(np.isnan(pred64).reshape(-1))
    path = os.path.join(GOLDEN, "nyu_eval.npz")
    np.savez_compressed(path, __meta__=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
