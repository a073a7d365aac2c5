"""KITTI evaluation cost on one GPU, with CUDA events after warm-up.

    python scripts/eval_bench.py [--frames 697] [--steps 5] [--warmup 2] [--oracle-frames 8]

Builds a synthetic Eigen-like split (``--frames`` ground truths at the four KITTI sizes, ~5 % LiDAR-like density) and
reports, per 697-frame split:
  (a) the evaluator alone (KittiDepthEvaluator.add over the whole split, in 16-frame batches) at 640x192 and 1024x320;
  (b) one threshold-sweep point: R18 640x192 SparseDepthWaveProgressiveDecoder (threshold 0.05, batches of 16 on
      synthetic features), then disp_to_depth, then the evaluator;
  (c) for context, the numpy oracle's per-frame loop on the host (timed on --oracle-frames frames, scaled to the split).
Every figure is milliseconds per split.
The card and its power limit are read in the same run and printed beside the numbers, as one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import kitti_eval as oke  # noqa: E402
from wavelet_monodepth_b200 import kitti_decoders as kd, synth  # noqa: E402
from wavelet_monodepth_b200.kitti_eval import KittiDepthEvaluator  # noqa: E402

BATCH = 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def split(frames, seed=0):
    rng = np.random.default_rng(seed)
    gt = []
    for i in range(frames):
        H, W = oke.GT_SIZES[i % len(oke.GT_SIZES)]
        g = np.where(rng.random((H, W)) < 0.05, rng.uniform(1.0, 90.0, (H, W)), 0.0).astype(np.float32)
        gt.append(g)
    return gt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=697)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-frames", type=int, default=8)
    a = ap.parse_args()
    gt = split(a.frames)
    ev = KittiDepthEvaluator(gt)
    res = {"card": card(), "frames": a.frames, "valid_pixels_per_frame": int(ev.offsets[-1]) / a.frames}
    g = torch.Generator(device="cuda").manual_seed(0)

    def sweep(disp):
        ev.reset()
        for i in range(0, a.frames, BATCH):
            ev.add(disp[i:i + BATCH])
    for h, w in oke.DISP_SIZES:
        disp = torch.rand((a.frames, 1, h, w), device="cuda", generator=g) * 0.3 + 0.01
        res["evaluator_ms_%dx%d" % (w, h)] = timed(lambda: sweep(disp), a.steps, a.warmup)

    ch = synth.RESNET18_CH
    hp = ["decoder.%d.2.conv." % k for k in (3, 4, 7, 8, 11, 12, 15, 16)]
    dec = kd.SparseDepthWaveProgressiveDecoder(np.array(ch))
    synth.load_random(dec, seed=3, gains={k: 4.0 for k in hp}, highpass=hp)
    dec = dec.cuda().eval()
    dec.count_ops = "async"
    feats = [f.cuda() for f in synth.blocky_features(synth.kitti_feature_shapes(BATCH, 192, 640, ch), seed=9, cell=4,
                                                       texture=0.01)]
    min_disp, max_disp = 1 / 100.0, 1 / 0.1

    def decode_only():
        with torch.no_grad():
            for _ in range(0, a.frames, BATCH):
                dec(feats, 0.05)

    def point():
        ev.reset()
        with torch.no_grad():
            for i in range(0, a.frames, BATCH):
                out = dec(feats, 0.05)
                n = min(BATCH, a.frames - i)
                ev.add((min_disp + (max_disp - min_disp) * out[("disp", 0)])[:n])
    res["decoder_only_ms"] = timed(decode_only, a.steps, a.warmup)
    res["sweep_point_ms"] = timed(point, a.steps, a.warmup)

    disp = np.random.default_rng(1).uniform(0.01, 0.3, (a.oracle_frames, 192, 640))
    t0 = time.perf_counter()
    for i in range(a.oracle_frames):
        oke.evaluate_frame(gt[i], disp[i])
    res["numpy_oracle_ms"] = (time.perf_counter() - t0) * 1e3 / a.oracle_frames * a.frames
    print(json.dumps(res))


if __name__ == "__main__":
    main()
