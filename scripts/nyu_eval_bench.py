"""NYUv2 evaluation cost on one GPU, with CUDA events after warm-up.

    python scripts/nyu_eval_bench.py [--frames 654] [--steps 3] [--warmup 1]

Builds a synthetic 654-frame split (480 x 640 ground truth, as NYUv2's labelled test set) and reports, in milliseconds
per split, for Eigen mode (240 x 320 disparities) and 224 mode (224 x 224), in batches of 16:
  (a) the evaluator alone (NyuDepthEvaluator.add over the whole split, then summary());
  (b) the reference's chain restated in torch float32 on CUDA: per frame, as utils.evaluate() runs it (resize, pad,
      resize, clamp, crop, then compute_errors_nyu over the concatenated split), and batched 16 frames at a time;
  (c) one threshold-sweep point: DenseNet161 640 x 480 SparseDecoderWave at threshold 0.1 on synthetic features, then
      the evaluator (Eigen mode only; the decoder alone is reported beside it).
The card and its power limit are read in the same run and printed beside the numbers, as one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from wavelet_monodepth_b200 import nyu_decoders as nd, synth  # noqa: E402
from wavelet_monodepth_b200.nyu_eval import NyuDepthEvaluator  # noqa: E402

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


def torch_chain(pred, use_224):
    """utils.py:219-229 and the Eigen crop, in float32 on the device (pred (n, 1, h, w), already / 100)."""
    if not use_224:
        pred = F.interpolate(pred, (224, 304), mode="bilinear", align_corners=True)
        pred = torch.nn.ReplicationPad2d(8)(pred)
        pred = F.interpolate(pred, scale_factor=2, mode="bilinear", align_corners=True)
    pred = torch.clamp(pred, min=0.4, max=10)
    return pred[:, 0] if use_224 else pred[:, 0, 20:460, 24:616]


def torch_errors(x, y):
    """utils.py:85-98 in float32"""
    thresh = torch.max((y / x), (x / y))
    return (torch.mean(torch.abs(y - x) / y), torch.sqrt(((y - x) ** 2).mean()),
            (torch.abs(torch.log10(y) - torch.log10(x))).mean(), (thresh < 1.25).float().mean(),
            (thresh < 1.25 ** 2).float().mean(), (thresh < 1.25 ** 3).float().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=654)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    n = a.frames
    g = torch.Generator(device="cuda").manual_seed(0)
    gt = torch.rand((n, 480, 640), device="cuda", generator=g) * 8.0 + 1.0
    res = {"card": card(), "frames": n, "batch": BATCH}
    for use_224, size in ((False, (240, 320)), (True, (224, 224))):
        tag = "224" if use_224 else "eigen"
        ev = NyuDepthEvaluator(gt, use_224=use_224)
        disp = torch.rand((n, 1) + size, device="cuda", generator=g) * 900.0 + 50.0
        gts = ev.gt

        def evaluator():
            ev.reset()
            for i in range(0, n, BATCH):
                ev.add(disp[i:i + BATCH])
            return ev.summary()

        def per_frame():
            preds = [torch_chain(disp[i:i + 1] / 100, use_224) for i in range(n)]
            return [float(v) for v in torch_errors(torch.cat(preds), gts)]

        def batched():
            preds = [torch_chain(disp[i:i + BATCH] / 100, use_224) for i in range(0, n, BATCH)]
            return [float(v) for v in torch_errors(torch.cat(preds), gts)]
        res["evaluator_ms_" + tag] = timed(evaluator, a.steps, a.warmup)
        res["torch_fp32_per_frame_ms_" + tag] = timed(per_frame, a.steps, a.warmup)
        res["torch_fp32_batched_ms_" + tag] = timed(batched, a.steps, a.warmup)
        del ev

    ch = synth.DENSENET161_CH
    dec = nd.SparseDecoderWave(enc_features=list(ch), decoder_width=0.5)
    synth.load_random(dec, seed=3)
    dec = dec.cuda().eval()
    feats = [f.cuda() for f in synth.blocky_features(synth.nyu_feature_shapes(BATCH, 480, 640, ch), seed=9, cell=16)]
    ev = NyuDepthEvaluator(gt)

    def decode_only():
        with torch.no_grad():
            for _ in range(0, n, BATCH):
                dec(feats, 0.1)

    def point():
        ev.reset()
        with torch.no_grad():
            for i in range(0, n, BATCH):
                out = dec(feats, 0.1)
                ev.add(out[("disp", 0)][:min(BATCH, n - i)])
        return ev.summary()

    res["decoder_only_ms"] = timed(decode_only, a.steps, a.warmup)
    res["sweep_point_ms"] = timed(point, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
