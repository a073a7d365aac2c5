"""Decoder training step (forward + backward, weight packing included) per mode, with CUDA events.

    python scripts/train_step_bench.py [--steps 10] [--warmup 3] [--runs 3] [--out DIR]

Workloads: KITTI ResNet18 640x192 with 12 frames (the KITTI options' default batch), KITTI ResNet50 1024x320 with 8
frames, NYU DenseNet161 640x480 with 8 frames, and the 224-pixel NYU decoder (DecoderWave224) on DenseNet161 and
MobileNetV2-light features with 8 frames (NYUv2/train.py --bs).  The 224 decoder's loss leaves out ("disp", 1), its
floor division, which torch cannot differentiate.  Modes: native (libwmd forward and backward, selected because
allow_tf32 is False), cudnn_fp32 (the decoder's cuDNN path with allow_tf32 False) and cudnn_tf32 (context only: it
computes a less precise result).  The three modes run alternated, --runs times each, in one process.  Also reported:
per-kernel times of the backward kernels (torch.profiler, a separate step), the largest gradient difference between
native and cuDNN fp32, per tensor relative to its largest cuDNN element, and the card with its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wavelet_monodepth_b200 import kitti_decoders as kd, nyu_decoders as nd, synth  # noqa: E402

WORKLOADS = {
    "kitti_r18_640x192_b12": ("kitti", [64, 64, 128, 256, 512], 12, 192, 640),
    "kitti_r50_1024x320_b8": ("kitti", [64, 256, 512, 1024, 2048], 8, 320, 1024),
    "nyu_d161_640x480_b8": ("nyu", [96, 96, 192, 384, 2208], 8, 480, 640),
    "nyu224_d161_b8": ("nyu224", [96, 96, 192, 384, 2208], 8, 224, 224),
    "nyu224_mnv2light_b8": ("nyu224", [32, 24, 32, 64, 160], 8, 224, 224),
}
MODES = ("native", "cudnn_fp32", "cudnn_tf32")
KERNELS = ("act_bwd_kernel", "conv_wgrad_kernel", "fold_src0_kernel", "fold_src1_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build(kind, ch, n, h, w):
    if kind == "kitti":
        mod = kd.DepthWaveProgressiveDecoder(np.array(ch))
        shapes = synth.kitti_feature_shapes(n, h, w, ch)
    else:
        mod = (nd.DecoderWave224 if kind == "nyu224" else nd.DecoderWave)(enc_features=ch, decoder_width=0.5)
        shapes = synth.nyu_feature_shapes(n, h, w, ch)
    synth.load_random(mod, seed=1)
    feats = [f.cuda().requires_grad_(True) for f in synth.blocky_features(shapes, seed=2)]
    return mod.cuda().train(), feats


def step(mod, feats, mode):
    torch.backends.cudnn.allow_tf32 = mode == "cudnn_tf32"
    mod.zero_grad(set_to_none=True)
    for f in feats:
        f.grad = None
    out = mod._autograd_forward(feats) if mode == "cudnn_fp32" else mod(feats)
    disp = [v for k, v in out.items() if k[0] == "disp" and not (k[1] == 1 and isinstance(mod, nd.DecoderWave224))]
    sum(d.mean() for d in disp).backward()


def time_mode(mod, feats, mode, steps, warmup):
    for _ in range(warmup):
        step(mod, feats, mode)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(mod, feats, mode)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def grads(mod, feats, mode):
    step(mod, feats, mode)
    torch.cuda.synchronize()
    return [p.grad.clone() for p in mod.parameters()] + [f.grad.clone() for f in feats if f.grad is not None]


def kernel_times(mod, feats):
    from torch.profiler import ProfilerActivity, profile
    step(mod, feats, "native")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(mod, feats, "native")
        torch.cuda.synchronize()
    res = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                res[k] = res.get(k, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    lines = []
    for name in a.workloads.split(","):
        mod, feats = build(*WORKLOADS[name])
        ms = {m: [] for m in MODES}
        for _ in range(a.runs):
            for m in MODES:
                ms[m].append(round(time_mode(mod, feats, m, a.steps, a.warmup), 3))
        gn, gc = grads(mod, feats, "native"), grads(mod, feats, "cudnn_fp32")
        diff = max((x - y).abs().max().item() / max(y.abs().max().item(), 1e-30) for x, y in zip(gn, gc))
        rec = dict(workload=name, gpu=gpu, ms_per_step=ms, native_kernels_ms=kernel_times(mod, feats),
                   max_grad_diff_vs_cudnn_fp32=float("%.3g" % diff))
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del mod, feats
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_step_bench.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
