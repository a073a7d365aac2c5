"""KITTI depth-hints training loss: libwmd's KittiDepthHintsLoss against the reference's float32 torch chain
(KITTI/trainer.py generate_images_pred + compute_losses_hints, restated in tests/test_gpu_kitti_loss.py:torch_chain).

    python scripts/kitti_loss_bench.py [--iters 50] [--runs 3]

Workloads: R18 640x192 with 12 frames (the trainer's defaults) and R50 1024x320 with 4 frames (the README command's
size).  Per workload:
  * the loss forward + backward (random disparities as leaf tensors), native and torch alternated --runs times,
    --iters calls each, timed with CUDA events -> ms per call;
  * the CUDA kernels one call launches, each implementation in a profiler run of its own;
  * the peak memory the loss adds with grad enabled;
  * a full native DepthWaveProgressiveDecoder training step (fp32 convolutions) with each loss, 3 runs: the number of
    parameter-gradient tensors whose bits differ from the first run's, and the median step time.
Also recorded: whether the torch chain's backward raises under torch.use_deterministic_algorithms(True).  The card's
name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import kitti_loss as okl  # noqa: E402
from test_gpu_kitti_loss import to_dev, torch_chain  # noqa: E402
from wavelet_monodepth_b200 import kitti_decoders as kd, synth  # noqa: E402
from wavelet_monodepth_b200.kitti_loss import KittiDepthHintsLoss  # noqa: E402

DEV = "cuda"
WORKLOADS = {"r18_640x192_x12": ((64, 64, 128, 256, 512), 12, 192, 640),
             "r50_1024x320_x4": ((64, 256, 512, 1024, 2048), 4, 320, 1024)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make(n, H, W, seed=5):
    case = dict(N=n, H=H, W=W, scales=okl.SCALES, loss_scales=okl.SCALES)
    inp, disps = okl.make_inputs(case, seed)
    return to_dev(inp, disps, case)


def loss_only(native, inputs, outputs, H, W):
    """one forward + backward"""
    if native:
        loss = KittiDepthHintsLoss(H, W)
        return lambda: loss(inputs, outputs)[0].backward()
    return lambda: torch_chain(inputs, outputs, okl.SCALES, okl.SCALES, H, W)[0].backward()


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def launches(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def peak_added(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def step(native, ch, n, H, W, runs=3):
    torch.backends.cudnn.allow_tf32 = False
    inputs, _ = make(n, H, W)
    grads, times = [], []
    for _ in range(runs):
        mod = kd.DepthWaveProgressiveDecoder(np.array(ch))
        synth.load_random(mod, seed=1)
        mod = mod.to(DEV).train()
        feats = [f.to(DEV) for f in synth.blocky_features(synth.kitti_feature_shapes(n, H, W, ch), seed=2)]
        torch.manual_seed(5)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = mod(feats)
        if native:
            total, _ = KittiDepthHintsLoss(H, W)(inputs, out)
        else:
            total, _ = torch_chain(inputs, out, okl.SCALES, okl.SCALES, H, W)
        total.backward()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
        grads.append([p.grad.clone() for p in mod.parameters() if p.grad is not None])
    differ = sum(int(not torch.equal(x, y)) for g in grads[1:] for x, y in zip(grads[0], g))
    return {"grad_tensors_differing": differ, "of": len(grads[0]) * (runs - 1), "step_ms_median": float(np.median(times))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    res = {"card": card(), "workloads": {}}
    for name, (ch, n, H, W) in WORKLOADS.items():
        inputs, outputs = make(n, H, W)
        r = {"native_ms": [], "torch_ms": []}
        fns = {True: loss_only(True, inputs, outputs, H, W), False: loss_only(False, inputs, outputs, H, W)}
        for _ in range(args.runs):
            r["native_ms"].append(round(timed(fns[True], args.iters), 3))
            r["torch_ms"].append(round(timed(fns[False], args.iters), 3))
        r["native_launches"], r["torch_launches"] = launches(fns[True]), launches(fns[False])
        r["native_peak_mib"], r["torch_peak_mib"] = round(peak_added(fns[True]), 1), round(peak_added(fns[False]), 1)
        r["step_native"] = step(True, ch, n, H, W)
        r["step_torch"] = step(False, ch, n, H, W)
        res["workloads"][name] = r
    torch.use_deterministic_algorithms(True)
    try:
        inputs, outputs = make(2, 192, 640)
        loss_only(False, inputs, outputs, 192, 640)()
        res["torch_chain_raises_under_deterministic"] = False
    except RuntimeError as e:
        res["torch_chain_raises_under_deterministic"] = str(e).splitlines()[0][:160]
    finally:
        torch.use_deterministic_algorithms(False)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
