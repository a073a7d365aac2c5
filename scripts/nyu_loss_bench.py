"""NYUv2 training loss: libwmd's NyuDepthLoss against the reference's float32 torch chain (train.py:279-327).

    python scripts/nyu_loss_bench.py [--iters 200] [--runs 3] [--out DIR]

Workloads (8 frames, NYUv2/train.py --bs):
  nyu_240x320   DecoderWave's pyramid: ("disp", s) at 240x320 / 2**s, default scales, no LL term (DecoderWave names its
                LL ("wavelets", 2, "LL"), so the reference skips it)
  nyu224        DecoderWave224's pyramid at 224x224 with its 14x14 LL, use_wavelets and supervise_LL
Per workload:
  * the loss forward + backward (random predictions as leaf tensors), native and torch alternated --runs times,
    --iters calls each, timed with CUDA events -> ms per call;
  * the CUDA kernels one call launches, each implementation in a profiler run of its own;
  * a full native DecoderWave / DecoderWave224 training step (DenseNet161 features, fp32 convolutions) with each loss,
    run 3 times: the number of parameter-gradient tensors whose bits differ from the first run's, and the step time.
Also recorded: whether the torch chain's backward raises under torch.use_deterministic_algorithms(True).  The card's
name and power limit are read in the same run.
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

from wavelet_monodepth_b200 import nyu_decoders as nd, synth, wavelets  # noqa: E402
from wavelet_monodepth_b200.nyu_loss import NyuDepthLoss  # noqa: E402

DEV = "cuda"
LL_KEY = ("wavelets", 3, "LL")
D161 = [96, 96, 192, 384, 2208]
# name -> (decoder, image H, W, depth H, W, NyuDepthLoss options)
WORKLOADS = {
    "nyu_240x320": (nd.DecoderWave, 480, 640, 240, 320, dict()),
    "nyu224": (nd.DecoderWave224, 224, 224, 224, 224, dict(use_wavelets=True, supervise_LL=True)),
}
N = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def torch_loss(outputs, depth, disparity=False, use_wavelets=False, supervise_LL=False):
    """train.py:279-327 in torch float32, as the reference computes it"""
    depth_n = 10.0 / depth if disparity else depth
    total = 0
    for s in range(4):
        pred = F.interpolate(outputs[("disp", s)], scale_factor=2 ** s, mode="bilinear", align_corners=True)
        total = total + 0.1 * F.l1_loss(pred, depth_n)
    if use_wavelets and LL_KEY in outputs:
        l_ll = F.l1_loss(outputs[LL_KEY], wavelets.DWT(J=4, wave="haar", mode="reflect")(depth_n)[0]) / 2 ** 4
        if supervise_LL:
            total = total + l_ll
    return total


def losses(opts):
    native = NyuDepthLoss(**opts)
    return {"native": lambda o, d: native(o, d)[0], "torch_f32": lambda o, d: torch_loss(o, d, **opts)}


def loss_inputs(dh, dw, opts):
    g = torch.Generator(device="cpu").manual_seed(0)
    depth = (torch.rand(N, 1, dh, dw, generator=g) * 990 + 10).to(DEV)
    outs = {("disp", s): (torch.rand(N, 1, dh >> s, dw >> s, generator=g) * 990 + 10).to(DEV).requires_grad_(True)
            for s in range(4)}
    if opts.get("use_wavelets"):
        outs[LL_KEY] = (torch.rand(N, 1, dh // 16, dw // 16, generator=g) * 16000).to(DEV).requires_grad_(True)
    return outs, depth


def loss_call(fn, outs, depth):
    fn(outs, depth).backward()


def time_calls(fn, outs, depth, iters):
    for _ in range(5):
        loss_call(fn, outs, depth)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        loss_call(fn, outs, depth)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernels(fn, outs, depth):
    from torch.profiler import ProfilerActivity, profile
    loss_call(fn, outs, depth)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loss_call(fn, outs, depth)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(names), sorted(set(names))


def torch_chain_raises_when_deterministic(opts):
    outs, depth = loss_inputs(16, 16, opts)
    torch.use_deterministic_algorithms(True)
    try:
        torch_loss(outs, depth, **opts).backward()
        return False
    except RuntimeError:
        return True
    finally:
        torch.use_deterministic_algorithms(False)


def decoder_steps(cls, ih, iw, dh, dw, fn):
    """3 native training steps with loss `fn` -> (tensors differing from the first run's bits, ms per step)"""
    torch.backends.cudnn.allow_tf32 = False
    mod = cls(enc_features=D161, decoder_width=0.5)
    synth.load_random(mod, seed=1)
    mod = mod.to(DEV).train()
    feats = [f.to(DEV) for f in synth.blocky_features(synth.nyu_feature_shapes(N, ih, iw, D161), seed=2)]
    depth = (torch.rand(N, 1, dh, dw, generator=torch.Generator().manual_seed(3)) * 990 + 10).to(DEV)
    runs, times = [], []
    for _ in range(4):                       # the first is a warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        mod.zero_grad(set_to_none=True)
        e0.record()
        fn(mod(feats), depth).backward()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        runs.append([p.grad.clone() for p in mod.parameters() if p.grad is not None])
    runs, times = runs[1:], times[1:]
    differ = sum(any(not torch.equal(a, r[i]) for r in runs[1:]) for i, a in enumerate(runs[0]))
    return differ, len(runs[0]), round(float(np.median(times)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    lines = []
    for name, (cls, ih, iw, dh, dw, opts) in WORKLOADS.items():
        fns = losses(opts)
        outs, depth = loss_inputs(dh, dw, opts)
        ms = {k: [] for k in fns}
        for _ in range(a.runs):
            for k, fn in fns.items():
                ms[k].append(round(time_calls(fn, outs, depth, a.iters), 4))
        launches = {k: kernels(fn, outs, depth) for k, fn in fns.items()}
        steps = {k: decoder_steps(cls, ih, iw, dh, dw, fn) for k, fn in fns.items()}
        raises = torch_chain_raises_when_deterministic(opts)
        rec = dict(workload=name, gpu=gpu, frames=N, loss_fwd_bwd_ms=ms,
                   launches_per_call={k: v[0] for k, v in launches.items()},
                   kernels={k: v[1] for k, v in launches.items()},
                   decoder_step={k: dict(grad_tensors_differing_over_3_runs=v[0], grad_tensors=v[1], ms_median=v[2])
                                 for k, v in steps.items()},
                   torch_chain_raises_under_deterministic_algorithms=raises)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "nyu_loss_bench.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
