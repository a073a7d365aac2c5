"""The baseline decoders against the wavelet decoders on one engine, with CUDA events.

    python scripts/baseline_bench.py [--parts a,b,c] [--steps 10] [--warmup 3] [--runs 3] [--out DIR]

(a) Inference (no_grad), ms per batch.  KITTI ResNet18 640x192 with 16 frames and ResNet50 1024x320 with 32 frames:
    DepthDecoder, DepthWaveProgressiveDecoder and SparseDepthWaveProgressiveDecoder at threshold 0.05.  NYU DenseNet161
    640x480 with 8 frames: Decoder, DecoderWave and SparseDecoderWave (threshold 0.1, its default).  Modes: native (libwmd,
    fp32-faithful), cudnn_tf32 (the cuDNN module graph with TF32 allowed, PyTorch's default) and cudnn_fp32 (the same
    graph with allow_tf32 False).  The sparse decoders have no cuDNN graph: native only.
(b) Training step (forward + backward, weight packing included) of each baseline: native, cudnn_fp32, cudnn_tf32; KITTI at
    ResNet18 640x192 with 12 frames (the KITTI options' default batch), NYU DenseNet161 640x480 with 8 frames.
(c) DepthDecoder's level-0 tail: the fused kernel (wmd_disp_tail16_f32) against the chain it replaces, upconv(0,1) on the
    gather-GEMM engine then dispconv(0) on head_conv3x3 (composed here from ``ops``), on the two KITTI shapes of (a);
    with the largest difference between their outputs.
Modes run alternated, --runs times each, in one process; the card and its power limit are read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wavelet_monodepth_b200 import kitti_decoders as kd, nyu_decoders as nd, ops, synth  # noqa: E402
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_SIGMOID, PAD_REFLECT, PAD_ZERO  # noqa: E402

KITTI = {"r18_640x192_b16": (synth.RESNET18_CH, 16, 192, 640), "r50_1024x320_b32": (synth.RESNET50_CH, 32, 320, 1024)}
NYU = {"d161_640x480_b8": (synth.DENSENET161_CH, 8, 480, 640)}
TRAIN = {"kitti_r18_640x192_b12": ("kitti", synth.RESNET18_CH, 12, 192, 640),
         "nyu_d161_640x480_b8": ("nyu", synth.DENSENET161_CH, 8, 480, 640)}
MODES = ("native", "cudnn_tf32", "cudnn_fp32")


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
    return round(e0.elapsed_time(e1) / steps, 3)


def alternate(fns, a):
    ms = {k: [] for k in fns}
    for _ in range(a.runs):
        for k, fn in fns.items():
            ms[k].append(timed(fn, a.steps, a.warmup))
    return ms


def infer(mod, feats, mode, *args):
    if mode == "native":
        return mod(feats, *args)
    torch.backends.cudnn.allow_tf32 = mode == "cudnn_tf32"
    return mod._autograd_forward(feats)


@torch.no_grad()
def part_a(a, gpu):
    recs = []
    for name, (ch, n, h, w) in KITTI.items():
        feats = [f.cuda() for f in synth.bench_kitti_features(n, h, w, ch)]
        base = kd.DepthDecoder(np.array(ch))
        synth.load_random(base, seed=1)
        wave, sparse = kd.DepthWaveProgressiveDecoder(np.array(ch)), kd.SparseDepthWaveProgressiveDecoder(np.array(ch))
        synth.bench_kitti_params(wave)
        synth.bench_kitti_params(sparse)
        sparse.count_ops = False
        mods = {"DepthDecoder": (base.cuda().eval(), ()), "DepthWaveProgressiveDecoder": (wave.cuda().eval(), ()),
                "SparseDepthWaveProgressiveDecoder@0.05": (sparse.cuda().eval(), (0.05,))}
        recs += _time_decoders("kitti_" + name, mods, feats, a, gpu)
        del feats, mods, base, wave, sparse
        torch.cuda.empty_cache()
    for name, (ch, n, h, w) in NYU.items():
        feats = [f.cuda() for f in synth.blocky_features(synth.nyu_feature_shapes(n, h, w, ch), seed=2)]
        mods = {}
        for cls, args in ((nd.Decoder, ()), (nd.DecoderWave, ()), (nd.SparseDecoderWave, (0.1,))):
            mod = cls(enc_features=list(ch), decoder_width=0.5)
            synth.load_random(mod, seed=1)
            if cls is nd.SparseDecoderWave:
                mod.count_ops = False
            mods[cls.__name__ + ("@0.1" if args else "")] = (mod.cuda().eval(), args)
        recs += _time_decoders("nyu_" + name, mods, feats, a, gpu)
        del feats, mods
        torch.cuda.empty_cache()
    return recs


def _time_decoders(workload, mods, feats, a, gpu):
    fns = {}
    for dname, (mod, args) in mods.items():
        for mode in (MODES if not args else ("native",)):
            fns[(dname, mode)] = (lambda m=mod, md=mode, ar=args: infer(m, feats, md, *ar))
    ms = alternate(fns, a)
    recs = []
    for dname, (mod, args) in mods.items():
        per = {mode: ms[(dname, mode)] for mode in MODES if (dname, mode) in ms}
        rec = dict(part="a", workload=workload, decoder=dname, gpu=gpu, ms_per_batch=per)
        if not args:
            ref = infer(mod, feats, "native")[("disp", 0)]
            rec["disp0_max_rel_diff_vs_native"] = {
                m: float("%.3g" % ((infer(mod, feats, m)[("disp", 0)] - ref).abs().max() / ref.abs().max()))
                for m in MODES[1:]}
        print(json.dumps(rec), flush=True)
        recs.append(rec)
    return recs


def part_b(a, gpu):
    recs = []
    for name, (kind, ch, n, h, w) in TRAIN.items():
        if kind == "kitti":
            mod = kd.DepthDecoder(np.array(ch))
            shapes = synth.kitti_feature_shapes(n, h, w, ch)
        else:
            mod = nd.Decoder(enc_features=list(ch), decoder_width=0.5)
            shapes = synth.nyu_feature_shapes(n, h, w, ch)
        synth.load_random(mod, seed=1)
        mod = mod.cuda().train()
        feats = [f.cuda().requires_grad_(True) for f in synth.blocky_features(shapes, seed=2)]

        def step(mode):
            torch.backends.cudnn.allow_tf32 = mode == "cudnn_tf32"
            mod.zero_grad(set_to_none=True)
            for f in feats:
                f.grad = None
            out = mod._autograd_forward(feats) if mode == "cudnn_fp32" else mod(feats)
            sum(v.mean() for v in out.values()).backward()

        ms = alternate({m: (lambda m=m: step(m)) for m in ("native", "cudnn_fp32", "cudnn_tf32")}, a)
        grads = {}
        for m in ("native", "cudnn_fp32"):
            step(m)
            grads[m] = [p.grad.clone() for p in mod.parameters()]
        diff = max((x - y).abs().max().item() / max(y.abs().max().item(), 1e-30)
                   for x, y in zip(grads["native"], grads["cudnn_fp32"]))
        rec = dict(part="b", workload=name, decoder=type(mod).__name__, gpu=gpu, ms_per_step=ms,
                   max_grad_diff_vs_cudnn_fp32=float("%.3g" % diff))
        print(json.dumps(rec), flush=True)
        recs.append(rec)
        del mod, feats, grads
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = False
    return recs


@torch.no_grad()
def part_c(a, gpu):
    """Level 0 from upconv(0,0)'s rows x (N*h*w, 16) at half resolution: the fused tail against conv_rows + head_conv3x3."""
    recs = []
    mod = kd.DepthDecoder(np.array(synth.RESNET18_CH))
    synth.load_random(mod, seed=1)
    mod = mod.cuda()
    c1, cd = mod.convs[("upconv", 0, 1)].conv.conv, mod.convs[("dispconv", 0)].conv
    packed = ops.pack_disp_tail16(c1.weight, c1.bias, cd.weight, cd.bias)
    w1 = ops.pack_weight(c1.weight)
    w2 = ops.pack_head_weight(cd.weight)
    for name, (_, n, h, w) in KITTI.items():
        h, w = h // 2, w // 2
        x = torch.rand((n * h * w, 16), dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(3))

        def fused():
            return ops.disp_tail16(x, packed, 1, n, h, w)

        def chain():
            u = ops.conv_rows(x, 16, w1, c1.bias, 16, n, 2 * h, 2 * w, pad=PAD_ZERO, act=ACT_ELU, shift0=1)
            return ops.head_conv3x3(u, 16, 0, w2, cd.bias, n, 2 * h, 2 * w, 1, act=ACT_SIGMOID, pad=PAD_REFLECT)

        ms = alternate({"fused": fused, "chain": chain}, a)
        rec = dict(part="c", workload="kitti_" + name, gpu=gpu, ms_per_call=ms,
                   max_abs_diff=float("%.3g" % (fused() - chain()).abs().max().item()),
                   bytes_fused=4 * n * h * w * 16 + 4 * n * 4 * h * w,
                   bytes_chain=4 * n * h * w * 16 + 2 * 4 * n * 4 * h * w * 16 + 4 * n * 4 * h * w)
        print(json.dumps(rec), flush=True)
        recs.append(rec)
        del x
        torch.cuda.empty_cache()
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="a,b,c")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    prev_tf32 = torch.backends.cudnn.allow_tf32
    lines = []
    for part in a.parts.split(","):
        lines += {"a": part_a, "b": part_b, "c": part_c}[part](a, gpu)
    torch.backends.cudnn.allow_tf32 = prev_tf32
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "baseline_bench.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
