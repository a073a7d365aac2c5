"""Inference (no_grad forward) of the 224-pixel NYU wavelet decoder per mode, with CUDA events.

    python scripts/decoder224_bench.py [--batches 8,32] [--encoders d161,mnv2light] [--steps 20] [--warmup 5] [--runs 3]
                                       [--out DIR]

Modes: native (DecoderWave224 on libwmd, fp32-faithful), cudnn_tf32 (the cuDNN module graph with TF32 allowed,
PyTorch's default and what this decoder ran before it had a native engine) and cudnn_fp32 (the same graph with
allow_tf32 False).  The modes run alternated, --runs times each, in one process.  Also reported: the largest relative
difference of ("disp", 0) from the native result per cuDNN mode, and the card with its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from wavelet_monodepth_b200 import nyu_decoders as nd, synth  # noqa: E402

ENCODERS = {"d161": [96, 96, 192, 384, 2208], "mnv2light": [32, 24, 32, 64, 160]}
MODES = ("native", "cudnn_tf32", "cudnn_fp32")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def forward(mod, feats, mode):
    if mode == "native":
        return mod(feats)
    torch.backends.cudnn.allow_tf32 = mode == "cudnn_tf32"
    return mod._autograd_forward(feats)


def time_mode(mod, feats, mode, steps, warmup):
    for _ in range(warmup):
        forward(mod, feats, mode)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        forward(mod, feats, mode)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--encoders", default=",".join(ENCODERS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    prev_tf32 = torch.backends.cudnn.allow_tf32
    lines = []
    torch.set_grad_enabled(False)
    for enc in a.encoders.split(","):
        ch = ENCODERS[enc]
        mod = nd.DecoderWave224(enc_features=ch, decoder_width=0.5)
        synth.load_random(mod, seed=1)
        mod = mod.cuda().eval()
        for n in (int(v) for v in a.batches.split(",")):
            feats = [f.cuda() for f in synth.blocky_features(synth.nyu_feature_shapes(n, 224, 224, ch), seed=2)]
            ms = {m: [] for m in MODES}
            for _ in range(a.runs):
                for m in MODES:
                    ms[m].append(round(time_mode(mod, feats, m, a.steps, a.warmup), 3))
            ref = forward(mod, feats, "native")[("disp", 0)]
            diff = {m: float("%.3g" % ((forward(mod, feats, m)[("disp", 0)] - ref).abs().max() / ref.abs().max()))
                    for m in MODES[1:]}
            rec = dict(decoder="DecoderWave224", encoder=enc, batch=n, gpu=gpu, ms_per_batch=ms,
                       disp0_max_rel_diff_vs_native=diff)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del feats
        del mod
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = prev_tf32
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decoder224_bench.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
