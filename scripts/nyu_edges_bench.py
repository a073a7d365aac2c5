"""NYUv2 depth-boundary-error cost on one GPU, with CUDA events after warm-up.

    python scripts/nyu_edges_bench.py [--frames 654] [--steps 3] [--warmup 1] [--host-frames 8]

Builds a synthetic 654-frame split (480 x 640 ground-truth depth and OC++-style binary edge maps of its depth steps,
240 x 320 disparities of a noisy copy of the scene) and reports, in milliseconds:
  (a) NyuDepthEvaluator.add over the whole split in batches of 16, then summary(), without and with edges;
  (b) the evaluator's one-off edge set-up per split (crop, float32 sums, ground-truth distance maps);
  (c) the reference's per-frame host path for the edges, as compute_depth_boundary_error runs it (normalise, the
      oracle's scikit-image 0.16.2 canny over scipy, two scipy distance transforms, the chamfer sums), per frame,
      averaged over the first --host-frames frames.
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

from oracle import nyu_edges as ne, nyu_eval as one  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=654)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-frames", type=int, default=8)
    a = ap.parse_args()
    n = a.frames
    base = ne.edge_split(0, n=min(n, 16))                 # 16 distinct scenes, repeated over the split
    rep = -(-n // base["gt"].shape[0])
    gt = np.tile(base["gt"], (rep, 1, 1))[:n]
    edges = np.tile(base["edges"], (rep, 1, 1))[:n]
    disp = torch.from_numpy(np.tile(base["disp"], (rep, 1, 1))[:n]).cuda()[:, None]
    res = {"card": card(), "frames": n, "batch": BATCH}
    plain = NyuDepthEvaluator(gt)
    torch.cuda.synchronize()
    t = time.perf_counter()
    ev = NyuDepthEvaluator(gt, edges_gt=edges)
    torch.cuda.synchronize()
    res["edges_setup_ms"] = (time.perf_counter() - t) * 1e3

    def run(e):
        def go():
            e.reset()
            for i in range(0, n, BATCH):
                e.add(disp[i:i + BATCH])
            return e.summary()
        return go
    res["evaluator_ms"] = timed(run(plain), a.steps, a.warmup)
    res["evaluator_with_edges_ms"] = timed(run(ev), a.steps, a.warmup)
    s = run(ev)()
    res["e_acc"], res["e_comp"] = s["e_acc"], s["e_comp"]

    k = min(a.host_frames, n)
    preds = one.predict(disp[:k, 0].cpu().numpy()).astype(np.float32)
    t = time.perf_counter()
    for i in range(k):
        ne.dbe_numpy(edges[i][20:460, 24:616], preds[i])
    res["host_per_frame_ms"] = (time.perf_counter() - t) * 1e3 / k
    res["host_split_estimate_ms"] = res["host_per_frame_ms"] * n
    print(json.dumps(res))


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
