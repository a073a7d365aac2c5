"""Time KITTI's depth hints at 1024x320: libwmd's twelve StereoSGBM matchers + fusion on device-resident uint8 views at
several batch sizes, per-kernel device times (torch.profiler), the CLI end to end on synthetic JPEGs through its loader,
and, where cv2 is importable, the script's cv2 CPU chain on the same host (one process, then one per core).

    python scripts/depth_hints_bench.py [--batches 1 4 8] [--iters 5] [--views 48] [--out DIR]

Prints the card's name and power limit with the numbers, and one JSON line; with --out also writes it there.
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import depth_hints as odh                                          # noqa: E402
from wavelet_monodepth_b200 import kitti_hints                                  # noqa: E402

H, W = 320, 1024


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def views(n, seed=0):
    pairs = [odh.make_pair(seed + k, H, W) for k in range(n)]
    base = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
    lookup = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
    return base, lookup, [k % 2 == 1 for k in range(n)]


def device_rate(batches, iters):
    gen = kitti_hints.DepthHintGenerator(H, W)
    out = {}
    for n in batches:
        base, lookup, right = views(n)
        gen(base, lookup, right)                                                # warm-up
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            gen(base, lookup, right)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / iters
        out[n] = {"ms_per_batch": round(ms, 3), "views_per_s": round(n * 1000.0 / ms, 1)}
        print("device, batch %d: %.2f ms per batch, %.1f views/s" % (n, ms, n * 1000.0 / ms))
    return out


def kernel_times(n):
    gen = kitti_hints.DepthHintGenerator(H, W)
    base, lookup, right = views(n)
    gen(base, lookup, right)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gen(base, lookup, right)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            rows[ev.key] = (rows.get(ev.key, (0.0, 0))[0] + t / 1000.0, ev.count)
    top = sorted(rows.items(), key=lambda kv: -kv[1][0])
    print("per-kernel device time, one batch of %d views (ms, launches):" % n)
    for k, (ms, cnt) in top[:16]:
        print("  %9.3f %4d  %s" % (ms, cnt, k[:100]))
    return {k[:100]: [round(ms, 4), cnt] for k, (ms, cnt) in top[:16]}


def end_to_end(nviews, batch, workers):
    from PIL import Image
    with tempfile.TemporaryDirectory() as tmp:
        data, lines = os.path.join(tmp, "raw"), []
        seq = "2011_09_26/2011_09_26_drive_0001_sync"
        for k in range(nviews // 2):
            left, right = odh.make_pair(1000 + k, 375, 1242)                   # KITTI's raw image size
            for cam, img in (("image_02", left), ("image_03", right)):
                d = os.path.join(data, seq, cam, "data")
                os.makedirs(d, exist_ok=True)
                Image.fromarray(img).save(os.path.join(d, "%010d.jpg" % k), quality=92)
            lines += ["%s %d l" % (seq, k), "%s %d r" % (seq, k)]
        split = os.path.join(tmp, "files.txt")
        with open(split, "w") as f:
            f.write("\n".join(lines) + "\n")
        argv = ["--data_path", data, "--filenames", split, "--save_path", os.path.join(tmp, "hints"),
                "--batch_size", str(batch), "--num_workers", str(workers), "--overwrite_saved_depths"]
        kitti_hints.run(kitti_hints.get_opts(argv))                               # warm-up: workers, first launches
        torch.cuda.synchronize()
        t = time.time()
        kitti_hints.run(kitti_hints.get_opts(argv))
        torch.cuda.synchronize()
        dt = time.time() - t
    r = {"views": len(lines), "seconds": round(dt, 3), "views_per_s": round(len(lines) / dt, 2), "batch": batch,
         "workers": workers}
    print("CLI end to end: %d views in %.2f s, %.2f views/s (batch %d, %d loader workers)"
          % (len(lines), dt, len(lines) / dt, batch, workers))
    return r


def _cv2_view(seed):
    import cv2
    cv2.setNumThreads(0)
    from oracle import sgbm
    left, right = odh.make_pair(seed, H, W)
    for nd, bs in sgbm.MATCHERS:
        cv2.StereoSGBM_create(minDisparity=0, numDisparities=nd, blockSize=bs,
                              **dict(sgbm.HINT_PARAMS)).compute(left, right)
    return seed


def cv2_chain(nviews):
    try:
        import cv2  # noqa: F401
    except ImportError:
        print("cv2 CPU chain: not measured (cv2 is not importable here)")
        return None
    t = time.time()
    for k in range(2):
        _cv2_view(k)
    single = (time.time() - t) / 2
    cores = os.cpu_count() or 1
    with mp.Pool(cores) as pool:
        t = time.time()
        pool.map(_cv2_view, range(nviews))
        par = nviews / (time.time() - t)
    print("cv2 CPU chain (twelve matchers, no fusion): %.2f s per view in one process; %.2f views/s on %d processes"
          % (single, par, cores))
    return {"s_per_view_single": round(single, 3), "views_per_s_all_cores": round(par, 2), "cores": cores}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--views", type=int, default=48)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "size": [H, W], "device": device_rate(a.batches, a.iters),
           "kernels": kernel_times(max(a.batches)),
           "cli": end_to_end(a.views, max(a.batches), min(12, os.cpu_count() or 1)), "cv2": cv2_chain(a.views)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "depth_hints_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
