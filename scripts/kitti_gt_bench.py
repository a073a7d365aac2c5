"""Time KITTI's ground-truth export: libwmd's wmd_velo_depth_f64 on device-resident full-size scans (one call for 32
scans, CUDA events, warmed up, median of repeats), the CLI's export end to end from .bin files in a temporary KITTI
tree through its loader, and oracle.kitti_gt's numpy port of generate_depth_map per frame on the host, on the same
scans (seeded ~120k-point scans of oracle.kitti_gt.synthetic_scan at the five calibration dates, camera 2, vel_depth).

    python scripts/kitti_gt_bench.py [--frames 32] [--repeats 20] [--e2e_frames 128] [--workers 8] [--out DIR]

Prints the card's name and power limit with the numbers, and one JSON line; with --out also writes it there.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_gt as og                                              # noqa: E402
from wavelet_monodepth_b200 import kitti_gt                                     # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def scans(n, calibs):
    """n full-size frames: (date, drive, frame, seed, points) over the five dates, with each date's P and size"""
    dates = sorted(og.DATES)
    frames, P, sizes = [], [], []
    for k in range(n):
        date = dates[k % len(dates)]
        frames.append((date, "%s_drive_%04d_sync" % (date, 1 + k % len(dates)), k, 1000 + k, None))
        p, hw = og.velo_to_image(og.read_calib_text(calibs[date][0]), og.read_calib_text(calibs[date][1]), 2)
        P.append(p)
        sizes.append(hw)
    return frames, np.stack(P), np.array(sizes, np.int32)


def device_time(points, P, sizes, repeats):
    offsets = np.concatenate([[0], np.cumsum([p.shape[0] for p in points])])
    pts = torch.from_numpy(np.concatenate(points)).cuda()
    for _ in range(3):
        kitti_gt.generate_depth_maps(pts, offsets, P, sizes, True)
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        kitti_gt.generate_depth_maps(pts, offsets, P, sizes, True)
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def end_to_end(n, calibs, workers, batch_size):
    with tempfile.TemporaryDirectory() as root:
        frames = [(d, dr, f, s, None) for d, dr, f, s, _ in scans(n, calibs)[0]]
        lines = []
        for date, drive, frame, seed, _ in frames:
            og.write_calib(os.path.join(root, date), calibs[date])
            d = os.path.join(root, date, drive, "velodyne_points", "data")
            os.makedirs(d, exist_ok=True)
            og.synthetic_scan(seed).tofile(os.path.join(d, "%010d.bin" % frame))
            lines.append("%s/%s %010d l" % (date, drive, frame))
        files = os.path.join(root, "test_files.txt")
        with open(files, "w") as f:
            f.write("\n".join(lines) + "\n")
        opt = kitti_gt.get_opts(["--data_path", root, "--split", "eigen", "--filenames", files, "--output",
                                 os.path.join(root, "gt_depths.npz"), "--batch_size", str(batch_size),
                                 "--num_workers", str(workers)])
        rates = []
        for _ in range(2):                                  # the first pass also warms the page cache
            t0 = time.perf_counter()
            maps = kitti_gt.export(opt)
            torch.cuda.synchronize()
            rates.append(len(maps) / (time.perf_counter() - t0))
        return rates


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--frames", type=int, default=32)
    p.add_argument("--repeats", type=int, default=20)
    p.add_argument("--e2e_frames", type=int, default=128)
    p.add_argument("--workers", type=int, default=8)
    p.add_argument("--batch_size", type=int, default=16)
    p.add_argument("--host_frames", type=int, default=8)
    p.add_argument("--out", type=str)
    a = p.parse_args()
    calibs = og.make_calibs()
    frames, P, sizes = scans(a.frames, calibs)
    points = [og.synthetic_scan(f[3]) for f in frames]
    ms, lo, hi = device_time(points, P, sizes, a.repeats)
    print("device: %d scans of %d points, one call %.3f ms (median of %d; min %.3f, max %.3f), %.0f frames/s"
          % (a.frames, points[0].shape[0], ms, a.repeats, lo, hi, a.frames * 1000.0 / ms))
    rates = end_to_end(a.e2e_frames, calibs, a.workers, a.batch_size)
    print("end to end through the CLI's loader (%d workers, batch %d, %d frames): %.1f frames/s (first pass %.1f)"
          % (a.workers, a.batch_size, a.e2e_frames, rates[1], rates[0]))
    host = []
    for k in range(a.host_frames):
        t0 = time.perf_counter()
        og.depth_map(points[k], P[k], int(sizes[k, 0]), int(sizes[k, 1]), True)
        host.append(time.perf_counter() - t0)
    host_ms = float(np.median(host)) * 1000
    print("host: oracle.kitti_gt.depth_map (numpy) %.1f ms per frame (median of %d)" % (host_ms, a.host_frames))
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "frames": a.frames, "points_per_frame": int(points[0].shape[0]),
           "device_ms_per_call": round(ms, 3), "device_ms_min": round(lo, 3), "device_ms_max": round(hi, 3),
           "e2e_frames_per_s": round(rates[1], 1), "e2e_first_pass_frames_per_s": round(rates[0], 1),
           "workers": a.workers, "host_oracle_ms_per_frame": round(host_ms, 1)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "kitti_gt_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
