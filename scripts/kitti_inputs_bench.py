"""Time KITTI's training inputs on libwmd: the device time of one KittiInputs call (batch 12, frames 0 and "s", so 24
views at mixed raw sizes, with jitter on half the items and depth hints) at 640x192 and 1024x320 from device-resident
views, and items/s end to end through a DataLoader on synthetic JPEGs: KittiInputsDataset + collate + KittiInputs
against the reference-equivalent host path (the PIL chain, torchvision's adjust_* and to_tensor in the workers, as
KITTI/datasets/mono_dataset.py does it) at the same worker count.

    python scripts/kitti_inputs_bench.py [--iters 50] [--workers 8] [--items 96] [--out DIR]

Prints the card's name and power limit with the numbers, and one JSON line; with --out also writes it there.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_inputs as oki                                          # noqa: E402
from wavelet_monodepth_b200 import kitti_inputs as ki                            # noqa: E402

FRAMES = [0, "s"]
BATCH = 12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def items(n, seed=0):
    rng = random.Random(seed)
    out = []
    for k in range(n):
        h, w = oki.RAW_SIZES[k % 5]
        view = oki.synthetic_view(seed + k, h, w)
        aug = k % 2 == 0
        out.append({"views": {0: view, "s": view[:, ::-1].copy()}, "do_color_aug": aug, "do_flip": k % 3 == 0,
                    "jitter": ki.get_params(rng) if aug else None, "side": "lr"[k % 2], "image_path": str(k),
                    "hint": oki.synthetic_hint(seed + k, 320, 1024)})
    return out


def device_time(height, width, iters):
    batch = ki.collate(items(BATCH))
    batch["src"] = batch["src"].cuda()                  # device-resident views
    batch["hint"] = batch["hint"].cuda()
    fn = ki.KittiInputs(height, width, FRAMES, use_depth_hints=True)
    for _ in range(3):
        fn(batch)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    s.record()
    for _ in range(iters):
        fn(batch)
    e.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / iters
    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
    with prof:
        for _ in range(5):
            fn(batch)
        torch.cuda.synchronize()
    kern = sum(ev.device_time_total for ev in prof.key_averages() if "inputs_" in ev.key) / 5 / 1e3
    return {"ms_per_call_events": s.elapsed_time(e) / iters, "ms_per_call_wall": wall * 1e3,
            "ms_per_call_kernels": kern, "views": BATCH * len(FRAMES)}


def write_tree(root, n):
    from PIL import Image
    lines = []
    for k in range(n):
        seq = "seq%d" % (k % 5)
        h, w = oki.RAW_SIZES[k % 5]
        for cam in (2, 3):
            path = os.path.join(root, seq, "image_0%d" % cam, "data", "%010d.jpg" % k)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            Image.fromarray(oki.synthetic_view(k * 10 + cam, h, w)).save(path, quality=92)
        lines.append("%s %d %s" % (seq, k, "lr"[k % 2]))
    return lines


class HostPath(ki.KittiInputsDataset):
    """the reference's preprocessing in the worker: PIL flip, the LANCZOS chain from scale -1, ColorJitter via
    torchvision's adjust_* in the drawn order and to_tensor of every scale, -1 included"""

    def __getitem__(self, index):
        import torchvision.transforms.functional as TF
        from PIL import Image
        it = super().__getitem__(index)
        adjust = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)
        out = {}
        for f, view in it["views"].items():
            img = Image.fromarray(view)
            if it["do_flip"]:
                img = img.transpose(Image.FLIP_LEFT_RIGHT)
            chain = {-1: img}
            for s in self.target_scales:
                img = img.resize((self.width >> s, self.height >> s), Image.LANCZOS)
                chain[s] = img
            for s, im in chain.items():
                out[("color", f, s)] = TF.to_tensor(im)
                aug = im
                if it["jitter"] is not None:
                    for op in it["jitter"][1]:
                        aug = adjust[op](aug, it["jitter"][0][op])
                out[("color_aug", f, s)] = TF.to_tensor(aug)
        for f in it["views"]:
            del out[("color", f, -1)], out[("color_aug", f, -1)]
        return out


def loader_rate(root, lines, height, width, workers, device):
    res = {}
    for name in ("device", "host"):
        cls = ki.KittiInputsDataset if name == "device" else HostPath
        ds = cls(root, lines, height, width, FRAMES, is_train=True)
        kw = dict(collate_fn=ki.collate) if name == "device" else {}
        dl = torch.utils.data.DataLoader(ds, batch_size=BATCH, shuffle=False, num_workers=workers, pin_memory=True,
                                         drop_last=True, persistent_workers=False, **kw)
        fn = ki.KittiInputs(height, width, FRAMES)
        done, t0 = 0, None
        for i, batch in enumerate(dl):
            if name == "device":
                out = fn(batch, device)
            else:
                out = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
            if i == 0:                                     # the workers' start-up is not the rate
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                continue
            done += BATCH
        torch.cuda.synchronize()
        res[name] = done / (time.perf_counter() - t0)
        del out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--items", type=int, default=96)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kitti_inputs_bench needs a CUDA device")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "batch": BATCH, "frames": [str(f) for f in FRAMES], "device": {},
           "loader_items_per_s": {}, "workers": a.workers}
    for h, w in ((192, 640), (320, 1024)):
        res["device"]["%dx%d" % (w, h)] = d = device_time(h, w, a.iters)
        print("%dx%d device: %.3f ms per call (events), %.3f ms wall, %.3f ms in the kernels, %d views"
              % (w, h, d["ms_per_call_events"], d["ms_per_call_wall"], d["ms_per_call_kernels"], d["views"]))
    with tempfile.TemporaryDirectory() as root:
        lines = write_tree(root, a.items)
        for h, w in ((192, 640), (320, 1024)):
            r = loader_rate(root, lines, h, w, a.workers, torch.device("cuda", 0))
            res["loader_items_per_s"]["%dx%d" % (w, h)] = r
            print("%dx%d loader, %d workers: %.1f items/s on the device path, %.1f items/s on the host path"
                  % (w, h, a.workers, r["device"], r["host"]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "kitti_inputs_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
