"""Time NYUv2's training inputs on libwmd: the device time of one NyuInputs call (batch --bs, 640x480 and 224x224, from
device-resident decoded items, CUDA events, median over --iters calls after warm-up), and items/s end to end through
a DataLoader over a seeded synthetic zip (JPEG images, PNG depths): NyuInputsDataset + collate + NyuInputs against the
reference's host path (NYUv2/data.py's flip, channel swap, adjust_gamma, crop, resize and to_tensor in the workers,
restated here with the same PIL and torchvision calls) at the same worker count, and the device path's loader alone
(decode, collate and pinning, without the device call).

    python scripts/nyu_inputs_bench.py [--bs 8] [--iters 100] [--workers 8] [--items 1024] [--out DIR]

Prints the card's name and power limit with the numbers, and one JSON line; with --out also writes it there.
"""
import argparse
import io
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import nyu_inputs as oni                                            # noqa: E402
from wavelet_monodepth_b200 import nyu_inputs as ni                              # noqa: E402


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
        flip, perm, gamma = ni.draws(True, rng)
        out.append({"image": oni.synthetic_image(seed + k), "depth": oni.synthetic_depth(seed + k), "flip": flip,
                    "perm": perm, "gamma": gamma})
    return out


def device_time(is_224, bs, iters):
    batch = ni.collate(items(bs))
    batch["image"], batch["depth"] = batch["image"].cuda(), batch["depth"].cuda()      # device-resident items
    fn = ni.NyuInputs(is_224)
    for _ in range(10):
        fn(batch)
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn(batch)
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
    with prof:
        for _ in range(10):
            fn(batch)
        torch.cuda.synchronize()
    kern = sum(ev.device_time_total for ev in prof.key_averages() if "nyu_inputs_" in ev.key) / 10 / 1e3
    return {"ms_per_call_median": statistics.median(times), "ms_per_call_min": min(times), "calls": iters,
            "ms_per_call_kernels": kern, "items": bs}


def write_zip(path, n):
    from PIL import Image
    rows = []
    with zipfile.ZipFile(path, "w") as zf:
        for k in range(n):
            img, dep = "data/nyu2_train/s%d/%d.jpg" % (k % 7, k), "data/nyu2_train/s%d/%d.png" % (k % 7, k)
            buf = io.BytesIO()
            Image.fromarray(oni.synthetic_image(k)).save(buf, "JPEG", quality=92)
            zf.writestr(img, buf.getvalue())
            buf = io.BytesIO()
            Image.fromarray(oni.synthetic_depth(k)).save(buf, "PNG")
            zf.writestr(dep, buf.getvalue())
            rows.append("%s,%s" % (img, dep))
        zf.writestr("data/nyu2_train.csv", "\n".join(rows) + "\n")


class HostPath(torch.utils.data.Dataset):
    """the reference's training transform in the worker: decode, flip, channel swap, torchvision's adjust_gamma, the
    16-pixel crop, resize with Pillow's default filter, to_tensor, depth * 1000 clamped to [10, 1000]"""

    def __init__(self, data, rows, is_224):
        self.data, self.rows = data, rows
        self.image_size, self.depth_size = ((224, 224), (224, 224)) if is_224 else ((640, 480), (320, 240))

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, idx):
        import torchvision.transforms.functional as TF
        from PIL import Image
        image = Image.open(io.BytesIO(self.data[self.rows[idx][0]]))
        depth = Image.open(io.BytesIO(self.data[self.rows[idx][1]]))
        if random.random() < 0.5:
            image, depth = image.transpose(Image.FLIP_LEFT_RIGHT), depth.transpose(Image.FLIP_LEFT_RIGHT)
        if random.random() < 0.1:
            image = Image.fromarray(np.asarray(image)[..., list(ni.PERMS[random.randint(0, 5)])])
        image = TF.adjust_gamma(image, random.uniform(1 / 0.8, 0.8), gain=1)
        box = (16, 16, 624, 464)
        image = TF.to_tensor(image.crop(box).resize(self.image_size))
        depth = torch.clamp(TF.to_tensor(depth.crop(box).resize(self.depth_size)).float() * 1000, 10, 1000)
        return {"image": image, "depth": depth}


def loader_rate(path, is_224, bs, workers, device):
    data, rows = ni.load_zip_to_mem(path)
    res = {}
    for name in ("device", "host", "loader_only"):
        if name != "host":
            ds, kw = ni.NyuInputsDataset(data, rows), dict(collate_fn=ni.collate)
        else:
            ds, kw = HostPath(data, rows, is_224), {}
        dl = torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=False, num_workers=workers, pin_memory=True,
                                         drop_last=True, **kw)
        fn = ni.NyuInputs(is_224)
        done, t0 = 0, None
        for i, batch in enumerate(dl):
            if name == "device":
                out = fn(batch, device)
            elif name == "loader_only":                    # the device path's loader without its device call
                out = batch
            else:
                out = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
            if i == 0:                                     # the workers' start-up is not the rate
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                continue
            done += bs
        torch.cuda.synchronize()
        res[name] = done / (time.perf_counter() - t0)
        del out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, default=8)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--items", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nyu_inputs_bench needs a CUDA device")
    if a.iters < 50:
        sys.exit("--iters must be at least 50")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "batch": a.bs, "device": {}, "loader_items_per_s": {},
           "workers": a.workers, "loader_items": a.items}
    for is_224 in (False, True):
        key = "224" if is_224 else "640x480"
        res["device"][key] = d = device_time(is_224, a.bs, a.iters)
        print("%s device: %.3f ms per call (median of %d, CUDA events), %.3f ms in the two kernels, %d items"
              % (key, d["ms_per_call_median"], d["calls"], d["ms_per_call_kernels"], d["items"]))
    with tempfile.TemporaryDirectory() as root:
        path = os.path.join(root, "nyu_data.zip")
        write_zip(path, a.items)
        for is_224 in (False, True):
            key = "224" if is_224 else "640x480"
            r = loader_rate(path, is_224, a.bs, a.workers, torch.device("cuda", 0))
            res["loader_items_per_s"][key] = r
            print("%s loader, %d workers: %.1f items/s on the device path (%.1f without its device call), %.1f items/s "
                  "on the host path" % (key, a.workers, r["device"], r["loader_only"], r["host"]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "nyu_inputs_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
