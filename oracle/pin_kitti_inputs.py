"""Pin oracle.kitti_inputs against the installed Pillow and the UNMODIFIED reference ``KITTIRAWDataset.__getitem__``,
and write tests/golden/kitti_inputs_*.npz.

Runs only where the reference checkout exists.  Three shims make the reference run with the installed packages, and
nothing else is changed:
  * ``Image.ANTIALIAS = Image.LANCZOS`` (removed in Pillow 10);
  * a ``skimage`` stub (``kitti_dataset.py`` imports ``skimage.transform``; ``__getitem__`` never uses it);
  * torchvision 0.8.2's ``ColorJitter.get_params``, which returns a Compose of the four adjustments (installed
    torchvision's ``TF.adjust_*``) after ``random.shuffle``; newer versions return a tuple the reference cannot call.

For each case a synthetic KITTI tree is written (views at the five raw sizes, ``.npy`` hints, some missing) and, from
one seed, the reference dataset and ``KittiInputsDataset`` are built and indexed: their draws must agree, and
``oracle.kitti_inputs.expected`` of our items must equal the reference's dict on every key, bit for bit.  The fixture
cases use PNG views, so the decoded views are ``synthetic_view(seed)`` exactly and tests can rebuild them; a JPEG tree
checks the same with the reference's own decode.  The fixtures hold each item's views (seed, size), draws and hint,
sha256 digests of every reference tensor, and the uint8 planes (x 255) of the scale-3 images.

Usage:  python -m oracle.pin_kitti_inputs
"""
import hashlib
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_inputs as oki                                          # noqa: E402
from wavelet_monodepth_b200 import kitti_inputs as ki                             # noqa: E402

REF_KITTI = "/root/reference/KITTI"
GOLDEN = os.path.join(REPO, "tests", "golden")
SEQUENCES = ["2011_09_%02d/2011_09_%02d_drive_%04d_sync" % (26 + k, 26 + k, k + 1) for k in range(5)]

# name: (height, width, frame_idxs, target_scales, is_train, use_depth_hints, seed, items)
CASES = {
    "train640": (192, 640, [0, "s"], [0, 1, 2, 3], True, True, 7, 12),
    "train1024": (320, 1024, [0, -1, 1, "s"], [0, 1, 2, 3], True, True, 11, 6),
    "eval640": (192, 640, [0], [0, 1, 2, 3], False, False, 5, 5),
}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def view_seed(seq, frame, cam):
    return 1000 * seq + 10 * frame + cam


def hint_shape(seq):
    return (188 + seq, 621 - 3 * seq)


def lines_of(n, seed):
    rng = np.random.default_rng(seed)
    return ["%s %d %s" % (SEQUENCES[k % 5], int(rng.integers(1, 8)), "lr"[int(rng.integers(0, 2))]) for k in range(n)]


def missing(line):
    """every third (sequence, frame) has no hint file"""
    seq, frame, _ = line.split()
    return (SEQUENCES.index(seq) + int(frame)) % 3 == 0


def write_tree(root, lines, frame_idxs, ext):
    from PIL import Image
    for line in lines:
        seq, frame, side = line.split()
        k, frame = SEQUENCES.index(seq), int(frame)
        h, w = oki.RAW_SIZES[k]
        for f in frame_idxs:
            cam = {"l": 2, "r": 3}[{"r": "l", "l": "r"}[side] if f == "s" else side]
            fr = frame if f == "s" else frame + f
            path = os.path.join(root, seq, "image_0%d" % cam, "data", "%010d%s" % (fr, ext))
            os.makedirs(os.path.dirname(path), exist_ok=True)
            if not os.path.exists(path):
                img = Image.fromarray(oki.synthetic_view(view_seed(k, fr, cam), h, w))
                img.save(path, quality=90) if ext == ".jpg" else img.save(path)
        if not missing(line):
            path = os.path.join(root, "depth_hints", seq, "image_02" if side == "l" else "image_03", "%010d.npy" % frame)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.save(path, oki.synthetic_hint(view_seed(k, frame, 9), *hint_shape(k))[None])


def shim_reference():
    """the three shims; returns KITTIRAWDataset"""
    from PIL import Image
    import torchvision.transforms as T
    import torchvision.transforms.functional as TF
    Image.ANTIALIAS = Image.LANCZOS
    sk = types.ModuleType("skimage")
    sk.transform = types.ModuleType("skimage.transform")
    sys.modules.update({"skimage": sk, "skimage.transform": sk.transform})

    def get_params(brightness, contrast, saturation, hue):           # torchvision 0.8.2
        transforms = []
        if brightness is not None:
            b = random.uniform(brightness[0], brightness[1])
            transforms.append(T.Lambda(lambda img: TF.adjust_brightness(img, b)))
        if contrast is not None:
            c = random.uniform(contrast[0], contrast[1])
            transforms.append(T.Lambda(lambda img: TF.adjust_contrast(img, c)))
        if saturation is not None:
            s = random.uniform(saturation[0], saturation[1])
            transforms.append(T.Lambda(lambda img: TF.adjust_saturation(img, s)))
        if hue is not None:
            h = random.uniform(hue[0], hue[1])
            transforms.append(T.Lambda(lambda img: TF.adjust_hue(img, h)))
        random.shuffle(transforms)
        return T.Compose(transforms)

    T.ColorJitter.get_params = staticmethod(get_params)
    sys.modules.pop("datasets", None)
    sys.path.insert(0, REF_KITTI)
    from datasets.kitti_dataset import KITTIRAWDataset
    return KITTIRAWDataset


def run_case(KITTIRAWDataset, name, ext):
    height, width, frame_idxs, scales, is_train, hints, seed, n = CASES[name]
    lines = lines_of(n, seed)
    with tempfile.TemporaryDirectory() as root:
        root = root + "/"
        write_tree(root, lines, frame_idxs, ext)
        kw = dict(target_scales=scales, use_depth_hints=hints, is_train=is_train, img_ext=ext)
        random.seed(seed)
        ref = KITTIRAWDataset(root, lines, height, width, frame_idxs, **kw)
        ref_items = [ref[i] for i in range(n)]
        random.seed(seed)
        ours = ki.KittiInputsDataset(root, lines, height, width, frame_idxs, **kw)
        our_items = [ours[i] for i in range(n)]
        if hints:
            assert (ours.with_hints, ours.without_hints) == (ref.with_hints, ref.without_hints)
    keys = sorted({k for r in ref_items for k in r if k != "image_path"}, key=repr)
    digests, planes = [], []
    for it, r in zip(our_items, ref_items):
        assert it["image_path"] == r["image_path"], (it["image_path"], r["image_path"])
        exp = oki.expected(it["views"], (it["do_color_aug"], it["do_flip"], it["jitter"]), it["side"], it.get("hint"),
                           height, width, scales, hints)
        got = {k: v for k, v in r.items() if k != "image_path"}
        assert set(exp) == set(got), set(exp) ^ set(got)
        for k, v in got.items():
            assert np.array_equal(v.numpy(), exp[k]) and v.dtype == torch.from_numpy(exp[k]).dtype, (name, k)
        digests.append([digest(got[k].numpy()) if k in got else "" for k in keys])
        planes.append(np.stack([np.rint(got[("color_aug", f, 3)].numpy() * 255).astype(np.uint8) for f in frame_idxs]))
    return lines, our_items, keys, digests, planes


def main():
    KITTIRAWDataset = shim_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    for name in CASES:
        run_case(KITTIRAWDataset, name, ".jpg")
        print("%s: the reference on a JPEG tree equals the oracle on every key" % name)
        lines, items, keys, digests, planes = run_case(KITTIRAWDataset, name, ".png")
        height, width, frame_idxs, scales, is_train, hints, seed, n = CASES[name]
        views = []
        for line in lines:
            seq, frame, side = line.split()
            k, frame = SEQUENCES.index(seq), int(frame)
            row = []
            for f in frame_idxs:
                cam = {"l": 2, "r": 3}[{"r": "l", "l": "r"}[side] if f == "s" else side]
                fr = frame if f == "s" else frame + f
                row.append((view_seed(k, fr, cam),) + oki.RAW_SIZES[k])
            views.append(row)
        found = [it.get("hint") is not None for it in items]
        hint_src = [(view_seed(SEQUENCES.index(ln.split()[0]), int(ln.split()[1]), 9),)
                    + hint_shape(SEQUENCES.index(ln.split()[0])) for ln in lines]
        np.savez_compressed(
            os.path.join(GOLDEN, "kitti_inputs_%s.npz" % name),
            config=np.array(repr(dict(height=height, width=width, frame_idxs=frame_idxs, scales=scales,
                                      use_depth_hints=hints))),
            lines=np.array(lines), views=np.array(views, np.int64), side=np.array([ln.split()[2] for ln in lines]),
            do_color_aug=np.array([it["do_color_aug"] for it in items]),
            do_flip=np.array([it["do_flip"] for it in items]),
            factors=np.array([it["jitter"][0] if it["jitter"] else (0.0,) * 4 for it in items], np.float64),
            order=np.array([it["jitter"][1] if it["jitter"] else (-1,) * 4 for it in items], np.int64),
            hint_found=np.array(found), hint_src=np.array(hint_src, np.int64),
            image_path=np.array([it["image_path"] for it in items]),
            keys=np.array([repr(k) for k in keys]), digests=np.array(digests), planes=np.stack(planes))
        print("%s: wrote %d items; aug %d, flip %d, hints found %d / %d" % (
            name, len(items), sum(it["do_color_aug"] for it in items), sum(it["do_flip"] for it in items),
            sum(found), len(found)))


if __name__ == "__main__":
    main()
