"""Pin oracle.nyu_inputs against the installed Pillow and the UNMODIFIED reference ``NYUv2/data.py``, and write
tests/golden/nyu_inputs_*.npz.

Runs only where the reference checkout exists.  For each case (640x480 or ``is_224``, BICUBIC or NEAREST) a synthetic
``nyu_data.zip`` is written: seeded 640x480 RGB views and L depths (``synthetic_image`` / ``synthetic_depth``), saved
losslessly as PNG so that tests can rebuild them from the seeds, and the reference's ``nyu2_train.csv``.  Both
``loadZipToMem`` and ``load_zip_to_mem`` load it, and must agree.  Each dataset index is then read from the reference
``depthDatasetMemory`` with ``getDefaultTrainTransform(is_224)`` (or ``getNoTransform`` for the testing items) and from
``NyuInputsDataset``, each after ``random.seed`` of that item's draw seed: both must leave ``random`` in the same state,
and ``oracle.nyu_inputs.expected`` of our item must equal the reference's tensors bit for bit.  The draw seeds are
chosen so that every flip x swap combination and all six permutations occur.  A JPEG zip checks the same with the
reference's own decode.

ToTensor calls ``resize`` without a filter.  The installed Pillow defaults to BICUBIC; the NEAREST cases run the
reference with one declared shim, ``Image.resize``'s default filter set to NEAREST (the default of the Pillow 6.2.1
the reference pins).

The fixtures hold each item's view seed, draw seed and draws and sha256 digests of the reference's image and depth.

Usage:  python -m oracle.pin_nyu_inputs
"""
import contextlib
import hashlib
import io
import os
import random
import sys
import tempfile
import zipfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import nyu_inputs as oni                                            # noqa: E402
from wavelet_monodepth_b200 import nyu_inputs as ni                              # noqa: E402

REF_NYU = "/root/reference/NYUv2"
GOLDEN = os.path.join(REPO, "tests", "golden")

# name: (is_224, resample)
CASES = {"640_bicubic": (False, "bicubic"), "224_bicubic": (True, "bicubic"),
         "640_nearest": (False, "nearest"), "224_nearest": (True, "nearest")}
# the training items' (flip, permutation index or -1): every flip x swap combination and all six permutations
TRAIN_DRAWS = [(False, -1), (True, -1), (False, 0), (True, 1), (False, 2), (True, 3), (False, 4), (True, 5), (True, 0),
               (False, 5)]
TEST_ITEMS = 2
VIEW_SEED0 = 100


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def draw_seeds(start=0):
    """the least seeds from `start` whose draws give TRAIN_DRAWS in turn"""
    seeds, s = [], start
    for want in TRAIN_DRAWS:
        while oni.draws(True, random.Random(s))[:2] != want:
            s += 1
        seeds.append(s)
        s += 1
    return seeds


def row_names(k, ext):
    return "data/nyu2_train/scene_%02d/%d%s" % (k, k, ext), "data/nyu2_train/scene_%02d/%d_depth.png" % (k, k)


def write_zip(path, n, ext):
    """n items; item k is synthetic_image(VIEW_SEED0 + k) and synthetic_depth(VIEW_SEED0 + k)"""
    from PIL import Image
    rows = []
    with zipfile.ZipFile(path, "w") as zf:
        for k in range(n):
            img, dep = row_names(k, ext)
            buf = io.BytesIO()
            Image.fromarray(oni.synthetic_image(VIEW_SEED0 + k)).save(buf, "JPEG" if ext == ".jpg" else "PNG",
                                                                       **({"quality": 90} if ext == ".jpg" else {}))
            zf.writestr(img, buf.getvalue())
            buf = io.BytesIO()
            Image.fromarray(oni.synthetic_depth(VIEW_SEED0 + k)).save(buf, "PNG")
            zf.writestr(dep, buf.getvalue())
            rows.append("%s,%s" % (img, dep))
        zf.writestr("data/nyu2_train.csv", "\n".join(rows) + "\n")


@contextlib.contextmanager
def default_filter(resample):
    """the declared shim: Image.resize's default filter is NEAREST for the NEAREST cases"""
    from PIL import Image
    orig = Image.Image.resize
    if resample == "nearest":
        def resize(self, size, resample=None, *args, **kwargs):
            return orig(self, size, Image.NEAREST if resample is None else resample, *args, **kwargs)
        Image.Image.resize = resize
    try:
        yield
    finally:
        Image.Image.resize = orig


def reference():
    sys.modules.pop("data", None)
    sys.path.insert(0, REF_NYU)
    import data as ref_data
    return ref_data


def run_case(ref_data, name, ext):
    is_224, resample = CASES[name]
    seeds = draw_seeds()
    n = len(seeds) + TEST_ITEMS
    with tempfile.TemporaryDirectory() as root:
        path = os.path.join(root, "nyu_data.zip")
        write_zip(path, n, ext)
        with contextlib.redirect_stdout(io.StringIO()):
            data, rows = ref_data.loadZipToMem(path)
        ours_data, ours_rows = ni.load_zip_to_mem(path)
    assert ours_data == data and ours_rows == rows, "load_zip_to_mem differs from loadZipToMem"
    view_seed = {row_names(k, ext)[0]: VIEW_SEED0 + k for k in range(n)}
    out = []
    for i in range(n):
        is_train = i < len(seeds)
        seed = seeds[i] if is_train else 0
        transform = (ref_data.getDefaultTrainTransform(is_224=is_224) if is_train
                     else ref_data.getNoTransform(is_224=is_224))
        with default_filter(resample):
            random.seed(seed)
            r = ref_data.depthDatasetMemory(data, rows, transform=transform)[i]
        after = random.getstate()
        random.seed(seed)
        it = ni.NyuInputsDataset(data, rows, is_train=is_train)[i]
        assert random.getstate() == after, (name, i, "the draws differ")
        if is_train:
            assert (it["flip"], it["perm"]) == TRAIN_DRAWS[i], (name, i)
        exp = oni.expected(it["image"], it["depth"], it["flip"], it["perm"], it["gamma"], is_224, resample)
        for k in ("image", "depth"):
            got = r[k]
            assert got.dtype == torch.float32 and np.array_equal(got.numpy(), exp[k]), (name, i, k)
        out.append(dict(view=view_seed[rows[i][0]], is_train=is_train, seed=seed, flip=it["flip"], perm=it["perm"],
                        gamma=np.nan if it["gamma"] is None else it["gamma"],
                        digests=(digest(r["image"].numpy()), digest(r["depth"].numpy()))))
    return out


def main():
    ref_data = reference()
    os.makedirs(GOLDEN, exist_ok=True)
    for name in CASES:
        run_case(ref_data, name, ".jpg")
        print("%s: the reference on JPEG images equals the oracle on every item" % name)
        items = run_case(ref_data, name, ".png")
        is_224, resample = CASES[name]
        np.savez_compressed(
            os.path.join(GOLDEN, "nyu_inputs_%s.npz" % name),
            config=np.array(repr(dict(is_224=is_224, resample=resample))),
            view=np.array([it["view"] for it in items], np.int64),
            is_train=np.array([it["is_train"] for it in items]),
            seed=np.array([it["seed"] for it in items], np.int64),
            flip=np.array([it["flip"] for it in items]),
            perm=np.array([it["perm"] for it in items], np.int64),
            gamma=np.array([it["gamma"] for it in items], np.float64),
            digests=np.array([it["digests"] for it in items]))
        print("%s: 0 mismatches over %d items (%d training, %d testing); wrote nyu_inputs_%s.npz"
              % (name, len(items), sum(it["is_train"] for it in items), sum(not it["is_train"] for it in items), name))


if __name__ == "__main__":
    main()
