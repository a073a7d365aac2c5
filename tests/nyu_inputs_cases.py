"""Shared by the NYUv2 input tests: rebuild the items of a tests/golden/nyu_inputs_*.npz fixture (its views are
oracle.nyu_inputs.synthetic_image / synthetic_depth of stored seeds) and compare outputs against its digests."""
import ast
import hashlib
import os

import numpy as np

from oracle import nyu_inputs as oni

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("640_bicubic", "224_bicubic", "640_nearest", "224_nearest")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load(name):
    with np.load(os.path.join(GOLDEN, "nyu_inputs_%s.npz" % name)) as f:
        fx = {k: f[k] for k in f.files}
    fx["config"] = ast.literal_eval(str(fx["config"]))
    return fx


def items(fx):
    """the fixture's items as NyuInputsDataset returns them"""
    out = []
    for n in range(len(fx["view"])):
        seed = int(fx["view"][n])
        gamma = float(fx["gamma"][n])
        out.append({"image": oni.synthetic_image(seed), "depth": oni.synthetic_depth(seed),
                    "flip": bool(fx["flip"][n]), "perm": int(fx["perm"][n]),
                    "gamma": None if np.isnan(gamma) else gamma})
    return out


def mismatches(fx, per_item):
    """(item, key) whose digest differs from the reference's, over per_item(n) -> {"image", "depth"} numpy arrays"""
    bad = []
    for n in range(len(fx["view"])):
        got = per_item(n)
        for k, want in zip(("image", "depth"), fx["digests"][n]):
            if digest(got[k]) != want:
                bad.append((n, k))
    return bad
