"""Shared by the KITTI input tests: rebuild the items of a tests/golden/kitti_inputs_*.npz fixture (its views are
oracle.kitti_inputs.synthetic_view of stored seeds) and compare a dict against the fixture's digests."""
import ast
import hashlib
import os

import numpy as np

from oracle import kitti_inputs as oki

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("train640", "train1024", "eval640")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load(name):
    with np.load(os.path.join(GOLDEN, "kitti_inputs_%s.npz" % name)) as f:
        fx = {k: f[k] for k in f.files}
    fx["config"] = ast.literal_eval(str(fx["config"]))
    fx["keys"] = [ast.literal_eval(str(k)) for k in fx["keys"]]
    return fx


def items(fx):
    """the fixture's items as KittiInputsDataset returns them"""
    cfg = fx["config"]
    out = []
    for n in range(len(fx["lines"])):
        views = {f: oki.synthetic_view(*map(int, fx["views"][n, k])) for k, f in enumerate(cfg["frame_idxs"])}
        it = {"views": views, "do_color_aug": bool(fx["do_color_aug"][n]), "do_flip": bool(fx["do_flip"][n]),
              "jitter": (tuple(map(float, fx["factors"][n])), tuple(map(int, fx["order"][n])))
              if fx["do_color_aug"][n] else None,
              "side": str(fx["side"][n]), "image_path": str(fx["image_path"][n])}
        if cfg["use_depth_hints"] and "s" in cfg["frame_idxs"]:
            it["hint"] = oki.synthetic_hint(*map(int, fx["hint_src"][n])) if fx["hint_found"][n] else None
        out.append(it)
    return out


def mismatches(fx, per_item):
    """keys whose digest differs from the fixture's, over per_item(n) -> {key: numpy array} ("" in the fixture: the
    reference has no such key for that item)"""
    bad = []
    for n in range(len(fx["lines"])):
        got = per_item(n)
        for k, want in zip(fx["keys"], fx["digests"][n]):
            if want == "":
                continue
            if k not in got or digest(got[k]) != want:
                bad.append((n, k))
    return bad
