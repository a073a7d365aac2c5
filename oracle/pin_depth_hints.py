"""Pin oracle.sgbm and oracle.depth_hints against OpenCV and the UNMODIFIED reference script, and write
tests/golden/kitti_depth_hints*.npz.

Runs only where cv2 (the pinned version, oracle.depth_hints.CV2_VERSION) and the reference checkout exist.
  * matcher: oracle.sgbm.compute equals cv2.StereoSGBM_create(...).compute bit for bit on every pair of the fixtures,
    for the twelve matchers of the script, both sides, and on stage-isolation variants (uniquenessRatio 0,
    speckleWindowSize 0, disp12MaxDiff 5 and -1, other P1 / P2 and preFilterCap), the smallest widths cv2 accepts, one
    row, and a pair made from the reference's assets/kitti_test_sample.jpg (stored, as GPU machines cannot read it);
    cv2 must refuse the next width down;
  * fusion: the reference's DepthHintDataset.__getitem__ (its cv2 matchers; ``pil_loader`` returns the stored views,
    whose size the resize keeps) and the fusion lines of run() on the CPU in float32 and float64: on every pixel the
    float64 run's choice is within 1e-12 (relative) of oracle.depth_hints' fp64-mode least error and its depth is that
    matcher's depth, bit for bit; where it differs from the oracle's first minimum (a near-tie that the reference's own
    float64 rounding decides) the pixel is counted (oracle.depth_hints.check_fp64); the contract mode's index flips
    against the float32 run are recorded per case;
  * full size (320x1024, two seeded pairs, both sides): sha256 of cv2's twelve maps and of the contract fusion's depth.

Usage:  python -m oracle.pin_depth_hints
"""
import argparse
import hashlib
import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import depth_hints as odh                                           # noqa: E402
from oracle import sgbm                                                         # noqa: E402

REF_KITTI = "/root/reference/KITTI"
REF_SAMPLE = "/root/reference/assets/kitti_test_sample.jpg"
GOLDEN = os.path.join(REPO, "tests", "golden")
VARIANTS = {
    "unique0_speckle0_lr5": dict(uniquenessRatio=0, speckleWindowSize=0, disp12MaxDiff=5),
    "speckle0": dict(speckleWindowSize=0),
    "lr5": dict(disp12MaxDiff=5),
    "lr_off": dict(disp12MaxDiff=-1),
    "lr1": dict(disp12MaxDiff=1),
    "p1_8_p2_32": dict(P1=8, P2=32),
    "p1_200_p2_3000": dict(P1=200, P2=3000),
    "cap15": dict(preFilterCap=15),
    "cap31": dict(preFilterCap=31),
}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cv2_maps(base, lookup, reverse, **kw):
    """cv2's twelve maps (12, H, W) int16, as the script calls them (mirrored views for a right base view)"""
    import cv2
    out = []
    for nd, bs in sgbm.MATCHERS:
        p = dict(sgbm.HINT_PARAMS, minDisparity=0, numDisparities=nd, blockSize=bs)
        p.update(kw)
        m = cv2.StereoSGBM_create(**p)
        if reverse:
            out.append(m.compute(np.ascontiguousarray(base[:, ::-1]), np.ascontiguousarray(lookup[:, ::-1]))[:, ::-1])
        else:
            out.append(m.compute(base, lookup))
    return np.ascontiguousarray(np.stack(out))


def check_oracle(base, lookup, reverse, maps, what, **kw):
    for (nd, bs), ref in zip(sgbm.MATCHERS, maps):
        got = sgbm.compute_side(base, lookup, nd, bs, reverse, **dict(sgbm.HINT_PARAMS, **kw))
        bad = int((got != ref).sum())
        if bad:
            raise SystemExit("oracle.sgbm differs from cv2 on %s, numDisparities %d blockSize %d: %d pixels"
                             % (what, nd, bs, bad))


def _reference():
    from PIL import Image
    if not hasattr(Image, "ANTIALIAS"):
        Image.ANTIALIAS = Image.LANCZOS
    sys.path.insert(0, REF_KITTI)
    import precompute_depth_hints as ref
    import layers
    return ref, layers


def run_reference(left, right, side, dtype):
    """the script's best_depth (1, H, W) and best_index for one view of a stored pair, on the CPU in dtype"""
    from PIL import Image
    ref, layers = _reference()
    H, W, _ = left.shape
    images = {"image_02": left, "image_03": right}
    ref.pil_loader = lambda path: Image.fromarray(images[path.split(os.sep)[-3]])
    ds = ref.DepthHintDataset("data", ["seq 0 %s" % side], H, W, "save", True)
    data = ds[0]
    data = {k: v.to(dtype) for k, v in data.items()}
    cam_to_world = layers.BackprojectDepth(12, H, W).to(dtype)
    world_to_cam = layers.Project3D(12, H, W)
    F = torch.nn.functional
    world_points = cam_to_world(data["depths"], data["invK"])
    cam_pix = world_to_cam(world_points, data["K"], data["T"])
    sample = F.grid_sample(data["lookup_image"], cam_pix, padding_mode="border")
    losses = ref.compute_reprojection_loss(sample, data["base_image"])
    best_index = torch.argmin(losses, dim=0)
    best_depth = torch.gather(data["depths"], dim=0, index=best_index)
    return best_depth.numpy(), best_index.numpy()


def pin_fusion(left, right, side, maps, out, key):
    base, lookup, rev = odh.views(left, right, side)
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        d, i = run_reference(left, right, side, dt)
        out["%s/%s/ref_%s_depth" % (key, side, tag)] = d.astype(np.float32)
        out["%s/%s/ref_%s_index" % (key, side, tag)] = i.astype(np.int8)
    d64, i64, errs = odh.fuse(base[None], lookup[None], maps[:, None], [rev], mode="fp64")
    ref_d = out["%s/%s/ref_f64_depth" % (key, side)]
    ref_i = out["%s/%s/ref_f64_index" % (key, side)].astype(np.int64)
    ties = odh.check_fp64(errs[:, 0], odh.depths(maps, odh.cameras(*base.shape[:2], [rev])[0][0, 0, 0]), i64[0, 0],
                          ref_i[0], ref_d[0])
    if ties is None:
        raise SystemExit("fp64 fusion differs from the float64 reference on %s/%s" % (key, side))
    out["%s/%s/ties_f64" % (key, side)] = np.int64(ties)
    dc, ic, _ = odh.fuse(base[None], lookup[None], maps[:, None], [rev], mode="contract")
    flips = int((ic[0] != out["%s/%s/ref_f32_index" % (key, side)]).sum())
    out["%s/%s/flips_f32" % (key, side)] = np.int64(flips)
    out["%s/%s/contract_depth" % (key, side)] = dc[0]
    out["%s/%s/contract_index" % (key, side)] = ic[0].astype(np.int8)
    print("  fusion %s/%s: fp64 agrees (%d near-ties decided otherwise), %d argmin flips against float32"
          % (key, side, ties, flips))


def main():
    argparse.ArgumentParser(description=__doc__.split("\n")[0]).parse_args()
    import cv2
    if cv2.__version__ != odh.CV2_VERSION:
        raise SystemExit("the fixtures pin cv2 %s; this is cv2 %s: not rewriting them" % (odh.CV2_VERSION, cv2.__version__))
    files = {}
    for name, (seed, H, W) in odh.SMALL.items():
        out = {"cv2_version": np.array(cv2.__version__)}
        left, right = odh.make_pair(seed, H, W)
        out["%s/left" % name], out["%s/right" % name] = left, right
        for side in "lr":
            base, lookup, rev = odh.views(left, right, side)
            maps = cv2_maps(base, lookup, rev)
            check_oracle(base, lookup, rev, maps, "%s/%s" % (name, side))
            assert np.array_equal(maps[4:8], maps[8:12]), "blockSize 2 and 3 differ"
            out["%s/%s/maps" % (name, side)] = maps
            pin_fusion(left, right, side, maps, out, name)
        files["kitti_depth_hints_%s.npz" % name] = out
        print("case %s: twelve matchers bit-equal, both sides" % name)

    st = {"cv2_version": np.array(cv2.__version__)}
    left, right = odh.make_pair(606, 48, 224)
    st["stages/left"], st["stages/right"] = left, right
    for vname, kw in VARIANTS.items():
        maps = cv2_maps(left, right, False, **kw)
        check_oracle(left, right, False, maps, vname, **kw)
        st["stages/%s" % vname] = maps
    # the smallest widths cv2 accepts (and its refusal of the next one down), and a single row
    for nd in sgbm.NUM_DISPARITIES:
        for bs in sgbm.BLOCK_SIZES:
            w = sgbm.min_width(nd, bs)
            l2, r2 = odh.make_pair(700 + nd + bs, 24, w)
            p = dict(sgbm.HINT_PARAMS, minDisparity=0, numDisparities=nd, blockSize=bs)
            ref = cv2.StereoSGBM_create(**p).compute(l2, r2)
            assert np.array_equal(sgbm.compute(l2, r2, nd, bs, **sgbm.HINT_PARAMS), ref), ("min width", nd, bs)
            try:
                cv2.StereoSGBM_create(**p).compute(l2[:, :-1].copy(), r2[:, :-1].copy())
            except cv2.error:
                pass
            else:
                raise SystemExit("cv2 accepted width %d for numDisparities %d blockSize %d" % (w - 1, nd, bs))
            st["minw/%d/%d/left" % (nd, bs)], st["minw/%d/%d/right" % (nd, bs)], st["minw/%d/%d/disp" % (nd, bs)] = \
                l2, r2, ref
    l1, r1 = odh.make_pair(808, 8, 256)
    maps = cv2_maps(l1[:1].copy(), r1[:1].copy(), False)
    check_oracle(l1[:1], r1[:1], False, maps, "one row")
    st["row/left"], st["row/right"], st["row/maps"] = l1[:1], r1[:1], maps
    from PIL import Image
    photo = np.asarray(Image.open(REF_SAMPLE).convert("RGB"))
    sl, sr = odh.sample_pair(photo, 96, 320)
    st["sample/left"], st["sample/right"] = sl, sr
    for side in "lr":
        base, lookup, rev = odh.views(sl, sr, side)
        maps = cv2_maps(base, lookup, rev)
        check_oracle(base, lookup, rev, maps, "sample/%s" % side)
        st["sample/%s/maps" % side] = maps
        pin_fusion(sl, sr, side, maps, st, "sample")
    files["kitti_depth_hints_stages.npz"] = st
    print("stage isolation, minimum widths, one row and the photo pair: bit-equal")

    full = {"cv2_version": np.array(cv2.__version__)}
    for name, (seed, H, W) in odh.FULL.items():
        left, right = odh.make_pair(seed, H, W)
        for side in "lr":
            base, lookup, rev = odh.views(left, right, side)
            maps = cv2_maps(base, lookup, rev)
            full["%s/%s/maps_sha256" % (name, side)] = np.array([digest(m) for m in maps])
            d, i, _ = odh.fuse(base[None], lookup[None], maps[:, None], [rev], mode="contract")
            full["%s/%s/depth_sha256" % (name, side)] = np.array(digest(d))
            full["%s/%s/index_sha256" % (name, side)] = np.array(digest(i.astype(np.int8)))
        print("full size %s: digests" % name)
    # the CPU test's one full-size matcher: the oracle itself against cv2's digest
    left, right = odh.make_pair(odh.FULL["full0"][0], 320, 1024)
    assert digest(sgbm.compute(left, right, 64, 1, **sgbm.HINT_PARAMS)) == full["full0/l/maps_sha256"][0]
    files["kitti_depth_hints_full.npz"] = full

    for name, keys in files.items():
        path = os.path.join(GOLDEN, name)
        with open(path, "wb") as f:
            np.savez_compressed(f, **keys)
        print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
