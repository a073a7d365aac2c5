"""Pin oracle.kitti_gt against the UNMODIFIED reference KITTI/kitti_utils.py and KITTI/export_gt_depth.py, and write
tests/golden/kitti_gt_*.npz.

Runs only where the reference checkout exists.  The reference needs two shims on current numpy, both declared here and
nowhere else: ``np.int = int`` (kitti_utils.py:92) and, for the export script, an ``np.array`` that makes a 1-D object
array of maps of different sizes, as numpy before 1.24 did (export_gt_depth.py:61).
  * calibration: KITTI-format files for five dates and their rectified sizes, and toy ones with small integer entries
    (focal 2, so exact half-pixel ties are reachable; one with T_z = -1 puts x < 1 behind the camera; 8x1 and 1x6
    images); the reference's P (P_rect . R_cam2rect . velo2cam, its read_calib_file) and sizes are stored;
  * engineered scans (points made by inverting P for chosen pixels and depths): one pixel hit in every order, the
    (y, W-1) / (y+1, 0) group collision either side first in groups of 2 and 3, pixel (0, 0), points behind the camera
    inside the image, x = +-0.0, exact .5 ties, NaN / inf in each coordinate, an empty scan, a scan with nothing in the
    image, H = 1 and W = 1, and thinned synthetic scans at the five dates: the oracle equals generate_depth_map bit for
    bit, for cams 2 and 3 and both vel_depth, and its projection equals np.dot(P, velo.T) on every point;
  * full size: seeded ~120k-point scans (oracle.kitti_gt.synthetic_scan) at the five dates, both cams and vel_depth:
    the oracle equals the reference and the sha256 of the reference's maps is stored;
  * end to end: export_gt_depths_kitti on a fake KITTI tree (oracle.kitti_gt.write_tree), both splits; the ``data``
    of the written gt_depths.npz is stored frame by frame.

Usage:  python -m oracle.pin_kitti_gt
"""
import hashlib
import itertools
import os
import sys
import tempfile
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_gt as og                                               # noqa: E402

REF_KITTI = "/root/reference/KITTI"
GOLDEN = os.path.join(REPO, "tests", "golden")
CAMS = (2, 3)
FULL_SEEDS = {"2011_09_26": 101, "2011_09_28": 102, "2011_09_29": 103, "2011_09_30": 104, "2011_10_03": 105}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def reference():
    np.int = int                                          # shim: kitti_utils.py:92's alias, removed in numpy 1.24
    sys.path.insert(0, REF_KITTI)
    import kitti_utils
    return kitti_utils


def sparse(depth):
    """flat indices and values of the pixels whose bits are not +0.0"""
    flat = depth.reshape(-1)
    idx = np.nonzero(flat.view(np.int64) != 0)[0]
    return idx.astype(np.int32), flat[idx]


def dense(idx, val, shape):
    out = np.zeros(int(np.prod(shape)), np.float64)
    out[idx] = val
    return out.reshape(shape)


# ----------------------------------------------------------------------------------------------------- engineered scans
def points(P, spec):
    """spec: (x, U, V[, reflectance]) with (U, V) the image coordinates before rint - 1 -> (M, 4) float32"""
    out = []
    for s in spec:
        x, U, V = s[:3]
        y, z = og.on_pixel(P, x, U, V)
        out.append((x, y, z, s[3] if len(s) > 3 else 0.5))
    return np.array(out, np.float32).reshape(-1, 4)


def engineered(calibs):
    """{case: (calib name, (M, 4) float32 points)}; toy coordinates are computed for camera 2"""
    P = {name: og.velo_to_image(og.read_calib_text(t[0]), og.read_calib_text(t[1]), 2)[0] for name, t in calibs.items()}
    toy, back = P["toy"], P["toy_back"]
    cases = {}
    perms = list(itertools.permutations((2.0, 4.0, 6.0)))
    spec = [(perm[r], 1 + k % 8, 1 + k // 8 + 2) for r in range(3) for k, perm in enumerate(perms)]
    spec += [(5.0, 8, 6), (5.0, 8, 6), (3.0, 8, 6), (3.0, 8, 6)]             # equal depths on one pixel
    cases["orders"] = ("toy", points(toy, spec))
    spec = []
    for row, (first, depths) in enumerate([("end", (4.0, 2.0)), ("start", (4.0, 2.0)), ("end", (2.0, 6.0, 4.0)),
                                           ("start", (6.0, 4.0, 2.0)), ("end", (6.0, 2.0, 2.0))]):
        sides = [(8, row + 1), (1, row + 2)]                                     # pixel (row, 7) and (row + 1, 0)
        if first == "start":
            sides = sides[::-1]
        for k, x in enumerate(depths):
            U, V = sides[k % 2]
            spec.append((x, U, V))
    cases["wrap"] = ("toy", points(toy, spec))
    cases["origin"] = ("toy", points(toy, [(4.0, 1, 1), (2.0, 1, 1), (6.0, 1, 1), (3.0, 2, 1), (1.0, 1, 2)]))
    spec = [(0.5, 2, 2), (2.0, 2, 2), (3.0, 4, 3), (0.25, 4, 3), (0.75, 6, 4), (0.5, 8, 6), (0.5, 1, 5),
            (2.0, 1, 5), (3.0, 3, 5)]                                            # q2 = x - 1 < 0 for x < 1
    cases["behind"] = ("toy_back", points(back, spec))
    spec = [(0.0, 2, 2), (-0.0, 2, 2), (-0.0, 3, 2), (0.0, 3, 2), (0.0, 4, 2), (-0.0, 4, 2), (0.0, 4, 2),
            (-0.0, 5, 3), (3.0, 5, 3), (3.0, 6, 3), (-0.0, 6, 3), (-0.0, 7, 4), (0.0, 2, 5), (-0.0, 8, 5),
            (0.0, 1, 6), (0.5, 8, 6), (-0.0, 8, 6)]
    cases["zeros"] = ("toy_back", points(back, spec))
    spec = [(4.0, U, V) for U in (-0.5, 0.5, 1.5, 2.5, 3.5, 4.5, 7.5, 8.5, 9.5) for V in (0.5, 1.5, 5.5, 6.5)]
    spec += [(2.0, U, 2.5) for U in (1.5, 2.5, 3.5)]
    cases["ties"] = ("toy", points(toy, spec))
    nf = points(toy, [(4.0, 2, 2), (4.0, 3, 3), (2.0, 3, 3), (4.0, 4, 4), (4.0, 5, 5, np.nan), (4.0, 6, 2, np.inf)])
    bad = []
    for c in range(3):
        for v in (np.nan, np.inf, -np.inf):
            p = points(toy, [(2.0, 3, 3)])[0].copy()
            p[c] = v
            bad.append(p)
    cases["nonfinite"] = ("toy", np.concatenate([nf[:2], np.array(bad, np.float32), nf[2:]]))
    cases["empty"] = ("toy", np.zeros((0, 4), np.float32))
    out = points(toy, [(4.0, -3, 2), (4.0, 2, 20), (4.0, 0.4, 2), (4.0, 9.5, 2), (4.0, 3, 0.49)])
    out = np.concatenate([out, np.array([[-1.0, 0.0, 0.0, 0.5], [-0.5, 0.2, 0.1, 0.5]], np.float32)])
    cases["outside"] = ("toy", out)
    cases["h1"] = ("toy_h1", points(P["toy_h1"], [(4.0, 1, 1), (2.0, 8, 1), (3.0, 1, 1), (2.0, 4, 1), (5.0, 4, 1),
                                                  (1.0, 2, 1), (2.0, 2, 0.6)]))
    cases["w1"] = ("toy_w1", points(P["toy_w1"], [(4.0, 1, 3), (2.0, 1, 1), (3.0, 1, 6), (1.5, 1, 3), (5.0, 1, 1),
                                                  (4.0, 1, 2)]))
    for k, (name, (W, H)) in enumerate(sorted(og.DATES.items())):
        Pd = P[name]
        spec = [(10.0, 1, 1), (12.0, 1, 1), (9.0, W, 11), (8.0, 1, 12), (11.0, 1, 13), (7.0, W, 12), (6.0, W, 12),
                (20.0, 600, 200), (15.0, 600, 200), (30.0, 600, 200), (0.1, 300, 150), (0.2, 300, 150),
                (5.0, 300, 150), (0.0, 400, 180), (-0.0, 400, 180)]
        pts = np.concatenate([points(Pd, spec), og.small_scan(300 + k, 3000)])
        cases["date_" + name] = (name, pts)
    return cases


# ----------------------------------------------------------------------------------------------------- end to end
class _RaggedNumpy(types.ModuleType):
    """numpy, with np.array making a 1-D object array of arrays of different shapes, as numpy < 1.24 did"""

    def __init__(self):
        super().__init__("numpy")

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def array(obj, *a, **k):
        try:
            return np.array(obj, *a, **k)
        except ValueError:
            out = np.empty(len(obj), dtype=object)
            for i, v in enumerate(obj):
                out[i] = v
            return out


def export_reference(calibs, split):
    """the reference script's gt_depths.npz ``data`` for the fake tree, as a list of float32 maps and its form"""
    import export_gt_depth
    with tempfile.TemporaryDirectory() as root:
        data_path = os.path.join(root, "kitti")
        lines = og.write_tree(data_path, calibs) if split == "eigen" else og.write_benchmark_tree(data_path)
        script_dir = os.path.join(root, "KITTI")
        os.makedirs(os.path.join(script_dir, "splits", split))
        with open(os.path.join(script_dir, "splits", split, "test_files.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
        export_gt_depth.__file__ = os.path.join(script_dir, "export_gt_depth.py")   # where it finds splits/
        export_gt_depth.np = _RaggedNumpy()
        argv = sys.argv
        sys.argv = ["export_gt_depth.py", "--data_path", data_path, "--split", split]
        try:
            export_gt_depth.export_gt_depths_kitti()
        finally:
            sys.argv = argv
        with np.load(os.path.join(script_dir, "splits", split, "gt_depths.npz"), allow_pickle=True) as f:
            data = f["data"]
    return data


def main():
    ku = reference()
    calibs = og.make_calibs()
    out_calib, parsed = {"names": np.array(sorted(calibs))}, {}
    with tempfile.TemporaryDirectory() as root:
        for name, texts in calibs.items():
            d = os.path.join(root, name)
            og.write_calib(d, texts)
            cam2cam = ku.read_calib_file(os.path.join(d, "calib_cam_to_cam.txt"))
            velo2cam = ku.read_calib_file(os.path.join(d, "calib_velo_to_cam.txt"))
            out_calib[name + "/cam_to_cam"], out_calib[name + "/velo_to_cam"] = np.array(texts[0]), np.array(texts[1])
            # generate_depth_map's lines 58-68, on the reference's parse
            Rt = np.vstack((np.hstack((velo2cam["R"].reshape(3, 3), velo2cam["T"][..., np.newaxis])),
                            np.array([0, 0, 0, 1.0])))
            R_cam2rect = np.eye(4)
            R_cam2rect[:3, :3] = cam2cam["R_rect_00"].reshape(3, 3)
            for cam in CAMS:
                P = np.dot(np.dot(cam2cam["P_rect_0%d" % cam].reshape(3, 4), R_cam2rect), Rt)
                out_calib["%s/P%d" % (name, cam)] = P
                mine = og.velo_to_image(og.read_calib_text(texts[0]), og.read_calib_text(texts[1]), cam)
                assert np.array_equal(mine[0].view(np.int64), P.view(np.int64)), (name, cam)
            size = cam2cam["S_rect_02"][::-1].astype(np.int32)
            out_calib[name + "/size"] = size
            parsed[name] = (d, {cam: out_calib["%s/P%d" % (name, cam)] for cam in CAMS}, tuple(int(v) for v in size))

        def check(name, pts, what):
            d, Ps, (H, W) = parsed[name]
            path = os.path.join(root, "scan.bin")
            pts.tofile(path)
            maps = {}
            for cam in CAMS:
                velo = pts[pts[:, 0] >= 0].copy()
                velo[:, 3] = 1.0
                q_ref = np.dot(Ps[cam], velo.T).T
                assert np.array_equal(og.project(velo, Ps[cam]).view(np.int64), q_ref.view(np.int64)), (what, cam)
                for vd in (0, 1):
                    ref = ku.generate_depth_map(d, path, cam, bool(vd))
                    mine = og.depth_map(pts, Ps[cam], H, W, bool(vd))
                    bad = int((ref.view(np.int64) != mine.view(np.int64)).sum())
                    if bad:
                        raise SystemExit("oracle.kitti_gt differs from generate_depth_map on %s cam %d vel_depth %d: "
                                         "%d pixels" % (what, cam, vd, bad))
                    maps[cam, vd] = ref
            return maps

        out_cases = {}
        cases = engineered(calibs)
        out_cases["cases"] = np.array(sorted(cases))
        for case, (name, pts) in sorted(cases.items()):
            maps = check(name, pts, case)
            out_cases[case + "/calib"], out_cases[case + "/points"] = np.array(name), pts
            for (cam, vd), ref in maps.items():
                idx, val = sparse(ref)
                out_cases["%s/%d/%d/index" % (case, cam, vd)], out_cases["%s/%d/%d/value" % (case, cam, vd)] = idx, val
            nz = {k: int((v != 0).sum()) for k, v in maps.items()}
            print("%-18s %-11s %6d points, nonzero pixels %s" % (case, name, pts.shape[0], nz))

        out_full = {"dates": np.array(sorted(FULL_SEEDS))}
        for name, seed in sorted(FULL_SEEDS.items()):
            pts = og.synthetic_scan(seed)
            maps = check(name, pts, "full " + name)
            out_full[name + "/seed"] = np.array(seed)
            out_full[name + "/points_sha256"] = np.array(digest(pts))
            for (cam, vd), ref in maps.items():
                out_full["%s/%d/%d/sha256" % (name, cam, vd)] = np.array(digest(ref))
            print("full %s: %d points, %d pixels (cam 2, vel_depth)" % (name, pts.shape[0], int((maps[2, 1] > 0).sum())))

    out_export = {}
    for split in ("eigen", "eigen_benchmark"):
        data = export_reference(calibs, split)
        out_export[split + "/object"] = np.array(data.dtype == object)
        out_export[split + "/frames"] = np.array(len(data))
        for i, m in enumerate(data):
            assert m.dtype == np.float32
            out_export["%s/%d" % (split, i)] = m
        if split == "eigen":
            for i, (date, drive, frame, seed, n) in enumerate(og.e2e_frames()):
                _, Ps, (H, W) = parsed[date]
                mine = og.depth_map(og.small_scan(seed, n), Ps[2], H, W, True).astype(np.float32)
                assert np.array_equal(mine.view(np.int32), data[i].view(np.int32)), (split, i)
        print("export %s: %d frames, object array %s" % (split, len(data), data.dtype == object))

    for name, arrays in (("calib", out_calib), ("cases", out_cases), ("full", out_full), ("export", out_export)):
        path = os.path.join(GOLDEN, "kitti_gt_%s.npz" % name)
        np.savez_compressed(path, **arrays)
        print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
