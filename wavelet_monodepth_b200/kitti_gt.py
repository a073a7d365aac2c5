"""KITTI's ground-truth depths on the device: ``KITTI/export_gt_depth.py`` as one batched command.

Before the Eigen split can be evaluated, the reference projects each test frame's velodyne scan into camera 2 with
``kitti_utils.generate_depth_map`` and saves the maps as ``splits/eigen/gt_depths.npz``.  Here the projection is
libwmd's ``wmd_velo_depth_f64`` (include/wmd_gt.h), the reference function bit for bit, for a batch of scans with
ragged point counts and mixed calibrations; the calibration is parsed and ``P`` formed on the host with numpy, exactly as
the reference does.

``generate_depth_maps`` is the batched device call: (N, Hmax, Wmax) fp64 maps on the device, which can go straight into
``kitti_eval.KittiDepthEvaluator``.  ``generate_depth_map`` is the reference function's signature for one scan.

    python -m wavelet_monodepth_b200.kitti_gt --data_path KITTI_RAW --split eigen|eigen_benchmark
        [--filenames splits/<split>/test_files.txt] [--output splits/<split>/gt_depths.npz] [--batch_size 16]
        [--num_workers 8]

run from the reference's ``KITTI/`` directory writes what the script writes there: ``np.savez_compressed(output,
data=...)`` with float32 (H, W) maps, stacked when all frames have one size, else a 1-D object array (what numpy
before 1.24 made of the script's ``np.array(gt_depths)``; later versions raise there).  ``eigen_benchmark`` reads the
split's ``proj_depth/groundtruth`` PNGs (value / 256) in the loader's workers; no kernel is involved.
"""
import argparse
import os

import numpy as np
import torch

from . import _lib
from .ops import _launch, _on_device


def read_calib_file(path):
    """A KITTI calibration file as {key: value}: float arrays where the value is a list of numbers, else the string."""
    numeric = set("0123456789.e+- ")
    data = {}
    with open(path, "r") as f:
        for line in f.readlines():
            key, value = line.split(":", 1)
            value = value.strip()
            data[key] = value
            if numeric.issuperset(value):
                try:
                    data[key] = np.array([float(v) for v in value.split(" ")])
                except ValueError:
                    pass
    return data


_CALIBS = {}


def _calib(calib_dir):
    key = os.path.abspath(calib_dir)
    if key not in _CALIBS:
        _CALIBS[key] = (read_calib_file(os.path.join(calib_dir, "calib_cam_to_cam.txt")),
                        read_calib_file(os.path.join(calib_dir, "calib_velo_to_cam.txt")))
    return _CALIBS[key]


def velo_to_image(calib_dir, cam=2):
    """(P, (H, W)): the (3, 4) fp64 velodyne-to-image projection P_rect_0{cam} . R_rect_00 . [R | T] of a calibration
    directory, formed with numpy as generate_depth_map forms it, and the rectified image size S_rect_02 (for either
    camera, as the reference reads it).  The two files are parsed once per directory."""
    cam2cam, velo2cam = _calib(calib_dir)
    Rt = np.vstack((np.hstack((velo2cam["R"].reshape(3, 3), velo2cam["T"][..., np.newaxis])), np.array([0, 0, 0, 1.0])))
    R_cam2rect = np.eye(4)
    R_cam2rect[:3, :3] = cam2cam["R_rect_00"].reshape(3, 3)
    P_rect = cam2cam["P_rect_0%d" % cam].reshape(3, 4)
    H, W = (int(v) for v in cam2cam["S_rect_02"][::-1].astype(np.int32))
    return np.dot(np.dot(P_rect, R_cam2rect), Rt), (H, W)


def _host(a, dtype, shape_tail, what):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    a = np.ascontiguousarray(a, dtype=dtype)
    if a.ndim != 1 + len(shape_tail) or tuple(a.shape[1:]) != shape_tail:
        raise _lib.WmdError("%s must be (N, %s), got %s" % (what, ", ".join(map(str, shape_tail)), a.shape))
    return a


@_on_device
def generate_depth_maps(points, offsets, P, sizes, vel_depth=False):
    """generate_depth_map for N scans at once: (N, Hmax, Wmax) fp64 CUDA maps, frame n's map in [n, :H_n, :W_n] and zero
    padding around it.

    points (M, 4) float32 (x, y, z, reflectance; a CUDA tensor, or a host tensor or array, pinned for an asynchronous
    upload): the scans one after another in file order; offsets (N + 1) ints, scan n being points[offsets[n] :
    offsets[n + 1]]; P (N, 3, 4) the projections of ``velo_to_image``; sizes (N, 2) each frame's (H, W).  Offsets, P
    and sizes are read on the host."""
    if not torch.is_tensor(points):
        points = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32))
    if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 4:
        raise _lib.WmdError("points must be (M, 4) float32, got %s %s" % (points.dtype, tuple(points.shape)))
    sizes = _host(sizes, np.int32, (2,), "sizes")
    P = _host(P, np.float64, (3, 4), "P")
    offsets = np.asarray(offsets.cpu() if torch.is_tensor(offsets) else offsets).astype(np.int64).reshape(-1)
    n, m = sizes.shape[0], points.shape[0]
    if (P.shape[0] != n or offsets.size != n + 1 or offsets[0] != 0 or offsets[-1] != m
            or (np.diff(offsets) < 0).any()):
        raise _lib.WmdError("offsets must be N + 1 = %d nondecreasing values from 0 to %d, with N P matrices (got %d "
                            "offsets, %d matrices)" % (n + 1, m, offsets.size, P.shape[0]))
    if n and (sizes < 1).any():
        raise _lib.WmdError("every frame needs H and W of at least 1: %s" % sizes[(sizes < 1).any(1)].tolist())
    h_max, w_max = (int(v) for v in sizes.max(0)) if n else (1, 1)
    device = points.device if points.is_cuda else torch.device("cuda", torch.cuda.current_device())
    depth = torch.empty((n, h_max, w_max), dtype=torch.float64, device=device)
    if n == 0:
        return depth
    lib = _lib.load()
    nbytes = int(lib.wmd_velo_depth_ws_bytes(n, h_max, w_max, m))
    if nbytes == 0:
        raise _lib.WmdError("wmd_velo_depth_f64 refuses %d frames of up to %dx%d with %d points" % (n, h_max, w_max, m))
    # a batch of empty scans still passes a non-null points pointer
    pts = points.to(device, non_blocking=True).contiguous() if m else torch.zeros((1, 4), device=device)
    offs = torch.from_numpy(offsets.astype(np.int32)).to(device, non_blocking=True)
    cams = torch.from_numpy(P).to(device, non_blocking=True)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
    _launch("velo_depth", lambda: dict(n=n, h=h_max, w=w_max, points=m)).wmd_velo_depth_f64(
        _lib.ptr(pts), _lib.ptr(offs), _lib.ptr(cams), sizes.ctypes.data, n, h_max, w_max, int(bool(vel_depth)),
        _lib.ptr(ws), nbytes, _lib.ptr(depth), _lib.stream_ptr())
    return depth


def load_velodyne_points(filename):
    """a KITTI .bin scan as (M, 4) float32"""
    return np.fromfile(filename, dtype=np.float32).reshape(-1, 4)


def generate_depth_map(calib_dir, velo_filename, cam=2, vel_depth=False):
    """kitti_utils.generate_depth_map on the device: the (H, W) fp64 CUDA map of one scan"""
    P, (H, W) = velo_to_image(calib_dir, cam)
    points = load_velodyne_points(velo_filename)
    return generate_depth_maps(points, [0, points.shape[0]], P[None], [(H, W)], vel_depth)[0]


# ---------------------------------------------------------------------------------------------------------- loading
class VeloScans(torch.utils.data.Dataset):
    """(velodyne .bin path, calibration directory) items -> (points (M, 4) float32, P (3, 4) fp64, (H, W)), read in
    the loader's workers"""

    def __init__(self, items, cam=2):
        self.items, self.cam = items, cam

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        velo, calib_dir = self.items[i]
        P, size = velo_to_image(calib_dir, self.cam)
        return load_velodyne_points(velo), P, size


def collate(batch):
    """a batch of VeloScans items -> {points (M, 4), offsets (N + 1) int32, P (N, 3, 4) fp64, sizes (N, 2) int32}
    CPU tensors (a loader with pin_memory=True pins them)"""
    counts = [b[0].shape[0] for b in batch]
    offsets = np.zeros(len(batch) + 1, np.int32)
    np.cumsum(counts, out=offsets[1:])
    points = np.concatenate([b[0] for b in batch]) if batch else np.zeros((0, 4), np.float32)
    return {"points": torch.from_numpy(points), "offsets": torch.from_numpy(offsets),
            "P": torch.from_numpy(np.stack([b[1] for b in batch]).reshape(-1, 3, 4)),
            "sizes": torch.from_numpy(np.array([b[2] for b in batch], np.int32).reshape(-1, 2))}


class BenchmarkDepths(torch.utils.data.Dataset):
    """eigen_benchmark's ground-truth PNG paths -> float32 (H, W) depths, uint16 / 256 as the script reads them"""

    def __init__(self, paths):
        self.paths = paths

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, i):
        from PIL import Image
        return np.array(Image.open(self.paths[i])).astype(np.float32) / 256


# ---------------------------------------------------------------------------------------------------------------- CLI
def save_gt_depths(path, maps):
    """np.savez_compressed(path, data=...) of float32 (H, W) maps as the script saves them under numpy < 1.24: stacked
    when every map has one shape, else a 1-D object array of the maps"""
    maps = [np.asarray(m, np.float32) for m in maps]
    if len({m.shape for m in maps}) <= 1:
        data = np.array(maps)
    else:
        data = np.empty(len(maps), dtype=object)
        for i, m in enumerate(maps):
            data[i] = m
    if os.path.dirname(path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, data=data)


def export(opt):
    """the float32 ground-truth maps of every line of opt.filenames, in order"""
    with open(opt.filenames) as f:
        lines = [ln.split() for ln in f.read().splitlines() if ln.strip()]
    loader_args = dict(batch_size=opt.batch_size, shuffle=False, num_workers=opt.num_workers)
    maps = []
    if opt.split == "eigen_benchmark":
        paths = [os.path.join(opt.data_path, folder, "proj_depth", "groundtruth", "image_02", "%010d.png" % int(frame))
                 for folder, frame, _ in lines]
        for batch in torch.utils.data.DataLoader(BenchmarkDepths(paths), collate_fn=list, **loader_args):
            maps.extend(batch)
        return maps
    items = [(os.path.join(opt.data_path, folder, "velodyne_points", "data", "%010d.bin" % int(frame)),
              os.path.join(opt.data_path, folder.split("/")[0])) for folder, frame, _ in lines]
    device = torch.device("cuda", torch.cuda.current_device())
    for batch in torch.utils.data.DataLoader(VeloScans(items, cam=2), collate_fn=collate, pin_memory=True,
                                             **loader_args):
        depth = generate_depth_maps(batch["points"].to(device, non_blocking=True), batch["offsets"], batch["P"],
                                    batch["sizes"], vel_depth=True).cpu().numpy()
        maps.extend(depth[k, :h, :w].astype(np.float32) for k, (h, w) in enumerate(batch["sizes"].tolist()))
    return maps


def get_opts(argv=None):
    p = argparse.ArgumentParser(description="KITTI's ground-truth depths (export_gt_depth.py) on the GPU")
    p.add_argument("--data_path", type=str, help="path to the root of the KITTI data", required=True)
    p.add_argument("--split", type=str, help="which split to export gt from", required=True,
                   choices=["eigen", "eigen_benchmark"])
    p.add_argument("--filenames", type=str, help="the split's lines; default splits/<split>/test_files.txt")
    p.add_argument("--output", type=str, help="default splits/<split>/gt_depths.npz")
    p.add_argument("--batch_size", type=int, default=16, help="frames per device call")
    p.add_argument("--num_workers", type=int, default=8, help="scan-reading worker processes")
    opt = p.parse_args(argv)
    split_folder = os.path.join("splits", opt.split)
    opt.filenames = opt.filenames or os.path.join(split_folder, "test_files.txt")
    opt.output = opt.output or os.path.join(split_folder, "gt_depths.npz")
    return opt


def run(opt):
    print("Exporting ground truth depths for {}".format(opt.split))
    maps = export(opt)
    print("Saving to {}".format(opt.output))
    save_gt_depths(opt.output, maps)
    return maps


if __name__ == "__main__":
    run(get_opts())
