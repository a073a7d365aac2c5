"""KITTI's depth hints on the device: ``KITTI/precompute_depth_hints.py`` as one batched command.

The reference script runs twelve ``cv2.StereoSGBM`` matchers on the CPU for every view (blockSize 1, 2, 3 x
numDisparities 64, 96, 128, 160), turns each disparity into a depth, warps the other view by each depth, and keeps per
pixel the depth whose SSIM + L1 reprojection error is least.  Here the matcher is libwmd's ``wmd_sgbm_u8``, OpenCV's
integer algorithm bit for bit, and the fusion is ``wmd_depth_hints_f32`` (include/wmd_hints.h).  blockSize 2 and 3 are
the same matcher (OpenCV uses the half-width blockSize / 2), so eight matchers run and the fusion reads the blockSize 2
maps twice; torch's argmin takes the first of equal errors, so the blockSize 3 index is never the one chosen.

``stereo_sgbm`` is ``matcher.compute`` with the script's parameters on (N, H, W, 3) uint8 CUDA views.
``DepthHintGenerator`` builds K, inv_K and the stereo transform exactly as the script does and maps a batch of
(base, lookup, right) views to the script's ``best_depth`` per view.

    python -m wavelet_monodepth_b200.kitti_hints --data_path KITTI_RAW [--filenames SPLIT] [--save_path DIR]
        [--height 320] [--width 1024] [--overwrite_saved_depths] [--batch_size 8] [--num_workers 12]

writes ``<save_path>/<sequence>/image_0{2,3}/<frame:010d>.npy``, (1, H, W) float32, which KITTI's ``mono_dataset``
loads as its depth hint.  Decode and resize are the script's: PIL ``convert('RGB')`` and a LANCZOS resize to (W, H).
One difference: without ``--overwrite_saved_depths`` the script stops with an AttributeError (it reads an
``old_save_path`` it never sets); here views whose file already exists are skipped.
"""
import argparse
import os
import time

import numpy as np
import torch

from . import _lib
from .ops import _launch, _on_device

NUM_DISPARITIES = (64, 96, 128, 160)
BLOCK_SIZES = (1, 2, 3)
MATCHERS = tuple((nd, bs) for bs in BLOCK_SIZES for nd in NUM_DISPARITIES)     # the script's order
BASELINE = 0.1


def _views(*ts):
    for t in ts:
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 4 and t.shape[3] == 3):
            raise _lib.WmdError("expected (N, H, W, 3) uint8 CUDA views, got %s"
                                % (tuple(t.shape) if torch.is_tensor(t) else type(t).__name__,))
    if any(t.shape != ts[0].shape for t in ts):
        raise _lib.WmdError("the views' shapes differ: %s" % [tuple(t.shape) for t in ts])
    return [t.contiguous() for t in ts]


def _flags(right, n, device):
    """per-frame right-view flags as a (N,) uint8 device tensor"""
    r = torch.as_tensor(right, dtype=torch.bool).reshape(-1)
    if r.numel() != n:
        raise _lib.WmdError("expected %d right-view flags, got %d" % (n, r.numel()))
    return r.to(device=device, dtype=torch.uint8)


@_on_device
def stereo_sgbm(left, right, num_disparities, block_size, reverse=None, out=None):
    """cv2.StereoSGBM_create(minDisparity=0, numDisparities, blockSize, P1=36, P2=288, preFilterCap=63,
    uniquenessRatio=10, speckleWindowSize=100, speckleRange=16).compute(left, right) per frame of (N, H, W, 3) uint8
    CUDA views: (N, H, W) int16, disparity x16, -16 where invalid.  reverse (N,) bools: match that frame mirrored (its
    base view is the right one), as the depth-hints script does; the map comes back in the views' orientation."""
    left, right = _views(left, right)
    n, h, w, _ = left.shape
    lib = _lib.load()
    nbytes = int(lib.wmd_sgbm_ws_bytes(n, h, w, num_disparities, block_size))
    if nbytes == 0 and n > 0:
        raise _lib.WmdError("wmd_sgbm_u8 refuses numDisparities %s, blockSize %s at %dx%d"
                            % (num_disparities, block_size, h, w))
    rev = None if reverse is None else _flags(reverse, n, left.device)
    if out is None:
        out = torch.empty((n, h, w), dtype=torch.int16, device=left.device)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=left.device)
    _launch("sgbm", lambda: dict(n=n, h=h, w=w, d=num_disparities, block=block_size)).wmd_sgbm_u8(
        _lib.ptr(left), _lib.ptr(right), _lib.ptr(rev), n, h, w, num_disparities, block_size, _lib.ptr(ws), ws.numel(),
        _lib.ptr(out), _lib.stream_ptr())
    return out


class DepthHintGenerator:
    """The depth-hints script's fused SGM depth for views of (height, width): K = [[0.58 W, 0, 0.5 W], [0, 1.92 H,
    0.5 H]] in float32, inv_K = pinv(K), the stereo transform T[0, 3] = -0.1 for a left base view and +0.1 for a right
    one.  ``gen(base, lookup, right)`` -> (N, 1, H, W) float32, the script's ``best_depth`` of each view (with
    ``return_index`` also the (N, 1, H, W) int32 index of the winning matcher)."""

    def __init__(self, height=320, width=1024):
        self.height, self.width = height, width
        K = np.array([[0.58, 0, 0.5, 0], [0, 1.92, 0.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float32)
        K[0] *= width
        K[1] *= height
        self.K = K
        self.inv_K = np.linalg.pinv(K)

    def cameras(self, right):
        """(K, inv_K, T), each (N, 4, 4) float32 CPU tensors, for per-view right flags"""
        r = torch.as_tensor(right, dtype=torch.bool).reshape(-1)
        n = r.numel()
        K = torch.from_numpy(self.K)[None].expand(n, 4, 4).contiguous()
        inv_K = torch.from_numpy(self.inv_K)[None].expand(n, 4, 4).contiguous()
        T = torch.eye(4)[None].repeat(n, 1, 1)
        T[:, 0, 3] = torch.where(r, torch.tensor(BASELINE), torch.tensor(-BASELINE))
        return K, inv_K, T

    def disparities(self, base, lookup, right):
        """the twelve matchers' maps, (12, N, H, W) int16, in the script's order"""
        base, lookup = _views(base, lookup)
        n, h, w, _ = base.shape
        maps = torch.empty((len(MATCHERS), n, h, w), dtype=torch.int16, device=base.device)
        for i, (nd, bs) in enumerate(MATCHERS):
            if bs == 3:                        # the blockSize 2 matcher: OpenCV's half-width is blockSize / 2
                maps[i].copy_(maps[i - len(NUM_DISPARITIES)])
            else:
                stereo_sgbm(base, lookup, nd, bs, reverse=right, out=maps[i])
        return maps

    def __call__(self, base, lookup, right, return_index=False):
        return self._run(base, lookup, right, return_index)

    @_on_device
    def _run(self, base, lookup, right, return_index):
        base, lookup = _views(base, lookup)
        n, h, w, _ = base.shape
        if (h, w) != (self.height, self.width):
            raise _lib.WmdError("views are %dx%d, the generator's cameras %dx%d" % (h, w, self.height, self.width))
        dev = base.device
        maps = self.disparities(base, lookup, right)
        K, inv_K, T = (t.to(dev) for t in self.cameras(right))
        depth = torch.empty((n, 1, h, w), dtype=torch.float32, device=dev)
        index = torch.empty((n, 1, h, w), dtype=torch.int32, device=dev) if return_index else None
        _fuse(base, lookup, maps, K, inv_K, T, depth, index)
        return (depth, index) if return_index else depth


def _fuse(base, lookup, maps, K, inv_K, T, depth, index):
    """wmd_depth_hints_f32 on (N, H, W, 3) uint8 views, the matchers' (12, N, H, W) int16 maps and (N, 4, 4) float32
    cameras: each pixel's least-error depth into depth (N, 1, H, W) float32 and, unless None, the winning matcher into
    index (N, 1, H, W) int32"""
    n, h, w, _ = base.shape
    nbytes = int(_lib.load().wmd_depth_hints_ws_bytes(n, h, w))
    if nbytes == 0 and n > 0:
        raise _lib.WmdError("wmd_depth_hints_f32 refuses %d views of %dx%d" % (n, h, w))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=base.device)
    _launch("depth_hints", lambda: dict(n=n, h=h, w=w)).wmd_depth_hints_f32(
        _lib.ptr(base), _lib.ptr(lookup), _lib.ptr(maps), _lib.ptr(K), _lib.ptr(inv_K), _lib.ptr(T), n, h, w,
        _lib.ptr(ws), ws.numel(), _lib.ptr(depth), _lib.ptr(index), _lib.stream_ptr())


# ---------------------------------------------------------------------------------------------------------------- CLI
def pil_rgb(path):
    from PIL import Image
    with open(path, "rb") as f:
        with Image.open(f) as img:
            return img.convert("RGB")


def load_view(path, height, width):
    """the script's decode and resize: PIL RGB, LANCZOS to (width, height), as (H, W, 3) uint8"""
    from PIL import Image
    return np.array(pil_rgb(path).resize((width, height), Image.LANCZOS), dtype=np.uint8)


def view_paths(data_path, save_path, line):
    """(base image, lookup image, output .npy, right) of one split line "sequence frame side" """
    sequence, frame, side = line.split()
    right = side != "l"
    this, other = ("image_03", "image_02") if right else ("image_02", "image_03")
    name = "%s.jpg" % str(frame).zfill(10)
    return (os.path.join(data_path, sequence, this, "data", name), os.path.join(data_path, sequence, other, "data", name),
            os.path.join(save_path, sequence, this, "%s.npy" % str(frame).zfill(10)), right)


class _Views(torch.utils.data.Dataset):
    def __init__(self, items, height, width):
        self.items, self.height, self.width = items, height, width

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        base, lookup, _, right = self.items[i]
        return (torch.from_numpy(load_view(base, self.height, self.width)),
                torch.from_numpy(load_view(lookup, self.height, self.width)), right, i)


def run(opt):
    """compute and save the depth hints of every view of opt.filenames; returns (views written, views skipped)"""
    save_path = opt.save_path or os.path.join(opt.data_path, "depth_hints")
    with open(opt.filenames) as f:
        lines = [ln for ln in f.read().splitlines() if ln.strip()]
    items = [view_paths(opt.data_path, save_path, ln) for ln in lines]
    todo = [it for it in items if opt.overwrite_saved_depths or not os.path.isfile(it[2])]
    print("Computing depth hints for %d views (%d skipped), saving to %s"
          % (len(todo), len(items) - len(todo), save_path))
    gen = DepthHintGenerator(opt.height, opt.width)
    loader = torch.utils.data.DataLoader(_Views(todo, opt.height, opt.width), batch_size=opt.batch_size,
                                         shuffle=False, num_workers=opt.num_workers, pin_memory=True)
    device = torch.device("cuda", torch.cuda.current_device())
    t0, done = time.time(), 0
    for base, lookup, right, idx in loader:
        depth = gen(base.to(device, non_blocking=True), lookup.to(device, non_blocking=True), right).cpu().numpy()
        for k, i in enumerate(idx.tolist()):
            out = todo[i][2]
            os.makedirs(os.path.dirname(out), exist_ok=True)
            np.save(out, depth[k])
        done += len(idx)
        print("%d / %d views, %.1f views/s" % (done, len(todo), done / max(time.time() - t0, 1e-9)))
    return len(todo), len(items) - len(todo)


def get_opts(argv=None):
    p = argparse.ArgumentParser(description="KITTI's depth hints (fused SGM) on the GPU")
    p.add_argument("--data_path", help="path to the KITTI raw images", type=str, required=True)
    p.add_argument("--filenames", help='text file of "sequence_name frame_number side" lines', type=str,
                   default="splits/eigen_full/all_files.txt")
    p.add_argument("--save_path", help="where to save the hints; default <data_path>/depth_hints", type=str)
    p.add_argument("--height", default=320, type=int)
    p.add_argument("--width", default=1024, type=int)
    p.add_argument("--overwrite_saved_depths", action="store_true",
                   help="recompute views whose hint file exists instead of skipping them")
    p.add_argument("--batch_size", default=8, type=int, help="views per device batch")
    p.add_argument("--num_workers", default=12, type=int, help="decode and resize worker processes")
    return p.parse_args(argv)


if __name__ == "__main__":
    run(get_opts())
