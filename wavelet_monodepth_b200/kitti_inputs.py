"""KITTI's training inputs on the device: ``KITTI/datasets/mono_dataset.py``'s ``__getitem__`` / ``preprocess`` with
``kitti_dataset.KITTIRAWDataset``, bit for bit, with only the JPEG decode left on the host.

The reference's DataLoader workers decode each view, flip it, run four chained Pillow LANCZOS resizes, apply one
ColorJitter to every scale and convert both the plain and the jittered image to float32.  Here:

- ``KittiInputsDataset`` takes ``MonoDataset``'s constructor arguments and makes the reference's random draws in its
  order (the constructor's probing ``get_params``, then per item ``do_color_aug``, ``do_flip`` and the jitter
  parameters of torchvision 0.8.2's ``ColorJitter.get_params``), but returns the decoded uint8 views unflipped, the
  draws, the raw depth hint and whether it was found, the side and ``image_path``.
- ``collate`` pads a list of items into one batch of CPU tensors (pinned by ``DataLoader(pin_memory=True)``).
- ``KittiInputs`` maps a batch to the reference's ``inputs`` dict on the device: the flip, the LANCZOS pyramid, the
  jitter and ToTensor run in libwmd's ``wmd_inputs_u8`` (include/wmd_inputs.h); the cameras are the reference's
  float32 K and ``np.linalg.pinv``, formed once on the host; the depth hint is flipped and nearest-resized by a
  gather and converted by ``depth_to_disp`` in float32 on the device.

The LANCZOS tables need libm's ``sin`` (Pillow's), so they are computed here in double with ``math.sin`` and uploaded
once per (source, target) size and device.  Scale -1 and its jitter are never computed: the reference discards them.

One difference: in a batch that mixes views with and without a hint file, the reference's ``default_collate`` raises on
the missing ``disp_hint``; here those items' ``disp_hint`` is zero, as their ``depth_hint`` and mask are.
"""
import ctypes
import math
import os
import random

import numpy as np
import torch

from . import _lib, pillow_tables
from .ops import _launch
from .pillow_tables import PRECISION_BITS

KITTI_K = np.array([[0.58, 0, 0.5, 0], [0, 1.92, 0.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float32)
JITTER_RANGES = ((0.8, 1.2), (0.8, 1.2), (0.8, 1.2), (-0.1, 0.1))      # brightness, contrast, saturation, hue
MIN_DEPTH, MAX_DEPTH = 0.1, 100.0

VIEW_DTYPE = np.dtype([("xtab", "<u8"), ("ytab", "<u8"), ("h", "<i4"), ("w", "<i4"), ("xk", "<i4"), ("yk", "<i4"),
                       ("flip", "<i4"), ("pad", "<i4")])                 # struct wmd_inputs_view
JITTER_DTYPE = np.dtype([("order", "<i4", 4), ("factor", "<f4", 3), ("hue_shift", "<i4")])  # struct wmd_inputs_jitter


# ------------------------------------------------------------------------------------------------- host-side tables
def lanczos_table(in_size, out_size):
    """Pillow's 8-bit LANCZOS coefficients for in_size -> out_size as (out_size, 2 + k) int32 rows of (first tap,
    taps, k coefficients); an unchanged extent is the identity, as Pillow copies the image."""
    if in_size == out_size:
        return np.stack([np.arange(out_size), np.ones(out_size, np.int64),
                         np.full(out_size, 1 << PRECISION_BITS)], 1).astype(np.int32)
    return pillow_tables.table(in_size, out_size, pillow_tables.lanczos, 3.0)


def hue_shift(hue_factor):
    """torchvision's hue byte: uint8(trunc(h * 255)), i.e. modulo 256"""
    return math.trunc(hue_factor * 255) % 256


def nearest_index(in_size, out_size):
    """cv2.resize INTER_NEAREST's source index of each output index"""
    return np.minimum(np.floor(np.arange(out_size) * (1.0 / (out_size / in_size))).astype(np.int64), in_size - 1)


def get_params(rng=random):
    """torchvision 0.8.2's ColorJitter.get_params with the reference's ranges: uniform draws for brightness, contrast,
    saturation and hue in that order, then random.shuffle of the four transforms.  Returns (factors, order)."""
    factors = tuple(rng.uniform(lo, hi) for lo, hi in JITTER_RANGES)
    order = [0, 1, 2, 3]
    rng.shuffle(order)
    return factors, tuple(order)


def cameras(height, width, scales):
    """{("K", s): K, ("inv_K", s): pinv(K)} as __getitem__ forms them (float32 numpy)"""
    out = {}
    for s in scales:
        K = KITTI_K.copy()
        K[0, :] *= width // (2 ** s)
        K[1, :] *= height // (2 ** s)
        out[("K", s)], out[("inv_K", s)] = K, np.linalg.pinv(K)
    return out


def _scales(target_scales):
    scales = [int(s) for s in target_scales]
    if not scales or len(set(scales)) != len(scales) or any(s < 0 or s > 3 for s in scales):
        raise ValueError("target_scales must be distinct scales in 0..3 (scale -1 is discarded by the reference and "
                         "never computed here), got %r" % (target_scales,))
    return scales


# ------------------------------------------------------------------------------------------------------ the dataset
def pil_rgb(path):
    from PIL import Image
    with open(path, "rb") as f:
        with Image.open(f) as img:
            return img.convert("RGB")


class KittiInputsDataset(torch.utils.data.Dataset):
    """KITTIRAWDataset's items before preprocessing: decoded uint8 (H, W, 3) views, unflipped, keyed by frame id, with
    the reference's random draws and the raw depth hint.  Same constructor arguments as MonoDataset."""

    def __init__(self, data_path, filenames, height, width, frame_idxs, target_scales=(0, 1, 2, 3),
                 use_depth_hints=False, depth_hint_path=None, is_train=False, img_ext=".jpg"):
        super().__init__()
        self.data_path, self.filenames = data_path, filenames
        self.height, self.width = height, width
        self.frame_idxs = list(frame_idxs)
        self.target_scales = _scales(target_scales)
        self.is_train, self.img_ext = is_train, img_ext
        self.use_depth_hints = use_depth_hints
        if use_depth_hints:
            self.with_hints = self.without_hints = 0
        self.depth_hint_path = os.path.join(data_path, "depth_hints") if depth_hint_path is None else depth_hint_path
        get_params()                # the reference's probing call, so a seeded process sees its augmentations
        self.side_map = {"2": 2, "3": 3, "l": 2, "r": 3}

    def __len__(self):
        return len(self.filenames)

    def get_image_path(self, folder, frame_index, side):
        return os.path.join(self.data_path, folder, "image_0{}/data".format(self.side_map[side]),
                            "{:010d}{}".format(frame_index, self.img_ext))

    def __getitem__(self, index):
        do_color_aug = self.is_train and random.random() > 0.5
        do_flip = self.is_train and random.random() > 0.5
        line = self.filenames[index].split()
        folder = line[0]
        frame_index = int(line[1]) if len(line) == 3 else 0
        side = line[2] if len(line) == 3 else None
        views, image_path = {}, None
        for i in self.frame_idxs:
            if i == "s":
                path = self.get_image_path(folder, frame_index, {"r": "l", "l": "r"}[side])
            else:
                path = self.get_image_path(folder, frame_index + i, side)
            views[i] = np.asarray(pil_rgb(path), dtype=np.uint8)
            image_path = path.split(self.data_path, 1)[-1]
        params = get_params() if do_color_aug else None
        item = {"views": views, "do_color_aug": do_color_aug, "do_flip": do_flip, "jitter": params, "side": side,
                "image_path": image_path}
        if "s" in self.frame_idxs and self.use_depth_hints:
            path = os.path.join(self.depth_hint_path, folder, "image_02" if side == "l" else "image_03",
                                str(frame_index).zfill(10) + ".npy")
            try:
                item["hint"] = np.load(path)[0]
                self.with_hints += 1
            except FileNotFoundError:
                item["hint"] = None
                self.without_hints += 1
        return item


def collate(items):
    """One padded batch of CPU tensors from KittiInputsDataset items: "src" (F N, Hmax, Wmax, 3) uint8 with the views
    frame-major (view f N + n is frame f of item n), "sizes" (F N, 2) int32 (h, w), "do_flip" and "do_color_aug" (N,)
    bool, "factors" (N, 4) float64 and "order" (N, 4) int64 (-1 without jitter), "side" and "image_path" lists, and
    with hints "hint" (N, Hh, Wh) float32, "hint_size" (N, 2) int64 and "hint_found" (N,) bool."""
    n = len(items)
    frames = list(items[0]["views"])
    views = [it["views"][f] for f in frames for it in items]
    hmax, wmax = max(v.shape[0] for v in views), max(v.shape[1] for v in views)
    src = torch.zeros((len(views), hmax, wmax, 3), dtype=torch.uint8)
    sizes = torch.empty((len(views), 2), dtype=torch.int32)
    for k, v in enumerate(views):
        src.numpy()[k, :v.shape[0], :v.shape[1]] = v
        sizes[k, 0], sizes[k, 1] = v.shape[0], v.shape[1]
    factors = torch.zeros((n, 4), dtype=torch.float64)
    order = torch.full((n, 4), -1, dtype=torch.int64)
    for k, it in enumerate(items):
        if it["jitter"] is not None:
            factors[k] = torch.tensor(it["jitter"][0], dtype=torch.float64)
            order[k] = torch.tensor(it["jitter"][1])
    batch = {"src": src, "sizes": sizes, "do_flip": torch.tensor([bool(it["do_flip"]) for it in items]),
             "do_color_aug": torch.tensor([bool(it["do_color_aug"]) for it in items]), "factors": factors,
             "order": order, "side": [it["side"] for it in items], "image_path": [it["image_path"] for it in items]}
    if "hint" in items[0]:
        found = [it["hint"] is not None for it in items]
        shapes = [it["hint"].shape if f else (1, 1) for it, f in zip(items, found)]
        hint = torch.zeros((n, max(s[0] for s in shapes), max(s[1] for s in shapes)), dtype=torch.float32)
        for k, it in enumerate(items):
            if found[k]:
                hint.numpy()[k, :shapes[k][0], :shapes[k][1]] = it["hint"]
        batch.update(hint=hint, hint_size=torch.tensor(shapes, dtype=torch.int64), hint_found=torch.tensor(found))
    return batch


# --------------------------------------------------------------------------------------------------- on the device
class KittiInputs:
    """``inputs = KittiInputs(height, width, frame_idxs, target_scales, use_depth_hints)(batch)``: the reference's
    ``inputs`` dict of a ``collate`` batch, on the current CUDA device (or ``device``): ("color", f, s) and
    ("color_aug", f, s) (N, 3, H >> s, W >> s) float32, ("K", s) and ("inv_K", s) (N, 4, 4), "stereo_T" when "s" is
    a frame, "depth_hint", "disp_hint" (when any item has a hint) and "depth_hint_mask" (N, 1, H, W) with hints, and
    "image_path"."""

    def __init__(self, height, width, frame_idxs, target_scales=(0, 1, 2, 3), use_depth_hints=False):
        self.height, self.width = height, width
        self.frame_idxs = list(frame_idxs)
        self.scales = _scales(target_scales)
        self.sizes = [(height >> s, width >> s) for s in self.scales]
        if min(min(hw) for hw in self.sizes) < 1:
            raise ValueError("%dx%d has no pixels at scale %d" % (height, width, max(self.scales)))
        self.use_depth_hints = use_depth_hints
        self.cams = {k: torch.from_numpy(v) for k, v in cameras(height, width, self.scales).items()}
        self._tables = {}
        self._dev_cams = {}

    def table(self, device, in_size, out_size):
        """(device int32 table, k) for in_size -> out_size, computed and uploaded once per device"""
        key = (device.index, in_size, out_size)
        if key not in self._tables:
            tab = lanczos_table(in_size, out_size)
            self._tables[key] = (torch.from_numpy(tab).to(device), tab.shape[1] - 2)
        return self._tables[key]

    def __call__(self, batch, device=None):
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        with torch.cuda.device(device):
            return self._run(batch, device)

    def _run(self, batch, device):
        frames = len(self.frame_idxs)
        src, sizes = batch["src"], batch["sizes"]
        V, src_h, src_w, _ = src.shape
        n = V // frames
        if src.dtype != torch.uint8 or src.shape[3] != 3 or V != n * frames or batch["do_flip"].numel() != n:
            raise _lib.WmdError("expected a collate batch of %d frames per item, got src %s" % (frames, tuple(src.shape)))
        hw = sizes.numpy().astype(np.int64)
        if (hw < 1).any() or (hw[:, 0] > src_h).any() or (hw[:, 1] > src_w).any():
            raise _lib.WmdError("view sizes must lie within the padded (%d, %d) source" % (src_h, src_w))
        flip = batch["do_flip"].numpy().astype(bool)
        out = {}
        (oh, ow) = self.sizes[0]
        views = np.zeros(V, VIEW_DTYPE)
        for v in range(V):
            xt, xk = self.table(device, int(hw[v, 1]), ow)
            yt, yk = self.table(device, int(hw[v, 0]), oh)
            views[v] = (xt.data_ptr(), yt.data_ptr(), hw[v, 0], hw[v, 1], xk, yk, int(flip[v % n]), 0)
        jit = np.zeros(n, JITTER_DTYPE)
        factors, order = batch["factors"].numpy(), batch["order"].numpy()
        jit["order"] = order
        jit["factor"] = factors[:, :3].astype(np.float32)
        jit["hue_shift"] = [hue_shift(float(h)) if o[0] >= 0 else 0 for h, o in zip(factors[:, 3], order)]
        jit = np.tile(jit, frames)                            # view f N + n takes item n's jitter
        meta = np.concatenate([views.view(np.uint8), jit.view(np.uint8)])
        meta_d = torch.from_numpy(meta).pin_memory().to(device, non_blocking=True)
        src_d = src.to(device, non_blocking=True).contiguous()

        desc = _lib.InputsDesc()
        desc.N, desc.src_h, desc.src_w, desc.n_scales = V, src_h, src_w, len(self.scales)
        desc.src = src_d.data_ptr()
        desc.views = meta_d.data_ptr()
        desc.jitter = meta_d.data_ptr() + views.nbytes
        color, color_aug = [], []
        for j, (h, w) in enumerate(self.sizes):
            desc.out_h[j], desc.out_w[j] = h, w
            if j:
                (ph, pw) = self.sizes[j - 1]
                xt, xk = self.table(device, pw, w)
                yt, yk = self.table(device, ph, h)
                desc.xtab[j], desc.ytab[j], desc.xk[j], desc.yk[j] = xt.data_ptr(), yt.data_ptr(), xk, yk
            color.append(torch.empty((V, 3, h, w), dtype=torch.float32, device=device))
            color_aug.append(torch.empty((V, 3, h, w), dtype=torch.float32, device=device))
            desc.color[j], desc.color_aug[j] = color[j].data_ptr(), color_aug[j].data_ptr()
        lib = _lib.load()
        nbytes = int(lib.wmd_inputs_ws_bytes(ctypes.byref(desc)))
        if nbytes == 0 and V > 0:
            raise _lib.WmdError("wmd_inputs_u8 refuses %d views of (%d, %d) -> %s" % (V, src_h, src_w, self.sizes))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
        _launch("kitti_inputs", lambda: dict(n=V, h=self.height, w=self.width)).wmd_inputs_u8(
            ctypes.byref(desc), ws.data_ptr(), ws.numel(), _lib.stream_ptr())

        for fi, f in enumerate(self.frame_idxs):
            for j, s in enumerate(self.scales):
                out[("color", f, s)] = color[j][fi * n:(fi + 1) * n]
                out[("color_aug", f, s)] = color_aug[j][fi * n:(fi + 1) * n]
        if device.index not in self._dev_cams:
            self._dev_cams[device.index] = {k: v.to(device) for k, v in self.cams.items()}
        for k, v in self._dev_cams[device.index].items():
            out[k] = v[None].expand(n, 4, 4).contiguous()
        if "s" in self.frame_idxs:
            T = torch.eye(4, dtype=torch.float32).repeat(n, 1, 1)
            for k, (side, f) in enumerate(zip(batch["side"], flip)):
                T[k, 0, 3] = (-1 if side == "l" else 1) * (-1 if f else 1) * 0.1
            out["stereo_T"] = T.to(device, non_blocking=True)
            if self.use_depth_hints:
                out.update(self._hints(batch, flip, device))
        out["image_path"] = list(batch["image_path"])
        return out

    def _hints(self, batch, flip, device):
        """flip, cv2 INTER_NEAREST to (W, H) and depth_to_disp of the raw hints, on the device"""
        n, H, W = len(flip), self.height, self.width
        found = batch["hint_found"].numpy().astype(bool)
        rows = np.zeros((n, H), np.int64)
        cols = np.zeros((n, W), np.int64)
        for k, (h0, w0) in enumerate(batch["hint_size"].numpy()):
            rows[k] = nearest_index(int(h0), H)
            cols[k] = nearest_index(int(w0), W)
            if flip[k]:
                cols[k] = w0 - 1 - cols[k]
        hint = batch["hint"].to(device, non_blocking=True)
        idx = torch.arange(n, device=device)[:, None, None]
        depth = hint[idx, torch.from_numpy(rows).to(device)[:, :, None], torch.from_numpy(cols).to(device)[:, None, :]]
        found_d = torch.from_numpy(found).to(device)[:, None, None, None]
        depth = torch.where(found_d, depth[:, None], torch.zeros((), device=device))
        out = {"depth_hint": depth, "depth_hint_mask": (depth > 0).float()}
        if found.any():
            # layers.depth_to_disp in float32; divisions by tensors, since torch multiplies by a scalar's reciprocal
            min_disp, max_disp = 1 / MAX_DEPTH, 1 / MIN_DEPTH
            one = torch.ones((), dtype=torch.float32, device=device)
            disp = one / (depth + 1e-5)
            disp = (disp - min_disp) / torch.tensor(max_disp - min_disp, dtype=torch.float32, device=device)
            disp = torch.where((depth <= 0) | (disp <= 0), torch.zeros((), device=device), disp)
            out["disp_hint"] = torch.where(found_d, disp, torch.zeros((), device=device))
        return out
