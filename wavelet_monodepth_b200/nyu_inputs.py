"""NYUv2's training inputs on the device: ``NYUv2/data.py``'s ``depthDatasetMemory`` with ``getDefaultTrainTransform``
(and ``getNoTransform`` for the testing loader), bit for bit, with only the image and depth decode left on the host.

The reference's DataLoader workers decode each item, flip it, maybe swap its channels, apply a random gamma, crop 16
pixels off every side, resize with Pillow and convert to float32.  Here:

- ``load_zip_to_mem`` is ``loadZipToMem``: the zip in memory and the shuffled ``nyu2_train.csv`` rows.
- ``NyuInputsDataset`` decodes with PIL as ``depthDatasetMemory`` does and makes the transform's random draws in its
  order (flip, swap and its permutation, gamma), but returns the decoded uint8 arrays and the draws.
- ``collate`` stacks a list of items into CPU tensors (pinned by ``DataLoader(pin_memory=True)``) and forms each
  item's gamma table with libm's ``pow``, as torchvision's ``adjust_gamma`` does.
- ``NyuInputs`` maps a batch to ``{"image", "depth"}`` on the device in one ``wmd_nyu_inputs_u8`` call
  (include/wmd_inputs_nyu.h): two launches for the flip, swap, gamma, crop, both resizes and ToTensor.

``resample`` picks the filter of ToTensor's ``resize``, which the reference calls without one: ``"bicubic"`` is
Pillow's default since 7.0 (and the reference's on a current Pillow), ``"nearest"`` the default of the Pillow 6.2.1 its
environment pins, with which the paper's models were trained.
"""
import ctypes
import io
import itertools
import random
import zipfile

import numpy as np
import torch

from . import _lib, pillow_tables
from .ops import _launch

SRC_H, SRC_W, CROP = _lib.NYU_SRC_H, _lib.NYU_SRC_W, _lib.NYU_CROP
CROP_H, CROP_W = SRC_H - 2 * CROP, SRC_W - 2 * CROP                     # 448, 608
PERMS = list(itertools.permutations(range(3), 3))                       # RandomChannelSwap's indices
SWAP_PROBABILITY, GAMMA = 0.1, 0.8
RESAMPLE = ("bicubic", "nearest")
ITEM_DTYPE = np.dtype([("flip", "<i4"), ("perm", "<i4", 3)])             # struct wmd_nyu_inputs_item


def sizes(is_224):
    """((image h, w), (depth h, w)) of ToTensor's resizes"""
    return ((224, 224), (224, 224)) if is_224 else ((480, 640), (240, 320))


def gamma_lut(gamma):
    """torchvision's adjust_gamma(img, gamma, gain=1) byte map (a Pillow point table), (256,) uint8; None: identity"""
    if gamma is None:
        return np.arange(256, dtype=np.uint8)
    return np.array([int((255 + 1 - 1e-3) * 1 * pow(v / 255.0, gamma)) for v in range(256)], np.uint8)


def resample_table(in_size, out_size, resample, offset=CROP):
    """the (out_size, 2 + k) int32 table of one resize pass, first taps offset by the crop"""
    if resample == "bicubic":
        return pillow_tables.table(in_size, out_size, pillow_tables.bicubic, 2.0, offset)
    return pillow_tables.nearest_table(in_size, out_size, offset)


# ------------------------------------------------------------------------------------------------------ the dataset
def load_zip_to_mem(path):
    """loadZipToMem: ({name: bytes} of the whole zip, the rows of data/nyu2_train.csv shuffled as sklearn's
    shuffle(random_state=0) shuffles them)"""
    with zipfile.ZipFile(path) as zf:
        data = {name: zf.read(name) for name in zf.namelist()}
    rows = [row.split(",") for row in data["data/nyu2_train.csv"].decode("utf-8").split("\n") if len(row) > 0]
    order = np.arange(len(rows))
    np.random.RandomState(0).shuffle(order)
    return data, [rows[i] for i in order]


def _decode(data, name, mode):
    from PIL import Image
    img = Image.open(io.BytesIO(data[name]))
    if img.mode != mode or img.size != (SRC_W, SRC_H):
        raise ValueError("%s: expected a %dx%d %s image, got %dx%d %s" % (name, SRC_W, SRC_H, mode, img.size[0],
                                                                          img.size[1], img.mode))
    return np.asarray(img, dtype=np.uint8)


def draws(is_train, rng=random):
    """getDefaultTrainTransform's draws in its order: (flip, permutation index or -1, gamma); the testing transform
    makes none: (False, -1, None)"""
    if not is_train:
        return False, -1, None
    flip = rng.random() < 0.5
    perm = rng.randint(0, len(PERMS) - 1) if rng.random() < SWAP_PROBABILITY else -1
    gamma = rng.uniform(1 / GAMMA, GAMMA)
    return flip, perm, gamma


class NyuInputsDataset(torch.utils.data.Dataset):
    """depthDatasetMemory's items before the transform: the decoded (480, 640, 3) RGB image and (480, 640) L depth as
    uint8 arrays, with the training transform's draws ("flip", "perm" an index into PERMS or -1, "gamma" or None).
    ``is_train=False`` is getNoTransform's loader, which draws nothing."""

    def __init__(self, data, nyu2_train, is_train=True):
        super().__init__()
        self.data, self.nyu_dataset, self.is_train = data, nyu2_train, is_train

    def __len__(self):
        return len(self.nyu_dataset)

    def __getitem__(self, idx):
        sample = self.nyu_dataset[idx]
        image = _decode(self.data, sample[0], "RGB")
        depth = _decode(self.data, sample[1], "L")
        flip, perm, gamma = draws(self.is_train)
        return {"image": image, "depth": depth, "flip": flip, "perm": perm, "gamma": gamma}


def collate(items):
    """One batch of CPU tensors from NyuInputsDataset items: "image" (N, 480, 640, 3) and "depth" (N, 480, 640) uint8,
    "flip" (N,) bool, "perm" (N, 3) int32 (output channel c takes input channel perm[c]), "lut" (N, 256) uint8 and
    "gamma" (N,) float64 (NaN without gamma)."""
    n = len(items)
    batch = {"image": torch.empty((n, SRC_H, SRC_W, 3), dtype=torch.uint8),
             "depth": torch.empty((n, SRC_H, SRC_W), dtype=torch.uint8),
             "flip": torch.tensor([bool(it["flip"]) for it in items], dtype=torch.bool),
             "perm": torch.tensor([PERMS[it["perm"]] if it["perm"] >= 0 else (0, 1, 2) for it in items],
                                  dtype=torch.int32).reshape(n, 3),
             "lut": torch.from_numpy(np.array([gamma_lut(it["gamma"]) for it in items], np.uint8).reshape(n, 256)),
             "gamma": torch.tensor([np.nan if it["gamma"] is None else it["gamma"] for it in items],
                                   dtype=torch.float64)}
    for k, it in enumerate(items):
        batch["image"].numpy()[k] = it["image"]
        batch["depth"].numpy()[k] = it["depth"]
    return batch


# --------------------------------------------------------------------------------------------------- on the device
class NyuInputs:
    """``inputs = NyuInputs(is_224, resample)(batch)``: ToTensor's ``{"image": (N, 3, H, W), "depth": (N, 1, h, w)}``
    float32 of a ``collate`` batch on the current CUDA device (or ``device``): 640x480 and 320x240, or 224x224 both
    with ``is_224``."""

    def __init__(self, is_224=False, resample="bicubic"):
        if resample not in RESAMPLE:
            raise ValueError("resample must be one of %s, got %r" % (RESAMPLE, resample))
        self.is_224, self.resample = bool(is_224), resample
        self.image_size, self.depth_size = sizes(self.is_224)
        self._tables = {}

    def table(self, device, in_size, out_size):
        """(device int32 table, k) for in_size -> out_size, computed and uploaded once per device"""
        key = (device.index, in_size, out_size)
        if key not in self._tables:
            tab = resample_table(in_size, out_size, self.resample)
            self._tables[key] = (torch.from_numpy(tab).to(device), tab.shape[1] - 2)
        return self._tables[key]

    def __call__(self, batch, device=None):
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        with torch.cuda.device(device):
            return self._run(batch, device)

    def _run(self, batch, device):
        image, depth, lut = batch["image"], batch["depth"], batch["lut"]
        n = image.shape[0]
        if (image.dtype != torch.uint8 or tuple(image.shape) != (n, SRC_H, SRC_W, 3) or depth.dtype != torch.uint8
                or tuple(depth.shape) != (n, SRC_H, SRC_W) or lut.dtype != torch.uint8 or tuple(lut.shape) != (n, 256)
                or tuple(batch["perm"].shape) != (n, 3) or batch["flip"].numel() != n):
            raise _lib.WmdError("expected a collate batch of (N, %d, %d, 3) images and (N, %d, %d) depths, got %s and %s"
                                % (SRC_H, SRC_W, SRC_H, SRC_W, tuple(image.shape), tuple(depth.shape)))
        (ih, iw), (dh, dw) = self.image_size, self.depth_size
        out = {"image": torch.empty((n, 3, ih, iw), dtype=torch.float32, device=device),
               "depth": torch.empty((n, 1, dh, dw), dtype=torch.float32, device=device)}
        if n == 0:
            return out
        items = np.zeros(n, ITEM_DTYPE)
        items["flip"] = batch["flip"].numpy().astype(np.int32)
        items["perm"] = batch["perm"].numpy()
        meta = np.concatenate([items.view(np.uint8), lut.numpy().reshape(-1)])
        meta_d = torch.from_numpy(meta).pin_memory().to(device, non_blocking=True)
        image_d = image.to(device, non_blocking=True).contiguous()
        depth_d = depth.to(device, non_blocking=True).contiguous()

        desc = _lib.NyuInputsDesc()
        desc.N, desc.image_h, desc.image_w, desc.depth_h, desc.depth_w = n, ih, iw, dh, dw
        ixt, desc.image_xk = self.table(device, CROP_W, iw)
        iyt, desc.image_yk = self.table(device, CROP_H, ih)
        dxt, desc.depth_xk = self.table(device, CROP_W, dw)
        dyt, desc.depth_yk = self.table(device, CROP_H, dh)
        desc.image_xtab, desc.image_ytab = ixt.data_ptr(), iyt.data_ptr()
        desc.depth_xtab, desc.depth_ytab = dxt.data_ptr(), dyt.data_ptr()
        desc.image_src, desc.depth_src = image_d.data_ptr(), depth_d.data_ptr()
        desc.items = meta_d.data_ptr()
        desc.lut = meta_d.data_ptr() + items.nbytes
        desc.image, desc.depth = out["image"].data_ptr(), out["depth"].data_ptr()
        nbytes = int(_lib.load().wmd_nyu_inputs_ws_bytes(ctypes.byref(desc)))
        if nbytes == 0:
            raise _lib.WmdError("wmd_nyu_inputs_u8 refuses %d items -> %s, %s" % (n, self.image_size, self.depth_size))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _launch("nyu_inputs", lambda: dict(n=n, is_224=self.is_224)).wmd_nyu_inputs_u8(
            ctypes.byref(desc), ws.data_ptr(), ws.numel(), _lib.stream_ptr())
        return out


def get_training_testing_data(batch_size, num_workers=8, is_224=False, zip_path="nyu_data.zip", resample="bicubic"):
    """getTrainingTestingData's two loaders, of collate batches: the training one (shuffled, with the training
    transform's draws) and the testing one (in order, no draws).  Each has a ``make_inputs``, the one NyuInputs(is_224,
    resample) both share, which maps its batches to ``{"image", "depth"}`` on the device."""
    make_inputs = NyuInputs(is_224, resample)
    data, nyu2_train = load_zip_to_mem(zip_path)
    training = NyuInputsDataset(data, nyu2_train, is_train=True)
    testing = NyuInputsDataset(data, nyu2_train, is_train=False)
    loaders = (torch.utils.data.DataLoader(training, batch_size, shuffle=True, num_workers=num_workers,
                                           pin_memory=True, collate_fn=collate),
               torch.utils.data.DataLoader(testing, batch_size, shuffle=False, num_workers=num_workers,
                                           pin_memory=True, collate_fn=collate))
    for loader in loaders:
        loader.make_inputs = make_inputs
    return loaders
