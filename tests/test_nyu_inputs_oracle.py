"""CPU: NYUv2's training inputs.  The BICUBIC and NEAREST tables, applied by oracle.nyu_inputs, equal the installed
Pillow's resize at every (608x448 -> target) pair in RGB and L; the gamma table equals torchvision's adjust_gamma and
the permutations RandomChannelSwap's; NyuInputsDataset makes the reference transform's draws; the shuffle restatement
equals sklearn's; the golden fixtures reproduce from the oracle; include/wmd_inputs_nyu.h matches its binding and the
library, and wmd_nyu_inputs_u8 refuses bad arguments before any CUDA call."""
import ctypes
import io
import os
import random
import re
import zipfile

import numpy as np
import pytest
from PIL import Image

from oracle import nyu_inputs as oni
from oracle.kitti_inputs import _pass
from wavelet_monodepth_b200 import _lib
from wavelet_monodepth_b200 import nyu_inputs as ni

import nyu_inputs_cases as nic

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TARGETS = ((640, 480), (320, 240), (224, 224))
PIL_FILTER = {"bicubic": Image.BICUBIC, "nearest": Image.NEAREST}


@pytest.mark.parametrize("resample", ["bicubic", "nearest"])
@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("target", TARGETS, ids=lambda wh: "%dx%d" % wh)
def test_tables_equal_pillow_resize(target, mode, resample):
    """the device tables (crop offset in their first taps) over the uncropped image, and the oracle's own resize of the
    cropped one, both equal Image.resize of the crop"""
    w, h = target
    rng = np.random.default_rng(w + h + len(mode))
    shape = (480, 640, 3) if mode == "RGB" else (480, 640)
    full = rng.integers(0, 256, shape, dtype=np.uint8)
    full[100:200] = rng.integers(0, 2, shape[1:], dtype=np.uint8) * 255           # hard edges, where taps clip
    crop = full[16:464, 16:624]
    want = np.asarray(Image.fromarray(full).crop((16, 16, 624, 464)).resize((w, h), PIL_FILTER[resample]))
    assert np.array_equal(oni.resize(crop, w, h, resample), want)
    xt, yt = ni.resample_table(608, w, resample), ni.resample_table(448, h, resample)
    got = _pass(_pass(full, (xt[:, :2], xt[:, 2:]), 1), (yt[:, :2], yt[:, 2:]), 0)
    assert np.array_equal(got, want)
    if resample == "nearest":
        assert xt.shape[1] == 3 and (xt[:, 1:] == (1, 1 << 22)).all()


def test_bicubic_tables_equal_the_oracles():
    for n_in, n_out in ((608, 640), (448, 480), (608, 320), (448, 240), (608, 224), (448, 224), (5, 9), (9, 2)):
        bounds, coeffs = oni.bicubic_table(n_in, n_out)
        tab = ni.resample_table(n_in, n_out, "bicubic", offset=0)
        assert np.array_equal(tab[:, :2], bounds) and np.array_equal(tab[:, 2:], coeffs), (n_in, n_out)
        assert np.array_equal(ni.resample_table(n_in, n_out, "nearest", offset=0)[:, 0], oni.nearest_index(n_in, n_out))


@pytest.mark.parametrize("gamma", [0.8, 1.0, 1.25] + list(np.linspace(0.8, 1.25, 17)))
def test_gamma_table_equals_adjust_gamma(gamma):
    import torchvision.transforms.functional as TF
    values = np.arange(256, dtype=np.uint8)
    img = np.stack([values, values[::-1], np.roll(values, 77)], -1).reshape(16, 16, 3)
    want = np.asarray(TF.adjust_gamma(Image.fromarray(img), float(gamma), gain=1))
    assert np.array_equal(ni.gamma_lut(float(gamma))[img], want)
    assert np.array_equal(oni.gamma_lut(float(gamma)), ni.gamma_lut(float(gamma)))
    assert np.array_equal(ni.gamma_lut(None), values)


def test_permutations_are_the_channel_swaps():
    import itertools
    assert ni.PERMS == oni.PERMS == list(itertools.permutations(range(3), 3))
    img, depth = oni.synthetic_image(1), oni.synthetic_depth(1)
    plain = oni.expected(img, depth, False, -1, None, True, "nearest")["image"]
    for p, perm in enumerate(ni.PERMS):
        # RandomChannelSwap: Image.fromarray(np.asarray(image)[..., list(indices[k])])
        swapped = np.asarray(Image.fromarray(np.asarray(Image.fromarray(img))[..., list(perm)]))
        e = oni.expected(img, depth, False, p, 1.1, True, "nearest")["image"]
        assert np.array_equal(e, oni.expected(swapped, depth, False, -1, 1.1, True, "nearest")["image"]), perm
        assert np.array_equal(oni.expected(img, depth, False, p, None, True, "nearest")["image"],
                              plain[list(perm)]), perm


def test_shuffle_restatement_equals_sklearn(tmp_path):
    shuffle = pytest.importorskip("sklearn.utils").shuffle
    rows = [["a%d" % k, "b%d" % k] for k in range(5077)]
    path = tmp_path / "nyu_data.zip"
    with zipfile.ZipFile(path, "w") as zf:
        zf.writestr("data/nyu2_train.csv", "\n".join(",".join(r) for r in rows) + "\n")
    data, got = ni.load_zip_to_mem(str(path))
    assert got == shuffle(rows, random_state=0)
    assert set(data) == {"data/nyu2_train.csv"}


@pytest.mark.parametrize("name", nic.CASES)
def test_fixtures_reproduce_from_the_oracle(name):
    fx = nic.load(name)
    cfg = fx["config"]
    its = nic.items(fx)
    exp = [oni.expected(it["image"], it["depth"], it["flip"], it["perm"], it["gamma"], cfg["is_224"], cfg["resample"])
           for it in its]
    assert nic.mismatches(fx, lambda n: exp[n]) == []
    draws = {(bool(f), int(p)) for f, p, t in zip(fx["flip"], fx["perm"], fx["is_train"]) if t}
    assert {p for _, p in draws} == set(range(-1, 6))                              # all six permutations
    assert {(f, p >= 0) for f, p in draws} == {(False, False), (False, True), (True, False), (True, True)}
    assert not fx["is_train"].all() and fx["is_train"].any()
    assert os.path.getsize(os.path.join(nic.GOLDEN, "nyu_inputs_%s.npz" % name)) < 1 << 20


def _zip(tmp_path, seeds, image_mode="RGB", image_size=(640, 480), depth_mode="L"):
    rows = []
    path = tmp_path / "nyu_data.zip"
    with zipfile.ZipFile(path, "w") as zf:
        for k, s in enumerate(seeds):
            img = Image.fromarray(oni.synthetic_image(s)).convert(image_mode).resize(image_size)
            dep = Image.fromarray(oni.synthetic_depth(s)).convert(depth_mode)
            for name, im in (("%d.png" % k, img), ("%d_depth.png" % k, dep)):
                buf = io.BytesIO()
                im.save(buf, "PNG")
                zf.writestr("data/nyu2_train/" + name, buf.getvalue())
            rows.append("data/nyu2_train/%d.png,data/nyu2_train/%d_depth.png" % (k, k))
        zf.writestr("data/nyu2_train.csv", "\n".join(rows) + "\n")
    return str(path)


def test_dataset_makes_the_references_draws(tmp_path):
    """a zip of the 640 BICUBIC fixture's views: each item of a NyuInputsDataset, after random.seed of its draw seed,
    has the reference's draws and views, and the oracle of it gives the reference's digests"""
    fx = nic.load("640_bicubic")
    data, rows = ni.load_zip_to_mem(_zip(tmp_path, [int(s) for s in fx["view"]]))
    order = {r[0]: int(r[0].split("/")[-1][:-4]) for r in rows}
    for i in range(len(fx["view"])):
        k = [j for j, r in enumerate(rows) if order[r[0]] == i][0]
        random.seed(int(fx["seed"][i]))
        it = ni.NyuInputsDataset(data, rows, is_train=bool(fx["is_train"][i]))[k]
        gamma = float(fx["gamma"][i])
        assert (it["flip"], it["perm"]) == (bool(fx["flip"][i]), int(fx["perm"][i]))
        assert (it["gamma"] is None and np.isnan(gamma)) or it["gamma"] == gamma
        assert np.array_equal(it["image"], oni.synthetic_image(int(fx["view"][i])))
        assert np.array_equal(it["depth"], oni.synthetic_depth(int(fx["view"][i])))
        exp = oni.expected(it["image"], it["depth"], it["flip"], it["perm"], it["gamma"], False, "bicubic")
        assert [nic.digest(exp["image"]), nic.digest(exp["depth"])] == list(fx["digests"][i])
    random.seed(5)
    assert ni.draws(True) == oni.draws(True, random.Random(5))
    assert ni.draws(False) == (False, -1, None)


@pytest.mark.parametrize("bad", [dict(image_mode="L"), dict(image_mode="RGBA"), dict(image_size=(640, 481)),
                                 dict(depth_mode="I;16"), dict(depth_mode="RGB")])
def test_dataset_refuses_other_modes_and_sizes(tmp_path, bad):
    data, rows = ni.load_zip_to_mem(_zip(tmp_path, [1], **bad))
    with pytest.raises(ValueError, match="data/nyu2_train/0"):
        ni.NyuInputsDataset(data, rows)[0]


def test_collate_stacks_items_and_forms_the_luts():
    its = [{"image": np.full((480, 640, 3), k, np.uint8), "depth": np.full((480, 640), 10 + k, np.uint8),
            "flip": k == 1, "perm": [-1, 4][k], "gamma": [None, 1.1][k]} for k in range(2)]
    b = ni.collate(its)
    assert tuple(b["image"].shape) == (2, 480, 640, 3) and tuple(b["depth"].shape) == (2, 480, 640)
    assert int(b["image"][1, 5, 5, 2]) == 1 and int(b["depth"][0, 0, 0]) == 10
    assert b["flip"].tolist() == [False, True]
    assert b["perm"].tolist() == [[0, 1, 2], list(ni.PERMS[4])]
    assert np.array_equal(b["lut"][0].numpy(), np.arange(256)) and np.array_equal(b["lut"][1].numpy(), ni.gamma_lut(1.1))
    assert np.isnan(float(b["gamma"][0])) and float(b["gamma"][1]) == 1.1


def test_options_are_checked():
    with pytest.raises(ValueError):
        ni.NyuInputs(resample="bilinear")
    assert ni.sizes(False) == ((480, 640), (240, 320)) and ni.sizes(True) == ((224, 224), (224, 224))


def header_text():
    return open(os.path.join(REPO, "include", "wmd_inputs_nyu.h")).read()


def test_header_binding_and_library_agree():
    text = re.sub(r"/\*.*?\*/", "", header_text(), flags=re.S)
    declared = set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", text))
    assert declared == set(_lib.NYU_INPUTS_SIGNATURES), declared ^ set(_lib.NYU_INPUTS_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.LOSS_SIGNATURES, _lib.KITTI_LOSS_SIGNATURES,
                  _lib.HINTS_SIGNATURES, _lib.INPUTS_SIGNATURES):
        assert not declared & set(other)
    lib = _lib.load()
    assert all(hasattr(lib, name) for name in declared)
    for macro, value in (("WMD_NYU_SRC_H", _lib.NYU_SRC_H), ("WMD_NYU_SRC_W", _lib.NYU_SRC_W),
                         ("WMD_NYU_CROP", _lib.NYU_CROP)):
        assert int(re.search(r"#define %s (\d+)" % macro, header_text()).group(1)) == value
    assert "(device memory, %d bytes)" % ni.ITEM_DTYPE.itemsize in header_text()
    # struct wmd_nyu_inputs_desc: nine int32 (padded to 40), then ten pointers
    assert ctypes.sizeof(_lib.NyuInputsDesc) == 40 + 10 * 8


def test_every_nyu_inputs_symbol_is_called_once():
    import inspect
    src = inspect.getsource(ni)
    assert src.count(".wmd_nyu_inputs_u8(") == 1 and ".wmd_nyu_inputs_u8(" in inspect.getsource(ni.NyuInputs._run)


def _desc(N=2, is_224=False):
    d = _lib.NyuInputsDesc()
    fake = 0x1000
    (ih, iw), (dh, dw) = ni.sizes(is_224)
    d.N, d.image_h, d.image_w, d.depth_h, d.depth_w = N, ih, iw, dh, dw
    d.image_xk = d.image_yk = d.depth_xk = d.depth_yk = 5
    for f in ("image_src", "depth_src", "items", "lut", "image_xtab", "image_ytab", "depth_xtab", "depth_ytab", "image",
              "depth"):
        setattr(d, f, fake)
    return d


def test_argument_errors_before_any_cuda_call():
    lib = _lib.load()
    fake = ctypes.c_void_p(0x1000)
    d = _desc()
    ok = lib.wmd_nyu_inputs_ws_bytes(ctypes.byref(d))
    assert ok >= 2 * 448 * (640 * 3 + 320) and lib.wmd_nyu_inputs_ws_bytes(None) == 0
    assert lib.wmd_nyu_inputs_u8(None, fake, ok, None) == -1
    for field, value in (("N", -1), ("N", 65536), ("image_h", 0), ("image_w", 32768), ("depth_h", -3), ("depth_w", 0),
                         ("N", 2331)):                       # 2331 sources of 640x480x3 exceed 2^31 values
        bad = _desc()
        setattr(bad, field, value)
        assert lib.wmd_nyu_inputs_ws_bytes(ctypes.byref(bad)) == 0, (field, value)
        assert lib.wmd_nyu_inputs_u8(ctypes.byref(bad), fake, 1 << 40, None) == -2, (field, value)
    big = _desc(N=1)
    big.image_h = big.image_w = 30000                         # one output of more than 2^31 values
    assert lib.wmd_nyu_inputs_u8(ctypes.byref(big), fake, 1 << 40, None) == -2
    assert lib.wmd_nyu_inputs_ws_bytes(ctypes.byref(_desc(N=2330))) > 0
    for field in ("image_src", "depth_src", "items", "lut", "image_xtab", "image_ytab", "depth_xtab", "depth_ytab",
                  "image", "depth"):
        bad = _desc()
        setattr(bad, field, None)
        assert lib.wmd_nyu_inputs_u8(ctypes.byref(bad), fake, ok, None) == -1, field
    for field in ("image_xk", "image_yk", "depth_xk", "depth_yk"):
        bad = _desc()
        setattr(bad, field, 0)
        assert lib.wmd_nyu_inputs_u8(ctypes.byref(bad), fake, ok, None) == -1, field
    assert lib.wmd_nyu_inputs_u8(ctypes.byref(d), None, ok, None) == -1
    assert lib.wmd_nyu_inputs_u8(ctypes.byref(d), fake, ok - 1, None) == -4
    empty = _desc(N=0)
    for f in ("image_src", "depth_src", "items", "lut", "image", "depth"):
        setattr(empty, f, None)
    assert lib.wmd_nyu_inputs_u8(ctypes.byref(empty), None, 0, None) == 0
