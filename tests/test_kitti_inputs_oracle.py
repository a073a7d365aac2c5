"""CPU: KITTI's training inputs.  oracle.kitti_inputs equals the installed Pillow bit for bit (LANCZOS tables and the
resample chain at the five raw sizes, blends over all 256 values, RGB -> L, RGB -> HSV and HSV -> RGB over all 2^24
colours, hue shifts both ways), the golden fixtures reproduce from it, KittiInputsDataset makes the reference's draws,
include/wmd_inputs.h matches its binding and the library, and wmd_inputs_u8 refuses bad arguments before any CUDA call."""
import ctypes
import os
import random
import re

import numpy as np
import pytest
from PIL import Image, ImageEnhance

from oracle import kitti_inputs as oki
from wavelet_monodepth_b200 import _lib
from wavelet_monodepth_b200 import kitti_inputs as ki

import kitti_inputs_cases as kic

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("hw", oki.RAW_SIZES, ids=lambda hw: "%dx%d" % (hw[1], hw[0]))
def test_tables_and_resample_chain_equal_pillow(hw):
    view = oki.synthetic_view(hw[1], *hw)
    for height, width in ((192, 640), (320, 1024)):
        for flip in (False, True):
            img = Image.fromarray(np.ascontiguousarray(view[:, ::-1] if flip else view))
            pyr = oki.pyramid(view, height, width, (0, 1, 2, 3), flip)
            for s in range(4):
                img = img.resize((width >> s, height >> s), Image.LANCZOS)
                assert np.array_equal(np.asarray(img), pyr[s]), (height, width, flip, s)
    for n_in, n_out in ((hw[1], 640), (hw[0], 192), (hw[1], 1024), (hw[0], 320), (640, 320), (96, 48), (7, 7)):
        bounds, coeffs = oki.lanczos_table(n_in, n_out)
        tab = ki.lanczos_table(n_in, n_out)
        assert np.array_equal(tab[:, :2], bounds) and np.array_equal(tab[:, 2:], coeffs), (n_in, n_out)


# the factor ends of the reference's ranges, 0 and 1, and float32 neighbours of the interpolate / extrapolate switch
FACTORS = (0.8, 1.2, 0.0, 1.0, -0.0, float(np.nextafter(np.float32(1), np.float32(2))),
           float(np.nextafter(np.float32(1), np.float32(0))), 1.0 + 2.0 ** -30, -1e-9, 0.5, 2.0, -0.5)


@pytest.mark.parametrize("factor", FACTORS)
def test_blend_over_all_values(factor):
    a, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    got = np.asarray(Image.blend(Image.fromarray(a), Image.fromarray(b), factor))
    assert np.array_equal(got, oki.blend(a, b, factor))


@pytest.mark.parametrize("op", range(4))
def test_enhance_ops_equal_pillow_and_torchvision(op):
    import torchvision.transforms.functional as TF
    img = oki.synthetic_view(9, 96, 160)
    factors = (0.8, 1.2, 1.0, 0.93) if op < 3 else (-0.1, 0.1, -0.05, 0.0, 0.0501, -0.5, 0.5)
    for f in factors:
        pil = Image.fromarray(img)
        want = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)[op](pil, f)
        assert np.array_equal(np.asarray(want), oki.adjust(img, op, f)), (op, f)
    if op == 1:
        assert oki.contrast_mean(img) == int(np.mean(np.asarray(Image.fromarray(img).convert("L"))) + 0.5)
        enh = ImageEnhance.Contrast(Image.fromarray(img)).degenerate
        assert np.asarray(enh)[0, 0, 0] == oki.contrast_mean(img)


def test_hue_shift_byte():
    assert [oki.hue_shift(h) for h in (-0.05, 0.05, -0.1, 0.1, 0.0, -0.0039)] == [244, 12, 231, 25, 0, 0]
    assert all(ki.hue_shift(h) == oki.hue_shift(h) for h in np.linspace(-0.5, 0.5, 1001))


@pytest.fixture(scope="module")
def all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def test_rgb_to_l_exhaustive(all_colours):
    assert np.array_equal(np.asarray(Image.fromarray(all_colours).convert("L")), oki.rgb_to_l(all_colours))


def test_rgb_to_hsv_exhaustive(all_colours):
    assert np.array_equal(np.asarray(Image.fromarray(all_colours).convert("HSV")), oki.rgb_to_hsv(all_colours))


def test_hsv_to_rgb_exhaustive(all_colours):
    got = np.asarray(Image.fromarray(all_colours, "HSV").convert("RGB"))
    assert np.array_equal(got, oki.hsv_to_rgb(all_colours))


@pytest.mark.parametrize("name", kic.CASES)
def test_fixtures_reproduce_from_the_oracle(name):
    fx = kic.load(name)
    cfg = fx["config"]
    its = kic.items(fx)
    exp = [oki.expected(it["views"], (it["do_color_aug"], it["do_flip"], it["jitter"]), it["side"], it.get("hint"),
                        cfg["height"], cfg["width"], cfg["scales"], cfg["use_depth_hints"]) for it in its]
    assert kic.mismatches(fx, lambda n: exp[n]) == []
    planes = np.stack([np.stack([np.rint(e[("color_aug", f, 3)] * 255).astype(np.uint8) for f in cfg["frame_idxs"]])
                       for e in exp])
    assert np.array_equal(planes, fx["planes"])
    assert os.path.getsize(os.path.join(kic.GOLDEN, "kitti_inputs_%s.npz" % name)) < 1 << 20


def test_dataset_makes_the_references_draws(tmp_path):
    """a tree of the train640 fixture's items: the draws of a seeded KittiInputsDataset are the reference's"""
    fx = kic.load("train640")
    cfg = fx["config"]
    for n, line in enumerate(fx["lines"]):
        seq, frame, side = str(line).split()
        for k, f in enumerate(cfg["frame_idxs"]):
            cam = {"l": 2, "r": 3}[{"r": "l", "l": "r"}[side] if f == "s" else side]
            path = tmp_path / seq / ("image_0%d" % cam) / "data" / ("%010d.png" % (int(frame) + (0 if f == "s" else f)))
            path.parent.mkdir(parents=True, exist_ok=True)
            Image.fromarray(oki.synthetic_view(*map(int, fx["views"][n, k]))).save(path)
    random.seed(7)                                                 # oracle.pin_kitti_inputs' seed of this case
    ds = ki.KittiInputsDataset(str(tmp_path) + "/", [str(x) for x in fx["lines"]], cfg["height"], cfg["width"],
                               cfg["frame_idxs"], cfg["scales"], is_train=True, img_ext=".png")
    for n in range(len(ds)):
        it = ds[n]
        assert (it["do_color_aug"], it["do_flip"]) == (bool(fx["do_color_aug"][n]), bool(fx["do_flip"][n]))
        if it["do_color_aug"]:
            assert it["jitter"] == (tuple(fx["factors"][n]), tuple(fx["order"][n]))
        assert it["image_path"] == str(fx["image_path"][n])
        for k, f in enumerate(cfg["frame_idxs"]):
            assert np.array_equal(it["views"][f], oki.synthetic_view(*map(int, fx["views"][n, k])))


def test_collate_pads_frame_major():
    its = [{"views": {0: np.full((3, 5, 3), 10 * k, np.uint8), "s": np.full((2, 4, 3), 10 * k + 1, np.uint8)},
            "do_color_aug": k == 1, "do_flip": k == 0, "jitter": ((1.1, 0.9, 1.0, 0.05), (2, 0, 3, 1)) if k == 1 else None,
            "side": "l", "image_path": str(k)} for k in range(2)]
    b = ki.collate(its)
    assert tuple(b["src"].shape) == (4, 3, 5, 3)
    assert b["sizes"].tolist() == [[3, 5], [3, 5], [2, 4], [2, 4]]
    assert [int(b["src"][v, 0, 0, 0]) for v in range(4)] == [0, 10, 1, 11]
    assert int(b["src"][2, 2:, :].sum()) == 0 and int(b["src"][2, :, 4:].sum()) == 0
    assert b["order"].tolist() == [[-1] * 4, [2, 0, 3, 1]] and b["do_flip"].tolist() == [True, False]


def test_camera_and_hint_helpers_agree_with_the_oracle():
    import cv2
    for h0, w0, H, W in ((188, 621, 192, 640), (375, 1242, 320, 1024), (320, 1024, 320, 1024), (10, 7, 3, 20)):
        assert np.array_equal(ki.nearest_index(w0, W), oki.nearest_index(w0, W))
        src = np.arange(h0 * w0, dtype=np.float32).reshape(h0, w0)
        want = cv2.resize(src, dsize=(W, H), interpolation=cv2.INTER_NEAREST)
        assert np.array_equal(src[oki.nearest_index(h0, H)][:, oki.nearest_index(w0, W)], want), (h0, w0, H, W)
    for k, v in ki.cameras(192, 640, (0, 1, 2, 3)).items():
        assert np.array_equal(v, oki.cameras(192, 640, (0, 1, 2, 3))[k]) and v.dtype == np.float32


def header_text():
    return open(os.path.join(REPO, "include", "wmd_inputs.h")).read()


def test_header_binding_and_library_agree():
    text = re.sub(r"/\*.*?\*/", "", header_text(), flags=re.S)
    declared = set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", text))
    assert declared == set(_lib.INPUTS_SIGNATURES), declared ^ set(_lib.INPUTS_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.LOSS_SIGNATURES, _lib.KITTI_LOSS_SIGNATURES,
                  _lib.HINTS_SIGNATURES):
        assert not declared & set(other)
    lib = _lib.load()
    assert all(hasattr(lib, name) for name in declared)
    assert int(re.search(r"#define WMD_INPUTS_MAX_SCALES (\d+)", header_text()).group(1)) == _lib.INPUTS_MAX_SCALES
    assert "(device memory, %d bytes)" % ki.VIEW_DTYPE.itemsize in header_text()
    assert "(device memory, %d bytes)" % ki.JITTER_DTYPE.itemsize in header_text()
    # struct wmd_inputs_desc: 4 + 8 int32, then pointers and int32 arrays at their natural alignment
    assert ctypes.sizeof(_lib.InputsDesc) == 48 + 8 * 2 + 8 * 8 + 4 * 8 + 8 + 8 * 8


def test_every_inputs_symbol_is_called_once():
    import inspect
    src = inspect.getsource(ki)
    assert src.count(".wmd_inputs_u8(") == 1 and ".wmd_inputs_u8(" in inspect.getsource(ki.KittiInputs._run)


def _desc(N=2, n_scales=4):
    d = _lib.InputsDesc()
    fake = 0x1000
    d.N, d.src_h, d.src_w, d.n_scales = N, 376, 1242, n_scales
    d.src = d.views = d.jitter = fake
    for j in range(4):
        d.out_h[j], d.out_w[j] = 192 >> j, 640 >> j
        d.xtab[j] = d.ytab[j] = d.color[j] = d.color_aug[j] = fake
        d.xk[j] = d.yk[j] = 13
    return d


def test_argument_errors_before_any_cuda_call():
    lib = _lib.load()
    fake = ctypes.c_void_p(0x1000)
    d = _desc()
    ok = lib.wmd_inputs_ws_bytes(ctypes.byref(d))
    assert ok > 0 and lib.wmd_inputs_ws_bytes(None) == 0
    assert lib.wmd_inputs_u8(None, fake, ok, None) == -1
    for field, value in (("N", -1), ("N", 65536), ("n_scales", 0), ("n_scales", 5), ("src_h", 0), ("src_w", 40000)):
        bad = _desc()
        setattr(bad, field, value)
        assert lib.wmd_inputs_ws_bytes(ctypes.byref(bad)) == 0, field
        assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, 1 << 40, None) == -2, field
    bad = _desc()
    bad.out_w[2] = 0
    assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, 1 << 40, None) == -2
    bad = _desc(N=30000)                                    # a stage of more than 2^31 values
    assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, 1 << 40, None) == -2
    for field in ("src", "views", "jitter"):
        bad = _desc()
        setattr(bad, field, None)
        assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, ok, None) == -1, field
    for arr in ("color", "color_aug", "xtab", "ytab"):
        bad = _desc()
        getattr(bad, arr)[3] = None
        assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, ok, None) == -1, arr
    bad = _desc()
    bad.xk[1] = 0
    assert lib.wmd_inputs_u8(ctypes.byref(bad), fake, ok, None) == -1
    assert lib.wmd_inputs_u8(ctypes.byref(d), None, ok, None) == -1
    assert lib.wmd_inputs_u8(ctypes.byref(d), fake, ok - 1, None) == -4
    assert lib.wmd_inputs_u8(ctypes.byref(_desc(N=0)), None, 0, None) == 0
    one = _desc(n_scales=1)
    one.color[1] = one.xtab[1] = None                       # stages past n_scales are not read
    assert lib.wmd_inputs_u8(ctypes.byref(one), fake, 0, None) == -4


def test_target_scales_are_checked():
    for bad in ((-1, 0), (0, 0), (4,), ()):
        with pytest.raises(ValueError):
            ki.KittiInputs(192, 640, [0], bad)
