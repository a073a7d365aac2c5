"""CPU: KITTI's ground-truth export.  oracle.kitti_gt reproduces generate_depth_map's maps stored in
tests/golden/kitti_gt_*.npz bit for bit, kitti_gt's calibration parsing reproduces the reference's P and sizes, its
writer reproduces the export script's gt_depths.npz, include/wmd_gt.h matches its binding and the library, and the
entry point refuses bad arguments before any CUDA call."""
import ctypes
import hashlib
import inspect
import os
import re
import types
from fractions import Fraction

import numpy as np
import pytest

from oracle import kitti_gt as og
from wavelet_monodepth_b200 import _lib, kitti_gt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
NAMES = ("calib", "cases", "full", "export")


def load(name):
    with np.load(os.path.join(GOLDEN, "kitti_gt_%s.npz" % name)) as f:
        return {k: f[k] for k in f.files}


CALIB, CASES = load("calib"), load("cases")


def case_map(case, cam, vd):
    """the reference's map of an engineered case, from its sparse form"""
    H, W = (int(v) for v in CALIB["%s/size" % CASES[case + "/calib"]])
    out = np.zeros(H * W, np.float64)
    out[CASES["%s/%d/%d/index" % (case, cam, vd)]] = CASES["%s/%d/%d/value" % (case, cam, vd)]
    return out.reshape(H, W)


@pytest.mark.parametrize("case", sorted(str(c) for c in CASES["cases"]))
def test_oracle_reproduces_generate_depth_map(case):
    name = str(CASES[case + "/calib"])
    H, W = (int(v) for v in CALIB[name + "/size"])
    for cam in (2, 3):
        for vd in (0, 1):
            got = og.depth_map(CASES[case + "/points"], CALIB["%s/P%d" % (name, cam)], H, W, bool(vd))
            assert np.array_equal(got.view(np.int64), case_map(case, cam, vd).view(np.int64)), (cam, vd)


def test_engineered_cases_reach_their_edges():
    """the fixture holds what the contract's edge cases need: signed zeros kept, ties, the (y, W-1) / (y+1, 0) group"""
    z = np.concatenate([CASES["zeros/%d/1/value" % cam] for cam in (2, 3)])
    assert (np.signbit(z) & (z == 0)).any() and (z > 0).any()
    pts = CASES["ties/points"]
    q = og.project(pts, CALIB["toy/P2"])
    assert (np.abs(q[:, 0] / q[:, 2] % 1) == 0.5).sum() >= 20
    wrap = case_map("wrap", 2, 0)
    assert (wrap[:5, -1] > 0).all() and (wrap[1:, 0] > 0).all()          # rows 0-4 collide with the next row
    assert CASES["empty/points"].shape == (0, 4) and not CASES["outside/2/0/index"].size
    assert CALIB["toy_h1/size"].tolist() == [1, 8] and CALIB["toy_w1/size"].tolist() == [6, 1]


def test_full_size_scans_against_their_digests():
    full = load("full")
    for name in (str(d) for d in full["dates"]):
        pts = og.synthetic_scan(int(full[name + "/seed"]))
        assert hashlib.sha256(pts.tobytes()).hexdigest() == str(full[name + "/points_sha256"])
        assert pts.shape[0] >= 120000
        H, W = (int(v) for v in CALIB[name + "/size"])
        got = og.depth_map(pts, CALIB["%s/P2" % name], H, W, True)
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(full["%s/2/1/sha256" % name])


def test_fma_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a = rng.normal(size=2000) * 10.0 ** rng.integers(-4, 4, 2000)
    b = rng.normal(size=2000).astype(np.float32).astype(np.float64)
    c = rng.normal(size=2000) * 10.0 ** rng.integers(-4, 4, 2000)
    c[:500] = -(a[:500] * b[:500])                                   # cancellation: the product's rounding error
    got = og.fma(a, b, c)
    for i in range(a.size):
        want = float(Fraction(a[i]) * Fraction(b[i]) + Fraction(c[i]))
        assert got[i] == want and np.signbit(got[i]) == np.signbit(want), i


def test_read_calib_file_and_velo_to_image_reproduce_the_reference(tmp_path):
    for name in (str(n) for n in CALIB["names"]):
        d = str(tmp_path / name)
        og.write_calib(d, (str(CALIB[name + "/cam_to_cam"]), str(CALIB[name + "/velo_to_cam"])))
        parsed = kitti_gt.read_calib_file(os.path.join(d, "calib_cam_to_cam.txt"))
        assert parsed["calib_time"] == "09-Jan-2012 13:57:47"
        for cam in (2, 3):
            P, size = kitti_gt.velo_to_image(d, cam)
            assert P.dtype == np.float64 and np.array_equal(P.view(np.int64), CALIB["%s/P%d" % (name, cam)].view(np.int64))
            assert size == tuple(int(v) for v in CALIB[name + "/size"])


def test_writer_reproduces_the_export_scripts_file(tmp_path):
    """the CLI's writer on the oracle's maps (eigen) and on the decoded PNGs (eigen_benchmark) writes the script's
    ``data``: a 1-D object array of float32 maps, bit for bit"""
    ex = load("export")
    calibs = {str(n): (str(CALIB[n + "/cam_to_cam"]), str(CALIB[n + "/velo_to_cam"])) for n in CALIB["names"]}
    maps = []
    for date, drive, frame, seed, n in og.e2e_frames():
        P, (H, W) = og.velo_to_image(og.read_calib_text(calibs[date][0]), og.read_calib_text(calibs[date][1]), 2)
        maps.append(og.depth_map(og.small_scan(seed, n), P, H, W, True).astype(np.float32))
    opt = types.SimpleNamespace(split="eigen_benchmark", data_path=str(tmp_path / "kitti"), batch_size=3,
                                num_workers=0, filenames=str(tmp_path / "bench_files.txt"))
    with open(opt.filenames, "w") as f:
        f.write("\n".join(og.write_benchmark_tree(opt.data_path)) + "\n")
    for split, frames in (("eigen", maps), ("eigen_benchmark", kitti_gt.export(opt))):
        path = str(tmp_path / split / "gt_depths.npz")
        kitti_gt.save_gt_depths(path, frames)
        with np.load(path, allow_pickle=True) as f:
            data = f["data"]
        assert (data.dtype == object) == bool(ex[split + "/object"]) and data.ndim == 1
        assert len(data) == int(ex[split + "/frames"])
        for i, m in enumerate(data):
            want = ex["%s/%d" % (split, i)]
            assert m.dtype == np.float32 and m.shape == want.shape
            assert np.array_equal(m.view(np.int32), want.view(np.int32)), (split, i)


def test_writer_stacks_maps_of_one_size(tmp_path):
    path = str(tmp_path / "gt.npz")
    kitti_gt.save_gt_depths(path, [np.ones((3, 4), np.float64), np.zeros((3, 4), np.float32)])
    with np.load(path) as f:
        assert f["data"].dtype == np.float32 and f["data"].shape == (2, 3, 4)


def test_fixtures_are_small():
    for name in NAMES:
        assert os.path.getsize(os.path.join(GOLDEN, "kitti_gt_%s.npz" % name)) < 1 << 20


def header_symbols():
    text = open(os.path.join(REPO, "include", "wmd_gt.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(wmd_[a-z0-9_]+)\s*\(", text))


def test_header_binding_and_library_agree():
    declared = header_symbols()
    assert declared == set(_lib.GT_SIGNATURES), declared ^ set(_lib.GT_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.LOSS_SIGNATURES, _lib.KITTI_LOSS_SIGNATURES,
                  _lib.HINTS_SIGNATURES, _lib.INPUTS_SIGNATURES, _lib.NYU_INPUTS_SIGNATURES):
        assert not declared & set(other)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name


def test_the_launch_symbol_is_called_from_generate_depth_maps_only():
    assert ".wmd_velo_depth_f64(" in inspect.getsource(kitti_gt.generate_depth_maps)
    assert inspect.getsource(kitti_gt).count(".wmd_velo_depth_f64(") == 1


def test_argument_errors_before_any_cuda_call():
    lib = _lib.load()
    fake = ctypes.c_void_p(0x1000)
    sizes = (ctypes.c_int32 * 4)(375, 1242, 370, 1224)
    ok = lib.wmd_velo_depth_ws_bytes(2, 375, 1242, 240000)
    assert ok >= 20 * 2 * 375 * 1242
    for N, H, W, M in ((-1, 375, 1242, 0), (2, 0, 1242, 0), (2, 375, 0, 0), (2, 375, 1242, -1),
                       (2, 375, 1242, (1 << 30) + 1), (2, 1 << 15, (1 << 15) + 1, 0)):
        assert lib.wmd_velo_depth_ws_bytes(N, H, W, M) == 0, (N, H, W, M)
    assert lib.wmd_velo_depth_f64(fake, fake, fake, sizes, -1, 375, 1242, 1, fake, ok, fake, None) == -2
    assert lib.wmd_velo_depth_f64(fake, fake, fake, sizes, 2, 0, 1242, 1, fake, ok, fake, None) == -2
    assert lib.wmd_velo_depth_f64(fake, fake, fake, sizes, 2, 374, 1242, 1, fake, ok, fake, None) == -2   # frame 0 > Hmax
    assert lib.wmd_velo_depth_f64(fake, fake, fake, sizes, 2, 375, 1241, 1, fake, ok, fake, None) == -2
    bad = (ctypes.c_int32 * 4)(375, 1242, 0, 1224)
    assert lib.wmd_velo_depth_f64(fake, fake, fake, bad, 2, 375, 1242, 1, fake, ok, fake, None) == -2
    for k in range(6):
        args = [fake, fake, fake, sizes]
        tail = [fake, ok, fake]
        if k < 4:
            args[k] = None
        else:
            tail[0 if k == 4 else 2] = None
        assert lib.wmd_velo_depth_f64(*args, 2, 375, 1242, 1, *tail, None) == -1, k
    assert lib.wmd_velo_depth_f64(ctypes.c_void_p(0x1004), fake, fake, sizes, 2, 375, 1242, 1, fake, ok, fake,
                                  None) == -1                                                           # misaligned
    assert lib.wmd_velo_depth_f64(fake, fake, fake, sizes, 2, 375, 1242, 1, fake, ok - 1, fake, None) == -4
    assert lib.wmd_velo_depth_f64(None, None, None, None, 0, 375, 1242, 1, None, 0, None, None) == 0
