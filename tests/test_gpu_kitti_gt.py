"""GPU: KITTI's ground-truth depths on libwmd.  generate_depth_maps equals generate_depth_map's maps stored in
tests/golden/kitti_gt_*.npz bit for bit (every engineered case, both cameras and vel_depth, the full-size scans by
digest), a mixed batch equals its frames run one by one, the bits repeat, and the CLI writes the export script's file,
which KittiDepthEvaluator scores exactly as it scores the device maps."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import kitti_gt as og
from wavelet_monodepth_b200 import _lib, kitti_gt
from wavelet_monodepth_b200.kitti_eval import KittiDepthEvaluator

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
pytestmark = pytest.mark.gpu


def load(name):
    with np.load(os.path.join(GOLDEN, "kitti_gt_%s.npz" % name)) as f:
        return {k: f[k] for k in f.files}


CALIB, CASES = load("calib"), load("cases")
CASE_NAMES = sorted(str(c) for c in CASES["cases"])


def size(calib):
    return tuple(int(v) for v in CALIB["%s/size" % calib])


def case_map(case, cam, vd):
    H, W = size(str(CASES[case + "/calib"]))
    out = np.zeros(H * W, np.float64)
    out[CASES["%s/%d/%d/index" % (case, cam, vd)]] = CASES["%s/%d/%d/value" % (case, cam, vd)]
    return out.reshape(H, W)


def run(frames, vel_depth):
    """frames: [(points, calib, cam)] -> the device's maps, each cropped to its frame, as fp64 numpy"""
    pts = [f[0] for f in frames]
    offsets = np.concatenate([[0], np.cumsum([p.shape[0] for p in pts])])
    P = np.stack([CALIB["%s/P%d" % (c, cam)] for _, c, cam in frames]) if frames else np.zeros((0, 3, 4))
    sizes = np.array([size(c) for _, c, _ in frames], np.int32).reshape(-1, 2)
    points = torch.from_numpy(np.concatenate(pts) if pts else np.zeros((0, 4), np.float32)).cuda()
    depth = kitti_gt.generate_depth_maps(points, offsets, P, sizes, vel_depth)
    assert depth.dtype == torch.float64 and depth.is_cuda
    out = depth.cpu().numpy()
    for k, (h, w) in enumerate(sizes.tolist()):                   # the padding is +0.0
        pad = out[k].copy()
        pad[:h, :w] = 0
        assert not pad.view(np.int64).any()
    return [out[k, :h, :w] for k, (h, w) in enumerate(sizes.tolist())]


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


@pytest.mark.parametrize("case", CASE_NAMES)
def test_engineered_cases_bit_for_bit(case):
    pts, calib = CASES[case + "/points"], str(CASES[case + "/calib"])
    for vd in (0, 1):
        before = _lib.launch_count()
        got = run([(pts, calib, 2), (pts, calib, 3)], bool(vd))
        assert _lib.launch_count() - before == 2
        for cam, g in zip((2, 3), got):
            assert same_bits(g, case_map(case, cam, vd)), (cam, vd, int((g != case_map(case, cam, vd)).sum()))


def mixed_frames():
    frames = []
    for k, case in enumerate(c for c in CASE_NAMES if c.startswith("date_")):
        pts, calib = CASES[case + "/points"], str(CASES[case + "/calib"])
        frames.append((pts[: 500 + 400 * k], calib, 2 + k % 2))
        frames.append((pts, calib, 3 - k % 2))
    frames.insert(3, (CASES["empty/points"], "toy", 2))
    frames.insert(6, (CASES["wrap/points"], "toy", 3))
    frames.append((og.synthetic_scan(7), "2011_09_26", 2))
    return frames


def test_mixed_batch_equals_frames_one_by_one():
    frames = mixed_frames()
    for vd in (False, True):
        batch = run(frames, vd)
        for f, got in zip(frames, batch):
            assert same_bits(got, run([f], vd)[0])


def test_full_size_scans_against_their_digests():
    full = load("full")
    frames = [(og.synthetic_scan(int(full[d + "/seed"])), d, cam) for d in (str(x) for x in full["dates"])
              for cam in (2, 3)]
    for vd in (0, 1):
        for (_, d, cam), got in zip(frames, run(frames, bool(vd))):
            assert hashlib.sha256(got.tobytes()).hexdigest() == str(full["%s/%d/%d/sha256" % (d, cam, vd)]), (d, cam)


def test_repeatable_and_deterministic():
    frames = mixed_frames()
    a = run(frames, True)
    torch.use_deterministic_algorithms(True)
    try:
        b = run(frames, True)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(same_bits(x, y) for x, y in zip(a, b))


def test_empty_batch():
    before = _lib.launch_count()
    out = kitti_gt.generate_depth_maps(torch.zeros((0, 4), device="cuda"), [0], np.zeros((0, 3, 4)),
                                       np.zeros((0, 2), np.int32))
    assert out.shape[0] == 0 and out.is_cuda and _lib.launch_count() == before


def test_bad_offsets_are_refused():
    pts = torch.zeros((5, 4), device="cuda")
    P, sizes = CALIB["toy/P2"][None], [size("toy")]
    for offsets in ([0, 4], [1, 5], [0, 6], [0, 2, 5]):
        with pytest.raises(_lib.WmdError):
            kitti_gt.generate_depth_maps(pts, offsets, P, sizes)


def test_generate_depth_map_signature(tmp_path):
    calib = "2011_09_28"
    d = str(tmp_path / calib)
    og.write_calib(d, (str(CALIB[calib + "/cam_to_cam"]), str(CALIB[calib + "/velo_to_cam"])))
    pts = CASES["date_%s/points" % calib]
    pts.tofile(str(tmp_path / "scan.bin"))
    for cam in (2, 3):
        got = kitti_gt.generate_depth_map(d, str(tmp_path / "scan.bin"), cam, True)
        assert got.is_cuda and same_bits(got.cpu().numpy(), case_map("date_" + calib, cam, 1))


def test_cli_writes_the_export_fixture_and_the_evaluator_agrees(tmp_path):
    ex = load("export")
    calibs = {str(n): (str(CALIB[n + "/cam_to_cam"]), str(CALIB[n + "/velo_to_cam"])) for n in CALIB["names"]}
    data_path = str(tmp_path / "kitti")
    split = tmp_path / "splits" / "eigen"
    split.mkdir(parents=True)
    (split / "test_files.txt").write_text("\n".join(og.write_tree(data_path, calibs)) + "\n")
    out = str(split / "gt_depths.npz")
    opt = kitti_gt.get_opts(["--data_path", data_path, "--split", "eigen", "--filenames",
                             str(split / "test_files.txt"), "--output", out, "--batch_size", "3",
                             "--num_workers", "2"])
    kitti_gt.run(opt)
    with np.load(out, allow_pickle=True) as f:
        data = f["data"]
    assert data.dtype == object and bool(ex["eigen/object"]) and len(data) == int(ex["eigen/frames"])
    for i, m in enumerate(data):
        assert m.dtype == np.float32 and np.array_equal(m.view(np.int32), ex["eigen/%d" % i].view(np.int32)), i

    # the evaluator on the device maps, and on the file as evaluate_depth.py loads it
    frames = [(og.small_scan(seed, n), date, 2) for date, _, _, seed, n in og.e2e_frames()]
    pts = [f[0] for f in frames]
    offsets = np.concatenate([[0], np.cumsum([p.shape[0] for p in pts])])
    P = np.stack([CALIB["%s/P2" % c] for _, c, _ in frames])
    sizes = np.array([size(c) for _, c, _ in frames], np.int32)
    dev = kitti_gt.generate_depth_maps(torch.from_numpy(np.concatenate(pts)).cuda(), offsets, P, sizes, True)
    from_device = KittiDepthEvaluator([dev[k, :h, :w] for k, (h, w) in enumerate(sizes.tolist())])
    from_file = KittiDepthEvaluator(list(data))
    pred = torch.rand((len(frames), 1, 192, 640), generator=torch.Generator().manual_seed(0)) * 0.3 + 0.01
    pred = pred.cuda()
    summaries = []
    for ev in (from_device, from_file):
        ev.add(pred)
        summaries.append({k: float(v).hex() for k, v in ev.summary().items()})
    assert summaries[0] == summaries[1]
