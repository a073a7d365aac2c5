"""GPU: KITTI's depth hints on libwmd.  stereo_sgbm equals OpenCV's maps stored in tests/golden/kitti_depth_hints*.npz
bit for bit (every matcher, both sides, mixed-side batches, the smallest widths, one row, full size by digest);
DepthHintGenerator equals oracle.depth_hints' contract mode on every pixel; the CLI writes the script's files."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import depth_hints as odh
from oracle import sgbm
from wavelet_monodepth_b200 import _lib, kitti_hints

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
pytestmark = pytest.mark.gpu


def load(name):
    with np.load(os.path.join(GOLDEN, "kitti_depth_hints_%s.npz" % name)) as f:
        return {k: f[k] for k in f.files}


def batch(items):
    """items: (fixture, key, side) -> base, lookup (N, H, W, 3) uint8 CUDA, right flags, the fixture maps (12, N, H, W)"""
    bases, lookups, rights, maps = [], [], [], []
    for fx, key, side in items:
        base, lookup, rev = odh.views(fx["%s/left" % key], fx["%s/right" % key], side)
        bases.append(base)
        lookups.append(lookup)
        rights.append(rev)
        maps.append(fx["%s/%s/maps" % (key, side)])
    cu = lambda a: torch.from_numpy(np.stack(a)).cuda()                               # noqa: E731
    return cu(bases), cu(lookups), rights, np.stack(maps, 1)


def _mixed():
    a, b = load("a"), load("b")
    return [(a, "a", "l"), (b, "b", "r"), (a, "a", "r"), (b, "b", "l")]


@pytest.mark.parametrize("which", ["ab_mixed", "c", "sample"])
def test_stereo_sgbm_equals_cv2_bit_for_bit(which):
    if which == "ab_mixed":
        items = _mixed()
    elif which == "c":
        c = load("c")
        items = [(c, "c", "r"), (c, "c", "l")]
    else:
        st = load("stages")
        items = [(st, "sample", "l"), (st, "sample", "r")]
    base, lookup, right, want = batch(items)
    for m, (nd, bs) in enumerate(sgbm.MATCHERS):
        got = kitti_hints.stereo_sgbm(base, lookup, nd, bs, reverse=right).cpu().numpy()
        bad = got != want[m]
        assert not bad.any(), (which, nd, bs, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def test_smallest_widths_one_row_and_refusals():
    st = load("stages")
    for nd in sgbm.NUM_DISPARITIES:
        for bs in sgbm.BLOCK_SIZES:
            k = "minw/%d/%d/" % (nd, bs)
            l2, r2 = (torch.from_numpy(st[k + s])[None].cuda() for s in ("left", "right"))
            got = kitti_hints.stereo_sgbm(l2, r2, nd, bs)[0].cpu().numpy()
            assert np.array_equal(got, st[k + "disp"]), (nd, bs)
            with pytest.raises(_lib.WmdError):
                kitti_hints.stereo_sgbm(l2[:, :, :-1].contiguous(), r2[:, :, :-1].contiguous(), nd, bs)
    l1, r1 = (torch.from_numpy(st["row/" + s])[None].cuda() for s in ("left", "right"))
    for m, (nd, bs) in enumerate(sgbm.MATCHERS):
        assert np.array_equal(kitti_hints.stereo_sgbm(l1, r1, nd, bs)[0].cpu().numpy(), st["row/maps"][m]), (nd, bs)


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_full_size_digests():
    """two seeded 320x1024 pairs, both sides, one mixed batch: cv2's twelve maps and the contract fusion's depth"""
    fx = load("full")
    items = []
    for name, (seed, H, W) in odh.FULL.items():
        left, right = odh.make_pair(seed, H, W)
        for side in "lr":
            items.append((name, side) + odh.views(left, right, side))
    base = torch.from_numpy(np.stack([it[2] for it in items])).cuda()
    lookup = torch.from_numpy(np.stack([it[3] for it in items])).cuda()
    right = [it[4] for it in items]
    gen = kitti_hints.DepthHintGenerator(320, 1024)
    maps = gen.disparities(base, lookup, right).cpu().numpy()
    depth, index = gen(base, lookup, right, return_index=True)
    depth, index = depth.cpu().numpy(), index.cpu().numpy()
    for n, (name, side) in enumerate(it[:2] for it in items):
        want = [str(v) for v in fx["%s/%s/maps_sha256" % (name, side)]]
        assert [_digest(maps[m, n]) for m in range(12)] == want, (name, side)
        assert _digest(depth[n:n + 1]) == str(fx["%s/%s/depth_sha256" % (name, side)]), (name, side)
        assert _digest(index[n:n + 1].astype(np.int8)) == str(fx["%s/%s/index_sha256" % (name, side)]), (name, side)


def _fusion_items():
    a, b, c, st = load("a"), load("b"), load("c"), load("stages")
    return {"ab_mixed": _mixed(), "c": [(c, "c", "l"), (c, "c", "r")],
            "sample": [(st, "sample", "r"), (st, "sample", "l")]}


@pytest.mark.parametrize("which", ["ab_mixed", "c", "sample"])
def test_generator_equals_contract_oracle_and_flips_stay_recorded(which):
    items = _fusion_items()[which]
    base, lookup, right, _ = batch(items)
    H, W = base.shape[1:3]
    depth, index = kitti_hints.DepthHintGenerator(H, W)(base, lookup, right, return_index=True)
    depth, index = depth.cpu().numpy(), index.cpu().numpy()
    for n, (fx, key, side) in enumerate(items):
        p = "%s/%s/" % (key, side)
        assert np.array_equal(depth[n].view(np.uint32), fx[p + "contract_depth"].view(np.uint32)), (key, side)
        assert np.array_equal(index[n], fx[p + "contract_index"].astype(np.int32)), (key, side)
        assert int((index[n] != fx[p + "ref_f32_index"]).sum()) <= int(fx[p + "flips_f32"]), (key, side)


def test_two_runs_give_the_same_bits_also_deterministic():
    base, lookup, right, _ = batch(_mixed())
    gen = kitti_hints.DepthHintGenerator(64, 256)
    first = gen(base, lookup, right).cpu()
    maps = gen.disparities(base, lookup, right).cpu()
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        again = gen(base, lookup, right).cpu()
        maps2 = gen.disparities(base, lookup, right).cpu()
    finally:
        torch.use_deterministic_algorithms(was)
    assert torch.equal(first.view(torch.int32), again.view(torch.int32)) and torch.equal(maps, maps2)


def test_empty_batch():
    e = torch.empty((0, 64, 256, 3), dtype=torch.uint8, device="cuda")
    assert kitti_hints.stereo_sgbm(e, e, 96, 2).shape == (0, 64, 256)
    assert kitti_hints.DepthHintGenerator(64, 256)(e, e, []).shape == (0, 1, 64, 256)


def test_cli_writes_the_scripts_files(tmp_path):
    """synthetic JPEGs in KITTI's raw layout; the CLI's files have the script's paths, shape (1, H, W) and dtype, their
    values are the generator's on the same decoded views, existing files are skipped unless overwriting"""
    from PIL import Image
    H, W = 64, 256
    data, lines = tmp_path / "raw", []
    for k, (seq, frame) in enumerate((("2011_09_26/2011_09_26_drive_0001_sync", 5),
                                      ("2011_09_26/2011_09_26_drive_0002_sync", 17))):
        left, right = odh.make_pair(900 + k, 80, 300)
        for cam, img in (("image_02", left), ("image_03", right)):
            d = data / seq / cam / "data"
            d.mkdir(parents=True, exist_ok=True)
            Image.fromarray(img).save(d / ("%010d.jpg" % frame), quality=95)
        lines += ["%s %d l" % (seq, frame), "%s %d r" % (seq, frame)]
    split = tmp_path / "files.txt"
    split.write_text("\n".join(lines) + "\n")
    out = tmp_path / "hints"
    argv = ["--data_path", str(data), "--filenames", str(split), "--save_path", str(out), "--height", str(H),
            "--width", str(W), "--batch_size", "3", "--num_workers", "0"]
    assert kitti_hints.run(kitti_hints.get_opts(argv)) == (4, 0)
    gen = kitti_hints.DepthHintGenerator(H, W)
    for line in lines:
        base_p, lookup_p, npy, right = kitti_hints.view_paths(str(data), str(out), line)
        seq, frame, side = line.split()
        assert npy == os.path.join(str(out), seq, "image_03" if side == "r" else "image_02", "%010d.npy" % int(frame))
        got = np.load(npy)
        assert got.shape == (1, H, W) and got.dtype == np.float32
        views = [torch.from_numpy(kitti_hints.load_view(p, H, W))[None].cuda() for p in (base_p, lookup_p)]
        want = gen(views[0], views[1], [right])[0].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), line
    # skip: existing files are left alone; overwrite: they are recomputed
    stamp = np.full((1, H, W), 7.0, np.float32)
    first = kitti_hints.view_paths(str(data), str(out), lines[0])[2]
    np.save(first, stamp)
    assert kitti_hints.run(kitti_hints.get_opts(argv)) == (0, 4)
    assert np.array_equal(np.load(first), stamp)
    assert kitti_hints.run(kitti_hints.get_opts(argv + ["--overwrite_saved_depths"])) == (4, 0)
    assert not np.array_equal(np.load(first), stamp)
