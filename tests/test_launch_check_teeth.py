"""The launch checkers of the evaluation, loss and data-pipeline entry points (tests/launch_check.py) have teeth: each
passes the oracle's own answer and raises LaunchError when one element of it is changed by the smallest step its bar
must see (a loss gradient one ulp off, one edge pixel toggled, one a_k count off by one, one KITTI median ratio one ulp
off, one KITTI loss mask pixel toggled, one SGBM disparity 1/16 px off, one fused depth one ulp off or its matcher index
changed, one input colour element one ulp off, one hint pixel toggled, one ground-truth depth one ulp off or one empty
ground-truth pixel given a depth).  CPU only: the checkers are called directly on CPU tensors, with stand-ins for the
evaluators' state; no GPU and no libwmd.

The footprint checks have teeth too, on CPU tensors the test owns (footprint.Footprint("cpu")): a write one element
into either guard, a poisoned cell that reaches a result, a channels_last buffer with the wrong strides, a changed input
that WRITES does not name, and a nonzero byte in a workspace's counter header are each caught."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import depth_hints as odh
from oracle import kitti_eval as oke
from oracle import kitti_gt as okg
from oracle import kitti_inputs as oki
from oracle import kitti_loss as okl
from oracle import nyu_edges as ne
from oracle import nyu_eval as one
from oracle import nyu_inputs as oni
from oracle import nyu_loss as onl
from oracle import sgbm as osgbm
from wavelet_monodepth_b200 import kitti_inputs as ki
from wavelet_monodepth_b200 import nyu_inputs as ni
from wavelet_monodepth_b200 import ops

import footprint
import kitti_inputs_cases as kic
import launch_check as lc
import nyu_inputs_cases as nic
from workloads import same


@pytest.fixture
def harness():
    """A Harness without its libwmd plumbing: the checkers only read the workload's name."""
    saved = dict(lc.REPORT)
    h = object.__new__(lc.Harness)
    h.current = "teeth"
    yield h
    lc.REPORT.clear()
    lc.REPORT.update(saved)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def ulp_up(a, index):
    """a copy of float array a with element `index` moved one ulp away from zero"""
    b = np.array(a, copy=True)
    b[index] = np.nextafter(b[index], np.copysign(np.inf, b[index]), dtype=b.dtype)
    return b


def both(check, good, bad):
    """check(good) passes; check(bad) raises LaunchError"""
    check(*good)
    with pytest.raises(lc.LaunchError):
        check(*bad)


# ------------------------------------------------------------------------------------------ NYUv2 training loss
def _loss_case():
    rng = np.random.default_rng(0)
    n, H, W = 2, 16, 24
    target = rng.uniform(10.0, 1000.0, (n, 1, H, W)).astype(np.float32)
    preds = [(target[..., ::1 << s, ::1 << s] * rng.uniform(0.7, 1.3, (n, 1, H >> s, W >> s))).astype(np.float32)
             for s in onl.SCALES]
    means = np.array([onl.term(p[:, 0], target[:, 0]) for p in preds], np.float32)
    signs = np.stack([onl.signs(onl.upsample(p[:, 0], H, W), target[:, 0]) for p in preds])
    return target, preds, means, signs


def test_loss_fwd_checker(harness):
    target, preds, means, signs = _loss_case()

    def call(means, signs):
        a = dict(target=t(target), preds=[t(p) for p in preds], log2s=onl.SCALES, means=t(means), want_signs=True)
        harness._check_loss_fwd(a, t(signs), None)
    both(call, (means, signs), (ulp_up(ulp_up(means, 2), 2), signs))     # one term two ulp off
    flipped = signs.copy()
    flipped[1, 0, 5, 7] = -flipped[1, 0, 5, 7] if flipped[1, 0, 5, 7] else 1
    both(call, (means, signs), (means, flipped))                          # one sign wrong


def test_loss_bwd_checker(harness):
    target, preds, _, signs = _loss_case()
    n, _, H, W = target.shape
    g = np.full(len(preds), 0.1, np.float32)
    grads = [(np.float64(g[k]) / np.float64(n * H * W) * onl.adjoint(signs[k], p.shape[2], p.shape[3]))
             .astype(np.float32)[:, None] for k, p in enumerate(preds)]

    def call(grads):
        a = dict(signs=t(signs), target_shape=(n, 1, H, W), preds=[t(p) for p in preds], log2s=onl.SCALES,
                 grad_means=t(g))
        harness._check_loss_bwd(a, [t(x) for x in grads], None)
    bad = list(grads)
    bad[2] = ulp_up(grads[2], (1, 0, 3, 4))                               # one gradient one ulp off
    assert grads[2][1, 0, 3, 4] != 0
    both(call, (grads,), (bad,))


# ------------------------------------------------------------------------------------------ NYUv2 evaluation
def test_nyu_evaluator_add_checker(harness):
    split = one.synthetic_split(0, n=2)
    disp = split["disp"][(60, 80, False)]
    gt = one.prepare_gt(split["gt"])
    gt_log10 = torch.log10(t(gt))
    depth = one.predict(disp)
    sums = one.frame_sums(depth, gt, gt_log10.numpy())
    assert sums[:, 3].min() > 0

    def call(depth_out, sums_out):
        ev = types.SimpleNamespace(gt=t(gt), gt_log10=gt_log10, sums=t(sums_out), use_224=False, use_disparity=False,
                                   next_frame=2)
        pre = (0, torch.full_like(ev.sums, float("nan")))
        harness._check_NyuDepthEvaluator_add(dict(self=ev, disp=t(disp)[:, None], depth_out=t(depth_out)), None, pre)
    count_off = sums.copy()
    count_off[1, 4] += 1                                                  # one a_2 count off by one
    both(call, (depth, sums), (depth, count_off))
    both(call, (depth, sums), (ulp_up(depth, (0, 100, 200)), sums))       # one map value one ulp off
    rel_off = sums.copy()
    rel_off[0, 0] *= 1 + 1e-11                                            # a sum past its 1e-12 bar
    both(call, (depth, sums), (depth, rel_off))


def test_compute_errors_nyu_checker(harness):
    rng = np.random.default_rng(1)
    gt = rng.uniform(0.5, 10.0, 5000)
    pred = gt * rng.uniform(0.6, 1.6, 5000)
    want = one.compute_errors_nyu(pred, gt)
    off = want.copy()
    off[3] += 1.0 / 5000                                                  # one a_1 count off by one

    def call(out):
        harness._check_compute_errors_nyu(dict(pred=t(pred), gt=t(gt)), t(out), None)
    both(call, (want,), (off,))


def _edge_case():
    rng = np.random.default_rng(2)
    h, w = 40, 56
    yy, xx = np.mgrid[0:h, 0:w] / np.array([h - 1, w - 1])[:, None, None]
    frames = []
    for k in range(2):
        d = 2.0 + yy + 0.5 * np.sin(6 * xx + k)
        d[h // 4:h // 2 + 1, w // 3:2 * w // 3 + 1] += 2.0
        frames.append((d * rng.uniform(0.97, 1.03, (h, w))).astype(np.float32))
    pred = np.stack(frames)
    edges_gt = np.stack([ne.step_edges(p, 0.5) for p in pred]).astype(np.float32)
    res = [ne.dbe(edges_gt[i], pred[i]) for i in range(2)]
    est = np.stack([r[2] for r in res])
    assert est.sum() > 0 and np.isfinite([r[:2] for r in res]).all()
    return pred, edges_gt, est, np.stack([r[3] for r in res]), np.array([r[:2] for r in res])


def test_edges_frames_checker(harness):
    pred, edges_gt, est, d_est, scores = _edge_case()

    def call(est, d_est, scores):
        a = dict(pred=t(pred.astype(np.float64)), edges_gt=t(edges_gt), scores=t(scores), low=ne.LOW, high=ne.HIGH)
        harness._check_edges_frames(a, (t(est), t(d_est)), None)
    toggled = est.copy()
    toggled[1, 10, 20] = ~toggled[1, 10, 20]                              # one edge pixel toggled
    both(call, (est, d_est, scores), (toggled, d_est, scores))
    both(call, (est, d_est, scores), (est, ulp_up(d_est, (0, 3, 3)), scores))
    off = scores.copy()
    off[0, 1] *= 1 + 1e-11
    both(call, (est, d_est, scores), (est, d_est, off))


def test_edt_checker(harness):
    _, _, est, d_est, _ = _edge_case()
    feats = est.astype(np.uint8)
    feats[1] = 0                                                          # no feature pixel: scipy's own answer
    dist = np.stack([ne.edt(f) for f in feats != 0])

    def call(dist):
        harness._check_edt(dict(features=t(feats)), t(dist), None)
    both(call, (dist,), (ulp_up(dist, (1, 7, 9)),))


# ------------------------------------------------------------------------------------------ KITTI evaluation
def _kitti_case():
    rng = np.random.default_rng(3)
    frames = []
    for H, W in ((40, 120), (38, 124)):
        lidar = rng.random((H, W)) < 0.3
        frames.append(np.where(lidar, rng.uniform(0.0, 100.0, (H, W)), 0.0).astype(np.float32))
    hm, wm = 40, 124
    padded = np.zeros((2, hm, wm), np.float32)
    for i, f in enumerate(frames):
        padded[i, :f.shape[0], :f.shape[1]] = f
    mask = np.zeros(padded.shape, bool)
    for i, f in enumerate(frames):
        mask[i, :f.shape[0], :f.shape[1]] = oke.valid_mask(f, "eigen")
    pixels = np.flatnonzero(mask).astype(np.int32)
    offsets = np.concatenate([[0], np.cumsum(mask.reshape(2, -1).sum(1))]).astype(np.int32)
    ev = types.SimpleNamespace(h_max=hm, w_max=wm, hw=t(np.array([f.shape for f in frames], np.int32)),
                               offsets=t(offsets), pixels=t(pixels), gt=t(padded.reshape(-1)[pixels]),
                               eval_split="eigen", median_scaling=True, pred_depth_scale_factor=1.0)
    assert offsets[1] > 10 and offsets[2] > offsets[1] + 10
    return frames, ev


def test_kitti_evaluator_init_checker(harness):
    frames, ev = _kitti_case()

    def call(offsets):
        e = types.SimpleNamespace(**dict(vars(ev), offsets=t(offsets)))
        harness._check_KittiDepthEvaluator_init(dict(self=e, gt_depths=frames, eval_split="eigen"), None, None)
    off = ev.offsets.numpy().copy()
    bad = off.copy()
    bad[1] += 1                                                           # one frame's valid count off by one
    both(call, (off,), (bad,))


def test_kitti_evaluator_add_checker(harness):
    frames, ev = _kitti_case()
    rng = np.random.default_rng(4)
    disp = (0.3 / rng.uniform(3.0, 60.0, (2, 16, 48))).astype(np.float32)
    want = [oke.evaluate_frame(g, d) for g, d in zip(frames, disp)]
    errors = np.stack([w[0] for w in want])
    ratios = np.array([w[1] for w in want])
    counts = np.array([w[2] for w in want], np.int32)

    def call(errors, ratios, counts):
        e = types.SimpleNamespace(**dict(vars(ev), errors=t(errors), ratios=t(ratios), counts=t(counts), next_frame=2))
        pre = (0, [torch.full((2, 7), float("nan"), dtype=torch.float64), torch.full((2,), float("nan"),
                   dtype=torch.float64), torch.zeros(2, dtype=torch.int32)])
        harness._check_KittiDepthEvaluator_add(dict(self=e, pred_disp=t(disp)), None, pre)
    both(call, (errors, ratios, counts), (errors, ulp_up(ratios, 1), counts))       # one median ratio one ulp off
    c = counts.copy()
    c[0] += 1
    both(call, (errors, ratios, counts), (errors, ratios, c))
    a1 = errors.copy()
    a1[1, 4] += 1.0 / counts[1]                                           # one a1 count off by one
    both(call, (errors, ratios, counts), (a1, ratios, counts))


def test_post_process_checker(harness):
    l_disp, r_disp = oke.post_process_inputs(5, n=2, h=8, w=16)
    r = r_disp[:, :, ::-1]
    want = oke.batch_post_process_disparity(l_disp, r)
    off = want.copy()
    off[1, 3, 5] *= 1 + 1e-14

    def call(out):
        harness._check_batch_post_process_disparity(dict(l_disp=t(l_disp), r_disp=t(r)), t(out), None)
    both(call, (want,), (off,))


def test_kitti_compute_errors_checker(harness):
    rng = np.random.default_rng(6)
    gt = rng.uniform(1.0, 80.0, 3000)
    pred = gt * rng.uniform(0.6, 1.6, 3000)
    want = np.array(oke.compute_errors(gt, pred))
    off = want.copy()
    off[6] -= 1.0 / 3000                                                  # one a3 count off by one

    def call(out):
        harness._check_compute_errors(dict(gt=t(gt), pred=t(pred)), t(out), None)
    both(call, (want,), (off,))


# ------------------------------------------------------------------------------------------ KITTI training loss
def _kitti_loss_case():
    """a 2-frame 32x48 case with a different camera per frame and loss scales (0, 1, 3), the call's arguments as
    kitti_loss._kitti_fwd / _kitti_bwd receive them (CPU tensors), and the contract-mode oracle's answer"""
    case = dict(N=2, H=32, W=48, scales=okl.SCALES, loss_scales=(0, 1, 3), camera=True)
    inp, disps = okl.make_inputs(case, 21)
    noise = okl.draw_noise(21, inp, case["loss_scales"])
    ls, opt = case["loss_scales"], (0.5, 80.0, 0.1)
    tt = {k: t(inp[k]) for k in ("target", "source", "K", "inv_K", "stereo_T", "depth_hint", "depth_hint_mask")}
    tt.update(color=[t(inp["colors"][s]) for s in ls], disp=[t(disps[s]) for s in ls], noise=[t(noise[s]) for s in ls])
    gt = np.array(okl.term_weights(ls), np.float32)
    o = okl.run(inp, disps, noise, okl.SCALES, ls, min_depth=0.5, max_depth=80.0, disparity_smoothness=0.1,
                grad_terms=gt)
    a = dict(t=tt, scales=okl.SCALES, loss_scales=ls, opt=opt)
    return a, o, gt


def test_kitti_fwd_checker(harness):
    a, o, _ = _kitti_loss_case()
    ls = a["loss_scales"]
    terms = np.array([o[k] for k in okl.term_keys(ls)], np.float32)
    masks = [np.stack([o[key][s] for s in ls])[:, :, None].astype(np.float32)
             for key in ("identity_selection", "depth_hint_pixels")]
    assert masks[1].sum() > 0 and masks[0].sum() > 0
    warped = np.stack([o["warped"][s] for s in ls]).astype(np.float32)

    def call(terms, idsel, hpix):
        res = (t(terms), t(o["color_depth_hint"].astype(np.float32)), t(warped), t(idsel), t(hpix), None)
        harness._check_kitti_fwd(a, res, None)
    both(call, (terms, *masks), (ulp_up(ulp_up(terms, 5), 5), *masks))     # one term two ulp off
    for k in (0, 1):
        toggled = [m.copy() for m in masks]
        toggled[k][1, 1, 0, 7, 9] = 1 - toggled[k][1, 1, 0, 7, 9]        # one mask pixel toggled
        both(call, (terms, *masks), (terms, *toggled))


def test_kitti_bwd_checker(harness):
    a, o, gt = _kitti_loss_case()
    ls = a["loss_scales"]
    idsel, hpix = (t(np.stack([o[key][s] for s in ls])[:, :, None].astype(np.float32))
                   for key in ("identity_selection", "depth_hint_pixels"))
    grads = [o["grad"][s].astype(np.float32) for s in ls]
    a = dict(a, grad_terms=t(gt), idsel=idsel, hpix=hpix)

    def call(grads, idsel=idsel):
        harness._check_kitti_bwd(dict(a, idsel=idsel), [t(g) for g in grads], None)
    for i, s in enumerate(ls):
        # the scale's largest gradient one ulp farther from the oracle's fp64 value
        want = o["grad"][s]
        j = np.unravel_index(np.argmax(np.abs(want)), want.shape)
        bad = list(grads)
        bad[i] = grads[i].copy()
        bad[i][j] = np.nextafter(grads[i][j], np.float32(np.inf if grads[i][j] >= want[j] else -np.inf))
        both(call, (grads,), (bad,))
    toggled = idsel.clone()
    toggled[0, 0, 0, 3, 4] = 1 - toggled[0, 0, 0, 3, 4]                   # one mask pixel toggled
    both(call, (grads,), (grads, toggled))


# ------------------------------------------------------------------------------------------ KITTI depth hints
def _hint_pair():
    """the 64x256 pair of tests/golden/kitti_depth_hints_a.npz as one mixed batch: its left view and its mirrored right
    view, with the twelve matchers' maps OpenCV made of each"""
    with np.load(os.path.join(kic.GOLDEN, "kitti_depth_hints_a.npz")) as f:
        left, right = f["a/left"], f["a/right"]
        maps = np.stack([f["a/l/maps"], f["a/r/maps"]], 1)
    base, lookup = np.stack([left, right]), np.stack([right, left])
    return base, lookup, maps, [False, True]


def test_stereo_sgbm_checker(harness):
    base, lookup, _, right = _hint_pair()
    want = np.stack([osgbm.compute_side(base[i], lookup[i], 96, 2, right[i]) for i in range(2)])
    assert (want != -16).mean() > 0.3

    def call(out):
        a = dict(left=t(base), right=t(lookup), num_disparities=96, block_size=2, reverse=right, out=None)
        harness._check_stereo_sgbm(a, t(out), None)
    moved = want.copy()
    moved[1, 30, 200] += 1                                                # one disparity 1/16 px off
    both(call, (want,), (moved,))
    border = want.copy()
    border[0, 0, 0] = 0                                                   # one unwritten border pixel written
    assert want[0, 0, 0] == -16
    both(call, (want,), (border,))


def test_fuse_checker(harness):
    base, lookup, maps, right = _hint_pair()
    K, inv_K, T = odh.cameras(64, 256, right)
    depth, index, _ = odh.fuse(base, lookup, maps, right, mode="contract")
    index = index.astype(np.int32)
    assert depth[0, 0, 20, 100] > 0 and len(np.unique(index)) > 2

    def call(depth, index):
        a = dict(base=t(base), lookup=t(lookup), maps=t(maps), K=t(K), inv_K=t(inv_K), T=t(T), depth=t(depth),
                 index=t(index))
        harness._check_fuse(a, None, None)
    both(call, (depth, index), (ulp_up(depth, (0, 0, 20, 100)), index))  # one fused depth one ulp off
    changed = index.copy()
    changed[1, 0, 40, 60] = (changed[1, 0, 40, 60] + 1) % 12              # one matcher index changed
    both(call, (depth, index), (depth, changed))


# ------------------------------------------------------------------------------------------ training inputs
def test_kitti_inputs_checker(harness):
    """two items of the train640 fixture (both frames, flips, jitter, hints) at 640x192"""
    fx = kic.load("train640")
    cfg = fx["config"]
    items = kic.items(fx)[:2]
    fn = ki.KittiInputs(cfg["height"], cfg["width"], cfg["frame_idxs"], cfg["scales"], cfg["use_depth_hints"])
    batch = ki.collate(items)
    exp = [oki.expected(it["views"], (it["do_color_aug"], it["do_flip"], it["jitter"]), it["side"], it.get("hint"),
                        fn.height, fn.width, fn.scales, fn.use_depth_hints) for it in items]
    keys = set(exp[0]) | set(exp[1])
    assert ("disp_hint" in exp[0]) != ("disp_hint" in exp[1])                    # an item without a hint: zeros
    out = {k: t(np.stack([e.get(k, np.zeros_like(exp[0].get(k, exp[1].get(k)))) for e in exp])) for k in keys}
    out["image_path"] = list(batch["image_path"])
    assert cfg["use_depth_hints"] and "s" in fn.frame_idxs and out["depth_hint_mask"].any()

    def call(out):
        harness._check_KittiInputs__run(dict(self=fn, batch=batch, device=None), out, None)
    key = ("color_aug", "s", 1)
    moved = dict(out)
    moved[key] = t(ulp_up(out[key].numpy(), (1, 2, 30, 40)))                     # one colour element one ulp off
    both(call, (out,), (moved,))
    h = 0 if "disp_hint" in exp[0] else 1
    mask = out["depth_hint_mask"].clone()
    mask[h, 0, 50, 60] = 1 - mask[h, 0, 50, 60]                                 # one hint pixel toggled
    both(call, (out,), (dict(out, depth_hint_mask=mask),))
    disp = out["disp_hint"].clone()
    disp[1 - h, 0, 5, 6] = 0.5                                                  # a hintless item's disp_hint not zero
    both(call, (out,), (dict(out, disp_hint=disp),))


def test_nyu_inputs_checker(harness):
    """two items of the 224_bicubic fixture"""
    fx = nic.load("224_bicubic")
    cfg = fx["config"]
    items = nic.items(fx)[:2]
    fn = ni.NyuInputs(cfg["is_224"], cfg["resample"])
    exp = [oni.expected(it["image"], it["depth"], it["flip"], it["perm"], it["gamma"], fn.is_224, fn.resample)
           for it in items]
    out = {k: np.stack([e[k] for e in exp]) for k in ("image", "depth")}

    def call(image, depth):
        harness._check_NyuInputs__run(dict(self=fn, batch=ni.collate(items), device=None),
                                      dict(image=t(image), depth=t(depth)), None)
    both(call, (out["image"], out["depth"]), (ulp_up(out["image"], (1, 0, 100, 50)), out["depth"]))
    both(call, (out["image"], out["depth"]), (out["image"], ulp_up(out["depth"], (0, 0, 10, 20))))


# ------------------------------------------------------------------------------------------ KITTI ground truth
def test_generate_depth_maps_checker(harness):
    """two 20000-point scans at two of the calibration dates' sizes, padded to one batch"""
    with np.load(os.path.join(kic.GOLDEN, "kitti_gt_calib.npz")) as f:
        frames = [("2011_09_26", 2), ("2011_09_28", 3)]
        P = np.stack([f["%s/P%d" % (d, cam)] for d, cam in frames])
        sizes = np.array([f["%s/size" % d] for d, _ in frames], np.int32)
    scans = [okg.small_scan(31 + k, 20000) for k in range(2)]
    offsets = np.array([0, scans[0].shape[0], scans[0].shape[0] + scans[1].shape[0]])
    hm, wm = sizes.max(0)
    depth = np.zeros((2, hm, wm))
    for k, (h, w) in enumerate(sizes):
        depth[k, :h, :w] = okg.depth_map(scans[k], P[k], h, w, True)
    hit = np.argwhere(depth[1] > 0)[0]
    assert depth[0].all() == 0 and (depth[1] > 0).sum() > 1000 and sizes[1, 0] < hm

    def call(depth):
        a = dict(points=t(np.concatenate(scans)), offsets=offsets, P=P, sizes=sizes, vel_depth=True)
        harness._check_generate_depth_maps(a, t(depth), None)
    both(call, (depth,), (ulp_up(depth, (1, *hit)),))                     # one depth one ulp off
    zero = np.argwhere(depth[0] == 0)[0]
    lit = depth.copy()
    lit[(0, *zero)] = 1.0                                                 # one empty pixel given a depth
    both(call, (depth,), (lit,))
    past = depth.copy()
    past[1, hm - 1, 0] = 1.0                                              # one pixel past frame 1's 370 rows written
    both(call, (depth,), (past,))


# ------------------------------------------------------------------------------------------ footprint
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.int16, torch.uint8])
@pytest.mark.parametrize("side", [-1, 1])
def test_a_write_one_element_into_a_guard_is_caught(dtype, side):
    with footprint.Footprint("cpu"):
        t = torch.empty((5, 7), dtype=dtype)
        t.fill_(3)                                                       # the whole buffer: allowed
    with pytest.raises(footprint.FootprintError, match="guard byte %s" % ("1 before" if side < 0 else "0 after")):
        with footprint.Footprint("cpu"):
            t = torch.empty((5, 7), dtype=dtype)
            at = t.storage_offset() + (-1 if side < 0 else t.numel())     # one element before / after the buffer
            t.as_strided((1,), (1,), at).fill_(3)
            del t                                                        # checked when it dies ...
    with pytest.raises(footprint.FootprintError, match="test_launch_check_teeth"):
        with footprint.Footprint("cpu"):
            keep = torch.zeros_like(torch.ones(3, 4, dtype=dtype)).t()  # ... or on exit while it lives
            keep.as_strided((1,), (1,), keep.storage_offset() + 12).fill_(1)


def _kernel(x, alloc):
    """writes every cell of its output but the first, and returns twice it: reads a cell it never wrote"""
    out = alloc(x.shape, dtype=x.dtype)
    out[1:] = x[1:]
    return {"y": out * 2}


def _kernel_ok(x, alloc):
    out = alloc(x.shape, dtype=x.dtype)
    out[:] = x
    return {"y": out * 2}


@pytest.mark.parametrize("dtype", [torch.float32, torch.int32])
def test_a_poisoned_cell_that_reaches_a_result_is_caught(dtype):
    """the plain run's allocator left zeros (a fresh process); under the footprint the cell is NaN / -1"""
    x = torch.arange(1, 9, dtype=dtype)
    for k in (_kernel_ok, _kernel):
        plain = k(x, torch.zeros)
        with footprint.Footprint("cpu"):
            checked = k(x, torch.empty)
        if k is _kernel_ok:
            same(plain, checked, "teeth")
        else:
            with pytest.raises(AssertionError, match="differs under the harness"):
                same(plain, checked, "teeth")


def test_buffers_have_torchs_layout_and_contents():
    """dtype, shape and strides equal torch's own allocation (channels_last, preserve_format of a permuted tensor),
    empty is all POISON bytes, zeros all zero, each buffer ALIGN-aligned; other devices pass through"""
    cl4 = torch.channels_last
    with footprint.Footprint("cpu") as fp:
        made = [(torch.empty((2, 8, 3, 5), memory_format=cl4), torch.empty((2, 8, 3, 5), device="meta", memory_format=cl4)),
                (torch.zeros((4, 6), dtype=torch.int64), torch.zeros((4, 6), dtype=torch.int64, device="meta")),
                (torch.empty_like(torch.ones(3, 4, 5).permute(2, 0, 1)), torch.ones(3, 4, 5).permute(2, 0, 1)),
                (torch.zeros_like(torch.ones(2, 3), dtype=torch.bool), torch.zeros(2, 3, dtype=torch.bool, device="meta")),
                (torch.empty(()), torch.empty((), device="meta"))]
        passed = torch.empty(3, device="meta")
    assert fp.allocated == len(made) and passed.device.type == "meta"
    for t, like in made:
        assert t.dtype == like.dtype and t.shape == like.shape and t.stride() == like.stride()
        assert t.data_ptr() % footprint.ALIGN == 0
    assert bool((made[0][0].view(torch.int32) == -1).all()) and bool((made[2][0].view(torch.int32) == -1).all())
    assert not made[1][0].any() and not made[3][0].any()


def test_a_channels_last_buffer_with_the_wrong_strides_is_caught(monkeypatch):
    def contiguous(arena, start, meta):
        return arena.view(meta.dtype)[start // meta.element_size():][:meta.numel()].view(meta.shape)
    monkeypatch.setattr(footprint, "_view", contiguous)
    with footprint.Footprint("cpu"):
        torch.empty((2, 4, 3, 3))                                        # contiguous: the strides agree
        with pytest.raises(footprint.FootprintError, match="strides"):
            torch.empty((2, 4, 3, 3), memory_format=torch.channels_last)


def test_a_changed_input_is_caught_unless_written_is_declared():
    args = {"x": torch.arange(12.0).reshape(3, 4), "feats": [torch.ones(5), {"s": torch.zeros(2, dtype=torch.int32)}],
            "out": torch.zeros(4), "scale": 2.0, "empty": torch.empty(0)}
    alias = args["out"][1:3]
    args["view"] = alias                                                 # shares memory with a written argument

    def call(mutate):
        snap = lc.snapshot(args, ("out",), device_type="cpu")
        mutate()
        return lc.changed_inputs(snap)
    assert call(lambda: args["out"].add_(1)) == []                       # named in WRITES (its alias too)
    assert call(lambda: None) == []
    assert call(lambda: args["x"].view(-1)[5].add_(1)) == ["x"]
    assert call(lambda: args["feats"][1]["s"].sub_(1)) == ["feats[1]['s']"]
    nan = args["feats"][0]
    nan[2] = float("nan")
    payload = torch.tensor([0x7FC00001], dtype=torch.int32).view(torch.float32)
    assert call(lambda: nan.__setitem__(2, payload[0])) == ["feats[0]"]  # another NaN: its bits changed


def test_a_nonzero_counter_header_is_caught():
    scratch = ops._Scratch()
    sizes = {"range": 1 << 17, "bwd": 8192, "splitk": 4096, "compact": 64}
    scratch.bufs = {(kind, 0, 0, 0): torch.zeros(n, dtype=torch.uint8) for kind, n in sizes.items()}
    scratch.bufs["compact", 0, 0, 0].fill_(7)                           # no header: not checked
    assert lc.scratch_header_faults(scratch) == (3, [])
    for kind, at in (("range", (1 << 16) - 1), ("bwd", 0), ("splitk", 4095)):
        scratch.bufs[kind, 0, 0, 0][at] = 1
        checked, faults = lc.scratch_header_faults(scratch)
        assert checked == 3 and len(faults) == 1 and faults[0].startswith(kind) and "byte %d " % at in faults[0]
        scratch.bufs[kind, 0, 0, 0][at] = 0
    scratch.bufs["range", 0, 0, 0][1 << 16] = 1                          # past the header: partial sums
    assert lc.scratch_header_faults(scratch) == (3, [])
