"""Pin oracle.kitti_loss against the UNMODIFIED reference trainer and write tests/golden/kitti_hints_loss*.npz.

Runs only where the reference checkout exists, like the other pin scripts.  For each case of ``CASES`` it calls the
reference's ``Trainer.generate_images_pred`` and ``Trainer.compute_losses_hints`` (KITTI/trainer.py) as unbound methods
on a stub ``self`` carrying ``opt`` (the depth-hints stereo configuration), ``SSIM()``, ``BackprojectDepth``,
``Project3D`` and ``num_scales``, on the CPU, once in float32 and once in float64, with the predictions as leaf tensors:
  * stub modules stand in for tensorboardX, the networks and the datasets, which the loss does not use;
  * ``Tensor.cuda()`` returns the tensor itself, so the noise is ``torch.randn`` on the CPU default generator, seeded
    with the case's seed before the call, as a seeded trainer step would draw it (float32 in both runs: the float64 run
    promotes it when it is added);
  * the gradient of ``losses["loss"]`` reaches the predictions' ``.grad``; the gradient of the weighted sum of every
    term, ``sum_k w_k losses[k]`` with the case's ``weights`` (``oracle.kitti_loss.term_keys`` order), is taken from the
    same graph with ``torch.autograd.grad``.
The case's ``min_depth``, ``max_depth`` and ``disparity_smoothness`` go to ``opt``, its intrinsics and stereo transforms
(one camera, or a different one per frame) to the inputs.
Each random case takes the first seed, counting up from its base seed, whose frames keep every fp64 decision (argmin
and the grid sample's floor) farther than 1e-9 relative from flipping, so the float64 run and the fp64 oracle decide
alike; exact ties, which every precision breaks alike, do not count (pixels whose scale and hint warps leave the image
past the same corner).  The "special" case is made of designed decisions: an all-zero and an all-one hint mask,
projections off both sides of the image, disparities of exactly 0 and 1 and exact ties between r and the hint loss.

The fixture holds each case's seed, the scalars of both runs, both runs' masks, the term weights, and the float64
gradients of the total and of the weighted terms: a seeded sample of each, at the same indices.  It is split over
``oracle.kitti_loss.FIXTURES`` so that every file stays well under 1 MiB: kitti_hints_loss.npz holds the first four
cases as they were first pinned, kitti_hints_loss_terms.npz their weights and weighted-term gradients, and
kitti_hints_loss_shapes.npz and kitti_hints_loss_cameras.npz the other cases whole, each file listing its own "cases".  Tests regenerate the inputs from the seeds (``oracle.kitti_loss.make_inputs``) and read the files
as one (``oracle.kitti_loss.load_fixture``).

Usage:  python -m oracle.pin_kitti_loss
"""
import argparse
import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import kitti_loss as okl                                          # noqa: E402

REF_KITTI = "/root/reference/KITTI"
GOLDEN = os.path.join(REPO, "tests", "golden")
GRAD_SAMPLES = 4096
NEAR = 1e-9


def _reference():
    for name in ("tensorboardX", "networks", "networks.network_constructors", "datasets"):
        mod = types.ModuleType(name)
        mod.SummaryWriter = object
        sys.modules.setdefault(name, mod)
    sys.path.insert(0, REF_KITTI)
    import trainer
    import layers
    return trainer.Trainer, layers


def run_reference(case, seed, dtype):
    """(scalars, masks {s: (identity_selection, depth_hint_pixels)}, grads {s}, weighted-term grads {s}, warped {s},
    color_depth_hint)"""
    Trainer, layers = _reference()
    inp, disps = okl.make_inputs(case, seed)
    N, _, H, W = inp["target"].shape
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype)                # noqa: E731
    opt = types.SimpleNamespace(loss_scales=list(case["loss_scales"]), scales=list(case["scales"]),
                                v1_multiscale=False, frame_ids=[0, "s"], pose_model_type="separate_resnet",
                                use_depth_hints=True, height=H, width=W, no_ssim=False, disable_automasking=False,
                                avg_reprojection=False, **okl.options(case))
    me = types.SimpleNamespace(opt=opt, ssim=layers.SSIM(), num_scales=len(opt.scales),
                               backproject_depth={0: layers.BackprojectDepth(N, H, W).to(dtype)},
                               project_3d={0: layers.Project3D(N, H, W)})
    me.compute_reprojection_loss = types.MethodType(Trainer.compute_reprojection_loss, me)
    me.compute_loss_masks = Trainer.compute_loss_masks
    me.compute_proxy_supervised_loss = Trainer.compute_proxy_supervised_loss
    inputs = {("color", 0, 0): t(inp["target"]), ("color", "s", 0): t(inp["source"]), ("K", 0): t(inp["K"]),
              ("inv_K", 0): t(inp["inv_K"]), "stereo_T": t(inp["stereo_T"]), "depth_hint": t(inp["depth_hint"]),
              "depth_hint_mask": t(inp["depth_hint_mask"])}
    for s in case["scales"]:
        inputs[("color", 0, s)] = t(inp["colors"][s])
    leaves = {s: t(disps[s]).requires_grad_() for s in case["scales"]}
    outputs = {("disp", s): leaves[s] for s in case["scales"]}
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        Trainer.generate_images_pred(me, inputs, outputs)
        torch.manual_seed(seed)
        losses = Trainer.compute_losses_hints(me, inputs, outputs)
    finally:
        torch.Tensor.cuda = cuda
    losses["loss"].backward(retain_graph=True)
    weighted = sum(w * losses[k] for w, k in zip(case["weights"], okl.term_keys(case["loss_scales"])))
    used = [s for s in case["scales"] if leaves[s].grad is not None]
    wg = dict(zip(used, torch.autograd.grad(weighted, [leaves[s] for s in used])))
    scalars = {k: float(v) for k, v in losses.items()}
    masks = {s: (outputs["identity_selection/%d" % s].detach().numpy()[:, 0].astype(np.float64),
                 outputs["depth_hint_pixels/%d" % s].detach().numpy()[:, 0].astype(np.float64))
             for s in case["loss_scales"]}
    grads = {s: (leaves[s].grad.numpy().astype(np.float64) if leaves[s].grad is not None
                 else np.zeros(disps[s].shape)) for s in case["scales"]}
    wgrads = {s: (wg[s].numpy().astype(np.float64) if s in wg else np.zeros(disps[s].shape)) for s in case["scales"]}
    warped = {s: outputs[("color", "s", s)].detach().numpy().astype(np.float64) for s in case["loss_scales"]}
    chint = outputs[("color_depth_hint", "s", 0)].detach().numpy().astype(np.float64)
    return scalars, masks, grads, wgrads, warped, chint


def _clear(case, seed):
    """True when no fp64 decision of the case at this seed lies within NEAR (relative) of flipping"""
    inp, disps = okl.make_inputs(case, seed)
    noise = okl.draw_noise(seed, inp, case["loss_scales"])
    return okl.decision_margin(inp, disps, noise, case) > NEAR


def main():
    argparse.ArgumentParser(description=__doc__.split("\n")[0]).parse_args()
    out = {}
    names = []
    for name, case in okl.CASES.items():
        seed = case["seed"]
        if case.get("random", True):
            while not _clear(case, seed):
                seed += 1
        names.append(name)
        out["%s/seed" % name] = np.int64(seed)
        keys = None
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            sc, masks, grads, wgrads, warped, chint = run_reference(case, seed, dt)
            keys = sorted(sc)
            out["%s/%s/scalars" % (name, tag)] = np.array([sc[k] for k in keys])
            for s, (ids, hp) in masks.items():
                out["%s/%s/identity_selection/%d" % (name, tag, s)] = np.packbits(ids.astype(bool))
                out["%s/%s/depth_hint_pixels/%d" % (name, tag, s)] = np.packbits(hp.astype(bool))
            if tag == "f64":
                rng = np.random.default_rng(seed)
                for s, g in grads.items():
                    flat = g.reshape(-1)
                    idx = np.sort(rng.choice(flat.size, min(GRAD_SAMPLES, flat.size), replace=False))
                    out["%s/grad_idx/%d" % (name, s)] = idx.astype(np.int64)
                    out["%s/f64/grad/%d" % (name, s)] = flat[idx]
                    out["%s/f64/wgrad/%d" % (name, s)] = wgrads[s].reshape(-1)[idx]
        out["%s/scalar_keys" % name] = np.array(keys)
        out["%s/weights" % name] = np.array(case["weights"])
    files = {name: {} for name in okl.FIXTURES}
    for k, v in out.items():
        files[okl.fixture_file(k)][k] = v
    for name in names:
        files[okl.fixture_file(name + "/seed")].setdefault("cases", []).append(name)
    for keys in files.values():
        if "cases" in keys:
            keys["cases"] = np.array(keys["cases"])
    for name, keys in files.items():
        path = os.path.join(GOLDEN, name)
        with open(path, "wb") as f:
            np.savez_compressed(f, **keys)
        print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
