"""Pin oracle.nyu_loss against the UNMODIFIED reference training loop and write tests/golden/nyu_loss.npz.

Runs only where the reference checkout exists, like the other pin scripts.  For each case of ``oracle.nyu_loss.CASES``
it runs the reference's ``NYUv2/train.py`` ``main()`` for one epoch of one batch on the CPU, once with float32 and once
with float64 tensors:
  * stub modules stand in for tensorboardX, matplotlib, imageio and skimage, and ``.cuda()`` returns the tensor or
    module itself;
  * ``oracle.haar`` is registered as ``pytorch_wavelets``; its DWT records the LL it returns (the reference's yl_gt),
    and returns nothing for a size that is not a multiple of 16, which only ``val()`` of the "thin" case passes it and
    does not use;
  * ``Model`` is a stub whose outputs are its own ``nn.Parameter``s (the case's predictions), so their ``.grad`` is the
    reference's loss gradient; ``torch.optim.Adam`` is a stub that records those gradients in ``step()``;
  * the loaders yield the case's batch; the test iterator has ``.next()``, which ``val()`` calls;
  * the loss scalars are captured from ``SummaryWriter.add_scalar`` of the "train" writer.
The float64 run takes its interpolation weights in fp64, so a target pixel within 1e-6 relative of a tie could take
the other sign there: each random case takes the first seed, counting up from its base seed, whose frames keep every
pixel farther than that from a tie (the "ties" case is made of exact ties on purpose).

The fixture holds each case's seed, the captured scalars of both runs, the float64 run's yl_gt, and the float64
gradients: all elements of small tensors, a seeded sample of the others.  Tests regenerate the inputs from the seeds.

Usage:  python -m oracle.pin_nyu_loss
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import haar, nyu_loss as onl                                     # noqa: E402

REF_NYU = "/root/reference/NYUv2"
GOLDEN = os.path.join(REPO, "tests", "golden")
SEED0 = 100
FULL_GRAD_MAX = 4800                       # gradients up to this size are stored whole
GRAD_SAMPLES = 2048
NEAR_TIE = 1e-6


class _Run:
    """What the stubs see and record during one main()"""
    depth = preds = ll = None
    dtype = torch.float32
    scalars, grads, yl = {}, None, []


class StubWriter:
    def __init__(self, path):
        self.mode = os.path.basename(path)

    def add_scalar(self, tag, v, niter):
        if self.mode == "train":
            _Run.scalars[tag] = float(v.detach()) if torch.is_tensor(v) else float(v)

    def add_image(self, *a, **k):
        pass

    add_histogram = add_image


class StubModel(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.keys = [("disp", s) for s in onl.SCALES]
        vals = [_Run.preds[s] for s in onl.SCALES]
        if _Run.ll is not None:
            self.keys.append(("wavelets", 3, "LL"))
            vals.append(_Run.ll)
        self.outs = nn.ParameterList([nn.Parameter(torch.from_numpy(v).to(_Run.dtype)) for v in vals])

    def forward(self, image):
        return dict(zip(self.keys, self.outs))


class StubAdam:
    def __init__(self, params, lr):
        self.params = list(params)

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    def step(self):
        _Run.grads = [None if p.grad is None else p.grad.detach().clone() for p in self.params]


class RecordingDWT(haar.DWTForward):
    def forward(self, x):
        if x.shape[-2] % 2 ** self.J or x.shape[-1] % 2 ** self.J:
            # val() transforms its target whatever the options and uses the result only with --use_wavelets; the
            # "thin" case (no wavelets) is not a multiple of 16, which oracle.haar does not restate in reflect mode
            return None, None
        yl, yh = super().forward(x)
        _Run.yl.append(yl.detach().clone())
        return yl, yh


class _TestIter:
    def __init__(self, batches):
        self.it = iter(batches)

    def next(self):
        return next(self.it)

    __next__ = next


class _TestLoader:
    def __init__(self, batches):
        self.batches = batches

    def __iter__(self):
        return _TestIter(self.batches)


def loaders(batch_size, num_workers, is_224=False):
    n, _, h, w = _Run.depth.shape
    batch = {"image": torch.zeros(n, 3, 2 * h, 2 * w, dtype=_Run.dtype),
             "depth": torch.from_numpy(_Run.depth).to(_Run.dtype)}
    return [batch], _TestLoader([batch])


def import_train():
    for name in ("matplotlib", "matplotlib.cm", "imageio", "skimage", "skimage.feature", "tensorboardX", "model",
                 "data", "pytorch_wavelets"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
    sys.modules["imageio"].imsave = sys.modules["imageio"].imread = None
    sys.modules["skimage"].feature = sys.modules["skimage.feature"]
    sys.modules["tensorboardX"].SummaryWriter = StubWriter
    sys.modules["model"].Model = StubModel
    sys.modules["data"].getTrainingTestingData = loaders
    sys.modules["pytorch_wavelets"].DWT = RecordingDWT
    sys.modules["pytorch_wavelets"].IDWT = haar.DWTInverse
    torch.Tensor.cuda = lambda self, *a, **k: self
    nn.Module.cuda = lambda self, *a, **k: self
    torch.optim.Adam = StubAdam
    if REF_NYU not in sys.path:
        sys.path.insert(0, REF_NYU)
    import train
    return train


def run_reference(train, name, depth, preds, ll, dtype):
    n, _, _, _, use_wavelets, supervise_ll, _ = onl.CASES[name]
    _Run.depth, _Run.preds, _Run.ll, _Run.dtype = depth, preds, ll, dtype
    _Run.scalars, _Run.grads, _Run.yl = {}, None, []
    flags = ["--disparity"] * onl.CASES[name][3] + ["--use_wavelets"] * use_wavelets + ["--supervise_LL"] * supervise_ll
    flags += ["--use_224"] * (depth.shape[2] == 224)
    with tempfile.TemporaryDirectory() as tmp:
        argv = sys.argv
        sys.argv = ["train.py", "--logdir", tmp, "--model_name", "pin", "--epochs", "1", "--bs", str(n)] + flags
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                train.main()
        finally:
            sys.argv = argv
    keys = ["disp_%d" % s for s in onl.SCALES] + (["LL"] if ll is not None else [])
    grads = {k: g.numpy() for k, g in zip(keys, _Run.grads) if g is not None}
    return dict(_Run.scalars), grads, (_Run.yl[0].numpy() if _Run.yl else None)


def nearest_tie(depth, preds, disparity):
    """smallest |sample - t| / |t| over the random case's pixels, in the oracle's fp64 samples"""
    t = (np.float32(1) / depth * np.float32(10)).astype(np.float32) if disparity else depth
    worst = np.inf
    for s in onl.SCALES:
        smp = onl.upsample(preds[s][:, 0], t.shape[2], t.shape[3])
        worst = min(worst, float(np.min(np.abs(smp - t[:, 0]) / np.abs(t[:, 0]))))
    return worst


def main():
    train = import_train()
    arrays, meta = {}, dict(cases={k: list(v) for k, v in onl.CASES.items()}, seeds={})
    for i, name in enumerate(onl.CASES):
        seed = SEED0 + 10 * i
        while True:                         # the first seed whose random frames keep clear of ties
            depth, preds, ll = onl.case_inputs(name, seed)
            if onl.CASES[name][6] != "random" or nearest_tie(depth, preds, onl.CASES[name][3]) > NEAR_TIE:
                break
            seed += 1
        meta["seeds"][name] = seed
        runs = {tag: run_reference(train, name, depth, preds, ll, dt)
                for tag, dt in (("f32", torch.float32), ("f64", torch.float64))}
        for tag, (scalars, _, _) in runs.items():
            arrays["%s__%s_scalars" % (name, tag)] = np.array([scalars[k] for k in sorted(scalars)], np.float64)
        meta.setdefault("scalar_keys", {})[name] = sorted(runs["f64"][0])
        _, grads, yl = runs["f64"]
        if yl is not None:
            arrays[name + "__yl_gt_f64"] = yl
        rng = np.random.default_rng(seed)
        for k, g in grads.items():
            flat = g.reshape(-1)
            idx = np.arange(flat.size) if flat.size <= FULL_GRAD_MAX else np.sort(
                rng.choice(flat.size, GRAD_SAMPLES, replace=False))
            arrays["%s__grad_%s_idx" % (name, k)] = idx.astype(np.int32)
            arrays["%s__grad_%s_f64" % (name, k)] = flat[idx]
        print(name, "seed", seed, {k: "%.7g" % v for k, v in runs["f64"][0].items()})
    path = os.path.join(GOLDEN, "nyu_loss.npz")
    np.savez_compressed(path, __meta__=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
