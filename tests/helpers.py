"""Shared test helpers: golden-fixture loading, seeded module construction, operands, comparison metrics."""
import glob
import json
import os

import numpy as np
import torch
import torch.nn.functional as F

from wavelet_monodepth_b200 import synth
from wavelet_monodepth_b200._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REL_TOL = 1e-4      # north_star: outputs within 1e-4 relative fp32 tolerance


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        arrays = {k: z[k] for k in z.files if k != "__meta__"}
        meta = json.loads(bytes(z["__meta__"]).decode())
    return arrays, meta


def golden_names(prefix):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, prefix + "*.npz")))


def key_str(k):
    return k if isinstance(k, str) else "_".join(str(v) for v in k)


def rnd(*shape, seed=0, lo=-1.0, hi=1.0):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(lo, hi, size=shape).astype(np.float32))


def rows_of(x):
    """(N, C, H, W) -> pixel-major rows (N*H*W, C)."""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).contiguous()


def close(got, want, tol=1e-12):
    """Two fp64 restatements of one sum, in different orders: max |got - want| <= tol max(max |want|, 1)."""
    return float((got - want).abs().max()) <= tol * max(float(want.abs().max()), 1.0)


def torch_conv(x, wt, b, pad, act):
    """A 3x3 convolution with the layers' padding and activation, in torch."""
    mode = {PAD_REFLECT: "reflect", PAD_REPLICATE: "replicate", PAD_ZERO: "constant"}[pad]
    y = F.conv2d(F.pad(x, (1, 1, 1, 1), mode=mode), wt, b)
    return {ACT_NONE: lambda t: t, ACT_ELU: F.elu, ACT_LRELU: lambda t: F.leaky_relu(t, 0.2),
            ACT_SIGMOID: torch.sigmoid}[act](y)


def rel_err(a, b):
    """max|a-b| / max(|b|, tiny): the 'relative fp32 tolerance' the parity statement uses."""
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    if a.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def kitti_features(meta, device="cpu"):
    shapes = synth.kitti_feature_shapes(2, meta["height"], meta["width"], meta["num_ch_enc"])
    feats = synth.blocky_features(shapes, seed=meta["feat_seed"], cell=meta["cell"])
    if "sample" in meta:
        feats = [f[meta["sample"]:meta["sample"] + 1] for f in feats]
    return [f.to(device) for f in feats]


def nyu_features(meta, device="cpu"):
    shapes = synth.nyu_feature_shapes(2, meta["height"], meta["width"], meta["enc_features"])
    feats = synth.blocky_features(shapes, seed=meta["feat_seed"], cell=meta["cell"])
    if "sample" in meta:
        feats = [f[meta["sample"]:meta["sample"] + 1] for f in feats]
    return [f.to(device) for f in feats]


def kitti_variant(want, meta, name):
    """(constructor kwargs, the variant's arrays keyed by key_str) of one DepthDecoder variant of the KITTI fixture."""
    prefix = name + "__"
    return meta["variants"][name], {k[len(prefix):]: v for k, v in want.items() if k.startswith(prefix)}


def seeded_params(module, meta):
    """state dict (CPU tensors, reference key names) for a module built from `meta`."""
    return synth.random_state_dict(synth.module_shapes(module), seed=meta["param_seed"], gains=meta.get("gains"))


def compare_outputs(got, want, what, float_tol=REL_TOL, exact_masks=True):
    """got: dict keyed by tuples / str (tensors or ints); want: dict keyed by key_str (numpy)."""
    got = {key_str(k): v for k, v in got.items()}
    missing = set(want) - set(got)
    assert not missing, (what, "missing keys", sorted(missing))
    worst = 0.0
    for k, wv in want.items():
        gv = got[k]
        if torch.is_tensor(gv):
            gv = gv.detach().float().cpu().numpy() if gv.dtype != torch.bool else gv.cpu().numpy()
        if "total_ops" in k:
            assert int(np.asarray(gv)) == int(wv), (what, k, gv, wv)
            continue
        assert tuple(np.shape(gv)) == tuple(wv.shape), (what, k, np.shape(gv), wv.shape)
        if "mask" in k:
            bad = int((np.asarray(gv).astype(bool) != wv.astype(bool)).sum())
            if exact_masks:
                assert bad == 0, (what, k, "mask pixels differ: %d of %d" % (bad, wv.size))
            continue
        e = rel_err(gv, wv)
        worst = max(worst, e)
        assert e <= float_tol, (what, k, "rel err %.3e > %.1e" % (e, float_tol))
    return worst
