"""Record the reference's module layout as tests/golden/reference_layout.json.

    python -m oracle.pin_reference_layout <path of the unmodified reference tree>

What tests/test_reference_integration.py checks our decoders against, stored so that the test needs no copy of the
reference: for every decoder the reference's own factories build (KITTI/networks/network_constructors.py
make_depth_decoder, NYUv2/model.py Model) the class name, the state-dict keys and shapes, the keys of ``.convs`` and how
``pyt_utils.group_weight`` splits its parameters; and the parameter names of the public functions of KITTI/layers.py.
``pytorch_wavelets`` is served by our drop-in (wavelets.py) while the reference is imported, as INTEGRATION.md A does.
"""
import argparse
import importlib
import inspect
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

OUT = os.path.join(REPO, "tests", "golden", "reference_layout.json")
KITTI_ENC = [64, 64, 128, 256, 512]
KITTI_CASES = {"wavelets": {}, "sparse": {"use_sparse": True}, "dense": {"use_wavelets": False}}
NYU_CASES = {"wavelets": {}, "sparse": {"use_sparse": True}, "wavelets_224": {"use_224": True},
             "dense": {"use_wavelets": False}, "dense_224": {"use_wavelets": False, "use_224": True}}
LAYER_NAMES = ("Conv3x3", "Conv1x1", "ConvBlock", "upsample", "sparse_select", "make_result", "mask2yx", "mask2idxmap",
               "sparse_conv1x1", "sparse_conv3x3", "sparse_upsample")


def _tree(ref, name):
    import wavelet_monodepth_b200.wavelets as w
    for mod in list(sys.modules):
        if mod in ("layers", "networks", "pyt_utils", "model", "load_save_utils") or mod.startswith("networks."):
            del sys.modules[mod]
    sys.path[:] = [p for p in sys.path if not p.startswith(ref)]
    sys.path.insert(0, os.path.join(ref, name))
    sys.modules["pytorch_wavelets"] = w
    importlib.invalidate_caches()


def _layout(module):
    sd = module.state_dict()
    return {"class": type(module).__name__, "keys": list(sd.keys()), "shapes": [list(v.shape) for v in sd.values()]}


def kitti(ref):
    _tree(ref, "KITTI")
    from networks.network_constructors import make_depth_decoder
    from pyt_utils import group_weight

    class Enc:
        num_ch_enc = np.array(KITTI_ENC)

    out = {}
    for case, kw in KITTI_CASES.items():
        opts = argparse.Namespace(use_wavelets=True, use_sparse=False, scales=range(4))
        opts.__dict__.update(kw)
        dec = make_depth_decoder(Enc(), opts)
        groups = []
        for _, weights in dec.convs.items():
            group_weight(groups, weights, 1e-4)
        entry = _layout(dec)
        entry["convs"] = list(dec.convs.keys())
        entry["grouped_params"] = sum(len(g["params"]) for g in groups)
        out[case] = entry
    layers = importlib.import_module("layers")
    sigs = {}
    for name in LAYER_NAMES:
        a = getattr(layers, name)
        sigs[name] = list(inspect.signature(a.__init__ if inspect.isclass(a) else a).parameters)
    return out, sigs


def nyu(ref):
    _tree(ref, "NYUv2")
    from model import Model
    out = {}
    for case, kw in NYU_CASES.items():
        opts = argparse.Namespace(encoder_type="densenet", normalize_input=False, pretrained_encoder=False, num_layers=18,
                                  use_wavelets=True, use_sparse=False, use_224=False, dw_waveconv=False, dw_upconv=False)
        opts.__dict__.update(kw)
        m = Model(opts)
        entry = _layout(m.decoder)
        entry["enc_features"] = [int(c) for c in m.encoder.num_ch_enc]
        out[case] = entry
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference", help="root of the unmodified reference tree (holds KITTI/ and NYUv2/)")
    ref = os.path.abspath(ap.parse_args().reference)
    k, sigs = kitti(ref)
    n = nyu(ref)
    with open(OUT, "w") as f:
        json.dump({"kitti_num_ch_enc": KITTI_ENC, "kitti": k, "nyu": n, "kitti_layer_signatures": sigs}, f, indent=1)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
