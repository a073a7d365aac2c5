"""Pin oracle.baseline against the UNMODIFIED reference and write its golden vectors.

Runs only in the build container (needs the reference checkout), like oracle/pin_against_reference.py, whose reference
import and comparison helpers it uses.  It
  1. runs the reference's DepthDecoder (depth_decoder.py:18-69) and ``kitti_baseline_forward`` on the tiny KITTI pyramid
     (N=2), with the default arguments and with scales=[1, 3], use_skips=False and num_output_channels=3, and asserts
     they agree bit for bit;
  2. does the same for the reference's Decoder and Decoder224 (densedepth_decoder.py:15-89) and
     ``nyu_baseline_forward`` on the tiny NYU pyramid (N=2);
  3. unless --skip-full-size: one frame each of ResNet18 640x192 (DepthDecoder), DenseNet161 640x480 (Decoder) and
     DenseNet161 224x224 (Decoder224);
  4. stores the reference's tiny outputs as tests/golden/kitti_tiny_baseline.npz, nyu_tiny_baseline.npz and
     nyu224_tiny_baseline.npz.  The NYU fixtures' meta also records the state-dict keys and shapes of the reference's
     Decoder / Decoder224 at their default (DenseNet161) widths.
No other fixture is written.

Usage:  python -m oracle.pin_baseline [--skip-full-size]
"""
import argparse
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import baseline                                                 # noqa: E402
from oracle.pin_against_reference import (GOLDEN, KITTI_TINY_CH, NYU_TINY_CH, REF, compare, import_reference,  # noqa: E402
                                          silence, to_npz_dict)
from oracle.pin_wave224 import save                                         # noqa: E402
from wavelet_monodepth_b200 import synth                                   # noqa: E402

# DepthDecoder variants pinned on the tiny pyramid: fixture key prefix -> constructor arguments
KITTI_VARIANTS = {
    "default": {},
    "scales13": {"scales": [1, 3]},
    "noskip": {"use_skips": False},
    "ch3": {"num_output_channels": 3},
}


def pin_kitti(full_size):
    _, dec = import_reference("KITTI")
    feats2 = synth.blocky_features(synth.kitti_feature_shapes(2, 64, 96, KITTI_TINY_CH), seed=5, cell=4)
    arrays = {}
    for name, kw in KITTI_VARIANTS.items():
        ref = dec.DepthDecoder(np.array(KITTI_TINY_CH), **kw).eval()
        sd = synth.random_state_dict(synth.module_shapes(ref), seed=11)
        ref.load_state_dict(sd)
        r = ref(feats2)
        compare(r, baseline.kitti_baseline_forward(sd, feats2, scales=kw.get("scales", range(4)),
                                                   use_skips=kw.get("use_skips", True)),
                "KITTI DepthDecoder %s (N=2)" % name, atol=0.0)
        arrays.update(to_npz_dict(r, prefix=name + "__"))
    save("kitti_tiny_baseline", arrays, dict(num_ch_enc=KITTI_TINY_CH, n=2, height=64, width=96, param_seed=11,
                                              feat_seed=5, cell=4, variants=KITTI_VARIANTS))
    if full_size:
        ch = synth.RESNET18_CH
        ref = dec.DepthDecoder(np.array(ch)).eval()
        sd = synth.random_state_dict(synth.module_shapes(ref), seed=11)
        ref.load_state_dict(sd)
        feats = synth.blocky_features(synth.kitti_feature_shapes(1, 192, 640, ch), seed=12)
        compare(ref(feats), baseline.kitti_baseline_forward(sd, feats), "KITTI DepthDecoder R18 640x192 (full size)",
                atol=0.0)


def pin_nyu(full_size):
    _, dec = import_reference("NYUv2")
    feats2 = synth.blocky_features(synth.nyu_feature_shapes(2, 96, 128, NYU_TINY_CH), seed=7, cell=4)
    for cls, fixture, extra in (("Decoder", "nyu_tiny_baseline", False), ("Decoder224", "nyu224_tiny_baseline", True)):
        ref = silence(getattr(dec, cls), enc_features=list(NYU_TINY_CH), decoder_width=0.5).eval()
        sd = synth.random_state_dict(synth.module_shapes(ref), seed=17)
        ref.load_state_dict(sd)
        r = ref(feats2)
        compare(r, baseline.nyu_baseline_forward(sd, feats2, extra_stage=extra), "NYU %s (N=2)" % cls, atol=0.0)
        full = silence(getattr(dec, cls))
        save(fixture, to_npz_dict(r), dict(enc_features=NYU_TINY_CH, n=2, height=96, width=128, param_seed=17,
                                           feat_seed=7, cell=4,
                                           state_dict={k: list(v.shape) for k, v in full.state_dict().items()}))
        if full_size:
            ch = synth.DENSENET161_CH
            size = (224, 224) if extra else (480, 640)
            sd = synth.random_state_dict(synth.module_shapes(full), seed=11)
            full.load_state_dict(sd)
            feats = synth.blocky_features(synth.nyu_feature_shapes(1, size[0], size[1], ch), seed=12)
            compare(full.eval()(feats), baseline.nyu_baseline_forward(sd, feats, extra_stage=extra),
                    "NYU %s DenseNet161 %dx%d (full size)" % (cls, size[1], size[0]), atol=0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-full-size", action="store_true", help="skip the three one-frame full-size checks")
    args = ap.parse_args()
    assert os.path.isdir(REF), "the reference checkout is only available in the build container"
    torch.set_grad_enabled(False)
    print("pinning oracle.baseline against the unmodified reference (%s)" % REF)
    pin_kitti(full_size=not args.skip_full_size)
    pin_nyu(full_size=not args.skip_full_size)
    print("golden vectors written to", GOLDEN)


if __name__ == "__main__":
    main()
