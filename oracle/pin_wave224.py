"""Pin oracle.wave224 against the UNMODIFIED reference and write its golden vectors.

Runs only in the build container (needs the reference checkout), like oracle/pin_against_reference.py, whose reference
import and comparison helpers it uses.  It
  1. runs the reference's DecoderWave224 (densedepth_decoder.py:151-221) and ``nyu224_dense_forward`` on the tiny NYU
     pyramid (N=2) and on DenseNet161 features of one 224x224 frame, and asserts they agree bit for bit,
  2. does the same for the reference's DepthWaveProgressiveDecoder(use_skips=False) and
     ``kitti_dense_noskip_forward`` on the tiny KITTI pyramid,
  3. stores the reference's tiny outputs as tests/golden/nyu224_tiny_dense.npz and kitti_tiny_dense_noskip.npz.
No other fixture is written.

Usage:  python -m oracle.pin_wave224 [--skip-full-size]
"""
import argparse
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import wave224                                                  # noqa: E402
from oracle.pin_against_reference import (GOLDEN, HEAD_GAIN_KITTI, KITTI_TINY_CH, NYU_TINY_CH, REF,  # noqa: E402
                                          compare, import_reference, to_npz_dict)
from wavelet_monodepth_b200 import synth                                   # noqa: E402

HEAD_GAIN_NYU224 = {"wave1_ll.": 4.0, "wave1.": 6.0, "wave2.": 6.0, "wave3.": 6.0, "wave4.": 6.0}


def save(name, arrays, meta):
    import json
    arrays = dict(arrays)
    arrays["__meta__"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **arrays)


def pin_nyu224(full_size):
    _, dec = import_reference("NYUv2")
    ref = dec.DecoderWave224(enc_features=list(NYU_TINY_CH), decoder_width=0.5).eval()
    sd = synth.random_state_dict(synth.module_shapes(ref), seed=17, gains=HEAD_GAIN_NYU224)
    ref.load_state_dict(sd, strict=False)
    feats2 = synth.blocky_features(synth.nyu_feature_shapes(2, 96, 128, NYU_TINY_CH), seed=7, cell=4)
    r = ref(feats2)
    compare(r, wave224.nyu224_dense_forward(sd, feats2), "NYU 224 dense decoder (N=2)", atol=0.0)
    d1 = r[("disp", 1)]
    print("      disp_1 (floor) takes %d distinct values in [%g, %g]" % (d1.unique().numel(), d1.min(), d1.max()))
    save("nyu224_tiny_dense", to_npz_dict(r), dict(enc_features=NYU_TINY_CH, n=2, height=96, width=128,
                                                  param_seed=17, feat_seed=7, cell=4, gains=HEAD_GAIN_NYU224))
    if full_size:
        ch = synth.DENSENET161_CH
        ref = dec.DecoderWave224(enc_features=list(ch), decoder_width=0.5).eval()
        sd = synth.random_state_dict(synth.module_shapes(ref), seed=11)
        ref.load_state_dict(sd, strict=False)
        feats = synth.blocky_features(synth.nyu_feature_shapes(1, 224, 224, ch), seed=12)
        compare(ref(feats), wave224.nyu224_dense_forward(sd, feats), "NYU 224 DenseNet161 224x224 (full size)", atol=0.0)


def pin_kitti_noskip():
    _, dec = import_reference("KITTI")
    ref = dec.DepthWaveProgressiveDecoder(np.array(KITTI_TINY_CH), use_skips=False).eval()
    sd = synth.random_state_dict(synth.module_shapes(ref), seed=11, gains=HEAD_GAIN_KITTI)
    ref.load_state_dict(sd, strict=False)
    feats2 = synth.blocky_features(synth.kitti_feature_shapes(2, 64, 96, KITTI_TINY_CH), seed=5, cell=4)
    r = ref(feats2)
    compare(r, wave224.kitti_dense_noskip_forward(sd, feats2), "KITTI dense decoder without skips (N=2)", atol=0.0)
    save("kitti_tiny_dense_noskip", to_npz_dict(r), dict(num_ch_enc=KITTI_TINY_CH, n=2, height=64, width=96,
                                                        param_seed=11, feat_seed=5, cell=4, gains=HEAD_GAIN_KITTI,
                                                        use_skips=False))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-full-size", action="store_true", help="skip the DenseNet161 224x224 check (~2 s)")
    args = ap.parse_args()
    assert os.path.isdir(REF), "the reference checkout is only available in the build container"
    torch.set_grad_enabled(False)
    print("pinning oracle.wave224 against the unmodified reference (%s)" % REF)
    pin_kitti_noskip()
    pin_nyu224(full_size=not args.skip_full_size)
    print("golden vectors written to", GOLDEN)


if __name__ == "__main__":
    main()
