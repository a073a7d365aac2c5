"""The decoder workloads that the launch-checking tests (tests/launch_check.py) share: the benchmark's encoder pyramids,
image sizes and synthetic features, the NYU wavelet decoders as the benchmark builds them, and the check that a
workload gives the same bits under the harness as without it."""
import torch

from wavelet_monodepth_b200 import nyu_decoders as nd, synth

DEV = "cuda"
NYU_HEADS = ["wave1.conv.", "wave2.conv.", "wave3.conv."]       # bench.py's NYU workload: high-pass heads x4
R50 = (synth.RESNET50_CH, 320, 1024)
R18 = (synth.RESNET18_CH, 192, 640)
D161 = (synth.DENSENET161_CH, 480, 640)


def kitti_feats(n, ch, h, w, layout="nchw"):
    host = synth.bench_kitti_features(n, h, w, ch, pin=layout == "pinned")
    if layout == "pinned":                          # the sparse levels' skip maps stay in pinned host memory
        return [f if k < 3 else f.to(DEV) for k, f in enumerate(host)]
    feats = [f.to(DEV) for f in host]
    if layout == "channels_last":
        feats = [f.contiguous(memory_format=torch.channels_last) for f in feats]
    return feats


def nyu_feats(n, ch, h, w):
    return [f.to(DEV) for f in synth.blocky_features(synth.nyu_feature_shapes(n, h, w, ch), seed=2000,
                                                      cell=synth.BENCH_SYNTH["cell"], texture=synth.BENCH_SYNTH["texture"])]


def nyu(cls, n, spec, thr=None):
    def run():
        dec = cls(enc_features=list(spec[0]), decoder_width=0.5)
        if cls is nd.Decoder:
            synth.load_random(dec, seed=11)
        else:
            synth.load_random(dec, seed=11, gains={k: synth.BENCH_SYNTH["head_gain"] for k in NYU_HEADS}, highpass=NYU_HEADS)
        dec = dec.to(DEV).eval()
        feats = nyu_feats(n, *spec)
        with torch.no_grad():
            return dec(feats, thr) if thr is not None else dec(feats)
    return run


def same(a, b, name):
    assert set(a) == set(b), (name, sorted(map(str, set(a) ^ set(b))))
    for k in a:
        x, y = a[k], b[k]
        if torch.is_tensor(x):
            assert x.shape == y.shape and x.dtype == y.dtype and torch.equal(x, y), (name, k, "differs under the harness")
        else:
            assert x == y, (name, k, x, y)
