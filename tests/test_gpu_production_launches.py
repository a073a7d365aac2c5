"""GPU: every libwmd launch of the benchmarked decoders, at the benchmark's sizes and on its synthetic inputs, against the
fp64 contract of its kernel (tests/launch_check.py).

The kernel contract tests run on synthetic shapes and data; the decoders' own launches have properties that only exist in
production: data-dependent row counts, stream-K cuts and balanced remainders; fp16-pair operand scales taken from the
decoders' amax slots (one per source for the whole batch); high-pass heads whose outputs cancel in flat regions; backward
paths such as the split-pixel weight gradient of a cout-1 layer over 1.5 M rows.  Each workload runs once plainly and once
under the harness, which checks each launch element by element at its kernel's bar, its preconditions, and that every
kernel launched ran inside a checked call, with every buffer guarded and poisoned, exactly sized workspaces and inputs
compared bit for bit after each call.  The two runs must agree bit for bit (outputs, and in training the gradients): the
harness does not change what it checks, and results depend neither on timing, nor on buffer reuse, nor on what was in
memory.  The launch symbols launch_check.REACH attributes to a workload must be called by it.
"""
import gc
import time

import numpy as np
import pytest
import torch

from wavelet_monodepth_b200 import kitti_decoders as kd, nyu_decoders as nd, synth

import launch_check as lc
from workloads import D161, DEV, R18, R50, kitti_feats, nyu, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from lc.REPORT.module_report()


@pytest.fixture(autouse=True)
def _fp32_convs():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def kitti_sparse(n, spec, thr, layout="nchw"):
    def run():
        dec = kd.SparseDepthWaveProgressiveDecoder(np.array(spec[0]))
        synth.bench_kitti_params(dec)
        dec = dec.to(DEV).eval()
        return dec(kitti_feats(n, *spec, layout=layout), thr)
    return run


def kitti_dense(n, spec):
    def run():
        dec = kd.DepthWaveProgressiveDecoder(np.array(spec[0]))
        synth.bench_kitti_params(dec)
        with torch.no_grad():
            return dec.to(DEV).eval()(kitti_feats(n, *spec))
    return run


def kitti_baseline(n, spec):
    def run():
        dec = kd.DepthDecoder(np.array(spec[0]))
        synth.load_random(dec, seed=7)
        with torch.no_grad():
            return dec.to(DEV).eval()(kitti_feats(n, *spec))
    return run


def train_step(kind, n, spec):
    """One native training step (scripts/train_step_bench.py): outputs, parameter and input-feature gradients."""
    def run():
        ch, h, w = spec
        if kind == "kitti_wave":
            mod = kd.DepthWaveProgressiveDecoder(np.array(ch))
        elif kind == "kitti_baseline":
            mod = kd.DepthDecoder(np.array(ch))
        else:
            mod = nd.DecoderWave(enc_features=list(ch), decoder_width=0.5)
        shapes = (synth.nyu_feature_shapes if kind == "nyu_wave" else synth.kitti_feature_shapes)(n, h, w, ch)
        synth.load_random(mod, seed=1)
        mod = mod.to(DEV).train()
        feats = [f.to(DEV).requires_grad_(True) for f in synth.blocky_features(shapes, seed=2)]
        out = mod(feats)
        sum(v.mean() for k, v in out.items() if k[0] == "disp").backward()
        res = {("out",) + tuple(k): v.detach() for k, v in out.items()}
        res.update({("grad", k): p.grad for k, p in mod.named_parameters() if p.grad is not None})
        res.update({("feature_grad", j): f.grad for j, f in enumerate(feats) if f.grad is not None})
        return res
    return run


WORKLOADS = {
    "sparse_r50_1024x320_x32_thr0.05": kitti_sparse(32, R50, 0.05),
    "sparse_r50_1024x320_x32_thr0": kitti_sparse(32, R50, 0.0),
    "sparse_r50_1024x320_x32_thr0.1": kitti_sparse(32, R50, 0.1),
    "sparse_r50_1024x320_x16_channels_last": kitti_sparse(16, R50, 0.05, "channels_last"),
    "sparse_r50_1024x320_x16_pinned_host": kitti_sparse(16, R50, 0.05, "pinned"),
    "dense_r50_1024x320_x32": kitti_dense(32, R50),
    "sparse_r18_640x192_x16_thr0.05": kitti_sparse(16, R18, 0.05),
    "nyu_sparse_d161_640x480_x8_thr0.1": nyu(nd.SparseDecoderWave, 8, D161, 0.1),
    "nyu_dense_d161_640x480_x8": nyu(nd.DecoderWave, 8, D161),
    "baseline_depthdecoder_r18_640x192_x16": kitti_baseline(16, R18),
    "baseline_densedepth_d161_640x480_x8": nyu(nd.Decoder, 8, D161),
    "train_wave_r18_640x192_x12": train_step("kitti_wave", 12, R18),
    "train_depthdecoder_r18_640x192_x12": train_step("kitti_baseline", 12, R18),
    "train_nyu_wave_d161_640x480_x8": train_step("nyu_wave", 8, D161),
}


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_every_launch_meets_its_contract(name, monkeypatch):
    run = WORKLOADS[name]
    t0 = time.perf_counter()
    plain = run()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    harness = lc.Harness(monkeypatch)
    with harness.workload(name):
        checked = run()
    monkeypatch.undo()
    t2 = time.perf_counter()
    same(plain, checked, name)
    assert not harness.reached(name), (name, "never called", harness.reached(name))
    print("%s (%.1f s plain, %.1f s checked; %s): %s" % (name, t1 - t0, t2 - t1, harness.report(),
                                                         ", ".join("%s x%d" % kv for kv in sorted(harness.calls.items()))))
    del plain, checked, harness
    gc.collect()
    torch.cuda.empty_cache()
