"""GPU: the window form of the tensor-core convolution (conv_rows_tc_kernel_window, csrc/conv_tc.cu).

A dense 3x3 launch (no pixel list, no index map, no gate, whole tiles or balanced) whose per-tile source windows fit a
slot runs in the window kernel.  The same launch with an identity map0 / map1 and an all-ones gate computes the same rows
through the gather kernel, so the two must give the same bits.  Every case is also checked against the fp64 contract
reference (tests/conv_ref.py) at the bars of test_gpu_conv_contract.py, including amax_out == max |y| and no writes
outside [0, rows) x [0, cout).
"""
import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from wavelet_monodepth_b200 import kitti_decoders as kd
from wavelet_monodepth_b200 import ops, synth
from wavelet_monodepth_b200._lib import PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

from test_gpu_conv_contract import Layer, operands, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
WIN, GATHER = "conv_rows_tc_kernel_window", "conv_rows_tc_kernel"


def tc_kernels(fn, launches):
    """Names (window / gather) of the tensor-core conv kernels fn launches, in launch order.  A short profiling session
    can come back without some kernel records; it is taken again until it holds all `launches`."""
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        evs = sorted((e for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and GATHER in e.name),
                     key=lambda e: e.time_range.start)
        if len(evs) >= launches:
            break
    return [WIN if WIN in e.name else GATHER for e in evs]


def twin(L):
    """The same launch through index maps and a gate that select every pixel: the gather kernel's rows."""
    total = L.n * L.h * L.w
    src0 = L.n * (L.h >> L.shift0) * (L.w >> L.shift0)
    map1 = torch.arange(total, dtype=torch.int32, device=DEV) if L.c1 else None
    return Layer(L.n, L.h, L.w, L.c0, L.cout, c1=L.c1, pad=L.pad, shift0=L.shift0,
                 map0=torch.arange(src0, dtype=torch.int32, device=DEV), map1=map1,
                 gate=torch.ones(total, dtype=torch.uint8, device=DEV))


# (n, h, w, c0, c1, cout, pad, shift0): H and W of 1, 2 and 3; tiles that span two images and row counts that are not
# multiples of 128; cin % 32 != 0 and cin % 4 != 0; cout tails of N = 128, 64 and 32; the widest windows that fit.
CASES = [
    (1, 1, 1, 20, 0, 33, PAD_ZERO, 0),
    (2, 1, 3, 6, 0, 63, PAD_REPLICATE, 0),
    (1, 2, 2, 36, 20, 129, PAD_REFLECT, 0),
    (3, 3, 1, 40, 0, 64, PAD_ZERO, 0),
    (2, 3, 2, 64, 6, 40, PAD_REFLECT, 0),
    (2, 3, 3, 33, 0, 96, PAD_REPLICATE, 0),
    (2, 2, 2, 40, 12, 96, PAD_REFLECT, 1),
    (3, 2, 2, 20, 0, 32, PAD_ZERO, 1),
    (2, 6, 10, 33, 0, 129, PAD_REPLICATE, 1),
    (2, 9, 45, 64, 20, 256, PAD_REFLECT, 0),       # 405 pixels per image
    (2, 10, 32, 96, 0, 256, PAD_REFLECT, 0),       # upconv(4, 0)'s geometry, fewer channels
    (2, 20, 64, 64, 128, 256, PAD_REFLECT, 1),     # upconv(4, 1)'s
    (2, 14, 38, 52, 36, 200, PAD_ZERO, 1),
    (1, 3, 79, 32, 8, 64, PAD_ZERO, 0),            # widest shift-0 window: 128 + 2 (79 + 1) = 288 rows
    (1, 4, 78, 20, 36, 48, PAD_REPLICATE, 1),      # widest with a full-resolution source 1 and shift0 = 1
    (1, 2, 192, 40, 0, 128, PAD_REFLECT, 1),       # widest half-resolution window: 3 x 96 rows
    (4, 40, 64, 64, 0, 256, PAD_REFLECT, 0),       # more tiles than SMs: data-parallel rounds + stream-K
    (4, 40, 64, 32, 64, 256, PAD_REPLICATE, 1),
]
# one past the widest window of each kind: the gather kernel runs them
TOO_WIDE = [
    (1, 3, 80, 32, 8, 64, PAD_ZERO, 0),
    (1, 4, 80, 20, 36, 48, PAD_REPLICATE, 1),
    (1, 2, 194, 40, 0, 128, PAD_REFLECT, 1),
]


def _layer(case):
    n, h, w, c0, c1, cout, pad, shift0 = case
    return Layer(n, h, w, c0, cout, c1=c1, pad=pad, shift0=shift0)


@pytest.mark.parametrize("dist", ["mixed", "same"])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("case", CASES + TOO_WIDE)
def test_window_kernel_gives_the_gather_kernels_bits(case, engine, splits, dist):
    L = _layer(case)
    ops_in = operands(L, dist, 7 * L.w + L.c0 + L.c1)
    got = run(L, engine, dist, "window", splits=splits, ops_in=ops_in)
    want = run(twin(L), engine, dist, "window", splits=splits, ops_in=ops_in)
    assert torch.equal(got, want)


@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
def test_dense_3x3_launches_whose_windows_fit_run_the_window_kernel(engine):
    launches = [(_layer(c), 0, WIN) for c in CASES] + [(_layer(c), 1, GATHER) for c in TOO_WIDE]
    launches.append((twin(_layer(CASES[11])), 0, GATHER))
    if engine == "tf32x3":
        launches.append((_layer(CASES[10]), 3, GATHER))       # split-K
    inputs = [operands(L, "mixed", 1) for L, _, _ in launches]
    names = tc_kernels(lambda: [run(L, engine, "mixed", "window", splits=s, ops_in=x)
                                for (L, s, _), x in zip(launches, inputs)], len(launches))
    assert names == [k for _, _, k in launches], names


def test_flagship_decoder_runs_its_dense_3x3_launches_in_the_window_kernel():
    mod = kd.SparseDepthWaveProgressiveDecoder(np.array(synth.RESNET50_CH))
    synth.bench_kitti_params(mod)
    mod = mod.to(DEV).eval()
    feats = [f.to(DEV) for f in synth.bench_kitti_features(2, 320, 1024, synth.RESNET50_CH)]
    mod(feats, 0.05)
    prof = ops.Profiler()
    ops.set_profiler(prof)
    try:
        mod(feats, 0.05)
        torch.cuda.synchronize()
    finally:
        ops.set_profiler(None)
    tc = [info for name, _, info in prof.results() if name == "conv_rows_tc"]
    names = tc_kernels(lambda: mod(feats, 0.05), len(tc))
    dense = [(info["taps"], info["c0"], info["c1"], info["cout"]) for info in tc]
    want = [WIN if d in ((9, 2048, 0, 256), (9, 256, 1024, 256)) else GATHER for d in dense]
    assert want.count(WIN) == 2, dense
    assert names == want, list(zip(dense, names))
