"""GPU: the window form of the tensor-core convolution (conv_rows_tc_kernel_window, csrc/conv_tc.cu).

A dense 3x3 launch (no pixel list, no index map, no gate, whole tiles or balanced) whose per-tile source windows fit a
slot runs in the window kernel.  The same launch with an identity map0 / map1 and an all-ones gate computes the same rows
through the row-set kernel (the gather kernel where tc_rowset_takes does not pick that), so the two must give the same
bits.  Every case is also checked against the fp64 contract reference (tests/conv_ref.py) at the bars of
test_gpu_conv_contract.py, including amax_out == max |y| and no writes outside [0, rows) x [0, cout).
"""
import pytest
import torch

from wavelet_monodepth_b200._lib import PAD_REFLECT, PAD_REPLICATE, PAD_ZERO

from conv_launch import (FLAGSHIP_DENSE, GATHER, SET, WIN, WORST, dense_layer, flagship_tc_kernels, operands, run,
                         tc_kernels, twin)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield from WORST.module_report()


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


@pytest.mark.parametrize("dist", ["mixed", "same"])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("case", CASES + TOO_WIDE)
def test_window_kernel_gives_the_gather_kernels_bits(case, engine, splits, dist):
    L = dense_layer(case)
    ops_in = operands(L, dist, 7 * L.w + L.c0 + L.c1)
    got = run(L, engine, dist, "window", splits=splits, ops_in=ops_in)
    want = run(twin(L), engine, dist, "window", splits=splits, ops_in=ops_in)
    assert torch.equal(got, want)


@pytest.mark.parametrize("engine", ["f16x3", "tf32x3"])
def test_dense_3x3_launches_whose_windows_fit_run_the_window_kernel(engine):
    launches = [(dense_layer(c), 0, WIN) for c in CASES] + [(dense_layer(c), 1, GATHER) for c in TOO_WIDE]
    # the same layer through identity maps and a gate: the row-set kernel, except on tf32x3's N = 128 tiles (cout 256)
    launches.append((twin(dense_layer(CASES[11])), 0, SET if engine == "f16x3" else GATHER))
    if engine == "tf32x3":
        launches.append((dense_layer(CASES[10]), 3, GATHER))       # split-K
    inputs = [operands(L, "mixed", 1) for L, _, _ in launches]
    names = tc_kernels(lambda: [run(L, engine, "mixed", "window", splits=s, ops_in=x)
                                for (L, s, _), x in zip(launches, inputs)], len(launches))
    assert names == [k for _, _, k in launches], names


def test_flagship_decoder_runs_its_dense_3x3_launches_in_the_window_kernel():
    shapes, names = flagship_tc_kernels()
    want = [WIN if s in FLAGSHIP_DENSE else (SET if s[0] == 9 else GATHER) for s in shapes]
    assert want.count(WIN) == 2, shapes
    assert names == want, list(zip(shapes, names))
