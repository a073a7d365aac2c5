"""CPU: the oracle's baseline decoders reproduce the unmodified reference's outputs (tests/golden/kitti_tiny_baseline.npz,
nyu_tiny_baseline.npz, nyu224_tiny_baseline.npz, written by oracle/pin_baseline.py) bit for bit, and the native modules
keep the reference's state-dict layout."""
import numpy as np
import pytest
import torch

from oracle import baseline
from wavelet_monodepth_b200 import kitti_decoders as kd, nyu_decoders as nd

from helpers import key_str, kitti_features, kitti_variant, load_golden, nyu_features, seeded_params

GOLDEN_THREADS = 8   # intra-op threads of the run that recorded the fixtures (see test_oracle_golden.py)


@pytest.fixture(autouse=True)
def _no_grad():
    was = torch.get_num_threads()
    torch.set_num_threads(GOLDEN_THREADS)
    try:
        with torch.no_grad():
            yield
    finally:
        torch.set_num_threads(was)


def _exact(got, want, what):
    got = {key_str(k): v for k, v in got.items()}
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    for k, wv in want.items():
        np.testing.assert_array_equal(got[k].numpy(), wv, err_msg="%s %s" % (what, k))


@pytest.mark.parametrize("name", ["default", "scales13", "noskip", "ch3"])
def test_kitti_baseline_matches_reference_golden_bit_exactly(name):
    want, meta = load_golden("kitti_tiny_baseline")
    kw, arrays = kitti_variant(want, meta, name)
    mod = kd.DepthDecoder(np.array(meta["num_ch_enc"]), **kw)
    got = baseline.kitti_baseline_forward(seeded_params(mod, meta), kitti_features(meta),
                                          scales=kw.get("scales", range(4)), use_skips=kw.get("use_skips", True))
    _exact(got, arrays, "kitti baseline " + name)
    cout = kw.get("num_output_channels", 1)
    for k, v in arrays.items():
        s = int(k.split("_")[1])
        assert v.shape == (2, cout, meta["height"] >> s, meta["width"] >> s)


@pytest.mark.parametrize("cls,fixture,extra", [(nd.Decoder, "nyu_tiny_baseline", False),
                                               (nd.Decoder224, "nyu224_tiny_baseline", True)])
def test_nyu_baseline_matches_reference_golden_bit_exactly(cls, fixture, extra):
    want, meta = load_golden(fixture)
    mod = cls(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    got = baseline.nyu_baseline_forward(seeded_params(mod, meta), nyu_features(meta), extra_stage=extra)
    _exact(got, want, fixture)
    assert want["disp_0"].shape == (2, 1, meta["height"] // (1 if extra else 2), meta["width"] // (1 if extra else 2))


@pytest.mark.parametrize("cls,fixture", [(nd.Decoder, "nyu_tiny_baseline"), (nd.Decoder224, "nyu224_tiny_baseline")])
def test_nyu_baseline_state_dict_is_the_references(cls, fixture):
    """Keys, order and shapes of the reference's module at its default (DenseNet161) widths, recorded in the fixture."""
    _, meta = load_golden(fixture)
    got = {k: list(v.shape) for k, v in cls().state_dict().items()}
    assert list(got.items()) == list(meta["state_dict"].items())


def test_kitti_baseline_slots_follow_the_module_list():
    mod = kd.DepthDecoder(np.array((8, 8, 16, 32, 64)), scales=[3, 1])
    order = list(mod.convs)
    for key, k in baseline.kitti_slots([3, 1]).items():
        assert order[k] == key
