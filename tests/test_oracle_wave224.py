"""CPU: the oracle's 224-pixel NYU decoder and its KITTI decoder without skips reproduce the unmodified reference's
outputs (tests/golden/nyu224_tiny_dense.npz, kitti_tiny_dense_noskip.npz, written by oracle/pin_wave224.py)
bit for bit, and the native modules keep the reference's state-dict layout."""
import numpy as np
import pytest
import torch

from oracle import wave224
from wavelet_monodepth_b200.kitti_decoders import DepthWaveProgressiveDecoder
from wavelet_monodepth_b200.nyu_decoders import DecoderWave224

from helpers import compare_outputs, key_str, kitti_features, load_golden, nyu_features, seeded_params

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


def test_nyu224_dense_matches_reference_golden_bit_exactly():
    want, meta = load_golden("nyu224_tiny_dense")
    mod = DecoderWave224(enc_features=list(meta["enc_features"]), decoder_width=0.5)
    got = wave224.nyu224_dense_forward(seeded_params(mod, meta), nyu_features(meta))
    _exact(got, want, "nyu224 dense")
    # the fixture exercises the floor division: ("disp", 1) holds several integers, and no other output is integral
    d1 = want["disp_1"]
    assert np.all(d1 == np.floor(d1)) and len(np.unique(d1)) >= 5
    assert not np.all(want["disp_2"] == np.floor(want["disp_2"]))


def test_kitti_dense_without_skips_matches_reference_golden_bit_exactly():
    want, meta = load_golden("kitti_tiny_dense_noskip")
    assert meta["use_skips"] is False
    mod = DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]), use_skips=False)
    feats = kitti_features(meta)
    got = wave224.kitti_dense_noskip_forward(seeded_params(mod, meta), feats)
    _exact(got, want, "kitti dense without skips")
    # only the coarsest map is read
    nan = [torch.full_like(f, float("nan")) for f in feats[:4]] + [feats[4]]
    _exact(wave224.kitti_dense_noskip_forward(seeded_params(mod, meta), nan), want, "kitti dense without skips, NaN skips")


def test_nyu224_fixture_keys_and_shapes():
    """Four IDWT levels: ("disp", 0) at the input resolution, the LL coefficients only at scale 3."""
    want, meta = load_golden("nyu224_tiny_dense")
    n, hh, ww = meta["n"], meta["height"], meta["width"]
    for s in range(4):
        assert want["disp_%d" % s].shape == (n, 1, hh >> s, ww >> s)
        for band in ("LH", "HL", "HH"):
            assert want["wavelets_%d_%s" % (s, band)].shape == (n, 1, hh >> (s + 1), ww >> (s + 1))
    assert want["wavelets_3_LL"].shape == (n, 1, hh >> 4, ww >> 4)
    assert not any(k.endswith("_LL") and k != "wavelets_3_LL" for k in want)


def test_decoder224_state_dict_layout_is_unchanged_by_the_shared_base():
    """The module order of the reference's DecoderWave224 (densedepth_decoder.py:152-179)."""
    mod = DecoderWave224()
    names = [k.rsplit(".", 1)[0] for k in mod.state_dict()]
    order = list(dict.fromkeys(n.split(".")[0] for n in names))
    assert order == ["iwt", "iwt_LL", "conv2", "up1", "wave1_ll", "wave1", "up2", "wave2", "up3", "wave3", "up4", "wave4"]
    shapes = {k: tuple(v.shape) for k, v in mod.state_dict().items()}
    assert shapes["conv2.conv.weight"] == (1104, 2208, 3, 3)
    assert shapes["up1.convA.conv.weight"] == (552, 1104 + 384, 3, 3)
    assert shapes["up4.convA.conv.weight"] == (69, 138 + 96, 3, 3)
    assert shapes["wave4.conv.weight"] == (3, 69, 3, 3)
