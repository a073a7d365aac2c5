"""CPU: the seam a maintainer of the reference touches (INTEGRATION.md section A), checked against the reference's own
module layout as oracle/pin_reference_layout.py recorded it from the UNMODIFIED reference tree
(tests/golden/reference_layout.json).  Not arithmetic:
  * for every decoder the reference's factories build (KITTI/networks/network_constructors.py:30-40, NYUv2/model.py:47-71)
    ours has the same class name, state-dict keys and shapes, so the three-line swap builds OUR classes in its place and
    checkpoints load STRICTLY in both directions (KITTI/test_simple.py:101-102);
  * ``.convs`` has the reference's keys and every parameter is reachable through it the way ``pyt_utils.group_weight``
    collects them (KITTI/trainer.py:74-75, KITTI/pyt_utils.py:12-29: Conv/Linear weights and biases only);
  * checkpoints survive the trainer's save / load code paths on disk (KITTI/trainer.py:733-773 pattern);
  * without CUDA the decoders fail loudly (no silent CPU path);
  * the public functions of KITTI/layers.py exist here with the same parameter names.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from helpers import GOLDEN

with open(os.path.join(GOLDEN, "reference_layout.json")) as _f:
    LAYOUT = json.load(_f)


class _Encoder:
    num_ch_enc = np.array(LAYOUT["kitti_num_ch_enc"])


def _kitti_decoder(case):
    from wavelet_monodepth_b200 import kitti_decoders as kd
    cls = getattr(kd, LAYOUT["kitti"][case]["class"])
    return cls(_Encoder.num_ch_enc) if cls is kd.SparseDepthWaveProgressiveDecoder else cls(_Encoder.num_ch_enc, range(4))


def _reference_state_dict(entry, seed):
    """A state dict with the reference module's keys and shapes (what its torch.save would have written), seeded values."""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.rand(tuple(s), generator=g) for k, s in zip(entry["keys"], entry["shapes"])}


def _grouped_params(convs):
    """Parameters pyt_utils.group_weight collects from the values of ``.convs``: Conv / Linear weights and biases."""
    n = 0
    for module in convs.values():
        for m in module.modules():
            if isinstance(m, (nn.Linear, nn.Conv2d, nn.Conv3d)):
                n += 1 + (m.bias is not None)
    return n


def _check_layout(module, entry):
    assert type(module).__name__ == entry["class"]
    sd = module.state_dict()
    assert list(sd.keys()) == entry["keys"], entry["class"]
    assert [list(v.shape) for v in sd.values()] == entry["shapes"], entry["class"]


def test_kitti_factory_builds_our_decoders_and_trainer_param_groups_accept_them():
    """Every configuration of make_depth_decoder (wavelets, sparse, dense): the class the factory builds, its state dict,
    ``.convs`` and group_weight's parameter count, and strict loading both ways."""
    for case, entry in sorted(LAYOUT["kitti"].items()):
        dec = _kitti_decoder(case)
        _check_layout(dec, entry)
        assert [list(k) if isinstance(k, tuple) else k for k in dec.convs.keys()] == entry["convs"], case   # JSON: tuples as lists
        assert _grouped_params(dec.convs) == entry["grouped_params"] == len(list(dec.parameters())) > 0, case
        ref_sd = _reference_state_dict(entry, seed=1)
        dec.load_state_dict(ref_sd, strict=True)                     # reference checkpoint -> ours
        twin = _kitti_decoder(case)
        twin.load_state_dict(dec.state_dict(), strict=True)          # ours -> a module with the reference's layout
        for k, v in ref_sd.items():
            assert torch.equal(twin.state_dict()[k], v), (case, k)


def test_kitti_checkpoints_round_trip_on_disk_through_the_trainers_code_path(tmp_path):
    entry = LAYOUT["kitti"]["sparse"]
    ours = _kitti_decoder("sparse")
    # trainer.save_model (:733-751): torch.save(model.state_dict(), "<name>.pth"); the reference module's file
    torch.save(ours.state_dict(), tmp_path / "depth.pth")
    torch.save(_reference_state_dict(entry, seed=2), tmp_path / "depth_ref.pth")
    # test_simple.py:101-102: strict load of depth.pth into a module with the reference's layout
    theirs = _kitti_decoder("sparse")
    theirs.load_state_dict(torch.load(tmp_path / "depth.pth", map_location="cpu"))
    for k, v in ours.state_dict().items():
        assert torch.equal(theirs.state_dict()[k], v), k
    # trainer.load_model (:753-773): filter by key, update, load
    model_dict = ours.state_dict()
    pretrained = {k: v for k, v in torch.load(tmp_path / "depth_ref.pth").items() if k in model_dict}
    assert set(pretrained) == set(model_dict)
    model_dict.update(pretrained)
    ours.load_state_dict(model_dict)
    for k, v in torch.load(tmp_path / "depth_ref.pth").items():      # what the reference module had saved
        assert torch.equal(ours.state_dict()[k], v), k
    # evaluate_depth.py:130 loads non-strictly
    ours.load_state_dict(torch.load(tmp_path / "depth_ref.pth"), strict=False)


def test_swapped_kitti_decoder_fails_loudly_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from wavelet_monodepth_b200 import kitti_decoders as kd
    from wavelet_monodepth_b200._lib import WmdError
    dec = kd.SparseDepthWaveProgressiveDecoder(_Encoder.num_ch_enc)
    feats = [torch.rand(1, c, 6 << (4 - k), 20 << (4 - k)) for k, c in enumerate(_Encoder.num_ch_enc)]
    with pytest.raises(WmdError):
        dec(feats, 0.05)


def test_nyu_model_builds_our_decoders_and_load_save_utils_round_trip(tmp_path):
    """Every decoder NYUv2 Model builds (wavelets, sparse, 224 variants, dense): class, state dict, strict loading both
    ways and a save / load round trip on disk."""
    from wavelet_monodepth_b200 import nyu_decoders as nd
    for case, entry in sorted(LAYOUT["nyu"].items()):
        cls = getattr(nd, entry["class"])
        dec = cls(enc_features=entry["enc_features"], decoder_width=0.5)
        _check_layout(dec, entry)
        ref_sd = _reference_state_dict(entry, seed=3)
        dec.load_state_dict(ref_sd, strict=True)
        path = tmp_path / ("%s.pth" % case)
        torch.save(dec.state_dict(), path)                           # load_save_utils.save_model / load_model pattern
        twin = cls(enc_features=entry["enc_features"], decoder_width=0.5)
        twin.load_state_dict(torch.load(path), strict=True)
        for k, v in ref_sd.items():
            assert torch.equal(twin.state_dict()[k], v), (case, k)


def test_functional_api_names_match_the_reference_layers():
    """Every public name of the hot path in KITTI/layers.py exists with the same parameter names here."""
    import inspect
    from wavelet_monodepth_b200 import kitti_layers as kl
    for name, pa in LAYOUT["kitti_layer_signatures"].items():
        b = getattr(kl, name)
        if inspect.isclass(b):
            assert issubclass(b, nn.Module)
            b = b.__init__
        pb = list(inspect.signature(b).parameters)
        assert pa == pb[:len(pa)], (name, pa, pb)
