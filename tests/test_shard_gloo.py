"""CPU, world_size 2 over gloo: batch sharding + the single all-gather of the output depth tensor."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from wavelet_monodepth_b200 import shard, synth

from helpers import load_golden, seeded_params


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, n_global, result_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import kitti as okitti               # tests may use the oracle as the stand-in decoder
        from wavelet_monodepth_b200.kitti_decoders import DepthWaveProgressiveDecoder
        torch.set_grad_enabled(False)
        _, meta = load_golden("kitti_tiny_dense")
        mod = DepthWaveProgressiveDecoder(np.array(meta["num_ch_enc"]))
        sd = seeded_params(mod, meta)
        shapes = synth.kitti_feature_shapes(n_global, meta["height"], meta["width"], meta["num_ch_enc"])
        feats = synth.blocky_features(shapes, seed=meta["feat_seed"], cell=meta["cell"])
        local = shard.shard_features(feats, world, rank)
        lo, hi = shard.shard_bounds(n_global, world, rank)
        assert local[0].shape[0] == hi - lo
        out, full = shard.sharded_decode(lambda f: okitti.dense_forward(sd, f), local, n_global)
        assert full.shape[0] == n_global
        # the overlapped form: three "steps" whose local output buffer is overwritten right after start() - what a
        # CUDA-graph replay does - each gathered through the double-buffered staging slots
        assert type(shard.make_gather(n_global)) is shard.OverlappedGather
        og = shard.OverlappedGather(n_global)
        buf = torch.empty_like(out[("disp", 0)])
        handles, wants = [], []
        for k in range(5):
            buf.copy_(out[("disp", 0)] * (k + 1))
            handles.append(og.start(buf))
            buf.fill_(-1.0)                                # the producer moves on before the gather is consumed
            wants.append(full * (k + 1))
            if k >= 1:                                     # consume step k-1 while step k is in flight
                got = handles[k - 1].wait()
                assert torch.equal(got, wants[k - 1]), ("overlapped gather", k - 1)
        assert torch.equal(handles[4].wait(), wants[4])
        if rank == 0:
            ref = okitti.dense_forward(sd, feats)[("disp", 0)]
            torch.save({"full": full, "ref": ref}, os.path.join(result_dir, "r0_%d.pt" % n_global))
    finally:
        dist.destroy_process_group()


def _run(n_global, tmp_path):
    port = _free_port()
    mp.spawn(_worker, args=(2, port, n_global, str(tmp_path)), nprocs=2, join=True)
    res = torch.load(os.path.join(str(tmp_path), "r0_%d.pt" % n_global))
    # batch-1 and batch-N convolutions may round differently on the CPU backend; the gather itself is exact
    assert float((res["full"] - res["ref"]).abs().max()) < 1e-5


def test_even_shards_through_the_overlapped_gather(tmp_path):
    _run(2, tmp_path)


def test_ragged_shards_through_the_overlapped_gather(tmp_path):
    _run(3, tmp_path)


def test_shard_bounds_cover_batch():
    for n in (1, 2, 7, 8, 32, 255, 256):
        for world in (1, 2, 4, 8):
            spans = [shard.shard_bounds(n, world, r) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1
