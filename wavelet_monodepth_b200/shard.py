"""Batch-sharded inference over one process per GPU (SURVEY 8e).

Every sample is independent (thresholds, masks and active lists are per sample; weights are
replicated), so the batch is partitioned contiguously over ranks, each rank runs encoder features ->
decoder locally, and exactly ONE collective moves data: an all-gather of the full-resolution
``("disp", 0)`` tensor.  The reference has no distributed code at all (single process, single device:
KITTI/trainer.py:45, evaluate_depth.py:116); this is the one parallelism the hot path admits.
"""
import torch
import torch.distributed as dist


def shard_bounds(n, world, rank):
    """Contiguous [lo, hi) slice of a batch of n for `rank`; sizes differ by at most one."""
    base, rem = divmod(int(n), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_features(feats, world, rank):
    """Slice every feature map of a global batch to this rank's shard (views, no copy)."""
    lo, hi = shard_bounds(feats[0].shape[0], world, rank)
    return [f[lo:hi] for f in feats]


def all_gather_batch(local, n_global, group=None):
    """All-gather a batch-sharded tensor (shards from shard_bounds) into the global (n_global, ...) tensor.

    One collective.  Ragged shards (n_global % world != 0) are padded to the largest shard and trimmed.
    Uses all_gather_into_tensor on NCCL (a single NVLink/NVSwitch all-gather into the output buffer) and
    the list form elsewhere (gloo in the CPU tests).
    """
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local
    rank = dist.get_rank(group)
    per = -(-n_global // world)
    lo, hi = shard_bounds(n_global, world, rank)
    assert local.shape[0] == hi - lo, (local.shape, lo, hi)
    if local.shape[0] != per:
        pad = torch.zeros((per - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], 0)
    local = local.contiguous()
    gathered = torch.empty((world * per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(gathered, local, group=group)
    else:
        dist.all_gather(list(gathered.chunk(world, 0)), local, group=group)
    if n_global % world == 0:
        return gathered
    parts = []
    for r in range(world):
        a, b = shard_bounds(n_global, world, r)
        parts.append(gathered[r * per:r * per + (b - a)])
    return torch.cat(parts, 0)


class GatherHandle:
    """An all-gather in flight.  ``wait()`` makes the CURRENT stream wait for it (no host block on NCCL) and returns
    the global (n_global, ...) tensor."""

    def __init__(self, work, gathered, n_global, world, per):
        self._work, self._gathered, self._n, self._world, self._per = work, gathered, n_global, world, per

    def wait(self):
        if self._work is not None:
            self._work.wait()
            self._work = None
        if self._n % self._world == 0:
            return self._gathered
        parts = []
        for r in range(self._world):
            a, b = shard_bounds(self._n, self._world, r)
            parts.append(self._gathered[r * self._per:r * self._per + (b - a)])
        return torch.cat(parts, 0)


class OverlappedGather:
    """The path's one collective, taken off the critical path (SURVEY 8e: "optionally launched from the last IDWT
    kernel's stream so it overlaps the tail").

    ``start(local)`` copies this rank's ``("disp", 0)`` shard into a private staging buffer on the current stream
    (42 MB at 1024x320 bs 32: ~15 us) and issues ``all_gather_into_tensor`` asynchronously: NCCL's stream waits for
    the staging copy only, so the caller can enqueue the NEXT step's decoder right away - the decoder may overwrite
    its output tensor (CUDA-graph replays do) while the gather of the previous step is still moving data over
    NVLink.  Staging and output buffers are double-buffered: step k uses slot k % 2, and a slot is reused only after
    its previous gather has been waited for."""

    def __init__(self, n_global, group=None):
        self.n_global, self.group = int(n_global), group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.per = -(-self.n_global // self.world)
        self._slots = [None, None]
        self._k = 0

    def start(self, local):
        if self.world == 1:
            return GatherHandle(None, local, self.n_global, 1, self.per)
        slot = self._k % 2
        self._k += 1
        ent = self._slots[slot]
        if ent is None or ent["stage"].shape[1:] != local.shape[1:] or ent["stage"].dtype != local.dtype:
            stage = torch.zeros((self.per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
            out = torch.empty((self.world * self.per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
            ent = self._slots[slot] = {"stage": stage, "out": out, "handle": None}
        elif ent["handle"] is not None:
            ent["handle"].wait()                             # slot reuse: its previous gather must have been consumed
        lo, hi = shard_bounds(self.n_global, self.world, self.rank)
        assert local.shape[0] == hi - lo, (local.shape, lo, hi)
        ent["stage"][:hi - lo].copy_(local)
        if dist.get_backend(self.group) == "nccl":
            work = dist.all_gather_into_tensor(ent["out"], ent["stage"], group=self.group, async_op=True)
        else:
            work = dist.all_gather(list(ent["out"].chunk(self.world, 0)), ent["stage"], group=self.group, async_op=True)
        ent["handle"] = GatherHandle(work, ent["out"], self.n_global, self.world, self.per)
        return ent["handle"]


def make_gather(n_global, group=None):
    """The overlapped all-gather of this build: NCCL (OverlappedGather)."""
    return OverlappedGather(n_global, group)


def sharded_decode(decoder, local_feats, n_global, *args, gather_key=("disp", 0), group=None, **kwargs):
    """Run `decoder` on this rank's shard and all-gather its full-resolution output.

    Returns (local_outputs, global_disp)."""
    out = decoder(local_feats, *args, **kwargs)
    return out, all_gather_batch(out[gather_key], n_global, group=group)
