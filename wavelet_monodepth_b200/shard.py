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


class PeerGather(OverlappedGather):
    """The same collective moved by the COPY ENGINES over NVLink peer memory instead of an NCCL kernel.

    Why: a persistent convolution CTA holds its SM's whole register file, so an NCCL all-gather kernel cannot run under
    the next step's decoder - it waits for a gap and its duration lands on the step (measured: 2 GPUs 3.84 vs 3.70 ms,
    4 GPUs 3.90 vs 3.70 ms, the difference = the collective's own 0.14 / 0.27 ms).  DMA engines need no SM.

    Every rank owns three (world x shard) output buffers whose CUDA IPC handles all ranks open once (`reduce_tensor`,
    exchanged with `all_gather_object`).  ``start(local)``: staging copy on the current stream (as OverlappedGather),
    then on a private copy stream one `cudaMemcpyPeerAsync` of the shard into slot k % 3 of EVERY rank's buffer, then a
    4-byte NCCL all-reduce as the arrival barrier: it is stream-ordered after this rank's copies, so its completion
    anywhere means every shard has landed everywhere.  ``handle.wait()`` makes the current stream wait for that barrier.
    Slot reuse: the copies of step k + 3 wait for the barrier of step k + 2, which every rank joined after the work its
    main stream held at ``start(k + 2)`` - i.e. after it consumed step k (consume a step before the second ``start``
    after it; OverlappedGather has the same rule with one step less slack).

    Falls back to the NCCL form (the parent class) when peer access, IPC or the start-up self-check fails.  Opt-in
    (make_gather): whether copy engines beat NCCL's SM kernels here depends on the platform's peer-copy rate."""

    SLOTS = 3

    def __init__(self, n_global, group=None):
        super().__init__(n_global, group)
        self._peer = None            # None = not set up yet, False = unavailable (NCCL form), dict = ready
        self.why_not = None

    def _agree(self, ok, dev):
        """True iff every rank says ok (one tiny all-reduce: all ranks call it at the same points whatever happened locally)."""
        t = torch.tensor([1.0 if ok else 0.0], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        return float(t) == 1.0

    def _setup(self, local):
        """Every rank runs the same sequence of collectives whatever fails locally; one failure anywhere = NCCL form everywhere."""
        if self.world == 1 or not local.is_cuda or dist.get_backend(self.group) != "nccl":
            self._peer, self.why_not = False, "needs NCCL ranks on CUDA devices"
            return
        dev = local.device
        outs = stage = payload = None
        try:                                          # phase A: local buffers + IPC handles
            from torch.multiprocessing.reductions import reduce_tensor
            shape = (self.world * self.per,) + tuple(local.shape[1:])
            outs = [torch.zeros(shape, dtype=local.dtype, device=dev) for _ in range(self.SLOTS)]
            stage = [torch.zeros((self.per,) + tuple(local.shape[1:]), dtype=local.dtype, device=dev) for _ in range(self.SLOTS)]
            payload = (dev.index, [reduce_tensor(t) for t in outs])
        except Exception as e:                        # noqa: BLE001
            self.why_not = "%s: %s" % (type(e).__name__, e)
        handles = [None] * self.world
        dist.all_gather_object(handles, payload, group=self.group)
        peers = None
        try:                                          # phase B: open every rank's buffers
            if any(h is None for h in handles):
                raise RuntimeError("a rank could not export its buffers")
            if len({h[0] for h in handles}) != self.world:
                raise RuntimeError("ranks do not see distinct device indices (masked CUDA_VISIBLE_DEVICES?)")
            for idx, _ in handles:
                if idx != dev.index and not torch.cuda.can_device_access_peer(dev.index, idx):
                    raise RuntimeError("no peer access %d -> %d" % (dev.index, idx))
            peers = [outs if r == self.rank else [fn(*a) for fn, a in hs] for r, (idx, hs) in enumerate(handles)]
        except Exception as e:                        # noqa: BLE001
            self.why_not = self.why_not or "%s: %s" % (type(e).__name__, e)
        if not self._agree(peers is not None, dev):
            self._peer, self.why_not = False, self.why_not or "another rank could not set up peer buffers"
            return
        self._peer = {"outs": outs, "stage": stage, "peers": peers, "stream": torch.cuda.Stream(dev),
                      "flag": torch.zeros(1, device=dev), "work": [None] * self.SLOTS, "shape": tuple(local.shape[1:]),
                      "dtype": local.dtype}
        # phase C: self-check against the NCCL all-gather on a rank-stamped pattern
        lo, hi = shard_bounds(self.n_global, self.world, self.rank)
        probe = torch.full((hi - lo,) + tuple(local.shape[1:]), float(self.rank + 1), dtype=local.dtype, device=dev)
        got = self._start_peer(probe).wait()
        torch.cuda.synchronize(dev)
        want = all_gather_batch(probe, self.n_global, self.group)
        if not self._agree(torch.equal(got, want), dev):
            self._peer, self.why_not = False, "self-check against the NCCL all-gather failed"
            return
        self._k = 0

    def _start_peer(self, local):
        st = self._peer
        slot = self._k % self.SLOTS
        self._k += 1
        lo, hi = shard_bounds(self.n_global, self.world, self.rank)
        assert local.shape[0] == hi - lo, (local.shape, lo, hi)
        if st["work"][slot] is not None:              # the slot's previous barrier (three steps ago) has long completed
            st["work"][slot].wait()
        st["stage"][slot][:hi - lo].copy_(local)
        ready = torch.cuda.Event()
        ready.record()
        prev = st["work"][(slot - 1) % self.SLOTS]
        with torch.cuda.stream(st["stream"]):
            st["stream"].wait_event(ready)
            if prev is not None:
                prev.wait()                           # everyone has consumed what this slot held (see the class docstring)
            for i in range(self.world):               # staggered: rank r starts with r + 1, so the links are used evenly
                p = (self.rank + 1 + i) % self.world
                st["peers"][p][slot][self.rank * self.per:self.rank * self.per + (hi - lo)].copy_(st["stage"][slot][:hi - lo],
                                                                                              non_blocking=True)
            work = dist.all_reduce(st["flag"], group=self.group, async_op=True)
        st["work"][slot] = work
        return GatherHandle(work, st["outs"][slot], self.n_global, self.world, self.per)

    def start(self, local):
        if self.world == 1:
            return GatherHandle(None, local, self.n_global, 1, self.per)
        if self._peer is None:
            self._setup(local)
        if self._peer is False or tuple(local.shape[1:]) != self._peer["shape"] or local.dtype != self._peer["dtype"]:
            return super().start(local)
        return self._start_peer(local)


def make_gather(n_global, group=None):
    """The overlapped all-gather of this build: NCCL (OverlappedGather); env WMD_PEER_GATHER=1 selects the copy-engine form.

    PeerGather is checked by scripts/peer_gather_check.py (even and ragged shards, 12 overlapped steps) and its copy rate
    by scripts/peer_copy_probe.py; neither has been measured on H100.  It stays opt-in for platforms whose DMA engines
    run at NVLink speed."""
    import os
    if os.environ.get("WMD_PEER_GATHER", "0") == "1" and dist.is_initialized() and dist.get_backend(group) == "nccl":
        return PeerGather(n_global, group)
    return OverlappedGather(n_global, group)


def sharded_decode(decoder, local_feats, n_global, *args, gather_key=("disp", 0), group=None, **kwargs):
    """Run `decoder` on this rank's shard and all-gather its full-resolution output.

    Returns (local_outputs, global_disp)."""
    out = decoder(local_feats, *args, **kwargs)
    return out, all_gather_batch(out[gather_key], n_global, group=group)
