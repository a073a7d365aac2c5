"""A guarded, poisoning allocator: what each libwmd launch writes past its buffers, and what it reads that it never wrote.

While a `Footprint` is active, `torch.empty`, `empty_like`, `zeros` and `zeros_like` for tensors on its device type
return views into arenas laid out [guard | buffer | guard] instead of blocks of PyTorch's caching allocator, which
rounds every block up to 512 B and to its size classes, so a write past a buffer lands in slack or in another live
tensor and nothing notices:
  - each guard is GUARD bytes of GUARD_BYTE; the buffer starts ALIGN-aligned and ends exactly where the tensor's last
    element ends, so a write one element before or after it lands in a guard;
  - an `empty` buffer is filled with POISON bytes (float and double NaN, integers -1, uint8 255) instead of what the
    allocator last left there (in a fresh process mostly zeros, which hides a read of a cell no one wrote); a `zeros`
    buffer is zero;
  - dtype, shape and memory format are torch's own: the strides come from the same call on device="meta".
Other devices, pinned host memory, `out=`, `requires_grad=True` and non-strided layouts pass through unchanged.

The modules look these functions up on the torch module at call time, so patching its attributes reaches every
allocation they make.  When a view dies its arena is queued; queued guards are checked in batches, one synchronize per
batch, so memory stays bounded, never while the current stream is capturing a CUDA graph.  An arena allocated during a
capture has its fills recorded into the graph rather than run, so its guards are checked only when the Footprint
ends: a graph captured under it must be replayed before then.  On exit every arena still held or alive is checked and
FootprintError names each written guard byte with the function that allocated the buffer.

Device-agnostic: Footprint("cpu") guards CPU tensors, which is how the CPU tests show that the checks catch what they
claim to.
"""
import sys
import threading
import weakref

import torch

GUARD = 256 << 10
GUARD_BYTE = 0xA5
POISON = 0xFF
ALIGN = 256
PATCHED = ("empty", "empty_like", "zeros", "zeros_like")
PACKAGE = "wavelet_monodepth_b200"
BATCH = 256                        # dead arenas per guard check
BATCH_BYTES = 4 << 30              # or this many bytes of them, whichever comes first


class FootprintError(AssertionError):
    pass


def _extent(shape, stride):
    """elements between a strided tensor's first and last element, both included (0 if it has none)"""
    if any(n == 0 for n in shape):
        return 0
    return 1 + sum((n - 1) * s for n, s in zip(shape, stride))


def _view(arena, start, meta):
    """the buffer of `arena` at byte `start` as a tensor of meta's dtype, shape and strides"""
    return arena.view(meta.dtype).as_strided(meta.shape, meta.stride(), start // meta.element_size())


def check_layout(view, meta):
    """view is what torch would have allocated: meta's dtype, shape and strides, on an ALIGN-aligned buffer"""
    if view.dtype != meta.dtype or view.shape != meta.shape or view.stride() != meta.stride():
        raise FootprintError("guarded %s %s with strides %s, torch allocates %s %s with strides %s"
                             % (view.dtype, tuple(view.shape), view.stride(), meta.dtype, tuple(meta.shape), meta.stride()))
    if view.data_ptr() % ALIGN:
        raise FootprintError("guarded buffer at %#x is not %d-byte aligned" % (view.data_ptr(), ALIGN))


def _caller():
    """'module.function' of the nearest package frame that asked for the allocation, else of the first frame outside
    this file"""
    f = sys._getframe(3)
    first = None
    while f is not None:
        mod = f.f_globals.get("__name__", "")
        if mod.startswith(PACKAGE):
            return "%s.%s" % (mod[len(PACKAGE) + 1:], f.f_code.co_qualname)
        if first is None and mod != __name__:
            first = "%s.%s" % (mod, f.f_code.co_qualname)
        f = f.f_back
    return first or "?"


class _Arena:
    __slots__ = ("arena", "start", "nbytes", "what", "captured", "fin")

    def __init__(self, arena, start, nbytes, what, captured):
        self.arena, self.start, self.nbytes, self.what, self.captured, self.fin = arena, start, nbytes, what, captured, None

    def guards(self):
        s, e = self.start, self.start + self.nbytes
        return self.arena[s - GUARD:s], self.arena[e:e + GUARD]


def guard_faults(before, after):
    """[(side, offset)] of the guard bytes that are not GUARD_BYTE: ("before", bytes before the buffer's start) for
    the nearest one in front, ("after", bytes past the buffer's end) for the nearest one behind"""
    out = []
    for side, g in (("before", before.flip(0)), ("after", after)):
        bad = (g != GUARD_BYTE).nonzero()
        if bad.numel():
            out.append((side, int(bad[0, 0]) + (side == "before")))
    return out


class Footprint:
    """with Footprint() as fp: ... - see the module docstring.  fp.checked arenas were checked, fp.guarded bytes of
    buffers lay between their guards, fp.allocated arenas were made."""

    def __init__(self, device_type="cuda"):
        self.device_type = device_type
        self.lock = threading.RLock()
        self.live = {}               # id -> _Arena whose view is alive
        self.queue = []              # dead, not yet checked
        self.queued_bytes = 0
        self.held = []               # allocated during a graph capture: checked on exit
        self.faults = []
        self.checked = self.guarded = self.allocated = 0
        self._orig = {}

    # ------------------------------------------------------------------------------------------ patching
    def __enter__(self):
        for name in PATCHED:
            self._orig[name] = getattr(torch, name)
            setattr(torch, name, self._patched(name))
        return self

    def __exit__(self, exc_type, exc, tb):
        for name, fn in self._orig.items():
            setattr(torch, name, fn)
        with self.lock:
            for rec in self.live.values():
                rec.fin.detach()
            pending = self.queue + self.held + list(self.live.values())
            self.live, self.queue, self.held, self.queued_bytes = {}, [], [], 0
        if exc_type is not None:
            return False
        self._check(pending)
        if self.faults:
            raise FootprintError("%d buffers written outside their bounds:\n  %s"
                                 % (len(self.faults), "\n  ".join(self.faults[:20])))
        return False

    def _patched(self, name):
        orig = self._orig[name]
        like = name.endswith("_like")
        zero = name.startswith("zeros")

        def alloc(*args, **kwargs):
            if (kwargs.get("out") is not None or kwargs.get("pin_memory") or kwargs.get("requires_grad")
                    or kwargs.get("layout", torch.strided) != torch.strided or kwargs.get("names") is not None):
                return orig(*args, **kwargs)
            dev = kwargs.get("device")
            if dev is None:
                dev = args[0].device if like else torch.get_default_device()
            dev = torch.device(dev)
            if dev.type != self.device_type:
                return orig(*args, **kwargs)
            meta_kw = dict(kwargs, device="meta")
            if like:
                t = args[0]
                src = torch.empty_strided(t.shape, t.stride(), dtype=t.dtype, device="meta")
                meta = orig(src, *args[1:], **meta_kw)
            else:
                meta = orig(*args, **meta_kw)
            return self._alloc(meta, dev, zero)
        alloc.__wrapped__ = orig
        return alloc

    # ------------------------------------------------------------------------------------------ arenas
    def _capturing(self):
        return self.device_type == "cuda" and torch.cuda.is_current_stream_capturing()

    def _alloc(self, meta, dev, zero):
        nbytes = _extent(meta.shape, meta.stride()) * meta.element_size()
        what = "%s (%s %s)" % (_caller(), str(meta.dtype).replace("torch.", ""), tuple(meta.shape))
        capturing = self._capturing()
        if not capturing and (len(self.queue) >= BATCH or self.queued_bytes >= BATCH_BYTES):
            self._drain()
        arena = self._orig["empty"](2 * GUARD + ALIGN + nbytes, dtype=torch.uint8, device=dev)
        start = GUARD + (-(arena.data_ptr() + GUARD)) % ALIGN
        arena.fill_(GUARD_BYTE)
        arena[start:start + nbytes].fill_(0 if zero else POISON)
        view = _view(arena, start, meta)
        check_layout(view, meta)
        rec = _Arena(arena, start, nbytes, what, capturing)
        with self.lock:
            self.allocated += 1
            self.live[id(rec)] = rec
            rec.fin = weakref.finalize(view, self._died, rec)
        return view

    def _died(self, rec):
        with self.lock:
            if self.live.pop(id(rec), None) is None:
                return
            if rec.captured:
                self.held.append(rec)
            else:
                self.queue.append(rec)
                self.queued_bytes += rec.arena.numel()

    def _drain(self):
        with self.lock:
            batch, self.queue, self.queued_bytes = self.queue, [], 0
        self._check(batch)

    def _check(self, recs):
        """one synchronize, then every guard of `recs` in one device-to-host copy"""
        if not recs:
            return
        if self.device_type == "cuda":
            torch.cuda.synchronize()
        flags = torch.stack([(g0 != GUARD_BYTE).any() | (g1 != GUARD_BYTE).any() for g0, g1 in map(_Arena.guards, recs)])
        for r, bad in zip(recs, flags.cpu().tolist()):
            if bad:
                for side, off in guard_faults(*r.guards()):
                    self.faults.append("%s: guard byte %d %s its %d-byte buffer written"
                                       % (r.what, off, side, r.nbytes))
        with self.lock:
            self.checked += len(recs)
            self.guarded += sum(r.nbytes for r in recs)
