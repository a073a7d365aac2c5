"""Tensor-level wrappers over the C ABI (include/wmd.h).

PyTorch is used for device memory and streams only: every function allocates
its outputs with torch, passes raw pointers to libwmd on torch's current stream
and returns tensors.  No arithmetic happens in torch here.
"""
import ctypes

import torch

from . import _lib
from ._lib import ACT_ELU, ACT_LRELU, ACT_NONE, ACT_SIGMOID, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO  # noqa: F401

_f32 = torch.float32
_i32 = torch.int32
_u8 = torch.uint8


def _dense(t, dtype=_f32):
    """Contiguous, 16-byte aligned tensor of `dtype` (copies only if needed)."""
    if t.dtype != dtype:
        t = t.to(dtype)
    if not t.is_contiguous():
        t = t.contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


class _Scratch:
    """Scratch buffers for the range / compaction / split-K kernels, one set per (device, stream).

    Two decoders on different streams of one device must not share the self-cleaning range counters or the split-K
    partial sums, so buffers are keyed by the stream they are used on.  A buffer that is outgrown is RETIRED, not
    freed: a captured CUDA graph (graphs.py) holds raw addresses of the buffers that were current at capture time and
    keeps replaying into them."""

    def __init__(self):
        self.bufs = {}
        self.retired = []

    @staticmethod
    def _key(kind, device, slot=0):
        return (kind, device.index if device.index is not None else torch.cuda.current_device(),
                torch.cuda.current_stream(device).cuda_stream, slot)

    def _get(self, key, device, nbytes, floor, zero):
        buf = self.bufs.get(key)
        if buf is None or buf.numel() < nbytes:
            if buf is not None:
                self.retired.append(buf)
            buf = (torch.zeros if zero else torch.empty)(max(nbytes, floor), dtype=_u8, device=device)
            self.bufs[key] = buf
        return buf

    def range(self, device, nbytes):
        return self._get(self._key("range", device), device, nbytes, 1 << 16, True)    # zeroed once; kernel keeps it zero

    def splitk(self, device, nbytes):
        """Split-K / stream-K workspace.  Its first 4 KiB hold the balanced mode's per-tile arrival counters, which must be
        zero before the first launch (the kernel leaves them zeroed): cleared once, when the buffer is created."""
        key = self._key("splitk", device)
        had = self.bufs.get(key)
        buf = self._get(key, device, (nbytes + 15) // 16 * 16, 4096, False)
        if buf is not had:
            buf[:4096].zero_()
        return buf.view(_f32)

    def compact(self, device, nbytes, slot=0):
        """slot: compactions that may run concurrently need different workspaces (side streams have their own key
        anyway; the slot also separates them when the caller serialises them on one stream)."""
        return self._get(self._key("compact", device, slot), device, nbytes, 1 << 16, False)


_scratch = _Scratch()


_SINGLE = []


def _single_gpu():
    if not _SINGLE:
        _SINGLE.append(torch.cuda.device_count() <= 1)
    return _SINGLE[0]


def _on_device(fn):
    """Run a wrapper with its tensors' device current.

    libwmd launches on the CUDA *current* device (it caches per-device attributes by cudaGetDevice()) and on the
    stream handed in, so both must belong to the device that owns the buffers.  The first CUDA tensor among the
    arguments decides; a decoder living on cuda:1 therefore works while cuda:0 is the process-wide current device."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        if _single_gpu():                      # one visible device: it is always the current one
            return fn(*args, **kwargs)
        dev = None
        for a in args:
            if torch.is_tensor(a) and a.is_cuda:
                dev = a.device
                break
        if dev is None:
            for a in kwargs.values():
                if torch.is_tensor(a) and a.is_cuda:
                    dev = a.device
                    break
            if dev is None and isinstance(kwargs.get("device"), torch.device) and kwargs["device"].type == "cuda":
                dev = kwargs["device"]
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)

    return wrapper


class Profiler:
    """Optional per-launch CUDA-event timing (bench.py's roofline pass).  Disabled unless installed."""

    def __init__(self):
        self.records = []          # (name, start_event, end_event, info dict)

    def results(self):
        """[(name, ms, info)] - call after a device synchronize."""
        return [(n, s.elapsed_time(e), i) for n, s, e, i in self.records]


_profiler = None


def set_profiler(p):
    global _profiler
    _profiler = p


class _prof:
    """with _prof(name, info_fn): <one C-ABI call>  - brackets the call with events on the current stream."""
    __slots__ = ("name", "info", "start")

    def __init__(self, name, info=None):
        self.name, self.info, self.start = name, info, None

    def __enter__(self):
        if _profiler is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record()
        return self

    def __exit__(self, *exc):
        if self.start is not None:
            end = torch.cuda.Event(enable_timing=True)
            end.record()
            info = self.info() if self.info else {}
            info["_stream"] = torch.cuda.current_stream().cuda_stream      # for scripts/step_timeline.py
            _profiler.records.append((self.name, self.start, end, info))
        return False


# --------------------------------------------------------------------------- Haar
def _epilogue_args(epilogue, like):
    """(mode, a, b, lo, hi, out0, out1, names) of a consumer epilogue spec; see head_idwt."""
    if epilogue is None:
        return _lib.EPI_NONE, 0.0, 0.0, 0.0, 0.0, None, None, ()
    if epilogue[0] == "disp_to_depth":
        min_depth, max_depth = float(epilogue[1]), float(epilogue[2])
        min_disp, max_disp = 1 / max_depth, 1 / min_depth                # Python doubles, as in the reference
        return (_lib.EPI_DISP_TO_DEPTH, min_disp, max_disp - min_disp, 0.0, 0.0, torch.empty_like(like), torch.empty_like(like),
                ("scaled_disp", "depth"))
    if epilogue[0] == "div_clamp":
        lo, hi = epilogue[2], epilogue[3]
        return (_lib.EPI_DIV_CLAMP, float(epilogue[1]), 0.0 if lo is None else 1.0, 0.0 if lo is None else float(lo),
                0.0 if lo is None else float(hi), torch.empty_like(like), None, ("depth",))
    raise _lib.WmdError("unknown consumer epilogue %r" % (epilogue,))


@_on_device
def idwt_haar(ll, hf, disp_scale=None, clamp01=False, epilogue=None):
    """ll (N,C,H,W), hf (N,C,3,H,W) -> out (N,C,2H,2W) [, disp = clamp?(out*disp_scale)] [, epilogue planes].

    epilogue (consumer of the last level, see head_idwt): returns the extra plane(s) after out / disp."""
    lib = _lib.load()
    ll, hf = _dense(ll), _dense(hf)
    n, c, h, w = ll.shape
    if tuple(hf.shape) != (n, c, 3, h, w):
        raise _lib.WmdError("idwt_haar: hf shape %s does not match ll %s" % (tuple(hf.shape), tuple(ll.shape)))
    out = torch.empty((n, c, 2 * h, 2 * w), dtype=_f32, device=ll.device)
    disp = torch.empty_like(out) if disp_scale is not None else None
    mode, ea, eb, elo, ehi, e0, e1, _ = _epilogue_args(epilogue, out)
    extra = tuple(t for t in (e0, e1) if t is not None)
    ret = (out,) + ((disp,) if disp_scale is not None else ()) + extra
    if out.numel() == 0:
        return ret if len(ret) > 1 else out
    with _prof('idwt_haar', lambda: dict(n=n, c=c, h=h, w=w, disp=disp is not None)):
        if mode == _lib.EPI_NONE:
            rc = lib.wmd_idwt_haar_f32(_lib.ptr(ll), _lib.ptr(hf), _lib.ptr(out), _lib.ptr(disp),
                                       float(disp_scale if disp_scale is not None else 1.0), int(bool(clamp01)),
                                       n, c, h, w, _lib.stream_ptr())
        else:
            rc = lib.wmd_idwt_haar_epi_f32(_lib.ptr(ll), _lib.ptr(hf), _lib.ptr(out), _lib.ptr(disp),
                                           float(disp_scale if disp_scale is not None else 1.0), int(bool(clamp01)),
                                           mode, ea, eb, elo, ehi, _lib.ptr(e0), _lib.ptr(e1), n, c, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_idwt_haar_f32")
    return ret if len(ret) > 1 else out


@_on_device
def idwt_bilinear(ll, hf, size, disp_scale=1.0, clamp01=False, align_corners=False):
    """Fused IDWT -> disp = [clamp](out*disp_scale) -> bilinear resize to `size` (F.interpolate semantics)."""
    lib = _lib.load()
    ll, hf = _dense(ll), _dense(hf)
    n, c, h, w = ll.shape
    full = torch.empty((n, c, int(size[0]), int(size[1])), dtype=_f32, device=ll.device)
    if full.numel() == 0:
        return full
    with _prof('idwt_bilinear', lambda: dict(n=n, c=c, h=h, w=w, fh=int(size[0]), fw=int(size[1]))):
        rc = lib.wmd_idwt_bilinear_f32(_lib.ptr(ll), _lib.ptr(hf), _lib.ptr(full), float(disp_scale), int(bool(clamp01)),
                                       int(size[0]), int(size[1]), int(bool(align_corners)), n, c, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_idwt_bilinear_f32")
    return full


@_on_device
def dwt_haar(x):
    """x (N,C,H,W) even H,W -> ll (N,C,H/2,W/2), hf (N,C,3,H/2,W/2)."""
    lib = _lib.load()
    x = _dense(x)
    n, c, h, w = x.shape
    ll = torch.empty((n, c, h // 2, w // 2), dtype=_f32, device=x.device)
    hf = torch.empty((n, c, 3, h // 2, w // 2), dtype=_f32, device=x.device)
    if x.numel() == 0:
        return ll, hf
    with _prof('dwt_haar', lambda: dict(n=n, c=c, h=h, w=w)):
        rc = lib.wmd_dwt_haar_f32(_lib.ptr(x), _lib.ptr(ll), _lib.ptr(hf), n, c, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_dwt_haar_f32")
    return ll, hf


# --------------------------------------------------------------------------- masks
@_on_device
def range_thresh(x, ratio, return_minmax=False):
    """Per-sample (max - min) * ratio over everything but dim 0 -> (N,) fp32 on device."""
    lib = _lib.load()
    x = _dense(x)
    n = x.shape[0]
    per = x.numel() // max(n, 1)
    thresh = torch.empty((n,), dtype=_f32, device=x.device)
    mm = torch.empty((n, 2), dtype=_f32, device=x.device) if return_minmax else None
    nbytes = lib.wmd_range_ws_bytes(n, per)
    ws = _scratch.range(x.device, nbytes)
    with _prof('range_thresh', lambda: dict(n=n, per=per)):
        rc = lib.wmd_range_thresh_f32(_lib.ptr(x), n, per, float(ratio), _lib.ptr(thresh), _lib.ptr(mm),
                                      _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    _lib.check(rc, "wmd_range_thresh_f32")
    return (thresh, mm) if return_minmax else thresh


@_on_device
def level_masks(yh, thresh, n=None, h=None, w=None, device=None, want=("S0", "S1", "S2", "S3", "S4", "S5")):
    """yh (N,3,H,W) or (N,1,3,H,W), thresh (N,) or None (all ones; then pass n,h,w,device).

    Returns dict of uint8 (N,1,H,W) [S0-S2] / (N,1,2H,2W) [S3-S5] tensors."""
    lib = _lib.load()
    if thresh is not None:
        yh = _dense(yh)
        n, h, w = yh.shape[0], yh.shape[-2], yh.shape[-1]
        device = yh.device
        thresh = _dense(thresh)
    out = {}
    ptrs = []
    for k in ("S0", "S1", "S2", "S3", "S4", "S5"):
        if k in want:
            hi = k in ("S3", "S4", "S5")
            out[k] = torch.empty((n, 1, 2 * h if hi else h, 2 * w if hi else w), dtype=_u8, device=device)
            ptrs.append(_lib.ptr(out[k]))
        else:
            ptrs.append(None)
    with _prof('level_masks', lambda: dict(n=n, h=h, w=w, thresh=thresh is not None)):
        rc = lib.wmd_level_masks(_lib.ptr(yh) if thresh is not None else None, _lib.ptr(thresh), *ptrs, n, h, w,
                                 _lib.stream_ptr())
    _lib.check(rc, "wmd_level_masks")
    return out


@_on_device
def compact(mask, want_idxmap=True, want_pixels=True, stream=None, ws_slot=0):
    """mask uint8 (N,1,H,W) or (N,H,W) -> idxmap int32 (N,H,W) | None, pixels int32 (N*H*W,) | None, offsets int32 (N+1,).

    stream: optional side stream to run on (it first waits for the current stream, which produced `mask`); then returns
    ((idxmap, pixels, offsets), event) and the consumer stream must wait for the event.  Outputs are allocated on the
    current stream.  ws_slot: workspace to use - concurrent compactions must not share one."""
    lib = _lib.load()
    mask = _dense(mask, _u8)
    n, h, w = mask.shape[0], mask.shape[-2], mask.shape[-1]
    dev = mask.device
    idxmap = torch.empty((n, h, w), dtype=_i32, device=dev) if want_idxmap else None
    pixels = torch.empty((n * h * w,), dtype=_i32, device=dev) if want_pixels else None
    offsets = torch.empty((n + 1,), dtype=_i32, device=dev)
    nbytes = lib.wmd_compact_ws_bytes(n, h, w)
    ws = _scratch.compact(dev, nbytes, ws_slot)

    def launch():
        with _prof('compact_mask', lambda: dict(n=n, h=h, w=w, idxmap=idxmap is not None, pixels=pixels is not None, offsets=offsets)):
            rc = lib.wmd_compact_mask(_lib.ptr(mask), _lib.ptr(idxmap), _lib.ptr(pixels), _lib.ptr(offsets), n, h, w,
                                      _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "wmd_compact_mask")

    if stream is None:
        launch()
        return idxmap, pixels, offsets
    stream.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(stream):
        launch()
        done = torch.cuda.Event()
        done.record(stream)
    return (idxmap, pixels, offsets), done


@_on_device
def gate_map(gate, idxmap=None):
    """int32 map: gate ? (idxmap or linear index) : -1, shaped like gate without the channel dim."""
    lib = _lib.load()
    gate = _dense(gate, _u8)
    out = torch.empty((gate.shape[0], gate.shape[-2], gate.shape[-1]), dtype=_i32, device=gate.device)
    with _prof('gate_map', lambda: dict(count=gate.numel())):
        rc = lib.wmd_gate_map(_lib.ptr(gate), _lib.ptr(idxmap), _lib.ptr(out), gate.numel(), _lib.stream_ptr())
    _lib.check(rc, "wmd_gate_map")
    return out


# --------------------------------------------------------------------------- layout
def pad4(c):
    return (int(c) + 3) // 4 * 4


def rows_view(x):
    """The zero-copy pixel-major rows of a channels_last feature map ((N*H*W, C) view), or None if x is not laid out so."""
    if not x.is_cuda or x.dtype != _f32 or x.dim() != 4:
        return None
    n, c, h, w = x.shape
    if c % 4 == 0 and x.permute(0, 2, 3, 1).is_contiguous() and x.data_ptr() % 16 == 0:
        return x.permute(0, 2, 3, 1).reshape(n * h * w, c)
    return None


@_on_device
def amax_rows(x, out):
    """out (1-element device tensor, pre-zeroed or holding a lower bound) = max(out, max |x|): for sources no libwmd kernel
    produced (channels_last maps used in place)."""
    lib = _lib.load()
    with _prof('amax', lambda: dict(count=x.numel())):
        rc = lib.wmd_amax_f32(_lib.ptr(x, _f32), x.numel(), _lib.ptr(out, _f32), _lib.stream_ptr())
    _lib.check(rc, "wmd_amax_f32")
    return out


@_on_device
def nchw_to_rows(x, ld=None, stream=None, gate=None, amax=None):
    """(N,C,H,W) -> rows (N*H*W, ld) pixel-major.  Zero-copy when x is channels_last and C % 4 == 0.

    gate: optional uint8 (N,1,H,W) / (N,H,W) mask of the pixels whose rows will be read later: only those rows are
    produced (wmd_nchw_to_rows_gated_f32); the other rows of the result are uninitialised memory.
    With a gate, x may also be a PINNED HOST tensor: the kernel then reads the marked parts of the map straight out of
    host memory (zero-copy over PCIe) - the host->device transfer of a skip map shrinks with the mask density.
    stream: optional side stream to run the transpose on (it first waits for the current stream, so `x` / `gate` may
    have been produced there).  Then returns (rows, event): the consumer stream must wait for `event` (None when no
    kernel was needed).  The output is allocated on the current stream, whose later work is what reads it."""
    lib = _lib.load()
    n, c, h, w = x.shape
    ld = pad4(c) if ld is None else ld
    on_host = not x.is_cuda
    if on_host:
        if gate is None:
            raise _lib.WmdError("nchw_to_rows: a host feature map needs a gate (only the gated move reads host memory)")
        if x.dtype != _f32 or not x.is_contiguous() or x.data_ptr() % 16:
            raise _lib.WmdError("nchw_to_rows: host feature maps must be contiguous fp32 NCHW, 16-byte aligned")
        dev = gate.device
    else:
        dev = x.device
        if x.dtype == _f32 and ld == c and x.permute(0, 2, 3, 1).is_contiguous() and x.data_ptr() % 16 == 0:
            rows = x.permute(0, 2, 3, 1).reshape(n * h * w, c)
            if amax is not None:
                amax_rows(rows, amax)
            return (rows, None) if stream is not None else rows
        x = _dense(x)
    if gate is not None:
        gate = _dense(gate, _u8)
        if gate.numel() != n * h * w:
            raise _lib.WmdError("nchw_to_rows: gate of %d pixels for a %dx%dx%d map" % (gate.numel(), n, h, w))
    rows = torch.empty((n * h * w, ld), dtype=_f32, device=dev)

    def launch():
        marked = _pm_count(gate)
        with _prof('nchw_to_rows', lambda: dict(n=n, c=c, hw=h * w, ld=ld, marked=marked, host=on_host)):
            if gate is None and amax is not None:
                rc = lib.wmd_nchw_to_rows_amax_f32(_lib.ptr(x), _lib.ptr(rows), n, c, h * w, ld, _lib.ptr(amax, _f32), _lib.stream_ptr())
            elif gate is None:
                rc = lib.wmd_nchw_to_rows_f32(_lib.ptr(x), _lib.ptr(rows), n, c, h * w, ld, _lib.stream_ptr())
            elif amax is not None:
                rc = lib.wmd_nchw_to_rows_gated_amax_f32(_lib.host_ptr(x, _f32), _lib.ptr(rows), _lib.ptr(gate), n, c, h * w, ld,
                                                         _lib.ptr(amax, _f32), _lib.stream_ptr())
            else:
                rc = lib.wmd_nchw_to_rows_gated_f32(_lib.host_ptr(x, _f32), _lib.ptr(rows), _lib.ptr(gate), n, c, h * w, ld,
                                                    _lib.stream_ptr())
        _lib.check(rc, "wmd_nchw_to_rows_f32")

    if stream is None:
        launch()
        return rows
    stream.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(stream):
        launch()
        done = torch.cuda.Event()
        done.record(stream)
    return rows, done


def _pm_count(gate):
    """Marked-pixel count of a gate for the profiler's byte accounting (None when not profiling or not gated)."""
    if gate is None or _profiler is None:
        return None
    return gate.sum()


@_on_device
def rows_to_nchw(rows, n, c, h, w):
    lib = _lib.load()
    rows = _dense(rows)
    out = torch.empty((n, c, h, w), dtype=_f32, device=rows.device)
    with _prof('rows_to_nchw', lambda: dict(n=n, c=c, hw=h * w)):
        rc = lib.wmd_rows_to_nchw_f32(_lib.ptr(rows), _lib.ptr(out), n, c, h * w, rows.shape[1], _lib.stream_ptr())
    _lib.check(rc, "wmd_rows_to_nchw_f32")
    return out


@_on_device
def gather_rows(x_nchw, pixels, count, max_rows=None, ld=None):
    """rows[m] = x[n, :, y, x] at the listed pixels (pixels/count None = every pixel)."""
    lib = _lib.load()
    x = _dense(x_nchw)
    n, c, h, w = x.shape
    ld = pad4(c) if ld is None else ld
    max_rows = n * h * w if max_rows is None else max_rows
    rows = torch.zeros((max(max_rows, 1), ld), dtype=_f32, device=x.device)
    rc = lib.wmd_gather_rows_nchw_f32(_lib.ptr(x), _lib.ptr(rows), ld, c, _lib.ptr(pixels), _lib.ptr(count),
                                      max_rows, n, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_gather_rows_nchw_f32")
    return rows


@_on_device
def gather_rows_list(x, pixels, count, ld=None, stream=None, amax=None):
    """Compact rows of the listed pixels of an NCHW map: rows[m] = x[n, :, y, x] for pixels[m] (wmd_gather_rows_list_f32).

    x: (N,C,H,W) CUDA tensor or PINNED HOST tensor (read in place over PCIe: only the listed pixels cross the bus).
    pixels / count: list + device count from `compact`.  Returns rows (N*H*W capacity, ld); rows past *count are
    uninitialised.  stream: as in nchw_to_rows (side stream; returns (rows, event))."""
    lib = _lib.load()
    n, c, h, w = x.shape
    ld = pad4(c) if ld is None else ld
    on_host = not x.is_cuda
    dev = pixels.device
    if on_host:
        if x.dtype != _f32 or not x.is_contiguous() or x.data_ptr() % 16:
            raise _lib.WmdError("gather_rows_list: host feature maps must be contiguous fp32 NCHW, 16-byte aligned")
    else:
        x = _dense(x)
    rows = torch.empty((max(n * h * w, 1), ld), dtype=_f32, device=dev)

    def launch():
        with _prof('gather_rows_list', lambda: dict(c=c, ld=ld, count=count, max_rows=n * h * w, host=on_host)):
            rc = lib.wmd_gather_rows_list_amax_f32(_lib.host_ptr(x, _f32), _lib.ptr(rows), ld, c, _lib.ptr(pixels, _i32),
                                                   _lib.ptr(count, _i32), n * h * w, n, h, w, _lib.ptr(amax, _f32),
                                                   _lib.stream_ptr())
        _lib.check(rc, "wmd_gather_rows_list_f32")

    if stream is None:
        launch()
        return rows
    stream.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(stream):
        launch()
        done = torch.cuda.Event()
        done.record(stream)
    return rows, done


@_on_device
def scatter_rows(rows, c, pixels, count, n, h, w, max_rows=None, out=None):
    """Dense (N,C,H,W), zero except at the listed pixels where it takes rows[m, :c]."""
    lib = _lib.load()
    rows = _dense(rows)
    if out is None:
        out = torch.zeros((n, c, h, w), dtype=_f32, device=rows.device)
    max_rows = min(rows.shape[0], n * h * w) if max_rows is None else max_rows
    rc = lib.wmd_scatter_rows_nchw_f32(_lib.ptr(rows), rows.shape[1], c, _lib.ptr(pixels), _lib.ptr(count),
                                       max_rows, _lib.ptr(out), n, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_scatter_rows_nchw_f32")
    return out


def tc_splits(max_rows, cout, nchunks, device, ldy=None):
    """Scheduling mode of the tensor-core (wgmma) engine for one launch: 1 = whole tiles, 0 = balanced (data-parallel + stream-K).

    At most one CTA per SM runs equal (128-row x N-channel) tiles, so with few tiles per SM the last round is mostly idle
    (320 tiles on 132 SMs = 81 %; the sparse levels' tile count is only known on the device) and a layer with fewer
    tiles than SMs leaves SMs dark.  Balanced mode runs the full rounds as whole tiles and deals the (tile, chunk)
    units of the remainder tiles out evenly on the device; only those tiles go through the fixed-order reduce pass
    (workspace: CTAs x 8 x 128 x 128 floats).  The extra pass only pays for long reductions, so it is used from
    TC_BALANCE_MIN_CHUNKS chunks on (per-layer times: scripts/conv_layers_env.py)."""
    return 0 if nchunks >= TC_BALANCE_MIN_CHUNKS else 1


TC_BALANCE_MIN_CHUNKS = int(__import__("os").environ.get("WMD_TC_BALANCE_MIN_CHUNKS", "80"))


class PackedW:
    """A conv weight packed for one of the two gather-GEMM engines ('simt' fp32 FMA, 'tc' wgmma 3xTF32)."""
    __slots__ = ("data", "kind", "taps", "c0", "c1", "cout", "data16")

    def __init__(self, data, kind, taps, c0, c1, cout, data16=None):
        self.data, self.kind, self.taps, self.c0, self.c1, self.cout = data, kind, taps, c0, c1, cout
        self.data16 = data16          # 'tc' only: fp16-pair image for precision f16x3 (wmd_pack_conv_weight_tc16_f32)


TC_MIN_K = 128        # shallower reductions (1x1 heads of the fine levels) do not amortise the tile prologue
TC_MIN_COUT = 32      # tensor-core tiles are 128 x {128, 64, 32}; below that the FMA tiles / head kernel take over


def default_conv_precision():
    """Operand form of the tensor-core engine: env WMD_CONV_PRECISION = tf32x3 (default) | f16x3.

    Both are fp32-faithful error-compensated splits with fp32 accumulation (22 mantissa bits per operand, three MMAs per
    product).  f16x3 feeds fp16 pairs of power-of-two scaled operands - half the MMA instructions - and needs the max |x|
    of each source (tracked on the device by the producers, see conv_rows amax*); launches that lack it use tf32x3.
    Opt-in: it costs the max tracking in every producer; its speed on H100 has not been measured."""
    import os
    return os.environ.get("WMD_CONV_PRECISION", "tf32x3")


def default_conv_kind():
    """Engine used when a caller does not ask for one: env WMD_CONV_IMPL = auto | simt | tc.

    auto (default): wgmma 3xTF32 for cout >= 32 (every upconv / 1x1 head stage of the decoders), fp32 FMA
    tiles below."""
    import os
    return os.environ.get("WMD_CONV_IMPL", "auto")


@_on_device
def pack_weight(weight, c1=0, kind=None, precision=None):
    """(Cout,Cin,k,k) conv weight -> PackedW.  c1 = trailing input channels that come from gather source 1.
    precision ('tc' only): 'f16x3' also builds the fp16-pair image (default: default_conv_precision()).

    simt: [k*k][Cin][ldw] rows (ldw = pad4(Cout)).  tc: per (n-tile, 32-channel chunk) swizzled smem images
    [tf32 hi | tf32 lo] (chunk boundaries follow the two gather sources, hence c1 matters)."""
    lib = _lib.load()
    kind = kind or default_conv_kind()
    wt = _dense(weight.detach())
    cout, cin = wt.shape[0], wt.shape[1]
    taps = wt.shape[2] * wt.shape[3]
    c0 = cin - c1
    if kind == "auto":
        kind = "tc" if (cout >= TC_MIN_COUT and taps * cin >= TC_MIN_K) else "simt"
    if kind == "tc":
        nfl = lib.wmd_conv_tc_weight_floats(cout, c0, c1, taps)
        packed = torch.empty((nfl,), dtype=_f32, device=wt.device)
        rc = lib.wmd_pack_conv_weight_tc_f32(_lib.ptr(wt), _lib.ptr(packed), cout, c0, c1, taps, _lib.stream_ptr())
        _lib.check(rc, "wmd_pack_conv_weight_tc_f32")
        packed16 = None
        if (precision or default_conv_precision()) == "f16x3":
            packed16 = torch.empty((lib.wmd_conv_tc16_weight_bytes(cout, c0, c1, taps),), dtype=_u8, device=wt.device)
            rc = lib.wmd_pack_conv_weight_tc16_f32(_lib.ptr(wt), _lib.ptr(packed16), cout, c0, c1, taps, _lib.stream_ptr())
            _lib.check(rc, "wmd_pack_conv_weight_tc16_f32")
        return PackedW(packed, "tc", taps, c0, c1, cout, packed16)
    ldw = pad4(cout)
    packed = torch.empty((taps * cin, ldw), dtype=_f32, device=wt.device)
    rc = lib.wmd_pack_conv_weight_f32(_lib.ptr(wt), _lib.ptr(packed), cout, cin, taps, ldw, _lib.stream_ptr())
    _lib.check(rc, "wmd_pack_conv_weight_f32")
    return PackedW(packed, "simt", taps, c0, c1, cout)


# --------------------------------------------------------------------------- conv
@_on_device
def conv_rows(x0, c0, wpacked, bias, cout, n, h, w, taps=9, pad=PAD_REFLECT, act=ACT_NONE, act_param=0.0,
              map0=None, shift0=0, x1=None, c1=0, gate=None, pixels=None, count=None, max_rows=None, out=None,
              m_in0=None, m_in1=None, splits=None, map1=None, amax0=None, amax1=None, amax_out=None):
    """Gather-GEMM convolution on pixel-major rows; see wmd_conv_rows_f32 in include/wmd.h.

    m_in0 / m_in1: optional active-row counts of the two sources (ints or 1-element device tensors), used only
    by the profiler's algorithmic-byte accounting.

    x0: rows (R0, ld0); x1: optional dense rows (N*H*W, ld1); wpacked: PackedW from pack_weight(weight, c1).
    Returns y rows (max_rows, pad4(cout)).
    """
    lib = _lib.load()
    dev = x0.device
    total = n * h * w
    max_rows = total if max_rows is None else int(max_rows)
    ldy = pad4(cout)
    if out is None:
        out = torch.empty((max(max_rows, 1), ldy), dtype=_f32, device=dev)
    assert isinstance(wpacked, PackedW) and (wpacked.taps, wpacked.c0, wpacked.c1, wpacked.cout) == (taps, c0, c1, cout), \
        ((wpacked.taps, wpacked.c0, wpacked.c1, wpacked.cout), (taps, c0, c1, cout))
    d = _lib.ConvDesc()
    d.N, d.H, d.W = n, h, w
    d.x0, d.c0, d.ld0 = _lib.ptr(x0, _f32), c0, x0.shape[1]
    d.map0, d.shift0 = _lib.ptr(map0, _i32), shift0
    d.x1, d.c1, d.ld1 = (_lib.ptr(x1, _f32), c1, x1.shape[1]) if x1 is not None else (None, 0, 0)
    d.gate = _lib.ptr(gate, _u8)
    d.map1 = _lib.ptr(map1, _i32) if x1 is not None else None
    d.w, d.bias = _lib.ptr(wpacked.data, _f32), _lib.ptr(bias, _f32)
    d.cout, d.ldw, d.taps, d.pad_mode = cout, (wpacked.data.shape[1] if wpacked.kind == "simt" else 0), taps, pad
    d.pixels, d.count, d.max_rows = _lib.ptr(pixels, _i32), _lib.ptr(count, _i32), max_rows
    d.y, d.ldy = _lib.ptr(out, _f32), out.shape[1]
    d.act, d.act_param = act, float(act_param)
    d.rows0 = int(x0.shape[0])
    # fp16-pair operands when the weights have that image and every source's max |x| is known (1-element device tensors);
    # amax_out (optional): device scalar raised to max |y|, for the consumers of this layer
    # (the split-K form with an external reduction keeps the tf32 operands: its reduction kernel adds unscaled slabs)
    if wpacked.kind == "tc" and splits is None:
        splits = tc_splits(max_rows, cout, taps * (-(-c0 // 32) + -(-c1 // 32)), dev, out.shape[1])
    use16 = (wpacked.kind == "tc" and wpacked.data16 is not None and amax0 is not None and
             (x1 is None or amax1 is not None) and splits in (0, 1))
    d.precision = _lib.PREC_F16X3 if use16 else _lib.PREC_TF32X3
    d.amax0, d.amax1 = (_lib.ptr(amax0, _f32), _lib.ptr(amax1, _f32) if x1 is not None else None) if use16 else (None, None)
    d.amax_out = _lib.ptr(amax_out, _f32)
    if use16:
        d.w = _lib.ptr(wpacked.data16, _u8)
    info = lambda: dict(n=n, h=h, w=w, taps=taps, c0=c0, c1=c1, cout=cout, shift0=shift0, count=count,   # noqa: E731
                        max_rows=max_rows, m_in0=m_in0, m_in1=m_in1, kind=wpacked.kind, f16=use16)
    if wpacked.kind == "tc":
        ws = None
        if splits != 1:
            ws = _scratch.splitk(dev, lib.wmd_conv_tc_splitk_ws_bytes(max_rows, out.shape[1], splits))
        with _prof('conv_rows_tc', info):
            rc = lib.wmd_conv_rows_tc_splitk_f32(ctypes.byref(d), splits, _lib.ptr(ws), ws.numel() * 4 if ws is not None else 0,
                                                 _lib.stream_ptr())
    else:
        with _prof('conv_rows', info):
            rc = lib.wmd_conv_rows_f32(ctypes.byref(d), _lib.stream_ptr())
    _lib.check(rc, "wmd_conv_rows_%sf32" % ("tc_" if wpacked.kind == "tc" else ""))
    return out


def head_mlp_supported(c, n1):
    return bool(_lib.load().wmd_head_mlp_supported(int(c), int(n1)))


@_on_device
def pack_head_mlp(w1, b1, wz):
    """(n1, c, 1, 1) 1x1 weight, (n1,) bias, (nz, n1, 1, 1) tap-product weight -> packed image for head_mlp."""
    lib = _lib.load()
    w1, wz = _dense(w1.detach()), _dense(wz.detach())
    n1, c, nz = int(w1.shape[0]), int(w1.shape[1]), int(wz.shape[0])
    if int(wz.shape[1]) != n1:
        raise _lib.WmdError("pack_head_mlp: wz expects %d inputs, w1 produces %d" % (wz.shape[1], n1))
    nfl = lib.wmd_head_mlp_weight_floats(c, n1)
    if nfl == 0:
        raise _lib.WmdError("head_mlp: unsupported shape c=%d n1=%d" % (c, n1))
    packed = torch.empty((nfl,), dtype=_f32, device=w1.device)
    rc = lib.wmd_pack_head_mlp_f32(_lib.ptr(w1), _lib.ptr(wz), _lib.ptr(_dense(b1.detach()) if b1 is not None else None),
                                   c, n1, nz, _lib.ptr(packed), _lib.stream_ptr())
    _lib.check(rc, "wmd_pack_head_mlp_f32")
    return packed


@_on_device
def head_mlp(x, c, packed, n1, slope=0.1, count=None, max_rows=None, nz=54):
    """z (max_rows, 56) = Wz . lrelu(W1 . x + b1) on pixel-major rows x (R, ld >= c); see wmd_head_mlp_f32."""
    lib = _lib.load()
    max_rows = x.shape[0] if max_rows is None else int(max_rows)
    z = torch.empty((max(max_rows, 1), 56), dtype=_f32, device=x.device)
    with _prof('head_mlp', lambda: dict(c=c, n1=n1, nz=nz, count=count, max_rows=max_rows)):
        rc = lib.wmd_head_mlp_f32(_lib.ptr(x, _f32), x.shape[1], c, _lib.ptr(packed, _f32), n1, float(slope),
                                  _lib.ptr(count, _i32), max_rows, _lib.ptr(z), 56, _lib.stream_ptr())
    _lib.check(rc, "wmd_head_mlp_f32")
    return z


@_on_device
def head_conv3x3(t, c, off_a, wa, ba, n, h, w, cout, scale=1.0, act=ACT_NONE, pad=PAD_REFLECT, off_b=-1, wb=None,
                 bb=None, idxmap=None, pixels=None, count=None, max_rows=None, out=None):
    """3x3 stage of the coefficient heads -> dense (N,cout,H,W); see wmd_head_conv3x3_f32.

    wa/wb: packed (9*c, cout) exactly (no padding: use pack_head_weight)."""
    lib = _lib.load()
    dev = t.device
    total = n * h * w
    max_rows = total if max_rows is None else int(max_rows)
    if out is None:
        out = (torch.zeros if pixels is not None else torch.empty)((n, cout, h, w), dtype=_f32, device=dev)
    d = _lib.HeadDesc()
    d.N, d.H, d.W = n, h, w
    d.t, d.ld, d.c, d.off_a, d.off_b = _lib.ptr(t, _f32), t.shape[1], c, off_a, off_b
    d.map = _lib.ptr(idxmap, _i32)
    d.wa, d.ba, d.wb, d.bb = _lib.ptr(wa, _f32), _lib.ptr(ba, _f32), _lib.ptr(wb, _f32), _lib.ptr(bb, _f32)
    d.cout, d.pad_mode, d.act, d.scale = cout, pad, act, float(scale)
    d.pixels, d.count, d.max_rows = _lib.ptr(pixels, _i32), _lib.ptr(count, _i32), max_rows
    d.out = _lib.ptr(out, _f32)
    with _prof('head_conv3x3', lambda: dict(n=n, h=h, w=w, c=c, cout=cout, dual=off_b >= 0, count=count, max_rows=max_rows)):
        rc = lib.wmd_head_conv3x3_f32(ctypes.byref(d), _lib.stream_ptr())
    _lib.check(rc, "wmd_head_conv3x3_f32")
    return out


@_on_device
def pack_head_weight(weight):
    """(cout<=4, c, 3, 3) -> (9*c, cout) contiguous, the layout wmd_head_conv3x3_f32 stages in shared memory."""
    lib = _lib.load()
    wt = _dense(weight.detach())
    cout, cin = wt.shape[0], wt.shape[1]
    packed = torch.empty((9 * cin, cout), dtype=_f32, device=wt.device)
    rc = lib.wmd_pack_conv_weight_f32(_lib.ptr(wt), _lib.ptr(packed), cout, cin, 9, cout, _lib.stream_ptr())
    _lib.check(rc, "wmd_pack_conv_weight_f32")
    return packed


def head_tap_weight(w_list, offsets, ctot):
    """1x1-conv weight (9*G, ctot, 1, 1) of the factored 3x3 head stage: row tap*G + g = head-group g's tap-th filter.

    w_list: 3x3 weights [(co_k, c_k, 3, 3)] of the heads; offsets: channel offset of each head's input inside the
    ctot-wide T row.  Groups are the heads' output channels concatenated in order (G = sum co_k)."""
    g_total = sum(int(w.shape[0]) for w in w_list)
    out = torch.zeros((9, g_total, ctot), dtype=_f32, device=w_list[0].device)
    g0 = 0
    for w, off in zip(w_list, offsets):
        co, c = int(w.shape[0]), int(w.shape[1])
        out[:, g0:g0 + co, off:off + c] = w.detach().permute(2, 3, 0, 1).reshape(9, co, c)
        g0 += co
    return out.reshape(9 * g_total, ctot, 1, 1)


@_on_device
def head_gather(z, groups, bias, n, h, w, cout, scale=1.0, act=ACT_NONE, dual=False, pad=PAD_REFLECT, idxmap=None,
                pixels=None, count=None, max_rows=None, out=None, col0=0):
    """Sum the nine per-tap products of z (rows x >= 9*groups) around every output pixel -> dense (N,cout,H,W).

    col0: first column of z that belongs to this head (its nine [tap][group] blocks start there)."""
    lib = _lib.load()
    if col0 < 0 or col0 + 9 * groups > z.shape[1]:
        raise _lib.WmdError("head_gather: columns %d..%d do not fit rows of %d" % (col0, col0 + 9 * groups, z.shape[1]))
    total = n * h * w
    max_rows = total if max_rows is None else int(max_rows)
    if out is None:
        out = (torch.zeros if pixels is not None else torch.empty)((n, cout, h, w), dtype=_f32, device=z.device)
    with _prof('head_gather', lambda: dict(n=n, h=h, w=w, groups=groups, cout=cout, count=count, max_rows=max_rows)):
        rc = lib.wmd_head_gather_f32(_lib.ptr(z, _f32) + 4 * col0, z.shape[1], groups, _lib.ptr(idxmap, _i32), _lib.ptr(bias, _f32),
                                     float(scale), act, int(bool(dual)), pad, _lib.ptr(pixels, _i32), _lib.ptr(count, _i32),
                                     max_rows, _lib.ptr(out, _f32), cout, n, h, w, _lib.stream_ptr())
    _lib.check(rc, "wmd_head_gather_f32")
    return out


@_on_device
def head_idwt(z, bias, yl, scale, disp_scale, idxmap=None, mask=None, pad=PAD_REFLECT, clamp01=True, col0=0,
              thresh_ratio=None, epilogue=None):
    """Fused tail of a decoder level (wmd_head_idwt_f32): factored +/- head stage -> yh -> IDWT -> disp [-> consumer
    epilogue] [-> next level's per-sample threshold].

    z rows (>= col0 + 54 columns of tap products), yl (N,1,H,W).  Returns dict(yh (N,3,H,W), out (N,1,2H,2W), disp,
    thresh (N,) if thresh_ratio is not None, plus the epilogue's planes).
    epilogue: None | ("disp_to_depth", min_depth, max_depth) -> "scaled_disp", "depth" (KITTI/layers.py:16-25)
                   | ("div_clamp", div, lo, hi)  (lo/hi None = no clamp) -> "depth" (NYUv2/utils.py:219,229)."""
    lib = _lib.load()
    yl = _dense(yl)
    n, _, h, w = yl.shape
    dev = yl.device
    if col0 < 0 or col0 + 54 > z.shape[1] or col0 % 2:
        raise _lib.WmdError("head_idwt: columns %d..%d do not fit rows of %d" % (col0, col0 + 54, z.shape[1]))
    res = {"yh": torch.empty((n, 3, h, w), dtype=_f32, device=dev),
           "out": torch.empty((n, 1, 2 * h, 2 * w), dtype=_f32, device=dev),
           "disp": torch.empty((n, 1, 2 * h, 2 * w), dtype=_f32, device=dev)}
    d = _lib.HeadIdwtDesc()
    d.N, d.H, d.W = n, h, w
    d.z, d.ldz = _lib.ptr(z, _f32) + 4 * col0, z.shape[1]
    d.map, d.mask, d.bias = _lib.ptr(idxmap, _i32), _lib.ptr(mask, _u8), _lib.ptr(bias, _f32)
    d.scale, d.pad_mode = float(scale), pad
    d.ll, d.yh, d.out, d.disp = _lib.ptr(yl), _lib.ptr(res["yh"]), _lib.ptr(res["out"]), _lib.ptr(res["disp"])
    d.disp_scale, d.clamp01 = float(disp_scale), int(bool(clamp01))
    mode, ea, eb, elo, ehi, e0, e1, names = _epilogue_args(epilogue, res["out"])
    d.epi_mode, d.epi_a, d.epi_b, d.epi_lo, d.epi_hi = mode, ea, eb, elo, ehi
    d.epi_out0, d.epi_out1 = _lib.ptr(e0), _lib.ptr(e1)
    for name, t in zip(names, (e0, e1)):
        res[name] = t
    ws = None
    if thresh_ratio is not None:
        res["thresh"] = torch.empty((n,), dtype=_f32, device=dev)
        d.thresh, d.thresh_ratio = _lib.ptr(res["thresh"]), float(thresh_ratio)
        ws = _scratch.range(dev, lib.wmd_head_idwt_ws_bytes(n, h, w))
    if n == 0:
        return res
    with _prof('head_idwt', lambda: dict(n=n, h=h, w=w, mask=mask, epi=d.epi_mode, thresh=thresh_ratio is not None)):
        rc = lib.wmd_head_idwt_f32(ctypes.byref(d), _lib.ptr(ws), ws.numel() if ws is not None else 0, _lib.stream_ptr())
    _lib.check(rc, "wmd_head_idwt_f32")
    return res
