"""Launch-checking harness: every libwmd launch a workload makes, checked against the fp64 contract of its kernel.

`Harness(monkeypatch)` wraps the entry points of ENTRY_POINTS, (owner, attribute) pairs whose owner is a module or a
class: the public functions of wavelet_monodepth_b200.ops, the evaluation and loss entry points of nyu_loss, nyu_eval,
kitti_eval and kitti_loss, and the data pipelines' launches (kitti_hints.stereo_sgbm and _fuse, KittiInputs._run,
NyuInputs._run, kitti_gt.generate_depth_maps).  The decoders, train_native and wavelets call `ops.<name>` through the
module, calls inside a module (conv_dgrad -> conv_rows, nchw_to_rows -> amax_rows, _NyuLossFn -> _loss_fwd / _loss_bwd,
_KittiLossFn -> _kitti_fwd / _kitti_bwd, NyuDepthEvaluator.add -> _edges_frames, DepthHintGenerator -> stereo_sgbm /
_fuse) resolve through its globals, and methods through their class, so wrapping the owners' attributes catches every
call, nested ones included.

Each call runs the original function, synchronises (compactions and list gathers run on side streams), recomputes the
result from the call's actual inputs with the references of the kernel contract tests (conv_ref, head_ref, disp_tail_ref,
conv_grad_ref, oracle.haar, oracle.nyu_loss, oracle.nyu_eval, oracle.nyu_edges, oracle.kitti_eval, oracle.kitti_loss,
oracle.sgbm, oracle.depth_hints, oracle.kitti_inputs, oracle.nyu_inputs, oracle.kitti_gt, plain torch restatements of
the wmd.h comments: none of them uses ops or libwmd) and compares at that kernel's bar.  It also checks the
preconditions a launch's contract relies on: source maxima that cover what an fp16-pair launch reads, exact amax
outputs, index maps inside their sources, strictly increasing pixel lists, count <= max_rows, views of one size per
launch, 0 / 1 mirror flags and scan offsets that rise from 0 to the point count.  Pack calls record the
plain weights behind each packed object; a pack is right when every launch that uses it is right.  State a checker needs
from before the call (an evaluator's next frame and the rows the call writes) comes from the entry's `_before_` hook.

Completeness: around each outermost wrapped call the harness takes the `launch_count()` delta; at the end of a workload the
checked deltas must add up to the whole delta, and any libwmd symbol called outside a wrapped call is named.

Footprint: a workload runs under footprint.Footprint, so every CUDA buffer the package allocates with torch.empty / zeros
(outputs, workspaces, the checkers' own) sits between guards and an `empty` one starts out as NaN / -1 bytes; the test's
plain-vs-checked comparison then also asserts that no result depends on what was in memory.  ops._scratch is swapped for
a _Scratch without its size floors, so each range / compaction / backward / split-K workspace is exactly its size
query.  At the end every guard must be intact and the counter header of every live range, backward and split-K
workspace zero (SCRATCH_HEADERS).  Around each outermost call every CUDA tensor reachable from its arguments must keep its
bits, except the arguments WRITES names.  REACH names the workload or direct case that calls each launch symbol.
"""
import contextlib
import inspect
import threading

import numpy as np
import torch
import torch.nn.functional as F

from oracle import depth_hints as odh
from oracle import haar as ohaar
from oracle import kitti_eval as oke
from oracle import kitti_gt as okg
from oracle import kitti_inputs as oki
from oracle import kitti_loss as okl
from oracle import nyu_edges as ne
from oracle import nyu_eval as one
from oracle import nyu_inputs as oni
from oracle import nyu_loss as onl
from oracle import sgbm as osgbm
from wavelet_monodepth_b200 import (_lib, kitti_eval, kitti_gt, kitti_hints, kitti_inputs, kitti_loss, nyu_eval, nyu_inputs,
                                    nyu_loss, ops)

import conv_grad_ref
import conv_ref as cr
import disp_tail_ref
import footprint
import haar_ref as har
import head_ref as hr
from contract import Worst, errors

_f32, _f64 = torch.float32, torch.float64
EPS = 2.0 ** -24

# ops entry points that launch kernels -> their checker (method name below); pack entry points; helpers without launches
CHECKED = ("conv_rows", "head_mlp", "head_gather", "head_conv3x3", "head_idwt", "idwt_haar", "dwt_haar", "idwt_bilinear",
           "disp_tail16", "range_thresh", "level_masks", "compact", "gate_map", "nchw_to_rows", "gather_rows",
           "gather_rows_list", "rows_to_nchw", "scatter_rows", "amax_rows", "act_backward", "conv_wgrad", "conv_dgrad")
PACKS = ("pack_weight", "pack_head_weight", "pack_head_mlp", "pack_disp_tail16")
# the evaluation and loss entry points that launch kernels, (owner, attribute)
EVAL_LOSS = ((nyu_loss, "_loss_fwd"), (nyu_loss, "_loss_bwd"),
             (nyu_eval, "compute_errors_nyu"), (nyu_eval, "_edt"), (nyu_eval, "_edges_frames"),
             (nyu_eval.NyuDepthEvaluator, "add"),
             (kitti_eval, "compute_errors"), (kitti_eval, "batch_post_process_disparity"),
             (kitti_eval.KittiDepthEvaluator, "__init__"), (kitti_eval.KittiDepthEvaluator, "add"),
             (kitti_loss, "_kitti_fwd"), (kitti_loss, "_kitti_bwd"))
# the depth-hint, training-input and ground-truth pipelines' entry points that launch kernels, (owner, attribute)
PIPELINES = ((kitti_hints, "stereo_sgbm"), (kitti_hints, "_fuse"), (kitti_inputs.KittiInputs, "_run"),
             (nyu_inputs.NyuInputs, "_run"), (kitti_gt, "generate_depth_maps"))
ENTRY_POINTS = tuple((ops, name) for name in CHECKED) + EVAL_LOSS + PIPELINES


def entry_name(owner, attr):
    """'conv_rows', '_loss_fwd', 'NyuDepthEvaluator.add', 'KittiDepthEvaluator.__init__'"""
    return attr if inspect.ismodule(owner) else "%s.%s" % (owner.__name__, attr)


ENTRIES = tuple(entry_name(o, a) for o, a in ENTRY_POINTS)


def hook(prefix, entry):
    """The Harness method of an entry point: hook("_check_", "KittiDepthEvaluator.__init__") is
    "_check_KittiDepthEvaluator_init", hook("_before_", "_loss_fwd") "_before_loss_fwd"."""
    return prefix + entry.replace(".__init__", ".init").strip("_").replace(".", "_")


# every symbol of the tables of _lib.TABLES: ("launch", entry point whose checker covers it) | ("pack", ops entry point) |
# "query"
SYMBOLS = {
    "wmd_version": "query", "wmd_status_string": "query", "wmd_last_cuda_error": "query", "wmd_launch_count": "query",
    "wmd_idwt_haar_f32": ("launch", "idwt_haar"),
    "wmd_idwt_haar_epi_f32": ("launch", "idwt_haar"),
    "wmd_idwt_bilinear_f32": ("launch", "idwt_bilinear"),
    "wmd_dwt_haar_f32": ("launch", "dwt_haar"),
    "wmd_range_ws_bytes": "query",
    "wmd_range_thresh_f32": ("launch", "range_thresh"),
    "wmd_level_masks": ("launch", "level_masks"),
    "wmd_compact_ws_bytes": "query",
    "wmd_compact_mask": ("launch", "compact"),
    "wmd_gate_map": ("launch", "gate_map"),
    "wmd_nchw_to_rows_f32": ("launch", "nchw_to_rows"),
    "wmd_nchw_to_rows_gated_f32": ("launch", "nchw_to_rows"),
    "wmd_nchw_to_rows_amax_f32": ("launch", "nchw_to_rows"),
    "wmd_nchw_to_rows_masked_amax_f32": ("launch", "nchw_to_rows"),
    "wmd_nchw_to_rows_gated_amax_f32": ("launch", "nchw_to_rows"),
    "wmd_rows_to_nchw_f32": ("launch", "rows_to_nchw"),
    "wmd_gather_rows_nchw_f32": ("launch", "gather_rows"),
    "wmd_gather_rows_list_f32": ("launch", "gather_rows_list"),
    "wmd_gather_rows_list_amax_f32": ("launch", "gather_rows_list"),
    "wmd_scatter_rows_nchw_f32": ("launch", "scatter_rows"),
    "wmd_amax_f32": ("launch", "amax_rows"),
    "wmd_amax_rows_masked_f32": ("launch", "amax_rows"),
    "wmd_pack_conv_weight_f32": ("pack", "pack_weight"),
    "wmd_pack_conv_weight_tc16_f32": ("pack", "pack_weight"),
    "wmd_pack_conv_weight_tc_f32": ("pack", "pack_weight"),
    "wmd_conv_tc_weight_floats": "query",
    "wmd_conv_tc16_weight_bytes": "query",
    "wmd_conv_tc_tile_n": "query",
    "wmd_conv_tc_set_reserved_sms": "query",
    "wmd_conv_tc_splitk_ws_bytes": "query",
    "wmd_conv_rows_f32": ("launch", "conv_rows"),
    "wmd_conv_rows_tc_f32": ("launch", "conv_rows"),
    "wmd_conv_rows_tc_splitk_f32": ("launch", "conv_rows"),
    "wmd_head_mlp_supported": "query",
    "wmd_head_mlp_weight_floats": "query",
    "wmd_pack_head_mlp_f32": ("pack", "pack_head_mlp"),
    "wmd_head_mlp_f32": ("launch", "head_mlp"),
    "wmd_head_conv3x3_f32": ("launch", "head_conv3x3"),
    "wmd_head_gather_f32": ("launch", "head_gather"),
    "wmd_head_idwt_ws_bytes": "query",
    "wmd_head_idwt_f32": ("launch", "head_idwt"),
    "wmd_pack_disp_tail16_f32": ("pack", "pack_disp_tail16"),
    "wmd_disp_tail16_f32": ("launch", "disp_tail16"),
    "wmd_act_bwd_ws_bytes": "query",
    "wmd_act_bwd_f32": ("launch", "act_backward"),
    "wmd_conv_wgrad_ws_bytes": "query",
    "wmd_conv_wgrad_f32": ("launch", "conv_wgrad"),
    "wmd_conv_dgrad_fold_f32": ("launch", "conv_dgrad"),
    # include/wmd_eval.h
    "wmd_eval_gt_mask": ("launch", "KittiDepthEvaluator.__init__"),
    "wmd_eval_gather_f32": ("launch", "KittiDepthEvaluator.__init__"),
    "wmd_eval_frames": ("launch", "KittiDepthEvaluator.add"),
    "wmd_eval_errors_f64": ("launch", "compute_errors"),
    "wmd_post_process_disparity": ("launch", "batch_post_process_disparity"),
    "wmd_eval_nyu_ws_bytes": "query",
    "wmd_eval_nyu_frames": ("launch", "NyuDepthEvaluator.add"),
    "wmd_eval_nyu_errors_ws_bytes": "query",
    "wmd_eval_nyu_errors_f64": ("launch", "compute_errors_nyu"),
    "wmd_eval_edges_ws_bytes": "query",
    "wmd_eval_edges_frames": ("launch", "_edges_frames"),
    "wmd_eval_edt_ws_bytes": "query",
    "wmd_eval_edt": ("launch", "_edt"),
    # include/wmd_loss.h
    "wmd_loss_nyu_ws_bytes": "query",
    "wmd_loss_nyu_fwd": ("launch", "_loss_fwd"),
    "wmd_loss_nyu_bwd": ("launch", "_loss_bwd"),
    # include/wmd_loss_kitti.h
    "wmd_loss_kitti_ws_bytes": "query",
    "wmd_loss_kitti_bwd_ws_bytes": "query",
    "wmd_loss_kitti_fwd": ("launch", "_kitti_fwd"),
    "wmd_loss_kitti_bwd": ("launch", "_kitti_bwd"),
    # include/wmd_hints.h
    "wmd_sgbm_ws_bytes": "query",
    "wmd_sgbm_u8": ("launch", "stereo_sgbm"),
    "wmd_depth_hints_ws_bytes": "query",
    "wmd_depth_hints_f32": ("launch", "_fuse"),
    # include/wmd_inputs.h
    "wmd_inputs_ws_bytes": "query",
    "wmd_inputs_u8": ("launch", "KittiInputs._run"),
    # include/wmd_inputs_nyu.h
    "wmd_nyu_inputs_ws_bytes": "query",
    "wmd_nyu_inputs_u8": ("launch", "NyuInputs._run"),
    # include/wmd_gt.h
    "wmd_velo_depth_ws_bytes": "query",
    "wmd_velo_depth_f64": ("launch", "generate_depth_maps"),
}

# launch symbol -> the workload (tests/test_gpu_production_launches.py, tests/test_gpu_workload_launches.py) or direct
# case (tests/test_gpu_launch_footprint.py, "direct:...") that calls it under the harness; each case asserts that the
# symbols given to it were called
_SPARSE, _NYU_DENSE, _TRAIN = "sparse_r50_1024x320_x32_thr0.05", "nyu_dense_d161_640x480_x8", "train_wave_r18_640x192_x12"
_KITTI_EVAL, _NYU_EVAL = "eval_kitti_sparse_r18_x16_postprocess", "eval_nyu_sparse_d161_x16_edges"
REACH = {
    "wmd_idwt_haar_f32": _NYU_DENSE, "wmd_idwt_haar_epi_f32": "direct:idwt_forms",
    "wmd_idwt_bilinear_f32": "direct:idwt_forms", "wmd_dwt_haar_f32": _TRAIN,
    "wmd_range_thresh_f32": "nyu_sparse_d161_640x480_x8_thr0.1", "wmd_level_masks": _SPARSE, "wmd_compact_mask": _SPARSE,
    "wmd_gate_map": _SPARSE,
    "wmd_nchw_to_rows_f32": _NYU_DENSE, "wmd_nchw_to_rows_gated_f32": "direct:gated_layout_moves",
    "wmd_nchw_to_rows_amax_f32": _SPARSE, "wmd_nchw_to_rows_masked_amax_f32": "direct:gated_layout_moves",
    "wmd_nchw_to_rows_gated_amax_f32": _SPARSE, "wmd_rows_to_nchw_f32": _TRAIN,
    "wmd_gather_rows_nchw_f32": "direct:gather_scatter_rows", "wmd_gather_rows_list_f32": "direct:gather_rows_list_abi",
    "wmd_gather_rows_list_amax_f32": _SPARSE, "wmd_scatter_rows_nchw_f32": "direct:gather_scatter_rows",
    "wmd_amax_f32": "sparse_r50_1024x320_x16_channels_last", "wmd_amax_rows_masked_f32": "sparse_r50_1024x320_x16_channels_last",
    "wmd_conv_rows_f32": "baseline_depthdecoder_r18_640x192_x16", "wmd_conv_rows_tc_f32": "direct:conv_rows_tc_abi",
    "wmd_conv_rows_tc_splitk_f32": _SPARSE,
    "wmd_head_mlp_f32": _SPARSE, "wmd_head_conv3x3_f32": _NYU_DENSE, "wmd_head_gather_f32": _SPARSE,
    "wmd_head_idwt_f32": _SPARSE, "wmd_disp_tail16_f32": "baseline_depthdecoder_r18_640x192_x16",
    "wmd_act_bwd_f32": _TRAIN, "wmd_conv_wgrad_f32": _TRAIN, "wmd_conv_dgrad_fold_f32": _TRAIN,
    "wmd_eval_gt_mask": _KITTI_EVAL, "wmd_eval_gather_f32": _KITTI_EVAL, "wmd_eval_frames": _KITTI_EVAL,
    "wmd_eval_errors_f64": _KITTI_EVAL, "wmd_post_process_disparity": _KITTI_EVAL,
    "wmd_eval_nyu_frames": _NYU_EVAL, "wmd_eval_nyu_errors_f64": _NYU_EVAL, "wmd_eval_edges_frames": _NYU_EVAL,
    "wmd_eval_edt": _NYU_EVAL,
    "wmd_loss_nyu_fwd": "train_nyu_wave_d161_640x480_x8_nyuloss", "wmd_loss_nyu_bwd": "train_nyu_wave_d161_640x480_x8_nyuloss",
    "wmd_loss_kitti_fwd": "train_baseline_r18_640x192_x12_kittiloss",
    "wmd_loss_kitti_bwd": "train_baseline_r18_640x192_x12_kittiloss",
    "wmd_sgbm_u8": "hints_320x1024_pair_both_sides", "wmd_depth_hints_f32": "hints_320x1024_pair_both_sides",
    "wmd_inputs_u8": "train_wave_r18_640x192_x12_from_kitti_inputs",
    "wmd_nyu_inputs_u8": "train_nyu_wave_d161_640x480_x8_from_nyu_inputs",
    "wmd_velo_depth_f64": "gt_export_full_scans_then_eval",
}

# bars of the checks this file adds on top of the contract tests' (units of 2^-24 of the element's scale)
ACT_BWD_ULP = 4        # dz = dy act'(y): at most three roundings (sigmoid: 1 - y, y (1 - y), the product with dy)
# bars of the evaluation and loss checks: those of their own tests (test_gpu_nyu_loss, test_gpu_nyu_eval,
# test_gpu_nyu_edges, test_gpu_kitti_eval, test_gpu_kitti_loss)
LOSS_MEAN_ULP = 1      # a loss term: the device's fp64 sum and the oracle's differ in order only, one fp32 rounding apart
KITTI_GRAD_ULP = 1     # a KITTI loss gradient: fp64 sums rounded once, within one fp32 ulp of its scale's largest
EVAL_REL = 1e-12       # fp64 sums of a fixed order against math.fsum / numpy's pairwise sums
NYU_SUM_ABS = 1e-15    # per pixel: the fp64 log10's ulp, all a log_10 sum of equal depths is made of
POST_REL = 1e-15       # batch_post_process_disparity: numpy's expression, evaluated in the same precision

REPORT = Worst("entry point, engine / precision, mode")     # err in the unit of the entry's bar


def _record(entry, engine, mode, err, bar, rows):
    REPORT.note((entry, engine, mode), err, bar=bar, rows=int(rows))


def _i(t):
    return int(t.reshape(-1)[0]) if torch.is_tensor(t) else int(t)


def _nhwc(x):
    n, c = x.shape[:2]
    return x.permute(0, 2, 3, 1).reshape(-1, c)


def _scalar(t):
    return float(t.reshape(-1)[0])


class LaunchError(AssertionError):
    pass


def _require(ok, what):
    if not ok:
        raise LaunchError(what)


class _LibSpy:
    """Stands in for the loaded CDLL: counts every launch and pack symbol it forwards, and records those called while
    no wrapped entry point is running."""

    def __init__(self, lib, harness):
        self._lib, self._h = lib, harness

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("wmd_") or SYMBOLS.get(name) == "query":
            return fn
        h = self._h

        def call(*args):
            if h.depth == 0:
                h.outside.append(name)
            h.launched[name] = h.launched.get(name, 0) + 1
            return fn(*args)
        return call


# ------------------------------------------------------------------------------------------ footprint
# the arguments each entry point writes in place (outputs passed in, amax slots, an evaluator's maps and scores); every
# other CUDA tensor reachable from a call's arguments must come back bit for bit
WRITES = {
    "conv_rows": ("out", "amax_out"), "head_gather": ("out",), "head_conv3x3": ("out",), "disp_tail16": ("out",),
    "nchw_to_rows": ("amax",), "gather_rows_list": ("amax",), "scatter_rows": ("out",), "amax_rows": ("out",),
    "act_backward": ("amax",), "_loss_fwd": ("means",), "_edt": ("out",), "_edges_frames": ("scores",),
    "NyuDepthEvaluator.add": ("depth_out",), "stereo_sgbm": ("out",), "_fuse": ("depth", "index"),
}

# the counter header of each ops._Scratch workspace kind, which the kernels must leave zero (wmd.h: wmd_range_thresh_f32
# and wmd_head_idwt_f32 64 KiB, wmd_act_bwd_f32 and wmd_conv_wgrad_f32 4 KiB, the balanced wmd_conv_rows_tc_splitk_f32
# 4 KiB)
SCRATCH_HEADERS = {"range": 1 << 16, "bwd": 4096, "splitk": 4096}


def _tensors(value, path):
    """(path, tensor) of every tensor in value, looking through lists, tuples and dicts"""
    if torch.is_tensor(value):
        yield path, value
    elif isinstance(value, (list, tuple)):
        for i, v in enumerate(value):
            yield from _tensors(v, "%s[%d]" % (path, i))
    elif isinstance(value, dict):
        for k, v in value.items():
            yield from _tensors(v, "%s[%r]" % (path, k))


def _span(t):
    """(device, first byte, end byte) of the memory a tensor's elements occupy"""
    n = footprint._extent(t.shape, t.stride()) * t.element_size()
    return t.device, t.data_ptr(), t.data_ptr() + n


def snapshot(args, writes, device_type="cuda"):
    """[(path, tensor, copy)] of every tensor on `device_type` reachable from the bound arguments `args` (a dict),
    except those of the arguments named in `writes` and any that shares memory with one of them"""
    out_spans = [_span(t) for name in writes for _, t in _tensors(args.get(name), name)]
    snap = []
    for name, value in args.items():
        if name in writes:
            continue
        for path, t in _tensors(value, name):
            if t.device.type != device_type or t.numel() == 0:
                continue
            d, b, e = _span(t)
            if any(d == od and b < oe and ob < e for od, ob, oe in out_spans):
                continue
            snap.append((path, t, t.detach().clone()))
    return snap


def _bitwise(t):
    """a tensor's bits as integers, so NaN payloads compare too"""
    t = t.detach()
    if t.is_floating_point() or t.is_complex():
        return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def changed_inputs(snap):
    """paths of the snapshot's tensors whose bits differ from their copies"""
    return [path for path, t, copy in snap if not torch.equal(_bitwise(t), _bitwise(copy))]


class _ExactScratch(ops._Scratch):
    """ops._Scratch without its size floors: each workspace is exactly as large as its size query asks"""

    def _get(self, key, device, nbytes, floor, zero):
        return super()._get(key, device, nbytes, 0, zero)


def scratch_header_faults(scratch):
    """(headers checked, ["kind: byte k of its counter header is v"]) over the live workspaces of an ops._Scratch"""
    faults, checked = [], 0
    for key, buf in scratch.bufs.items():
        n = SCRATCH_HEADERS.get(key[0])
        if n is None:
            continue
        head = buf[:n]
        bad = head.nonzero()
        checked += 1
        if bad.numel():
            k = int(bad[0, 0])
            faults.append("%s workspace of %d bytes: byte %d of its %d-byte counter header is %d"
                          % (key[0], buf.numel(), k, n, int(head[k])))
    return checked, faults


class Harness:
    def __init__(self, monkeypatch):
        self.packs = {}            # data_ptr of a packed image -> (packed object, plain weights)
        self.depth = 0
        self.main = threading.get_ident()
        self.current = None
        self.checked = 0
        self.outside = []
        self.gaps = []             # kernels launched between two checked calls of a thread other than the workload's
        self.last_end = {}         # thread -> launch_count() when its last outermost checked call returned
        self.calls = {}
        self.launched = {}         # launch / pack symbol -> calls
        self.snapshots = 0         # input tensors compared after their call
        self.stats = None          # the footprint figures of the last workload
        lib = _lib.load()
        monkeypatch.setattr(_lib, "_lib", _LibSpy(lib, self))
        for owner, attr in ENTRY_POINTS:
            name = entry_name(owner, attr)
            monkeypatch.setattr(owner, attr, self._wrap(name, getattr(owner, attr), getattr(self, hook("_check_", name))))
        for name in PACKS:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name), getattr(self, "_pack_" + name)))

    # ------------------------------------------------------------------------------------------ plumbing
    def _wrap(self, name, orig, check):
        sig = inspect.signature(orig)
        before = getattr(self, hook("_before_", name), None)
        writes = WRITES.get(name, ())

        def wrapped(*args, **kwargs):
            a = sig.bind(*args, **kwargs)
            a.apply_defaults()
            a = dict(a.arguments)
            outer = self.depth == 0
            if outer:
                torch.cuda.synchronize()
                c0 = _lib.launch_count()
                tid = threading.get_ident()
                if tid != self.main and tid in self.last_end and c0 != self.last_end[tid]:
                    self.gaps.append((name, c0 - self.last_end[tid]))
                snap = snapshot(a, writes)
            pre = before(a) if before is not None else None
            self.depth += 1
            try:
                res = orig(*args, **kwargs)
            finally:
                self.depth -= 1
            torch.cuda.synchronize()
            if outer:
                c1 = _lib.launch_count()
                self.last_end[tid] = c1
                if tid == self.main:
                    self.checked += c1 - c0
                changed = changed_inputs(snap)
                self.snapshots += len(snap)
                del snap
                _require(not changed, "%s: %s changed its inputs %s" % (self.current, name, changed))
            self.calls[name] = self.calls.get(name, 0) + 1
            check(a, res, pre)
            return res
        return wrapped

    @contextlib.contextmanager
    def workload(self, name):
        """Checks that every kernel launched inside the block ran inside a checked call.  launch_count() counts per host
        thread: on the calling thread the checked deltas must add up to the whole; autograd runs the backward on its own
        thread, whose counter must not move between two checked calls.  The block runs under footprint.Footprint with
        exactly sized workspaces; its guards and the workspaces' counter headers are checked at the end (self.stats)."""
        torch.cuda.synchronize()
        self.current, self.checked, self.outside, self.gaps, self.last_end = name, 0, [], [], {}
        self.launched, self.snapshots = {}, 0
        self.main = threading.get_ident()
        saved, scratch = ops._scratch, _ExactScratch()
        ops._scratch = scratch
        try:
            with footprint.Footprint() as fp:
                c0 = _lib.launch_count()
                yield self
                torch.cuda.synchronize()
                total = _lib.launch_count() - c0
        finally:
            ops._scratch = saved
        _require(not self.outside and not self.gaps and total == self.checked,
                 "%s: %d kernels launched, %d inside checked calls; libwmd called outside them: %s; launched between "
                 "checked calls of the backward thread, before: %s" % (name, total, self.checked, sorted(set(self.outside)),
                                                                        self.gaps))
        _require(total > 0, "%s launched nothing" % name)
        headers, faults = scratch_header_faults(scratch)
        _require(not faults, "%s: workspace counters left nonzero: %s" % (name, faults))
        self.stats = dict(arenas=fp.checked, guarded=fp.guarded, snapshots=self.snapshots, headers=headers)

    def report(self):
        """the footprint figures of the last workload, one line"""
        s = self.stats
        return ("%d arenas checked, %.1f MB guarded, %d input snapshots compared, %d scratch headers checked"
                % (s["arenas"], s["guarded"] / 1e6, s["snapshots"], s["headers"]))

    def reached(self, case):
        """the launch symbols REACH attributes to `case` that this harness has not seen called"""
        return sorted(s for s, c in REACH.items() if c == case and not self.launched.get(s))

    def _weights(self, packed):
        key = packed.data.data_ptr() if isinstance(packed, ops.PackedW) else packed.data_ptr()
        _require(key in self.packs, "a launch uses a packed weight no pack call of this harness produced")
        return self.packs[key][1]

    def _keep(self, packed, weights):
        key = packed.data.data_ptr() if isinstance(packed, ops.PackedW) else packed.data_ptr()
        self.packs[key] = (packed, weights)

    # ------------------------------------------------------------------------------------------ packs
    def _pack_pack_weight(self, a, res, pre):
        self._keep(res, a["weight"].detach().clone())

    def _pack_pack_head_weight(self, a, res, pre):
        self._keep(res, a["weight"].detach().clone())

    def _pack_pack_head_mlp(self, a, res, pre):
        b1 = a["b1"].detach().clone() if a["b1"] is not None else None
        self._keep(res, (a["w1"].detach().clone(), b1, a["wz"].detach().clone()))

    def _pack_pack_disp_tail16(self, a, res, pre):
        self._keep(res, tuple(t.detach().clone() if t is not None else None for t in (a["w1"], a["b1"], a["w2"], a["b2"])))

    # ------------------------------------------------------------------------------------------ shared preconditions
    def _check_list(self, entry, pixels, count, max_rows, total):
        """count <= max_rows; the first min(count, max_rows) entries of the list strictly increasing, inside the grid."""
        if pixels is None:
            return total
        cnt = _i(count)
        _require(0 <= cnt <= max_rows, "%s: count %d outside [0, max_rows = %d]" % (entry, cnt, max_rows))
        p = pixels.reshape(-1)[:cnt].long()
        if cnt:
            _require(bool((p[1:] > p[:-1]).all()), "%s: pixel list not strictly increasing" % entry)
            _require(int(p[0]) >= 0 and int(p[-1]) < total, "%s: pixel list leaves the %d-pixel grid" % (entry, total))
        return cnt

    def _check_map(self, entry, m, rows):
        if m is not None and m.numel():
            _require(int(m.max()) < rows, "%s: index map entry %d past the %d rows of its source" % (entry, int(m.max()), rows))
            _require(int(m.min()) >= -1, "%s: index map entry below -1" % entry)

    def _before_amax(self, t):
        return t.clone() if t is not None else None

    def _check_amax_out(self, entry, old, new, values):
        want = max(_scalar(old), cr.finite_max(values))      # NaN and +-Inf do not count (wmd.h, amax_out)
        _require(_scalar(new) == want, "%s: amax %.9g, want exactly %.9g" % (entry, _scalar(new), want))

    # ------------------------------------------------------------------------------------------ convolution
    def _before_conv_rows(self, a):
        return self._before_amax(a["amax_out"])

    def _check_conv_rows(self, a, out, old_amax):
        wp = a["wpacked"]
        weight = self._weights(wp)
        n, h, w, taps, c0, c1, cout = a["n"], a["h"], a["w"], a["taps"], a["c0"], a["c1"], a["cout"]
        x0, x1 = a["x0"], a["x1"]
        total = n * h * w
        max_rows = total if a["max_rows"] is None else int(a["max_rows"])
        splits = a["splits"]
        if wp.kind == "tc" and splits is None:
            nchunks = taps * (-(-c0 // 32) + -(-c1 // 32))
            splits = 0 if nchunks >= ops.TC_BALANCE_MIN_CHUNKS else 1
        use16 = (wp.kind == "tc" and wp.data16 is not None and a["amax0"] is not None
                 and (x1 is None or a["amax1"] is not None) and splits in (0, 1))
        engine = "simt" if wp.kind == "simt" else ("f16x3" if use16 else "tf32x3")
        mode = "-" if wp.kind == "simt" else {1: "whole", 0: "balanced"}.get(splits, "split-K")
        dense3 = taps == 9 and a["pixels"] is None and a["map0"] is None and a["map1"] is None and a["gate"] is None
        mode += "/dense3x3" if dense3 else ("/1x1" if taps == 1 else "/gather")
        entry = "conv_rows"
        rows = min(self._check_list(entry, a["pixels"], a["count"], max_rows, total), max_rows)
        rows0 = int(x0.shape[0])
        self._check_map(entry, a["map0"], rows0)
        if x1 is not None:
            self._check_map(entry, a["map1"], int(x1.shape[0]))
        amax16 = max(_scalar(a["amax0"]), _scalar(a["amax1"]) if x1 is not None else 0.0) if use16 else None
        ref = cr.conv_ref(x0, c0, weight, a["bias"], n, h, w, taps=taps, pad=a["pad"], act=a["act"],
                          act_param=a["act_param"], map0=a["map0"], shift0=a["shift0"], x1=x1, c1=c1,
                          map1=a["map1"], gate=a["gate"], pixels=a["pixels"], count=a["count"],
                          max_rows=max_rows, rows0=rows0 if (taps == 1 and a["map0"] is None) else None,
                          read_max=True, f16_amax=amax16, floor=engine)
        y64, s, m0, m1 = ref[:4]
        floor = ref[4]                          # BAR S + F with the engine's floor (conv_ref, the f16x3 / tf32x3 / FMA bounds)
        if use16:
            _require(_scalar(a["amax0"]) >= m0, "conv_rows: amax0 %.9g below the largest |x0| read, %.9g"
                     % (_scalar(a["amax0"]), m0))
            if x1 is not None:
                _require(_scalar(a["amax1"]) >= m1, "conv_rows: amax1 %.9g below the largest |x1| read, %.9g"
                         % (_scalar(a["amax1"]), m1))
        y = out[:rows, :cout]
        if wp.kind == "tc" and a["amax_out"] is not None:
            self._check_amax_out(entry, old_amax, a["amax_out"], y)
        allow = 0.0 if a["act"] in (cr.ACT_NONE, cr.ACT_LRELU) else cr.ACT_ALLOW
        err = errors(y, y64, s, allow + floor)[0]
        bar = cr.BAR[engine]
        _record(entry, engine, mode, err, bar, rows)
        _require(err <= bar, "%s: conv_rows %s %s (n %d, %dx%d, c0 %d, c1 %d, cout %d, taps %d, %d rows): err/S %.3g > %.3g"
                 % (self.current, engine, mode, n, h, w, c0, c1, cout, taps, rows, err, bar))

    # ------------------------------------------------------------------------------------------ coefficient heads
    def _check_head_mlp(self, a, z, pre):
        w1, b1, wz = self._weights(a["packed"])
        x = a["x"]
        max_rows = x.shape[0] if a["max_rows"] is None else int(a["max_rows"])
        count = _i(a["count"]) if a["count"] is not None else None
        if count is not None:
            _require(count <= max_rows, "head_mlp: count %d > max_rows %d" % (count, max_rows))
        rows = max_rows if count is None else min(count, max_rows)
        want, s, floor = hr.head_mlp_ref(x, a["c"], w1, b1, wz, a["slope"], count, max_rows, floor=True)
        nz = a["nz"]
        _require(bool((z[:rows, nz:56] == 0).all()), "head_mlp: columns nz..55 are not zero")
        err = errors(z[:rows, :nz], want, s, floor)[0]
        bar = hr.BAR["head_mlp"]
        _record("head_mlp", "tf32x3", "-", err, bar, rows)
        _require(err <= bar, "%s: head_mlp err/S %.3g > %.3g" % (self.current, err, bar))

    def _written(self, out, pixels, rows, cout):
        flat = out.permute(0, 2, 3, 1).reshape(-1, cout)
        return flat[pixels.reshape(-1)[:rows].long()] if pixels is not None else flat

    def _check_head_gather(self, a, out, pre):
        z, groups, n, h, w, cout = a["z"], a["groups"], a["n"], a["h"], a["w"], a["cout"]
        total = n * h * w
        max_rows = total if a["max_rows"] is None else int(a["max_rows"])
        rows = min(self._check_list("head_gather", a["pixels"], a["count"], max_rows, total), max_rows)
        self._check_map("head_gather", a["idxmap"], z.shape[0])
        want, s = hr.head_gather_ref(z, z.shape[1], a["col0"], groups, a["idxmap"], a["bias"], a["scale"], a["act"],
                                     a["dual"], a["pad"], a["pixels"], a["count"], max_rows, cout, n, h, w)
        allow = 0.0 if a["act"] == cr.ACT_NONE else cr.ACT_ALLOW * abs(a["scale"]) * (2 if a["dual"] else 1)
        err = errors(self._written(out, a["pixels"], rows, cout), want, s, allow)[0]
        bar = hr.BAR["head_gather"]
        _record("head_gather", "fp32", "list" if a["pixels"] is not None else "dense", err, bar, rows)
        _require(err <= bar, "%s: head_gather err/S %.3g > %.3g" % (self.current, err, bar))

    def _check_head_conv3x3(self, a, out, pre):
        t, n, h, w, cout, c = a["t"], a["n"], a["h"], a["w"], a["cout"], a["c"]
        total = n * h * w
        max_rows = total if a["max_rows"] is None else int(a["max_rows"])
        rows = min(self._check_list("head_conv3x3", a["pixels"], a["count"], max_rows, total), max_rows)
        self._check_map("head_conv3x3", a["idxmap"], t.shape[0])
        dual = a["off_b"] >= 0
        wa = self._weights(a["wa"])
        wb = self._weights(a["wb"]) if dual else None
        want, s = hr.head_conv3x3_ref(t, t.shape[1], c, a["off_a"], a["off_b"], wa, a["ba"], wb, a["bb"], cout, a["scale"],
                                      a["act"], a["pad"], a["idxmap"], a["pixels"], a["count"], max_rows, n, h, w)
        allow = 0.0 if a["act"] == cr.ACT_NONE else cr.ACT_ALLOW * abs(a["scale"]) * (2 if dual else 1)
        err = errors(self._written(out, a["pixels"], rows, cout), want, s, allow)[0]
        bar = hr.BAR["head_conv3x3"]
        _record("head_conv3x3", "fp32", "list" if a["pixels"] is not None else "dense", err, bar, rows)
        _require(err <= bar, "%s: head_conv3x3 (c %d, cout %d) err/S %.3g > %.3g" % (self.current, c, cout, err, bar))

    def _check_head_idwt(self, a, res, pre):
        z, yl = a["z"], a["yl"]
        n, _, h, w = yl.shape
        self._check_map("head_idwt", a["idxmap"], z.shape[0])
        ref = hr.head_idwt_ref(z, a["col0"], a["idxmap"], a["mask"], a["bias"], a["scale"], a["pad"], yl, a["disp_scale"],
                               a["clamp01"], n, h, w)
        al = cr.ACT_ALLOW * abs(a["scale"])
        err = max(errors(res["yh"], ref["yh"], ref["s_yh"], 2 * al)[0],
                  errors(res["out"], ref["out"], ref["s_out"], 3 * al)[0],
                  errors(res["disp"], ref["disp"], ref["s_disp"], 3 * al * abs(a["disp_scale"]))[0])
        if a["mask"] is not None:
            off = (a["mask"].reshape(n, 1, h, w) == 0).expand(-1, 3, -1, -1)
            _require(bool((res["yh"][off] == 0).all()), "head_idwt: coefficients outside the wavelet mask are not zero")
        bar = hr.BAR["head_idwt"]
        _record("head_idwt", "fp32", "masked" if a["mask"] is not None else "dense", err, bar, n * h * w)
        _require(err <= bar, "%s: head_idwt err/S %.3g > %.3g" % (self.current, err, bar))
        if a["thresh_ratio"] is not None:
            o = res["out"].reshape(n, -1)
            want = (o.amax(1) - o.amin(1)) * torch.tensor(a["thresh_ratio"], dtype=_f32, device=o.device)
            _require(har.same_bits(res["thresh"], want), "head_idwt: threshold is not (max - min)(out) * ratio")
        self._check_epilogue("head_idwt", a["epilogue"], res["out"], res["disp"],
                             [res[k] for k in ("scaled_disp", "depth") if k in res])

    def _check_epilogue(self, entry, epi, out, disp, planes):
        """The consumer epilogue planes against the torch expressions on the kernel's own reconstruction / disparity: NaN
        exactly where they are NaN, and equal values elsewhere."""
        if epi is None:
            return
        for p, want in zip(planes, epilogue_ref(epi, out, disp)):
            _require(har.same_values(p, want), "%s: %s epilogue plane" % (entry, epi[0]))

    # ------------------------------------------------------------------------------------------ Haar transforms
    def _oracle_idwt(self, ll, hf):
        """oracle.haar's synthesis in fp32 on the CPU (the order the kernel claims bit-identity with)."""
        return ohaar.DWTInverse("haar", "zero")((ll.detach().float().cpu(), [hf.detach().float().cpu()]))

    def _check_idwt_haar(self, a, res, pre):
        """The reconstruction bit for bit (NaN where the oracle's is NaN), the disparity and epilogue planes by value."""
        ll, hf = a["ll"], a["hf"]
        n, c, h, w = ll.shape
        res_t = res if isinstance(res, tuple) else (res,)
        want = self._oracle_idwt(ll, hf.reshape(n, c, 3, h, w))
        _require(har.same_bits(res_t[0], want), "idwt_haar: reconstruction differs from oracle.haar.DWTInverse")
        disp = har.disp(want, a["disp_scale"] if a["disp_scale"] is not None else 1.0, a["clamp01"])
        k = 1
        if a["disp_scale"] is not None:
            _require(har.same_values(res_t[1], disp), "idwt_haar: disparity plane")
            k = 2
        if a["epilogue"] is not None:
            self._check_epilogue("idwt_haar", a["epilogue"], res_t[0], disp.to(res_t[0].device), list(res_t[k:]))
        _record("idwt_haar", "fp32", "-", 0.0, 0, n * c * h * w)

    def _check_dwt_haar(self, a, res, pre):
        """One analysis level against oracle.haar in fp64: |err| <= DWT_ULP 2^-24 S + DWT_FLOOR, S = 1/2 the sum of the four
        |x| (haar_ref)."""
        x = a["x"]
        ll, hf = res
        n, c, hh, ww = x.shape
        x64 = x.detach().double()
        rl, rh = ohaar.DWTForward(J=1, wave="haar", mode="zero").to(x.device).double()(x64)
        sc = 0.5 * F.avg_pool2d(x64.abs(), 2) * 4
        bar = har.DWT_ULP * EPS
        e_l, f_l = errors(ll, rl, sc, floor=har.DWT_FLOOR, bar=bar)
        e_h, f_h = errors(hf, rh[0], sc.unsqueeze(2).expand_as(rh[0]), floor=har.DWT_FLOOR, bar=bar)
        ol, oh = ohaar.DWTForward(J=1, wave="haar", mode="zero")(x.detach().float().cpu())
        exact = har.same_bits(ll, ol) and har.same_bits(hf, oh[0])
        REPORT.note(("dwt_haar", "fp32", "exact" if exact else "bounded"), max(e_l, e_h), max(f_l, f_h), bar=bar,
                    rows=n * c * hh * ww // 4)
        _require(max(f_l, f_h) <= 1, "%s: dwt_haar err %.3g > DWT_ULP 2^-24 S + DWT_FLOOR" % (self.current, max(f_l, f_h)))

    def _check_idwt_bilinear(self, a, full, pre):
        ll, hf, size, ac = a["ll"], a["hf"], a["size"], bool(a["align_corners"])
        n, c, h, w = ll.shape
        disp = har.disp(self._oracle_idwt(ll, hf.reshape(n, c, 3, h, w)), a["disp_scale"], a["clamp01"])
        disp = disp.to(full.device).double()
        ulps = hr.bilinear_ulps(full, disp, size, ac)
        _record("idwt_bilinear", "fp32", "ac" if ac else "-", ulps, hr.BILINEAR_ULP, full.numel())
        _require(ulps <= hr.BILINEAR_ULP, "%s: idwt_bilinear %.3g ulp > %.3g" % (self.current, ulps, hr.BILINEAR_ULP))

    # ------------------------------------------------------------------------------------------ baseline tail
    def _check_disp_tail16(self, a, out, pre):
        n = a["n"]
        if n == 0:
            return
        w1, b1, w2, b2 = self._weights(a["packed"])
        want, s, floor = disp_tail_ref.disp_tail_ref(a["x"], w1, b1, w2, b2, n, a["h"], a["w"], floor=True)
        err = errors(out, want, s, floor)[0]
        _record("disp_tail16", "tf32x3", "-", err, disp_tail_ref.BAR, n * a["h"] * a["w"] * 4)
        _require(err <= disp_tail_ref.BAR, "%s: disp_tail16 err/S %.3g > %.3g" % (self.current, err, disp_tail_ref.BAR))

    # ------------------------------------------------------------------------------------------ masks and compaction
    def _check_range_thresh(self, a, res, pre):
        x = a["x"]
        n = x.shape[0]
        xs = x.reshape(n, -1).float()
        mn, mx = xs.amin(1), xs.amax(1)
        want = (mx - mn) * torch.tensor(a["ratio"], dtype=_f32, device=x.device)
        got = res[0] if a["return_minmax"] else res
        _require(torch.equal(got, want), "range_thresh: not (max - min) * ratio")
        if a["return_minmax"]:
            _require(torch.equal(res[1], torch.stack([mn, mx], 1)), "range_thresh: minmax")
        _record("range_thresh", "fp32", "-", 0.0, 0, n)

    def _check_level_masks(self, a, res, pre):
        if a["thresh"] is not None:
            yh = a["yh"]
            n, h, w = yh.shape[0], yh.shape[-2], yh.shape[-1]
        else:
            yh, n, h, w = None, a["n"], a["h"], a["w"]
        want = level_masks_ref(yh, a["thresh"], n, h, w, a["device"])
        for k, m in res.items():
            _require(torch.equal(m, want[k]), "level_masks: %s" % k)
        _record("level_masks", "-", "-", 0.0, 0, n * h * w)

    def _check_compact(self, a, res, pre):
        if a["stream"] is not None:
            res = res[0]
        idxmap, pixels, offsets = res
        mask = a["mask"]
        n, h, w = mask.shape[0], mask.shape[-2], mask.shape[-1]
        m = mask.reshape(n, h, w)
        per = (m != 0).reshape(n, -1).sum(1)
        want_off = torch.cat([per.new_zeros(1), per.cumsum(0)]).to(torch.int32)
        _require(torch.equal(offsets, want_off), "compact: offsets")
        if idxmap is not None:
            _require(torch.equal(idxmap, cr.index_map(m)), "compact: index map")
        if pixels is not None:
            lst = cr.pixel_list(m)
            _require(torch.equal(pixels[:len(lst)], lst), "compact: pixel list")
        _record("compact", "-", "-", 0.0, 0, n * h * w)

    def _check_gate_map(self, a, out, pre):
        gate = a["gate"]
        n, h, w = gate.shape[0], gate.shape[-2], gate.shape[-1]
        g = gate.reshape(n, h, w) != 0
        src = a["idxmap"].reshape(n, h, w) if a["idxmap"] is not None else \
            torch.arange(n * h * w, dtype=torch.int32, device=gate.device).reshape(n, h, w)
        _require(torch.equal(out, torch.where(g, src, torch.full_like(src, -1))), "gate_map")
        _record("gate_map", "-", "-", 0.0, 0, n * h * w)

    # ------------------------------------------------------------------------------------------ layout moves
    def _before_nchw_to_rows(self, a):
        return self._before_amax(a["amax"])

    def _check_nchw_to_rows(self, a, rows, old_amax):
        x = a["x"]
        n, c, h, w = x.shape
        xr = _nhwc(x.to(rows.device) if not x.is_cuda else x)
        gate = a["gate"]
        if gate is not None:
            sel = gate.reshape(-1) != 0
            got, want = rows[sel], xr[sel]
            mode = "gated-host" if not x.is_cuda else "gated"
        else:
            sel = None
            got, want = rows, xr
            mode = "view" if rows.data_ptr() == x.data_ptr() else "plain"
        _require(torch.equal(got[:, :c], want), "nchw_to_rows (%s): rows differ from the map" % mode)
        if got.shape[1] > c:
            _require(bool((got[:, c:] == 0).all()), "nchw_to_rows: pad columns are not zero")
        if a["amax"] is not None:
            cover = gate if gate is not None else a["amax_mask"]
            vals = xr[cover.reshape(-1) != 0] if cover is not None else xr
            self._check_amax_out("nchw_to_rows (%s)" % mode, old_amax, a["amax"], vals)
            mode += "+amax" if a["amax_mask"] is None or gate is not None else "+masked amax"
        _record("nchw_to_rows", "-", mode, 0.0, 0, n * h * w)

    def _check_rows_to_nchw(self, a, out, pre):
        rows, n, c, h, w = a["rows"], a["n"], a["c"], a["h"], a["w"]
        _require(torch.equal(out, rows[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2)), "rows_to_nchw")
        _record("rows_to_nchw", "-", "-", 0.0, 0, n * h * w)

    def _check_gather_rows(self, a, rows, pre):
        x = a["x_nchw"]
        n, c, h, w = x.shape
        total = n * h * w
        max_rows = total if a["max_rows"] is None else a["max_rows"]
        r = min(self._check_list("gather_rows", a["pixels"], a["count"], max_rows, total), max_rows)
        xr = _nhwc(x)
        want = xr[a["pixels"].reshape(-1)[:r].long()] if a["pixels"] is not None else xr[:r]
        _require(torch.equal(rows[:r, :c], want), "gather_rows")
        _record("gather_rows", "-", "-", 0.0, 0, r)

    def _before_gather_rows_list(self, a):
        return self._before_amax(a["amax"])

    def _check_gather_rows_list(self, a, res, old_amax):
        rows = res[0] if a["stream"] is not None else res
        x = a["x"]
        n, c, h, w = x.shape
        total = n * h * w
        r = self._check_list("gather_rows_list", a["pixels"], a["count"], total, total)
        xr = _nhwc(x.to(rows.device) if not x.is_cuda else x)
        want = xr[a["pixels"].reshape(-1)[:r].long()]
        _require(torch.equal(rows[:r, :c], want), "gather_rows_list: rows differ from the listed pixels")
        if rows.shape[1] > c:
            _require(bool((rows[:r, c:] == 0).all()), "gather_rows_list: pad columns are not zero")
        if a["amax"] is not None:
            self._check_amax_out("gather_rows_list", old_amax, a["amax"], want)
        _record("gather_rows_list", "-", "host" if not x.is_cuda else "device", 0.0, 0, r)

    def _before_scatter_rows(self, a):
        return a["out"].clone() if a["out"] is not None else None

    def _check_scatter_rows(self, a, out, old):
        rows, c, n, h, w = a["rows"], a["c"], a["n"], a["h"], a["w"]
        total = n * h * w
        max_rows = min(rows.shape[0], total) if a["max_rows"] is None else a["max_rows"]
        r = min(self._check_list("scatter_rows", a["pixels"], a["count"], max_rows, total), max_rows)
        want = (old if old is not None else torch.zeros_like(out)).permute(0, 2, 3, 1).reshape(total, c).clone()
        want[a["pixels"].reshape(-1)[:r].long()] = rows[:r, :c]
        _require(torch.equal(out, want.reshape(n, h, w, c).permute(0, 3, 1, 2)), "scatter_rows")
        _record("scatter_rows", "-", "-", 0.0, 0, r)

    def _before_amax_rows(self, a):
        return self._before_amax(a["out"])

    def _check_amax_rows(self, a, res, old):
        x, mask = a["x"], a["mask"]
        vals = x.reshape(x.shape[0], -1)[mask.reshape(-1) != 0] if mask is not None else x
        self._check_amax_out("amax_rows", old, a["out"], vals)
        _record("amax_rows", "-", "masked" if mask is not None else "all", 0.0, 0, x.shape[0])

    # ------------------------------------------------------------------------------------------ backward
    def _dz64(self, y, dy, cout, act, act_param):
        """dy act'(y) in fp64 from the fp32 inputs (act_param as the fp32 the kernel receives)."""
        y64, dy64 = y[:, :cout].double(), dy[:, :cout].double()
        slope = float(torch.tensor(act_param, dtype=_f32))
        d = {cr.ACT_NONE: torch.ones_like(y64), cr.ACT_ELU: torch.where(y64 > 0, 1.0, y64 + 1),
             cr.ACT_LRELU: torch.where(y64 > 0, 1.0, slope), cr.ACT_SIGMOID: y64 * (1 - y64)}[act]
        return dy64 * d

    def _before_act_backward(self, a):
        return self._before_amax(a["amax"])

    def _check_act_backward(self, a, res, old_amax):
        dz, db = res
        cout = a["cout"]
        want = self._dz64(a["y"], a["dy"], cout, a["act"], a["act_param"])
        rows = want.shape[0]
        dz_floor, db_floor = conv_grad_ref.act_bwd_floor(a["dy"][:, :cout], rows_summed=rows)
        err = errors(dz[:, :cout], want, want.abs().clamp(min=1e-38), dz_floor)[0]
        bar = ACT_BWD_ULP * EPS
        _record("act_backward", "fp32", "dz", err, bar, rows)
        _require(err <= bar, "%s: act_backward dz %.3g > %.3g relative" % (self.current, err, bar))
        if a["amax"] is not None:
            self._check_amax_out("act_backward", old_amax, a["amax"], dz[:, :cout])
        if db is not None:
            gb, sb = want.sum(0), want.abs().sum(0)
            err = errors(db, gb, sb, db_floor)[0]
            bar = conv_grad_ref.BARS["db"]
            _record("act_backward", "fp32", "db", err, bar, rows)
            _require(err <= bar, "%s: act_backward db err/S %.3g > %.3g" % (self.current, err, bar))

    def _grad_sources(self, a, rows0, with_data):
        x0, x1 = a.get("x0"), a.get("x1")
        c0, c1 = a["c0"], a["c1"]
        dev = a["dz"].device
        x0r = x0[:, :c0] if with_data else torch.zeros(rows0, c0, dtype=_f32, device=dev)
        x1r = None
        if c1:
            x1r = x1[:, :c1] if with_data else torch.zeros(a["n"] * a["h"] * a["w"], c1, dtype=_f32, device=dev)
        return x0r, x1r

    def _check_conv_wgrad(self, a, dw, pre):
        n, h, w, taps, c0, c1, cout = a["n"], a["h"], a["w"], a["taps"], a["c0"], a["c1"], a["cout"]
        _require(a["map0"] is None, "conv_wgrad: the harness restates dense layers only")
        x0r, x1r = self._grad_sources(a, None, True)
        k = 3 if taps == 9 else 1
        wzero = torch.zeros(cout, c0 + c1, k, k, dtype=_f32, device=dw.device)
        with torch.enable_grad():                               # the autograd backward calling this runs without
            ref = conv_grad_ref.conv_grads(x0r, c0, x1r, c1, wzero, a["dz"][:, :cout], n, h, w, taps=taps, pad=a["pad"],
                                           shift0=a["shift0"])
            floor = conv_grad_ref.wgrad_floor(x0r, c0, x1r, c1, wzero, a["dz"][:, :cout], n, h, w, taps=taps,
                                              pad=a["pad"], shift0=a["shift0"])
        err = errors(dw, *ref["w"], floor)[0]
        bar = conv_grad_ref.BARS["dW"]
        _record("conv_wgrad", "tf32x3", "cout<=8" if cout <= 8 else "-", err, bar, n * h * w)
        _require(err <= bar, "%s: conv_wgrad (n %d, %dx%d, c0 %d, c1 %d, cout %d) err/S %.3g > %.3g"
                 % (self.current, n, h, w, c0, c1, cout, err, bar))

    def _check_conv_dgrad(self, a, res, pre):
        dx0, dx1 = res
        n, h, w, taps, c0, c1, cout, shift0 = a["n"], a["h"], a["w"], a["taps"], a["c0"], a["c1"], a["cout"], a["shift0"]
        wt = self._weights(a["wt_packed"])                      # W.transpose(0, 1).flip(2, 3)
        weight = wt.flip(2, 3).transpose(0, 1)
        rows0 = n * (h >> shift0) * (w >> shift0)
        a = dict(a, x0=None, x1=None)
        x0r, x1r = self._grad_sources(a, rows0, False)
        with torch.enable_grad():
            ref = conv_grad_ref.conv_grads(x0r, c0, x1r, c1, weight, a["dz"][:, :cout], n, h, w, taps=taps, pad=a["pad"],
                                           shift0=shift0)
        floor = {"x0": 0.0, "x1": 0.0}
        if a["amax"] is not None:           # the fp16-pair form: BAR S + F (conv_grad_ref.dgrad_floor)
            floor = conv_grad_ref.dgrad_floor(c0, c1, weight, a["dz"][:, :cout], n, h, w, _scalar(a["amax"]), taps=taps,
                                              pad=a["pad"], shift0=shift0)
        err0 = errors(dx0[:, :c0], *ref["x0"], allow=floor["x0"])[0]
        _require(bool((dx0[:, c0:] == 0).all()), "conv_dgrad: dx0 pad columns are not zero")
        _record("conv_dgrad", "dx0", "taps%d" % taps, err0, conv_grad_ref.BARS["dx0"], rows0)
        _require(err0 <= conv_grad_ref.BARS["dx0"], "%s: conv_dgrad dx0 err/S %.3g > %.3g"
                 % (self.current, err0, conv_grad_ref.BARS["dx0"]))
        if dx1 is not None:
            want, s = ref["x1"]
            err1 = errors(_nhwc(dx1), want, s, allow=floor["x1"])[0]
            _record("conv_dgrad", "dx1", "taps%d" % taps, err1, conv_grad_ref.BARS["dx1"], n * h * w)
            _require(err1 <= conv_grad_ref.BARS["dx1"], "%s: conv_dgrad dx1 err/S %.3g > %.3g"
                     % (self.current, err1, conv_grad_ref.BARS["dx1"]))

    # ------------------------------------------------------------------------------------------ NYUv2 training loss
    def _check_loss_fwd(self, a, signs, pre):
        """means[k] within LOSS_MEAN_ULP fp32 ulp of oracle.nyu_loss.term, NaN where it is NaN; int8 signs equal"""
        target = _np(a["target"])[:, 0]
        n, H, W = target.shape
        means = _np(a["means"])
        worst = 0.0
        for k, (p, lg) in enumerate(zip(a["preds"], a["log2s"])):
            pk = _np(p)[:, 0]
            _require(pk.shape[1] << lg == H and pk.shape[2] << lg == W, "_loss_fwd: term %d is not the target / 2^%d"
                     % (k, lg))
            want = onl.term(pk, target)
            _require(np.isnan(means[k]) == np.isnan(want), "_loss_fwd: term %d is %r, want %r" % (k, means[k], want))
            if not np.isnan(want):
                worst = max(worst, _ulps(means[k], want))
            if signs is not None:
                ws = onl.signs(onl.upsample(pk, H, W), target)
                bad = int((_np(signs[k]) != ws).sum())
                _require(bad == 0, "%s: _loss_fwd term %d (%dx%d, factor 2^%d): %d signs differ"
                         % (self.current, k, pk.shape[1], pk.shape[2], lg, bad))
        _record("_loss_fwd", "fp64", "ulp" + ("+signs" if signs is not None else ""), worst, LOSS_MEAN_ULP,
                n * H * W * len(a["preds"]))
        _require(worst <= LOSS_MEAN_ULP, "%s: _loss_fwd %.3g fp32 ulp > %d" % (self.current, worst, LOSS_MEAN_ULP))

    def _check_loss_bwd(self, a, grads, pre):
        """grads[k] = fp32((g_k / (N H W)) S) of oracle.nyu_loss.adjoint on the call's own signs, bit for bit"""
        n, _, H, W = a["target_shape"]
        sg = _np(a["signs"])
        g = _np(a["grad_means"]).astype(np.float32)
        worst = 0.0
        for k, p in enumerate(a["preds"]):
            h, w = int(p.shape[2]), int(p.shape[3])
            coef = np.float64(g[k]) / np.float64(n * H * W)
            want = (coef * onl.adjoint(sg[k], h, w)).astype(np.float32)
            got = _np(grads[k])[:, 0]
            if not np.array_equal(got, want, equal_nan=True):
                bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
                worst = max(worst, float(np.nan_to_num(_ulps(got[bad], want[bad]), nan=np.inf).max()))
                _require(False, "%s: _loss_bwd term %d (%dx%d from %dx%d): %d gradients differ, worst %.3g ulp"
                         % (self.current, k, h, w, H, W, int(bad.sum()), worst))
        _record("_loss_bwd", "fp64", "bits", worst, 0, n * H * W * len(a["preds"]))

    # ------------------------------------------------------------------------------------------ KITTI training loss
    def _kitti_oracle(self, a, grads):
        """oracle.kitti_loss.run in contract mode on the call's own inputs, noise, options and (backward) grad_terms"""
        t, loss_scales = a["t"], tuple(a["loss_scales"])
        inp = {k: _np(t[k]) for k in ("target", "source", "K", "inv_K", "stereo_T", "depth_hint", "depth_hint_mask")}
        inp["colors"] = {s: _np(c) for s, c in zip(loss_scales, t["color"])}
        disps = {s: _np(d) for s, d in zip(loss_scales, t["disp"])}
        noise = {s: _np(z) for s, z in zip(loss_scales, t["noise"])}
        min_depth, max_depth, smooth = a["opt"]
        gt = _np(a["grad_terms"]) if grads else None
        return okl.run(inp, disps, noise, tuple(a["scales"]), loss_scales, min_depth=min_depth, max_depth=max_depth,
                       disparity_smoothness=smooth, grads=grads, grad_terms=gt)

    def _kitti_masks(self, entry, o, loss_scales, idsel, hpix):
        for i, s in enumerate(loss_scales):
            for key, m in (("identity_selection", idsel), ("depth_hint_pixels", hpix)):
                bad = int((_np(m[i])[:, 0] != o[key][s]).sum())
                _require(bad == 0, "%s: %s scale %d: %d mask pixels differ from oracle.kitti_loss" % (entry, key, s, bad))

    def _check_kitti_fwd(self, a, res, pre):
        """oracle.kitti_loss.run (contract mode): color_depth_hint, the warped colours and both masks bit for bit; the
        terms within LOSS_MEAN_ULP fp32 ulp, NaN exactly where the oracle's are"""
        terms, chint, warped, idsel, hpix, _ = res
        loss_scales = tuple(a["loss_scales"])
        o = self._kitti_oracle(a, False)
        _require(np.array_equal(_np(chint), o["color_depth_hint"].astype(np.float32), equal_nan=True),
                 "%s: _kitti_fwd: color_depth_hint differs from oracle.kitti_loss" % self.current)
        for i, s in enumerate(loss_scales):
            _require(np.array_equal(_np(warped[i]), o["warped"][s].astype(np.float32), equal_nan=True),
                     "%s: _kitti_fwd: the warped colours of scale %d differ from oracle.kitti_loss" % (self.current, s))
        self._kitti_masks("%s: _kitti_fwd" % self.current, o, loss_scales, idsel, hpix)
        got = _np(terms)
        worst = 0.0
        for k, key in enumerate(okl.term_keys(loss_scales)):
            want = float(o[key])
            _require(np.isnan(got[k]) == np.isnan(want), "_kitti_fwd: %s is %r, want %r" % (key, got[k], want))
            if not np.isnan(want):
                worst = max(worst, float(_ulps(got[k], want)))
        n, _, H, W = a["t"]["target"].shape
        _record("_kitti_fwd", "fp64", "ulp+masks", worst, LOSS_MEAN_ULP, n * H * W * len(loss_scales))
        _require(worst <= LOSS_MEAN_ULP, "%s: _kitti_fwd term %.3g fp32 ulp > %d" % (self.current, worst, LOSS_MEAN_ULP))

    def _check_kitti_bwd(self, a, grads, pre):
        """oracle.kitti_loss.run (contract mode) with the call's grad_terms, on masks equal to the call's: each gradient
        element within KITTI_GRAD_ULP fp32 ulp of its scale's largest, NaN exactly where the oracle's are"""
        loss_scales = tuple(a["loss_scales"])
        o = self._kitti_oracle(a, True)
        self._kitti_masks("%s: _kitti_bwd" % self.current, o, loss_scales, a["idsel"], a["hpix"])
        worst = 0.0
        for i, s in enumerate(loss_scales):
            got, want = _np(grads[i]).astype(np.float64), o["grad"][s]
            nan = np.isnan(want)
            _require(np.array_equal(np.isnan(got), nan), "%s: _kitti_bwd scale %d: %d NaN gradients, want %d"
                     % (self.current, s, int(np.isnan(got).sum()), int(nan.sum())))
            if nan.all():
                continue
            scale = float(np.float32(np.abs(want[~nan]).max()))
            err = float(np.abs(got[~nan] - want[~nan]).max()) / max(scale * EPS, 1e-300)
            worst = max(worst, err)
            _require(err <= KITTI_GRAD_ULP, "%s: _kitti_bwd scale %d (%dx%d): %.3g fp32 ulp of the largest gradient > %d"
                     % (self.current, s, got.shape[2], got.shape[3], err, KITTI_GRAD_ULP))
        n, _, H, W = a["t"]["target"].shape
        _record("_kitti_bwd", "fp64", "ulp of largest", worst, KITTI_GRAD_ULP, n * H * W * len(loss_scales))

    # ------------------------------------------------------------------------------------------ NYUv2 evaluation
    def _before_NyuDepthEvaluator_add(self, a):
        ev = a["self"]
        return ev.next_frame, ev.sums.clone()

    def _check_NyuDepthEvaluator_add(self, a, res, pre):
        """oracle.nyu_eval.predict and frame_sums fed the evaluator's own gt / gt_log10: the map bit for bit, NaN pattern
        included; counts exact; the three sums within EVAL_REL relative plus NYU_SUM_ABS per pixel; other rows kept"""
        ev = a["self"]
        f0, old = pre
        disp = a["disp"]
        d = disp[:, 0] if disp.dim() == 4 and disp.shape[1] == 1 else disp
        n = int(d.shape[0])
        if n == 0:
            return
        _require(ev.next_frame == f0 + n, "NyuDepthEvaluator.add: next_frame %d, want %d" % (ev.next_frame, f0 + n))
        want_map = one.predict(_np(d), ev.use_224, ev.use_disparity)
        if a["depth_out"] is not None:
            dm = _np(a["depth_out"])
            _require(np.array_equal(dm, want_map, equal_nan=True),
                     "%s: NyuDepthEvaluator.add: %d prediction-map values differ from oracle.nyu_eval.predict"
                     % (self.current, int((~((dm == want_map) | (np.isnan(dm) & np.isnan(want_map)))).sum())))
        want = one.frame_sums(want_map, _np(ev.gt[f0:f0 + n]), _np(ev.gt_log10[f0:f0 + n]))
        got = _np(ev.sums[f0:f0 + n])
        _require(np.array_equal(got[:, 3:], want[:, 3:]), "%s: NyuDepthEvaluator.add: a_k / pixel counts %s, want %s"
                 % (self.current, got[:, 3:].tolist(), want[:, 3:].tolist()))
        err = _rel_err(got[:, :3], want[:, :3], "NyuDepthEvaluator.add sums", NYU_SUM_ABS * want[:, 6:7])
        rest = old.clone()
        rest[f0:f0 + n] = ev.sums[f0:f0 + n]
        _require(torch.equal(_bits(rest), _bits(ev.sums)), "NyuDepthEvaluator.add wrote rows outside its frames")
        mode = ("224" if ev.use_224 else "eigen") + ("/disparity" if ev.use_disparity else "")
        _record("NyuDepthEvaluator.add", "fp64", mode, err, EVAL_REL, n * want_map[0].size)
        _require(err <= EVAL_REL, "%s: NyuDepthEvaluator.add sums err %.3g > %.3g" % (self.current, err, EVAL_REL))

    def _check_compute_errors_nyu(self, a, out, pre):
        want = one.compute_errors_nyu(_np(a["pred"]), _np(a["gt"]))
        err = _rel_err(_np(out), want, "compute_errors_nyu")
        _record("compute_errors_nyu", "fp64", "-", err, EVAL_REL, a["pred"].numel())
        _require(err <= EVAL_REL, "%s: compute_errors_nyu err %.3g > %.3g" % (self.current, err, EVAL_REL))

    def _check_edt(self, a, out, pre):
        """each frame's distance map equals scipy's distance_transform_edt bit for bit"""
        f = _np(a["features"]) != 0
        got = _np(out)
        for i in range(f.shape[0]):
            _require(np.array_equal(got[i].view(np.int64), ne.edt(f[i]).view(np.int64)),
                     "%s: _edt frame %d (%dx%d) differs from scipy's distance transform" % (self.current, i, *f.shape[1:]))
        _record("_edt", "fp64", "-", 0.0, 0, f.size)

    def _check_edges_frames(self, a, res, pre):
        """oracle.nyu_edges.dbe per frame on the prediction rounded to fp32: edges and distance map bit for bit, scores
        within EVAL_REL relative, NaN and 10 exact"""
        edges_est, d_est = _np(res[0]), _np(res[1])
        p = _np(a["pred"]).astype(np.float32)
        g, scores = _np(a["edges_gt"]), _np(a["scores"])
        worst = 0.0
        for i in range(p.shape[0]):
            acc, comp, e, d = ne.dbe(g[i], p[i], a["low"], a["high"])
            _require(np.array_equal(edges_est[i] != 0, e), "%s: _edges_frames frame %d: %d edge pixels differ"
                     % (self.current, i, int(((edges_est[i] != 0) != e).sum())))
            _require(np.array_equal(d_est[i].view(np.int64), d.view(np.int64)),
                     "%s: _edges_frames frame %d: the distance map differs from scipy's" % (self.current, i))
            want = np.array([acc, comp])
            ten = want == ne.MAX_DIST
            _require(np.array_equal(scores[i][ten], want[ten]), "_edges_frames frame %d: score not exactly 10" % i)
            worst = max(worst, _rel_err(scores[i], want, "_edges_frames frame %d scores" % i))
        _record("_edges_frames", "fp64", "-", worst, EVAL_REL, p.size)
        _require(worst <= EVAL_REL, "%s: _edges_frames scores err %.3g > %.3g" % (self.current, worst, EVAL_REL))

    # ------------------------------------------------------------------------------------------ KITTI evaluation
    def _check_KittiDepthEvaluator_init(self, a, res, pre):
        """oracle.kitti_eval.valid_mask of each frame: frame sizes, offsets, the pixel list and the gathered ground
        truth exact"""
        ev = a["self"]
        frames = [(g.detach().cpu().numpy() if torch.is_tensor(g) else np.asarray(g)).astype(np.float32)
                  for g in a["gt_depths"]]
        hm, wm = ev.h_max, ev.w_max
        pixels, values, counts = [], [], [0]
        for i, g in enumerate(frames):
            ys, xs = np.nonzero(oke.valid_mask(g, a["eval_split"]))
            pixels.append(i * hm * wm + ys * wm + xs)
            values.append(g[ys, xs])
            counts.append(ys.size)
        off = np.cumsum(counts)
        total = int(off[-1])
        _require(np.array_equal(_np(ev.hw), np.array([g.shape for g in frames])), "KittiDepthEvaluator: frame sizes")
        _require(np.array_equal(_np(ev.offsets), off), "%s: KittiDepthEvaluator: valid counts %s, want %s"
                 % (self.current, np.diff(_np(ev.offsets)).tolist(), counts[1:]))
        _require(np.array_equal(_np(ev.pixels[:total]), np.concatenate(pixels)), "KittiDepthEvaluator: pixel list")
        _require(np.array_equal(_np(ev.gt[:total]), np.concatenate(values)), "KittiDepthEvaluator: gathered gt")
        _record("KittiDepthEvaluator.__init__", "-", a["eval_split"], 0.0, 0, total)

    def _before_KittiDepthEvaluator_add(self, a):
        ev = a["self"]
        return ev.next_frame, [t.clone() for t in (ev.errors, ev.ratios, ev.counts)]

    def _check_KittiDepthEvaluator_add(self, a, res, pre):
        """oracle.kitti_eval.evaluate_frame on each frame's ground truth (rebuilt from the split's checked valid pixels):
        counts, a1..a3 and the median ratio exact, the other metrics within EVAL_REL relative; other rows kept"""
        ev = a["self"]
        f0, old = pre
        d = a["pred_disp"]
        d = _np(d[:, 0] if d.dim() == 4 and d.shape[1] == 1 else d)
        n = d.shape[0]
        _require(ev.next_frame == f0 + n, "KittiDepthEvaluator.add: next_frame %d, want %d" % (ev.next_frame, f0 + n))
        hw, off, pix, gtv = _np(ev.hw), _np(ev.offsets), _np(ev.pixels), _np(ev.gt)
        errors, ratios, counts = _np(ev.errors), _np(ev.ratios), _np(ev.counts)
        split = ev.eval_split
        worst = 0.0
        for i in range(n):
            f = f0 + i
            g = np.zeros(tuple(hw[f]), np.float32)
            p = pix[off[f]:off[f + 1]].astype(np.int64) - f * ev.h_max * ev.w_max
            g[p // ev.w_max, p % ev.w_max] = gtv[off[f]:off[f + 1]]
            we, wr, wc = oke.evaluate_frame(g, d[i], split, ev.median_scaling, ev.pred_depth_scale_factor)
            _require(int(counts[f]) == wc, "%s: KittiDepthEvaluator.add frame %d: count %d, want %d"
                     % (self.current, f, counts[f], wc))
            _require(np.array_equal(errors[f, 4:], we[4:], equal_nan=True), "%s: KittiDepthEvaluator.add frame %d: "
                     "a1..a3 %s, want %s" % (self.current, f, errors[f, 4:].tolist(), we[4:].tolist()))
            _require(ratios[f] == wr or (np.isnan(ratios[f]) and np.isnan(wr)),
                     "%s: KittiDepthEvaluator.add frame %d: ratio %r, want %r" % (self.current, f, ratios[f], wr))
            worst = max(worst, _rel_err(errors[f, :4], we[:4], "KittiDepthEvaluator.add frame %d" % f))
        for t, o in zip((ev.errors, ev.ratios, ev.counts), old):
            rest = o.clone()
            rest[f0:f0 + n] = t[f0:f0 + n]
            _require(torch.equal(_bits(rest), _bits(t)), "KittiDepthEvaluator.add wrote rows outside its frames")
        mode = "%s/%s" % (split, "median" if ev.median_scaling else "x%g" % ev.pred_depth_scale_factor)
        _record("KittiDepthEvaluator.add", "fp64", mode, worst, EVAL_REL, int(off[f0 + n] - off[f0]))
        _require(worst <= EVAL_REL, "%s: KittiDepthEvaluator.add err %.3g > %.3g" % (self.current, worst, EVAL_REL))

    def _check_batch_post_process_disparity(self, a, out, pre):
        """the reference's numpy expression on the call's inputs, in their precision"""
        want = oke.batch_post_process_disparity(_np(a["l_disp"]), _np(a["r_disp"]))
        err = _rel_err(_np(out), want, "batch_post_process_disparity")
        _record("batch_post_process_disparity", "fp64", str(a["l_disp"].dtype).split(".")[-1], err, POST_REL, out.numel())
        _require(err <= POST_REL, "%s: batch_post_process_disparity err %.3g > %.3g" % (self.current, err, POST_REL))

    def _check_compute_errors(self, a, out, pre):
        want = np.array(oke.compute_errors(_np(a["gt"]).astype(np.float64), _np(a["pred"]).astype(np.float64)))
        err = _rel_err(_np(out), want, "compute_errors")
        _record("compute_errors", "fp64", "-", err, EVAL_REL, a["gt"].numel())
        _require(err <= EVAL_REL, "%s: compute_errors err %.3g > %.3g" % (self.current, err, EVAL_REL))

    # ------------------------------------------------------------------------------------------ KITTI depth hints
    def _check_stereo_sgbm(self, a, out, pre):
        """each frame equals oracle.sgbm.compute_side on the call's views and mirror flag, int16 bits, the borders the
        matcher never writes included"""
        left, right = _np(a["left"]), _np(a["right"])
        n, h, w, _ = left.shape
        _require(right.shape == left.shape, "stereo_sgbm: views of %s and %s" % (left.shape, right.shape))
        rev = np.zeros(n, bool)
        if a["reverse"] is not None:
            r = np.asarray(_np(a["reverse"]) if torch.is_tensor(a["reverse"]) else a["reverse"]).reshape(-1)
            _require(r.size == n and np.isin(r, (0, 1)).all(), "stereo_sgbm: reverse flags %s, want %d of 0 / 1"
                     % (r.tolist(), n))
            rev = r.astype(bool)
        nd, bs = a["num_disparities"], a["block_size"]
        got = _np(out)
        _require(got.dtype == np.int16 and got.shape == (n, h, w), "stereo_sgbm: map %s %s" % (got.dtype, got.shape))
        for i in range(n):
            want = osgbm.compute_side(left[i], right[i], nd, bs, bool(rev[i]))
            bad = int((got[i] != want).sum())
            _require(bad == 0, "%s: stereo_sgbm (%d, %d) frame %d (%dx%d%s): %d disparities differ from oracle.sgbm"
                     % (self.current, nd, bs, i, h, w, ", mirrored" if rev[i] else "", bad))
        _record("stereo_sgbm", "int16", "nd%d/bs%d" % (nd, bs), 0.0, 0, n * h * w)

    def _check_fuse(self, a, res, pre):
        """oracle.depth_hints.fuse (contract mode) on the launch's own views and maps: depth bits and index equal; the
        cameras are the generator's for each view's side"""
        base, lookup, maps = _np(a["base"]), _np(a["lookup"]), _np(a["maps"])
        n, h, w, _ = base.shape
        _require(lookup.shape == base.shape and maps.shape == (len(osgbm.MATCHERS), n, h, w),
                 "_fuse: views %s, %s and maps %s" % (base.shape, lookup.shape, maps.shape))
        right = _np(a["T"])[:, 0, 3] > 0
        for name, want in zip(("K", "inv_K", "T"), odh.cameras(h, w, right)):
            _require(np.array_equal(_np(a[name]).view(np.uint32), want.view(np.uint32)),
                     "_fuse: %s is not the generator's camera" % name)
        depth, index, _ = odh.fuse(base, lookup, maps, right, mode="contract")
        got = _np(a["depth"])
        bad = int((got.view(np.uint32) != depth.view(np.uint32)).sum())
        _require(bad == 0, "%s: _fuse (%d views of %dx%d): %d depths differ from oracle.depth_hints" % (self.current, n, h,
                                                                                                        w, bad))
        if a["index"] is not None:
            bad = int((_np(a["index"]) != index).sum())
            _require(bad == 0, "%s: _fuse: %d matcher indices differ from oracle.depth_hints" % (self.current, bad))
        _record("_fuse", "fp32", "contract" + ("+index" if a["index"] is not None else ""), 0.0, 0, n * h * w)

    # ------------------------------------------------------------------------------------------ training inputs
    def _check_KittiInputs__run(self, a, out, pre):
        """oracle.kitti_inputs.expected of each item of the call's host batch and draws: every key bit for bit (pyramid,
        flip, jitter order and factors, cameras, stereo_T, hints); disp_hint zero for an item without a hint"""
        fn, batch = a["self"], a["batch"]
        frames = fn.frame_idxs
        src, sizes = _np(batch["src"]), _np(batch["sizes"])
        n = len(batch["side"])
        _require(src.shape[0] == n * len(frames), "KittiInputs._run: %d views for %d items" % (src.shape[0], n))
        flip, aug = _np(batch["do_flip"]).astype(bool), _np(batch["do_color_aug"]).astype(bool)
        factors, order = _np(batch["factors"]), _np(batch["order"])
        hints = fn.use_depth_hints and "s" in frames
        _require(out["image_path"] == list(batch["image_path"]), "KittiInputs._run: image_path")
        for k in range(n):
            _require(aug[k] == (order[k, 0] >= 0), "KittiInputs._run: item %d do_color_aug %s with jitter order %s"
                     % (k, aug[k], order[k].tolist()))
            views = {}
            for fi, f in enumerate(frames):
                h, w = sizes[fi * n + k]
                views[f] = src[fi * n + k, :h, :w]
            params = (tuple(map(float, factors[k])), tuple(map(int, order[k]))) if aug[k] else None
            hint = None
            if hints and batch["hint_found"][k]:
                hh, hw = _np(batch["hint_size"])[k]
                hint = _np(batch["hint"])[k, :hh, :hw]
            want = oki.expected(views, (aug[k], flip[k], params), batch["side"][k], hint, fn.height, fn.width,
                                fn.scales, fn.use_depth_hints)
            extra = set(out) - set(want) - {"image_path"}
            _require(extra <= {"disp_hint"}, "KittiInputs._run: item %d has keys %s the reference does not" % (k, extra))
            for key in extra:
                _require(not _np(out[key][k]).any(), "KittiInputs._run: item %d's %s is not zero" % (k, key))
            for key, wv in want.items():
                _require(key in out, "KittiInputs._run: no %s" % (key,))
                g = _np(out[key][k])
                _require(g.dtype == wv.dtype and g.shape == wv.shape and g.tobytes() == wv.tobytes(),
                         "%s: KittiInputs._run item %d (%dx%d views, flip %d, jitter %s): %s differs from "
                         "oracle.kitti_inputs" % (self.current, k, *sizes[k], flip[k], params, key))
        mode = "%dx%d" % (fn.width, fn.height) + ("+hints" if hints else "")
        _record("KittiInputs._run", "u8/fp32", mode, 0.0, 0, len(src) * fn.height * fn.width)

    def _check_NyuInputs__run(self, a, out, pre):
        """oracle.nyu_inputs.expected of each item of the call's host batch and draws: image and depth bit for bit"""
        fn, batch = a["self"], a["batch"]
        image, depth, perm = _np(batch["image"]), _np(batch["depth"]), _np(batch["perm"])
        flip, gamma = _np(batch["flip"]).astype(bool), _np(batch["gamma"])
        for k in range(image.shape[0]):
            p = tuple(int(v) for v in perm[k])
            _require(p in oni.PERMS, "NyuInputs._run: item %d's channel order %s is not a permutation" % (k, p))
            want = oni.expected(image[k], depth[k], flip[k], oni.PERMS.index(p),
                                None if np.isnan(gamma[k]) else float(gamma[k]), fn.is_224, fn.resample)
            for key, wv in want.items():
                g = _np(out[key][k])
                _require(g.dtype == wv.dtype and g.shape == wv.shape and g.tobytes() == wv.tobytes(),
                         "%s: NyuInputs._run item %d (flip %d, perm %s, gamma %s): %s differs from oracle.nyu_inputs"
                         % (self.current, k, flip[k], p, gamma[k], key))
        mode = ("224" if fn.is_224 else "640") + "/" + fn.resample
        _record("NyuInputs._run", "u8/fp32", mode, 0.0, 0, out["image"].numel())

    # ------------------------------------------------------------------------------------------ KITTI ground truth
    def _check_generate_depth_maps(self, a, depth, pre):
        """oracle.kitti_gt.depth_map of each scan: the fp64 bits of its (H, W) map, and +0.0 everywhere past (H, W)"""
        pts = a["points"]
        pts = _np(pts) if torch.is_tensor(pts) else np.asarray(pts, np.float32)
        off = np.asarray(_np(a["offsets"]) if torch.is_tensor(a["offsets"]) else a["offsets"], np.int64).reshape(-1)
        P = np.asarray(_np(a["P"]) if torch.is_tensor(a["P"]) else a["P"], np.float64).reshape(-1, 3, 4)
        sizes = np.asarray(_np(a["sizes"]) if torch.is_tensor(a["sizes"]) else a["sizes"], np.int64).reshape(-1, 2)
        n = sizes.shape[0]
        _require(off.size == n + 1 and off[0] == 0 and off[-1] == pts.shape[0] and (np.diff(off) >= 0).all(),
                 "generate_depth_maps: offsets %s for %d scans of %d points" % (off.tolist(), n, pts.shape[0]))
        got = _np(depth)
        for i, (h, w) in enumerate(sizes):
            want = okg.depth_map(pts[off[i]:off[i + 1]], P[i], int(h), int(w), bool(a["vel_depth"]))
            bad = int((got[i, :h, :w].view(np.int64) != want.view(np.int64)).sum())
            _require(bad == 0, "%s: generate_depth_maps frame %d (%dx%d, %d points): %d depths differ from "
                     "oracle.kitti_gt" % (self.current, i, h, w, off[i + 1] - off[i], bad))
            pad = got[i].copy()
            pad[:h, :w] = 0
            _require(not pad.view(np.int64).any(), "%s: generate_depth_maps frame %d: written past its %dx%d"
                     % (self.current, i, h, w))
        _record("generate_depth_maps", "fp64", "vel_depth" if a["vel_depth"] else "camera", 0.0, 0, int(off[-1]))


def epilogue_ref(epi, out, disp):
    """The consumer epilogue planes in torch on a reconstruction and its disparity: disp_to_depth (KITTI/layers.py:16-25)
    -> [scaled_disp, depth], div_clamp (NYUv2/utils.py:219,229) -> [depth].  torch.clamp keeps a NaN."""
    if epi[0] == "disp_to_depth":
        lo, span = 1 / float(epi[2]), 1 / float(epi[1]) - 1 / float(epi[2])
        scaled = torch.tensor(lo, dtype=_f32, device=disp.device) + torch.tensor(span, dtype=_f32, device=disp.device) * disp
        return [scaled, 1 / scaled]
    v = out * (torch.tensor(1.0, dtype=_f32) / torch.tensor(float(epi[1]), dtype=_f32)).to(out.device)
    if epi[2] is not None:
        v = torch.clamp(v, min=float(epi[2]), max=float(epi[3]))
    return [v]


def level_masks_ref(yh, thresh, n, h, w, device):
    """The six pixel sets of wmd_level_masks in torch, uint8 (N, 1, H, W) / (N, 1, 2H, 2W): S0 = max_band |yh| > thresh (a
    NaN band or threshold sets no bit), S1 / S2 its 3x3 / 5x5 dilations, S5 = up2(S0), S4 / S3 up2(S0)'s 3x3 / 5x5
    dilations; thresh None: every S0 bit set."""
    if thresh is not None:
        s0 = yh.reshape(n, 3, h, w).abs().amax(1, keepdim=True) > thresh.reshape(n, 1, 1, 1)
    else:
        s0 = torch.ones((n, 1, h, w), dtype=torch.bool, device=device)
    f = s0.float()
    s5 = f.repeat_interleave(2, 2).repeat_interleave(2, 3)
    want = {"S0": f, "S1": F.max_pool2d(f, 3, 1, 1), "S2": F.max_pool2d(f, 5, 1, 2),
            "S5": s5, "S4": F.max_pool2d(s5, 3, 1, 1), "S3": F.max_pool2d(s5, 5, 1, 2)}
    return {k: v.to(torch.uint8) for k, v in want.items()}


def _np(t):
    return t.detach().cpu().numpy()


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int64) if t.dtype == torch.float64 else t


def _ulps(got, want):
    """|got - want| in units of the fp32 spacing at want"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def _rel_err(got, want, what, allow=0.0):
    """max over the elements of (|got - want| - allow) / |want|, after requiring the same NaN pattern and +-Inf exact"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    _require(np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN pattern %s, want %s" % (what, got, want))
    inf = np.isinf(want)
    _require(np.array_equal(got[inf], want[inf]), "%s: %s, want %s" % (what, got, want))
    f = np.isfinite(want)
    if not f.any():
        return 0.0
    allow = np.broadcast_to(np.asarray(allow, np.float64), want.shape)
    e = (np.abs(got[f] - want[f]) - allow[f]).clip(min=0) / np.maximum(np.abs(want[f]), 1e-300)
    return float(e.max())
