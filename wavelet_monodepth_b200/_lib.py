"""ctypes binding of libwmd.so (the C ABI declared in include/wmd.h).

There is deliberately NO fallback: if the shared library is missing or a call
fails, the product raises.  (The torch-CPU oracle under oracle/ is test
infrastructure and is never imported from here.)
"""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_longlong, c_size_t, c_void_p)

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libwmd.so")

PAD_ZERO, PAD_REFLECT, PAD_REPLICATE = 0, 1, 2
ACT_NONE, ACT_ELU, ACT_LRELU, ACT_SIGMOID = 0, 1, 2, 3
PAD_BY_NAME = {"zero": PAD_ZERO, "constant": PAD_ZERO, "reflect": PAD_REFLECT, "reflection": PAD_REFLECT,
               "replicate": PAD_REPLICATE}


class ConvDesc(Structure):
    """struct wmd_conv_desc (include/wmd.h)."""
    _fields_ = [
        ("N", c_int32), ("H", c_int32), ("W", c_int32),
        ("x0", c_void_p), ("c0", c_int32), ("ld0", c_int32),
        ("map0", c_void_p), ("shift0", c_int32),
        ("x1", c_void_p), ("c1", c_int32), ("ld1", c_int32),
        ("gate", c_void_p),
        ("w", c_void_p), ("bias", c_void_p),
        ("cout", c_int32), ("ldw", c_int32), ("taps", c_int32), ("pad_mode", c_int32),
        ("pixels", c_void_p), ("count", c_void_p), ("max_rows", c_int32),
        ("y", c_void_p), ("ldy", c_int32),
        ("act", c_int32), ("act_param", c_float),
        ("map1", c_void_p),
        ("precision", c_int32), ("amax0", c_void_p), ("amax1", c_void_p), ("amax_out", c_void_p),
        ("rows0", c_int32),
    ]


class HeadDesc(Structure):
    """struct wmd_head_desc (include/wmd.h)."""
    _fields_ = [
        ("N", c_int32), ("H", c_int32), ("W", c_int32),
        ("t", c_void_p), ("ld", c_int32), ("c", c_int32), ("off_a", c_int32), ("off_b", c_int32),
        ("map", c_void_p),
        ("wa", c_void_p), ("ba", c_void_p), ("wb", c_void_p), ("bb", c_void_p),
        ("cout", c_int32), ("pad_mode", c_int32), ("act", c_int32), ("scale", c_float),
        ("pixels", c_void_p), ("count", c_void_p), ("max_rows", c_int32),
        ("out", c_void_p),
    ]


class HeadIdwtDesc(Structure):
    """struct wmd_head_idwt_desc (include/wmd.h)."""
    _fields_ = [
        ("N", c_int32), ("H", c_int32), ("W", c_int32),
        ("z", c_void_p), ("ldz", c_int32),
        ("map", c_void_p), ("mask", c_void_p), ("bias", c_void_p),
        ("scale", c_float), ("pad_mode", c_int32),
        ("ll", c_void_p), ("yh", c_void_p), ("out", c_void_p), ("disp", c_void_p),
        ("disp_scale", c_float), ("clamp01", c_int32),
        ("epi_mode", c_int32), ("epi_a", c_float), ("epi_b", c_float), ("epi_lo", c_float), ("epi_hi", c_float),
        ("epi_out0", c_void_p), ("epi_out1", c_void_p),
        ("thresh", c_void_p), ("thresh_ratio", c_float),
    ]


EPI_NONE, EPI_DISP_TO_DEPTH, EPI_DIV_CLAMP = 0, 1, 2
PREC_TF32X3, PREC_F16X3 = 0, 1

# name -> (restype, argtypes); must list every symbol include/wmd.h declares (tests/test_abi.py checks)
SIGNATURES = {
    "wmd_version": (c_int, []),
    "wmd_status_string": (c_char_p, [c_int]),
    "wmd_last_cuda_error": (c_int, []),
    "wmd_launch_count": (c_longlong, []),
    "wmd_idwt_haar_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_int,
                                  c_int, c_void_p]),
    "wmd_idwt_haar_epi_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_float, c_float, c_float,
                                      c_float, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_idwt_bilinear_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_int, c_int, c_int,
                                      c_int, c_int, c_void_p]),
    "wmd_dwt_haar_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_range_ws_bytes": (c_size_t, [c_int, c_longlong]),
    "wmd_range_thresh_f32": (c_int, [c_void_p, c_int, c_longlong, c_float, c_void_p, c_void_p, c_void_p, c_size_t,
                                     c_void_p]),
    "wmd_level_masks": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_int, c_int, c_int, c_void_p]),
    "wmd_compact_ws_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wmd_compact_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t,
                                 c_void_p]),
    "wmd_gate_map": (c_int, [c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]),
    "wmd_nchw_to_rows_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p]),
    "wmd_nchw_to_rows_gated_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p]),
    "wmd_rows_to_nchw_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p]),
    "wmd_gather_rows_nchw_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_int, c_void_p]),
    "wmd_gather_rows_list_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_int, c_void_p]),
    "wmd_scatter_rows_nchw_f32": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                                          c_int, c_void_p]),
    "wmd_pack_conv_weight_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_head_mlp_supported": (c_int, [c_int, c_int]),
    "wmd_head_mlp_weight_floats": (c_size_t, [c_int, c_int]),
    "wmd_pack_head_mlp_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "wmd_head_mlp_f32": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_float, c_void_p, c_int, c_void_p, c_int,
                                 c_void_p]),
    "wmd_conv_rows_f32": (c_int, [POINTER(ConvDesc), c_void_p]),
    "wmd_conv_tc_tile_n": (c_int, [c_int]),
    "wmd_conv_tc16_weight_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wmd_pack_conv_weight_tc16_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_amax_f32": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p]),
    "wmd_amax_rows_masked_f32": (c_int, [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_void_p]),
    "wmd_nchw_to_rows_amax_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p, c_void_p]),
    "wmd_nchw_to_rows_masked_amax_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p,
                                                 c_void_p]),
    "wmd_nchw_to_rows_gated_amax_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_longlong, c_int, c_void_p, c_void_p]),
    "wmd_gather_rows_list_amax_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                              c_int, c_void_p, c_void_p]),
    "wmd_conv_tc_set_reserved_sms": (c_int, [c_int]),
    "wmd_conv_tc_weight_floats": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wmd_pack_conv_weight_tc_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_conv_rows_tc_f32": (c_int, [POINTER(ConvDesc), c_void_p]),
    "wmd_conv_tc_splitk_ws_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wmd_conv_rows_tc_splitk_f32": (c_int, [POINTER(ConvDesc), c_int, c_void_p, c_size_t, c_void_p]),
    "wmd_head_conv3x3_f32": (c_int, [POINTER(HeadDesc), c_void_p]),
    "wmd_head_idwt_ws_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wmd_head_idwt_f32": (c_int, [POINTER(HeadIdwtDesc), c_void_p, c_size_t, c_void_p]),
    "wmd_head_gather_f32": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_act_bwd_ws_bytes": (c_size_t, [c_int, c_int]),
    "wmd_act_bwd_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int, c_void_p,
                                c_void_p, c_void_p, c_size_t, c_void_p]),
    "wmd_conv_wgrad_ws_bytes": (c_size_t, [POINTER(ConvDesc)]),
    "wmd_conv_wgrad_f32": (c_int, [POINTER(ConvDesc), c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "wmd_conv_dgrad_fold_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                        c_void_p, c_void_p]),
    "wmd_pack_disp_tail16_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "wmd_disp_tail16_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
}
# include/wmd_eval.h: the KITTI evaluation entry points (tests/test_oracle_kitti_eval.py checks this table against it)
EVAL_SIGNATURES = {
    "wmd_eval_gt_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "wmd_eval_gather_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "wmd_eval_frames": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_int, c_int, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p]),
    "wmd_eval_errors_f64": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "wmd_post_process_disparity": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
}
EVAL_EIGEN, EVAL_GT_POSITIVE = 0, 1
DISP_TAIL16_PACKED_FLOATS = 5332          # WMD_DISP_TAIL16_PACKED_FLOATS

_lib = None


class WmdError(RuntimeError):
    pass


def load():
    """Load libwmd.so once; raises WmdError (never falls back) if it cannot be loaded."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise WmdError("%s is missing: build it with `python -m wavelet_monodepth_b200.build` "
                       "(or __graft_entry__.build()); there is no CPU/PyTorch fallback." % LIB_PATH)
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError:
        # libcudart.so.12 is normally already mapped by `import torch`; otherwise take the toolkit's copy
        for cand in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so.12"):
            try:
                ctypes.CDLL(cand, mode=ctypes.RTLD_GLOBAL)
                break
            except OSError:
                continue
        lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in list(SIGNATURES.items()) + list(EVAL_SIGNATURES.items()):
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        lib = load()
        msg = lib.wmd_status_string(rc).decode()
        raise WmdError("%s failed: %s (status %d, cudaError %d)" % (what, msg, rc, lib.wmd_last_cuda_error()))


def stream_ptr():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def host_ptr(t, dtype=None):
    """Pointer of a contiguous PINNED host tensor, for the one entry point that may read host memory in place
    (wmd_nchw_to_rows_gated_f32's src: page-locked memory is mapped into the device's address space under UVA, so a
    kernel reads it across PCIe at the same address).  Pageable memory is refused."""
    if t.is_cuda:
        return ptr(t, dtype)
    if not t.is_pinned():
        raise WmdError("host features must be pinned (page-locked) to be read by the device; got pageable memory")
    if dtype is not None and t.dtype != dtype:
        raise WmdError("expected dtype %s, got %s" % (dtype, t.dtype))
    if not t.is_contiguous():
        raise WmdError("expected a contiguous tensor")
    return t.data_ptr()


def ptr(t, dtype=None):
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise WmdError("libwmd operates on CUDA tensors only (got a %s tensor); there is no CPU path" % t.device)
    if dtype is not None and t.dtype != dtype:
        raise WmdError("expected dtype %s, got %s" % (dtype, t.dtype))
    if not t.is_contiguous():
        raise WmdError("expected a contiguous tensor")
    return t.data_ptr()


def launch_count():
    return int(load().wmd_launch_count())
