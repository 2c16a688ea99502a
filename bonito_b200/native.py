"""
ctypes binding of `libbonito_b200.so` (C ABI: include/bonito_b200.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C bonito_b200/csrc`.
There is no CPU fallback: if the library (or a CUDA device) is missing, the native
path raises -- see `require()`.
"""

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_longlong, c_size_t, c_void_p

import numpy as np
import torch

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libbonito_b200.so")
_lib = None

ACT_NONE, ACT_SWISH, ACT_TANH, ACT_CLAMP, ACT_SCALE, ACT_SWIGLU, ACT_TANH_SCALE, ACT_SWISH_CLAMP, ACT_RELU = 0, 1, 2, 3, 4, 5, 6, 7, 8
GEMM_AUTO, GEMM_TCGEN05, GEMM_MMA_SYNC = 0, 1, 2

MAX_LSTM_LAYERS = 8
LSTM_CHAINS = 4


class LstmCrfPlanStruct(ctypes.Structure):
    """`b200_lstm_crf_plan` of include/bonito_b200.h."""
    _fields_ = [("n", c_int), ("l", c_int), ("t", c_int), ("tp", c_int),
                ("c1", c_int), ("k1", c_int), ("act1", c_int), ("c2", c_int), ("k2", c_int), ("act2", c_int),
                ("hidden", c_int), ("k3", c_int), ("s3", c_int), ("pad3", c_int), ("act3", c_int),
                ("n_lstm", c_int), ("n_scores", c_int), ("act_l", c_int),
                ("lo", c_float), ("hi", c_float),
                ("reverse", c_int * MAX_LSTM_LAYERS),
                ("w1", c_void_p), ("b1", c_void_p), ("w2", c_void_p), ("b2", c_void_p), ("w3", c_void_p), ("b3", c_void_p),
                ("wl", c_void_p), ("bl", c_void_p),
                ("wih", c_void_p * MAX_LSTM_LAYERS), ("bias", c_void_p * MAX_LSTM_LAYERS), ("whh", c_void_p * MAX_LSTM_LAYERS),
                ("stem", c_void_p), ("ya", c_void_p), ("yb", c_void_p), ("gx", c_void_p), ("hx", c_void_p),
                ("chain_streams", c_void_p * (LSTM_CHAINS - 1))]


# name -> (restype, argtypes); must list every symbol declared in include/bonito_b200.h
SIGNATURES = {
    "b200_version": (c_int, []),
    "b200_last_error": (c_char_p, []),
    "b200_conv_stem_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                   c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "b200_conv_stem_fwd_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_float,
                                      c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_float, c_void_p, c_int, c_int,
                                      c_void_p]),
    "b200_gemm_fwd": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int,
                              c_int, c_float, c_float, c_int, c_int, c_longlong, c_longlong, c_int, c_void_p]),
    "b200_gemm_fwd_ex": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int,
                                 c_int, c_float, c_float, c_int, c_int, c_longlong, c_longlong, c_int, c_longlong, c_int, c_int,
                                 c_int, c_int, c_void_p]),
    "b200_conv_first_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                    c_int, c_void_p]),
    "b200_conv_first_fwd_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_float,
                                       c_void_p, c_longlong, c_int, c_int, c_void_p]),
    "b200_depthwise_conv_fwd": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int, c_int,
                                        c_void_p]),
    "b200_ctc_head_fwd": (c_int, [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_sw_align_workspace_bytes": (c_size_t, [c_int, c_int]),
    "b200_sw_align": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_pair_align_trace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b200_pair_align_workspace_bytes": (c_size_t, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_int]),
    "b200_pair_align": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "b200_rmsnorm_residual_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_void_p, c_longlong, c_int,
                                          c_void_p]),
    "b200_swiglu_fwd": (c_int, [c_void_p, c_void_p, c_longlong, c_int, c_void_p]),
    "b200_lstm_cluster_size": (c_int, [c_int]),
    "b200_lstm_rec_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b200_lstm_tile_chunks": (c_int, [c_int]),
    "b200_lstm_tile_cluster": (c_int, [c_int]),
    "b200_lstm_rec_tile_workspace_bytes": (c_size_t, [c_int]),
    "b200_lstm_rec_tile_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b200_lstm_fused_tile_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_int, c_void_p]),
    "b200_lstm_wide_ctas": (c_int, [c_int]),
    "b200_lstm_wide_max_chunks": (c_int, [c_int]),
    "b200_lstm_wide_resident": (c_int, [c_int]),
    "b200_lstm_rec_wide_workspace_bytes": (c_size_t, [c_int, c_int]),
    "b200_lstm_rec_wide_status_offset": (c_size_t, [c_int, c_int]),
    "b200_lstm_rec_wide_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b200_crf_decode_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_quantize_i8": (c_int, [c_void_p, c_void_p, c_longlong, c_float, c_void_p]),
    "b200_stream_create": (c_int, [c_void_p]),
    "b200_chunk_count": (c_int, [c_longlong, c_int, c_int]),
    "b200_chunk_signal": (c_int, [c_void_p, c_int, c_longlong, c_int, c_int, c_void_p, c_longlong, c_void_p]),
    "b200_gemm_i8_fwd": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int,
                                 c_int, c_float, c_float, c_int, c_int, c_longlong, c_longlong, c_int, c_longlong, c_int, c_int,
                                 c_int, c_void_p]),
    "b200_lstm_crf_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_lstm_crf_lstm_fwd": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "b200_crf_beam_search": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_int, c_float, c_float, c_float,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_crf_decode": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_float, c_float,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_crf_decode_lb": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_float,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_crf_sparse_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b200_ctc_crf_sparse_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_crf_sparse_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_ctc_crf_sparse_grad": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_crf_target_max_states": (c_int, []),
    "b200_ctc_crf_target_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b200_ctc_crf_target_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                        c_void_p]),
    "b200_ctc_crf_target_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p]),
    "b200_ctc_loss_max_target": (c_int, []),
    "b200_ctc_loss_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_ctc_loss_fwd": (c_int, [c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_void_p, c_void_p, c_longlong,
                                  c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_loss_grad": (c_int, [c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_void_p, c_void_p, c_longlong,
                                   c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_beam_workspace_bytes": (c_size_t, [c_int, c_longlong, c_int]),
    "b200_ctc_beam_search": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_float, c_void_p, c_size_t,
                                     c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_wgrad_gemm_workspace_bytes": (c_size_t, [c_longlong, c_int, c_int]),
    "b200_wgrad_gemm": (c_int, [c_void_p, c_longlong, c_longlong, c_void_p, c_longlong, c_longlong, c_int, c_int, c_int, c_int,
                                c_void_p, c_void_p, c_void_p]),
    "b200_depthwise_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b200_depthwise_wgrad": (c_int, [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p]),
    "b200_conv_first_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b200_conv_first_wgrad": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "b200_bn_stats_workspace_bytes": (c_size_t, [c_longlong, c_int]),
    "b200_bn_stats": (c_int, [c_void_p, c_longlong, c_longlong, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_void_p]),
    "b200_bn_act_fwd": (c_int, [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p]),
    "b200_bn_act_bwd_workspace_bytes": (c_size_t, [c_longlong, c_int]),
    "b200_bn_act_bwd": (c_int, [c_void_p, c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p]),
    "b200_ctc_head_train_fwd": (c_int, [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_ctc_head_bwd_workspace_bytes": (c_size_t, [c_longlong, c_int]),
    "b200_ctc_head_bwd": (c_int, [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "b200_map_minimizers": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_map_anchors": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_int, c_void_p, c_longlong, c_void_p, c_void_p,
                                 c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_map_chain": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200_map_extract": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200_map_align_trace_bytes": (c_size_t, [c_int, c_int]),
    "b200_map_align": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_void_p]),
    "b200_bgzf_workspace_bytes": (c_size_t, [c_longlong]),
    "b200_bgzf_compress": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b200_bgzf_decompress": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_void_p, c_longlong, c_void_p, c_void_p]),
    "b200_zstd_decompress": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_void_p, c_longlong, c_void_p, c_void_p,
                                     c_void_p]),
    "b200_svb16_decode": (c_int, [c_void_p, c_longlong, c_void_p, c_int, c_void_p, c_longlong, c_void_p, c_void_p]),
}

BGZF_MEMBER_INPUT = 65280   # B200_BGZF_MEMBER_INPUT
BGZF_MEMBER_MAX = 65536     # output bytes per member at most
# B200_INFLATE_* status codes of b200_bgzf_decompress
INFLATE_STATUS = {1: "block type 3", 2: "stored block LEN is not the complement of NLEN",
                  3: "invalid Huffman code lengths", 4: "invalid code-length repeat",
                  5: "invalid literal/length or distance code", 6: "distance reaches before the member's first byte",
                  7: "output longer than ISIZE", 8: "output shorter than ISIZE", 9: "DEFLATE data ends before the final block",
                  10: "CRC32 mismatch", 11: "member outside the launch's buffers"}


class BnActStruct(ctypes.Structure):
    """`b200_bn_act` of include/bonito_b200.h."""
    _fields_ = [("m", c_longlong), ("c", c_int), ("t", c_int), ("act", c_int), ("p", c_float), ("seed", ctypes.c_ulonglong),
                ("unit", c_int), ("z", c_void_p), ("ldz", c_longlong), ("mean", c_void_p), ("invstd", c_void_p),
                ("gamma", c_void_p), ("beta", c_void_p), ("zr", c_void_p), ("ldzr", c_longlong), ("mean_r", c_void_p),
                ("invstd_r", c_void_p), ("gamma_r", c_void_p), ("beta_r", c_void_p), ("mask", c_void_p)]


class NativeError(RuntimeError):
    pass


def lib_path():
    return _LIB_PATH


def load():
    """Load the shared library (no CUDA calls are made by loading it)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise NativeError(
                f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C bonito_b200/csrc` (there is no CPU fallback for the native path)")
        lib = ctypes.CDLL(_LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = lib
    return _lib


def require(device=None):
    """Library + CUDA device, or a loud failure."""
    lib = load()
    if not torch.cuda.is_available():
        raise NativeError("bonito_b200 native path needs a CUDA device (sm_90a); none is visible")
    return lib


def _check(rc, what):
    if rc != 0:
        msg = load().b200_last_error().decode(errors="replace")
        raise NativeError(f"{what} failed ({rc}): {msg}")


def _ptr(t):
    return None if t is None else c_void_p(t.data_ptr())


def _stream(stream=None):
    """cudaStream_t for the C ABI: an explicit torch stream, or the current one."""
    return c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def _f16(t, name):
    if t.dtype != torch.float16 or not t.is_cuda or not t.is_contiguous():
        raise NativeError(f"{name}: expected a contiguous CUDA fp16 tensor, got {t.dtype} {t.device}")
    return t


def version():
    return load().b200_version()


def conv_stem(x, w1, b1, act1, w2, b2, act2, out, lp, padl, bounds=None):
    """x [N,L] -> out [N,lp,C2] channels-last, zero padded (see b200_conv_stem_fwd).  `bounds=(lo1, hi1, lo2, hi2)`: the
    bounds of act1 / act2 (B200_ACT_SWISH_CLAMP), through b200_conv_stem_fwd_ex."""
    lib = require()
    n, l = x.shape
    c1, _, k1 = w1.shape
    c2, _, k2 = w2.shape
    with torch.cuda.device(x.device):
        if bounds is None:
            rc = lib.b200_conv_stem_fwd(_ptr(_f16(x, "x")), n, l, c1, k1, _ptr(_f16(w1, "w1")), _ptr(b1), act1,
                                        c2, k2, _ptr(_f16(w2, "w2")), _ptr(b2), act2, _ptr(out), lp, padl, _stream())
        else:
            lo1, hi1, lo2, hi2 = (float(v) for v in bounds)
            rc = lib.b200_conv_stem_fwd_ex(_ptr(_f16(x, "x")), n, l, c1, k1, _ptr(_f16(w1, "w1")), _ptr(b1), act1, lo1, hi1,
                                           c2, k2, _ptr(_f16(w2, "w2")), _ptr(b2), act2, lo2, hi2, _ptr(out), lp, padl,
                                           _stream())
    _check(rc, "b200_conv_stem_fwd")
    return out


def gemm(a_ptr_tensor, lda, b, bias, c, ldc, m, n, k, act=ACT_NONE, lo=0.0, hi=0.0,
         rows_inner=None, valid_inner=None, stride_inner=1, stride_outer=0, impl=GEMM_AUTO, stream=None, max_ctas=0,
         cb_width=0, cb_rows=0, group=0, stride_group=0):
    """C = act(A B^T + bias); `a_ptr_tensor` / `c` only supply base pointers (rows may overlap / be remapped; `cb_*`:
    column blocks, see b200_gemm_fwd_ex)."""
    lib = require()
    if rows_inner is None:
        rows_inner, valid_inner = m, m
    with torch.cuda.device(c.device):
        rc = lib.b200_gemm_fwd_ex(_ptr(a_ptr_tensor), lda, _ptr(_f16(b, "b")), _ptr(bias), _ptr(c), ldc, m, n, k,
                                  act, float(lo), float(hi), rows_inner, valid_inner, stride_inner, stride_outer,
                                  int(group), int(stride_group), int(cb_width), int(cb_rows), impl, int(max_ctas),
                                  _stream(stream))
    _check(rc, "b200_gemm_fwd")
    return c


def conv_first(x, w, bias, act, out, lp, padl, stream=None):
    """x [N,L] -> out [N,lp,C] channels-last with zero halo (see b200_conv_first_fwd)."""
    lib = require()
    n, l = x.shape
    c, _, k = w.shape
    with torch.cuda.device(out.device):
        rc = lib.b200_conv_first_fwd(_ptr(_f16(x, "x")), n, l, c, k, _ptr(_f16(w, "w")), _ptr(bias), act, _ptr(out), lp,
                                     padl, _stream(stream))
    _check(rc, "b200_conv_first_fwd")
    return out


def conv_first_ex(x, w, bias, act, out, ldo, lp, padl, stride=1, lo=0.0, hi=0.0, stream=None):
    """x [N,L] -> rows n*lp + padl + t (t < (L-1)//stride + 1) of `out`, pitch `ldo` elements (see b200_conv_first_fwd_ex);
    `out` only supplies the base pointer, so it may be a column offset into a wider buffer."""
    lib = require()
    n, l = x.shape
    c, _, k = w.shape
    with torch.cuda.device(x.device):
        rc = lib.b200_conv_first_fwd_ex(_ptr(_f16(x, "x")), n, l, c, k, int(stride), _ptr(_f16(w, "w")), _ptr(bias), act,
                                        float(lo), float(hi), _ptr(out), int(ldo), lp, padl, _stream(stream))
    _check(rc, "b200_conv_first_fwd_ex")
    return out


def depthwise_conv(x, ldx, w, y, ldy, n, t, stream=None):
    """Depthwise Conv1d over n chunks of t channels-last rows (see b200_depthwise_conv_fwd); w [C, 1, K]; `x` / `y` only
    supply base pointers (column ranges of wider buffers with pitches ldx / ldy)."""
    lib = require()
    c, _, k = w.shape
    with torch.cuda.device(y.device):
        rc = lib.b200_depthwise_conv_fwd(_ptr(x), int(ldx), _ptr(_f16(w, "w")), _ptr(y), int(ldy), int(n), int(t), c, k,
                                         _stream(stream))
    _check(rc, "b200_depthwise_conv_fwd")
    return y


def ctc_head(x, m, w, bias, labels, probs, logp=None, stream=None):
    """x [m, F] -> labels uint8 [m], probs fp32 [m] and, when given, logp fp16 [m, 5] (see b200_ctc_head_fwd)."""
    lib = require()
    f = w.shape[-1]
    with torch.cuda.device(labels.device):
        rc = lib.b200_ctc_head_fwd(_ptr(_f16(x, "x")), int(m), f, _ptr(_f16(w, "w")), _ptr(bias), _ptr(logp), _ptr(labels),
                                   _ptr(probs), _stream(stream))
    _check(rc, "b200_ctc_head_fwd")
    return labels, probs


def sw_align_workspace_bytes(n_pairs, max_ref_len):
    return load().b200_sw_align_workspace_bytes(int(n_pairs), int(max_ref_len))


def sw_align(query, query_off, query_len, ref, ref_off, ref_len, workspace, out, stream=None):
    """Batched Smith-Waterman (see b200_sw_align): query / ref packed CUDA uint8 buffers; query_off / ref_off CPU int64 and
    query_len / ref_len CPU int32 tensors of n_pairs entries; workspace CUDA uint8 of sw_align_workspace_bytes(n_pairs,
    max(ref_len)) bytes; out CUDA int32 [n_pairs, 7]."""
    lib = require()
    n = query_len.numel()
    for t, dtype, name in ((query_off, torch.int64, "query_off"), (ref_off, torch.int64, "ref_off"),
                           (query_len, torch.int32, "query_len"), (ref_len, torch.int32, "ref_len")):
        if t.is_cuda or t.dtype != dtype or not t.is_contiguous() or t.numel() != n:
            raise NativeError(f"sw_align: {name} must be a contiguous host {dtype} tensor of {n} entries")
    for t, dtype, name in ((query, torch.uint8, "query"), (ref, torch.uint8, "ref"), (workspace, torch.uint8, "workspace"),
                           (out, torch.int32, "out")):
        if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
            raise NativeError(f"sw_align: {name} must be a contiguous CUDA {dtype} tensor")
    if out.shape != (n, 7):
        raise NativeError(f"sw_align: out must have shape ({n}, 7), got {tuple(out.shape)}")
    with torch.cuda.device(out.device):
        rc = lib.b200_sw_align(_ptr(query), _ptr(query_off), _ptr(query_len), _ptr(ref), _ptr(ref_off), _ptr(ref_len), n,
                               _ptr(workspace), _ptr(out), _stream(stream))
    _check(rc, "b200_sw_align")
    return out


PAIR_GLOBAL_EDIT, PAIR_SEMIGLOBAL_AFFINE = 0, 1


def _host_i32(a, n, name):
    """A contiguous int32 numpy copy of `n` entries (the per-pair host arrays of b200_pair_align)."""
    a = np.ascontiguousarray(a, dtype=np.int32)
    if a.shape != (n,):
        raise NativeError(f"pair_align: {name} must have {n} entries, got shape {a.shape}")
    return a


def pair_align_trace_bytes(mode, query_len, ref_len, band=0):
    return load().b200_pair_align_trace_bytes(int(mode), int(query_len), int(ref_len), int(band))


def pair_align_workspace_bytes(mode, query_len, ref_len, band=None, traceback=True):
    n = len(query_len)
    ql, rl = _host_i32(query_len, n, "query_len"), _host_i32(ref_len, n, "ref_len")
    bd = None if band is None else _host_i32(band, n, "band")
    return load().b200_pair_align_workspace_bytes(int(mode), n, ql.ctypes.data, rl.ctypes.data,
                                                  None if bd is None else bd.ctypes.data, int(bool(traceback)))


def pair_align(mode, query, query_off, query_len, ref, ref_off, ref_len, band, workspace, out, ops=None, ops_off=None,
               traceback=True, stream=None):
    """Batched banded edit / semi-global affine alignment (see b200_pair_align): query / ref / ops / workspace CUDA uint8
    buffers, out CUDA int32 [n, 2]; query_off / ref_off / ops_off int64 and query_len / ref_len / band int32 host numpy
    arrays (copied into the workspace on `stream` before this returns)."""
    lib = require()
    n = len(query_len)
    q_off, r_off = (np.ascontiguousarray(a, dtype=np.int64) for a in (query_off, ref_off))
    ql, rl = _host_i32(query_len, n, "query_len"), _host_i32(ref_len, n, "ref_len")
    bd = None if band is None else _host_i32(band, n, "band")
    o_off = None if ops_off is None else np.ascontiguousarray(ops_off, dtype=np.int64)
    for a, name in ((q_off, "query_off"), (r_off, "ref_off"), (o_off, "ops_off")):
        if a is not None and a.shape != (n,):
            raise NativeError(f"pair_align: {name} must have {n} entries")
    for t, dtype, name in ((query, torch.uint8, "query"), (ref, torch.uint8, "ref"), (workspace, torch.uint8, "workspace"),
                           (out, torch.int32, "out"), (ops, torch.uint8, "ops")):
        if t is not None and (not t.is_cuda or t.dtype != dtype or not t.is_contiguous()):
            raise NativeError(f"pair_align: {name} must be a contiguous CUDA {dtype} tensor")
    if out.shape != (n, 2):
        raise NativeError(f"pair_align: out must have shape ({n}, 2), got {tuple(out.shape)}")
    need = pair_align_workspace_bytes(mode, ql, rl, bd, traceback)
    if workspace.numel() < need:
        raise NativeError(f"pair_align: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(out.device):
        rc = lib.b200_pair_align(int(mode), _ptr(query), q_off.ctypes.data, ql.ctypes.data, _ptr(ref), r_off.ctypes.data,
                                 rl.ctypes.data, None if bd is None else bd.ctypes.data, n, int(bool(traceback)),
                                 _ptr(workspace), _ptr(ops), None if o_off is None else o_off.ctypes.data, _ptr(out),
                                 _stream(stream))
    _check(rc, "b200_pair_align")
    return out


def attention(qkv, cos_sin, out, n, t, heads, head_dim, wl, wr, stream=None):
    lib = require()
    with torch.cuda.device(out.device):
        rc = lib.b200_attention_fwd(_ptr(_f16(qkv, "qkv")), _ptr(_f16(cos_sin, "cos_sin")), _ptr(out), n, t, heads,
                                    head_dim, wl, wr, _stream(stream))
    _check(rc, "b200_attention_fwd")
    return out


def rmsnorm_residual(a, x, w, alpha, eps, out, m, d, stream=None):
    lib = require()
    with torch.cuda.device(out.device):
        rc = lib.b200_rmsnorm_residual_fwd(_ptr(_f16(a, "a")), _ptr(_f16(x, "x")), _ptr(_f16(w, "w")), float(alpha),
                                           float(eps), _ptr(out), m, d, _stream(stream))
    _check(rc, "b200_rmsnorm_residual_fwd")
    return out


def swiglu(h, out, m, f, stream=None):
    lib = require()
    with torch.cuda.device(out.device):
        rc = lib.b200_swiglu_fwd(_ptr(_f16(h, "h")), _ptr(out), m, f, _stream(stream))
    _check(rc, "b200_swiglu_fwd")
    return out


def lstm_cluster_size(hidden):
    return load().b200_lstm_cluster_size(hidden)


def lstm_rec(gx, whh, y, t, n, hidden, reverse, stream=None):
    lib = require()
    with torch.cuda.device(y.device):
        rc = lib.b200_lstm_rec_fwd(_ptr(gx), _ptr(_f16(whh, "whh")), _ptr(y), t, n, hidden,
                                   int(bool(reverse)), _stream(stream))
    _check(rc, "b200_lstm_rec_fwd")
    return y


def lstm_tile_chunks(hidden):
    """Chunks per tile of the tile-layout recurrent kernel (0: this hidden size only has the generic-layout kernel)."""
    return load().b200_lstm_tile_chunks(hidden)


def lstm_tile_cluster(hidden):
    return load().b200_lstm_tile_cluster(hidden)


def lstm_rec_tile_workspace_bytes(n):
    return load().b200_lstm_rec_tile_workspace_bytes(n)


def lstm_rec_tile(gx, whh, y, t, n, hidden, reverse, stream=None, workspace=None):
    """gx [tiles][T][8][64][192], y [tiles][T][64][H] (see b200_lstm_rec_tile_fwd); n chunks = ceil(n/64) tiles.
    `workspace`: uint8 tensor of lstm_rec_tile_workspace_bytes(n) bytes (allocated here when omitted)."""
    lib = require()
    if workspace is None:
        workspace = torch.empty(lstm_rec_tile_workspace_bytes(n), dtype=torch.uint8, device=y.device)
    with torch.cuda.device(y.device):
        rc = lib.b200_lstm_rec_tile_fwd(_ptr(gx), _ptr(_f16(whh, "whh")), _ptr(y), _ptr(workspace), t, n, hidden,
                                        int(bool(reverse)), _stream(stream))
    _check(rc, "b200_lstm_rec_tile_fwd")
    return y


def lstm_fused_tile(x, wih, bias, whh, y, t, n, hidden, reverse, stream=None, workspace=None):
    """One whole fp16 LSTM layer in the tile layout, input projection included: x, y [tiles][T][64][H]; wih / bias in gx
    column order, whh in W_hh row order (see b200_lstm_fused_tile_fwd).  `workspace`: uint8 tensor of
    lstm_rec_tile_workspace_bytes(n) bytes (allocated here when omitted)."""
    lib = require()
    if workspace is None:
        workspace = torch.empty(lstm_rec_tile_workspace_bytes(n), dtype=torch.uint8, device=y.device)
    with torch.cuda.device(y.device):
        rc = lib.b200_lstm_fused_tile_fwd(_ptr(x), _ptr(_f16(wih, "wih")), _ptr(_f16(bias, "bias")), _ptr(_f16(whh, "whh")),
                                          _ptr(y), _ptr(workspace), t, n, hidden, int(bool(reverse)), _stream(stream))
    _check(rc, "b200_lstm_fused_tile_fwd")
    return y


def lstm_wide_ctas(hidden):
    """CTAs of the wide recurrent kernel (hidden / 8; 0: this hidden size has no wide kernel)."""
    return load().b200_lstm_wide_ctas(hidden)


def lstm_wide_max_chunks(hidden):
    return load().b200_lstm_wide_max_chunks(hidden)


def lstm_wide_resident(hidden, device=None):
    """CTAs of the wide kernel that fit on the device at once (the grid needs lstm_wide_ctas(hidden) of them)."""
    lib = require()
    with torch.cuda.device(device if device is not None else torch.cuda.current_device()):
        rc = lib.b200_lstm_wide_resident(hidden)
    if rc < 0:
        _check(rc, "b200_lstm_wide_resident")
    return rc


def lstm_rec_wide_workspace_bytes(n, hidden):
    return load().b200_lstm_rec_wide_workspace_bytes(n, hidden)


def lstm_rec_wide_status_offset(n, hidden):
    return load().b200_lstm_rec_wide_status_offset(n, hidden)


def lstm_rec_wide(gx, whh, y, t, n, hidden, reverse, stream=None, workspace=None):
    """gx [T][G][n][32], y [T][n][H] (see b200_lstm_rec_wide_fwd).  `workspace`: uint8 tensor of
    lstm_rec_wide_workspace_bytes(n, hidden) bytes (allocated here when omitted); its status word is not checked here."""
    lib = require()
    if workspace is None:
        workspace = torch.empty(lstm_rec_wide_workspace_bytes(n, hidden), dtype=torch.uint8, device=y.device)
    with torch.cuda.device(y.device):
        rc = lib.b200_lstm_rec_wide_fwd(_ptr(gx), _ptr(_f16(whh, "whh")), _ptr(y), _ptr(workspace), t, n, hidden,
                                        int(bool(reverse)), _stream(stream))
    _check(rc, "b200_lstm_rec_wide_fwd")
    return y


def crf_decode_workspace_bytes(n, t, state_len):
    return load().b200_crf_decode_workspace_bytes(n, t, state_len)


def crf_decode(scores, state_len, blank_score, qscale, qbias, workspace, moves, sequence, qstring, stream=None):
    lib = require()
    n, t, _ = scores.shape
    with torch.cuda.device(scores.device):
        rc = lib.b200_crf_decode(_ptr(scores), n, t, state_len, float(blank_score), float(qscale),
                                 float(qbias), _ptr(workspace), _ptr(moves), _ptr(sequence), _ptr(qstring),
                                 _stream(stream))
    _check(rc, "b200_crf_decode")
    return moves, sequence, qstring


def crf_decode_lb(scores, state_len, qscale, qbias, workspace, moves, sequence, qstring, stream=None):
    """Learned-blank decode (see b200_crf_decode_lb): scores [N, T, 5 * 4**state_len] in the [state][stay, m0..m3] layout;
    workspace of crf_decode_workspace_bytes(N, T, state_len) bytes."""
    lib = require()
    n, t, _ = scores.shape
    with torch.cuda.device(scores.device):
        rc = lib.b200_crf_decode_lb(_ptr(scores), n, t, state_len, float(qscale), float(qbias), _ptr(workspace), _ptr(moves),
                                    _ptr(sequence), _ptr(qstring), _stream(stream))
    _check(rc, "b200_crf_decode_lb")
    return moves, sequence, qstring


def crf_beam_search(scores, state_len, blank_score, beam_width, beam_cut, qscale, qbias, workspace, moves, sequence, qstring,
                    stream=None):
    lib = require()
    n, t, _ = scores.shape
    with torch.cuda.device(scores.device):
        rc = lib.b200_crf_beam_search(_ptr(scores), n, t, state_len, float(blank_score), int(beam_width), float(beam_cut),
                                      float(qscale), float(qbias), _ptr(workspace), _ptr(moves), _ptr(sequence),
                                      _ptr(qstring), _stream(stream))
    _check(rc, "b200_crf_beam_search")
    return moves, sequence, qstring


SEMIRING_LOG, SEMIRING_MAX = 0, 1


def _dev(t, dtype, name, what, shape=None):
    """A contiguous CUDA tensor of `dtype` (and `shape`), or NativeError."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        got = f"{t.dtype} {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
        raise NativeError(f"{what}: {name} must be a contiguous CUDA {dtype} tensor, got {got}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise NativeError(f"{what}: {name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
    return t


def _semiring(semiring, what):
    if semiring not in (SEMIRING_LOG, SEMIRING_MAX):
        raise NativeError(f"{what}: unknown semiring {semiring!r}")
    return semiring


def _sparse_shape(scores, state_len, what):
    _dev(scores, torch.float32, "scores", what)
    if scores.dim() != 3 or scores.shape[2] != 5 * 4 ** state_len:
        raise NativeError(f"{what}: scores must be [T, N, {5 * 4 ** state_len}] for state_len {state_len}, "
                          f"got {tuple(scores.shape)}")
    if scores.data_ptr() % 16:
        raise NativeError(f"{what}: scores must be 16-byte aligned")
    t, n, _ = scores.shape
    return t, n


def ctc_crf_sparse_workspace_bytes(n, t, state_len, semiring):
    return load().b200_ctc_crf_sparse_workspace_bytes(int(n), int(t), int(state_len), int(semiring))


def ctc_crf_sparse_fwd(scores, state_len, semiring, logz, alpha=None, workspace=None, stream=None):
    """k-mer lattice forward (see b200_ctc_crf_sparse_fwd): scores [T, N, 5*4**state_len] fp32 -> logz [N]; alpha
    [T+1, N, S] when given; `workspace` (uint8, ctc_crf_sparse_workspace_bytes bytes) keeps what ctc_crf_sparse_grad needs."""
    lib = require()
    what = "ctc_crf_sparse_fwd"
    t, n = _sparse_shape(scores, state_len, what)
    _dev(logz, torch.float32, "logz", what, (n,))
    if alpha is not None:
        _dev(alpha, torch.float32, "alpha", what, (t + 1, n, 4 ** state_len))
    if workspace is not None:
        _dev(workspace, torch.uint8, "workspace", what)
        need = ctc_crf_sparse_workspace_bytes(n, t, state_len, semiring)
        if workspace.numel() < need:
            raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(scores.device):
        rc = lib.b200_ctc_crf_sparse_fwd(_ptr(scores), t, n, int(state_len), _semiring(semiring, what), _ptr(logz),
                                         _ptr(alpha), _ptr(workspace), _stream(stream))
    _check(rc, "b200_ctc_crf_sparse_fwd")
    return logz


def ctc_crf_sparse_bwd(scores, state_len, semiring, beta, stream=None):
    """k-mer lattice backward scores beta [T+1, N, S] (see b200_ctc_crf_sparse_bwd)."""
    lib = require()
    what = "ctc_crf_sparse_bwd"
    t, n = _sparse_shape(scores, state_len, what)
    _dev(beta, torch.float32, "beta", what, (t + 1, n, 4 ** state_len))
    with torch.cuda.device(scores.device):
        rc = lib.b200_ctc_crf_sparse_bwd(_ptr(scores), t, n, int(state_len), _semiring(semiring, what), _ptr(beta),
                                         _stream(stream))
    _check(rc, "b200_ctc_crf_sparse_bwd")
    return beta


def ctc_crf_sparse_grad(scores, state_len, semiring, g, workspace, grad, stream=None):
    """grad [T, N, C] = g[n] * dlogz[n]/dscores from the workspace of ctc_crf_sparse_fwd (see b200_ctc_crf_sparse_grad)."""
    lib = require()
    what = "ctc_crf_sparse_grad"
    t, n = _sparse_shape(scores, state_len, what)
    _dev(g, torch.float32, "g", what, (n,))
    _dev(grad, torch.float32, "grad", what, tuple(scores.shape))
    _dev(workspace, torch.uint8, "workspace", what)
    need = ctc_crf_sparse_workspace_bytes(n, t, state_len, semiring)
    if workspace.numel() < need:
        raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(scores.device):
        rc = lib.b200_ctc_crf_sparse_grad(_ptr(scores), t, n, int(state_len), _semiring(semiring, what), _ptr(g),
                                          _ptr(workspace), _ptr(grad), _stream(stream))
    _check(rc, "b200_ctc_crf_sparse_grad")
    return grad


def ctc_crf_target_max_states():
    return load().b200_ctc_crf_target_max_states()


def ctc_crf_target_workspace_bytes(n, t, l, semiring):
    return load().b200_ctc_crf_target_workspace_bytes(int(n), int(t), int(l), int(semiring))


def _target_shape(stay, move, lengths, what):
    _dev(stay, torch.float32, "stay", what)
    if stay.dim() != 3:
        raise NativeError(f"{what}: stay must be [T, N, L], got {tuple(stay.shape)}")
    t, n, l = stay.shape
    _dev(move, torch.float32, "move", what, (t, n, l - 1))
    _dev(lengths, torch.int32, "lengths", what, (n,))
    return t, n, l


def ctc_crf_target_fwd(stay, move, lengths, semiring, logz, workspace=None, stream=None):
    """Target-lattice logZ (see b200_ctc_crf_target_fwd): stay [T, N, L], move [T, N, L-1] fp32, lengths [N] int32 ->
    logz [N]; `workspace` (ctc_crf_target_workspace_bytes bytes) keeps what ctc_crf_target_grad needs."""
    lib = require()
    what = "ctc_crf_target_fwd"
    t, n, l = _target_shape(stay, move, lengths, what)
    _dev(logz, torch.float32, "logz", what, (n,))
    if workspace is not None:
        _dev(workspace, torch.uint8, "workspace", what)
        need = ctc_crf_target_workspace_bytes(n, t, l, semiring)
        if workspace.numel() < need:
            raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(stay.device):
        rc = lib.b200_ctc_crf_target_fwd(_ptr(stay), _ptr(move), _ptr(lengths), t, n, l, _semiring(semiring, what),
                                         _ptr(logz), _ptr(workspace), _stream(stream))
    _check(rc, "b200_ctc_crf_target_fwd")
    return logz


def ctc_crf_target_grad(stay, move, lengths, semiring, g, workspace, dstay, dmove, stream=None):
    """dstay / dmove = g[n] * dlogz[n]/d(stay, move) from the workspace of ctc_crf_target_fwd (see b200_ctc_crf_target_grad)."""
    lib = require()
    what = "ctc_crf_target_grad"
    t, n, l = _target_shape(stay, move, lengths, what)
    _dev(g, torch.float32, "g", what, (n,))
    _dev(dstay, torch.float32, "dstay", what, (t, n, l))
    _dev(dmove, torch.float32, "dmove", what, (t, n, l - 1))
    _dev(workspace, torch.uint8, "workspace", what)
    need = ctc_crf_target_workspace_bytes(n, t, l, semiring)
    if workspace.numel() < need:
        raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(stay.device):
        rc = lib.b200_ctc_crf_target_grad(_ptr(stay), _ptr(move), _ptr(lengths), t, n, l, _semiring(semiring, what),
                                          _ptr(g), _ptr(workspace), _ptr(dstay), _ptr(dmove), _stream(stream))
    _check(rc, "b200_ctc_crf_target_grad")
    return dstay, dmove


def ctc_loss_max_target():
    return load().b200_ctc_loss_max_target()


def ctc_loss_workspace_bytes(n, t, max_target):
    return load().b200_ctc_loss_workspace_bytes(int(n), int(t), int(max_target))


def _ctc_loss_shape(log_probs, input_lengths, targets, target_off, target_lengths, what):
    if not isinstance(log_probs, torch.Tensor) or not log_probs.is_cuda or log_probs.dtype != torch.float32 \
            or log_probs.dim() != 3 or (log_probs.stride(2) != 1 and log_probs.shape[2] != 1):
        raise NativeError(f"{what}: log_probs must be a CUDA fp32 [T, N, C] tensor with a contiguous class axis")
    t, n, _ = log_probs.shape
    _dev(input_lengths, torch.int32, "input_lengths", what, (n,))
    _dev(target_lengths, torch.int32, "target_lengths", what, (n,))
    _dev(target_off, torch.int64, "target_off", what, (n,))
    _dev(targets, torch.int32, "targets", what)
    return log_probs.shape


def ctc_loss_fwd(log_probs, input_lengths, targets, target_off, target_lengths, max_target, blank, nll, workspace=None,
                 stream=None):
    """CTC negative log-likelihood (see b200_ctc_loss_fwd): log_probs CUDA fp32 [T, N, C] (any strides on T and N);
    input_lengths / target_lengths int32 [N]; sample n's labels are targets.view(-1)[target_off[n]:][:target_lengths[n]]
    (int32 targets, int64 target_off) -> nll [N]; `workspace` (uint8, ctc_loss_workspace_bytes bytes) keeps what
    ctc_loss_grad needs."""
    lib = require()
    what = "ctc_loss_fwd"
    t, n, c = _ctc_loss_shape(log_probs, input_lengths, targets, target_off, target_lengths, what)
    _dev(nll, torch.float32, "nll", what, (n,))
    if workspace is not None:
        _dev(workspace, torch.uint8, "workspace", what)
        need = ctc_loss_workspace_bytes(n, t, max_target)
        if workspace.numel() < need:
            raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(log_probs.device):
        rc = lib.b200_ctc_loss_fwd(_ptr(log_probs), log_probs.stride(0), log_probs.stride(1), t, n, c, _ptr(input_lengths),
                                   _ptr(targets), targets.numel(), _ptr(target_off), _ptr(target_lengths), int(max_target),
                                   int(blank), _ptr(nll), _ptr(workspace), _stream(stream))
    _check(rc, "b200_ctc_loss_fwd")
    return nll


def ctc_loss_grad(log_probs, input_lengths, targets, target_off, target_lengths, max_target, blank, g, zero_infinity,
                  workspace, grad, stream=None):
    """grad [T, N, C] = g[n] * dnll[n]/dlog_probs in torch's form, from the workspace of ctc_loss_fwd with the same
    arguments (see b200_ctc_loss_grad)."""
    lib = require()
    what = "ctc_loss_grad"
    t, n, c = _ctc_loss_shape(log_probs, input_lengths, targets, target_off, target_lengths, what)
    _dev(g, torch.float32, "g", what, (n,))
    _dev(grad, torch.float32, "grad", what, (t, n, c))
    _dev(workspace, torch.uint8, "workspace", what)
    need = ctc_loss_workspace_bytes(n, t, max_target)
    if workspace.numel() < need:
        raise NativeError(f"{what}: workspace has {workspace.numel()} bytes, {need} needed")
    with torch.cuda.device(log_probs.device):
        rc = lib.b200_ctc_loss_grad(_ptr(log_probs), log_probs.stride(0), log_probs.stride(1), t, n, c, _ptr(input_lengths),
                                    _ptr(targets), targets.numel(), _ptr(target_off), _ptr(target_lengths), int(max_target),
                                    int(blank), _ptr(g), int(bool(zero_infinity)), _ptr(workspace), _ptr(grad),
                                    _stream(stream))
    _check(rc, "b200_ctc_loss_grad")
    return grad


def ctc_beam_workspace_bytes(n_reads, total_frames, beam_width):
    return load().b200_ctc_beam_workspace_bytes(int(n_reads), int(total_frames), int(beam_width))


def ctc_beam_search(logp, frame_off, frame_len, beam_width, threshold, qscale, qbias, workspace, sequence, qstring, moves,
                    stream=None):
    """CTC prefix beam search over packed reads (see b200_ctc_beam_search): logp CUDA fp16 [frames, 5]; frame_off int64 and
    frame_len int32 host arrays of one entry per read (copied into the workspace on `stream` before this returns);
    workspace CUDA uint8 of ctc_beam_workspace_bytes(n_reads, sum(frame_len), beam_width) bytes; sequence / qstring /
    moves CUDA uint8 [frames]."""
    lib = require()
    what = "ctc_beam_search"
    _dev(logp, torch.float16, "logp", what)
    if logp.dim() != 2 or logp.shape[1] != 5:
        raise NativeError(f"{what}: logp must be [frames, 5], got {tuple(logp.shape)}")
    frames = logp.shape[0]
    ln = np.ascontiguousarray(frame_len, dtype=np.int32)
    off = np.ascontiguousarray(frame_off, dtype=np.int64)
    if ln.ndim != 1 or off.shape != ln.shape:
        raise NativeError(f"{what}: frame_off and frame_len must have one entry per read, got shapes {off.shape} / {ln.shape}")
    n = ln.shape[0]
    if n and (int(ln.min()) < 0 or int(off.min()) < 0 or int((off + ln).max()) > frames):
        raise NativeError(f"{what}: a read lies outside the {frames} frames of logp")
    if not 1 <= int(beam_width) <= 32:
        raise NativeError(f"{what}: beam_width {beam_width} is outside [1, 32]")
    for t, name in ((sequence, "sequence"), (qstring, "qstring"), (moves, "moves")):
        _dev(t, torch.uint8, name, what, (frames,))
    _dev(workspace, torch.uint8, "workspace", what)
    with torch.cuda.device(logp.device):
        rc = lib.b200_ctc_beam_search(_ptr(logp), off.ctypes.data, ln.ctypes.data, n, int(beam_width), float(threshold),
                                      float(qscale), float(qbias), _ptr(workspace), workspace.numel(), _ptr(sequence),
                                      _ptr(qstring), _ptr(moves), _stream(stream))
    _check(rc, "b200_ctc_beam_search")
    return sequence, qstring, moves


# ---- QuartzNet CTC training (b200_wgrad_gemm ... b200_ctc_head_bwd) ----
def _f32(t, name):
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise NativeError(f"{name}: expected a contiguous CUDA fp32 tensor, got {t.dtype} {t.device}")
    return t


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def wgrad_gemm(dz, ldz, x, ldx, m, cout, k, dw, rows_inner=None, valid_inner=None, lpz=None, stream=None):
    """dw [cout, k] fp32 = dZ^T X over m GEMM rows with the row map of `gemm` (see b200_wgrad_gemm); `dz` / `x` only supply
    base pointers."""
    lib = require()
    if rows_inner is None:
        rows_inner = valid_inner = m
    lpz = valid_inner if lpz is None else lpz
    with torch.cuda.device(dw.device):
        ws = _workspace(lib.b200_wgrad_gemm_workspace_bytes(int(m), int(cout), int(k)), dw.device)
        rc = lib.b200_wgrad_gemm(_ptr(dz), int(ldz), int(lpz), _ptr(x), int(ldx), int(m), int(cout), int(k), int(rows_inner),
                                 int(valid_inner), _ptr(ws), _ptr(_f32(dw, "dw")), _stream(stream))
    _check(rc, "b200_wgrad_gemm")
    return dw


def depthwise_wgrad(dy, ldy, x, ldx, n, t, dw, stream=None):
    """dw [C, 1, K] fp32: the depthwise convolution's weight gradient (see b200_depthwise_wgrad)."""
    lib = require()
    c, _, k = dw.shape
    with torch.cuda.device(dw.device):
        ws = _workspace(lib.b200_depthwise_wgrad_workspace_bytes(int(n), int(t), c, k), dw.device)
        rc = lib.b200_depthwise_wgrad(_ptr(dy), int(ldy), _ptr(x), int(ldx), int(n), int(t), c, k, _ptr(ws),
                                      _ptr(_f32(dw, "dw")), _stream(stream))
    _check(rc, "b200_depthwise_wgrad")
    return dw


def conv_first_wgrad(dz, ldz, x, stride, dw, stream=None):
    """dw [C, 1, K] fp32: the first convolution's weight gradient against the signal x [N, L] (see b200_conv_first_wgrad)."""
    lib = require()
    n, l = x.shape
    c, _, k = dw.shape
    t = (l - 1) // stride + 1
    with torch.cuda.device(dw.device):
        ws = _workspace(lib.b200_conv_first_wgrad_workspace_bytes(n, t, c, k), dw.device)
        rc = lib.b200_conv_first_wgrad(_ptr(dz), int(ldz), _ptr(_f16(x, "x")), n, l, c, k, int(stride), _ptr(ws),
                                       _ptr(_f32(dw, "dw")), _stream(stream))
    _check(rc, "b200_conv_first_wgrad")
    return dw


def bn_stats(z, ldz, m, c, eps, momentum, mean, invstd, running_mean=None, running_var=None, stream=None):
    """Batch statistics of z [m, c] (pitch ldz) into mean / invstd, updating the running statistics (see b200_bn_stats)."""
    lib = require()
    with torch.cuda.device(mean.device):
        ws = _workspace(lib.b200_bn_stats_workspace_bytes(int(m), int(c)), mean.device)
        rc = lib.b200_bn_stats(_ptr(z), int(ldz), int(m), int(c), float(eps), float(momentum), _ptr(ws), _ptr(_f32(mean, "mean")),
                               _ptr(_f32(invstd, "invstd")), _ptr(running_mean), _ptr(running_var), _stream(stream))
    _check(rc, "b200_bn_stats")


def bn_act_struct(m, c, t, act, p, seed, unit, z, ldz, mean, invstd, gamma, beta, residual=None, mask=None):
    """A `b200_bn_act`; `residual` = (zr, ldzr, mean_r, invstd_r, gamma_r, beta_r) or None.  The struct holds raw pointers:
    the caller keeps the tensors alive."""
    s = BnActStruct(m=int(m), c=int(c), t=int(t), act=int(act), p=float(p), seed=int(seed) & (2**64 - 1), unit=int(unit),
                    z=z.data_ptr(), ldz=int(ldz), mean=_f32(mean, "mean").data_ptr(), invstd=_f32(invstd, "invstd").data_ptr(),
                    gamma=_f32(gamma, "gamma").data_ptr(), beta=_f32(beta, "beta").data_ptr(),
                    mask=None if mask is None else mask.data_ptr())
    if residual is not None:
        zr, ldzr, mr, ir, gr, br = residual
        s.zr, s.ldzr, s.mean_r, s.invstd_r, s.gamma_r, s.beta_r = (zr.data_ptr(), int(ldzr), _f32(mr, "mean_r").data_ptr(),
                                                                   _f32(ir, "invstd_r").data_ptr(), _f32(gr, "gamma_r").data_ptr(),
                                                                   _f32(br, "beta_r").data_ptr())
    return s


def bn_act_fwd(args, out, ldo, lpo, stream=None):
    """BatchNorm [+ residual BatchNorm] -> activation -> dropout into rows of `out` (see b200_bn_act_fwd)."""
    lib = require()
    with torch.cuda.device(out.device):
        rc = lib.b200_bn_act_fwd(ctypes.byref(args), _ptr(out), int(ldo), int(lpo), _stream(stream))
    _check(rc, "b200_bn_act_fwd")
    return out


def bn_act_bwd(args, dy, ldy, dgamma, dbeta, dz, ldo, lpo, dy2=None, ldy2=0, dgamma_r=None, dbeta_r=None, dzr=None, stream=None):
    """Gradient of `bn_act_fwd` (see b200_bn_act_bwd)."""
    lib = require()
    for t, name in ((dy, "dy"), (dy2, "dy2")):
        if t is not None and t.stride(-1) != 1:
            raise NativeError(f"bn_act_bwd: {name} must have unit stride along its last dimension (rows of pitch ld)")
    with torch.cuda.device(dz.device):
        ws = _workspace(lib.b200_bn_act_bwd_workspace_bytes(args.m, args.c), dz.device)
        rc = lib.b200_bn_act_bwd(ctypes.byref(args), _ptr(dy), int(ldy), _ptr(dy2), int(ldy2), _ptr(ws), _ptr(_f32(dgamma, "dgamma")),
                                 _ptr(_f32(dbeta, "dbeta")), _ptr(dgamma_r), _ptr(dbeta_r), _ptr(dz), _ptr(dzr), int(ldo), int(lpo),
                                 _stream(stream))
    _check(rc, "b200_bn_act_bwd")


def ctc_head_train_fwd(x, m, w, bias, logp, stream=None):
    """logp [m, 5] fp32 = log_softmax(fp16(x w^T + bias)) (see b200_ctc_head_train_fwd)."""
    lib = require()
    with torch.cuda.device(logp.device):
        rc = lib.b200_ctc_head_train_fwd(_ptr(_f16(x, "x")), int(m), w.shape[-1], _ptr(_f16(w, "w")), _ptr(bias),
                                         _ptr(_f32(logp, "logp")), _stream(stream))
    _check(rc, "b200_ctc_head_train_fwd")
    return logp


def ctc_head_bwd(x, m, w, logp, g, dw, db, dx, stream=None):
    """Gradient of `ctc_head_train_fwd` from g = dL/dlogp (see b200_ctc_head_bwd)."""
    lib = require()
    f = w.shape[-1]
    with torch.cuda.device(dx.device):
        ws = _workspace(lib.b200_ctc_head_bwd_workspace_bytes(int(m), f), dx.device)
        rc = lib.b200_ctc_head_bwd(_ptr(_f16(x, "x")), int(m), f, _ptr(_f16(w, "w")), _ptr(_f32(logp, "logp")), _ptr(_f32(g, "g")),
                                   _ptr(ws), _ptr(_f32(dw, "dw")), _ptr(db), _ptr(_f16(dx, "dx")), _stream(stream))
    _check(rc, "b200_ctc_head_bwd")


def lstm_crf_fwd(plan_struct, x, scores, stream=None):
    """Whole encoder forward from one C call (see b200_lstm_crf_fwd); `plan_struct`: a filled LstmCrfPlanStruct."""
    lib = require()
    with torch.cuda.device(scores.device):
        rc = lib.b200_lstm_crf_fwd(ctypes.byref(plan_struct), _ptr(_f16(x, "x")), _ptr(scores), _stream(stream))
    _check(rc, "b200_lstm_crf_fwd")
    return scores


def chunk_signal(signal, chunksize, overlap, out=None, stream=None):
    """bonito.util.chunk for ONE read already on the device: signal [length] (or [1, length]) fp16 / fp32 ->
    [n_chunks, 1, chunksize] fp16 from one gather kernel (see b200_chunk_signal)."""
    lib = require()
    sig = signal.reshape(-1)
    if not sig.is_cuda or sig.dtype not in (torch.float16, torch.float32) or not sig.is_contiguous():
        raise ValueError("chunk_signal: a contiguous float16 / float32 CUDA tensor expected")
    n = lib.b200_chunk_count(sig.numel(), int(chunksize), int(overlap))
    if n <= 0:
        raise ValueError(f"chunk_signal: bad geometry (length {sig.numel()}, chunksize {chunksize}, overlap {overlap})")
    if out is None:
        out = torch.empty(n, 1, chunksize, dtype=torch.float16, device=sig.device)
    with torch.cuda.device(sig.device):
        rc = lib.b200_chunk_signal(_ptr(sig), int(sig.dtype == torch.float32), sig.numel(), int(chunksize), int(overlap),
                                   _ptr(out), int(chunksize), _stream(stream))
    _check(rc, "b200_chunk_signal")
    return out


def lstm_crf_lstm_fwd(plan_struct, first, count, stream=None):
    """LSTM layers [first, first + count) of a filled LstmCrfPlanStruct, in chains of tiles (see b200_lstm_crf_lstm_fwd)."""
    lib = require()
    rc = lib.b200_lstm_crf_lstm_fwd(ctypes.byref(plan_struct), int(first), int(count), _stream(stream))
    _check(rc, "b200_lstm_crf_lstm_fwd")


def new_stream(device):
    """A CUDA stream of its own (cudaStreamCreateWithFlags, non-blocking) wrapped for torch.  torch.cuda.Stream() returns
    one of 32 pooled streams per device round-robin, so streams that must run concurrently can silently be the same stream."""
    lib = require()
    handle = c_void_p()
    with torch.cuda.device(device):
        rc = lib.b200_stream_create(ctypes.byref(handle))
    _check(rc, "b200_stream_create")
    return torch.cuda.ExternalStream(handle.value, device=device)


def quantize_i8(x, out, scale=127.0, stream=None):
    """fp16 -> int8 (see b200_quantize_i8); `out`: int8 tensor with x.numel() elements."""
    lib = require()
    with torch.cuda.device(out.device):
        rc = lib.b200_quantize_i8(_ptr(_f16(x, "x")), _ptr(out), x.numel(), float(scale), _stream(stream))
    _check(rc, "b200_quantize_i8")
    return out


def gemm_i8(a, lda, b, col_scale, bias, c, ldc, m, n, k, act=ACT_NONE, lo=0.0, hi=0.0, rows_inner=None, valid_inner=None,
            stride_inner=1, stride_outer=0, group=0, stride_group=0, cb_width=0, cb_rows=0, stream=None, max_ctas=0):
    """C = act(col_scale * (A_i8 B_i8^T) + bias) (see b200_gemm_i8_fwd)."""
    lib = require()
    if rows_inner is None:
        rows_inner, valid_inner = m, m
    with torch.cuda.device(c.device):
        rc = lib.b200_gemm_i8_fwd(_ptr(a), lda, _ptr(b), _ptr(col_scale), _ptr(bias), _ptr(c), ldc, m, n, k, act, float(lo),
                                  float(hi), rows_inner, valid_inner, stride_inner, stride_outer, int(group), int(stride_group),
                                  int(cb_width), int(cb_rows), int(max_ctas), _stream(stream))
    _check(rc, "b200_gemm_i8_fwd")
    return c


# ------------------------------------------------------------------------------------------------ mapping (map.cu)
def _map_dev(t, dtype, name, what):
    if t is None or not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise NativeError(f"{what}: {name} must be a contiguous CUDA {dtype} tensor")
    return _ptr(t)


def map_minimizers(seq, seq_off, k, w, kmer, mm, stream=None):
    """mm[p] = hash << 1 | strand of the minimizer at base p, else -1 (see b200_map_minimizers)."""
    lib = require()
    n = seq.numel()
    for t, dtype, name in ((seq, torch.uint8, "seq"), (seq_off, torch.int64, "seq_off"), (kmer, torch.int64, "kmer"),
                           (mm, torch.int64, "mm")):
        _map_dev(t, dtype, name, "map_minimizers")
    if kmer.numel() < n or mm.numel() < n:
        raise NativeError("map_minimizers: kmer and mm need one entry per base")
    with torch.cuda.device(seq.device):
        _check(lib.b200_map_minimizers(_ptr(seq), n, _ptr(seq_off), seq_off.numel() - 1, int(k), int(w), _ptr(kmer), _ptr(mm),
                                       _stream(stream)), "b200_map_minimizers")


def map_anchors(mm, seq_off, k, uniq, start, val, max_occ, count=None, aoff=None, akey=None, aq=None, stream=None):
    """Anchors per position into `count`, or (count None) the anchors themselves into akey / aq at aoff."""
    lib = require()
    with torch.cuda.device(mm.device):
        _check(lib.b200_map_anchors(_ptr(mm), mm.numel(), _ptr(seq_off), seq_off.numel() - 1, int(k), _ptr(uniq), uniq.numel(),
                                    _ptr(start), _ptr(val), int(max_occ), _ptr(count), _ptr(aoff), _ptr(akey), _ptr(aq),
                                    _stream(stream)), "b200_map_anchors")


def map_chain(akey, aq, read_aoff, ctg_off, k, f, pred, stream=None):
    lib = require()
    for t, dtype, name in ((akey, torch.int64, "akey"), (aq, torch.int32, "aq"), (read_aoff, torch.int64, "read_aoff"),
                           (ctg_off, torch.int64, "ctg_off"), (f, torch.int32, "f"), (pred, torch.int32, "pred")):
        _map_dev(t, dtype, name, "map_chain")
    with torch.cuda.device(akey.device):
        _check(lib.b200_map_chain(_ptr(akey), _ptr(aq), _ptr(read_aoff), read_aoff.numel() - 1, _ptr(ctg_off),
                                  ctg_off.numel() - 1, int(k), _ptr(f), _ptr(pred), _stream(stream)), "b200_map_chain")


def map_extract(akey, aq, f, pred, order, read_aoff, seq_off, k, max_band, taken, chain, out, stream=None):
    lib = require()
    n_reads = read_aoff.numel() - 1
    if out.shape != (n_reads, 9) or out.dtype != torch.int64:
        raise NativeError(f"map_extract: out must be int64 ({n_reads}, 9)")
    with torch.cuda.device(out.device):
        _check(lib.b200_map_extract(_ptr(akey), _ptr(aq), _ptr(f), _ptr(pred), _ptr(order), _ptr(read_aoff), _ptr(seq_off),
                                    n_reads, int(k), int(max_band), _ptr(taken), _ptr(chain), _ptr(out), _stream(stream)),
               "b200_map_extract")


def map_align_trace_bytes(query_len, band):
    return load().b200_map_align_trace_bytes(int(query_len), int(band))


def map_align(query, target, chain, meta, max_band, cen, trace, ops, out, stream=None):
    """Banded local alignment of each pair along its chain (see b200_map_align); meta CUDA int64 [n, 9]."""
    lib = require()
    n = meta.shape[0]
    if meta.shape != (n, 9) or out.shape != (n, 6):
        raise NativeError("map_align: meta must be (n, 9) and out (n, 6)")
    for t, dtype, name in ((query, torch.uint8, "query"), (target, torch.uint8, "target"), (chain, torch.int64, "chain"),
                           (meta, torch.int64, "meta"), (cen, torch.int32, "cen"), (trace, torch.uint8, "trace"),
                           (ops, torch.uint8, "ops"), (out, torch.int32, "out")):
        _map_dev(t, dtype, name, "map_align")
    with torch.cuda.device(out.device):
        _check(lib.b200_map_align(_ptr(query), _ptr(target), _ptr(chain), _ptr(meta), n, int(max_band), _ptr(cen), _ptr(trace),
                                  _ptr(ops), _ptr(out), _stream(stream)), "b200_map_align")


# ------------------------------------------------------------------------------------------------ BGZF (bgzf.cu)
def bgzf_members(in_bytes):
    return -(-int(in_bytes) // BGZF_MEMBER_INPUT)


def bgzf_workspace_bytes(in_bytes):
    return load().b200_bgzf_workspace_bytes(int(in_bytes))


def bgzf_compress(inp, out, out_offsets, workspace, stream=None):
    """BGZF members of the CUDA uint8 buffer `inp`, back to back into `out` (CUDA uint8, >= members * 65536 bytes);
    out_offsets (CUDA int64 [members + 1]) receives their offsets and the total length (see b200_bgzf_compress)."""
    lib = require()
    what = "bgzf_compress"
    _dev(inp, torch.uint8, "inp", what)
    _dev(out, torch.uint8, "out", what)
    _dev(workspace, torch.uint8, "workspace", what)
    n = bgzf_members(inp.numel())
    _dev(out_offsets, torch.int64, "out_offsets", what)
    if out_offsets.numel() < n + 1 or out.numel() < n * BGZF_MEMBER_MAX:
        raise NativeError(f"{what}: {n} members need {n + 1} offsets and {n * BGZF_MEMBER_MAX} output bytes")
    with torch.cuda.device(inp.device):
        rc = lib.b200_bgzf_compress(_ptr(inp), inp.numel(), _ptr(out), _ptr(out_offsets), _ptr(workspace), workspace.numel(),
                                    _stream(stream))
    _check(rc, "b200_bgzf_compress")
    return out_offsets


def bgzf_decompress(inp, meta, out, status, stream=None):
    """Inflate BGZF members (see b200_bgzf_decompress): inp CUDA uint8 (the members' raw DEFLATE data), meta CUDA int64
    [n, 5] (raw start, raw length, output offset, ISIZE, CRC32 per member), out CUDA uint8, status CUDA int32 [n]
    (INFLATE_STATUS codes, 0 = inflated and CRC32 verified)."""
    lib = require()
    what = "bgzf_decompress"
    _dev(inp, torch.uint8, "inp", what)
    _dev(out, torch.uint8, "out", what)
    n = meta.shape[0] if isinstance(meta, torch.Tensor) else 0
    _dev(meta, torch.int64, "meta", what, (n, 5))
    _dev(status, torch.int32, "status", what, (n,))
    with torch.cuda.device(out.device):
        rc = lib.b200_bgzf_decompress(_ptr(inp), inp.numel(), _ptr(meta), n, _ptr(out), out.numel(), _ptr(status),
                                      _stream(stream))
    _check(rc, "b200_bgzf_decompress")
    return status


# ------------------------------------------------------------------------------------------------ zstd / svb16 (zstd.cu)
# B200_ZSTD_* status codes of b200_zstd_decompress
ZSTD_STATUS = {0: "ok", 1: "not a zstd frame", 2: "reserved frame header bit, dictionary ID or window too large",
               3: "reserved block type or block too large", 4: "invalid literals section size or type",
               5: "invalid Huffman weights or literal stream", 6: "invalid FSE table or accuracy log",
               7: "invalid sequence count or bit stream", 8: "offset before the frame's first byte",
               9: "output past capacity", 10: "content size mismatch", 11: "truncated input", 12: "checksum mismatch",
               13: "stream outside the launch's buffers"}
# B200_SVB16_* status codes of b200_svb16_decode
SVB16_STATUS = {0: "ok", 1: "svb16 length is not keys + data", 2: "row outside the launch's buffers"}


def zstd_decompress(inp, meta, out, out_len, status, stream=None):
    """Decompress zstd streams (see b200_zstd_decompress): inp CUDA uint8, meta CUDA int64 [n, 4] (input offset, input
    length, output offset, output capacity per stream), out CUDA uint8, out_len CUDA int64 [n] (bytes produced), status
    CUDA int32 [n] (ZSTD_STATUS codes, 0 = decoded)."""
    lib = require()
    what = "zstd_decompress"
    _dev(inp, torch.uint8, "inp", what)
    _dev(out, torch.uint8, "out", what)
    n = meta.shape[0] if isinstance(meta, torch.Tensor) else 0
    _dev(meta, torch.int64, "meta", what, (n, 4))
    _dev(out_len, torch.int64, "out_len", what, (n,))
    _dev(status, torch.int32, "status", what, (n,))
    with torch.cuda.device(out.device):
        rc = lib.b200_zstd_decompress(_ptr(inp), inp.numel(), _ptr(meta), n, _ptr(out), out.numel(), _ptr(out_len),
                                      _ptr(status), _stream(stream))
    _check(rc, "b200_zstd_decompress")
    return status


def svb16_decode(inp, meta, out, status, stream=None):
    """Decode svb16 rows into int16 samples (see b200_svb16_decode): inp CUDA uint8, meta CUDA int64 [n, 4] (svb16
    offset, svb16 length, sample count, sample offset per row), out CUDA int16, status CUDA int32 [n] (SVB16_STATUS)."""
    lib = require()
    what = "svb16_decode"
    _dev(inp, torch.uint8, "inp", what)
    _dev(out, torch.int16, "out", what)
    n = meta.shape[0] if isinstance(meta, torch.Tensor) else 0
    _dev(meta, torch.int64, "meta", what, (n, 4))
    _dev(status, torch.int32, "status", what, (n,))
    with torch.cuda.device(out.device):
        rc = lib.b200_svb16_decode(_ptr(inp), inp.numel(), _ptr(meta), n, _ptr(out), out.numel(), _ptr(status),
                                   _stream(stream))
    _check(rc, "b200_svb16_decode")
    return status
