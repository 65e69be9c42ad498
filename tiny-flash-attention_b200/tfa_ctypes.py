"""ctypes binding of the C ABI (include/tfa_b200.h) for callers that hold raw device/host pointers.

This is the same stub INTEGRATION.md shows for a reference maintainer.  torch is used only to get
`data_ptr()` / streams of tensors the caller already owns.  There is NO fallback: if libtfa_b200.so
is missing or the device is not sm_90, calls raise.
"""
from __future__ import annotations

import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TFA_LIB", os.path.join(HERE, "libtfa_b200.so"))   # TFA_LIB: tuning variants only

TFA_BF16, TFA_FP16 = 0, 1
TFA_FP8_E4M3 = 2
_LIB = None
_WORKSPACES = {}     # (device, stream) -> last split-KV workspace, see _split_workspace()


class TfaError(RuntimeError):
    def __init__(self, code, msg, record=None):
        super().__init__(f"tfa error {code}: {msg}" + (f" debug={record}" if record else ""))
        self.code = code
        self.record = record


class FwdArgs(ctypes.Structure):
    _fields_ = [
        ("q", ctypes.c_void_p), ("k", ctypes.c_void_p), ("v", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("lse", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("S", ctypes.c_int32), ("D", ctypes.c_int32),
        ("stride_b", ctypes.c_int64), ("stride_h", ctypes.c_int64), ("stride_s", ctypes.c_int64),
        ("dtype", ctypes.c_int32), ("is_causal", ctypes.c_int32), ("softmax_scale", ctypes.c_float),
        ("out_fp32", ctypes.c_int32), ("stream", ctypes.c_void_p),
    ]


class AttnArgs(ctypes.Structure):
    """struct tfa_attn_args (include/tfa_b200.h)."""
    _fields_ = [
        ("q", ctypes.c_void_p), ("k", ctypes.c_void_p), ("v", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("lse", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("Hq", ctypes.c_int32), ("Hkv", ctypes.c_int32), ("Sq", ctypes.c_int32),
        ("Sk", ctypes.c_int32), ("D", ctypes.c_int32),
        ("q_stride_b", ctypes.c_int64), ("q_stride_h", ctypes.c_int64), ("q_stride_s", ctypes.c_int64),
        ("kv_stride_b", ctypes.c_int64), ("kv_stride_h", ctypes.c_int64), ("kv_stride_s", ctypes.c_int64),
        ("dtype", ctypes.c_int32), ("is_causal", ctypes.c_int32), ("softmax_scale", ctypes.c_float),
        ("out_fp32", ctypes.c_int32), ("num_splits", ctypes.c_int32),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t), ("stream", ctypes.c_void_p),
    ]


class VarlenArgs(ctypes.Structure):
    """struct tfa_attn_varlen_args (include/tfa_b200.h)."""
    _fields_ = [
        ("q", ctypes.c_void_p), ("k", ctypes.c_void_p), ("v", ctypes.c_void_p), ("out", ctypes.c_void_p),
        ("lse", ctypes.c_void_p), ("cu_seqlens_q", ctypes.c_void_p), ("cu_seqlens_k", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("Hq", ctypes.c_int32), ("Hkv", ctypes.c_int32), ("D", ctypes.c_int32),
        ("total_q", ctypes.c_int32), ("total_k", ctypes.c_int32), ("max_seqlen_q", ctypes.c_int32),
        ("q_stride_s", ctypes.c_int64), ("q_stride_h", ctypes.c_int64),
        ("kv_stride_s", ctypes.c_int64), ("kv_stride_h", ctypes.c_int64),
        ("dtype", ctypes.c_int32), ("is_causal", ctypes.c_int32), ("softmax_scale", ctypes.c_float),
        ("out_fp32", ctypes.c_int32), ("stream", ctypes.c_void_p),
    ]


class KvcacheArgs(ctypes.Structure):
    """struct tfa_attn_kvcache_args (include/tfa_b200.h)."""
    _fields_ = [
        ("q", ctypes.c_void_p), ("k_cache", ctypes.c_void_p), ("v_cache", ctypes.c_void_p),
        ("k_new", ctypes.c_void_p), ("v_new", ctypes.c_void_p), ("out", ctypes.c_void_p), ("lse", ctypes.c_void_p),
        ("cache_seqlens", ctypes.c_void_p), ("block_table", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("Hq", ctypes.c_int32), ("Hkv", ctypes.c_int32), ("Sq", ctypes.c_int32),
        ("D", ctypes.c_int32), ("num_blocks", ctypes.c_int32), ("page_block_size", ctypes.c_int32),
        ("max_blocks_per_seq", ctypes.c_int32), ("Snew", ctypes.c_int32),
        ("q_stride_b", ctypes.c_int64), ("q_stride_s", ctypes.c_int64), ("q_stride_h", ctypes.c_int64),
        ("cache_stride_block", ctypes.c_int64), ("cache_stride_s", ctypes.c_int64), ("cache_stride_h", ctypes.c_int64),
        ("block_table_stride", ctypes.c_int64),
        ("new_stride_b", ctypes.c_int64), ("new_stride_s", ctypes.c_int64), ("new_stride_h", ctypes.c_int64),
        ("dtype", ctypes.c_int32), ("is_causal", ctypes.c_int32), ("softmax_scale", ctypes.c_float),
        ("out_fp32", ctypes.c_int32), ("num_splits", ctypes.c_int32),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t), ("stream", ctypes.c_void_p),
    ]


class VarlenKvcacheArgs(ctypes.Structure):
    """struct tfa_attn_varlen_kvcache_args (include/tfa_b200.h)."""
    _fields_ = [
        ("q", ctypes.c_void_p), ("k_cache", ctypes.c_void_p), ("v_cache", ctypes.c_void_p),
        ("k_new", ctypes.c_void_p), ("v_new", ctypes.c_void_p), ("out", ctypes.c_void_p), ("lse", ctypes.c_void_p),
        ("cu_seqlens_q", ctypes.c_void_p), ("cache_seqlens", ctypes.c_void_p), ("block_table", ctypes.c_void_p),
        ("B", ctypes.c_int32), ("Hq", ctypes.c_int32), ("Hkv", ctypes.c_int32), ("D", ctypes.c_int32),
        ("total_q", ctypes.c_int32), ("max_seqlen_q", ctypes.c_int32),
        ("num_blocks", ctypes.c_int32), ("page_block_size", ctypes.c_int32), ("max_blocks_per_seq", ctypes.c_int32),
        ("q_stride_s", ctypes.c_int64), ("q_stride_h", ctypes.c_int64),
        ("cache_stride_block", ctypes.c_int64), ("cache_stride_s", ctypes.c_int64), ("cache_stride_h", ctypes.c_int64),
        ("block_table_stride", ctypes.c_int64), ("new_stride_s", ctypes.c_int64), ("new_stride_h", ctypes.c_int64),
        ("dtype", ctypes.c_int32), ("is_causal", ctypes.c_int32), ("softmax_scale", ctypes.c_float),
        ("out_fp32", ctypes.c_int32), ("stream", ctypes.c_void_p),
    ]


class KvQuantArgs(ctypes.Structure):
    """struct tfa_kv_quant_args (include/tfa_b200.h)."""
    _fields_ = [("cache_dtype", ctypes.c_int32), ("k_scale", ctypes.c_float), ("v_scale", ctypes.c_float)]


class QkvQuantArgs(ctypes.Structure):
    """struct tfa_qkv_quant_args (include/tfa_b200.h)."""
    _fields_ = [("qkv_dtype", ctypes.c_int32), ("q_scale", ctypes.c_float), ("k_scale", ctypes.c_float),
                ("v_scale", ctypes.c_float)]


class SplitArgs(ctypes.Structure):
    """struct tfa_split_args (include/tfa_b200.h)."""
    _fields_ = [("num_splits", ctypes.c_int32), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t)]


class RotaryArgs(ctypes.Structure):
    """struct tfa_rotary_args (include/tfa_b200.h)."""
    _fields_ = [
        ("cos", ctypes.c_void_p), ("sin", ctypes.c_void_p), ("seqlen_ro", ctypes.c_int32),
        ("rotary_dim", ctypes.c_int32), ("interleaved", ctypes.c_int32), ("q_rot", ctypes.c_void_p),
    ]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} not built -- run `python tiny-flash-attention_b200/build.py` "
                                    "(there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        L.tfa_abi_version.restype = ci
        L.tfa_fwd.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp]
        L.tfa_fwd.restype = ci
        L.tfa_fwd_ex.argtypes = [ctypes.POINTER(FwdArgs)]
        L.tfa_fwd_ex.restype = ci
        L.tfa_fwd_multi.argtypes = [ctypes.POINTER(FwdArgs), ctypes.POINTER(ctypes.c_void_p), ci]
        L.tfa_fwd_multi.restype = ci
        L.tfa_attn_fwd.argtypes = [ctypes.POINTER(AttnArgs)]
        L.tfa_attn_fwd.restype = ci
        L.tfa_attn_num_splits.argtypes = [ctypes.POINTER(AttnArgs)]
        L.tfa_attn_num_splits.restype = ci
        L.tfa_attn_workspace_bytes.argtypes = [ctypes.POINTER(AttnArgs), ci]
        L.tfa_attn_workspace_bytes.restype = ctypes.c_size_t
        L.tfa_attn_varlen_fwd.argtypes = [ctypes.POINTER(VarlenArgs)]
        L.tfa_attn_varlen_fwd.restype = ci
        L.tfa_attn_kvcache_fwd.argtypes = [ctypes.POINTER(KvcacheArgs)]
        L.tfa_attn_kvcache_fwd.restype = ci
        L.tfa_attn_kvcache_rotary_fwd.argtypes = [ctypes.POINTER(KvcacheArgs), ctypes.POINTER(RotaryArgs)]
        L.tfa_attn_kvcache_rotary_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs)]
        L.tfa_attn_varlen_kvcache_fwd.restype = ci
        L.tfa_attn_kvcache_fp8_fwd.argtypes = [ctypes.POINTER(KvcacheArgs), ctypes.POINTER(RotaryArgs),
                                               ctypes.POINTER(KvQuantArgs)]
        L.tfa_attn_kvcache_fp8_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_fp8_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ctypes.POINTER(KvQuantArgs)]
        L.tfa_attn_varlen_kvcache_fp8_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_rotary_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ctypes.POINTER(RotaryArgs),
                                                         ctypes.POINTER(KvQuantArgs)]
        L.tfa_attn_varlen_kvcache_rotary_fwd.restype = ci
        L.tfa_attn_fp8_fwd.argtypes = [ctypes.POINTER(AttnArgs), ctypes.POINTER(QkvQuantArgs)]
        L.tfa_attn_fp8_fwd.restype = ci
        L.tfa_attn_varlen_fp8_fwd.argtypes = [ctypes.POINTER(VarlenArgs), ctypes.POINTER(QkvQuantArgs)]
        L.tfa_attn_varlen_fp8_fwd.restype = ci
        L.tfa_attn_kvcache_qkv8_fwd.argtypes = [ctypes.POINTER(KvcacheArgs), ctypes.POINTER(QkvQuantArgs)]
        L.tfa_attn_kvcache_qkv8_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_qkv8_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ctypes.POINTER(QkvQuantArgs)]
        L.tfa_attn_varlen_kvcache_qkv8_fwd.restype = ci
        L.tfa_attn_kvcache_qkv8_q16_fwd.argtypes = [ctypes.POINTER(KvcacheArgs), ctypes.POINTER(RotaryArgs),
                                                    ctypes.POINTER(QkvQuantArgs), vp]
        L.tfa_attn_kvcache_qkv8_q16_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_qkv8_q16_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs),
                                                           ctypes.POINTER(RotaryArgs), ctypes.POINTER(QkvQuantArgs), vp]
        L.tfa_attn_varlen_kvcache_qkv8_q16_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_split_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ctypes.POINTER(RotaryArgs),
                                                        ctypes.POINTER(KvQuantArgs), ctypes.POINTER(SplitArgs)]
        L.tfa_attn_varlen_kvcache_split_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_qkv8_split_fwd.argtypes = [ctypes.POINTER(VarlenKvcacheArgs),
                                                             ctypes.POINTER(RotaryArgs), ctypes.POINTER(QkvQuantArgs),
                                                             vp, ctypes.POINTER(SplitArgs)]
        L.tfa_attn_varlen_kvcache_qkv8_split_fwd.restype = ci
        L.tfa_attn_varlen_kvcache_num_splits.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ci]
        L.tfa_attn_varlen_kvcache_num_splits.restype = ci
        L.tfa_attn_varlen_kvcache_workspace_bytes.argtypes = [ctypes.POINTER(VarlenKvcacheArgs), ci]
        L.tfa_attn_varlen_kvcache_workspace_bytes.restype = ctypes.c_size_t
        L.tfa_selftest_wgmma_fp8.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp]
        L.tfa_selftest_wgmma_fp8.restype = ci
        L.tfa_fwd_host.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, ci]
        L.tfa_fwd_host.restype = ci
        L.tfa_host_release.restype = None
        L.tfa_launch_count.restype = ctypes.c_ulonglong
        L.tfa_debug_record.argtypes = [ctypes.POINTER(ctypes.c_uint * 8)]
        L.tfa_debug_record.restype = ci
        L.tfa_debug_clear.restype = None
        L.tfa_error_string.argtypes = [ci]
        L.tfa_error_string.restype = ctypes.c_char_p
        L.tfa_selftest_tma.argtypes = [vp, ci, ci, ci, ci, ci, ci, vp, vp]
        L.tfa_selftest_tma.restype = ci
        L.tfa_selftest_umma.argtypes = [vp, vp, vp, ci, ci, ci, ci, ctypes.POINTER(ci * 4), vp]
        L.tfa_selftest_umma.restype = ci
        _LIB = L
    return _LIB


def debug_record():
    rec = (ctypes.c_uint * 8)()
    lib().tfa_debug_record(ctypes.byref(rec))
    return list(rec)


def check(rc):
    if rc != 0:
        rec = debug_record()
        raise TfaError(rc, lib().tfa_error_string(rc).decode(), rec if rec[0] else None)


def _dtype_code(t):
    import torch
    if t.dtype == torch.bfloat16:
        return TFA_BF16
    if t.dtype == torch.float16:
        return TFA_FP16
    raise TypeError(f"q/k/v must be bfloat16 or float16, got {t.dtype}")


def fwd(q, k, v, is_causal, softmax_scale, out_fp32=False, layout="bhsd", stream=None, out=None, lse=None):
    """Device tensors in, (out, lse) device tensors back -- straight through tfa_fwd_ex()."""
    import torch
    assert q.is_cuda and k.is_cuda and v.is_cuda, "device tensors required"
    assert q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    if layout == "bhsd":
        B, H, S, D = q.shape
        sb, sh, ss = H * S * D, S * D, D
    elif layout == "bshd":
        B, S, H, D = q.shape
        sb, ss, sh = S * H * D, H * D, D
    else:
        raise ValueError(layout)
    if out is None:
        out = torch.empty(q.shape, dtype=torch.float32 if out_fp32 else q.dtype, device=q.device)
    if lse is None:
        lse = torch.empty((B, H, S), dtype=torch.float32, device=q.device)
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = FwdArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), B, H, S, D, sb, sh, ss,
                _dtype_code(q), int(bool(is_causal)), float(softmax_scale), int(bool(out_fp32)), st)
    check(lib().tfa_fwd_ex(ctypes.byref(a)))
    return out, lse


def _split_workspace(dense, args, device, stream):
    """Split count of the dense problem `dense` (AttnArgs).  When it splits, allocates the workspace on `device` and
    sets num_splits / workspace / workspace_bytes in `args` (`dense` itself, or the call's own argument struct)."""
    import torch
    L = lib()
    n = int(L.tfa_attn_num_splits(ctypes.byref(dense)))
    if n > 1:
        need = int(L.tfa_attn_workspace_bytes(ctypes.byref(dense), n))
        ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=device)
        args.workspace, args.workspace_bytes, args.num_splits = ws.data_ptr(), need, n
        # the launch is asynchronous: keep the workspace alive until the next call on the same stream (which is
        # ordered behind this one) instead of handing it back to the allocator while the kernels may still run
        _WORKSPACES[(device.index, int(stream))] = ws
    return n


def _qkv_quant(q, q_scale, k_scale, v_scale, out_dtype):
    """(tfa_qkv_quant_args, output dtype) for float8_e4m3fn q / k / v, or (None, q's dtype) for 16-bit ones, which
    take no scales."""
    import torch
    if q.dtype != torch.float8_e4m3fn:
        if (q_scale, k_scale, v_scale) != (1.0, 1.0, 1.0) or out_dtype not in (None, q.dtype):
            raise ValueError(f"q_scale / k_scale / v_scale / out_dtype apply to float8_e4m3fn inputs only; q is {q.dtype}")
        return None, q.dtype
    if out_dtype not in (torch.bfloat16, torch.float16):
        raise TypeError(f"float8_e4m3fn inputs need out_dtype bfloat16 or float16, got {out_dtype}")
    return QkvQuantArgs(TFA_FP8_E4M3, float(q_scale), float(k_scale), float(v_scale)), out_dtype


def attn_fwd(q, k, v, is_causal, softmax_scale, num_splits=1, out_fp32=False, stream=None, return_splits=False,
             out=None, lse=None, q_scale=1.0, k_scale=1.0, v_scale=1.0, out_dtype=None):
    """Generalised problem through tfa_attn_fwd(): q (B,Hq,Sq,D), k/v (B,Hkv,Sk,D) contiguous device tensors,
    bottom-right causal mask, optional split-KV (num_splits: 1 none, n > 1 as asked, 0 library heuristic).  `out`
    (contiguous, q's shape) / `lse` (contiguous (B, Hq, Sq) fp32) may be given to write into caller-owned buffers.
    torch.float8_e4m3fn q / k / v go through tfa_attn_fp8_fwd() with the per-tensor q_scale / k_scale / v_scale and
    the output dtype out_dtype (bfloat16 or float16)."""
    import torch
    assert q.is_cuda and q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    B, Hq, Sq, D = q.shape
    _, Hkv, Sk, _ = k.shape
    if not (q.dtype == k.dtype == v.dtype):
        raise TypeError(f"q, k and v must share one dtype, got {q.dtype}, {k.dtype}, {v.dtype}")
    quant, odt = _qkv_quant(q, q_scale, k_scale, v_scale, out_dtype)
    if out is None:
        out = torch.empty(q.shape, dtype=torch.float32 if out_fp32 else odt, device=q.device)
    if lse is None:
        lse = torch.empty((B, Hq, Sq), dtype=torch.float32, device=q.device)
    assert out.shape == q.shape and out.is_contiguous() and out.dtype == (torch.float32 if out_fp32 else odt)
    assert lse.shape == (B, Hq, Sq) and lse.is_contiguous() and lse.dtype == torch.float32
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = AttnArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), B, Hq, Hkv, Sq, Sk, D,
                 Hq * Sq * D, Sq * D, D, Hkv * Sk * D, Sk * D, D,
                 (TFA_BF16 if odt == torch.bfloat16 else TFA_FP16) if quant else _dtype_code(q),
                 int(bool(is_causal)), float(softmax_scale), int(bool(out_fp32)), int(num_splits), None, 0, st)
    n = _split_workspace(a, a, q.device, st)
    if quant is not None:
        check(lib().tfa_attn_fp8_fwd(ctypes.byref(a), ctypes.byref(quant)))
    else:
        check(lib().tfa_attn_fwd(ctypes.byref(a)))
    if return_splits:
        return out, lse, n
    return out, lse


def attn_varlen_fwd(q, k, v, cu_q, cu_k, max_seqlen_q, is_causal, scale, out_fp32=False, out=None, lse=None,
                    stream=None, q_scale=1.0, k_scale=1.0, v_scale=1.0, out_dtype=None):
    """Packed variable-length batch through tfa_attn_varlen_fwd(): q (total_q, Hq, D), k/v (total_k, Hkv, D) device
    tensors with unit head_dim stride (views of a packed qkv tensor are fine; k and v share strides), cu_q / cu_k
    int32 device tensors of B + 1 offsets.  Returns out (total_q, Hq, D) and lse (Hq, total_q); `out` / `lse` may be
    given to write into caller-owned buffers.
    torch.float8_e4m3fn q / k / v go through tfa_attn_varlen_fp8_fwd() with the per-tensor q_scale / k_scale / v_scale
    and the output dtype out_dtype (bfloat16 or float16)."""
    import torch
    assert q.is_cuda and q.dim() == 3 and k.dim() == 3 and k.shape == v.shape and k.stride() == v.stride()
    assert q.stride(2) == 1 and k.stride(2) == 1
    assert cu_q.dtype == torch.int32 and cu_k.dtype == torch.int32 and cu_q.numel() == cu_k.numel() >= 2
    total_q, Hq, D = q.shape
    total_k, Hkv, _ = k.shape
    fp8 = [t.dtype == torch.float8_e4m3fn for t in (q, k, v)]
    if any(fp8) and not all(fp8):
        raise TypeError(f"q, k and v must all be float8_e4m3fn or none, got {q.dtype}, {k.dtype}, {v.dtype}")
    quant, odt = _qkv_quant(q, q_scale, k_scale, v_scale, out_dtype)
    if out is None:
        out = torch.empty((total_q, Hq, D), dtype=torch.float32 if out_fp32 else odt, device=q.device)
    if lse is None:
        lse = torch.empty((Hq, total_q), dtype=torch.float32, device=q.device)
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = VarlenArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), cu_q.data_ptr(),
                   cu_k.data_ptr(), cu_q.numel() - 1, Hq, Hkv, D, total_q, total_k, int(max_seqlen_q),
                   q.stride(0), q.stride(1), k.stride(0), k.stride(1),
                   (TFA_BF16 if odt == torch.bfloat16 else TFA_FP16) if quant else _dtype_code(q),
                   int(bool(is_causal)), float(scale), int(bool(out_fp32)), st)
    if quant is not None:
        check(lib().tfa_attn_varlen_fp8_fwd(ctypes.byref(a), ctypes.byref(quant)))
    else:
        check(lib().tfa_attn_varlen_fwd(ctypes.byref(a)))
    return out, lse


def _cache_args(block_table, k_new, v_new, new_dims):
    """What the two cache calls take of block_table, k_new and v_new: (max_blocks_per_seq, the table's row stride, its
    pointer), or (1, 1, None) for a contiguous cache; then the k_new / v_new pointers and k_new's first `new_dims`
    strides, or None, None and zeros without an append."""
    import torch
    if block_table is not None:
        assert block_table.dtype == torch.int32 and block_table.dim() == 2 and block_table.stride(1) == 1
        bt = (block_table.shape[1], block_table.stride(0), block_table.data_ptr())
    else:
        bt = (1, 1, None)
    if k_new is None:
        return bt, None, None, (0,) * new_dims
    assert k_new.shape == v_new.shape and k_new.stride() == v_new.stride() and k_new.stride(-1) == 1
    return bt, k_new.data_ptr(), v_new.data_ptr(), k_new.stride()[:new_dims]


def _quant(k_cache, k_scale, v_scale):
    """The tfa_kv_quant_args of an FP8 (torch.float8_e4m3fn) cache, or None for a 16-bit one, which takes no scales."""
    import torch
    if k_cache.dtype != torch.float8_e4m3fn:
        if k_scale != 1.0 or v_scale != 1.0:
            raise ValueError(f"k_scale / v_scale apply to a float8_e4m3fn cache only; this cache is {k_cache.dtype}")
        return None
    return KvQuantArgs(TFA_FP8_E4M3, float(k_scale), float(v_scale))


def _cache_quant(q, k_cache, k_new, rotary_cos, q_scale, k_scale, v_scale, out_dtype, q8_scale=None):
    """What a cache call takes of its element types and scales: (tfa_kv_quant_args or None, tfa_qkv_quant_args or None,
    the output dtype).  A float8_e4m3fn q needs a float8_e4m3fn cache (the e4m3-query calls, out in out_dtype, k_new in
    out_dtype) and takes no rotary; a 16-bit q takes a cache of its own dtype or an FP8 one, and no q_scale / out_dtype.
    q8_scale: a 16-bit q quantized with it for the e4m3-query calls on a float8_e4m3fn cache (out and k_new in q's
    dtype, rotary allowed)."""
    import torch
    if q8_scale is not None:
        if q.dtype == torch.float8_e4m3fn:
            raise ValueError("q8_scale quantizes a 16-bit q; this q is float8_e4m3fn already (pass q_scale)")
        if k_cache.dtype != torch.float8_e4m3fn:
            raise TypeError(f"q8_scale needs a float8_e4m3fn cache, got {k_cache.dtype}")
        if q_scale != 1.0 or out_dtype not in (None, q.dtype):
            raise ValueError(f"q_scale / out_dtype apply to a float8_e4m3fn q only; q is {q.dtype}")
        return None, QkvQuantArgs(TFA_FP8_E4M3, float(q8_scale), float(k_scale), float(v_scale)), q.dtype
    if q.dtype != torch.float8_e4m3fn:
        if q_scale != 1.0 or out_dtype not in (None, q.dtype):
            raise ValueError(f"q_scale / out_dtype apply to a float8_e4m3fn q only; q is {q.dtype}")
        return _quant(k_cache, k_scale, v_scale), None, q.dtype
    if k_cache.dtype != torch.float8_e4m3fn:
        raise TypeError(f"a float8_e4m3fn q needs a float8_e4m3fn cache, got {k_cache.dtype}")
    if rotary_cos is not None:
        raise ValueError("a float8_e4m3fn q takes no rotary: rotate q before quantizing it, or pass a 16-bit q")
    qkv8, odt = _qkv_quant(q, q_scale, k_scale, v_scale, out_dtype)
    if k_new is not None and k_new.dtype != odt:
        raise TypeError(f"k_new / v_new must have out_dtype {odt} with a float8_e4m3fn q, got {k_new.dtype}")
    return None, qkv8, odt


def _cache_dtype_code(q, qkv8, odt):
    """args->dtype of a cache call: q's, or with a float8_e4m3fn q (qkv8) the output's."""
    import torch
    if qkv8 is None:
        return _dtype_code(q)
    return TFA_BF16 if odt == torch.bfloat16 else TFA_FP16


def _rotary_args(q, rotary_cos, rotary_sin, rotary_interleaved, q_rot, stream, need_q_rot=True):
    """The RotaryArgs of a cache call with q (its q_rot: a contiguous tensor of q's shape and dtype, or a buffer
    allocated here and kept alive as the split workspace is; none unless given when not `need_q_rot`), or None without
    rotary_cos."""
    import torch
    if rotary_cos is None:
        return None
    assert rotary_sin is not None and rotary_cos.dim() == 2 and rotary_cos.shape == rotary_sin.shape
    assert rotary_cos.is_contiguous() and rotary_sin.is_contiguous()
    if q_rot is None and not need_q_rot:
        return RotaryArgs(rotary_cos.data_ptr(), rotary_sin.data_ptr(), rotary_cos.shape[0], 2 * rotary_cos.shape[1],
                          int(bool(rotary_interleaved)), None)
    if q_rot is None:
        q_rot = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        _WORKSPACES[("q_rot", q.device.index, int(stream))] = q_rot
    assert q_rot.shape == q.shape and q_rot.dtype == q.dtype and q_rot.is_contiguous()
    return RotaryArgs(rotary_cos.data_ptr(), rotary_sin.data_ptr(), rotary_cos.shape[0], 2 * rotary_cos.shape[1],
                      int(bool(rotary_interleaved)), q_rot.data_ptr())


def _q8_scratch(q, q8, stream):
    """The e4m3 scratch a 16-bit q is quantized into: `q8`, a contiguous float8_e4m3fn tensor of q's shape, or a buffer
    allocated here and kept alive as the split workspace is."""
    import torch
    if q8 is None:
        q8 = torch.empty(q.shape, dtype=torch.float8_e4m3fn, device=q.device)
        _WORKSPACES[("q8", q.device.index, int(stream))] = q8
    assert q8.shape == q.shape and q8.dtype == torch.float8_e4m3fn and q8.is_contiguous()
    return q8


def attn_kvcache_fwd(q, k_cache, v_cache, cache_seqlens, block_table=None, k_new=None, v_new=None, is_causal=False,
                     scale=None, num_splits=1, out_fp32=False, out=None, lse=None, stream=None, return_splits=False,
                     rotary_cos=None, rotary_sin=None, rotary_interleaved=False, q_rot=None, k_scale=1.0, v_scale=1.0,
                     q_scale=1.0, out_dtype=None, q8_scale=None, q8=None):
    """Attention against a KV cache through tfa_attn_kvcache_fwd(): q (B, Sq, Hq, D) with unit head_dim stride;
    k_cache / v_cache (num_blocks, page, Hkv, D) with a block_table (B, max_blocks_per_seq) int32, or (B, capacity,
    Hkv, D) with block_table None; cache_seqlens (B,) int32; optional k_new / v_new (B, Snew, Hkv, D) appended in
    place.  num_splits: 1 none, n > 1 as asked, 0 library heuristic (a workspace is allocated here when it splits).
    rotary_cos / rotary_sin (seqlen_ro, rotary_dim / 2) in q's dtype: rotate q and k_new first, through
    tfa_attn_kvcache_rotary_fwd().  The rotated queries go to `q_rot`, a contiguous (B, Sq, Hq, D) tensor of q's dtype
    that holds them after the call, or to a buffer allocated here.
    torch.float8_e4m3fn caches go through tfa_attn_kvcache_fp8_fwd() with the per-tensor k_scale / v_scale.  A
    torch.float8_e4m3fn q with them goes through tfa_attn_kvcache_qkv8_fwd() with q_scale too, the output (and k_new /
    v_new) in out_dtype (bfloat16 or float16), without rotary.  A 16-bit q with them and q8_scale goes through
    tfa_attn_kvcache_qkv8_q16_fwd(): q (rotated with rotary_cos / rotary_sin) is quantized with q8_scale into `q8`, a
    contiguous float8_e4m3fn tensor of q's shape that holds the codes after the call, or into a buffer allocated here.
    Returns out (q's shape and strides) and lse (B, Hq, Sq)."""
    import torch
    assert q.is_cuda and q.dim() == 4 and k_cache.dim() == 4 and k_cache.shape == v_cache.shape
    assert k_cache.stride() == v_cache.stride() and q.stride(3) == 1 and k_cache.stride(3) == 1
    assert cache_seqlens.dtype == torch.int32
    B, Sq, Hq, D = q.shape
    nblk, page, Hkv, _ = k_cache.shape
    quant, qkv8, odt = _cache_quant(q, k_cache, k_new, rotary_cos, q_scale, k_scale, v_scale, out_dtype, q8_scale)
    (mbps, bts, bt_ptr), nptr, vptr, ns = _cache_args(block_table, k_new, v_new, 3)
    snew = k_new.shape[1] if k_new is not None else 0
    if scale is None:
        scale = D ** -0.5
    if out is None:
        out = torch.empty_strided(q.shape, q.stride(), dtype=torch.float32 if out_fp32 else odt, device=q.device)
    if lse is None:
        lse = torch.empty((B, Hq, Sq), dtype=torch.float32, device=q.device)
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = KvcacheArgs(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), nptr, vptr, out.data_ptr(), lse.data_ptr(),
                    cache_seqlens.data_ptr(), bt_ptr, B, Hq, Hkv, Sq, D, nblk, page, mbps, snew,
                    q.stride(0), q.stride(1), q.stride(2), k_cache.stride(0), k_cache.stride(1), k_cache.stride(2),
                    bts, ns[0], ns[1], ns[2], _cache_dtype_code(q, qkv8, odt), int(bool(is_causal)), float(scale),
                    int(bool(out_fp32)), int(num_splits), None, 0, st)
    # the split count and workspace of the dense problem with Sk = capacity
    dense = AttnArgs(None, None, None, None, None, B, Hq, Hkv, Sq, mbps * page, D, 0, 0, 0, 0, 0, 0, 0,
                     int(bool(is_causal)), 0.0, 0, int(num_splits), None, 0, None)
    n = _split_workspace(dense, a, q.device, st)
    r = _rotary_args(q, rotary_cos, rotary_sin, rotary_interleaved, q_rot, st, q8_scale is None)
    if q8_scale is not None:
        q8 = _q8_scratch(q, q8, st)
        check(lib().tfa_attn_kvcache_qkv8_q16_fwd(ctypes.byref(a), ctypes.byref(r) if r is not None else None,
                                                  ctypes.byref(qkv8), q8.data_ptr()))
    elif qkv8 is not None:
        check(lib().tfa_attn_kvcache_qkv8_fwd(ctypes.byref(a), ctypes.byref(qkv8)))
    elif quant is not None:
        check(lib().tfa_attn_kvcache_fp8_fwd(ctypes.byref(a), ctypes.byref(r) if r is not None else None,
                                             ctypes.byref(quant)))
    elif r is None:
        check(lib().tfa_attn_kvcache_fwd(ctypes.byref(a)))
    else:
        check(lib().tfa_attn_kvcache_rotary_fwd(ctypes.byref(a), ctypes.byref(r)))
    if return_splits:
        return out, lse, n
    return out, lse


def attn_varlen_kvcache_fwd(q, k_cache, v_cache, cu_q, max_seqlen_q, cache_seqlens, block_table=None, k_new=None,
                            v_new=None, is_causal=False, scale=None, out_fp32=False, out=None, lse=None, stream=None,
                            k_scale=1.0, v_scale=1.0, rotary_cos=None, rotary_sin=None, rotary_interleaved=False,
                            q_rot=None, q_scale=1.0, out_dtype=None, q8_scale=None, q8=None, num_splits=1,
                            return_splits=False, workspace=None):
    """A packed variable-length batch of queries against a KV cache through tfa_attn_varlen_kvcache_fwd(): q
    (total_q, Hq, D) with unit head_dim stride and cu_q int32 (B + 1) offsets, as attn_varlen_fwd; k_cache / v_cache
    and block_table as attn_kvcache_fwd; cache_seqlens (B,) int32; optional k_new / v_new packed (total_q, Hkv, D),
    sharing cu_q, appended in place.  torch.float8_e4m3fn caches go through tfa_attn_varlen_kvcache_fp8_fwd() with
    the per-tensor k_scale / v_scale.  rotary_cos / rotary_sin (seqlen_ro, rotary_dim / 2) in q's dtype: rotate q and
    k_new first, through tfa_attn_varlen_kvcache_rotary_fwd() (with `quant` for an FP8 cache).  The rotated queries go
    to `q_rot`, a contiguous (total_q, Hq, D) tensor of q's dtype, or to a buffer allocated here.  A
    torch.float8_e4m3fn q with an FP8 cache goes through tfa_attn_varlen_kvcache_qkv8_fwd() as attn_kvcache_fwd's, and
    a 16-bit q with q8_scale through tfa_attn_varlen_kvcache_qkv8_q16_fwd() (`q8`: (total_q, Hq, D)) as its.
    num_splits != 1 takes the split-KV forms (tfa_attn_varlen_kvcache_split_fwd() /
    tfa_attn_varlen_kvcache_qkv8_split_fwd()): n > 1 as asked, 0 library heuristic, with a workspace allocated here
    when it splits, or the caller's `workspace` (a device tensor, passed as is with num_splits; given, it takes the
    split-KV form at num_splits = 1 too).  Returns out (total_q, Hq, D) and lse (Hq, total_q), and with return_splits the split count;
    `out` / `lse` may be given to write into caller-owned buffers."""
    import torch
    assert q.is_cuda and q.dim() == 3 and k_cache.dim() == 4 and k_cache.shape == v_cache.shape
    assert k_cache.stride() == v_cache.stride() and q.stride(2) == 1 and k_cache.stride(3) == 1
    assert cu_q.dtype == torch.int32 and cu_q.numel() >= 2 and cache_seqlens.dtype == torch.int32
    total_q, Hq, D = q.shape
    nblk, page, Hkv, _ = k_cache.shape
    quant, qkv8, odt = _cache_quant(q, k_cache, k_new, rotary_cos, q_scale, k_scale, v_scale, out_dtype, q8_scale)
    (mbps, bts, bt_ptr), nptr, vptr, ns = _cache_args(block_table, k_new, v_new, 2)
    if scale is None:
        scale = D ** -0.5
    if out is None:
        out = torch.empty((total_q, Hq, D), dtype=torch.float32 if out_fp32 else odt, device=q.device)
    if lse is None:
        lse = torch.empty((Hq, total_q), dtype=torch.float32, device=q.device)
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = VarlenKvcacheArgs(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), nptr, vptr, out.data_ptr(),
                          lse.data_ptr(), cu_q.data_ptr(), cache_seqlens.data_ptr(), bt_ptr, cu_q.numel() - 1, Hq, Hkv,
                          D, total_q, int(max_seqlen_q), nblk, page, mbps, q.stride(0), q.stride(1),
                          k_cache.stride(0), k_cache.stride(1), k_cache.stride(2), bts, ns[0], ns[1],
                          _cache_dtype_code(q, qkv8, odt),
                          int(bool(is_causal)), float(scale), int(bool(out_fp32)), st)
    r = _rotary_args(q, rotary_cos, rotary_sin, rotary_interleaved, q_rot, st, q8_scale is None)
    if num_splits != 1 or workspace is not None:
        n = _varlen_split(a, num_splits, q.device, st, q, q8, q8_scale, qkv8, quant, r, workspace)
        return (out, lse, n) if return_splits else (out, lse)
    if q8_scale is not None:
        q8 = _q8_scratch(q, q8, st)
        check(lib().tfa_attn_varlen_kvcache_qkv8_q16_fwd(ctypes.byref(a), ctypes.byref(r) if r is not None else None,
                                                         ctypes.byref(qkv8), q8.data_ptr()))
    elif qkv8 is not None:
        check(lib().tfa_attn_varlen_kvcache_qkv8_fwd(ctypes.byref(a), ctypes.byref(qkv8)))
    elif r is not None:
        check(lib().tfa_attn_varlen_kvcache_rotary_fwd(ctypes.byref(a), ctypes.byref(r),
                                                       ctypes.byref(quant) if quant is not None else None))
    elif quant is not None:
        check(lib().tfa_attn_varlen_kvcache_fp8_fwd(ctypes.byref(a), ctypes.byref(quant)))
    else:
        check(lib().tfa_attn_varlen_kvcache_fwd(ctypes.byref(a)))
    return (out, lse, 1) if return_splits else (out, lse)


def _varlen_split(a, num_splits, device, stream, q, q8, q8_scale, qkv8, quant, r, workspace):
    """The split-KV form of attn_varlen_kvcache_fwd's call on the filled argument struct `a`; returns the split count."""
    import torch
    L = lib()
    n = int(L.tfa_attn_varlen_kvcache_num_splits(ctypes.byref(a), int(num_splits)))
    sp = SplitArgs(int(num_splits), None, 0)
    if workspace is not None:
        sp = SplitArgs(int(num_splits), workspace.data_ptr() if workspace.numel() else None,
                       workspace.numel() * workspace.element_size())
    elif n > 1:
        need = int(L.tfa_attn_varlen_kvcache_workspace_bytes(ctypes.byref(a), n))
        ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=device)
        sp = SplitArgs(n, ws.data_ptr(), need)
        _WORKSPACES[(device.index, int(stream))] = ws       # kept alive as _split_workspace keeps its own
    rp = ctypes.byref(r) if r is not None else None
    if q8_scale is not None:
        q8 = _q8_scratch(q, q8, stream)
        check(L.tfa_attn_varlen_kvcache_qkv8_split_fwd(ctypes.byref(a), rp, ctypes.byref(qkv8), q8.data_ptr(),
                                                       ctypes.byref(sp)))
    elif qkv8 is not None:
        check(L.tfa_attn_varlen_kvcache_qkv8_split_fwd(ctypes.byref(a), None, ctypes.byref(qkv8), None,
                                                       ctypes.byref(sp)))
    else:
        check(L.tfa_attn_varlen_kvcache_split_fwd(ctypes.byref(a), rp, ctypes.byref(quant) if quant is not None else None,
                                                  ctypes.byref(sp)))
    return n


def fwd_multi(q, k, v, is_causal, softmax_scale, out, extra_ptrs, lse=None, stream=None):
    """Fused compute + exchange: like fwd() on (B,H,S,D) device tensors, and the same kernel also stores every chunk
    of O to the raw device addresses in `extra_ptrs` (peer GPUs' buffers with the same strides, <= 7 of them)."""
    import torch
    B, H, S, D = q.shape
    if lse is None:
        lse = torch.empty((B, H, S), dtype=torch.float32, device=q.device)
    st = stream if stream is not None else torch.cuda.current_stream(q.device).cuda_stream
    a = FwdArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), B, H, S, D, H * S * D, S * D, D,
                _dtype_code(q), int(bool(is_causal)), float(softmax_scale), 0, st)
    n = len(extra_ptrs)
    arr = (ctypes.c_void_p * max(n, 1))(*[ctypes.c_void_p(int(x)) for x in extra_ptrs])
    check(lib().tfa_fwd_multi(ctypes.byref(a), arr, n))
    return out, lse


def fwd_host(q, k, v, out, lse, is_causal, softmax_scale, n_chunks=8):
    """HOST (ideally pinned) (B,H,S,D) tensors in, results written into host `out` / `lse`;
    H2D, kernel and D2H are all inside the call (the e2e path bench.py times)."""
    assert not q.is_cuda and not out.is_cuda
    B, H, S, D = q.shape
    check(lib().tfa_fwd_host(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(),
                             lse.data_ptr() if lse is not None else None, B, H, S, D, _dtype_code(q),
                             int(bool(is_causal)), float(softmax_scale), int(n_chunks)))
    return out, lse


def launch_count() -> int:
    return int(lib().tfa_launch_count())
