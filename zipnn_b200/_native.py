"""ctypes binding of libzipnn_b200.so (the C ABI in include/zipnn_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is
visible, the codec raises.  The library is built in-tree by `build()` (also called by
`__graft_entry__.build()`), so it travels with the source tree.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libzipnn_b200.so")
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-diag-suppress", "128", "-Xcompiler", "-fPIC", "-shared"]

OK, E_ARG, E_CAPACITY, E_CORRUPT, E_CUDA, E_UNSUPPORTED, E_INDEX = 0, 1, 2, 3, 4, 5, 6
MATVEC_MAX_TOKENS = 8   # ZIPNN_B200_MATVEC_MAX_TOKENS
EXPERTS_MATVEC_MAX_TOKENS = 4   # ZIPNN_B200_EXPERTS_MATVEC_MAX_TOKENS
MATMUL_MAX_TOKENS = 64  # ZIPNN_B200_MATMUL_MAX_TOKENS
FP8_E4M3, FP8_E5M2 = 0, 1   # ZIPNN_B200_FP8_E4M3 / _E5M2

_lib = None
_lock = threading.Lock()


class BatchItem(C.Structure):
    """zipnn_b200_batch_item (include/zipnn_b200.h)."""
    _fields_ = [("d_body", C.c_void_p), ("body_len", C.c_size_t), ("num_buf", C.c_int), ("bits_mode", C.c_int),
                ("bytes_mode", C.c_int), ("chunk", C.c_size_t), ("orig", C.c_size_t), ("d_out", C.c_void_p)]


class SliceItem(C.Structure):
    """zipnn_b200_slice_item (include/zipnn_b200.h)."""
    _fields_ = [("d_body", C.c_void_p), ("body_len", C.c_size_t), ("num_buf", C.c_int), ("bits_mode", C.c_int),
                ("bytes_mode", C.c_int), ("chunk", C.c_size_t), ("orig", C.c_size_t), ("base", C.c_size_t),
                ("rows", C.c_size_t), ("pitch", C.c_size_t), ("len", C.c_size_t), ("d_out", C.c_void_p)]


class CompressItem(C.Structure):
    """zipnn_b200_compress_item (include/zipnn_b200.h)."""
    _fields_ = [("d_in", C.c_void_p), ("n", C.c_size_t), ("h_hdr", C.c_void_p), ("hdr_len", C.c_size_t),
                ("num_buf", C.c_int), ("bits_mode", C.c_int), ("bytes_mode", C.c_int), ("chunk", C.c_size_t),
                ("threshold", C.c_float), ("d_out", C.c_void_p), ("out_cap", C.c_size_t)]


class Fp8SelectItem(C.Structure):
    """zipnn_b200_fp8_select_item (include/zipnn_b200.h)."""
    _fields_ = [("in_features", C.c_size_t), ("d_scale", C.c_void_p), ("block_rows", C.c_size_t), ("block_cols", C.c_size_t),
                ("d_out", C.c_void_p)]


class DecodePlanStruct(C.Structure):
    """zipnn_b200_decode_plan (include/zipnn_b200.h): host memory, filled by zipnn_b200_decode_plan_create."""
    _fields_ = [("opaque", C.c_uint64 * 16)]


class ZipNNNativeError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"zipnn_b200: {msg} (status {status})")
        self.status = status


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".inc"))] + \
        [os.path.join(os.path.dirname(_HERE), "include", "zipnn_b200.h")]


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/zipnn_b200.cu for sm_90a into csrc/libzipnn_b200.so (no GPU needed)."""
    newest = max(os.path.getmtime(p) for p in sources())
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= newest:
        return LIB_PATH
    nvcc = os.environ.get("NVCC") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH, os.path.join(CSRC, "zipnn_b200.cu")]
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB_PATH


def lib() -> C.CDLL:
    """Load the shared library (building it first if the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            try:
                build()   # no-op when the library is newer than every source file
            except Exception as exc:  # pragma: no cover
                if not os.path.exists(LIB_PATH):
                    raise ZipNNNativeError(-1, f"libzipnn_b200.so is missing and could not be built: {exc}") from exc
                import warnings
                warnings.warn(f"zipnn_b200: libzipnn_b200.so looks older than its sources and could not be rebuilt ({exc}); loading it as is")
            # experiments only: a variant build of the same sources (tools/decode_probe.py)
            L = C.CDLL(os.environ.get("ZIPNN_B200_LIB_VARIANT") or LIB_PATH)
            vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
            szp = C.POINTER(C.c_size_t)
            sig = {
                "zipnn_b200_version": (i32, []),
                "zipnn_b200_strerror": (C.c_char_p, [i32]),
                "zipnn_b200_last_cuda_error": (i32, []),
                "zipnn_b200_sm_count": (i32, []),
                "zipnn_b200_peek": (i32, [vp, sz, vp, vp]),
                "zipnn_b200_launch_count": (C.c_ulonglong, []),
                "zipnn_b200_compress_bound": (i32, [sz, i32, sz, sz, szp]),
                "zipnn_b200_compress_workspace_size": (i32, [sz, i32, sz, szp]),
                "zipnn_b200_decompress_workspace_size": (i32, [sz, i32, sz, szp]),
                "zipnn_b200_decompress_workspace_size_full": (i32, [sz, i32, sz, szp]),
                "zipnn_b200_compress": (i32, [vp, sz, vp, sz, i32, i32, i32, sz, C.c_float, vp, sz, szp, vp, sz, vp]),
                "zipnn_b200_compress_batch_workspace_size": (i32, [C.POINTER(CompressItem), i32, szp]),
                "zipnn_b200_compress_batch": (i32, [C.POINTER(CompressItem), i32, szp, vp, sz, vp]),
                "zipnn_b200_decompress": (i32, [vp, sz, i32, i32, i32, sz, sz, vp, vp, sz, vp, i32]),
                "zipnn_b200_decompress_batch_workspace_size": (i32, [C.POINTER(BatchItem), i32, szp]),
                "zipnn_b200_decompress_batch": (i32, [C.POINTER(BatchItem), i32, vp, sz, vp, i32]),
                "zipnn_b200_decompress_slices_workspace_size": (i32, [C.POINTER(SliceItem), i32, szp]),
                "zipnn_b200_decompress_slices": (i32, [C.POINTER(SliceItem), i32, vp, sz, vp, i32]),
                "zipnn_b200_decode_plan_size": (i32, [C.POINTER(SliceItem), i32, vp, szp, szp]),
                "zipnn_b200_decode_plan_create": (i32, [C.POINTER(SliceItem), i32, vp, sz, vp, sz, C.POINTER(DecodePlanStruct), vp]),
                "zipnn_b200_decode_plan_run": (i32, [C.POINTER(DecodePlanStruct), vp]),
                "zipnn_b200_decode_plan_status": (i32, [C.POINTER(DecodePlanStruct), vp]),
                "zipnn_b200_decode_plan_index": (i32, [C.POINTER(DecodePlanStruct), szp, szp]),
                "zipnn_b200_decode_plan_run_shifted": (i32, [C.POINTER(DecodePlanStruct), C.c_int64, i32, vp]),
                "zipnn_b200_decode_plan_gather_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, sz, sz, szp]),
                "zipnn_b200_decode_plan_gather": (i32, [C.POINTER(DecodePlanStruct), i32, sz, vp, sz, i32, vp, vp, sz, vp]),
                "zipnn_b200_decode_plan_select_scratch_size": (i32, [C.POINTER(DecodePlanStruct), sz, szp]),
                "zipnn_b200_decode_plan_run_select": (i32, [C.POINTER(DecodePlanStruct), sz, vp, sz, i32, vp, sz, vp]),
                "zipnn_b200_decode_plan_matvec_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, i32, sz, sz, szp]),
                "zipnn_b200_decode_plan_matvec": (i32, [C.POINTER(DecodePlanStruct), i32, i32, sz, vp, sz, sz, vp, vp, sz, vp, sz, vp]),
                "zipnn_b200_decode_plan_matmul_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, i32, sz, sz, szp]),
                "zipnn_b200_decode_plan_matmul": (i32, [C.POINTER(DecodePlanStruct), i32, i32, sz, vp, sz, sz, vp, vp, sz, vp, sz, vp]),
                "zipnn_b200_decode_plan_matvec_fp8_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, sz, sz, szp]),
                "zipnn_b200_decode_plan_matvec_fp8": (i32, [C.POINTER(DecodePlanStruct), i32, i32, i32, sz, vp, sz, sz, vp, sz, sz, vp, vp, sz,
                                                             vp, sz, vp]),
                "zipnn_b200_decode_plan_matmul_fp8_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, sz, sz, szp]),
                "zipnn_b200_decode_plan_matmul_fp8": (i32, [C.POINTER(DecodePlanStruct), i32, i32, i32, sz, vp, sz, sz, vp, sz, sz, vp, vp, sz,
                                                             vp, sz, vp]),
                "zipnn_b200_decode_plan_dequant_fp8": (i32, [C.POINTER(DecodePlanStruct), i32, i32, i32, sz, vp, sz, sz, vp, vp]),
                "zipnn_b200_decode_plan_dequant_fp8_select": (i32, [C.POINTER(DecodePlanStruct), sz, vp, sz, i32, i32, i32, i32,
                                                                    C.POINTER(Fp8SelectItem), vp, sz, vp]),
                "zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size": (i32, [C.POINTER(DecodePlanStruct), i32, sz, sz, sz, sz, szp]),
                "zipnn_b200_decode_plan_experts_matvec_fp8": (i32, [C.POINTER(DecodePlanStruct), i32, sz, vp, sz, i32, sz, i32, i32, sz,
                                                                    vp, sz, i32, vp, sz, sz, vp, sz, vp, sz, vp]),
                "zipnn_b200_split": (i32, [vp, sz, i32, i32, vp, sz, vp]),
                "zipnn_b200_regroup": (i32, [vp, sz, sz, i32, i32, vp, vp]),
                "zipnn_b200_compress_host": (i32, [vp, sz, vp, sz, i32, i32, i32, sz, C.c_float, vp, sz, szp]),
                "zipnn_b200_decompress_host": (i32, [vp, sz, i32, i32, i32, sz, sz, vp]),
                "zipnn_b200_timing_enable": (None, [i32]),
                "zipnn_b200_timing_kernel_count": (i32, []),
                "zipnn_b200_timing_kernel_name": (C.c_char_p, [i32]),
                "zipnn_b200_timing_collect": (i32, [C.POINTER(C.c_double), C.POINTER(C.c_ulonglong), i32]),
            }
            for name, (res, args) in sig.items():
                f = getattr(L, name)
                f.restype, f.argtypes = res, args
            _lib = L
    return _lib


EXPORTS = [
    "zipnn_b200_version", "zipnn_b200_strerror", "zipnn_b200_last_cuda_error", "zipnn_b200_sm_count", "zipnn_b200_peek",
    "zipnn_b200_launch_count", "zipnn_b200_compress_bound", "zipnn_b200_compress_workspace_size",
    "zipnn_b200_decompress_workspace_size", "zipnn_b200_decompress_workspace_size_full", "zipnn_b200_compress",
    "zipnn_b200_compress_batch_workspace_size", "zipnn_b200_compress_batch", "zipnn_b200_decompress", "zipnn_b200_decompress_batch_workspace_size", "zipnn_b200_decompress_batch",
    "zipnn_b200_decompress_slices_workspace_size", "zipnn_b200_decompress_slices", "zipnn_b200_decode_plan_size",
    "zipnn_b200_decode_plan_create", "zipnn_b200_decode_plan_run", "zipnn_b200_decode_plan_status", "zipnn_b200_decode_plan_index", "zipnn_b200_decode_plan_run_shifted",
    "zipnn_b200_decode_plan_gather_scratch_size", "zipnn_b200_decode_plan_gather",
    "zipnn_b200_decode_plan_select_scratch_size", "zipnn_b200_decode_plan_run_select",
    "zipnn_b200_decode_plan_matvec_scratch_size", "zipnn_b200_decode_plan_matvec",
    "zipnn_b200_decode_plan_matmul_scratch_size", "zipnn_b200_decode_plan_matmul",
    "zipnn_b200_decode_plan_matvec_fp8_scratch_size", "zipnn_b200_decode_plan_matvec_fp8",
    "zipnn_b200_decode_plan_matmul_fp8_scratch_size", "zipnn_b200_decode_plan_matmul_fp8",
    "zipnn_b200_decode_plan_dequant_fp8", "zipnn_b200_decode_plan_dequant_fp8_select",
    "zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size", "zipnn_b200_decode_plan_experts_matvec_fp8", "zipnn_b200_split", "zipnn_b200_regroup", "zipnn_b200_compress_host", "zipnn_b200_decompress_host",
    "zipnn_b200_timing_enable", "zipnn_b200_timing_kernel_count", "zipnn_b200_timing_kernel_name",
    "zipnn_b200_timing_collect",
]


def check(status: int) -> None:
    if status == OK:
        return
    L = lib()
    msg = L.zipnn_b200_strerror(status).decode()
    if status == E_CUDA:
        msg += f" (cudaError {L.zipnn_b200_last_cuda_error()})"
    if status == E_CORRUPT:
        raise ZipNNNativeError(status, msg)
    raise ZipNNNativeError(status, msg)


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise ZipNNNativeError(E_CUDA, "no CUDA device: zipnn_b200 has no CPU fallback")


# The sizes depend on the arguments alone: kept, so that a call in a loop asks the library once.
@functools.lru_cache(maxsize=256)
def compress_bound(n: int, num_buf: int, chunk: int, hdr_len: int) -> int:
    out = C.c_size_t(0)
    check(lib().zipnn_b200_compress_bound(n, num_buf, chunk, hdr_len, C.byref(out)))
    return out.value


@functools.lru_cache(maxsize=256)
def compress_workspace_size(n: int, num_buf: int, chunk: int) -> int:
    out = C.c_size_t(0)
    check(lib().zipnn_b200_compress_workspace_size(n, num_buf, chunk, C.byref(out)))
    return out.value


@functools.lru_cache(maxsize=256)
def decompress_workspace_size(orig: int, num_buf: int, chunk: int, full: bool = False) -> int:
    out = C.c_size_t(0)
    f = lib().zipnn_b200_decompress_workspace_size_full if full else lib().zipnn_b200_decompress_workspace_size
    check(f(orig, num_buf, chunk, C.byref(out)))
    return out.value


def launch_count() -> int:
    return int(lib().zipnn_b200_launch_count())


def timing_enable(on: bool) -> None:
    lib().zipnn_b200_timing_enable(1 if on else 0)


def timing_collect() -> dict:
    """-> {kernel name: (total ms, launches)} since the last collect; synchronises the device."""
    L = lib()
    k = L.zipnn_b200_timing_kernel_count()
    ms = (C.c_double * k)()
    cnt = (C.c_ulonglong * k)()
    check(L.zipnn_b200_timing_collect(ms, cnt, k))
    return {L.zipnn_b200_timing_kernel_name(i).decode(): (ms[i], int(cnt[i])) for i in range(k)}
