"""ctypes front-end for the test oracle (TEST INFRASTRUCTURE ONLY).

Two checkers live here:

* ``port``  -- ``libzipnn_oracle.so``, our plain-C restatement of the reference
  algorithm (``zipnn_oracle.c``; every function cites the reference file:line).
* ``ref``   -- ``_ref/zipnn_core*.so``, the UNMODIFIED reference C extension
  compiled from ``/root/reference`` by ``make -C oracle ref`` (git-ignored,
  shipped to the GPU box as a binary).  Optional: ``ref_core()`` returns None
  when it has not been built.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import this module.  The product package
``zipnn_b200`` never does.
"""
from __future__ import annotations

import ctypes as C
import importlib.util
import os
import subprocess
import sysconfig

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
ERR = C.c_size_t(-1).value


def build(ref: bool = True) -> None:
    """Compile the restatement, and the reference itself when its sources are present."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "all"])
    if ref and os.path.isdir("/root/reference/csrc"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libzipnn_oracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = C.CDLL(path)
        u8p = C.c_void_p
        L.zo_huf_compress.restype = C.c_size_t
        L.zo_huf_compress.argtypes = [u8p, C.c_size_t, u8p, C.c_size_t]
        L.zo_huf_decompress.restype = C.c_size_t
        L.zo_huf_decompress.argtypes = [u8p, C.c_size_t, u8p, C.c_size_t]
        L.zo_huf_table_from_counts.restype = C.c_size_t
        L.zo_huf_table_from_counts.argtypes = [u8p, C.c_uint, C.c_size_t, u8p, u8p, u8p, C.c_size_t, u8p]
        L.zo_compress_bound.restype = C.c_size_t
        L.zo_compress_bound.argtypes = [C.c_size_t, C.c_int, C.c_size_t, C.c_size_t]
        L.zo_zipnn_compress.restype = C.c_longlong
        L.zo_zipnn_compress.argtypes = [u8p, C.c_size_t, u8p, C.c_size_t, C.c_int, C.c_int, C.c_int,
                                        C.c_size_t, C.c_float, u8p, C.c_size_t, C.c_int]
        L.zo_zipnn_decompress.restype = C.c_int
        L.zo_zipnn_decompress.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_size_t,
                                          C.c_size_t, u8p, C.c_int]
        L.zo_huf_read_table.restype = C.c_size_t
        L.zo_huf_read_table.argtypes = [u8p, C.c_size_t, u8p, u8p, u8p]
        L.zo_split_chunk.restype = None
        L.zo_split_chunk.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, u8p, C.c_size_t]
        _LIB = L
    return _LIB


def _u8(a) -> np.ndarray:
    if isinstance(a, np.ndarray):
        return np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return np.frombuffer(a, dtype=np.uint8)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------- port: HUF block level
def huf_compress(src, cap: int | None = None):
    """Restatement of HUF_compress.  -> (ret, bytes) with ret 0=raw, 1=RLE, ERR=error."""
    s = _u8(src)
    cap = cap if cap is not None else 256 * 1024
    dst = np.zeros(cap + 64, dtype=np.uint8)
    r = lib().zo_huf_compress(_ptr(dst), cap, _ptr(s), s.size)
    if r == ERR or r == 0:
        return r, b""
    return r, dst[:r].tobytes()


def huf_decompress(src, n: int):
    s = _u8(src)
    dst = np.zeros(max(n, 1), dtype=np.uint8)
    r = lib().zo_huf_decompress(_ptr(dst), n, _ptr(s), s.size)
    if r == ERR:
        raise ValueError("oracle: corrupt HUF block")
    return dst[:n]


def huf_read_table(block):
    """Table description at the start of a HUF block -> (size in bytes, weights[nsym], tableLog)."""
    s = _u8(block)
    w = np.zeros(256, dtype=np.uint8)
    nsym = np.zeros(1, dtype=np.uint32)
    log = np.zeros(1, dtype=np.uint32)
    h = lib().zo_huf_read_table(_ptr(s), s.size, _ptr(w), _ptr(nsym), _ptr(log))
    if h == ERR:
        raise ValueError("oracle: corrupt HUF table description")
    return int(h), w[: int(nsym[0])].copy(), int(log[0])


def huf_table_from_counts(counts, n: int):
    """-> (nbBits[256], val[256], header bytes or None on error, tableLog)."""
    cnt = np.ascontiguousarray(counts, dtype=np.uint32)
    nz = np.nonzero(cnt)[0]
    max_sym = int(nz[-1])
    nb = np.zeros(256, dtype=np.uint8)
    val = np.zeros(256, dtype=np.uint16)
    hdr = np.zeros(512, dtype=np.uint8)
    log = np.zeros(1, dtype=np.uint32)
    h = lib().zo_huf_table_from_counts(_ptr(cnt), max_sym, n, _ptr(nb), _ptr(val), _ptr(hdr), 512, _ptr(log))
    return nb, val, (None if h == ERR else hdr[:h].tobytes()), int(log[0])


# ---------------------------------------------------------------- port: stream level
def split_chunk(chunk_bytes, G: int, bits_mode: int):
    s = _u8(chunk_bytes)
    stride = s.size // G + 1
    planes = np.zeros(G * stride, dtype=np.uint8)
    lib().zo_split_chunk(_ptr(s), s.size, G, bits_mode, _ptr(planes), stride)
    return [planes[g * stride: g * stride + s.size // G + (1 if g < s.size % G else 0)].copy() for g in range(G)]


def zipnn_compress(header, data, num_buf: int, bits_mode: int, bytes_mode: int, chunk: int,
                   threshold: float = 0.95, threads: int = 1) -> np.ndarray:
    """Restatement of zipnn_core.zipnn_core(header, data, ...) -> full stream (uint8 array)."""
    h = _u8(bytes(header))
    d = _u8(data)
    cap = lib().zo_compress_bound(d.size, num_buf, chunk, h.size)
    out = np.empty(cap + 64, dtype=np.uint8)
    r = lib().zo_zipnn_compress(_ptr(h), h.size, _ptr(d), d.size, num_buf, bits_mode, bytes_mode, chunk,
                                threshold, _ptr(out), cap, threads)
    if r < 0:
        raise RuntimeError("oracle compress failed")
    return out[:r]


def zipnn_decompress(body, num_buf: int, bits_mode: int, bytes_mode: int, chunk: int, orig: int,
                     threads: int = 1) -> np.ndarray:
    """Restatement of zipnn_core.combine_dtype(stream_after_header, ...)."""
    b = _u8(body)
    out = np.empty(max(orig, 1), dtype=np.uint8)
    r = lib().zo_zipnn_decompress(_ptr(b), b.size, num_buf, bits_mode, bytes_mode, chunk, orig, _ptr(out), threads)
    if r != 0:
        raise RuntimeError("oracle decompress failed")
    return out[:orig]


# ---------------------------------------------------------------- ref: the compiled reference
_REF = None
_REF_TRIED = False


def ref_path() -> str:
    return os.path.join(_HERE, "_ref", "zipnn_core" + sysconfig.get_config_var("EXT_SUFFIX"))


def ref_core():
    """The reference's own `zipnn_core` extension module, or None if not built."""
    global _REF, _REF_TRIED
    if not _REF_TRIED:
        _REF_TRIED = True
        p = ref_path()
        if os.path.exists(p):
            spec = importlib.util.spec_from_file_location("zipnn_core", p)
            m = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(m)
            _REF = m
    return _REF


def ref_cdll():
    """ctypes view of the same .so: HUF_compress, HUF_decompress and its two decoders (4X1: one symbol per
    table cell, 4X2: two) are exported."""
    p = ref_path()
    if not os.path.exists(p):
        return None
    L = C.CDLL(p)
    for name in ("HUF_compress", "HUF_decompress", "HUF_decompress4X1", "HUF_decompress4X2"):
        f = getattr(L, name)
        f.restype = C.c_size_t
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.HUF_isError.restype = C.c_uint
    L.HUF_isError.argtypes = [C.c_size_t]
    return L


def ref_huf_compress(src, cap: int = 256 * 1024):
    L = ref_cdll()
    s = _u8(src)
    dst = np.zeros(cap + 64, dtype=np.uint8)
    r = L.HUF_compress(_ptr(dst), cap, _ptr(s), s.size)
    if L.HUF_isError(r):
        return ERR, b""
    if r == 0:
        return 0, b""
    return r, dst[:r].tobytes()


def ref_huf_decoders(block, n: int) -> dict:
    """What the reference's HUF_decompress, HUF_decompress4X1 and HUF_decompress4X2 make of one block for an n-byte
    destination: {name: the decoded bytes, or None when it reports an error}."""
    L = ref_cdll()
    s = _u8(block)
    out = {}
    for name in ("HUF_decompress", "HUF_decompress4X1", "HUF_decompress4X2"):
        dst = np.zeros(max(n, 1) + 64, dtype=np.uint8)
        r = getattr(L, name)(_ptr(dst), n, _ptr(s), s.size)
        out[name] = None if L.HUF_isError(r) or r != n else dst[:n].tobytes()
    return out
