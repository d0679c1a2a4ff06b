"""Sliced reads of compressed tensors: decode only the chunks an index touches.

A ZipNN stream is a sequence of independent chunks of the tensor's bytes, so an index into a row-major tensor is
a *box* over the decoded bytes: row r is [base + r * pitch, base + r * pitch + len), r in [0, rows).  The kernels
(`zipnn_b200_decompress_slices`, include/zipnn_b200.h) decode the chunks the box meets and write only its bytes.

  * `plan_index` turns (shape, element size, index) into the box, the shape of the result and a residual (steps and
    restrictions the box cannot express, applied with torch indexing to the decoded box);
  * `StreamIndex` holds the header and size tables of one stream; `read_substream` reads only the payload of a
    chunk range and lays it out as a self-contained stream (size rows rebased), ready for one H2D copy;
  * `slice_stream` is `ZipNN.decompress_slice`; `CompressedSlice` is what `SafeOpen(..., slices=True).get_slice`
    returns for a compressed entry.
"""
from __future__ import annotations

import ctypes as C
import math
import operator
import os
from typing import NamedTuple

import numpy as np
import torch

from . import _native
from .util_header import EnumFormat
from .util_torch import torch_dtype_of_code

_ST_DTYPES = {torch.float64: "F64", torch.float32: "F32", torch.float16: "F16", torch.bfloat16: "BF16",
              torch.float8_e4m3fn: "F8_E4M3", torch.float8_e5m2: "F8_E5M2"}


# ---------------------------------------------------------------------------------------------- index planning
class Residual(NamedTuple):
    view: tuple          # the decoded box as (rows, elements of the restricted dim it spans, *inner dims)
    rows: object         # numpy int64 array of the box rows the index selects, or None for all of them
    step: int            # step inside the restricted dim


class SlicePlan(NamedTuple):
    box: tuple           # (base, rows, pitch, len) in bytes of the decoded tensor
    out_shape: tuple
    residual: Residual   # None: the box, reshaped to out_shape, is the result


def _dims(shape, index):
    """Per dim (start, count, step, kept) with the semantics of safetensors' PySafeSlice.__getitem__: ints (negative
    ones count from the end) drop their dim, slices take positive steps, one Ellipsis stands for the missing dims."""
    if not isinstance(index, tuple):
        index = (index,)
    n_ell = sum(1 for x in index if x is Ellipsis)
    if n_ell > 1:
        raise IndexError("an index can only have a single ellipsis ('...')")
    n_real = len(index) - n_ell
    if n_real > len(shape):
        raise IndexError(f"too many indices for tensor of dimension {len(shape)}")
    fill = (slice(None),) * (len(shape) - n_real)
    if n_ell:
        at = index.index(Ellipsis)
        index = index[:at] + fill + index[at + 1:]
    else:
        index = index + fill
    dims = []
    for d, (x, size) in enumerate(zip(index, shape)):
        if isinstance(x, slice):
            if x.step is not None and operator.index(x.step) <= 0:
                raise ValueError("step must be greater than zero")
            start, stop, step = x.indices(size)
            dims.append((start, len(range(start, stop, step)), step, True))
        else:
            i = operator.index(x)
            if not -size <= i < size:
                raise IndexError(f"index {i} is out of bounds for dimension {d} with size {size}")
            dims.append((i + size if i < 0 else i, 1, 1, False))
    return dims


def plan_index(shape, esize: int, index) -> SlicePlan:
    """The box that covers `tensor[index]` for a row-major tensor of `shape` with `esize`-byte elements.

    With d the last restricted dim, the dims after d are one contiguous block, and the box takes one run of dim d
    per selected index of the dims in front of it.  The box is exact when those indices are evenly spaced (only a
    leading range of the dims before d restricted, or one of them stepped) and dim d has step 1, or when nothing in
    front of d is selected more than once (then the elements of a stepped dim d are the rows).  Otherwise it is the
    smallest such box that covers the index, and the residual picks the result out of it."""
    shape = tuple(int(s) for s in shape)
    dims = _dims(shape, index)
    out_shape = tuple(c for _, c, _, kept in dims if kept)
    total = esize * math.prod(shape)
    if any(c == 0 for _, c, _, _ in dims):
        return SlicePlan((0, 0, 0, 0), out_shape, None)
    restricted = [d for d, (s, c, st, _) in enumerate(dims) if not (s == 0 and c == shape[d])]
    if not restricted:
        return SlicePlan((0, 1, total, total), out_shape, None)
    d = restricted[-1]
    inner = esize * math.prod(shape[d + 1:])
    row_bytes = shape[d] * inner
    s_d, c_d, st_d, _ = dims[d]
    sel = np.zeros(1, dtype=np.int64)           # selected indices of the dims in front of d, flattened (C order)
    for i in range(d):
        s, c, st, _ = dims[i]
        sel = (sel[:, None] * shape[i] + (s + st * np.arange(c, dtype=np.int64))[None, :]).reshape(-1)
    first = int(sel[0])
    if sel.size == 1 and st_d > 1:
        return SlicePlan((first * row_bytes + s_d * inner, c_d, st_d * inner, inner), out_shape, None)
    span = (c_d - 1) * st_d + 1
    gap = int(np.gcd.reduce(np.diff(sel))) if sel.size > 1 else 1
    rows = (int(sel[-1]) - first) // gap + 1
    box = (first * row_bytes + s_d * inner, rows, gap * row_bytes if rows > 1 else span * inner, span * inner)
    pick = None if rows == sel.size else (sel - first) // gap
    if pick is None and st_d == 1:
        return SlicePlan(box, out_shape, None)
    return SlicePlan(box, out_shape, Residual((rows, span) + shape[d + 1:], pick, st_d))


def apply_residual(x, plan: SlicePlan):
    """The decoded box (a flat numpy array or torch tensor of elements) -> tensor[index]."""
    if plan.residual is None:
        return x.reshape(plan.out_shape)
    view, pick, step = plan.residual
    y = x.reshape(view)
    if pick is not None:
        y = y[torch.from_numpy(pick).to(y.device)] if isinstance(y, torch.Tensor) else y[pick]
    if step > 1:
        y = y[:, ::step]
    y = y.reshape(plan.out_shape)
    return y.contiguous() if isinstance(y, torch.Tensor) else np.ascontiguousarray(y)


# ---------------------------------------------------------------------------------------------- sub-streams
class FileSource:
    """Bytes [offset, offset + nbytes) of an open file."""

    def __init__(self, fd: int, offset: int, nbytes: int):
        self.fd, self.offset, self.nbytes = fd, offset, nbytes

    def read(self, off: int, n: int) -> bytes:
        b = os.pread(self.fd, n, self.offset + off)
        if len(b) != n:
            raise RuntimeError("corrupt ZipNN stream: truncated")
        return b

    def read_into(self, off: int, mv: memoryview) -> None:
        got = 0
        while got < len(mv):
            k = os.preadv(self.fd, [mv[got:]], self.offset + off + got)
            if k <= 0:
                raise RuntimeError("corrupt ZipNN stream: truncated")
            got += k


class MemorySource:
    """A stream held in host memory (uint8 numpy array)."""

    def __init__(self, arr: np.ndarray):
        self.arr, self.nbytes = arr, arr.size

    def read(self, off: int, n: int) -> bytes:
        if off + n > self.nbytes:
            raise RuntimeError("corrupt ZipNN stream: truncated")
        return self.arr[off: off + n].tobytes()

    def read_into(self, off: int, mv: memoryview) -> None:
        if off + len(mv) > self.nbytes:
            raise RuntimeError("corrupt ZipNN stream: truncated")
        np.frombuffer(mv, dtype=np.uint8)[:] = self.arr[off: off + len(mv)]


class StreamIndex:
    """Header (and, with `tables`, the size tables) of one torch-format stream, read from `src` exactly: the
    32-byte header, the packed shape, then the 9 * G * K table bytes."""

    def __init__(self, src, tables: bool = True):
        from .zipnn import HEADER_LEN, HUF_MAX_BLOCK, ZipNN
        head = src.read(0, HEADER_LEN + 1)
        if head[0:2] != b"ZN":
            raise ValueError("Header should start with ZN")
        if head[8] != EnumFormat.TORCH.value or head[13] > 127 or head[9] != 0:
            raise ValueError("slices need a torch-format stream (not a streaming frame or a delta stream)")
        packed = bytearray(head[HEADER_LEN:])
        at = HEADER_LEN + 1
        for _ in range(head[HEADER_LEN]):
            k = src.read(at, 1)
            if k[0] not in (1, 2, 4, 8):
                raise ValueError("corrupt shape descriptor in ZipNN header")
            packed += k + src.read(at + 1, k[0])
            at += 1 + k[0]
        z = ZipNN(input_format="torch")
        self.after = z._retrieve_header(head[:HEADER_LEN] + bytes(packed))
        self.G = z._num_buf_of_dtype()
        self.chunk = z.compression_chunk if self.G != 1 else min(HUF_MAX_BLOCK, z.compression_chunk)
        self.n = z.original_len
        self.K = -(-self.n // self.chunk)
        self.bits_mode, self.bytes_mode = z._bit_reorder, z._byte_reorder
        self.dtype = torch_dtype_of_code(z.dtype)
        self.shape = tuple(z.shape_bytes)
        self.total_len = src.nbytes
        self.types = self.cum = self.group_off = None
        if tables and self.K:
            G, K = self.G, self.K
            tab = np.frombuffer(src.read(self.after, 9 * G * K), dtype=np.uint8)
            self.types = tab[: G * K].reshape(G, K)
            self.cum = tab[G * K:].view("<u8").reshape(G, K)
            totals = [int(t) for t in self.cum[:, -1]]
            payload0 = self.after + 9 * G * K
            if payload0 + sum(totals) > self.total_len:
                raise RuntimeError("corrupt ZipNN stream: size table past the end of the stream")
            self.group_off = [payload0 + sum(totals[:g]) for g in range(G)]

    def covering(self, box) -> tuple:
        """Chunk range [k0, k1) a non-empty box meets."""
        base, rows, pitch, ln = box
        return base // self.chunk, -(-(base + (rows - 1) * pitch + ln) // self.chunk)

    def _spans(self, k0: int, k1: int):
        lo = [int(x) for x in self.cum[:, k0 - 1]] if k0 else [0] * self.G
        hi = [int(x) for x in self.cum[:, k1 - 1]]
        tot = [int(x) for x in self.cum[:, -1]]
        if any(not (a <= b <= t) for a, b, t in zip(lo, hi, tot)):
            raise RuntimeError("corrupt ZipNN stream: size table")
        return lo, hi

    def substream_len(self, k0: int, k1: int) -> int:
        lo, hi = self._spans(k0, k1)
        return 9 * self.G * (k1 - k0) + sum(hi) - sum(lo)

    def substream_orig(self, k0: int, k1: int) -> int:
        return min(self.n, k1 * self.chunk) - k0 * self.chunk

    def read_substream(self, src, k0: int, k1: int, dst: np.ndarray) -> None:
        """Chunks [k0, k1) as a stream body of their own, into dst[:substream_len(k0, k1)]: their type bytes, their
        size rows rebased to the range, then per group only the payload bytes of the range, read from `src`."""
        G, Kl = self.G, k1 - k0
        lo, hi = self._spans(k0, k1)
        dst[: G * Kl] = self.types[:, k0:k1].reshape(-1)
        rows = self.cum[:, k0:k1].astype(np.uint64) - np.array(lo, dtype=np.uint64).reshape(G, 1)
        dst[G * Kl: 9 * G * Kl] = rows.astype("<u8").reshape(-1).view(np.uint8)
        w = 9 * G * Kl
        for g in range(G):
            ln = hi[g] - lo[g]
            if ln:
                src.read_into(self.group_off[g] + lo[g], memoryview(dst[w: w + ln]))
            w += ln


# ---------------------------------------------------------------------------------------------- decode
def decode_box(dbody: torch.Tensor, idx: StreamIndex, box, orig: int) -> torch.Tensor:
    """One `zipnn_b200_decompress_slices` call: the box of a stream body (or sub-stream of `orig` decoded bytes)
    on the GPU -> CUDA uint8 tensor of rows * len bytes."""
    base, rows, pitch, ln = box
    dev = dbody.device
    out = torch.empty(max(rows * ln, 1), dtype=torch.uint8, device=dev)[: rows * ln]
    if rows * ln == 0:
        return out
    it = (_native.SliceItem * 1)()
    it[0].d_body, it[0].body_len = dbody.data_ptr(), dbody.numel()
    it[0].num_buf, it[0].bits_mode, it[0].bytes_mode = idx.G, idx.bits_mode, idx.bytes_mode
    it[0].chunk, it[0].orig = idx.chunk, orig
    it[0].base, it[0].rows, it[0].pitch, it[0].len = base, rows, pitch, ln
    it[0].d_out = out.data_ptr()
    L = _native.lib()
    with torch.cuda.device(dev):
        wsz = C.c_size_t(0)
        _native.check(L.zipnn_b200_decompress_slices_workspace_size(it, 1, C.byref(wsz)))
        ws = torch.empty(wsz.value, dtype=torch.uint8, device=dev)
        rc = L.zipnn_b200_decompress_slices(it, 1, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream, 1)
    if rc == _native.E_CORRUPT:
        raise RuntimeError("Thread processing failed: corrupt ZipNN stream")
    _native.check(rc)
    return out


def _decode_host_box(src, idx: StreamIndex, plan: SlicePlan, dev) -> torch.Tensor:
    """Header, tables and covered payload from `src` into one pinned buffer, one H2D copy, one decode."""
    k0, k1 = idx.covering(plan.box)
    n = idx.substream_len(k0, k1)
    host = torch.empty(max(n, 1), dtype=torch.uint8, pin_memory=True)
    idx.read_substream(src, k0, k1, host.numpy())
    dbody = host[:n].to(dev, non_blocking=True)
    base, rows, pitch, ln = plan.box
    return decode_box(dbody, idx, (base - k0 * idx.chunk, rows, pitch, ln), idx.substream_orig(k0, k1))


def _result(u8: torch.Tensor, idx: StreamIndex, plan: SlicePlan) -> torch.Tensor:
    return apply_residual(u8.view(idx.dtype), plan)


def slice_stream(stream, index) -> torch.Tensor:
    """`ZipNN.decompress_slice`: `stream` is a CUDA uint8 tensor (decoded whole-stream with the box: the meta kernel
    skips the chunks outside it) or a host uint8 array (cut to the covering sub-stream first)."""
    from .zipnn import HEADER_LEN
    _native.require_cuda()
    if isinstance(stream, torch.Tensor):
        head = stream[: HEADER_LEN + 1 + 9 * 255].cpu().numpy()
        src = MemorySource(head)
        src.nbytes = stream.numel()
        idx = StreamIndex(src, tables=False)
        plan = plan_index(idx.shape, idx.dtype.itemsize, index)
        if stream.numel() < idx.after:
            raise RuntimeError("corrupt ZipNN stream: truncated header")
        return _result(decode_box(stream[idx.after:], idx, plan.box, idx.n), idx, plan)
    src = MemorySource(stream)
    idx = StreamIndex(src)
    plan = plan_index(idx.shape, idx.dtype.itemsize, index)
    if plan.box[1] * plan.box[3] == 0:
        return torch.empty(plan.out_shape, dtype=idx.dtype)
    dev = torch.device("cuda", torch.cuda.current_device())
    return _result(_decode_host_box(src, idx, plan, dev), idx, plan).cpu()


class CompressedSlice:
    """A compressed safetensors entry opened for slicing (the interface of safetensors' PySafeSlice:
    `get_shape()`, `get_dtype()`, `[index]`).  An index reads the stream's header, tables and only the payload
    of the chunks it covers from the file, copies them to the GPU at once and decodes them with one call; the
    tables are read once per entry."""

    def __init__(self, fd: int, offset: int, nbytes: int, device=None):
        """`device`: the CUDA device the result stays on, or None for a host result (decoded on the current GPU)."""
        self._src = FileSource(fd, offset, nbytes)
        self._device = device
        self._idx = None

    def _index(self) -> StreamIndex:
        if self._idx is None:
            self._idx = StreamIndex(self._src)
        return self._idx

    def get_shape(self) -> list:
        return list(self._index().shape)

    def get_dtype(self) -> str:
        return _ST_DTYPES[self._index().dtype]

    def __getitem__(self, index) -> torch.Tensor:
        idx = self._index()
        plan = plan_index(idx.shape, idx.dtype.itemsize, index)
        if plan.box[1] * plan.box[3] == 0:
            return torch.empty(plan.out_shape, dtype=idx.dtype, device=self._device or "cpu")
        _native.require_cuda()
        dev = self._device if self._device is not None else torch.device("cuda", torch.cuda.current_device())
        t = _result(_decode_host_box(self._src, idx, plan, dev), idx, plan)
        return t if self._device is not None else t.cpu()
