"""`ZipNN` -- host-side mirror of the reference codec object, routed to the CUDA kernels.

Same constructor, same `compress()` / `decompress()` contract and the same stream bytes as
reference `zipnn/zipnn.py:27-1218`; the native calls `zipnn_core.zipnn_core(...)`
(`zipnn/zipnn.py:714-725`) and `zipnn_core.combine_dtype(...)` (`:1143-1151`) are replaced by
the C ABI in `include/zipnn_b200.h`.

What is new relative to the reference:
  * a CUDA tensor in gives a CUDA tensor out (the compressed stream as `uint8`, or the
    decoded tensor), with no host round trip;
  * host inputs (CPU tensors, bytes, numpy) still work -- they are copied to the GPU, coded
    there and copied back (there is NO CPU codec in this package);
  * the input is never modified (the reference rotates sign bits in place, SURVEY Q1).

Not carried over (out of the hot path, SURVEY.md section 2): zstd/lz4/snappy methods, lossy
modes (dead code in the reference), the uint32/numpy truncation paths (they raise in the
reference as well), file-path arguments.
"""
from __future__ import annotations

import ctypes as C
import contextlib
import functools
import math
import multiprocessing
import os
import threading

import numpy as np
import torch

from . import _native
from .util_header import EnumFormat, EnumLossy, EnumMethod
from .util_torch import (
    BFLOAT16, FLOAT, FLOAT16, FLOAT32, FLOAT8_E4M3FN, FLOAT8_E5M2, HALF, UINT32,
    dtype_code, torch_dtype_of_code, zipnn_is_floating_point, zipnn_pack_shape, zipnn_unpack_shape,
)

HEADER_LEN = 32
HUF_MAX_BLOCK = 128 * 1024  # fp8 planes are whole chunks, and a Huffman block holds at most 128 KiB


def _as_u8_numpy(data) -> np.ndarray:
    """Zero-copy uint8 view of a bytes-like object / numpy array."""
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data).reshape(-1).view(np.uint8)
    return np.frombuffer(data, dtype=np.uint8)


def _torch_flat_u8(data: torch.Tensor) -> torch.Tensor:
    """Flat contiguous uint8 view of a tensor's bytes (a copy only when it is not contiguous)."""
    t = data.detach().contiguous().reshape(-1)
    if t.numel() == 0:   # (an empty tensor may carry a zero stride, which view() refuses)
        t = torch.empty(0, dtype=t.dtype, device=t.device)
    return t.view(torch.uint8) if t.dtype != torch.uint8 else t


def _xor_bytes(a, b):
    """Delta step (reference: np.bitwise_xor on host bytes, zipnn/zipnn.py:636-640, 997-1004).  If either side
    lives on a GPU the XOR runs there and a CUDA uint8 tensor comes back; otherwise a numpy array."""
    ta, tb = isinstance(a, torch.Tensor) and a.is_cuda, isinstance(b, torch.Tensor) and b.is_cuda
    if ta or tb:
        dev = a.device if ta else b.device

        def dev_u8(x):
            if isinstance(x, torch.Tensor):
                x = x.detach().contiguous().reshape(-1)
                return (x if x.dtype == torch.uint8 else x.view(torch.uint8)).to(dev, non_blocking=True)
            return torch.from_numpy(np.array(_as_u8_numpy(x), copy=True)).to(dev, non_blocking=True)
        ua, ub = dev_u8(a), dev_u8(b)
        if ua.numel() != ub.numel():
            raise ValueError("Length of delta file has to match the length of the original file.")
        return torch.bitwise_xor(ua, ub)
    return np.bitwise_xor(_as_u8_numpy(a), _as_u8_numpy(b))


@functools.lru_cache(maxsize=None)
def _default_threads() -> int:
    """min(cores, 16), the reference's default thread count, asked once: os.cpu_count() reads sysfs, which costs a
    fraction of a millisecond on a large host, and a ZipNN object is often made per tensor."""
    return min(multiprocessing.cpu_count(), 16)


def _layout_for_dtype(code: int):
    """(bit_reorder, byte_reorder, num_buf) per dtype: reference zipnn/zipnn.py:788-815."""
    if code in (FLOAT8_E4M3FN, FLOAT8_E5M2):
        return 1, 10, 1          # bit_reorder is recorded but ignored by the fp8 path
    if code in (FLOAT32, FLOAT):
        return 1, 220, 4
    if code == BFLOAT16:
        return 1, 10, 2
    if code in (FLOAT16, HALF):
        return 0, 10, 2
    raise ValueError("Support only torch.dtype float32/bfloat16/float16")


class ZipNN:
    def __init__(
        self,
        method: str = "AUTO",
        input_format: str = "byte",
        bytearray_dtype: str = "bfloat16",
        is_monotonic: int = 0,
        threads: int = 0,
        compression_threshold=0.95,
        check_th_after_percent=10,
        byte_reorder: int = 0,
        reorder_signbit: int = 0,
        delta_compressed_type: str = 0,
        lossy_compressed_type: str = 0,
        lossy_compressed_factor=27,
        compression_chunk=256 * 1024,
        is_streaming: bool = False,
        streaming_chunk: int = 1024 * 1024,
        input_file: str = None,
        compressed_file: str = None,
        decompressed_file: str = None,
        zstd_level: int = 3,
        lz4_compression_level: int = 0,
    ):
        """Same keyword arguments as the reference (zipnn/zipnn.py:29-51).

        `threads`, `check_th_after_percent`, `is_monotonic`, `zstd_level`,
        `lz4_compression_level` are accepted for compatibility and have no effect on the GPU
        path (`check_th_after_percent` has none in the reference either,
        csrc/zipnn_core.c:555-558).
        """
        self.method = EnumMethod(method).value
        self.input_format = EnumFormat(input_format).value
        self.bytearray_dtype = bytearray_dtype
        self.is_monotonic = is_monotonic
        self.threads = threads or _default_threads()
        self.compression_threshold = compression_threshold
        self.check_th_after_percent = check_th_after_percent
        self.byte_reorder = byte_reorder
        self.reorder_signbit = reorder_signbit
        self.delta_compressed_type = delta_compressed_type
        self.lossy_compressed_type = EnumLossy.NONE if lossy_compressed_type is None else EnumLossy(lossy_compressed_type)
        self.lossy_compressed_factor = lossy_compressed_factor

        if compression_chunk > 0 and (compression_chunk & (compression_chunk - 1)) == 0:
            self.compression_chunk = compression_chunk
        else:
            raise ValueError("compression_chunk must be a number that is a power of 2.")
        if self.input_format != EnumFormat.BYTE.value and is_streaming:
            raise ValueError("Streaming is currently implemented only for bytes data type.")
        self.is_streaming = is_streaming
        if streaming_chunk > 0 and (streaming_chunk & (streaming_chunk - 1)) == 0:
            self.streaming_chunk = streaming_chunk
        else:
            raise ValueError("streaming_chunk must be a number that is a power of 2.")

        self.input_file = input_file
        self.compressed_file = compressed_file
        self.decompressed_file = decompressed_file
        self.lz4_compression_level = lz4_compression_level

        self._version_major, self._version_minor, self._version_tiny = 0, 5, 3
        if self.method not in (EnumMethod.AUTO.value, EnumMethod.HUFFMAN.value):
            # reference: these need the optional zstandard / lz4 / snappy wheels and are only
            # reachable for one-group byte_reorder modes that no float dtype selects
            raise ImportError(f"method {EnumMethod(self.method).name} is not part of the GPU path; use AUTO or HUFFMAN")
        if self.lossy_compressed_type != EnumLossy.NONE and self.input_format != EnumFormat.TORCH.value:
            raise ValueError("When use lossy compression the input have to be torch.tensor")

        self.header_length = HEADER_LEN
        self._header = bytearray(self.header_length)
        self._ext_header = b""
        self._shape_size = 0
        self._update_header()

    # ------------------------------------------------------------------ header
    # [0:2]="ZN" [2:5]=version [5]=byte_reorder [6]=bit_reorder [7]=method [8]=format [9]=delta
    # [10:13]=lossy [13]=streaming [14]=log2(chunk) [15]=dtype [16:24]=orig len [24:32]=stream len
    # (zipnn/zipnn.py:287-303, 355-394)
    def _update_header(self):
        h = self._header
        h[0:2] = b"ZN"
        h[2], h[3], h[4] = self._version_major, self._version_minor, self._version_tiny
        h[7] = self.method
        h[8] = self.input_format
        h[9] = 1 if self.delta_compressed_type == "byte" else 2 if self.delta_compressed_type == "file" else 0
        h[13] = 128 + int(math.log(self.streaming_chunk, 2)) if self.is_streaming else 0
        h[14] = int(math.log(self.compression_chunk, 2))

    def _retrieve_header(self, head: bytes) -> int:
        """Parse the 32-byte header (+ packed shape); returns where the body starts
        (zipnn/zipnn.py:396-438)."""
        header = head[: self.header_length]
        if len(header) < self.header_length or header[0:2] != b"ZN":
            raise ValueError("Header should start with ZN")
        self.version_major, self.version_minor, self.version_tiny = header[2], header[3], header[4]
        self._byte_reorder = header[5]
        self._bit_reorder = header[6]
        self.method = header[7]
        self.input_format = header[8]
        self.lossy_compressed_type = header[10]
        self.lossy_compressed_factor = header[11]
        self._lossy_is_int = header[12]
        self.is_streaming = 1 if header[13] > 127 else 0
        self.compression_chunk = 2 ** header[14]
        self.dtype = header[15]
        self.original_len = int.from_bytes(header[16:24], "little")
        self._shape_size = 0
        if self.input_format in (EnumFormat.TORCH.value, EnumFormat.NUMPY.value):
            self.shape_bytes, self._shape_size = zipnn_unpack_shape(head[self.header_length:])
        return self.header_length + self._shape_size

    # ------------------------------------------------------------------ compress
    def compress(self, data, compress_cpu_gpu="cpu", delta_second_data=None, lossy_compressed_type: str = None,
                 lossy_compressed_factor: int = None, out=None):
        """zipnn/zipnn.py:560-643.  Returns a `memoryview` for host inputs (as the reference
        does) or a CUDA `uint8` tensor for CUDA inputs (or when compress_cpu_gpu == "gpu").
        `out=` (extension): a CPU uint8 tensor, ideally pinned, to receive a host result --
        lets a caller that codes many tensors reuse one staging buffer."""
        self._want_device_result = (compress_cpu_gpu == "gpu")
        self._out = out
        if self.delta_compressed_type == "byte":
            if len(data) != len(delta_second_data):
                raise ValueError("Length of delta file has to match the length of the original file.")
        elif self.delta_compressed_type == "file":
            try:
                with open(delta_second_data, "rb") as file:
                    delta_second_data = file.read()
            except Exception:
                raise FileNotFoundError("Encountered an error when reading the delta file")
            if len(data) != len(delta_second_data):
                raise ValueError("Length of delta file has to match the length of the original file.")
        elif delta_second_data is not None:
            raise ValueError("ZipNN isn't set for delta compression, but delta_second_data is not null.")

        if self.is_streaming and self.input_format == EnumFormat.BYTE.value:
            # independent frames of `streaming_chunk` input bytes (zipnn/zipnn.py:612-635)
            src = _as_u8_numpy(data)
            dlt = _as_u8_numpy(delta_second_data) if delta_second_data is not None else None
            if dlt is not None:
                src = np.bitwise_xor(src, dlt)
            fast = self._compress_frames_at_once(src)
            if fast is not None:
                return fast
            out = bytearray()
            for off in range(0, src.size, self.streaming_chunk):
                out.extend(self.compress_torch_numpy_byte(src[off: off + self.streaming_chunk]))
            return out
        if delta_second_data is not None:
            data = _xor_bytes(data, delta_second_data)
        return self.compress_torch_numpy_byte(data)

    def _compress_frames_at_once(self, src: np.ndarray):
        """All streaming frames from ONE pass of the codec.  A frame is the stream of `streaming_chunk` input
        bytes compressed alone (zipnn/zipnn.py:612-635); when a frame is a whole number of chunks, that is
        the frame's rows of the type / size tables (sizes rebased to the frame) and its slices of the
        per-group payload of the stream of the WHOLE input, because chunks are coded independently.  One H2D
        copy and one set of kernel launches instead of one per MiB.  -> bytearray, or None (caller loops)."""
        code = dtype_code(self.bytearray_dtype)
        _, _, num_buf = _layout_for_dtype(code)
        chunk = self.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, self.compression_chunk)
        n = src.size
        if n == 0 or self.streaming_chunk % chunk or self.streaming_chunk < chunk:
            return None
        whole = np.frombuffer(self.compress_torch_numpy_byte(src), dtype=np.uint8)
        H, G = HEADER_LEN, num_buf
        K = (n + chunk - 1) // chunk
        types = whole[H: H + G * K].reshape(G, K)
        cum = np.frombuffer(whole[H + G * K: H + 9 * G * K].tobytes(), dtype="<u8").reshape(G, K).astype(np.int64)
        payload0 = H + 9 * G * K
        base = payload0 + np.concatenate([[0], np.cumsum(cum[:, -1])[:-1]])
        per = self.streaming_chunk // chunk
        out = bytearray()
        hdr = bytearray(whole[:H].tobytes())
        for c0 in range(0, K, per):
            c1 = min(K, c0 + per)
            lo = cum[:, c0 - 1] if c0 else np.zeros(G, dtype=np.int64)
            hi = cum[:, c1 - 1]
            flen = H + 9 * G * (c1 - c0) + int((hi - lo).sum())
            hdr[16:24] = int(min(n, c1 * chunk) - c0 * chunk).to_bytes(8, "little")
            hdr[24:32] = int(flen).to_bytes(8, "little")
            out.extend(hdr)
            out.extend(np.ascontiguousarray(types[:, c0:c1]).tobytes())
            out.extend((cum[:, c0:c1] - lo.reshape(G, 1)).astype("<u8").tobytes())
            for g in range(G):
                out.extend(whole[int(base[g] + lo[g]): int(base[g] + hi[g])].tobytes())
        return out

    def compress_torch_numpy_byte(self, data, lossy_compressed_type=None, lossy_compressed_factor=None):
        """dtype dispatch + byte view of the input: zipnn/zipnn.py:748-867."""
        fmt = self.input_format
        if fmt == EnumFormat.BYTE.value:
            code = dtype_code(self.bytearray_dtype)
            shape = None
        else:
            code = dtype_code(data.dtype)
            shape = tuple(data.shape)
        if not zipnn_is_floating_point(fmt, data, self.bytearray_dtype):
            if code == UINT32 and fmt == EnumFormat.NUMPY.value:
                raise ValueError("Not support uint32 with NumPy format")
            raise ValueError("Support only uint32 with NumPy format")
        bit_reorder, byte_reorder, num_buf = _layout_for_dtype(code)
        self._header[5], self._header[6], self._header[15] = byte_reorder, bit_reorder, code

        if fmt == EnumFormat.TORCH.value:
            # a contiguous CUDA tensor goes as it is: the device call needs its address and byte size only
            flat = data if data.is_cuda and data.is_contiguous() else _torch_flat_u8(data)
        elif fmt == EnumFormat.NUMPY.value:
            flat = torch.from_numpy(np.ascontiguousarray(data).reshape(-1).view(np.uint8))
        elif isinstance(data, torch.Tensor):   # byte format, bytes held in a (possibly CUDA) uint8 tensor
            flat = data.detach().contiguous().reshape(-1).view(torch.uint8)
        else:
            flat = _as_u8_numpy(data)     # host bytes: stays a numpy view (may be read-only)
        return self.compress_bin(flat, bit_reorder, byte_reorder, num_buf, shape)

    def _plan_header(self, n: int, num_buf: int, shape):
        """-> (python_header bytes, chunk) for an input of n bytes (zipnn/zipnn.py:709-721)."""
        self._header[16:24] = int(n).to_bytes(8, "little")
        self._ext_header = zipnn_pack_shape(shape) if self.input_format in (EnumFormat.TORCH.value, EnumFormat.NUMPY.value) else b""
        chunk = self.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, self.compression_chunk)
        return bytes(self._header) + self._ext_header, chunk

    def compress_bin(self, flat_u8, bit_reorder: int, byte_reorder: int, num_buf: int, shape):
        """Header assembly + the native call (zipnn/zipnn.py:670-746).  `flat_u8` holds the input's bytes: a flat
        uint8 torch tensor (CPU or CUDA), a contiguous CUDA tensor of any dtype, or a numpy array (host bytes)."""
        n = flat_u8.nbytes if isinstance(flat_u8, torch.Tensor) else flat_u8.size
        python_header, chunk = self._plan_header(n, num_buf, shape)
        self._last_plan = dict(header=python_header, num_buf=num_buf, bit_reorder=bit_reorder,
                               byte_reorder=byte_reorder, chunk=chunk, threshold=self.compression_threshold)
        if getattr(self, "_plan_only", False):
            return None
        if isinstance(flat_u8, torch.Tensor) and flat_u8.is_cuda:
            return _compress_device(flat_u8, python_header, num_buf, bit_reorder, byte_reorder, chunk, self.compression_threshold)
        out = _compress_host(flat_u8, python_header, num_buf, bit_reorder, byte_reorder, chunk, self.compression_threshold,
                             out=getattr(self, "_out", None))
        if getattr(self, "_want_device_result", False):
            return torch.from_numpy(np.asarray(out)).cuda()
        return out

    def compress_batch(self, tensors) -> list:
        """Many CUDA tensors (one device) in one `zipnn_b200_compress_batch` call: one launch per encode
        kernel and byte-group class, one host synchronisation.  Element i equals `self.compress(tensors[i])`;
        the streams are views into one output buffer.  Torch input format only, without streaming or delta."""
        if self.input_format != EnumFormat.TORCH.value or self.is_streaming or self.delta_compressed_type:
            raise ValueError("compress_batch takes torch tensors, without streaming or delta compression")
        tensors = list(tensors)
        if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in tensors):
            raise ValueError("compress_batch takes CUDA tensors")
        if len({t.device for t in tensors}) > 1:
            raise ValueError("compress_batch takes tensors on one device")
        if not tensors:
            return []
        plans = [self.plan(t) for t in tensors]
        return _compress_device_batch([_torch_flat_u8(t) for t in tensors], plans)

    def plan(self, data) -> dict:
        """Everything `compress(data)` would hand to the native call, without calling it:
        {header, num_buf, bit_reorder, byte_reorder, chunk, threshold}.  Needs no GPU."""
        self._plan_only = True
        try:
            self.compress_torch_numpy_byte(data)
        finally:
            self._plan_only = False
        return self._last_plan

    # ------------------------------------------------------------------ decompress
    def decompress(self, data, decompress_cpu_gpu="cpu", delta_second_data=None, out=None):
        """zipnn/zipnn.py:928-1005.  CUDA `uint8` tensor in -> CUDA result; host bytes in -> host result.
        `out=` (extension): CPU tensor (ideally pinned) that receives a host result."""
        self._out = out
        if self.delta_compressed_type == "byte":
            if delta_second_data is None:
                raise ValueError("delta_second_data is None or not set for delta copression")
        elif self.delta_compressed_type == "file":
            try:
                with open(delta_second_data, "rb") as file:
                    delta_second_data = file.read()
            except Exception:
                raise FileNotFoundError("Encountered an error when reading the delta file")
        elif delta_second_data is not None:
            raise ValueError("ZipNN isn't set for delta compression, but delta_second_data is not null.")

        stream = _as_stream(data)
        # one look at the stream start serves this check and decompress_bin's header parse (for a CUDA
        # stream every look is a synchronising device-to-host copy)
        head = _peek(stream, HEADER_LEN + 1 + 9 * 255)
        if len(head) < HEADER_LEN:
            raise ValueError("Header should start with ZN")
        was_delta = head[9]
        if was_delta == 0 and self.delta_compressed_type != 0:
            raise ValueError("The data wasn't compressed using delta compression and you're trying to delta-decompress it.")
        if was_delta != 0 and self.delta_compressed_type == 0:
            raise ValueError("The data was compressed using delta compression and you're trying to decompress it normally.")

        if self.input_format == EnumFormat.BYTE.value and head[13] > 127:
            # concatenated frames, each [32-byte header][body]; frame length at header[24:32]
            if isinstance(stream, torch.Tensor):
                stream = stream.cpu().numpy()
            dlt = _as_u8_numpy(delta_second_data) if delta_second_data is not None else None
            fast = self._decompress_frames_at_once(stream)
            if fast is not None:
                if dlt is not None:
                    if fast.size != dlt.size:
                        raise ValueError("Length of delta file has to match the length of the decompressed file.")
                    fast = np.bitwise_xor(fast, dlt)
                return bytearray(fast.tobytes())
            out = bytearray()
            off, doff = 0, 0
            while off < stream.size:
                flen = int.from_bytes(stream[off + 24: off + 32].tobytes(), "little")
                if flen < HEADER_LEN or off + flen > stream.size:
                    raise RuntimeError("corrupt ZipNN streaming frame")
                piece = np.frombuffer(self.decompress_bin(stream[off: off + flen]), dtype=np.uint8)
                if dlt is not None:
                    if doff + piece.size > dlt.size:
                        raise ValueError("Length of delta file has to match the length of the decompressed file.")
                    piece = np.bitwise_xor(piece, dlt[doff: doff + piece.size])
                    doff += piece.size
                out.extend(piece.tobytes())
                off += flen
            if dlt is not None and doff != dlt.size:
                raise ValueError("Length of delta file has to match the length of the decompressed file.")
            return out

        result = self.decompress_bin(stream, head=head)
        if delta_second_data is not None:
            on_gpu = (isinstance(result, torch.Tensor) and result.is_cuda) or (isinstance(delta_second_data, torch.Tensor) and delta_second_data.is_cuda)
            nres = result.numel() * result.element_size() if isinstance(result, torch.Tensor) else len(_as_u8_numpy(result))
            ndlt = delta_second_data.numel() * delta_second_data.element_size() if isinstance(delta_second_data, torch.Tensor) else len(_as_u8_numpy(delta_second_data))
            if nres != ndlt:
                raise ValueError("Length of delta file has to match the length of the decompressed file.")
            x = _xor_bytes(result, delta_second_data)
            return x if on_gpu else x.tobytes()
        return result

    def decompress_slice(self, data, index):
        """`decompress(data)[index]` while decoding only the chunks the index touches (zipnn_b200/slicing.py).
        `data` is a torch-format stream; `index` takes ints, slices with positive steps and one Ellipsis, as
        safetensors' slices do.  A CUDA stream is decoded in place with a window; a host stream is first cut to
        the chunks the index covers, which are copied to the GPU at once.  The result lies where `decompress`
        would put it: on the stream's GPU, or on the host for a host stream.  Streaming frames and delta streams
        raise ValueError."""
        from .slicing import slice_stream
        if self.delta_compressed_type != 0:
            raise ValueError("decompress_slice does not take delta streams")
        return slice_stream(_as_stream(data), index)

    def _decompress_frames_at_once(self, stream: np.ndarray):
        """Every frame of a streaming file in one batched decode (zipnn_b200_decompress_batch): one H2D copy of
        the file, one launch per kernel, one D2H copy -- instead of a copy, five launches and two
        synchronisations per 1 MiB frame.  -> uint8 array, or None when a frame does not fit the fast path."""
        H = HEADER_LEN
        frames = []
        off = doff = 0
        total = stream.size
        while off < total:
            if off + H > total:
                raise RuntimeError("corrupt ZipNN streaming frame")
            hd = stream[off: off + H].tobytes()
            flen = int.from_bytes(hd[24:32], "little")
            if hd[0:2] != b"ZN" or flen < H or off + flen > total:
                raise RuntimeError("corrupt ZipNN streaming frame")
            z = ZipNN(input_format="byte", bytearray_dtype=self.bytearray_dtype)
            z._retrieve_header(hd)
            num_buf = z._num_buf_of_dtype()
            chunk = z.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, z.compression_chunk)
            if doff % 16:
                return None        # (a frame whose output would not start on a 16-byte boundary: per-frame loop)
            frames.append((off + H, flen - H, num_buf, z._bit_reorder, z._byte_reorder, chunk, z.original_len, doff))
            off += flen
            doff += z.original_len
        if not frames:
            return np.empty(0, dtype=np.uint8)
        _native.require_cuda()
        L = _native.lib()
        dev = torch.device("cuda", torch.cuda.current_device())
        src_t = _host_tensor(np.ascontiguousarray(stream))
        dbuf = torch.empty(64 + total + 16, dtype=torch.uint8, device=dev)
        dbuf[64: 64 + total].copy_(src_t, non_blocking=True)
        out = torch.empty(max(doff, 1), dtype=torch.uint8, device=dev)
        arr = (_native.BatchItem * len(frames))()
        for i, (boff, blen, num_buf, bits, bytes_mode, chunk, n, o) in enumerate(frames):
            arr[i].d_body = dbuf.data_ptr() + 64 + boff
            arr[i].body_len = blen
            arr[i].num_buf, arr[i].bits_mode, arr[i].bytes_mode = num_buf, bits, bytes_mode
            arr[i].chunk, arr[i].orig = chunk, n
            arr[i].d_out = out.data_ptr() + o if n else None
        wsz = C.c_size_t(0)
        _native.check(L.zipnn_b200_decompress_batch_workspace_size(arr, len(frames), C.byref(wsz)))
        ws = torch.empty(wsz.value, dtype=torch.uint8, device=dev)
        rc = L.zipnn_b200_decompress_batch(arr, len(frames), ws.data_ptr(), ws.numel(), _cuda_stream_handle(), 1)
        if rc == _native.E_CORRUPT:
            raise RuntimeError("Thread processing failed: corrupt ZipNN stream")
        _native.check(rc)
        host = _host_out(doff, None)
        host.copy_(out[:doff], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return host.numpy()

    def _num_buf_of_dtype(self) -> int:
        code = self.dtype
        if code in (FLOAT8_E4M3FN, FLOAT8_E5M2):
            return 1
        if code in (FLOAT32, FLOAT):
            return 4
        if code in (BFLOAT16, FLOAT16, HALF):
            return 2
        if code == UINT32:
            raise ValueError("Unsupported uinit32 in this version yet! please try version 0.1.1")
        raise ValueError(f"Unsupported Dtype {self.dtype}")

    def decompress_bin(self, stream, head=None):
        """Header parse, native call, tensor re-wrap (zipnn/zipnn.py:1072-1198)."""
        stream = _as_stream(stream)
        if head is None:
            head = _peek(stream, HEADER_LEN + 1 + 9 * 255)
        after_header = self._retrieve_header(head)
        code = self.dtype
        num_buf = self._num_buf_of_dtype()
        chunk = self.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, self.compression_chunk)
        n = self.original_len
        total = stream.numel() if isinstance(stream, torch.Tensor) else stream.size
        if total < after_header:
            raise RuntimeError("corrupt ZipNN stream: truncated header")
        if isinstance(stream, torch.Tensor):
            tdt = torch_dtype_of_code(code) if self.input_format == EnumFormat.TORCH.value else None
            if tdt is not None and math.prod(self.shape_bytes) * tdt.itemsize == n:
                # the tensor itself is the destination: no views to make of the decoded bytes
                out = torch.empty(self.shape_bytes, dtype=tdt, device=stream.device)
                return _decompress_device(stream, num_buf, self._bit_reorder, self._byte_reorder, chunk, n, after_header, out)
            out_u8 = _decompress_device(stream, num_buf, self._bit_reorder, self._byte_reorder, chunk, n, after_header)
        else:
            out_u8 = _decompress_host(stream[after_header:], num_buf, self._bit_reorder, self._byte_reorder, chunk, n,
                                      out=getattr(self, "_out", None))

        fmt = self.input_format
        if fmt == EnumFormat.BYTE.value:
            if isinstance(out_u8, torch.Tensor) and out_u8.is_cuda:
                return out_u8
            return memoryview(out_u8.numpy()) if isinstance(out_u8, torch.Tensor) else memoryview(out_u8)
        tdt = torch_dtype_of_code(code)
        t = out_u8 if isinstance(out_u8, torch.Tensor) else torch.from_numpy(out_u8)
        if fmt == EnumFormat.TORCH.value:
            return t.view(tdt).reshape(self.shape_bytes)
        if fmt == EnumFormat.NUMPY.value:
            arr = t.cpu().numpy()
            if code in (FLOAT32, FLOAT):
                return arr.view(np.float32).reshape(self.shape_bytes)
            if code in (FLOAT16, HALF):
                return arr.view(np.float16).reshape(self.shape_bytes)
            raise ValueError(f"Unsupported Dtype {self.dtype}")
        raise ValueError(f"Unsupported input_format {self.input_format}")



class DecodePipe:
    """Decode many host- or file-resident streams onto one GPU without a host synchronisation per
    tensor (the load path: `SafeOpen(..., device="cuda")`, SURVEY.md section 8f N1).

    One bitstream of a chunk is decoded serially, so a decode takes the same time however small the tensor
    is, and a checkpoint has hundreds of tensors.  `submit*` therefore (1) parses the header on the
    host, (2) moves the body through a ring of pinned 64 MiB slabs -- filled by a few threads with
    `preadv` straight from the file (a memory-mapped source costs a page fault per 4 KiB) --
    (3) enqueues the H2D copies and the decode on one of a few side streams, each of which owns its
    body and workspace buffers, with the error word left on the device, and (4) makes the caller's
    current stream wait for that decode: the tensor that comes back is safe to use on the current
    stream, and the next submit runs beside this one.  `finish` synchronises once, raises what a
    per-tensor check would have raised, and re-decodes in place the rare tensor that needed the
    large workspace."""

    SLAB_BYTES = 64 << 20      # pinned staging slab; a stream larger than this goes through several
    COPY_PIECE = 8 << 20       # granule handed to one worker thread
    _shared_pool = None
    _shared_streams = {}
    _slab_cache = []           # pinned slabs of finished pipes, reused by the next one
    # the three above: pipes are built and released on a loader's threads at once.  Re-entrant: a pipe left in a
    # reference cycle (its pending redo closures hold it) is released by __del__ on whatever thread the cyclic
    # collector runs, which may be a thread inside this lock already
    _shared_lock = threading.RLock()

    def __init__(self, device, streams: int = 4, stage_buffers: int = 4, copy_threads: int = 0):
        _native.require_cuda()
        self.device = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        # side streams are process-wide per device: the caching allocator keeps one pool per stream, so a
        # second file loaded through fresh streams would pay cudaMalloc for every tensor again
        key = (self.device.index, streams)
        with DecodePipe._shared_lock:
            if key not in DecodePipe._shared_streams:
                DecodePipe._shared_streams[key] = [torch.cuda.Stream(self.device) for _ in range(streams)]
            self._streams = DecodePipe._shared_streams[key]
        self._body = [None] * streams      # per side stream, reused in stream order
        self._ws = [None] * streams
        self._stage = [None] * stage_buffers
        self._stage_evt = [None] * stage_buffers
        self._slab = 0
        self._n = 0
        self._flags = None                 # int32[cap] on the device, one word per submitted tensor
        self._nflags = 0
        self._pending = []                 # (flag index, redo closure)
        # pinned slabs and reader threads are process-wide: page-locking 256 MiB costs tens to hundreds
        # of milliseconds, more than a small checkpoint takes to load
        nthreads = copy_threads or max(1, min(16, (multiprocessing.cpu_count() or 2) // 2))
        with DecodePipe._shared_lock:
            if nthreads > 1 and DecodePipe._shared_pool is None:
                from concurrent.futures import ThreadPoolExecutor
                DecodePipe._shared_pool = ThreadPoolExecutor(max_workers=nthreads)
            self._pool = DecodePipe._shared_pool if nthreads > 1 else None
        for j, sl in enumerate(DecodePipe._take_slabs(self.SLAB_BYTES, stage_buffers)):
            self._stage[j] = sl

    @staticmethod
    def _take_slabs(nbytes: int, most: int) -> list:
        """Up to `most` cached slabs of `nbytes` bytes, each handed to this caller alone.  Slabs of another size
        are dropped: SLAB_BYTES may have changed since they were cached."""
        with DecodePipe._shared_lock:
            cache = DecodePipe._slab_cache
            cache[:] = [sl for sl in cache if sl.numel() == nbytes]
            return [cache.pop() for _ in range(min(most, len(cache)))]

    @staticmethod
    def _give_slab(sl: torch.Tensor) -> None:
        """Keep a slab no pipe uses any more for the next one (at most 8 are kept)."""
        with DecodePipe._shared_lock:
            if len(DecodePipe._slab_cache) < 8:
                DecodePipe._slab_cache.append(sl)

    # ---- host side: fill a pinned slab
    def _fill_from_host(self, dst: torch.Tensor, src: torch.Tensor):
        n = src.numel()
        if self._pool is None or n <= self.COPY_PIECE:
            dst.copy_(src)
            return
        futs = [self._pool.submit(dst[a: min(n, a + self.COPY_PIECE)].copy_, src[a: min(n, a + self.COPY_PIECE)])
                for a in range(0, n, self.COPY_PIECE)]
        for f in futs:
            f.result()

    @staticmethod
    def _pread_into(fd: int, mv, off: int):
        got = 0
        n = len(mv)
        while got < n:
            r = os.preadv(fd, [mv[got:]], off + got)
            if r <= 0:
                raise RuntimeError("corrupt ZipNN stream: file is shorter than its index says")
            got += r

    def _fill_from_file(self, dst: torch.Tensor, fd: int, off: int):
        n = dst.numel()
        mv = memoryview(dst.numpy())
        if self._pool is None or n <= self.COPY_PIECE:
            self._pread_into(fd, mv, off)
            return
        futs = [self._pool.submit(self._pread_into, fd, mv[a: min(n, a + self.COPY_PIECE)], off + a)
                for a in range(0, n, self.COPY_PIECE)]
        for f in futs:
            f.result()

    def _upload(self, dbody: torch.Tensor, blen: int, fill, st):
        """body -> device through the pinned slab ring, enqueued on `st` (which the caller made current).
        fill(dst_pinned, a, b) puts body bytes [a, b) into dst_pinned."""
        for a in range(0, blen, self.SLAB_BYTES):
            b = min(blen, a + self.SLAB_BYTES)
            j = self._slab % len(self._stage)
            self._slab += 1
            if self._stage_evt[j] is not None:
                self._stage_evt[j].synchronize()       # the H2D copy out of this slab is done
            if self._stage[j] is None:
                self._stage[j] = _pinned_empty(self.SLAB_BYTES)
            fill(self._stage[j][: b - a], a, b)
            dbody[a:b].copy_(self._stage[j][: b - a], non_blocking=True)
            evt = torch.cuda.Event()
            evt.record(st)
            self._stage_evt[j] = evt

    def _grown(self, bufs, k: int, nbytes: int) -> torch.Tensor:
        if bufs[k] is None or bufs[k].numel() < nbytes:
            bufs[k] = None
            bufs[k] = torch.empty(max(nbytes + (nbytes >> 2), 1 << 20), dtype=torch.uint8, device=self.device)
        return bufs[k]

    # ---- the common part
    def _decode(self, znn: "ZipNN", head: bytes, total_len: int, fill, refetch) -> torch.Tensor:
        """head = the first bytes of the stream; fill(dst, a, b) delivers body bytes; refetch() -> the
        whole body as a host array (only for the rare redo)."""
        after = znn._retrieve_header(head)
        num_buf = znn._num_buf_of_dtype()
        chunk = znn.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, znn.compression_chunk)
        n = znn.original_len
        if total_len < after:
            raise RuntimeError("corrupt ZipNN stream: truncated header")
        if znn.input_format != EnumFormat.TORCH.value or znn.is_streaming:
            return None
        tdt = torch_dtype_of_code(znn.dtype)
        shape = znn.shape_bytes
        blen = total_len - after
        L = _native.lib()
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            if n == 0:
                return torch.empty(0, dtype=torch.uint8, device=self.device).view(tdt).reshape(shape)
            k = self._n % len(self._streams)
            st = self._streams[k]
            self._n += 1
            if self._flags is None or self._nflags == self._flags.numel():
                self._flags = torch.zeros(1024, dtype=torch.int32, device=self.device)
                self._nflags = 0
                for side in self._streams:      # the zero fill runs on the current stream
                    side.wait_stream(cur)
            fi = self._nflags
            self._nflags += 1
            flags = self._flags
            with torch.cuda.stream(st):
                dbody = self._grown(self._body, k, 64 + blen + 16)[64: 64 + blen]
                self._upload(dbody, blen, lambda dst, a, b: fill(dst, after + a, after + b), st)
                out = torch.empty(n, dtype=torch.uint8, device=self.device)
                ws = self._grown(self._ws, k, _native.decompress_workspace_size(n, num_buf, chunk))
                rc = L.zipnn_b200_decompress(dbody.data_ptr(), blen, num_buf, znn._bit_reorder, znn._byte_reorder, chunk, n,
                                             out.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream, 0)
                if rc == _native.E_CORRUPT:
                    raise RuntimeError("Thread processing failed: corrupt ZipNN stream")
                _native.check(rc)
                flags[fi: fi + 1].copy_(ws[:4].view(torch.int32), non_blocking=True)
                done = torch.cuda.Event()
                done.record(st)
            cur.wait_event(done)
            out.record_stream(cur)
            bits, bytes_mode = znn._bit_reorder, znn._byte_reorder

            def redo(out=out):
                body = torch.from_numpy(np.ascontiguousarray(refetch()[after:])).to(self.device)
                out.copy_(_decompress_device(body, num_buf, bits, bytes_mode, chunk, n))

            self._pending.append((flags, fi, redo))
        return out.view(tdt).reshape(shape)

    def submit(self, host_stream, znn: "ZipNN" = None) -> torch.Tensor:
        """A stream held in host memory (bytes, numpy, CPU tensor) -> CUDA tensor."""
        znn = znn if znn is not None else ZipNN(input_format="torch")
        src = _as_stream(host_stream)
        if isinstance(src, torch.Tensor):          # already on a GPU: plain stream-ordered decode
            return znn.decompress(src)
        src_t = _host_tensor(src)
        r = self._decode(znn, src[: HEADER_LEN + 1 + 9 * 255].tobytes(), src.size,
                         lambda dst, a, b: self._fill_from_host(dst, src_t[a:b]), lambda: src)
        if r is None:
            return znn.decompress(torch.from_numpy(np.ascontiguousarray(src)).to(self.device))
        return r

    def submit_file(self, fd: int, offset: int, nbytes: int, znn: "ZipNN" = None) -> torch.Tensor:
        """A stream stored at [offset, offset + nbytes) of an open file -> CUDA tensor."""
        znn = znn if znn is not None else ZipNN(input_format="torch")
        head = os.pread(fd, min(nbytes, HEADER_LEN + 1 + 9 * 255), offset)

        def whole():
            buf = np.empty(nbytes, dtype=np.uint8)
            self._pread_into(fd, memoryview(buf), offset)
            return buf

        r = self._decode(znn, head, nbytes, lambda dst, a, b: self._fill_from_file(dst, fd, offset + a), whole)
        if r is None:
            return znn.decompress(torch.from_numpy(whole()).to(self.device))
        return r

    def submit_file_batch(self, fd: int, entries) -> list:
        """Every stream of a checkpoint shard at once: entries = [(file offset, byte length)], each a
        ZipNN torch-format stream -> list of CUDA tensors (None for an entry this path does not take:
        the caller falls back to `submit_file`).

        The byte range that holds the entries is read into pinned slabs by the reader threads, copied
        to ONE device buffer, and all tensors are decoded by one `zipnn_b200_decompress_batch` call:
        one launch per kernel for the whole shard instead of five per tensor (the reference and the
        side-stream path above decode per tensor, zipnn/zipnn.py:1601-1607)."""
        if not entries:
            return []
        L = _native.lib()
        lo = min(off for off, _ in entries)
        hi = max(off + n for off, n in entries)
        span = hi - lo
        cur = torch.cuda.current_stream(self.device)
        k = self._n % len(self._streams)
        st = self._streams[k]
        self._n += 1
        outs = [None] * len(entries)
        with torch.cuda.device(self.device):
            if self._flags is None or self._nflags == self._flags.numel():
                self._flags = torch.zeros(1024, dtype=torch.int32, device=self.device)
                self._nflags = 0
                for side in self._streams:
                    side.wait_stream(cur)
            fi = self._nflags
            self._nflags += 1
            flags = self._flags
            items = []
            keep = []
            for j, (off, nbytes) in enumerate(entries):
                znn = ZipNN(input_format="torch")
                head = os.pread(fd, min(nbytes, HEADER_LEN + 1 + 9 * 255), off)
                try:
                    after = znn._retrieve_header(head)
                except ValueError:
                    continue
                if znn.input_format != EnumFormat.TORCH.value or znn.is_streaming or nbytes < after:
                    continue
                num_buf = znn._num_buf_of_dtype()
                chunk = znn.compression_chunk if num_buf != 1 else min(HUF_MAX_BLOCK, znn.compression_chunk)
                items.append((j, off - lo + after, nbytes - after, num_buf, znn._bit_reorder, znn._byte_reorder, chunk, znn.original_len,
                              torch_dtype_of_code(znn.dtype), znn.shape_bytes))
            if not items:
                return outs
            with torch.cuda.stream(st):
                dbuf = torch.empty(64 + span + 16, dtype=torch.uint8, device=self.device)
                dspan = dbuf[64: 64 + span]
                self._upload(dspan, span, lambda dst, a, b: self._fill_from_file(dst, fd, lo + a), st)
                arr = (_native.BatchItem * len(items))()
                for i, (j, boff, blen, num_buf, bits, bytes_mode, chunk, n, tdt, shape) in enumerate(items):
                    out = torch.empty(max(n, 1), dtype=torch.uint8, device=self.device)[:n]
                    keep.append(out)
                    arr[i].d_body = dspan.data_ptr() + boff
                    arr[i].body_len = blen
                    arr[i].num_buf, arr[i].bits_mode, arr[i].bytes_mode = num_buf, bits, bytes_mode
                    arr[i].chunk, arr[i].orig = chunk, n
                    arr[i].d_out = out.data_ptr() if n else None
                    outs[j] = out.view(tdt).reshape(shape)
                wsz = C.c_size_t(0)
                _native.check(L.zipnn_b200_decompress_batch_workspace_size(arr, len(items), C.byref(wsz)))
                ws = torch.empty(wsz.value, dtype=torch.uint8, device=self.device)
                rc = L.zipnn_b200_decompress_batch(arr, len(items), ws.data_ptr(), ws.numel(), st.cuda_stream, 0)
                if rc == _native.E_CORRUPT:
                    raise RuntimeError("Thread processing failed: corrupt ZipNN stream")
                _native.check(rc)
                flags[fi: fi + 1].copy_(ws[:4].view(torch.int32), non_blocking=True)
                done = torch.cuda.Event()
                done.record(st)
            cur.wait_event(done)
            for t in keep:
                t.record_stream(cur)
            dbuf.record_stream(st)
            ws.record_stream(st)
            self._pending.append((flags, fi, lambda: None))
        return outs

    def finish(self):
        """Wait for everything submitted and report errors."""
        pending, self._pending = self._pending, []
        for st in self._streams:
            st.synchronize()
        if not pending:
            return
        host = {}
        for fl, _, _ in pending:
            if id(fl) not in host:
                host[id(fl)] = fl.cpu().numpy()
        vals = [int(host[id(fl)][fi]) for fl, fi, _ in pending]
        if any(v & 1 for v in vals):
            raise RuntimeError("Thread processing failed: corrupt ZipNN stream")
        if any(v & 2 for v in vals):
            _native.check(_native.E_UNSUPPORTED)
        for v, (_, _, redo) in zip(vals, pending):
            if v & 4:
                redo()
        torch.cuda.current_stream(self.device).synchronize()

    def release(self):
        """Give the pinned slabs back for the next pipe (after `finish`)."""
        for j, evt in enumerate(self._stage_evt):
            if evt is not None:
                evt.synchronize()
        for j, sl in enumerate(self._stage):
            if sl is not None and sl.numel() == self.SLAB_BYTES:
                DecodePipe._give_slab(sl)
            self._stage[j] = None
            self._stage_evt[j] = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


# ---------------------------------------------------------------------- native calls
def _as_stream(data):
    """CUDA/CPU uint8 tensor stays a tensor if on CUDA; everything else becomes a uint8 ndarray."""
    if isinstance(data, torch.Tensor):
        if data.is_cuda and data.dtype == torch.uint8 and data.dim() == 1 and data.is_contiguous():
            return data    # what compress returns: no view ops on the way in
        t = data.detach().contiguous().reshape(-1)
        t = t if t.dtype == torch.uint8 else t.view(torch.uint8)
        return t if t.is_cuda else t.numpy()
    return _as_u8_numpy(data)


def _peek(stream, nbytes: int) -> bytes:
    """The first nbytes of a stream.  For a CUDA stream, one synchronising copy through the library's pinned block:
    a tensor slice copied to the host costs several torch calls and a pageable copy while the GPU waits."""
    if isinstance(stream, torch.Tensor):
        n = min(nbytes, stream.numel())
        buf = C.create_string_buffer(n)
        with _on_device(stream.device):
            _native.check(_native.lib().zipnn_b200_peek(stream.data_ptr(), n, buf, _cuda_stream_handle(stream.device)))
        return buf.raw
    return stream[:nbytes].tobytes()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _cuda_stream_handle(device=None) -> int:
    """cudaStream_t of the current stream of `device` (default: the current device)."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device() if device is None or device.index is None else device.index)
    return torch.cuda.current_stream(device).cuda_stream


def _on_device(device):
    """The native calls launch on the current device: make it `device` for the call, when it is not already."""
    if device.index is None or device.index == torch.cuda.current_device():
        return contextlib.nullcontext()
    return torch.cuda.device(device)


def _aligned(t: torch.Tensor) -> torch.Tensor:
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _compress_device(flat_u8: torch.Tensor, header: bytes, num_buf: int, bits_mode: int, bytes_mode: int,
                     chunk: int, threshold: float) -> torch.Tensor:
    """`flat_u8`: a contiguous CUDA tensor of any dtype, coded as its bytes."""
    flat_u8 = _aligned(flat_u8)
    n = flat_u8.nbytes
    dev = flat_u8.device
    bound = _native.compress_bound(n, num_buf, chunk, len(header))
    wsz = _native.compress_workspace_size(n, num_buf, chunk)
    with _on_device(dev):
        out = torch.empty(bound, dtype=torch.uint8, device=dev)
        ws = torch.empty(wsz, dtype=torch.uint8, device=dev)
        out_len = C.c_size_t(0)
        _native.check(_native.lib().zipnn_b200_compress(flat_u8.data_ptr() if n else None, n, header, len(header), num_buf,
                                                        bits_mode, bytes_mode, chunk, threshold, out.data_ptr(), bound,
                                                        C.byref(out_len), ws.data_ptr(), wsz, _cuda_stream_handle(dev)))
    return out[: out_len.value]


def _batch_items(flats: list, plans: list):
    """-> (zipnn_b200_compress_item array without d_out, header buffers to keep alive, output offsets, output
    bytes): item i codes flats[i] as `plan()` i says, into its bound at its offset (256-byte steps) of one buffer."""
    items = (_native.CompressItem * len(flats))()
    hdrs, offs, at = [], [], 0
    for it, f, p in zip(items, flats, plans):
        hdr = C.create_string_buffer(p["header"], len(p["header"]))
        hdrs.append(hdr)
        it.d_in, it.n = (f.data_ptr() if f.numel() else None), f.numel()
        it.h_hdr, it.hdr_len = C.cast(hdr, C.c_void_p), len(p["header"])
        it.num_buf, it.bits_mode, it.bytes_mode = p["num_buf"], p["bit_reorder"], p["byte_reorder"]
        it.chunk, it.threshold = p["chunk"], p["threshold"]
        it.out_cap = _native.compress_bound(f.numel(), p["num_buf"], p["chunk"], len(p["header"]))
        offs.append(at)
        at += (it.out_cap + 255) // 256 * 256
    return items, hdrs, offs, at


def _compress_device_batch(flats: list, plans: list) -> list:
    """Flat uint8 CUDA tensors (one device) and their `ZipNN.plan()`s -> their streams, views into one
    output buffer, from one `zipnn_b200_compress_batch` call and one workspace."""
    _native.require_cuda()
    L = _native.lib()
    flats = [_aligned(f) for f in flats]
    n = len(flats)
    items, hdrs, offs, at = _batch_items(flats, plans)   # (hdrs: alive until the call returns, which copies them)
    dev = flats[0].device
    with torch.cuda.device(dev):
        out = torch.empty(at, dtype=torch.uint8, device=dev)
        for it, o in zip(items, offs):
            it.d_out = out.data_ptr() + o
        wsz = C.c_size_t(0)
        _native.check(L.zipnn_b200_compress_batch_workspace_size(items, n, C.byref(wsz)))
        ws = torch.empty(max(wsz.value, 1), dtype=torch.uint8, device=dev)
        lens = (C.c_size_t * n)()
        _native.check(L.zipnn_b200_compress_batch(items, n, lens, ws.data_ptr(), ws.numel(), _cuda_stream_handle()))
    return [out[o: o + lens[i]] for i, o in enumerate(offs)]


def _decompress_device(body: torch.Tensor, num_buf: int, bits_mode: int, bytes_mode: int, chunk: int,
                       orig: int, body_off: int = 0, out: torch.Tensor = None) -> torch.Tensor:
    """Decode body[body_off:] (a flat uint8 CUDA tensor) into `out` (a contiguous tensor of orig bytes on the same
    device; by default a new uint8 one) and return `out`."""
    dev = body.device
    with _on_device(dev):
        if out is None:
            out = torch.empty(orig, dtype=torch.uint8, device=dev)
        if orig == 0:
            return out
        st = _native.E_CAPACITY
        for full in (False, True):   # the full workspace is only needed by unusual streams
            wsz = _native.decompress_workspace_size(orig, num_buf, chunk, full=full)
            ws = torch.empty(wsz, dtype=torch.uint8, device=dev)
            st = _native.lib().zipnn_b200_decompress(body.data_ptr() + body_off, body.numel() - body_off, num_buf, bits_mode,
                                                     bytes_mode, chunk, orig, out.data_ptr(), ws.data_ptr(), wsz,
                                                     _cuda_stream_handle(dev), 1)
            if st != _native.E_CAPACITY:
                break
    if st == _native.E_CORRUPT:
        raise RuntimeError("Thread processing failed: corrupt ZipNN stream")  # reference: zipnn_core.c:1089
    _native.check(st)
    return out


def _pinned_empty(nbytes: int) -> torch.Tensor:
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)


def _host_tensor(a) -> torch.Tensor:
    """Flat uint8 CPU tensor over host bytes without copying (numpy arrays may be read-only)."""
    if isinstance(a, torch.Tensor):
        return a
    if a.size == 0:
        return torch.empty(0, dtype=torch.uint8)
    if a.flags.writeable:
        return torch.from_numpy(a)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return torch.from_numpy(a)   # only ever read from


def _host_out(nbytes: int, out):
    """Host destination for a result: the caller's buffer (`out=`), else fresh pinned memory
    (torch's caching host allocator makes repeated calls cheap)."""
    if out is None:
        return _pinned_empty(nbytes)[:nbytes]
    o = out.detach().reshape(-1)
    o = o if o.dtype == torch.uint8 else o.view(torch.uint8)
    if o.is_cuda or not o.is_contiguous() or o.numel() < nbytes:
        raise ValueError("out= must be a contiguous CPU tensor with room for the result")
    return o[:nbytes]


def _compress_host(flat_u8, header: bytes, num_buf: int, bits_mode: int, bytes_mode: int, chunk: int,
                   threshold: float, out=None):
    """Host bytes in, host bytes out through `zipnn_b200_compress_host` (include/zipnn_b200.h): the library
    moves the input through the device slab by slab, with the copies in both directions and the kernels
    overlapped.  Pinned buffers (torch pin_memory) get the full PCIe rate; any host memory works."""
    _native.require_cuda()
    L = _native.lib()
    src = _host_tensor(flat_u8)
    n = src.numel()
    if out is None:
        host = _host_out(_native.compress_bound(n, num_buf, chunk, len(header)), None)
    else:   # the size is not known in advance: use whatever room the caller gave, the library checks as it goes
        host = out.detach().reshape(-1)
        host = host if host.dtype == torch.uint8 else host.view(torch.uint8)
        if host.is_cuda or not host.is_contiguous():
            raise ValueError("out= must be a contiguous CPU tensor with room for the result")
    hdr = (C.c_char * len(header)).from_buffer_copy(header)
    out_len = C.c_size_t(0)
    rc = L.zipnn_b200_compress_host(src.data_ptr() if n else None, n, hdr, len(header), num_buf, bits_mode, bytes_mode, chunk, threshold,
                                    host.data_ptr(), host.numel(), C.byref(out_len))
    if rc == _native.E_CAPACITY:
        raise ValueError("out= must be a contiguous CPU tensor with room for the result")
    _native.check(rc)
    return memoryview(host.numpy()[: out_len.value])


def _decompress_host(body: np.ndarray, num_buf: int, bits_mode: int, bytes_mode: int, chunk: int, orig: int, out=None) -> torch.Tensor:
    """Host stream in, host bytes out through `zipnn_b200_decompress_host`: chunk ranges of 256 MiB are a
    stream of their own once their table rows are rebased, so the library decodes slab by slab on two
    CUDA streams with the H2D copy, the kernels and the D2H copy of neighbouring slabs overlapped."""
    _native.require_cuda()
    host = _host_out(orig, out)
    if orig == 0:
        return host
    src = _host_tensor(np.ascontiguousarray(body))
    rc = _native.lib().zipnn_b200_decompress_host(src.data_ptr(), src.numel(), num_buf, bits_mode, bytes_mode, chunk, orig, host.data_ptr())
    if rc == _native.E_CORRUPT:
        raise RuntimeError("Thread processing failed: corrupt ZipNN stream")   # reference: zipnn_core.c:1089
    _native.check(rc)
    return host
