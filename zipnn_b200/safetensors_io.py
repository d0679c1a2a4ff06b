"""safetensors load-path plugin and the .znn.safetensors writer/reader.

Mirrors reference zipnn/zipnn.py:1584-1643 (`decompress_safetensors_tensor`, `SafeOpen`,
`zipnn_safetensors`), scripts/zipnn_compress_safetensors.py:37-148 and
scripts/zipnn_decompress_safetensors.py:34-136.

GPU behaviour: `SafeOpen(..., device="cuda")` reads a compressed entry as uint8 bytes,
moves the COMPRESSED bytes to the GPU, decodes there and returns a CUDA tensor, so a
consumer such as vLLM's weight iterator (`for name in f.keys(): f.get_tensor(name)`) pays
the H2D copy on ~2/3 of the bytes and the decode on the GPU.  With device="cpu" the tensor
comes back on the host, as in the reference.
"""
from __future__ import annotations

import functools
import os

import torch
from safetensors import safe_open as _safe_open
from safetensors.torch import save_file as _save_file

from .slicing import CompressedSlice
from .util_header import EnumFormat
from .util_patch import multi_process_patcher
from .util_safetensors import (COMPRESSED_DTYPE, COMPRESSION_METHOD, build_compressed_tensor_info,
                               get_compressed_tensors_metadata, set_compressed_tensors_metadata)
from .util_torch import zipnn_is_floating_point
from .zipnn import DecodePipe, ZipNN


def decompress_safetensors_tensor(tensor: torch.Tensor, device=None) -> torch.Tensor:
    """Decode one compressed entry (a uint8 tensor holding a ZipNN stream).
    zipnn/zipnn.py:1584-1589.  `device` cuda => decode on that GPU and return a CUDA tensor."""
    znn = ZipNN(input_format="torch", bytearray_dtype=COMPRESSED_DTYPE, method=COMPRESSION_METHOD)
    dev = torch.device(device) if device is not None else tensor.device
    if dev.type == "cuda":
        return znn.decompress(tensor.contiguous().to(dev, non_blocking=True))
    return znn.decompress(tensor.contiguous())


def _safetensors_index(filename) -> dict:
    """{tensor name: (absolute file offset, byte length)} from the safetensors header
    (8-byte little-endian length, JSON with `data_offsets` relative to the end of the header)."""
    import json
    with open(filename, "rb") as f:
        hlen = int.from_bytes(f.read(8), "little")
        meta = json.loads(f.read(hlen))
    base = 8 + hlen
    return {k: (base + v["data_offsets"][0], v["data_offsets"][1] - v["data_offsets"][0])
            for k, v in meta.items() if k != "__metadata__"}


class SafeOpen:
    """`safetensors.safe_open` wrapper that decodes compressed tensors on access
    (zipnn/zipnn.py:1592-1626)."""

    def __init__(self, filename, framework, device="cpu", batch=True, slices=False):
        """`batch` (CUDA devices only): decode all compressed tensors of the file with one batched call on
        the first access instead of one call per tensor; costs device memory for the whole file at once.
        `slices`: `get_slice` of a compressed entry returns a `CompressedSlice`, whose `[index]` reads and
        decodes only the chunks the index covers (a tensor-parallel loader's shards).  Off by default, where
        `get_slice` answers as the reference does."""
        self._device = device
        self._batch = batch
        self._slices = slices
        self._slice_fd = None      # own descriptor of the slices' reads (payload ranges straight into pinned memory)
        self._slice_index = None
        self._slice_cache = {}
        self._ready = {}
        self._filename = filename
        self._f = _safe_open(filename, framework, device)
        self.compressed_tensors_metadata = get_compressed_tensors_metadata(self._f.metadata())
        dev = torch.device(device) if isinstance(device, (str, torch.device)) else torch.device("cuda", device)
        self._cuda = dev if dev.type == "cuda" else None
        self._fd = None         # own descriptor: compressed bytes are read straight into pinned staging slabs
        self._index = None
        self._pipe = None

    def get_tensor(self, name):
        if name not in self.compressed_tensors_metadata:
            return self._f.get_tensor(name)
        if self._cuda is None:
            return decompress_safetensors_tensor(self._f.get_tensor(name))
        # GPU load path: header parsed on the host, compressed bytes through a pinned staging buffer,
        # decode on a side stream, no host synchronisation per tensor (errors surface in close()).
        if self._pipe is None:
            self._index = _safetensors_index(self._filename)
            self._fd = os.open(self._filename, os.O_RDONLY)
            self._pipe = DecodePipe(self._cuda)
            if self._batch:
                # every compressed entry of the file in one go: one read of the byte range, one H2D buffer,
                # ONE launch per decode kernel for the whole shard; tensors are handed out as they are asked for
                names = sorted(self.compressed_tensors_metadata, key=lambda k: self._index[k][0])
                names = [k for k in names if k in self._index]
                got = self._pipe.submit_file_batch(self._fd, [self._index[k] for k in names])
                self._ready = {k: t for k, t in zip(names, got) if t is not None}
        if name in self._ready:
            return self._ready.pop(name)
        off, nbytes = self._index[name]
        znn = ZipNN(input_format="torch", bytearray_dtype=COMPRESSED_DTYPE, method=COMPRESSION_METHOD)
        return self._pipe.submit_file(self._fd, off, nbytes, znn)

    def close(self):
        """Wait for the decodes still in flight and raise what they found (corrupt stream, ...)."""
        pipe, self._pipe = self._pipe, None
        fd, self._fd = self._fd, None
        self._ready = {}
        self._close_slices()
        try:
            if pipe is not None:
                pipe.finish()
        finally:
            if pipe is not None:
                pipe.release()
            if fd is not None:
                os.close(fd)

    def get_slice(self, name):
        if name not in self.compressed_tensors_metadata:
            return self._f.get_slice(name)
        if not self._slices:
            return NotImplementedError  # as the reference: slices of compressed tensors are unsupported
        if name not in self._slice_cache:
            if self._slice_fd is None:
                self._slice_index = _safetensors_index(self._filename)
                self._slice_fd = os.open(self._filename, os.O_RDONLY)
            off, nbytes = self._slice_index[name]
            self._slice_cache[name] = CompressedSlice(self._slice_fd, off, nbytes, self._cuda)
        return self._slice_cache[name]

    def _close_slices(self):
        fd, self._slice_fd = self._slice_fd, None
        self._slice_cache = {}
        if fd is not None:
            os.close(fd)

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_value, traceback):
        try:
            if exc_type is None:
                self.close()
        finally:
            self._pipe = None
            self._close_slices()
            if self._fd is not None:
                os.close(self._fd)
                self._fd = None
            r = self._f.__exit__(exc_type, exc_value, traceback)
        return r

    def __del__(self):
        try:
            if self._pipe is not None:
                self._pipe.finish()
        except Exception:
            pass

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return getattr(self._f, name)


def load_file(filename, device="cpu") -> dict:
    """Whole-file load (the shape of `safetensors.torch.load_file`): every tensor of a
    `.znn.safetensors` (or plain) file, compressed entries decoded -- on the GPU, many at a time,
    when `device` is a CUDA device."""
    with SafeOpen(filename, "pt", device) as f:
        return {name: f.get_tensor(name) for name in f.keys()}


def _zipnn_safetensors(slices=False):
    import safetensors.torch
    safetensors.torch.safe_open = functools.partial(SafeOpen, slices=True) if slices else SafeOpen


# one object per variant: the patcher applies each patch function once, and pickles it into spawned processes
_zipnn_safetensors_slices = functools.partial(_zipnn_safetensors, slices=True)


def zipnn_safetensors(slices=False):
    """Patch `safetensors.torch.safe_open` in this process and in every process spawned
    from it (zipnn/zipnn.py:1629-1643).  `slices=True` installs a SafeOpen whose `get_slice`
    of a compressed entry returns a `CompressedSlice`."""
    multi_process_patcher(_zipnn_safetensors_slices if slices else _zipnn_safetensors)


def compress_safetensors_file(filename, delete=False, force=True, method=None, threads=None, device="cuda"):
    """`x.safetensors` -> `x.znn.safetensors` (scripts/zipnn_compress_safetensors.py:37-148).

    Floating-point tensors are stored as uint8 streams under their own name; a tensor whose
    stream is not smaller stays raw.  Deliberate divergence: the raw fallback stores the
    ORIGINAL bytes (the reference stores its in-place-rotated copy, SURVEY.md section 8b),
    and the metadata key is written even when the source file had no metadata dict.
    Returns (compressed_path, compressed_bytes, original_bytes).
    """
    assert filename.endswith(".safetensors")
    compressed_path = filename[: -len(".safetensors")] + ".znn.safetensors"
    if not force and os.path.exists(compressed_path):
        raise FileExistsError(compressed_path)
    tensors, infos = {}, {}
    comp_len = og_len = 0
    with _safe_open(filename, "pt", "cpu") as f:
        for name in f.keys():
            tensor = f.get_tensor(name)
            if not zipnn_is_floating_point(EnumFormat.TORCH.value, tensor, tensor.dtype):
                tensors[name] = tensor
                continue
            znn = ZipNN(input_format="torch", bytearray_dtype=tensor.dtype,
                        method=method if method is not None else COMPRESSION_METHOD, threads=threads)
            size = tensor.element_size() * tensor.nelement()
            og_len += size
            src = tensor.to(device, non_blocking=True) if device else tensor
            buf = znn.compress(src)
            clen = buf.numel() if isinstance(buf, torch.Tensor) else len(buf)
            if clen >= size:
                tensors[name] = tensor
                comp_len += size
                continue
            comp_len += clen
            tensors[name] = buf.cpu() if isinstance(buf, torch.Tensor) else torch.frombuffer(bytearray(buf), dtype=COMPRESSED_DTYPE)
            infos[name] = build_compressed_tensor_info(tensor)
        metadata = f.metadata()
    metadata = dict(metadata) if metadata else {}
    set_compressed_tensors_metadata(infos, metadata)
    _save_file(tensors, compressed_path, metadata)
    if delete:
        os.remove(filename)
    return compressed_path, comp_len, og_len


def decompress_safetensors_file(filename, delete=False, force=True, device="cuda"):
    """`x.znn.safetensors` -> `x.safetensors` (scripts/zipnn_decompress_safetensors.py:34-136)."""
    assert filename.endswith(".znn.safetensors")
    out_path = filename[: -len(".znn.safetensors")] + ".safetensors"
    if not force and os.path.exists(out_path):
        raise FileExistsError(out_path)
    tensors = {}
    with SafeOpen(filename, "pt", "cpu") as f:
        meta = f.metadata()
        for name in f.keys():
            if name in f.compressed_tensors_metadata:
                raw = f._f.get_tensor(name)
                t = decompress_safetensors_tensor(raw, device=device)
                tensors[name] = t.cpu()
            else:
                tensors[name] = f._f.get_tensor(name)
    meta = {k: v for k, v in (meta or {}).items() if k != "znn_compressed_vectors"}
    _save_file(tensors, out_path, meta or None)
    if delete:
        os.remove(filename)
    return out_path
