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
import time

import torch
from safetensors import safe_open as _safe_open
from safetensors.torch import save_file as _save_file

from .slicing import CompressedSlice
from .util_header import EnumFormat
from .util_patch import multi_process_patcher
from .util_safetensors import (COMPRESSED_DTYPE, COMPRESSION_METHOD, METADATA_KEY, build_compressed_tensor_info,
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


def _safetensors_header(filename) -> tuple:
    """-> (file offset of the data, the header's JSON dict) of a safetensors file
    (8-byte little-endian length, JSON with `data_offsets` relative to the end of the header)."""
    import json
    with open(filename, "rb") as f:
        hlen = int.from_bytes(f.read(8), "little")
        meta = json.loads(f.read(hlen))
    return 8 + hlen, meta


def _safetensors_index(filename) -> dict:
    """{tensor name: (absolute file offset, byte length)} from the safetensors header."""
    base, meta = _safetensors_header(filename)
    return {k: (base + v["data_offsets"][0], v["data_offsets"][1] - v["data_offsets"][0])
            for k, v in meta.items() if k != "__metadata__"}


class FileEntry:
    """One tensor of a safetensors / .znn.safetensors file, from the header alone: `nbytes` at `offset` of `file`,
    the tensor's dtype and shape (for a compressed entry those of `znn_compressed_vectors`, not of its uint8
    stream), whether it is compressed, and whether the file is a .znn file (one with that metadata key)."""

    def __init__(self, file, offset, nbytes, dtype, shape, compressed, znn_file):
        self.file, self.offset, self.nbytes, self.dtype, self.shape = file, offset, nbytes, dtype, tuple(shape)
        self.compressed, self.znn_file = compressed, znn_file

    @property
    def floating(self) -> bool:
        return self.dtype in _FLOAT_DTYPES


def file_entries(filenames) -> dict:
    """{name: FileEntry} over the headers of several files, the shards of one checkpoint (no tensor data is read).
    ValueError for a name found in two files or a dtype the header names that torch lacks."""
    import json
    from safetensors.torch import _getdtype
    out, dups, bad = {}, [], []
    for fn in filenames:
        base, meta = _safetensors_header(fn)
        file_meta = meta.get("__metadata__") or {}
        comp = get_compressed_tensors_metadata(file_meta)
        znn = METADATA_KEY in file_meta
        for k, v in meta.items():
            if k == "__metadata__":
                continue
            if k in out:
                dups.append(k)
                continue
            a, b = v["data_offsets"]
            info = comp.get(k)
            try:
                if info is not None:
                    dtype, shape = getattr(torch, info["dtype"]), json.loads(info["shape"])
                    if not isinstance(dtype, torch.dtype):
                        raise AttributeError(info["dtype"])
                else:
                    dtype, shape = _getdtype(v["dtype"]), v["shape"]
            except (AttributeError, KeyError, TypeError, ValueError):
                bad.append(k)
                continue
            out[k] = FileEntry(fn, base + a, b - a, dtype, shape, info is not None, znn)
    if dups:
        raise ValueError(f"keys found in more than one file: {sorted(set(dups))}")
    if bad:
        raise ValueError(f"keys with a dtype or shape this reader does not know: {bad}")
    return out


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


# Input bytes per batched compress call when a file is written from many tensors: bounds the device memory
# of one group (its inputs, the streams' bound and the workspace).  A larger tensor is a group on its own.
SAVE_GROUP_BYTES = 1 << 30


def _plan_groups(sizes, budget: int) -> list:
    """Consecutive index groups whose byte sizes add up to at most `budget`; an entry larger than the budget
    is a group on its own.  Order is kept."""
    groups, cur, acc = [], [], 0
    for i, s in enumerate(sizes):
        if cur and acc + s > budget:
            groups.append(cur)
            cur, acc = [], 0
        cur.append(i)
        acc += s
    if cur:
        groups.append(cur)
    return groups


# safetensors dtype names of the floating-point types (anything else is stored as it is)
_ST_DTYPES = {"F64": "float64", "F32": "float32", "F16": "float16", "BF16": "bfloat16", "F8_E4M3": "float8_e4m3fn",
              "F8_E5M2": "float8_e5m2"}
_FLOAT_DTYPES = frozenset(getattr(torch, v) for v in _ST_DTYPES.values())


class _FileRange:
    """A tensor's bytes in a file: `nbytes` at `offset` of the open descriptor `fd`."""

    def __init__(self, fd: int, offset: int, nbytes: int, dtype: torch.dtype, shape):
        self.fd, self.offset, self.nbytes, self.dtype, self.shape = fd, offset, nbytes, dtype, list(shape)


def _entry_bytes(src) -> int:
    return src.nbytes if isinstance(src, _FileRange) else src.element_size() * src.nelement()


def _pread_into(fd: int, mv, off: int) -> None:
    while len(mv):
        got = os.preadv(fd, [mv], off)
        if got <= 0:
            raise OSError(f"short read at offset {off}")
        mv, off = mv[got:], off + got


def _cuda_index(device) -> torch.device:
    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _align256(v: int) -> int:
    return (v + 255) // 256 * 256


class _Group:
    """One compressed group of `compress_groups`: `grp` indices into its entries, `flats` the inputs on the device,
    `streams` their streams (views of the batch's output buffer, sized by the bound), `stage` / `place` the pinned
    staging buffer and each staged entry's offset in it, `events` [before h2d, after h2d, after the kernels]."""

    def __init__(self, grp, flats, streams, stage, place, events):
        self.grp, self.flats, self.streams, self.stage, self.place, self.events = grp, flats, streams, stage, place, events


def compress_groups(entries, device, timings=None):
    """Floating-point entries [(key, CPU/CUDA tensor or _FileRange)] -> one `_Group` per group of SAVE_GROUP_BYTES
    input bytes, compressed on `device` but not synchronised.  Host bytes are staged in pinned memory (file ranges
    read with pread) and copied with one host-to-device copy per group; a group is one `ZipNN.compress_batch` call.
    A group's device memory (its inputs, the streams' bound, the workspace) is released when the consumer moves on
    to the next one, so that one group at a time is on the device.  `timings` (a dict): seconds of staging, added up."""
    from .zipnn import _pinned_empty
    dev = _cuda_index(device)
    sizes = [_entry_bytes(src) for _, src in entries]
    for grp in _plan_groups(sizes, SAVE_GROUP_BYTES):
        t0 = time.perf_counter()
        host = [i for i in grp if not (isinstance(entries[i][1], torch.Tensor) and entries[i][1].is_cuda)]
        at, place = 0, {}
        for i in host:
            place[i] = at
            at += _align256(sizes[i])
        stage = _pinned_empty(at)
        for i in host:
            src, a = entries[i][1], place[i]
            if isinstance(src, _FileRange):
                _pread_into(src.fd, memoryview(stage.numpy())[a: a + src.nbytes], src.offset)
            elif sizes[i]:
                stage[a: a + sizes[i]].copy_(src.detach().contiguous().reshape(-1).view(torch.uint8))
        if timings is not None:
            timings["stage"] = timings.get("stage", 0.0) + (time.perf_counter() - t0)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record(stream)
            d_stage = stage[:at].to(dev, non_blocking=True) if host else None
            ev[1].record(stream)
            flats = []
            for i in grp:
                src = entries[i][1]
                if i in place:
                    s = d_stage[place[i]: place[i] + sizes[i]]
                    dt = src.dtype
                    shape = src.shape if isinstance(src, _FileRange) else tuple(src.shape)
                    flats.append(s.view(dt).view(shape) if sizes[i] else torch.empty(shape, dtype=dt, device=dev))
                else:
                    flats.append(src)
            streams = ZipNN(input_format="torch", method=COMPRESSION_METHOD).compress_batch(flats)
            ev[2].record(stream)
        yield _Group(grp, flats, streams, stage, place, ev)
        del flats, streams, d_stage   # before the next group is allocated


def _compress_entries(entries, device, timings=None):
    """Floating-point entries [(name, CPU/CUDA tensor or _FileRange)] -> ({name: CPU tensor}, infos,
    compressed bytes, original bytes), the choices `compress_safetensors_file` makes per tensor (a stream
    that is not smaller keeps the original bytes).  The groups of `compress_groups`; every stream is copied
    back into pinned memory.
    `timings` (a dict): seconds per phase, added up -- stage, h2d, kernels, d2h (device phases by events)."""
    from .zipnn import _pinned_empty
    dev = _cuda_index(device)
    out, infos = {}, {}
    comp_len = og_len = 0
    sizes = [_entry_bytes(src) for _, src in entries]
    for g in compress_groups(entries, dev, timings):
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream()
            lens = [s.numel() for s in g.streams]
            keep = [k for k, i in enumerate(g.grp) if lens[k] < sizes[i]]
            at, hplace = 0, {}
            for k in keep:
                hplace[k] = at
                at += _align256(lens[k])
            hout = _pinned_empty(at)
            for k in keep:
                hout[hplace[k]: hplace[k] + lens[k]].copy_(g.streams[k], non_blocking=True)
            done = torch.cuda.Event(enable_timing=True)
            done.record(stream)
            stream.synchronize()
        for k, i in enumerate(g.grp):
            name, src = entries[i]
            og_len += sizes[i]
            if k in hplace:
                comp_len += lens[k]
                out[name] = hout[hplace[k]: hplace[k] + lens[k]]
                infos[name] = build_compressed_tensor_info(g.flats[k])
            else:   # not smaller: the original bytes
                comp_len += sizes[i]
                if isinstance(src, _FileRange):
                    out[name] = g.stage[g.place[i]: g.place[i] + sizes[i]].clone().view(src.dtype).view(src.shape)
                else:
                    out[name] = src.cpu()
        if timings is not None:
            ev = g.events + [done]
            for key, a, b in (("h2d", 0, 1), ("kernels", 1, 2), ("d2h", 2, 3)):
                timings[key] = timings.get(key, 0.0) + ev[a].elapsed_time(ev[b]) / 1e3
        del g
    return out, infos, comp_len, og_len


def _check_like_safetensors(tensors) -> None:
    """What `safetensors.torch.save_file` refuses, before any GPU work: a non-dict, non-tensors, sparse or
    non-contiguous tensors and tensors sharing storage."""
    from safetensors.torch import _find_shared_tensors
    if not isinstance(tensors, dict):
        raise ValueError(f"Expected a dict of [str, torch.Tensor] but received {type(tensors)}")
    for k, v in tensors.items():
        if not isinstance(v, torch.Tensor):
            raise ValueError(f"Key `{k}` is invalid, expected torch.Tensor but received {type(v)}")
    sparse = [k for k, v in tensors.items() if v.layout != torch.strided]
    if sparse:
        raise ValueError(f"You are trying to save a sparse tensors: `{sparse}` which this library does not support.")
    failing = [names for names in _find_shared_tensors(tensors) if len(names) > 1]
    if failing:
        raise RuntimeError(f"Some tensors share memory, this will lead to duplicate memory on disk: {failing}.")
    for k, v in tensors.items():
        if not v.is_contiguous():
            raise ValueError(f"You are trying to save a non contiguous tensor: `{k}` which is not allowed.")


def _write_compressed(tensors, infos, metadata, path) -> None:
    metadata = dict(metadata) if metadata else {}
    set_compressed_tensors_metadata(infos, metadata)
    _save_file(tensors, path, metadata)


def _cuda_device(device):
    """The CUDA device that `device` names (a torch.device, "cuda" / "cuda:i", or a device index), else None."""
    if isinstance(device, bool) or device is None:
        return None
    if isinstance(device, int):
        return torch.device("cuda", device)
    try:
        d = torch.device(device)
    except (RuntimeError, TypeError, ValueError):
        return None
    return d if d.type == "cuda" else None


def save_file(tensors, filename, metadata=None) -> None:
    """The counterpart of `load_file`: a dict of CUDA and/or CPU tensors -> a `.znn.safetensors` file,
    byte for byte what `safetensors.torch.save_file` of the tensors followed by `compress_safetensors_file`
    writes.  Floating-point tensors are compressed on the GPU (CPU ones are staged in pinned memory and
    copied over), many per kernel launch; the file is written by `safetensors.torch.save_file`."""
    save_coded(tensors, {}, filename, metadata)


def save_coded(tensors, coded, filename, metadata=None) -> None:
    """`save_file` of `tensors` plus entries that are already compressed: `coded` = {name: (CUDA uint8 stream,
    dtype, shape)}, written as they are (one device-to-host copy each, no decode or encode)."""
    from .zipnn import _pinned_empty
    _check_like_safetensors(tensors)
    plain, floats = {}, []
    for name in sorted(tensors):   # the order a reader of the plain file lists them in, which the metadata JSON follows
        t = tensors[name]
        if zipnn_is_floating_point(EnumFormat.TORCH.value, t, t.dtype):
            floats.append((name, t))
        else:
            plain[name] = t.cpu()
    devices = {t.device for _, t in floats if t.is_cuda} | {s.device for s, _, _ in coded.values()}
    if len(devices) > 1:
        raise ValueError(f"save_file compresses on one GPU, but the tensors are on {sorted(map(str, devices))}: "
                         "move them to one device (or to the CPU) first")
    dev = devices.pop() if devices else torch.device("cuda")
    out, infos, _, _ = _compress_entries(floats, dev)
    plain.update(out)
    if coded:
        at, place = 0, {}
        for name, (s, _, _) in coded.items():
            place[name] = at
            at += _align256(s.numel())
        hout = _pinned_empty(at)
        with torch.cuda.device(dev):
            for name, (s, _, _) in coded.items():
                hout[place[name]: place[name] + s.numel()].copy_(s, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        for name, (s, dtype, shape) in coded.items():
            plain[name] = hout[place[name]: place[name] + s.numel()]
            infos[name] = build_compressed_tensor_info(torch.empty(shape, dtype=dtype, device="meta"))
        infos = {k: infos[k] for k in sorted(infos)}
    _write_compressed(plain, infos, metadata, filename)


def compress_safetensors_file(filename, delete=False, force=True, method=None, threads=None, device="cuda"):
    """`x.safetensors` -> `x.znn.safetensors` (scripts/zipnn_compress_safetensors.py:37-148).

    Floating-point tensors are stored as uint8 streams under their own name; a tensor whose
    stream is not smaller stays raw.  Deliberate divergence: the raw fallback stores the
    ORIGINAL bytes (the reference stores its in-place-rotated copy, SURVEY.md section 8b),
    and the metadata key is written even when the source file had no metadata dict.
    With a CUDA `device` ("cuda", "cuda:i", a torch.device or a device index), the floating-point entries are
    read with pread into pinned memory and compressed a group at a time by the batched encoder on that device
    (as `save_file`); any other `device` keeps the per-tensor path (tensor.to(device), then ZipNN.compress).
    Returns (compressed_path, compressed_bytes, original_bytes).
    """
    assert filename.endswith(".safetensors")
    compressed_path = filename[: -len(".safetensors")] + ".znn.safetensors"
    if not force and os.path.exists(compressed_path):
        raise FileExistsError(compressed_path)
    cuda = _cuda_device(device)
    if cuda is not None and method in (None, COMPRESSION_METHOD):
        index = _safetensors_index(filename)
        tensors, floats = {}, []
        fd = os.open(filename, os.O_RDONLY)
        try:
            with _safe_open(filename, "pt", "cpu") as f:
                for name in f.keys():
                    sl = f.get_slice(name)
                    dtype = getattr(torch, _ST_DTYPES.get(sl.get_dtype(), "uint8"))
                    if dtype.is_floating_point:
                        floats.append((name, _FileRange(fd, *index[name], dtype, sl.get_shape())))
                    else:
                        tensors[name] = f.get_tensor(name)
                metadata = f.metadata()
            out, infos, comp_len, og_len = _compress_entries(floats, cuda)
        finally:
            os.close(fd)
        tensors.update(out)
        _write_compressed(tensors, infos, metadata, compressed_path)
        if delete:
            os.remove(filename)
        return compressed_path, comp_len, og_len
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
