"""`DecodePlan` -- decode the same compressed tensors again and again with no host work per decode.

A plan is made once from a list of CUDA torch-format ZipNN streams: their headers are parsed (one synchronising
device-to-host copy for all of them), the outputs are laid out in one buffer, and `zipnn_b200_decode_plan_create`
validates the streams, builds everything that depends only on them and decodes once, recording where every segment
of the per-bitstream-CTA decoder starts.  `run()` then only enqueues the decode kernels, which decode each segment
once from its recorded start, on the current CUDA stream (a fixed number of launches, capturable in a CUDA graph) and
rewrites the same output tensors.  This is what keeps weights compressed in HBM (resident.py): a module's weights
are decoded just before it runs.

Lifetime rules (include/zipnn_b200.h): the streams must not change while the plan lives (the plan keeps references
to them); plans that share a scratch buffer must run ordered on one stream; plans that share an output buffer
overwrite each other's outputs.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import torch

from . import _native
from .util_header import EnumFormat
from .util_torch import torch_dtype_of_code
from .zipnn import HEADER_LEN, HUF_MAX_BLOCK, ZipNN, _cuda_stream_handle

_HEAD = HEADER_LEN + 1 + 9 * 255   # the 32-byte header and the longest packed shape (as decompress peeks)
_ALIGN = 16
GATHER_SLOTS = 64   # chunk slots of gather's default scratch: 16 MiB for 256 KiB chunks
MATVEC_MAX_TOKENS = _native.MATVEC_MAX_TOKENS
MATMUL_MAX_TOKENS = _native.MATMUL_MAX_TOKENS
EXPERTS_MATVEC_MAX_TOKENS = _native.EXPERTS_MATVEC_MAX_TOKENS
_MATVEC_DTYPES = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 2}   # ZIPNN_B200_MATVEC_*
_MATMUL_DTYPES = (torch.bfloat16, torch.float16)
_FP8_FORMATS = {torch.float8_e4m3fn: _native.FP8_E4M3, torch.float8_e5m2: _native.FP8_E5M2}   # ZIPNN_B200_FP8_*
_SELECT_FP8_MAX_ITEMS = 4   # outputs of a plan dequant_fp8_select takes (kSelectFp8MaxItems)


class _Product(NamedTuple):
    """What sets one product of `DecodePlan` apart from the others."""
    name: str        # the method's, and zipnn_b200_decode_plan_{name} / _{name}_scratch_size
    limit: int       # rows of x
    weights: dict    # weight dtype -> its code in the native calls (the fp8 format, or the dtype)
    x_dtypes: tuple  # x's dtypes, or None: the weights'
    scaled: bool     # fp8 weights with a scale grid: the native calls take the format and x's dtype, and the grid

    def native(self, suffix: str = ""):
        return getattr(_native.lib(), f"zipnn_b200_decode_plan_{self.name}{suffix}")


_MATVEC = _Product("matvec", MATVEC_MAX_TOKENS, _MATVEC_DTYPES, None, False)
_MATMUL = _Product("matmul", MATMUL_MAX_TOKENS, {dt: _MATVEC_DTYPES[dt] for dt in _MATMUL_DTYPES}, None, False)
_MATVEC_FP8 = _Product("matvec_fp8", MATVEC_MAX_TOKENS, _FP8_FORMATS, _MATMUL_DTYPES, True)
_MATMUL_FP8 = _Product("matmul_fp8", MATMUL_MAX_TOKENS, _FP8_FORMATS, _MATMUL_DTYPES, True)


def _round(n: int, a: int) -> int:
    return (n + a - 1) // a * a


class _Stream:
    """What the header of one torch-format stream says: where the body starts, the decoded bytes and layout."""

    def __init__(self, stream: torch.Tensor, head: bytes):
        z = ZipNN(input_format="torch")
        if len(head) < HEADER_LEN:
            raise ValueError("Header should start with ZN")
        after = z._retrieve_header(head)
        if z.input_format != EnumFormat.TORCH.value or head[9] != 0 or z.is_streaming:
            raise ValueError("DecodePlan takes torch-format streams without delta compression or streaming frames")
        if stream.numel() < after:
            raise RuntimeError("corrupt ZipNN stream: truncated header")
        self.stream = stream
        self.after = after
        self.num_buf = z._num_buf_of_dtype()
        self.bits_mode, self.bytes_mode = z._bit_reorder, z._byte_reorder
        self.chunk = z.compression_chunk if self.num_buf != 1 else min(HUF_MAX_BLOCK, z.compression_chunk)
        self.nbytes = z.original_len
        self.dtype = torch_dtype_of_code(z.dtype)
        self.shape = tuple(z.shape_bytes)


def _parse(streams) -> list:
    streams = [s for s in streams]
    for s in streams:
        if not (isinstance(s, torch.Tensor) and s.is_cuda and s.dtype == torch.uint8 and s.dim() == 1 and s.is_contiguous()):
            raise ValueError("DecodePlan takes flat contiguous CUDA uint8 streams")
    if len({s.device for s in streams}) > 1:
        raise ValueError("DecodePlan takes streams on one device")
    if not streams:
        return []
    heads = torch.cat([s[:_HEAD] for s in streams]).cpu().numpy().tobytes()   # one synchronising copy
    out, at = [], 0
    for s in streams:
        k = min(s.numel(), _HEAD)
        out.append(_Stream(s, heads[at: at + k]))
        at += k
    return out


def _offsets(parsed) -> tuple:
    offs, at = [], 0
    for p in parsed:
        offs.append(at)
        at = _round(at + p.nbytes, _ALIGN)
    return offs, at


def _items(parsed, offs, out_ptr: int):
    arr = (_native.SliceItem * max(1, len(parsed)))()
    for it, p, o in zip(arr, parsed, offs):
        it.d_body, it.body_len = p.stream.data_ptr() + p.after, p.stream.numel() - p.after
        it.num_buf, it.bits_mode, it.bytes_mode = p.num_buf, p.bits_mode, p.bytes_mode
        it.chunk, it.orig = p.chunk, p.nbytes
        it.base, it.rows, it.pitch, it.len = 0, 1, p.nbytes, p.nbytes
        it.d_out = out_ptr + o
    return arr


def _sizes(parsed) -> tuple:
    """-> (out bytes, plan bytes, scratch bytes)."""
    offs, out_bytes = _offsets(parsed)
    arr = _items(parsed, offs, 1 << 12)   # (any aligned non-null address: sizing reads no output)
    pb, sb = C.c_size_t(0), C.c_size_t(0)
    # (synchronising: reads the streams' type rows to size the segment index)
    _native.check(_native.lib().zipnn_b200_decode_plan_size(arr, len(parsed), _cuda_stream_handle(), C.byref(pb), C.byref(sb)))
    return out_bytes, pb.value, sb.value


def _raise_status(rc: int) -> None:
    if rc == _native.E_CORRUPT:
        raise _native.ZipNNNativeError(rc, "Thread processing failed: corrupt ZipNN stream")
    if rc == _native.E_INDEX:
        raise IndexError("zipnn_b200: a gather or selected run of this plan met an id outside [0, rows) (a gather zeroed "
                         "its rows, a selected run selected nothing for it)")
    _native.check(rc)


class DecodePlan:
    """Decode `streams` (CUDA uint8 torch-format ZipNN streams on one device, as `ZipNN(input_format="torch")
    .compress` or `compress_batch` return them) into `.outputs` now and on every `run()`.

    out:     optional CUDA uint8 buffer of at least `DecodePlan.sizes(streams)[0]` bytes that receives the outputs
             (at 16-byte aligned offsets); allocated when not given.
    scratch: optional CUDA uint8 buffer of at least `DecodePlan.sizes(streams)[1]` bytes, 256-byte aligned, for the
             plane pools of a run; allocated when not given.  Plans whose runs are ordered on one stream may share it.
    Raises like `ZipNN.decompress` when a stream is corrupt or unsupported.
    """

    @staticmethod
    def sizes(streams) -> tuple:
        """-> (out_bytes, scratch_bytes) a plan of these streams needs, so that callers can share buffers."""
        out_bytes, _, scratch_bytes = _sizes(_parse(streams))
        return out_bytes, scratch_bytes

    def __init__(self, streams, out: torch.Tensor = None, scratch: torch.Tensor = None):
        _native.require_cuda()
        parsed = _parse(streams)
        dev = parsed[0].stream.device if parsed else torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev):
            out_bytes, plan_bytes, scratch_bytes = _sizes(parsed)
            if out is None:
                out = torch.empty(max(out_bytes, 1), dtype=torch.uint8, device=dev)
            if scratch is None:
                scratch = torch.empty(max(scratch_bytes, 1), dtype=torch.uint8, device=dev)
            for name, buf, need, align in (("out", out, out_bytes, _ALIGN), ("scratch", scratch, scratch_bytes, 256)):
                if not (buf.is_cuda and buf.device == dev and buf.dtype == torch.uint8 and buf.is_contiguous()):
                    raise ValueError(f"{name} must be a contiguous CUDA uint8 tensor on the streams' device")
                if buf.numel() < need or buf.data_ptr() % align:
                    raise ValueError(f"{name} needs {need} bytes, {align}-byte aligned")
            self._meta = torch.empty(plan_bytes, dtype=torch.uint8, device=dev)
            offs, _ = _offsets(parsed)
            arr = _items(parsed, offs, out.data_ptr())
            self._plan = _native.DecodePlanStruct()
            rc = _native.lib().zipnn_b200_decode_plan_create(arr, len(parsed), self._meta.data_ptr(), plan_bytes, scratch.data_ptr(),
                                                              scratch_bytes, C.byref(self._plan), _cuda_stream_handle())
        _raise_status(rc)
        self._streams = [p.stream for p in parsed]   # the plan reads them on every run
        self._out, self._scratch = out, scratch
        self.device = dev
        self.outputs = [out[o: o + p.nbytes].view(p.dtype).reshape(p.shape) for p, o in zip(parsed, offs)]
        index_bytes, coded = C.c_size_t(0), C.c_size_t(0)
        _native.check(_native.lib().zipnn_b200_decode_plan_index(C.byref(self._plan), C.byref(index_bytes), C.byref(coded)))
        self.coded_items = coded.value
        self.nbytes = {"plan": plan_bytes, "scratch": scratch_bytes, "index": index_bytes.value, "out": out_bytes,
                       "streams": sum(p.stream.numel() for p in parsed), "dense": sum(p.nbytes for p in parsed)}
        self._run = _native.lib().zipnn_b200_decode_plan_run
        self._run_shifted = _native.lib().zipnn_b200_decode_plan_run_shifted
        self._gather = _native.lib().zipnn_b200_decode_plan_gather
        self._ref = C.byref(self._plan)
        self._offs = [(o, p.nbytes, p.dtype, p.shape) for p, o in zip(parsed, offs)]
        self._scratches = {}          # method name -> that call's default scratch, grown on demand
        self._product_ok = {}         # (method name, output, in_features) -> eligible?
        self._select_ok = None        # select_ok(), once asked

    def _check_out(self) -> None:
        if self._out is None:
            raise RuntimeError("DecodePlan: the output buffer was released (release_out); only gather runs")

    def _check_ids(self, name: str, ids) -> None:
        if not (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.device == self.device and ids.dtype in (torch.int32, torch.int64)):
            raise ValueError(f"{name} takes CUDA int32 or int64 ids on the plan's device")

    def _scratch_for(self, name: str, scratch, need) -> torch.Tensor:
        """The caller's `scratch` for method `name` once checked, or, for None, the plan's default scratch of that
        method, grown to `need()` bytes."""
        if scratch is None:
            n = need()
            own = self._scratches.get(name)
            if own is None or own.numel() < n:
                own = self._scratches[name] = torch.empty(n, dtype=torch.uint8, device=self.device)
            return own
        if not (isinstance(scratch, torch.Tensor) and scratch.is_cuda and scratch.device == self.device
                and scratch.dtype == torch.uint8 and scratch.is_contiguous()):
            raise ValueError(f"{name}'s scratch must be a contiguous CUDA uint8 tensor on the plan's device")
        return scratch

    def run(self) -> list:
        """Enqueue the decode on the current CUDA stream (launches only) and return `.outputs`."""
        self._check_out()
        rc = self._run(self._ref, torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return self.outputs

    def views(self, out: torch.Tensor) -> list:
        """The outputs' views of another buffer `out` (same offsets, dtypes and shapes as `.outputs`); ValueError
        unless `out` is a contiguous CUDA uint8 tensor on the plan's device, 16-byte aligned, of at least
        `nbytes["out"]` bytes."""
        self._check_out()
        if not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == torch.uint8
                and out.dim() == 1 and out.is_contiguous()):
            raise ValueError("run_into takes a flat contiguous CUDA uint8 tensor on the plan's device")
        if out.numel() < self.nbytes["out"] or out.data_ptr() % _ALIGN:
            raise ValueError(f"run_into needs {self.nbytes['out']} bytes, {_ALIGN}-byte aligned")
        return [out[o: o + n].view(dt).reshape(sh) for o, n, dt, sh in self._offs]

    def run_into(self, out: torch.Tensor, max_ctas: int = 0) -> list:
        """Enqueue the decode on the current CUDA stream as ONE kernel launch of at most `max_ctas` CTAs (0: as many
        as fit on the device) with the outputs in `out` instead of the create-time buffer, and return their views
        of `out` (as `views(out)`).  Runs of one plan, and of plans sharing a scratch buffer, must stay ordered on
        one stream, whichever of `run` and `run_into` enqueues them.  Needs a plan with a segment index (the
        default)."""
        views = self.views(out)
        rc = self._run_shifted(self._ref, out.data_ptr() - self._out.data_ptr(), int(max_ctas),
                               torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return views

    def release_out(self) -> None:
        """Drop the plan's reference to its output buffer (the one create decoded into), for a plan that only
        gathers: `run`, `run_into` and `views` raise RuntimeError from then on, `outputs` is None."""
        self._out, self.outputs = None, None

    def _gather_row(self, k: int) -> tuple:
        if not 0 <= k < len(self._offs):
            raise IndexError(f"DecodePlan has {len(self._offs)} outputs, not {k + 1}")
        _, n, dt, sh = self._offs[k]
        if len(sh) == 0 or sh[0] == 0:
            raise ValueError("gather takes rows along dim 0 of a non-empty output with at least one dimension")
        return n // sh[0], dt, sh

    def gather_scratch_bytes(self, k: int, slots: int) -> int:
        """Bytes of a gather scratch for output `k` with `slots` chunk slots (capped to the output's chunks): each
        gather pass decodes up to `slots` chunks, so more slots mean fewer launches and more memory."""
        row, _, _ = self._gather_row(k)
        out = C.c_size_t(0)
        _native.check(_native.lib().zipnn_b200_decode_plan_gather_scratch_size(self._ref, k, row, int(slots), C.byref(out)))
        return out.value

    def gather(self, k: int, ids: torch.Tensor, out: torch.Tensor = None, scratch: torch.Tensor = None) -> torch.Tensor:
        """Rows of output `k` along dim 0, as `outputs[k][ids]` would give them, decoded from the chunks the ids
        touch and no others (zipnn_b200_decode_plan_gather): enqueued on the current CUDA stream, launches only,
        the ids never read on the host, so it can be captured in a CUDA graph and replayed with new ids.

        ids:     CUDA int32 or int64 tensor of any shape on the plan's device.
        out:     optional contiguous tensor of shape `ids.shape + outputs[k].shape[1:]` and the output's dtype.
        scratch: optional 256-byte aligned CUDA uint8 buffer of at least `gather_scratch_bytes(k, 1)` bytes; its slot
                 count sets the passes.  It holds nothing between calls: calls (and plan runs) that share it must
                 be ordered on one stream.  Default: a buffer of GATHER_SLOTS slots kept by the plan.
        -> out.  An id outside [0, rows) gets a zero row and makes `check()` raise IndexError (from then on: the
        plan's error word is sticky).  Works without the plan's output buffer (`release_out`)."""
        row, dt, sh = self._gather_row(k)
        self._check_ids("gather", ids)
        ids_c = ids.contiguous()
        shape = tuple(ids.shape) + tuple(sh[1:])
        if out is None:
            out = torch.empty(shape, dtype=dt, device=self.device)
        elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == dt
                  and tuple(out.shape) == shape and out.is_contiguous()):
            raise ValueError(f"gather's out must be a contiguous {dt} CUDA tensor of shape {shape} on the plan's device")
        n = ids_c.numel()
        if n == 0:
            return out
        scratch = self._scratch_for("gather", scratch, lambda: self.gather_scratch_bytes(k, GATHER_SLOTS))
        rc = self._gather(self._ref, k, row, ids_c.data_ptr(), n, ids_c.element_size(), out.data_ptr(), scratch.data_ptr(),
                          scratch.numel(), torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return out

    def _select_size(self) -> tuple:
        """-> (status, scratch bytes) of zipnn_b200_decode_plan_select_scratch_size for rows = shape[0] of the outputs."""
        rows = {sh[0] if len(sh) else None for _, _, _, sh in self._offs}
        if len(rows) != 1 or None in rows or 0 in rows:
            return _native.E_UNSUPPORTED, 0
        out = C.c_size_t(0)
        rc = _native.lib().zipnn_b200_decode_plan_select_scratch_size(self._ref, rows.pop(), C.byref(out))
        return rc, out.value

    def select_ok(self) -> bool:
        """Can `run_select` decode slices of this plan's outputs?  True when every output has at least one dimension
        and the same `shape[0]` as the others, and is a whole tensor in one piece (not empty, at most 16383 chunks) of
        a plan with a segment index.  Never raises."""
        if self._select_ok is None:
            self._select_ok = self._select_size()[0] == _native.OK
        return self._select_ok

    def select_scratch_bytes(self) -> int:
        """Bytes of a `run_select` scratch for this plan (a few bytes per chunk; it depends on the plan alone)."""
        rc, n = self._select_size()
        _native.check(rc)
        return n

    def run_select(self, ids: torch.Tensor, scratch: torch.Tensor = None) -> list:
        """Enqueue the decode of the slices `outputs[k][e]` (along dim 0) of every output k for every id e in `ids`
        on the current CUDA stream, and return `.outputs` (zipnn_b200_decode_plan_run_select): only the chunks that
        meet a selected slice are decoded (whole), no other byte of the outputs is written, so the slices that were
        not selected hold unspecified bytes.  Launches only, a fixed number of them, the ids never read on the host:
        capturable in a CUDA graph and replayable with new ids copied into the captured tensor.

        ids:     CUDA int32 or int64 tensor of any shape on the plan's device; duplicates allowed; empty: nothing runs.
        scratch: optional 256-byte aligned CUDA uint8 buffer of at least `select_scratch_bytes()` bytes, not the plan's
                 own scratch.  It holds nothing between calls: calls that share it must be ordered on one stream.
                 Default: a buffer kept by the plan.
        An id outside [0, shape[0]) selects nothing and makes `check()` raise IndexError (from then on: the plan's
        error word is sticky).  ValueError for a plan `select_ok` refuses."""
        self._check_out()
        self._check_ids("run_select", ids)
        if not self.select_ok():
            raise ValueError("run_select needs outputs that share shape[0], each a whole tensor in one piece (see select_ok)")
        ids_c = ids.contiguous()
        n = ids_c.numel()
        if n == 0:
            return self.outputs
        scratch = self._scratch_for("run_select", scratch, self.select_scratch_bytes)
        rc = _native.lib().zipnn_b200_decode_plan_run_select(self._ref, self._offs[0][3][0], ids_c.data_ptr(), n, ids_c.element_size(),
                                                             scratch.data_ptr(), scratch.numel(),
                                                             torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return self.outputs

    def _product_item(self, k: int) -> tuple:
        """-> (dtype, elements) of output k."""
        if not 0 <= k < len(self._offs):
            raise IndexError(f"DecodePlan has {len(self._offs)} outputs, not {k + 1}")
        _, _, dt, sh = self._offs[k]
        return dt, math.prod(sh)

    def _product_size(self, kind: _Product, k: int, in_features: int, n_tokens: int) -> tuple:
        """-> (status, scratch bytes) of zipnn_b200_decode_plan_{kind.name}_scratch_size."""
        dt, _ = self._product_item(k)
        out = C.c_size_t(0)
        if dt not in kind.weights or in_features <= 0:
            return _native.E_UNSUPPORTED, 0
        dtype = () if kind.scaled else (kind.weights[dt],)
        with torch.cuda.device(self.device):
            rc = kind.native("_scratch_size")(self._ref, k, *dtype, int(in_features), int(n_tokens), C.byref(out))
        return rc, out.value

    def _ok(self, kind: _Product, k: int, in_features: int) -> bool:
        dt, n = self._product_item(k)
        if dt not in kind.weights or in_features <= 0 or n == 0 or n % in_features:
            return False
        key = (kind.name, k, in_features)
        if key not in self._product_ok:
            self._product_ok[key] = self._product_size(kind, k, in_features, 1)[0] == _native.OK
        return self._product_ok[key]

    def _scratch_bytes(self, kind: _Product, k: int, in_features: int, n_tokens: int) -> int:
        rc, n = self._product_size(kind, k, in_features, n_tokens)
        _native.check(rc)
        return n

    def matvec_ok(self, k: int, in_features: int) -> bool:
        """Can `matvec` multiply by output `k` seen as rows of `in_features` elements?  True for a bf16 / fp16 / fp32
        output in one piece whose rows are a multiple of 16 bytes and whose chunks all decode in the fused mode (what
        float weights produce; a constant tensor or a ragged tail does not).  The first call for an output
        synchronises (it reads the chunk modes); never raises for an output that exists."""
        return self._ok(_MATVEC, k, in_features)

    def matvec_scratch_bytes(self, k: int, in_features: int, n_tokens: int = MATVEC_MAX_TOKENS) -> int:
        """Bytes of a matvec scratch for output `k`, rows of `in_features` elements and `n_tokens` rows of x."""
        return self._scratch_bytes(_MATVEC, k, in_features, n_tokens)

    def matvec(self, k: int, x: torch.Tensor, bias: torch.Tensor = None, out: torch.Tensor = None,
               scratch: torch.Tensor = None) -> torch.Tensor:
        """`x @ W.T (+ bias)` with W = output `k` seen as [out_features, in_features], in_features = x.shape[-1],
        computed from the coded streams: W is neither written nor read dense (zipnn_b200_decode_plan_matvec).  Two
        launches on the current CUDA stream, no host read: capturable in a CUDA graph and replayable with new x.
        Products and sums are fp32, each result is rounded once; two calls with the same inputs give the same bits.

        x:       CUDA tensor [..., in_features] of the output's dtype on the plan's device, at most MATVEC_MAX_TOKENS
                 rows (product of the leading dims); rows that are not 16-byte aligned are copied first.
        bias:    optional contiguous [out_features] tensor of the same dtype.
        out:     optional tensor of shape x.shape[:-1] + (out_features,), same dtype, contiguous in its last dim
                 with equally spaced rows (e.g. a column slice of a wider buffer).
        scratch: optional 256-byte aligned CUDA uint8 buffer of at least `matvec_scratch_bytes(k, in_features, rows)`
                 bytes.  It holds nothing between calls: calls (and plan runs) that share it must be ordered on one
                 stream.  Default: a buffer kept by the plan.
        -> out.  ValueError for an output `matvec_ok` refuses.  Works without the plan's output buffer."""
        return self._product(_MATVEC, k, x, bias, out, scratch)

    def matmul_ok(self, k: int, in_features: int) -> bool:
        """Can `matmul` multiply by output `k` seen as rows of `in_features` elements?  What `matvec_ok` accepts, for
        bf16 and fp16 outputs only (an fp32 output decodes).  Never raises for an output that exists."""
        return self._ok(_MATMUL, k, in_features)

    def matmul_scratch_bytes(self, k: int, in_features: int, n_tokens: int = MATMUL_MAX_TOKENS) -> int:
        """Bytes of a matmul scratch for output `k`, rows of `in_features` elements and `n_tokens` rows of x."""
        return self._scratch_bytes(_MATMUL, k, in_features, n_tokens)

    def matmul(self, k: int, x: torch.Tensor, bias: torch.Tensor = None, out: torch.Tensor = None,
               scratch: torch.Tensor = None) -> torch.Tensor:
        """`matvec` for up to MATMUL_MAX_TOKENS rows of x, on tensor cores (zipnn_b200_decode_plan_matmul): the same
        arguments and rules, with `matmul_ok` and `matmul_scratch_bytes` in place of the matvec's.  bf16 and fp16
        weights only.  Products and sums are fp32 (the tensor cores' sums are not rounded to nearest at each step, so
        a result may differ from the matvec's in the last bits), each result is rounded once; two calls with the same
        inputs give the same bits.  x must be finite: an infinity may give NaN where the dense product gives one.
        Subnormal weights are kept, not flushed: on an H100 80GB HBM3, x = 1 times bf16 exponent-0 weights (fp32
        subnormal products) returns each weight bit for bit, as the matvec and decode + F.linear do."""
        return self._product(_MATMUL, k, x, bias, out, scratch)

    def matvec_fp8_ok(self, k: int, in_features: int) -> bool:
        """Can `matvec_fp8` multiply by output `k` seen as rows of `in_features` elements?  True for a float8_e4m3fn or
        float8_e5m2 output in one piece whose rows are a multiple of 16 elements and whose chunks all decode in the
        fused mode (what fp8 weights produce).  The first call for an output synchronises (it reads the chunk modes);
        never raises for an output that exists."""
        return self._ok(_MATVEC_FP8, k, in_features)

    def matvec_fp8_scratch_bytes(self, k: int, in_features: int, n_tokens: int = MATVEC_MAX_TOKENS) -> int:
        """Bytes of a matvec_fp8 scratch for output `k`, rows of `in_features` elements and `n_tokens` rows of x."""
        return self._scratch_bytes(_MATVEC_FP8, k, in_features, n_tokens)

    def matvec_fp8(self, k: int, x: torch.Tensor, scale: torch.Tensor, block: tuple = None, bias: torch.Tensor = None,
                   out: torch.Tensor = None, scratch: torch.Tensor = None) -> torch.Tensor:
        """`x @ (S * W).T (+ bias)` with W = output `k`, an fp8 tensor (float8_e4m3fn or float8_e5m2) seen as
        [out_features, in_features], in_features = x.shape[-1], and S its fp32 scale grid, computed from the coded
        streams: W is neither written nor read dense (zipnn_b200_decode_plan_matvec_fp8).  The weight the product uses
        is float(W[o][i]) * scale[o // bn][i // bk] -- the stored scale multiplies, as `weight_scale_inv` does in fp8
        checkpoints.  Two launches on the current CUDA stream, no host read: capturable in a CUDA graph.  Each group of
        16 consecutive weights of a row is multiplied with x in fp32 and scaled once; the sums and the single rounding
        are `matvec`'s, and two calls with the same inputs give the same bits.  An e4m3fn NaN or an e5m2 infinity or NaN
        gives what the dense product of the dequantized matrix gives: NaN or an infinity in that row.

        x:       CUDA bf16 or fp16 tensor [..., in_features] on the plan's device, at most MATVEC_MAX_TOKENS rows;
                 rows that are not 16-byte aligned are copied first.
        scale:   contiguous CUDA float32 tensor of ceil(out_features / bn) * ceil(in_features / bk) elements, row-major.
        block:   (bn, bk), bn >= 1, bk >= 16 and a multiple of 16: (out_features, in_features) is one scale for the
                 tensor, (1, in_features) one per row, (128, 128) DeepSeek's blocks.  None: a one-element scale, per
                 tensor.
        bias, out, scratch: as for `matvec`, in x's dtype; the scratch at least `matvec_fp8_scratch_bytes(k,
                 in_features, rows)` bytes.
        -> out.  ValueError for an output `matvec_fp8_ok` refuses.  Works without the plan's output buffer."""
        return self._product(_MATVEC_FP8, k, x, bias, out, scratch, scale=scale, block=block)

    def matmul_fp8_ok(self, k: int, in_features: int) -> bool:
        """Can `matmul_fp8` multiply by output `k` seen as rows of `in_features` elements?  What `matvec_fp8_ok`
        accepts.  Never raises for an output that exists."""
        return self._ok(_MATMUL_FP8, k, in_features)

    def matmul_fp8_scratch_bytes(self, k: int, in_features: int, n_tokens: int = MATMUL_MAX_TOKENS) -> int:
        """Bytes of a matmul_fp8 scratch for output `k`, rows of `in_features` elements and `n_tokens` rows of x."""
        return self._scratch_bytes(_MATMUL_FP8, k, in_features, n_tokens)

    def matmul_fp8(self, k: int, x: torch.Tensor, scale: torch.Tensor, block: tuple = None, bias: torch.Tensor = None,
                   out: torch.Tensor = None, scratch: torch.Tensor = None) -> torch.Tensor:
        """`matvec_fp8` for up to MATMUL_MAX_TOKENS rows of x, on tensor cores (zipnn_b200_decode_plan_matmul_fp8): the
        same arguments and rules, with `matmul_fp8_ok` and `matmul_fp8_scratch_bytes` in place of the matvec's.  Each
        weight is dequantized to x's dtype exactly as `dequant_fp8` writes it, D = dtype(float(W) * S), and the products
        and sums are the tensor cores' in fp32 (as `matmul`'s), each result rounded once: F.linear(x, D) up to the order
        of the fp32 sums, never writing D.  Two calls with the same inputs give the same bits.  x must be finite: an
        infinity may give NaN where the dense product gives one.  An e4m3fn NaN, an e5m2 infinity or NaN, or an fp16
        overflow in D gives NaN or an infinity in that row, as F.linear of D does."""
        return self._product(_MATMUL_FP8, k, x, bias, out, scratch, scale=scale, block=block)

    def _fp8_grid(self, name: str, in_features: int, scale, block, out_features: int, experts: int = 1) -> tuple:
        """-> (bn, bk) after checking `scale` against the grid the block implies (for method `name`); `experts` > 1: a
        weight [experts, out_features, in_features] with one grid per expert, back to back."""
        if not (isinstance(scale, torch.Tensor) and scale.is_cuda and scale.device == self.device and scale.dtype == torch.float32
                and scale.is_contiguous()):
            raise ValueError(f"{name}'s scale must be a contiguous CUDA float32 tensor on the plan's device")
        if block is None:
            if scale.numel() != experts:
                raise ValueError(f"{name} takes block=None for one scale per {'expert' if experts > 1 else 'tensor'} only, "
                                 f"not {scale.numel()} elements")
            return out_features, in_features
        bn, bk = (int(b) for b in block)
        if bn < 1 or bk < 16 or bk % 16:
            raise ValueError(f"{name}'s block (bn, bk) needs bn >= 1 and bk a multiple of 16 of at least 16, not {(bn, bk)}")
        grid = experts * -(-out_features // bn) * -(-in_features // bk)
        if scale.numel() != grid:
            lead = f"{experts}, " if experts > 1 else ""
            raise ValueError(f"{name}'s scale for block {(bn, bk)} of a [{lead}{out_features}, {in_features}] weight has {grid} "
                             f"elements, not {scale.numel()}")
        return bn, bk

    def dequant_fp8(self, k: int, in_features: int, scale: torch.Tensor, block: tuple = None, dtype: torch.dtype = torch.bfloat16,
                    out: torch.Tensor = None) -> torch.Tensor:
        """The dequantized weight S * W as a [out_features, in_features] tensor of `dtype` (bf16 or fp16), W = output `k`
        (an fp8 tensor that `matvec_fp8_ok(k, in_features)` accepts) and S its fp32 scale grid, written straight from the
        coded streams: the fp8 bytes are neither written nor read dense (zipnn_b200_decode_plan_dequant_fp8).  Bit for bit
        torch's `(W.to(torch.float32) * S_expanded).to(dtype)`: one fp32 product per element and one rounding to nearest
        even (fp16 overflow gives +-inf); NaN stays NaN, its payload may differ.  Two launches on the current CUDA stream,
        no scratch, no host read: capturable in a CUDA graph and replayable with a new scale.

        scale, block: as for `matvec_fp8`.
        out:     optional contiguous tensor of shape (out_features, in_features) and `dtype` on the plan's device, 16-byte
                 aligned; exactly its elements are written.
        -> out.  ValueError for an output `matvec_fp8_ok` refuses, and for a bad scale, block, dtype or out.  Works
        without the plan's output buffer.  A decode error surfaces through `check()`."""
        if dtype not in _MATMUL_DTYPES:
            raise ValueError(f"dequant_fp8 writes bf16 or fp16, not {dtype}")
        if not self._ok(_MATVEC_FP8, k, in_features):
            raise ValueError(f"dequant_fp8 cannot dequantize output {k} with in_features {in_features} (see matvec_fp8_ok)")
        wdt, total = self._product_item(k)
        shape = (total // in_features, in_features)
        bn, bk = self._fp8_grid("dequant_fp8", in_features, scale, block, shape[0])
        if out is None:
            out = torch.empty(shape, dtype=dtype, device=self.device)
        elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == dtype
                  and tuple(out.shape) == shape and out.is_contiguous() and out.data_ptr() % 16 == 0):
            raise ValueError(f"dequant_fp8's out must be a contiguous 16-byte aligned {dtype} CUDA tensor of shape {shape} on the plan's device")
        rc = _native.lib().zipnn_b200_decode_plan_dequant_fp8(self._ref, k, _FP8_FORMATS[wdt], _MATVEC_DTYPES[dtype], in_features,
                                                              scale.data_ptr(), bn, bk, out.data_ptr(),
                                                              torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return out

    def dequant_fp8_select_ok(self, in_features) -> bool:
        """Can `dequant_fp8_select` dequantize slices of this plan's outputs, output k seen as rows of `in_features[k]`
        elements?  True when `select_ok` is, the plan has at most 4 outputs, all of one fp8 dtype, `matvec_fp8_ok(k,
        in_features[k])` accepts each, and each slice [e] (along dim 0) is whole rows.  The first call for an output
        synchronises (it reads the chunk modes); never raises."""
        try:
            inf = [int(i) for i in in_features]
        except (TypeError, ValueError):
            return False
        if len(inf) != len(self._offs) or not 1 <= len(inf) <= _SELECT_FP8_MAX_ITEMS or not self.select_ok():
            return False
        if len({dt for _, _, dt, _ in self._offs}) != 1:
            return False
        for k, i in enumerate(inf):
            _, _, dt, sh = self._offs[k]
            if not self._ok(_MATVEC_FP8, k, i) or (math.prod(sh) // sh[0]) % i:
                return False
        return True

    def dequant_fp8_select(self, ids: torch.Tensor, in_features, scales, blocks, dtype: torch.dtype = torch.bfloat16,
                           outs=None, scratch: torch.Tensor = None) -> list:
        """`dequant_fp8` of the slices [e] (along dim 0) that `ids` select, written straight from the coded streams of
        the chunks that meet them (zipnn_b200_decode_plan_dequant_fp8_select): the routed experts of an fp8
        mixture-of-experts layer, output k = an expert weight [E, out_k, in_k] with a scale grid per expert.  Every
        element of a selected slice is bit for bit torch's `(W[e].to(torch.float32) * S[e]_expanded).to(dtype)`.  Each
        chunk that meets a selected slice is written whole (a chunk that straddles slices writes its neighbours'
        elements too, correctly); no other element of the outputs is written, so the slices that were not selected
        hold whatever they held.  Three launches on the current CUDA stream, a fixed number, the ids never read on the
        host: capturable in a CUDA graph and replayable with new ids and new scales.

        ids:     CUDA int32 or int64 tensor of any shape on the plan's device; duplicates allowed; empty: nothing runs.
        in_features: per output, in_k (its rows' elements).
        scales:  per output, the contiguous CUDA float32 grid [E, ceil(out_k / bn), ceil(in_k / bk)] (any shape of that
                 many elements), as transformers' `FP8Experts` holds it in `*_scale_inv`.
        blocks:  per output, (bn, bk) as for `matvec_fp8`, or None: one scale per expert ([E, 1, 1]).
        dtype:   bf16 or fp16.
        outs:    optional list of contiguous 16-byte aligned tensors [E, out_k, in_k] of `dtype` on the plan's device.
        scratch: as for `run_select` (at least `select_scratch_bytes()` bytes, not the plan's own scratch); default: a
                 buffer kept by the plan.
        -> the list of outputs.  An id outside [0, E) selects nothing and makes `check()` raise IndexError (sticky).
        ValueError for a plan `dequant_fp8_select_ok` refuses, and for bad ids, scales, blocks, dtype or outs.  Works
        without the plan's output buffer."""
        name = "dequant_fp8_select"
        self._check_ids(name, ids)
        if dtype not in _MATMUL_DTYPES:
            raise ValueError(f"{name} writes bf16 or fp16, not {dtype}")
        inf = list(in_features) if isinstance(in_features, (list, tuple)) else None
        if inf is None or not self.dequant_fp8_select_ok(inf):
            raise ValueError(f"{name} cannot dequantize this plan's outputs with in_features {in_features} (see {name}_ok)")
        inf = [int(i) for i in inf]
        n_out = len(self._offs)
        scales, blocks = list(scales), list(blocks)
        if len(scales) != n_out or len(blocks) != n_out:
            raise ValueError(f"{name} takes one scale and one block per output ({n_out})")
        if outs is not None:
            outs = list(outs)
            if len(outs) != n_out:
                raise ValueError(f"{name} takes one out per output ({n_out})")
        E = self._offs[0][3][0]
        arr = (_native.Fp8SelectItem * n_out)()
        result = []
        for k, (it, i) in enumerate(zip(arr, inf)):
            wdt, total = self._product_item(k)
            shape = (E, total // (E * i), i)
            bn, bk = self._fp8_grid(name, i, scales[k], blocks[k], shape[1], experts=E)
            out = None if outs is None else outs[k]
            if out is None:
                out = torch.empty(shape, dtype=dtype, device=self.device)
            elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == dtype
                      and tuple(out.shape) == shape and out.is_contiguous() and out.data_ptr() % 16 == 0):
                raise ValueError(f"{name}'s out {k} must be a contiguous 16-byte aligned {dtype} CUDA tensor of shape {shape} "
                                 "on the plan's device")
            it.in_features, it.d_scale, it.block_rows, it.block_cols, it.d_out = i, scales[k].data_ptr(), bn, bk, out.data_ptr()
            result.append(out)
        ids_c = ids.contiguous()
        n = ids_c.numel()
        if n == 0:
            return result
        scratch = self._scratch_for(name, scratch, self.select_scratch_bytes)
        rc = _native.lib().zipnn_b200_decode_plan_dequant_fp8_select(self._ref, E, ids_c.data_ptr(), n, ids_c.element_size(),
                                                                     _FP8_FORMATS[self._offs[0][2]], _MATVEC_DTYPES[dtype], n_out, arr,
                                                                     scratch.data_ptr(), scratch.numel(),
                                                                     torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return result

    def experts_matvec_fp8_ok(self, k: int, in_features: int) -> bool:
        """Can `experts_matvec_fp8` multiply by the experts of output `k`, seen as [E, out, in_features] (E = shape[0])?
        True when `select_ok` is, `matvec_fp8_ok(k, in_features)` accepts the output and each expert is whole rows.
        The first call for an output synchronises (it reads the chunk modes); never raises."""
        try:
            k, i = int(k), int(in_features)
        except (TypeError, ValueError):
            return False
        if not 0 <= k < len(self._offs) or i <= 0 or not self.select_ok():
            return False
        _, _, dt, sh = self._offs[k]
        return dt in _FP8_FORMATS and self._ok(_MATVEC_FP8, k, i) and (math.prod(sh) // sh[0]) % i == 0

    def experts_matvec_fp8_scratch_bytes(self, k: int, in_features: int, top_k: int, n_tokens: int = EXPERTS_MATVEC_MAX_TOKENS) -> int:
        """Bytes of an `experts_matvec_fp8` scratch for output `k`, rows of `in_features` elements, `top_k` experts per
        token and `n_tokens` tokens: the select scratch, the pair tables and the matvec's partial sums."""
        out = C.c_size_t(0)
        with torch.cuda.device(self.device):
            rc = _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size(self._ref, int(k), self._offs[0][3][0], int(in_features),
                                                                                       int(n_tokens) * int(top_k), int(top_k), C.byref(out))
        _native.check(rc)
        return out.value

    def experts_matvec_fp8(self, k: int, ids: torch.Tensor, x: torch.Tensor, scale: torch.Tensor, block: tuple = None,
                           out: torch.Tensor = None, scratch: torch.Tensor = None) -> torch.Tensor:
        """The routed experts of output `k` times x, from the coded streams of the chunks they meet
        (zipnn_b200_decode_plan_experts_matvec_fp8): output k is an fp8 expert weight [E, out, in] with a scale grid
        per expert, and for every pair (t, j) of `ids`, y[t, j] = x_tj @ (S[e] * W[e]).T with e = ids[t, j].  No weight
        is written.  Each result is bit for bit `matvec_fp8` of the output seen as [E * out, in] with x = x_tj, rows
        e * out ... (e + 1) * out - 1.  Five launches on the current CUDA stream, a fixed number, the ids never read on
        the host: capturable in a CUDA graph and replayable with new ids, x and scales.

        ids:     CUDA int32 or int64 tensor [T, top_k] on the plan's device, T <= EXPERTS_MATVEC_MAX_TOKENS.  Empty: nothing
                 runs.
        x:       CUDA bf16 or fp16 tensor [T, in] (pair (t, j) multiplies x[t]: the first projection) or [T, top_k, in]
                 (it multiplies x[t, j]: the down projection); rows that are not 16-byte aligned are copied first.
        scale, block: as for `dequant_fp8_select` (a grid per expert, [E, ceil(out / bn), ceil(in / bk)], or block=None
                 for one scale per expert).
        out:     optional [T, top_k, out] tensor of x's dtype with contiguous, equally spaced rows.
        scratch: optional 256-byte aligned CUDA uint8 buffer of at least `experts_matvec_fp8_scratch_bytes(k, in,
                 top_k, T)` bytes, not the plan's own scratch; it holds nothing between calls.  Default: a buffer kept
                 by the plan.
        -> out.  An id outside [0, E), or an expert routed more than once by one token, makes `check()` raise
        IndexError (sticky).  ValueError for an output `experts_matvec_fp8_ok` refuses, and for bad ids, x, scale, block,
        out or scratch.  Works without the plan's output buffer."""
        name = "experts_matvec_fp8"
        self._check_ids(name, ids)
        if ids.dim() != 2:
            raise ValueError(f"{name} takes ids [T, top_k], not {tuple(ids.shape)}")
        T, top_k = ids.shape
        if T > EXPERTS_MATVEC_MAX_TOKENS:
            raise ValueError(f"{name} takes at most {EXPERTS_MATVEC_MAX_TOKENS} tokens, not {T}")
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.device == self.device and x.dtype in _MATMUL_DTYPES
                and tuple(x.shape[:-1]) in ((T,), (T, top_k))):
            raise ValueError(f"{name} takes a CUDA bf16 or fp16 x [T, in] or [T, top_k, in] on the plan's device, T, top_k = {T}, {top_k}")
        per_pair = x.dim() == 3
        in_features = x.shape[-1]
        if not self.experts_matvec_fp8_ok(k, in_features):
            raise ValueError(f"{name} cannot multiply by output {k} with in_features {in_features} (see {name}_ok)")
        wdt, total = self._product_item(k)
        E = self._offs[0][3][0]
        rows = total // (E * in_features)
        bn, bk = self._fp8_grid(name, in_features, scale, block, rows, experts=E)
        shape = (T, top_k, rows)
        if out is None:
            out = torch.empty(shape, dtype=x.dtype, device=self.device)
        elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == x.dtype
                  and tuple(out.shape) == shape):
            raise ValueError(f"{name}'s out must be a {x.dtype} CUDA tensor of shape {shape} on the plan's device")
        n = T * top_k
        if n == 0:
            return out
        try:
            y2 = out.view(n, rows)
        except RuntimeError:
            y2 = None
        if y2 is None or y2.stride(1) != 1:
            raise ValueError(f"{name}'s out must have contiguous rows, equally spaced")
        xr = n if per_pair else T
        x2 = x.reshape(xr, in_features)
        if x2.stride(1) != 1 or x2.data_ptr() % 16 or (xr > 1 and (x2.stride(0) * x.element_size()) % 16):
            x2 = x2.contiguous()
            if x2.data_ptr() % 16:
                x2 = x2.clone()
        ids_c = ids.contiguous()
        scratch = self._scratch_for(name, scratch, lambda: self.experts_matvec_fp8_scratch_bytes(k, in_features, top_k, T))
        rc = _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8(
            self._ref, k, E, ids_c.data_ptr(), n, ids_c.element_size(), top_k, _FP8_FORMATS[wdt], _MATVEC_DTYPES[x.dtype],
            in_features, x2.data_ptr(), x2.stride(0), int(per_pair), scale.data_ptr(), bn, bk, y2.data_ptr(), y2.stride(0),
            scratch.data_ptr(), scratch.numel(), torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return out

    def _product(self, kind: _Product, k: int, x, bias, out, scratch, scale=None, block=None) -> torch.Tensor:
        """matvec, matmul, matvec_fp8 and matmul_fp8: the checks and the call."""
        name = kind.name
        wdt, total = self._product_item(k)
        dt = x.dtype if kind.x_dtypes and isinstance(x, torch.Tensor) and x.dtype in kind.x_dtypes else wdt
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.device == self.device and x.dtype == dt and x.dim() >= 1):
            raise ValueError(f"{name} takes a CUDA {'bf16 or fp16' if kind.x_dtypes else dt} tensor [..., in_features] on the plan's device")
        in_features = x.shape[-1]
        lead = tuple(x.shape[:-1])
        n = math.prod(lead)
        if n > kind.limit:
            raise ValueError(f"{name} takes at most {kind.limit} rows of x, not {n}")
        if not self._ok(kind, k, in_features):
            raise ValueError(f"{name} cannot multiply by output {k} with in_features {in_features} (see {name}_ok)")
        out_features = total // in_features
        if kind.scaled:
            bn, bk = self._fp8_grid(name, in_features, scale, block, out_features)
        es = x.element_size()
        x2 = x.reshape(max(n, 1), in_features) if n else x.reshape(0, in_features)
        if n and (x2.stride(1) != 1 or x2.data_ptr() % 16 or (n > 1 and (x2.stride(0) * es) % 16)):
            x2 = x2.contiguous()
            if x2.data_ptr() % 16:
                x2 = x2.clone()
        if bias is not None and not (isinstance(bias, torch.Tensor) and bias.device == self.device and bias.dtype == dt
                                     and tuple(bias.shape) == (out_features,) and bias.is_contiguous()):
            raise ValueError(f"{name}'s bias must be a contiguous {dt} CUDA tensor of shape ({out_features},) on the plan's device")
        shape = lead + (out_features,)
        if out is None:
            out = torch.empty(shape, dtype=dt, device=self.device)
        elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.device == self.device and out.dtype == dt
                  and tuple(out.shape) == shape):
            raise ValueError(f"{name}'s out must be a {dt} CUDA tensor of shape {shape} on the plan's device")
        if n == 0:
            return out
        try:
            y2 = out.view(n, out_features)
        except RuntimeError:
            y2 = None
        if y2 is None or y2.stride(1) != 1:
            raise ValueError(f"{name}'s out must have contiguous rows, equally spaced")
        scratch = self._scratch_for(name, scratch, lambda: self._scratch_bytes(kind, k, in_features, kind.limit))
        if kind.scaled:
            dtypes, grid = (kind.weights[wdt], _MATVEC_DTYPES[dt]), (scale.data_ptr(), bn, bk)
        else:
            dtypes, grid = (kind.weights[dt],), ()
        rc = kind.native()(self._ref, k, *dtypes, in_features, x2.data_ptr(), x2.stride(0), n, *grid,
                           bias.data_ptr() if bias is not None else None, y2.data_ptr(), y2.stride(0), scratch.data_ptr(),
                           scratch.numel(), torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _native.check(rc)
        return out

    def check(self) -> None:
        """Synchronise the current stream and raise if a run so far found an error."""
        with torch.cuda.device(self.device):
            _raise_status(_native.lib().zipnn_b200_decode_plan_status(C.byref(self._plan), _cuda_stream_handle()))
