"""The host-memory paths against the oracle at every slab and frame boundary (models: test_host_pipelines_host.py).

  a. zipnn_b200_decompress_host's slab decoder, on plane-built streams of every layout, at slab knobs below one
     chunk, of one chunk, 3*chunk - 1 and 3*chunk, into pinned and pageable buffers, and on corrupt streams;
  b. zipnn_b200_compress_host's slab encoder and its early-copy bet: bets kept, lost in slab 0, in a middle slab and
     in the last one, out_cap at the stream length (lost-bet copies skipped), one byte short and below the tables;
  c. error exits: whatever a failing call returns, nothing it queued still writes to the caller's buffer;
  d. DecodePipe's pinned ring shrunk to a few KiB: bodies span many slabs, the ring wraps, the reader threads split
     every slab, the 1024-entry error-flag buffer rolls over, and slabs cached at one size are not reused at another;
  e. streaming frames: every frame equals the oracle's stream of its byte range, through the at-once paths and the
     per-frame loops, with delta, and on a stream whose last frame runs past the end.
Every output lies between canaries; every stream is compared byte for byte with the oracle's.
"""
import ctypes as C
import functools
import math
import os

import numpy as np
import pytest
import torch

import plane_inputs as P
import test_host_pipelines_host as HM
from oracle import oracle as O
from zipnn_b200 import DecodePipe, ZipNN, _native
from zipnn_b200 import zipnn as Z
from zipnn_b200.util_torch import dtype_code, zipnn_pack_shape

pytestmark = pytest.mark.gpu

CANARY = 0xA5
PAD = 256
BM = HM.BYTES_MODE
DEFAULT_RING = DecodePipe.SLAB_BYTES
TORCH_DTYPE = {"bf16": torch.bfloat16, "bf16_256k": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32,
               "fp8": torch.float8_e4m3fn}

_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.argtypes = [C.c_void_p]


@pytest.fixture
def knob(monkeypatch):
    """set(v): ZIPNN_B200_HOST_SLAB_BYTES = v (None: unset); host_knobs() reads it on every call."""
    def set_(v):
        if v is None:
            monkeypatch.delenv(HM.KNOB, raising=False)
        else:
            monkeypatch.setenv(HM.KNOB, str(v))
    set_(None)
    return set_


class HostBuf:
    """nbytes of pinned (torch pin_memory) or pageable (malloc) host memory, filled with the canary."""

    def __init__(self, nbytes: int, kind: str):
        self.kind, self.n = kind, nbytes
        if kind == "pinned":
            self.t = torch.full((nbytes,), CANARY, dtype=torch.uint8, pin_memory=True)
            self.ptr = self.t.data_ptr()
            self.a = self.t.numpy()
        else:
            self.ptr = _libc.malloc(nbytes)
            self.a = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))
            self.a[:] = CANARY

    def free(self):
        if self.kind == "malloc" and self.ptr:
            self.a = None
            _libc.free(self.ptr)
            self.ptr = 0


@pytest.fixture
def host_buf():
    bufs = []

    def make(nbytes, kind):
        bufs.append(HostBuf(nbytes, kind))
        return bufs[-1]
    yield make
    for b in bufs:
        b.free()


def decode_host(body, G, bits, chunk, orig, out: HostBuf) -> int:
    body = np.ascontiguousarray(body)
    return _native.lib().zipnn_b200_decompress_host(body.ctypes.data, body.size, G, bits, BM[G], chunk, orig, out.ptr)


def encode_host(data, hdr, G, bits, chunk, out: HostBuf, out_cap):
    """-> (rc, out_len)."""
    data = np.ascontiguousarray(data)
    hbuf = (C.c_char * len(hdr)).from_buffer_copy(bytes(hdr))
    out_len = C.c_size_t(0)
    rc = _native.lib().zipnn_b200_compress_host(data.ctypes.data, data.size, hbuf, len(hdr), G, bits, BM[G], chunk, 0.95,
                                                out.ptr, out_cap, C.byref(out_len))
    return rc, out_len.value


def torch_stream(hdr: bytes, body: np.ndarray) -> bytes:
    """A torch-format stream from a ZipNN.plan() header and a body the oracle wrote after another header."""
    h = bytearray(hdr)
    h[24:32] = int(len(h) + body.size).to_bytes(8, "little")
    return bytes(h) + body.tobytes()


# ================================================================== a. the slab decoder
@functools.lru_cache(maxsize=None)
def decode_layout(name):
    G, bits, chunk, n = HM.DECODE_LAYOUTS[name]
    data = HM.planned_bytes(HM.DECODE_PATTERN[G], G, bits, chunk, n, seed=len(name) * 7 + G)
    want = O.zipnn_compress(HM.header32(n), data, G, bits, BM[G], chunk, threads=8)
    return data, want


@pytest.mark.parametrize("k", range(4))
@pytest.mark.parametrize("name", list(HM.DECODE_LAYOUTS))
def test_slab_decoder(name, k, knob, host_buf):
    G, bits, chunk, n = HM.DECODE_LAYOUTS[name]
    data, want = decode_layout(name)
    assert HM.realised(HM.DECODE_PATTERN[G], want, 32, G, chunk, n), "the planes did not code as built"
    slab = HM.decode_knobs(chunk)[k]
    plan = HM.slab_plan(n, chunk, slab)
    assert plan.piped and plan.per == [1, 1, 2, 3][k] and plan.nslabs > 1
    knob(slab)
    out = host_buf(n + PAD, "pinned" if k % 2 else "malloc")
    assert decode_host(want[32:], G, bits, chunk, n, out) == 0
    assert np.array_equal(out.a[:n], data), f"{name}: slab decode != input"
    assert np.all(out.a[n:] == CANARY), "wrote past orig"
    # the same stream in torch format through ZipNN.decompress(bytes)
    t = torch.from_numpy(data.copy()).view(TORCH_DTYPE[name])
    hdr = ZipNN(input_format="torch", compression_chunk=chunk if G > 1 else 262144).plan(t)["header"]
    back = ZipNN(input_format="torch").decompress(torch_stream(hdr, want[32:]))
    assert back.dtype == t.dtype and np.array_equal(back.view(torch.uint8).numpy(), data)


def test_slab_decoder_many_general_chunks_per_slab(knob, host_buf):
    """fp32 values upcast from a narrower type: the two low byte groups are zero (RLE), the two high ones are coded,
    so every chunk takes a pool slot; 100 of them per slab is more than the 64 slots of the normal workspace."""
    chunk, per = 4096, 100
    g = torch.Generator().manual_seed(17)
    t = (torch.randn(250 * chunk // 4, generator=g) * 0.02).to(torch.float8_e4m3fn).to(torch.float32)
    data = t.view(torch.uint8).numpy()
    n = data.size
    hdr = ZipNN(input_format="torch", compression_chunk=chunk).plan(t)["header"]
    want = O.zipnn_compress(hdr, data, 4, 1, 220, chunk, threads=8)
    body = want[len(hdr):]
    pr = P.predict(body, 4, 1, chunk, n)
    plan = HM.slab_plan(n, chunk, per * chunk)
    assert plan.piped and plan.nslabs == 3
    for c0, c1 in plan.ranges[:-1]:
        assert sum(m == "general" for m in pr["mode"][c0:c1]) > 64
    knob(per * chunk)
    out = host_buf(n + PAD, "malloc")
    assert decode_host(body, 4, 1, chunk, n, out) == 0
    assert np.array_equal(out.a[:n], data) and np.all(out.a[n:] == CANARY)
    back = ZipNN(input_format="torch").decompress(want.tobytes())
    assert torch.equal(back.view(torch.int32), t.view(torch.int32))


def test_slab_decoder_corrupt_streams(knob, host_buf):
    """A bad type byte in the last slab (found on the device), a size row that decreases across the edge into the
    last slab (found by the host check, at the slab the model names) and a truncated body: each is E_CORRUPT, and a
    good decode through the same process cache right after is exact."""
    name = "bf16"
    G, bits, chunk, n = HM.DECODE_LAYOUTS[name]
    data, want = decode_layout(name)
    slab = 3 * chunk - 1
    plan = HM.slab_plan(n, chunk, slab)
    K, per = plan.K, plan.per
    c_last = plan.ranges[-1][0]
    knob(slab)
    body = want[32:].copy()
    bad_type = body.copy()
    bad_type[1 * K + K - 1] = 9
    bad_row = body.copy()
    cum = bad_row[G * K: 9 * G * K].view("<u8").reshape(G, K)
    cum[G - 1, K - 1] = cum[G - 1, c_last - 1] - 1
    cases = [(bad_type, ("ok", None)), (bad_row, ("row", plan.nslabs - 1)), (body[:-7], ("room", None))]
    for bad, where in cases:
        assert HM.decode_host_check(bad, G, chunk, n, per) == where
        out = host_buf(n + PAD, "pinned")
        assert decode_host(bad, G, bits, chunk, n, out) == HM.E_CORRUPT, where
        assert np.all(out.a[n:] == CANARY)
        good = host_buf(n + PAD, "malloc")
        assert decode_host(body, G, bits, chunk, n, good) == 0
        assert np.array_equal(good.a[:n], data) and np.all(good.a[n:] == CANARY)


# ================================================================== b. the slab encoder and its early bet
ENC_CHUNK, ENC_PER = 4096, 2
FP32 = ("raw", "raw", "raw", "huf")      # float32 weights: three raw mantissa planes, a coded exponent plane
BF16 = ("raw", "huf")


def _enc_pattern(default, K, at):
    """K chunks of `default`, with chunk c replaced by at[c]."""
    return [at.get(c, default) for c in range(K)]


# name: (G, bits, chunk count, pattern overrides, expected {taken, lost})
ENC_CASES = {
    "fp32_kept": (4, 1, 7, FP32, {}, dict(taken={1: True, 2: True, 3: True}, lost={1: None, 2: None, 3: None})),
    "fp32_g1_slab0": (4, 1, 7, FP32, {0: ("raw", "huf", "raw", "huf")},
                      dict(taken={1: True, 2: False, 3: False}, lost={1: None, 2: None, 3: None})),
    "fp32_g1_middle": (4, 1, 7, FP32, {3: ("raw", "huf", "raw", "huf")},
                       dict(taken={1: True, 2: True, 3: True}, lost={1: None, 2: 1, 3: 1})),
    "fp32_g1_last": (4, 1, 7, FP32, {6: ("raw", "rle", "raw", "huf")},
                     dict(taken={1: True, 2: True, 3: True}, lost={1: None, 2: 3, 3: 3}, skip=True)),
    "fp32_g2_only": (4, 1, 8, FP32, {4: ("raw", "raw", "huf", "huf")},
                     dict(taken={1: True, 2: True, 3: True}, lost={1: None, 2: None, 3: 2})),
    "bf16_g0_last": (2, 1, 7, BF16, {6: ("huf", "huf")}, dict(taken={1: True}, lost={1: 3}, skip=True)),
    "fp8": (1, 0, 7, ("huf",), {2: ("raw",), 5: ("rle",)}, dict(taken={}, lost={})),
}
# header variants: 32 bytes, and torch-format headers with 1-D and 2-D shapes
HEADERS = {"h32": (), "h36": (7143,), "h40": (3, 70000), "h41": (300, 70000)}


def enc_input(name):
    G, bits, K, default, at, _ = ENC_CASES[name]
    n = K * ENC_CHUNK - 100 if K % 2 else K * ENC_CHUNK     # a ragged last chunk in the odd-sized cases
    pattern = _enc_pattern(default, K, at)
    data = HM.planned_bytes(pattern, G, bits, ENC_CHUNK, n, seed=K * 31 + G)
    return data, pattern


def enc_header(hname, n):
    h = bytearray(HM.header32(n))
    shape = HEADERS[hname]
    if not shape:
        return bytes(h)
    h[8] = 2                                                # torch format (the library copies the header as it is)
    return bytes(h) + zipnn_pack_shape(shape)


@pytest.mark.parametrize("hname", list(HEADERS))
@pytest.mark.parametrize("name", list(ENC_CASES))
def test_slab_encoder_bets(name, hname, knob, host_buf):
    G, bits, K, _, _, expect = ENC_CASES[name]
    data, pattern = enc_input(name)
    n = data.size
    hdr = enc_header(hname, n)
    H = len(hdr)
    assert H == {"h32": 32, "h36": 36, "h40": 40, "h41": 41}[hname]
    want = O.zipnn_compress(hdr, data, G, bits, BM[G], ENC_CHUNK)
    assert HM.realised(pattern, want, H, G, ENC_CHUNK, n), "the planes did not code as built"
    plan = HM.slab_plan(n, ENC_CHUNK, ENC_PER * ENC_CHUNK, "encode")
    assert plan.piped and plan.per == ENC_PER
    knob(ENC_PER * ENC_CHUNK)
    L = want.size
    bound = _native.compress_bound(n, G, ENC_CHUNK, H)
    m = HM.bet_model(want, H, G, ENC_CHUNK, n, ENC_PER, bound)
    assert m["status"] == HM.OK and m["out_len"] == L and not m["skipped"]
    assert m["taken"] == expect["taken"] and m["lost"] == expect["lost"], (m["taken"], m["lost"])
    if expect.get("skip"):
        # a bet lost late: at out_cap == L the early copies of the slabs before the loss would pass out_cap
        assert HM.bet_model(want, H, G, ENC_CHUNK, n, ENC_PER, L)["skipped"]
    K_ = plan.K
    payload0 = H + 9 * G * K_
    _, cum, _, _ = HM.tables(want, H, G, K_)
    g0_slab0 = int(cum[0, ENC_PER - 1])
    caps = {"bound": bound, "exact": L, "short": L - 1, "payload0": payload0 - 1, "g0_mid": payload0 + g0_slab0 + 1}
    for i, (cname, cap) in enumerate(caps.items()):
        mc = HM.bet_model(want, H, G, ENC_CHUNK, n, ENC_PER, cap)
        if cname == "short":
            assert mc["site"] == ("final" if G > 1 else ("g0", plan.nslabs - 1))
        if cname == "payload0":
            assert mc["site"] == "payload0"
        if cname == "g0_mid":
            assert mc["site"] == ("g0", 1)
        out = host_buf(max(cap, L) + PAD, "pinned" if (i + len(hname)) % 2 else "malloc")
        rc, out_len = encode_host(data, hdr, G, bits, ENC_CHUNK, out, cap)
        torch.cuda.synchronize()
        assert rc == mc["status"], (cname, rc, mc["site"])
        assert np.all(out.a[cap:] == CANARY), f"{cname}: wrote past out_cap"
        if rc == HM.OK:
            assert out_len == L and np.array_equal(out.a[:L], want), f"{name}/{hname}/{cname}: stream != oracle"


def test_zipnn_compress_host_out(knob):
    """ZipNN.compress(host tensor, out=): the stream at out_cap == its length equals the oracle's; one byte less
    is a ValueError."""
    data, _ = enc_input("fp32_g1_middle")
    t = torch.from_numpy(data.copy()).view(torch.float32).reshape(3, -1)
    z = ZipNN(input_format="torch", compression_chunk=ENC_CHUNK)
    hdr = z.plan(t)["header"]
    want = O.zipnn_compress(hdr, data, 4, 1, 220, ENC_CHUNK)
    knob(ENC_PER * ENC_CHUNK)
    out = torch.full((want.size + PAD,), CANARY, dtype=torch.uint8, pin_memory=True)
    got = z.compress(t.pin_memory(), out=out[: want.size])
    assert bytes(got) == want.tobytes() and torch.all(out[want.size:] == CANARY)
    with pytest.raises(ValueError):
        z.compress(t, out=torch.empty(want.size - 1, dtype=torch.uint8, pin_memory=True))


# ================================================================== c. error exits leave nothing in flight
BIG_SLAB = 24 << 20


def _settled(buf: torch.Tensor, last: slice):
    """Snapshot the range the last queued copy writes, then everything, then let the device finish: nothing may
    change after the call returned."""
    first = buf[last].clone()
    snap = buf.clone()
    torch.cuda.synchronize()
    assert torch.equal(buf[last], first) and torch.equal(buf, snap), "the call returned with copies into h_out in flight"


def test_error_exits_leave_nothing_in_flight(knob):
    L = _native.lib()
    chunk, G = 262144, 2
    n = 3 * BIG_SLAB
    g = torch.Generator().manual_seed(41)
    t = (torch.randn(n // 2, generator=g) * 0.02).to(torch.bfloat16)
    data = t.view(torch.uint8).numpy()
    plan = HM.slab_plan(n, chunk, BIG_SLAB)
    assert plan.piped and plan.nslabs == 3
    hdr = HM.header32(n)
    stream = ZipNN(input_format="byte").compress(torch.from_numpy(data).cuda()).cpu().numpy()   # (byte-format header)
    K = plan.K
    H = 32
    knob(BIG_SLAB)
    # decompress: a size row that decreases into the last slab, found by the host check after slabs 0 and 1 are queued
    body = stream[H:].copy()
    cum = body[G * K: 9 * G * K].view("<u8").reshape(G, K)
    c_last = plan.ranges[-1][0]
    cum[G - 1, K - 1] = cum[G - 1, c_last - 1] - 1
    assert HM.decode_host_check(body, G, chunk, n, plan.per) == ("row", 2)
    h_out = torch.full((n,), CANARY, dtype=torch.uint8, pin_memory=True)
    rc = L.zipnn_b200_decompress_host(body.ctypes.data, body.size, G, 1, 10, chunk, n, h_out.data_ptr())
    last = slice(plan.ranges[1][1] * chunk - 4096, plan.ranges[1][1] * chunk)     # the end of slab 1's output
    _settled(h_out, last)
    assert rc == HM.E_CORRUPT
    # compress with out_cap one byte short: fails at the final check right after the last slab's group-0 copy
    Lw = stream.size
    m = HM.bet_model(stream, H, G, chunk, n, plan.per, Lw - 1)
    assert m["status"] == HM.E_CAPACITY and m["site"] == "final"
    g0 = [c for c in m["copies"] if c[0] == 0][-1]
    h_out = torch.full((Lw,), CANARY, dtype=torch.uint8, pin_memory=True)
    src = torch.from_numpy(data.copy()).pin_memory()
    hbuf = (C.c_char * 32).from_buffer_copy(hdr)
    out_len = C.c_size_t(0)
    rc = L.zipnn_b200_compress_host(src.data_ptr(), n, hbuf, 32, G, 1, 10, chunk, 0.95, h_out.data_ptr(), Lw - 1, C.byref(out_len))
    _settled(h_out, slice(g0[2] + g0[3] - 4096, g0[2] + g0[3]))
    assert rc == HM.E_CAPACITY
    # the same through ZipNN: a too-small out= (ValueError) and a corrupt stream decoded into out= (RuntimeError)
    z = ZipNN(input_format="torch")
    ts = bytes(z.compress(t))
    Ht = len(ts) - (stream.size - H)
    mt = HM.bet_model(np.frombuffer(ts, np.uint8), Ht, G, chunk, n, plan.per, len(ts) - 1)
    assert mt["site"] == "final"
    g0 = [c for c in mt["copies"] if c[0] == 0][-1]
    small = torch.full((len(ts) - 1,), CANARY, dtype=torch.uint8, pin_memory=True)
    with pytest.raises(ValueError):
        z.compress(t, out=small)
    _settled(small, slice(g0[2] + g0[3] - 4096, g0[2] + g0[3]))
    bad = bytearray(ts)
    tcum = np.frombuffer(bad, dtype=np.uint8)[Ht + G * K: Ht + 9 * G * K].view("<u8").reshape(G, K)
    tcum[G - 1, K - 1] = tcum[G - 1, c_last - 1] - 1
    out = torch.full((n,), CANARY, dtype=torch.uint8, pin_memory=True)
    with pytest.raises(RuntimeError, match="corrupt"):
        ZipNN(input_format="torch").decompress(bytes(bad), out=out)
    _settled(out, last)


# ================================================================== d. DecodePipe's pinned ring
SMALL_RING, SMALL_PIECE = 65536 + 48, 4096 + 16


@pytest.fixture
def small_ring(monkeypatch):
    DecodePipe._slab_cache.clear()
    monkeypatch.setattr(DecodePipe, "SLAB_BYTES", SMALL_RING)
    monkeypatch.setattr(DecodePipe, "COPY_PIECE", SMALL_PIECE)
    yield
    DecodePipe._slab_cache.clear()


def _tensors():
    g = torch.Generator().manual_seed(23)
    return [
        (torch.randn(600_000, generator=g) * 0.02).to(torch.bfloat16),
        (torch.randn(200_001, generator=g)).reshape(-1),
        (torch.randn(300_007, generator=g) * 0.1).to(torch.float8_e4m3fn),
        (torch.randn(1000, generator=g)).to(torch.float16).reshape(10, 100),
    ]


def _streams(ts):
    return [ZipNN(input_format="torch").compress(t.cuda()).cpu().numpy() for t in ts]


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.cpu().view(torch.uint8), b.cpu().view(torch.uint8))


def test_pipe_ring_wraps(small_ring, tmp_path):
    ts = _tensors()
    ss = _streams(ts)
    assert max(s.size for s in ss) > 8 * SMALL_RING            # a body wraps the 4-slab ring more than twice
    pipe = DecodePipe("cuda")
    got = [pipe.submit(ss[0].tobytes()), pipe.submit(ss[1]), pipe.submit(torch.from_numpy(ss[2].copy())),
           pipe.submit(ss[3].tobytes())]
    path = str(tmp_path / "streams.bin")
    empty = ZipNN(input_format="torch").compress(torch.empty(0, dtype=torch.bfloat16).cuda()).cpu().numpy()
    other = np.frombuffer(bytes(ZipNN(input_format="byte").compress(ts[0].view(torch.uint8).numpy().tobytes())), np.uint8)
    blobs = ss + [empty, other]
    offs, at = [], 13                                              # an odd start: every body sits off alignment
    with open(path, "wb") as f:
        f.write(b"\0" * at)
        for b in blobs:
            offs.append(at)
            f.write(b.tobytes())
            at += b.size
    fd = os.open(path, os.O_RDONLY)
    try:
        got += [pipe.submit_file(fd, offs[i], ss[i].size) for i in range(len(ss))]
        batch = pipe.submit_file_batch(fd, [(offs[i], blobs[i].size) for i in range(len(blobs))])
        slabs_used = pipe._slab
        pipe.finish()
    finally:
        os.close(fd)
    pipe.release()
    assert slabs_used > 3 * 4
    for i, t in enumerate(ts + ts):
        assert _same(got[i], t), i
    for i, t in enumerate(ts):
        assert _same(batch[i], t), i
    assert batch[len(ts)].numel() == 0 and batch[len(ts)].dtype == torch.bfloat16
    assert batch[len(ts) + 1] is None
    assert all(s.numel() == SMALL_RING for s in DecodePipe._slab_cache)


def test_pipe_load_module(small_ring, tmp_path, monkeypatch):
    from test_resident_gpu import make_model
    from test_resident_load_gpu import build, dealiased
    from zipnn_b200 import decompress_module, load_module, save_file
    dense = make_model(torch.bfloat16)
    path = str(tmp_path / "m.znn.safetensors")
    save_file(dealiased(dense), path)

    def load():
        m = build("cuda", torch.bfloat16)
        load_module(m, path)
        decompress_module(m)
        return {k: v.detach().clone() for k, v in m.state_dict().items()}
    small = load()
    with monkeypatch.context() as mp:
        mp.setattr(DecodePipe, "SLAB_BYTES", DEFAULT_RING)
        mp.setattr(DecodePipe, "COPY_PIECE", 8 << 20)
        DecodePipe._slab_cache.clear()
        default = load()
        DecodePipe._slab_cache.clear()
    assert list(small) == list(default)
    for k in default:
        assert _same(small[k], default[k]) and _same(small[k], dense.state_dict()[k]), k


def test_pipe_error_flags_roll_over(small_ring):
    g = torch.Generator().manual_seed(29)
    t = (torch.randn(300, generator=g) * 0.02).to(torch.bfloat16)
    s = ZipNN(input_format="torch").compress(t.cuda()).cpu().numpy()
    H = 32 + 1 + 1 + 2                                             # header + a 1-D shape with a 2-byte dimension
    assert s[H] == 0 and s.size > H
    bad = s.copy()
    bad[H] = 9                                                     # a type byte out of range: found on the device
    pipe = DecodePipe("cuda")
    got = [pipe.submit(s) for _ in range(1100)]
    first_flags = pipe._pending[0][0]
    assert pipe._pending[-1][0] is not first_flags and pipe._pending[-1][1] == 1100 - 1024 - 1
    pipe.finish()
    pipe.release()
    assert all(_same(x, t) for x in got)
    for at in (5, 1050):
        pipe = DecodePipe("cuda")
        for i in range(1100):
            pipe.submit(bad if i == at else s)
        with pytest.raises(RuntimeError, match="corrupt"):
            pipe.finish()
        pipe.release()


def test_pipe_slab_cache_keeps_sizes_apart(small_ring, monkeypatch):
    """Slabs cached by a pipe with one SLAB_BYTES are not handed to a pipe built with another."""
    g = torch.Generator().manual_seed(31)
    t = (torch.randn(700_000, generator=g) * 0.02).to(torch.bfloat16)
    s = ZipNN(input_format="torch").compress(t.cuda()).cpu().numpy()
    pipe = DecodePipe("cuda")
    x = pipe.submit(s)
    pipe.finish()
    pipe.release()
    assert _same(x, t) and DecodePipe._slab_cache and all(c.numel() == SMALL_RING for c in DecodePipe._slab_cache)
    for size in (3 * 65536 + 16, DEFAULT_RING):
        with monkeypatch.context() as mp:
            mp.setattr(DecodePipe, "SLAB_BYTES", size)
            pipe = DecodePipe("cuda")
            y = pipe.submit(s)
            pipe.finish()
            pipe.release()
        assert _same(y, t), size
    assert s.size > 2 * (3 * 65536 + 16)


# ================================================================== e. streaming frames
FRAME_DTYPES = {"bfloat16": 2, "float16": 2, "float32": 4, "float8_e4m3fn": 1}


def _frame_chunk(dtype, cc):
    G = FRAME_DTYPES[dtype]
    return cc if G != 1 else min(HM.HUF_MAX_BLOCK, cc)


def _streaming_chunks(chunk):
    """one chunk, several chunks, 1 MiB, below one chunk (per-frame compress loop), 8 bytes (decode fallback)."""
    return {"one": chunk, "several": 4 * chunk, "mib": 1 << 20, "below": chunk // 2, "tiny": 8}


def _frame_data(dtype, sc, kind, seed):
    n = {"exact": 3 * sc, "ragged": 2 * sc + sc // 2 + 6 if sc > 16 else 2 * sc + 6, "short": sc // 2 + 6 if sc > 16 else 6}[kind]
    G = FRAME_DTYPES[dtype]
    bits = 0 if G == 1 else 1
    rng = np.random.default_rng(seed)
    pattern = HM.DECODE_PATTERN[G]
    return HM.planned_bytes(pattern, G, bits, 4096, n, int(rng.integers(1 << 30))) if n >= 4096 else \
        rng.integers(0, 4, n).astype(np.uint8)


def oracle_frames(data, dtype, cc, sc, delta=0):
    code = dtype_code(dtype)
    bit_reorder, byte_reorder, G = Z._layout_for_dtype(code)
    chunk = _frame_chunk(dtype, cc)
    head = bytearray(32)
    head[0:5] = b"ZN" + bytes([0, 5, 3])
    head[5], head[6], head[7], head[8], head[9] = byte_reorder, bit_reorder, 0, 1, delta     # AUTO, byte format
    head[13], head[14], head[15] = 128 + int(math.log2(sc)), int(math.log2(cc)), code
    frames = []
    for off in range(0, data.size, sc):
        part = data[off: off + sc]
        h = bytearray(head)
        h[16:24] = part.size.to_bytes(8, "little")
        frames.append(O.zipnn_compress(h, part, G, bit_reorder, byte_reorder, chunk).tobytes())
    return frames


def _no_fast(monkeypatch):
    monkeypatch.setattr(ZipNN, "_compress_frames_at_once", lambda self, src: None)
    monkeypatch.setattr(ZipNN, "_decompress_frames_at_once", lambda self, stream: None)


@pytest.mark.parametrize("sck", ["one", "several", "mib", "below", "tiny"])
@pytest.mark.parametrize("cc", [4096, 262144])
@pytest.mark.parametrize("dtype", list(FRAME_DTYPES))
def test_streaming_frames(dtype, cc, sck, monkeypatch):
    chunk = _frame_chunk(dtype, cc)
    sc = _streaming_chunks(chunk)[sck]
    G = FRAME_DTYPES[dtype]
    for i, kind in enumerate(("exact", "ragged", "short")):
        data = _frame_data(dtype, sc, kind, seed=i)
        paths = HM.frame_paths(data.size, G, cc, sc)
        assert paths["compress"] == ("at_once" if sck in ("one", "several", "mib") else "loop")
        if sck == "tiny" and kind != "short":
            assert paths["decompress"] == "fallback"
        z = ZipNN(input_format="byte", bytearray_dtype=dtype, compression_chunk=cc, is_streaming=True, streaming_chunk=sc)
        want = oracle_frames(data, dtype, cc, sc)
        assert len(want) == len(paths["frames"])
        got = bytes(z.compress(data.tobytes()))
        at = 0
        for j, (w, (off, ln)) in enumerate(zip(want, paths["frames"])):
            f = got[at: at + len(w)]
            assert f[13] == 128 + int(math.log2(sc)) and int.from_bytes(f[16:24], "little") == ln
            assert int.from_bytes(f[24:32], "little") == len(w)
            assert f == w, f"frame {j} of {len(want)} != oracle"
            at += len(w)
        assert at == len(got)
        whole = b"".join(want)
        back = ZipNN(input_format="byte", bytearray_dtype=dtype, is_streaming=True).decompress(whole)
        assert bytes(back) == data.tobytes()
        with monkeypatch.context() as mp:
            _no_fast(mp)
            assert bytes(ZipNN(input_format="byte", bytearray_dtype=dtype, compression_chunk=cc, is_streaming=True,
                               streaming_chunk=sc).compress(data.tobytes())) == whole
            assert bytes(ZipNN(input_format="byte", bytearray_dtype=dtype, is_streaming=True).decompress(whole)) == data.tobytes()


def test_streaming_delta_and_errors(monkeypatch):
    dtype, cc, sc = "bfloat16", 4096, 8192
    rng = np.random.default_rng(5)
    data = HM.planned_bytes(HM.DECODE_PATTERN[2], 2, 1, 4096, 5 * sc + 1000, 7)
    base = data.copy()
    base[rng.choice(data.size, 500, replace=False)] ^= 0x10
    mk = lambda: ZipNN(input_format="byte", bytearray_dtype=dtype, compression_chunk=cc, is_streaming=True,  # noqa: E731
                       streaming_chunk=sc, delta_compressed_type="byte")
    want = b"".join(oracle_frames(np.bitwise_xor(data, base), dtype, cc, sc, delta=1))
    assert bytes(mk().compress(data.tobytes(), delta_second_data=base.tobytes())) == want
    with pytest.raises(ValueError, match="Length of delta"):
        mk().compress(data.tobytes(), delta_second_data=base[:-1].tobytes())
    for fast in (True, False):
        with monkeypatch.context() as mp:
            if not fast:
                _no_fast(mp)
            assert bytes(mk().decompress(want, delta_second_data=base.tobytes())) == data.tobytes()
            with pytest.raises(ValueError, match="Length of delta"):
                mk().decompress(want, delta_second_data=base[:-1].tobytes())       # short: at once, or mid-loop
            with pytest.raises(ValueError, match="Length of delta"):
                mk().decompress(want, delta_second_data=base.tobytes() + b"\0")    # long: at once, or after the loop
    # a frame whose length field runs past the end
    plain = b"".join(oracle_frames(data, dtype, cc, sc))
    bad = bytearray(plain)
    last = len(plain) - len(oracle_frames(data[-1000:], dtype, cc, sc)[0])
    bad[last + 24: last + 32] = (len(plain) - last + 1).to_bytes(8, "little")
    for fast in (True, False):
        with monkeypatch.context() as mp:
            if not fast:
                _no_fast(mp)
            with pytest.raises(RuntimeError, match="corrupt"):
                ZipNN(input_format="byte", bytearray_dtype=dtype, is_streaming=True).decompress(bytes(bad))
