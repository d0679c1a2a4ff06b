"""The device codec at every chunk size and threshold the stream format accepts (tests/chunk_settings.py).

Every case first asserts on the host that it reaches the branch it names: chunks too small for the warp-per-
stream emission kernel, the fused decode kernel taking 512-byte chunks, planes past 128 KiB that are always raw,
the planes where HUF_compress's destination capacity (the chunk) or the strict threshold comparison keeps a
block raw.  Then, against the oracle's stream:
  * encoders: zipnn_b200_compress, zipnn_b200_compress_host (one pass, and the slab pipeline with slabs of three
    chunks) and ZipNN(compression_chunk=..., compression_threshold=...) write it byte for byte, into buffers
    pre-filled with a canary so that unwritten payload bytes cannot pass as zeros, and leave the input alone;
  * decoders: it decodes to the input with both decoder families (ZIPNN_B200_SYNC_MAX 0 and large), through
    the batch entry point, and through zipnn_b200_decompress_slices on boxes that cross chunk edges, with and
    without forced piece splits; the bytes around every output stay untouched.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import chunk_settings as CS
import plane_inputs as P
from oracle import oracle as O
from zipnn_b200 import ZipNN, _native

pytestmark = pytest.mark.gpu

CANARY = 0xA5
PAD = 64
KNOBS = ("ZIPNN_B200_SYNC_MAX", "ZIPNN_B200_HOST_SLAB_BYTES", "ZIPNN_B200_SLICE_PIECE_CHUNKS")
CASES = CS.settings_inputs()
ZIPNN_DTYPE = {(1, 0): torch.float8_e4m3fn, (2, 0): torch.float16, (2, 1): torch.bfloat16, (4, 1): torch.float32}


def _env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bm(G):
    return 220 if G == 4 else 10


def _types(stream, G, K):
    return np.frombuffer(stream, dtype=np.uint8)[32: 32 + G * K].reshape(G, K)


# ------------------------------------------------------------------ coverage: each case reaches its branch
def assert_reaches_branch(c, stream):
    G, chunk, n = c["G"], c["chunk"], c["data"].size
    K = -(-n // chunk)
    types = _types(stream, G, K)
    if chunk < 64 * G:
        # no chunk is a multiple of 64*G: none suits the warp kernel, the general kernel writes every payload
        lens = [min(chunk, n - k * chunk) for k in range(K)]
        assert all(L % (64 * G) for L in lens)
    if c["kind"] == "chunk" and chunk == 512 and c["family"] == "gauss":
        pr = P.predict(np.frombuffer(stream, np.uint8)[32:], G, c["bits"], chunk, n)
        assert any(v == "fused" for v in pr["fused"].values()), "no chunk reaches the fused decode kernel"
    if chunk // G > 128 * 1024:
        assert not types[:, : n // chunk].any(), "a plane past 128 KiB was coded"
    if c["kind"] in ("capflip", "capslack", "exact"):
        planes = c["data"].reshape(-1, c["plen"])
        assert not types.any()
        for p in planes:
            if c["kind"] == "exact":
                assert O.huf_compress(p, c["plen"])[0] == c["plen"] * c["thr"]
            else:
                assert CS.stored_size(p, 1 << 20, c["thr"]) > 1, "an unbounded destination would not code it"
    if c["kind"] == "rle":
        col = types[:, -1] if c["plen"] == 3 else types[:, 0]
        assert (col == (1 if 1 < c["plen"] * np.float32(c["thr"]) else 0)).all()


# ------------------------------------------------------------------ encoders
def device_compress(c):
    G, n, chunk = c["G"], c["data"].size, c["chunk"]
    d_in = torch.from_numpy(c["data"].copy()).cuda()
    bound = _native.compress_bound(n, G, chunk, 32)
    d_out = torch.full((bound + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.compress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
    out_len = C.c_size_t(0)
    hbuf = (C.c_char * 32).from_buffer_copy(CS.header())
    rc = _native.lib().zipnn_b200_compress(d_in.data_ptr(), n, hbuf, 32, G, c["bits"], _bm(G), chunk, c["thr"], d_out.data_ptr(),
                                           bound, C.byref(out_len), ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, rc
    assert np.array_equal(d_in.cpu().numpy(), c["data"]), "the encoder changed its input"
    host = d_out.cpu().numpy()
    assert np.all(host[out_len.value:] == CANARY), "wrote past the stream"
    return host[: out_len.value]


def host_compress(c):
    G, n, chunk = c["G"], c["data"].size, c["chunk"]
    src = c["data"].copy()
    bound = _native.compress_bound(n, G, chunk, 32)
    out = np.full(bound + PAD, CANARY, dtype=np.uint8)
    out_len = C.c_size_t(0)
    hbuf = (C.c_char * 32).from_buffer_copy(CS.header())
    rc = _native.lib().zipnn_b200_compress_host(src.ctypes.data, n, hbuf, 32, G, c["bits"], _bm(G), chunk, c["thr"], out.ctypes.data,
                                                bound, C.byref(out_len))
    assert rc == 0, rc
    assert np.array_equal(src, c["data"])
    assert np.all(out[bound:] == CANARY)
    return out[: out_len.value]


def check_encoders(c, want, monkeypatch):
    name = c["name"]
    assert np.array_equal(device_compress(c), want), f"{name}: device stream != oracle stream"
    _env(monkeypatch, {})
    assert np.array_equal(host_compress(c), want), f"{name}: host-buffer stream != oracle stream"
    if c["data"].size > 3 * c["chunk"]:
        _env(monkeypatch, {"ZIPNN_B200_HOST_SLAB_BYTES": str(3 * c["chunk"])})
        assert np.array_equal(host_compress(c), want), f"{name}: slab pipeline stream != oracle stream"
        _env(monkeypatch, {})
    dt = ZIPNN_DTYPE.get((c["G"], c["bits"]))
    if dt is not None:
        t = torch.from_numpy(c["data"].copy()).view(dt)
        z = ZipNN(input_format="torch", compression_chunk=c["chunk"], compression_threshold=c["thr"])
        plan = z.plan(t)
        ref = O.zipnn_compress(plan["header"], c["data"], plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], plan["chunk"],
                               plan["threshold"], threads=8)
        got = z.compress(t.cuda()).cpu().numpy()
        assert np.array_equal(got, ref), f"{name}: ZipNN stream != oracle stream"


# ------------------------------------------------------------------ decoders
def decode_single(c, body):
    G, n, chunk = c["G"], c["data"].size, c["chunk"]
    d_body = torch.from_numpy(body.copy()).cuda()
    out = torch.full((PAD + n + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.decompress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
    rc = _native.lib().zipnn_b200_decompress(d_body.data_ptr(), body.size, G, c["bits"], _bm(G), chunk, n, out[PAD:].data_ptr(),
                                             ws.data_ptr(), ws.numel(), _stream(), 1)
    host = out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY), f"{c['name']}: wrote outside the output"
    return rc, host[PAD: PAD + n]


def decode_batch(c, body):
    G, n = c["G"], c["data"].size
    arr = (_native.BatchItem * 1)()
    d_body = torch.from_numpy(body.copy()).cuda()
    out = torch.full((PAD + n + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    arr[0].d_body, arr[0].body_len = d_body.data_ptr(), body.size
    arr[0].num_buf, arr[0].bits_mode, arr[0].bytes_mode = G, c["bits"], _bm(G)
    arr[0].chunk, arr[0].orig, arr[0].d_out = c["chunk"], n, out[PAD:].data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(arr, 1, C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decompress_batch(arr, 1, ws.data_ptr(), ws.numel(), _stream(), 1)
    host = out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY), f"{c['name']}: batch wrote outside"
    return rc, host[PAD: PAD + n]


def decode_slice(c, body, base, rows, pitch, length):
    G, n = c["G"], c["data"].size
    it = (_native.SliceItem * 1)()
    d_body = torch.from_numpy(body.copy()).cuda()
    n_out = rows * length
    out = torch.full((PAD + n_out + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    it[0].d_body, it[0].body_len = d_body.data_ptr(), body.size
    it[0].num_buf, it[0].bits_mode, it[0].bytes_mode = G, c["bits"], _bm(G)
    it[0].chunk, it[0].orig = c["chunk"], n
    it[0].base, it[0].rows, it[0].pitch, it[0].len, it[0].d_out = base, rows, pitch, length, out[PAD:].data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_slices_workspace_size(it, 1, C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decompress_slices(it, 1, ws.data_ptr(), ws.numel(), _stream(), 1)
    host = out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n_out:] == CANARY), f"{c['name']}: slice wrote outside"
    return rc, host[PAD: PAD + n_out]


def slice_boxes(c):
    """One run that starts and ends inside chunks and crosses several chunk edges, and a band of columns of the
    tensor viewed as rows of 2.5 chunks (each row crossing chunk edges), in whole elements."""
    G, chunk, n = c["G"], c["chunk"], c["data"].size
    base = min(chunk // 2 + G, n - G) // G * G
    run = (base, 1, 0, max(G, min(n - base, 5 * chunk + 7 * G) // G * G))
    pitch = max(G, (5 * chunk // 2 + G) // G * G)
    rows = n // pitch
    boxes = [run]
    if rows >= 2:
        c0 = (pitch // 4) // G * G
        boxes.append((c0, rows, pitch, max(G, (pitch // 2) // G * G)))
    return boxes


def check_decoders(c, body, monkeypatch):
    name, data = c["name"], c["data"]
    for env in ({"ZIPNN_B200_SYNC_MAX": "0"}, {"ZIPNN_B200_SYNC_MAX": str(1 << 24)}):
        _env(monkeypatch, env)
        rc, got = decode_single(c, body)
        assert rc == 0 and np.array_equal(got, data), (name, env, rc)
    _env(monkeypatch, {})
    rc, got = decode_batch(c, body)
    assert rc == 0 and np.array_equal(got, data), (name, "batch", rc)
    for env in ({}, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "2"}):
        _env(monkeypatch, env)
        for box in slice_boxes(c):
            base, rows, pitch, length = box
            want = np.concatenate([data[base + r * pitch: base + r * pitch + length] for r in range(rows)])
            rc, got = decode_slice(c, body, *box)
            assert rc == 0 and np.array_equal(got, want), (name, env, box, rc)
    _env(monkeypatch, {})


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c["name"] for c in CASES])
def test_setting(idx, monkeypatch):
    c = CASES[idx]
    want = O.zipnn_compress(CS.header(), c["data"], c["G"], c["bits"], _bm(c["G"]), c["chunk"], c["thr"], threads=8)
    assert_reaches_branch(c, want.tobytes())
    check_encoders(c, want, monkeypatch)
    check_decoders(c, want[32:], monkeypatch)


# ------------------------------------------------------------------ the largest chunk the ABI accepts
def test_largest_chunk_two_chunks_second_ragged():
    """bf16 at chunk 2^31: two chunks, the second 1 MiB.  Every plane is raw (the first chunk's planes are 1 GiB,
    the second's 512 KiB), so the stream is the format's raw layout; it is assembled here from the oracle's split
    rather than by O.zipnn_compress, whose per-thread scratch of one chunk per plane would need 10 GiB of host
    memory at this size."""
    G, bits, chunk = 2, 1, 1 << 31
    n = chunk + (1 << 20)
    rng = np.random.default_rng(31)
    data = rng.integers(0, 256, n, dtype=np.uint8)
    planes = [O.split_chunk(data[:chunk], G, bits), O.split_chunk(data[chunk:], G, bits)]
    sizes = np.array([[p[g].size for p in planes] for g in range(G)], dtype=np.uint64)
    hdr = bytearray(CS.header())
    total = 32 + 9 * G * 2 + n
    hdr[24:32] = total.to_bytes(8, "little")
    want = np.concatenate([np.frombuffer(bytes(hdr), np.uint8), np.zeros(G * 2, np.uint8),
                           np.cumsum(sizes, axis=1).astype("<u8").view(np.uint8).reshape(-1)] +
                          [p[g] for g in range(G) for p in planes])
    del planes
    c = {"name": "chunk-2^31", "G": G, "bits": bits, "chunk": chunk, "thr": 0.95, "data": data}
    got = device_compress(c)
    assert got.size == want.size and np.array_equal(got, want)
    del got
    rc, back = decode_single(c, want[32:])
    assert rc == 0 and np.array_equal(back, data)


# ------------------------------------------------------------------ below G
@pytest.mark.parametrize("G,chunk", [(2, 1), (4, 1), (4, 2)])
def test_chunk_below_group_is_rejected(G, chunk):
    bits, bm = 1, _bm(G)
    n = 64 * G
    L = _native.lib()
    d_in = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(4 * n + 4096, dtype=torch.uint8, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    h_in = np.zeros(n, np.uint8)
    h_out = np.zeros(4 * n + 4096, np.uint8)
    out_len = C.c_size_t(0)
    hbuf = (C.c_char * 32).from_buffer_copy(CS.header())
    assert L.zipnn_b200_compress(d_in.data_ptr(), n, hbuf, 32, G, bits, bm, chunk, 0.95, d_out.data_ptr(), d_out.numel(),
                                 C.byref(out_len), ws.data_ptr(), ws.numel(), _stream()) == _native.E_ARG
    assert L.zipnn_b200_compress_host(h_in.ctypes.data, n, hbuf, 32, G, bits, bm, chunk, 0.95, h_out.ctypes.data, h_out.size,
                                      C.byref(out_len)) == _native.E_ARG
    assert L.zipnn_b200_decompress(d_out.data_ptr(), 2048, G, bits, bm, chunk, n, d_in.data_ptr(), ws.data_ptr(), ws.numel(),
                                   _stream(), 1) == _native.E_ARG
    assert L.zipnn_b200_decompress_host(h_out.ctypes.data, 2048, G, bits, bm, chunk, n, h_in.ctypes.data) == _native.E_ARG
    arr = (_native.BatchItem * 1)()
    arr[0].d_body, arr[0].body_len, arr[0].num_buf, arr[0].bits_mode, arr[0].bytes_mode = d_out.data_ptr(), 2048, G, bits, bm
    arr[0].chunk, arr[0].orig, arr[0].d_out = chunk, n, d_in.data_ptr()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(arr, 1, C.byref(wsz)) == _native.E_ARG
    assert L.zipnn_b200_decompress_batch(arr, 1, ws.data_ptr(), ws.numel(), _stream(), 1) == _native.E_ARG
    it = (_native.SliceItem * 1)()
    it[0].d_body, it[0].body_len, it[0].num_buf, it[0].bits_mode, it[0].bytes_mode = d_out.data_ptr(), 2048, G, bits, bm
    it[0].chunk, it[0].orig, it[0].base, it[0].rows, it[0].pitch, it[0].len, it[0].d_out = chunk, n, 0, 1, 0, G, d_in.data_ptr()
    assert L.zipnn_b200_decompress_slices_workspace_size(it, 1, C.byref(wsz)) == _native.E_ARG
    assert L.zipnn_b200_decompress_slices(it, 1, ws.data_ptr(), ws.numel(), _stream(), 1) == _native.E_ARG
    dt = torch.bfloat16 if G == 2 else torch.float32
    with pytest.raises(_native.ZipNNNativeError):
        ZipNN(input_format="torch", compression_chunk=chunk).compress(torch.zeros(64, dtype=dt, device="cuda"))
    with pytest.raises(_native.ZipNNNativeError):
        ZipNN(input_format="torch", compression_chunk=chunk).compress(torch.zeros(64, dtype=dt))
