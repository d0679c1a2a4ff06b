"""What the device calls keep between calls -- launch plans per (kernel, device), pinned read-back blocks, cached sizes
-- must never carry one call's tensor into the next.  Calls of several sizes, dtypes and layouts are interleaved on one
stream, on side streams and on every visible device, and each result is checked against its own input (and the
stream against the oracle's, where the oracle is fast enough)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as O
from zipnn_b200 import ZipNN, _native
from zipnn_b200.zipnn import HEADER_LEN

gpu = pytest.mark.gpu

# (dtype, shape): every dtype, multi-dimensional shapes, sizes on both sides of the per-bitstream-CTA /
# one-thread-per-bitstream crossover (3072 chunks of 256 KiB for two groups, 1536 for four), ragged last chunks and an
# empty tensor
CASES = [
    (torch.bfloat16, (3, 5, 7)),
    (torch.float32, (70001,)),
    (torch.float16, (257, 129)),
    (torch.float8_e4m3fn, (200000,)),
    (torch.bfloat16, (3200 * 131072 + 999,)),
    (torch.float32, (1536 * 65536 + 13,)),
    (torch.bfloat16, (0,)),
    (torch.float16, (4099,)),
]


def _make(dtype, shape, seed, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    n = int(np.prod(shape))
    sigma = 0.5 if dtype == torch.float8_e4m3fn else 0.02
    return (torch.randn(n, generator=g, device=device, dtype=torch.float32) * sigma).to(dtype).reshape(shape)


def _bytes(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


def _oracle_stream(t):
    plan = ZipNN(input_format="torch").plan(t.cpu())
    raw = _bytes(t).cpu().numpy()
    return O.zipnn_compress(plan["header"], raw, plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], plan["chunk"],
                            plan["threshold"], threads=2)


@gpu
def test_interleaved_sizes_and_dtypes_on_one_stream():
    inputs = [_make(dt, shape, 100 + i) for i, (dt, shape) in enumerate(CASES)]
    small = {i for i, t in enumerate(inputs) if t.numel() * t.element_size() < (8 << 20)}
    want = {i: _oracle_stream(inputs[i]) for i in small}
    # forwards, backwards and forwards again: every call follows a call of another size, dtype or layout
    order = list(range(len(CASES))) + list(reversed(range(len(CASES)))) + list(range(len(CASES)))
    for i in order:
        x = inputs[i]
        s = ZipNN(input_format="torch").compress(x)
        if i in small:
            assert np.array_equal(s.cpu().numpy(), want[i]), f"stream of case {i}"
        y = ZipNN(input_format="torch").decompress(s)
        assert y.is_cuda and y.dtype == x.dtype and tuple(y.shape) == tuple(x.shape) and y.is_contiguous()
        assert torch.equal(_bytes(y), _bytes(x)), f"round trip of case {i}"


@gpu
def test_past_4gib_between_small_calls():
    """A tensor of more than 4 GiB (input offsets past 2^32) between two small ones, twice."""
    small = _make(torch.float16, (4099,), 7)
    big = _make(torch.bfloat16, ((4 << 30) // 2 + 3 * 131072 + 5,), 8)
    want_small = _oracle_stream(small)
    first = None
    for _ in range(2):
        s0 = ZipNN(input_format="torch").compress(small)
        sb = ZipNN(input_format="torch").compress(big)
        assert sb.numel() > (1 << 32) * 0.6
        if first is None:
            first = sb.clone()
        else:
            assert torch.equal(sb, first), "the same tensor coded twice gave two streams"
        assert np.array_equal(s0.cpu().numpy(), want_small)
        yb = ZipNN(input_format="torch").decompress(sb)
        assert torch.equal(_bytes(yb), _bytes(big))
        y0 = ZipNN(input_format="torch").decompress(s0)
        assert torch.equal(_bytes(y0), _bytes(small))
        del sb, yb
    del first, big
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("where", ["size_table", "total"])
def test_corrupt_stream_raises_and_the_next_call_is_clean(where):
    x = _make(torch.bfloat16, (3200 * 131072,), 11)   # the one-thread-per-bitstream decoder
    s = ZipNN(input_format="torch").compress(x)
    bad = s.clone()
    hdr = len(ZipNN(input_format="torch").plan(x)["header"])
    G, K = 2, (x.numel() * 2 + 262143) // 262144
    cum = hdr + G * K                                  # u64 cumulative sizes, group-major
    if where == "size_table":
        bad[cum + 8 * (K + 7): cum + 8 * (K + 8)] = 0xFF   # a group-1 entry far past the payload
    else:
        bad[cum + 8 * (K - 1): cum + 8 * K] = 0x7F         # group 0's total
    with pytest.raises(RuntimeError, match="corrupt"):
        ZipNN(input_format="torch").decompress(bad)
    # the error word belongs to that call's workspace: a good stream right after decodes
    y = ZipNN(input_format="torch").decompress(s)
    assert torch.equal(_bytes(y), _bytes(x))
    with pytest.raises(RuntimeError, match="corrupt"):
        ZipNN(input_format="torch").decompress(bad)


@gpu
def test_side_streams_interleaved():
    """Calls on two side streams and the default one, enqueued back to back: each call's read-backs wait for its own
    stream only, and each result is its own input's."""
    xs = [_make(dt, shape, 200 + i) for i, (dt, shape) in enumerate(CASES[:6])]
    streams = [torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.current_stream()]
    outs = []
    for i, x in enumerate(xs):
        st = streams[i % 3]
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            s = ZipNN(input_format="torch").compress(x)
            outs.append((st, s, ZipNN(input_format="torch").decompress(s)))
    torch.cuda.synchronize()
    for x, (_, _, y) in zip(xs, outs):
        assert torch.equal(_bytes(y), _bytes(x))


@gpu
def test_every_device_with_another_current():
    """A tensor on each visible device while another device is current: the launch plans (shared-memory attributes,
    occupancy) are the tensor's device's, and the result lands there."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("one visible device")
    xs = [_make(torch.bfloat16, (3200 * 131072 + 77,), 300 + d, device=f"cuda:{d}") for d in range(n)]
    for rounds in range(2):
        for d in range(n):
            torch.cuda.set_device((d + 1) % n)
            x = xs[d]
            s = ZipNN(input_format="torch").compress(x)
            y = ZipNN(input_format="torch").decompress(s)
            assert s.device == x.device and y.device == x.device
            assert torch.equal(_bytes(y), _bytes(x))
    torch.cuda.set_device(0)


@gpu
def test_peek_reads_after_the_stream_work():
    """zipnn_b200_peek sees what the work enqueued before it wrote, on a busy side stream."""
    st = torch.cuda.Stream()
    L = _native.lib()
    with torch.cuda.stream(st):
        big = torch.zeros(1 << 28, dtype=torch.uint8, device="cuda")
        for v in (3, 5, 9):
            big.fill_(v)
            got = C.create_string_buffer(4096)
            _native.check(L.zipnn_b200_peek(big.data_ptr() + 12345, 4096, got, st.cuda_stream))
            assert got.raw == bytes([v]) * 4096


def test_peek_rejects_more_than_a_block():
    L = _native.lib()
    buf = C.create_string_buffer(8192)
    assert L.zipnn_b200_peek(None, 0, None, None) == _native.OK
    assert L.zipnn_b200_peek(1 << 20, 4097, buf, None) == _native.E_ARG
    assert L.zipnn_b200_peek(None, 16, buf, None) == _native.E_ARG


def test_size_queries_are_the_library_answers():
    out = C.c_size_t(0)
    for n, G, chunk in ((1 << 21, 2, 1 << 18), (12345, 4, 1 << 18), (0, 1, 1 << 17), ((5 << 30) + 3, 2, 1 << 18)):
        for _ in range(2):   # the second answer comes from the binding's cache
            _native.check(_native.lib().zipnn_b200_compress_workspace_size(n, G, chunk, C.byref(out)))
            assert _native.compress_workspace_size(n, G, chunk) == out.value
            _native.check(_native.lib().zipnn_b200_decompress_workspace_size(n, G, chunk, C.byref(out)))
            assert _native.decompress_workspace_size(n, G, chunk) == out.value
            _native.check(_native.lib().zipnn_b200_compress_bound(n, G, chunk, HEADER_LEN + 10, C.byref(out)))
            assert _native.compress_bound(n, G, chunk, HEADER_LEN + 10) == out.value


def test_default_threads_unchanged():
    import multiprocessing
    assert ZipNN().threads == min(multiprocessing.cpu_count(), 16)
    assert ZipNN(threads=3).threads == 3
