"""Sliced reads on the GPU: ZipNN.decompress_slice and SafeOpen(..., slices=True).get_slice equal indexing the whole
tensor, bit for bit, and decode only the chunks the index covers."""
import json
import os

import numpy as np
import pytest
import torch
from safetensors import safe_open
from safetensors.torch import save_file

from golden_safetensors_inputs import make_checkpoint

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "ref_model.znn.safetensors")
DTYPES = [torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn]


def _t(shape, dt, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * (0.5 if dt == torch.float8_e4m3fn else 0.02)).to(dt)


def _bits(x):
    return x.contiguous().reshape(-1).view(torch.uint8).cpu()


def _same(a, b):
    return a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and torch.equal(_bits(a), _bits(b))


def _indexes(shape):
    out = [(), Ellipsis, 0, -1, slice(None), slice(2, 2), slice(5, 1), slice(None, None, 3), slice(-3, None)]
    for d, n in enumerate(shape):
        pre = (slice(None),) * d
        out += [pre + (slice(1, n - 1),), pre + (n // 2,), pre + (-2,), pre + (slice(0, n, 2),), pre + (slice(n // 3, None, 5),)]
    if len(shape) >= 2:
        out += [(slice(1, 4), slice(2, 7)), (2, Ellipsis, slice(1, 3)), (Ellipsis, 1), (slice(None, None, 2), slice(3, None, 4))]
    return out


def _check_stream(t, chunk, indexes=None):
    from zipnn_b200 import ZipNN
    full = t.cuda()
    s = ZipNN(input_format="torch", compression_chunk=chunk).compress(full)
    host = s.cpu()
    for idx in indexes if indexes is not None else _indexes(tuple(t.shape)):
        want = full[idx]
        got = ZipNN(input_format="torch").decompress_slice(s, idx)
        assert got.is_cuda and _same(got, want), (t.dtype, tuple(t.shape), idx)
        got = ZipNN(input_format="torch").decompress_slice(host, idx)
        assert not got.is_cuda and _same(got, want), ("host", t.dtype, tuple(t.shape), idx)


@pytest.mark.parametrize("dt", DTYPES)
def test_decompress_slice_equals_full_index(dt):
    _check_stream(_t((70001,), dt, 1), 4096)                       # ragged last chunk
    _check_stream(_t((301, 256), dt, 2), 4096)
    _check_stream(_t((7, 33, 65), dt, 3), 4096)
    _check_stream(_t((300, 257), dt, 4), 256 * 1024)               # the default chunk


def test_both_store_classes():
    t = _t((301, 256), torch.bfloat16, 5)                           # 512-byte rows
    _check_stream(t, 4096, [(slice(None), slice(8, 16)),            # base, pitch, len multiples of 16
                            (slice(3, 200), slice(64, 192)),
                            (slice(None), slice(3, 10)),            # 2-byte granular
                            (slice(None), 7)])
    _check_stream(_t((40, 33, 5), torch.bfloat16, 6), 4096, [(Ellipsis, slice(1, 3)), (slice(2, 30), slice(None), 4)])  # pitch < 16


def test_stream_shapes():
    _check_stream(torch.zeros(5000, 64, dtype=torch.bfloat16), 4096, [slice(7, 900), (slice(None), slice(5, 9))])     # RLE
    up = _t((100, 65536), torch.bfloat16, 7).to(torch.float32)     # two coded groups in every chunk: general chunks
    _check_stream(up, 256 * 1024, [slice(None), slice(1, 99), (slice(None), slice(5, 9000)), (slice(None, None, 3), slice(100, 101))])
    big = _t((4100, 1024), torch.bfloat16, 8)                       # 4100 chunks
    _check_stream(big, 2048, [slice(10, 4000), (slice(None), slice(100, 700)), (slice(None), 5)])


def test_piece_splitting(monkeypatch):
    monkeypatch.setenv("ZIPNN_B200_SLICE_PIECE_CHUNKS", "3")
    _check_stream(_t((301, 256), torch.bfloat16, 9), 4096, [slice(None), slice(5, 290), (slice(None), slice(3, 10)),
                                                            (slice(None), slice(16, 48)), (slice(None), slice(0, 255))])
    _check_stream(_t((9001, 3), torch.float32, 10), 4096, [(slice(None), 1), slice(17, 8000)])
    _check_stream(_t((70001,), torch.float8_e4m3fn, 11), 4096, [slice(3, 69999), slice(None, None, 7)])


def test_only_covered_chunks_are_used():
    from zipnn_b200 import ZipNN
    from zipnn_b200.slicing import MemorySource, StreamIndex
    t = _t((64, 2048), torch.bfloat16, 12)                          # one 4 KiB chunk per row
    s = ZipNN(input_format="torch", compression_chunk=4096).compress(t.cuda()).cpu()
    idx = StreamIndex(MemorySource(s.numpy()))
    c = 10
    assert idx.types[1, c] == 1 and int(idx.cum[1, c]) - int(idx.cum[1, c - 1]) > 1
    bad = s.clone()
    bad[idx.group_off[1] + int(idx.cum[1, c]) - 1] = 0              # the chunk's last bitstream loses its end mark
    for stream in (bad, bad.cuda()):
        got = ZipNN(input_format="torch").decompress_slice(stream, slice(20, 30))
        assert _same(got, t[20:30])
        got = ZipNN(input_format="torch").decompress_slice(stream, (slice(None, 10), slice(5, 9)))
        assert _same(got, t[:10, 5:9])
        with pytest.raises(RuntimeError, match="corrupt"):
            ZipNN(input_format="torch").decompress_slice(stream, slice(5, 12))
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="corrupt"):
            ZipNN(input_format="torch").decompress_slice(stream, (slice(None), 3))
        torch.cuda.synchronize()


def test_launch_count_is_fixed():
    from zipnn_b200 import ZipNN, _native
    t = _t((2000, 1024), torch.bfloat16, 13)
    s = ZipNN(input_format="torch", compression_chunk=4096).compress(t.cuda())
    counts = []
    for idx in (slice(3, 4), slice(0, 2000), (slice(None), slice(1, 5)), slice(None, None, 2)):
        before = _native.launch_count()
        ZipNN(input_format="torch").decompress_slice(s, idx)
        counts.append(_native.launch_count() - before)
    assert len(set(counts)) == 1 and counts[0] > 0, counts


def test_streaming_frames_are_refused():
    from zipnn_b200 import ZipNN
    s = ZipNN(input_format="byte", bytearray_dtype="bfloat16", is_streaming=True).compress(bytes(4096))
    with pytest.raises(ValueError):
        ZipNN(input_format="torch").decompress_slice(bytes(s), slice(0, 4))


def _twin(tmp_path):
    from zipnn_b200 import compress_safetensors_file
    want = {"bf16": _t((300, 257), torch.bfloat16, 14), "fp16": _t((64, 3, 129), torch.float16, 15),
            "fp32": _t((1000, 96), torch.float32, 16), "fp8": _t((513, 64), torch.float8_e4m3fn, 17),
            "ids": torch.arange(600, dtype=torch.int64).reshape(6, 100)}
    src = str(tmp_path / "m.safetensors")
    save_file(want, src)
    path, _, _ = compress_safetensors_file(src)
    return src, path


def _compare_slices(plain_path, znn_path, device):
    from zipnn_b200 import CompressedSlice, SafeOpen
    with safe_open(plain_path, "pt", "cpu") as p, SafeOpen(znn_path, "pt", device, slices=True) as f:
        assert set(f.keys()) == set(p.keys())
        for name in p.keys():
            a, b = p.get_slice(name), f.get_slice(name)
            if name in f.compressed_tensors_metadata:
                assert isinstance(b, CompressedSlice)
            assert b.get_shape() == a.get_shape() and b.get_dtype() == a.get_dtype(), name
            for idx in _indexes(tuple(a.get_shape())):
                want, got = a[idx], b[idx]
                assert got.device.type == torch.device(device).type, (name, idx)
                assert _same(got, want), (name, idx)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
def test_safe_open_slices_match_safetensors(tmp_path, device):
    src, path = _twin(tmp_path)
    _compare_slices(src, path, device)
    with safe_open(GOLD, "pt", "cpu") as f:
        assert set(json.loads(f.metadata()["znn_compressed_vectors"])) == {"w_bf16", "w_fp16", "w_fp32", "w_fp8", "big_bf16"}
    plain = str(tmp_path / "ref_plain.safetensors")
    save_file(make_checkpoint(), plain)
    _compare_slices(plain, GOLD, device)


def test_patch_with_slices(tmp_path):
    import safetensors.torch
    from zipnn_b200 import CompressedSlice, zipnn_safetensors
    src, path = _twin(tmp_path)
    saved = safetensors.torch.safe_open
    try:
        zipnn_safetensors(slices=True)
        with safetensors.torch.safe_open(path, framework="pt", device="cuda") as f:
            sl = f.get_slice("bf16")
            assert isinstance(sl, CompressedSlice)
            with safe_open(src, "pt", "cpu") as p:
                assert _same(sl[10:20, 3:9], p.get_slice("bf16")[10:20, 3:9])
    finally:
        safetensors.torch.safe_open = saved


def test_transformers_tensor_parallel_shards(tmp_path):
    from transformers.integrations.tensor_parallel import get_tensor_shard
    from zipnn_b200 import SafeOpen
    src, path = _twin(tmp_path)
    with safe_open(src, "pt", "cpu") as p, SafeOpen(path, "pt", "cuda", slices=True) as f:
        for name in ("bf16", "fp32", "fp8"):
            a, b = p.get_slice(name), f.get_slice(name)
            empty = torch.empty(a.get_shape(), device="meta")
            for world in (1, 2, 3, 8, 14):
                mesh = torch.empty(world)
                for dim in (0, 1, -1):
                    for rank in range(world):
                        want = get_tensor_shard(a, empty, mesh, rank, dim)
                        got = get_tensor_shard(b, empty, mesh, rank, dim)
                        assert tuple(got.shape) == tuple(want.shape), (name, world, dim, rank)
                        if want.numel():
                            assert _same(got, want), (name, world, dim, rank)
    _ = np
