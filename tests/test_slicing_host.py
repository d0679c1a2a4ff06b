"""Host side of sliced reads (zipnn_b200/slicing.py): the index planner against numpy indexing, a restatement of
the meta kernel's "chunk meets box" rule against brute force, and the sub-stream reader against the oracle."""
import os
import random

import numpy as np
import pytest
import torch

from zipnn_b200 import slicing
from zipnn_b200.slicing import FileSource, MemorySource, StreamIndex, apply_residual, plan_index

ESIZES = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def cut_box(buf: np.ndarray, box) -> np.ndarray:
    base, rows, pitch, ln = box
    if rows * ln == 0:
        return buf[:0]
    return np.concatenate([buf[base + r * pitch: base + r * pitch + ln] for r in range(rows)])


def random_index(rng, shape):
    items = []
    for size in shape:
        k = rng.random()
        if k < 0.2:
            items.append(rng.randrange(-size, size))
        elif k < 0.35:
            items.append(slice(None))
        else:
            a = rng.choice([None, rng.randrange(-size - 2, size + 3)])
            b = rng.choice([None, rng.randrange(-size - 2, size + 3)])
            st = rng.choice([None, 1, 1, 2, 3, rng.randrange(1, size + 2)])
            items.append(slice(a, b, st))
    k = rng.random()
    if k < 0.15:                          # leave trailing dims out
        items = items[: rng.randint(0, len(items))]
    elif k < 0.35:                        # an Ellipsis stands for a run of dims (every item keeps its dim)
        a = rng.randint(0, len(items))
        b = rng.randint(a, len(items))
        items = items[:a] + [Ellipsis] + items[b:]
    if len(items) == 1 and rng.random() < 0.5:
        return items[0]
    return tuple(items)


def test_planner_matches_numpy():
    rng = random.Random(11)
    cases = 0
    while cases < 2400:
        ndim = rng.randint(1, 4)
        shape = tuple(rng.choice([1, 2, 3, 5, 7, 8, 16]) for _ in range(ndim))
        esize = rng.choice(list(ESIZES))
        idx = random_index(rng, shape)
        n = int(np.prod(shape))
        arr = np.arange(n, dtype=ESIZES[esize]).reshape(shape)
        buf = arr.reshape(-1).view(np.uint8)
        want = arr[idx]
        plan = plan_index(shape, esize, idx)
        assert plan.out_shape == want.shape, (shape, idx)
        base, rows, pitch, ln = plan.box
        if rows * ln:
            assert base + (rows - 1) * pitch + ln <= buf.size and (rows == 1 or ln <= pitch), (shape, idx, plan.box)
            assert ln % esize == 0 and base % esize == 0
        got = apply_residual(cut_box(buf, plan.box).view(ESIZES[esize]), plan)
        assert np.array_equal(got, want), (shape, esize, idx, plan)
        cases += 1


def test_planner_boxes_are_exact_for_tensor_parallel_shards():
    # column-parallel (dim 0) and row-parallel (dim 1) shards are one box with no residual
    for idx, box in (((slice(4, 8),), (4 * 12 * 2, 1, 4 * 12 * 2, 4 * 12 * 2)),
                     ((slice(None), slice(3, 6)), (3 * 2, 16, 12 * 2, 3 * 2)),
                     ((Ellipsis, slice(0, 6)), (0, 16, 12 * 2, 6 * 2)),
                     ((slice(None, None, 2),), (0, 8, 2 * 12 * 2, 12 * 2)),
                     ((3, slice(1, 12, 5)), (3 * 12 * 2 + 2, 3, 10, 2))):
        plan = plan_index((16, 12), 2, idx)
        assert plan.box == box and plan.residual is None, (idx, plan)


def test_planner_errors_like_safetensors():
    with pytest.raises(ValueError):
        plan_index((4, 5), 2, slice(None, None, -1))
    with pytest.raises(ValueError):
        plan_index((4, 5), 2, (slice(None), slice(None, None, 0)))
    with pytest.raises(IndexError):
        plan_index((4, 5), 2, 4)
    with pytest.raises(IndexError):
        plan_index((4, 5), 2, (0, 0, 0))
    with pytest.raises(IndexError):
        plan_index((4, 5), 2, (Ellipsis, 0, Ellipsis))


# ---- the meta kernel's skip rule (zipnn_b200/csrc/decode.cuh: box_meets), restated on the host ----
def box_meets(box, a, n):
    base, rows, pitch, ln = box
    e0 = base + ln
    r = 0 if a < e0 else (a - e0) // pitch + 1
    return r < rows and base + r * pitch < a + n


def brute_meets(box, a, n):
    base, rows, pitch, ln = box
    return any(base + r * pitch < a + n and a < base + r * pitch + ln for r in range(rows))


def test_skip_rule_matches_brute_force():
    rng = random.Random(5)
    for _ in range(3000):
        chunk = rng.choice([16, 64, 256])
        kind = rng.random()
        if kind < 0.3:                 # rows == 1 (the pitch only has to be >= len)
            rows, ln = 1, rng.randint(1, 5 * chunk)
            pitch = -(-ln // 16) * 16
        elif kind < 0.65:              # pitch < chunk
            pitch = rng.randint(1, chunk - 1)
            ln, rows = rng.randint(1, pitch), rng.randint(2, 40)
        else:                          # pitch > chunk
            pitch = rng.randint(chunk + 1, 6 * chunk)
            ln, rows = rng.randint(1, pitch), rng.randint(2, 12)
        base = rng.randint(0, 4 * chunk)
        end = base + (rows - 1) * pitch + ln
        K = -(-end // chunk) + 2
        for c in range(K):
            n = chunk if rng.random() < 0.9 else rng.randint(1, chunk)
            assert box_meets((base, rows, pitch, ln), c * chunk, n) == brute_meets((base, rows, pitch, ln), c * chunk, n), \
                (base, rows, pitch, ln, c, chunk, n)


# ---- the sub-stream reader against the oracle ----
def _stream(t: torch.Tensor, chunk: int):
    from oracle import oracle as O
    from zipnn_b200 import ZipNN
    plan = ZipNN(input_format="torch", compression_chunk=chunk).plan(t)
    raw = t.contiguous().view(torch.uint8).numpy().reshape(-1)
    s = O.zipnn_compress(plan["header"], raw, plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], plan["chunk"],
                         plan["threshold"], threads=2)
    return s, raw, plan


def _tensors():
    g = torch.Generator().manual_seed(9)
    bf = (torch.randn(50_001, generator=g) * 0.02).to(torch.bfloat16)
    bf[10_000:30_000] = 0                         # whole chunks of zeros: RLE planes
    f32 = (torch.randn(3, 7_001, generator=g) * 0.02).to(torch.float32)
    f32[1] = 0
    f8 = (torch.randn(90_001, generator=g) * 0.5).to(torch.float8_e4m3fn)
    f8[:20_000] = 0
    return {"bf16": bf, "fp32": f32, "fp8": f8}


@pytest.mark.parametrize("name", ["bf16", "fp32", "fp8"])
def test_substream_reader_matches_the_oracle(name, tmp_path, monkeypatch):
    from oracle import oracle as O
    t = _tensors()[name]
    stream, raw, plan = _stream(t, 4096)
    path = tmp_path / "s.bin"
    pad = 123                                     # the stream sits inside a larger file, as in a safetensors file
    path.write_bytes(b"x" * pad + stream.tobytes() + b"y" * 77)
    reads = []
    orig_read, orig_into = FileSource.read, FileSource.read_into
    monkeypatch.setattr(FileSource, "read", lambda self, off, n: (reads.append((off, n)), orig_read(self, off, n))[1])
    monkeypatch.setattr(FileSource, "read_into", lambda self, off, mv: (reads.append((off, len(mv))), orig_into(self, off, mv))[1])
    fd = os.open(path, os.O_RDONLY)
    try:
        idx = StreamIndex(FileSource(fd, pad, stream.size))
        assert idx.chunk == plan["chunk"] and idx.G == plan["num_buf"]
        assert sum(n for _, n in reads) == idx.after + 9 * idx.G * idx.K       # header + tables, nothing more
        n, chunk, K = idx.n, idx.chunk, idx.K
        assert n % chunk and K > 6
        mem = StreamIndex(MemorySource(stream))
        rng = random.Random(3)
        ranges = [(0, K), (0, 1), (K - 1, K), (2, 5)] + [tuple(sorted(rng.sample(range(K + 1), 2))) for _ in range(6)]
        for k0, k1 in ranges:
            if k1 <= k0:
                continue
            reads.clear()
            m = idx.substream_len(k0, k1)
            sub = np.zeros(m, dtype=np.uint8)
            idx.read_substream(FileSource(fd, pad, stream.size), k0, k1, sub)
            lo = idx.cum[:, k0 - 1].astype(np.int64) if k0 else np.zeros(idx.G, dtype=np.int64)
            covered = int((idx.cum[:, k1 - 1].astype(np.int64) - lo).sum())
            assert sum(n for _, n in reads) == covered                          # only the covered payload
            sub_mem = np.zeros(m, dtype=np.uint8)
            mem.read_substream(MemorySource(stream), k0, k1, sub_mem)
            assert np.array_equal(sub, sub_mem)
            a, b = k0 * chunk, min(n, k1 * chunk)
            assert idx.substream_orig(k0, k1) == b - a
            dec = O.zipnn_decompress(sub, idx.G, idx.bits_mode, idx.bytes_mode, chunk, b - a)
            assert np.array_equal(dec, raw[a:b]), (k0, k1)
            part = raw[a:b]
            want = O.zipnn_compress(plan["header"], part, plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], chunk,
                                    plan["threshold"], threads=2)
            assert np.array_equal(want[len(plan["header"]):], sub), (k0, k1)   # the oracle's own stream of those bytes
    finally:
        os.close(fd)


def test_rle_planes_are_covered():
    stream, _, _ = _stream(_tensors()["bf16"], 4096)
    idx = StreamIndex(MemorySource(stream))
    hi = idx.cum.astype(np.int64)
    sizes = np.diff(np.concatenate([np.zeros((idx.G, 1), dtype=np.int64), hi], axis=1), axis=1)
    assert ((idx.types == 1) & (sizes == 1)).any()    # some item is an RLE byte


def test_slices_reject_streaming_frames():
    from zipnn_b200 import ZipNN
    from zipnn_b200.util_torch import zipnn_pack_shape
    z = ZipNN(input_format="torch")
    h = bytearray(z._header)
    h[13] = 128 + 20
    h[15] = 6
    with pytest.raises(ValueError):
        StreamIndex(MemorySource(np.frombuffer(bytes(h) + zipnn_pack_shape((4,)), dtype=np.uint8)))


def test_safe_open_slices_default_and_patch_is_picklable():
    import pickle
    from zipnn_b200 import safetensors_io
    p = pickle.loads(pickle.dumps(safetensors_io._zipnn_safetensors_slices))
    assert p.func is safetensors_io._zipnn_safetensors and p.keywords == {"slices": True}
    import inspect
    assert inspect.signature(safetensors_io.SafeOpen).parameters["slices"].default is False
    _ = slicing
