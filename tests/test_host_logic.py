"""Host-side logic that needs no GPU: header/shape packing, dtype dispatch, the C-ABI
library's exports and sizing functions, and the single-thread device routines compiled for
the host (tests/host_emu) against the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import oracle as O
from zipnn_b200 import ZipNN, _native
from zipnn_b200.util_torch import dtype_code, zipnn_pack_shape, zipnn_unpack_shape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_layout_matches_reference_bytes():
    # reference header for ZipNN(method="HUFFMAN", bytearray_dtype="bfloat16") on 2 MiB of bytes
    # (SURVEY.md section 8c): 5a4e0005030a0101 0100000000001206 0000200000000000 ...
    z = ZipNN(method="HUFFMAN", bytearray_dtype="bfloat16")
    plan = z.plan(bytes(2 * 1024 * 1024))
    assert plan["header"][:24].hex() == "5a4e0005030a0101010000000000120600002000" + "00000000"
    assert (plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], plan["chunk"]) == (2, 1, 10, 262144)


@pytest.mark.parametrize("dt,exp", [(torch.float32, (1, 220, 4, 1)), (torch.bfloat16, (1, 10, 2, 6)),
                                    (torch.float16, (0, 10, 2, 4)), (torch.float8_e4m3fn, (1, 10, 1, 29)),
                                    (torch.float8_e5m2, (1, 10, 1, 30))])
def test_dtype_dispatch(dt, exp):
    t = torch.zeros(5, 3).to(dt)
    z = ZipNN(input_format="torch")
    p = z.plan(t)
    assert (p["bit_reorder"], p["byte_reorder"], p["num_buf"], p["header"][15]) == exp
    assert p["header"][32:] == zipnn_pack_shape((5, 3))
    assert p["chunk"] == (131072 if exp[2] == 1 else 262144)


def test_rejects_non_float_and_bad_params():
    with pytest.raises(ValueError):
        ZipNN(input_format="torch").plan(torch.zeros(4, dtype=torch.int32))
    with pytest.raises(ValueError):
        ZipNN(compression_chunk=3000)
    with pytest.raises(ValueError):
        ZipNN(input_format="torch", is_streaming=True)
    with pytest.raises(ImportError):
        ZipNN(method="zstd")
    with pytest.raises(ValueError):
        ZipNN(input_format="byte", bytearray_dtype="uint32").plan(b"1234")


def test_shape_pack_roundtrip():
    for shape in [(), (1,), (255, 256), (65535, 65536, 3), (4294967295,), (4294967296, 2)]:
        packed = zipnn_pack_shape(shape)
        got, used = zipnn_unpack_shape(packed + b"\xff\xff")
        assert got == tuple(shape) and used == len(packed)
    assert dtype_code("float") == 2 and dtype_code("half") == 5 and dtype_code(torch.float) == 1


def test_cabi_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "zipnn_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(zipnn_b200_[a-z0-9_]+)\s*\(", hdr)))
    assert declared, "no declarations parsed"
    _native.build()
    L = C.CDLL(_native.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), name
    assert sorted(_native.EXPORTS) == declared


def test_cabi_sizing_without_gpu():
    assert _native.lib().zipnn_b200_version() == 0x000200
    # worst case: every plane raw -> header + 9 bytes of metadata per (group, chunk) + n
    assert _native.compress_bound(1 << 21, 2, 1 << 18, 34) == 34 + 9 * 2 * 8 + (1 << 21)
    assert _native.compress_bound(0, 2, 1 << 18, 32) == 32
    assert _native.compress_workspace_size(1 << 21, 2, 1 << 18) > 0
    assert _native.decompress_workspace_size(1 << 21, 4, 1 << 18) > 0
    out = C.c_size_t(0)
    assert _native.lib().zipnn_b200_compress_bound(10, 3, 1 << 18, 32, C.byref(out)) == _native.E_ARG
    assert b"corrupt" in _native.lib().zipnn_b200_strerror(_native.E_CORRUPT)


def _emu():
    so = os.path.join(ROOT, "tests", "host_emu", "libemu_serial.so")
    E = C.CDLL(so)
    E.emu_table_from_counts.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    E.emu_read_weights.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    E.emu_block_decision.restype = C.c_uint32
    E.emu_block_decision.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_double]
    return E


def test_device_serial_routines_match_oracle():
    """huf_serial.cuh (what one GPU thread runs) vs the oracle: code lengths, canonical values,
    table description bytes, and the decoder's weight parse of those bytes."""
    E = _emu()
    rng = np.random.default_rng(5)
    forms = set()
    for it in range(600):
        kind = it % 6
        size = int(rng.choice([20, 64, 300, 2000, 32768, 131072, int(rng.integers(13, 131073))]))
        if kind == 0:
            x = (rng.standard_normal(size) * 0.02).astype(np.float32)
            src = (x.view(np.uint32) >> 23).astype(np.uint8)
        elif kind == 1:
            k = int(rng.integers(2, 20))
            src = rng.choice(k, size, p=rng.dirichlet(np.ones(k) * rng.uniform(0.05, 2))).astype(np.uint8)
        elif kind == 2:
            k = int(rng.integers(2, 256))
            src = rng.choice(k, size, p=rng.dirichlet(np.ones(k) * rng.uniform(0.01, 1))).astype(np.uint8)
        elif kind == 3:
            src = np.minimum(rng.geometric(rng.uniform(0.02, 0.9), size), 255).astype(np.uint8)
        elif kind == 4:
            src = (rng.standard_normal(size) * rng.uniform(0.5, 40) + 128).clip(0, 255).astype(np.uint8)
        else:
            src = np.minimum(rng.zipf(rng.uniform(1.1, 3), size), 255).astype(np.uint8)
        cnt = np.bincount(src, minlength=256).astype(np.uint32)
        if (cnt > 0).sum() < 2:
            continue
        nb0, val0, hdr0, log0 = O.huf_table_from_counts(cnt, size)
        nb = np.zeros(256, np.uint8)
        val = np.zeros(256, np.uint16)
        hdr = np.zeros(512, np.uint8)
        lg = C.c_int(0)
        h = E.emu_table_from_counts(cnt.ctypes.data, size, nb.ctypes.data, val.ctypes.data, hdr.ctypes.data, C.byref(lg))
        assert np.array_equal(nb, nb0) and lg.value == log0
        present = cnt > 0
        assert np.array_equal(val[present], val0[present])
        assert (h < 0) == (hdr0 is None)
        if h > 0:
            assert hdr[:h].tobytes() == hdr0
            forms.add("fse" if hdr[0] < 128 else "nibble")
            w = np.zeros(256, np.uint8)
            ns, l2 = C.c_int(0), C.c_int(0)
            buf = np.concatenate([hdr[:h], np.zeros(8, np.uint8)])
            assert E.emu_read_weights(buf.ctypes.data, h, w.ctypes.data, C.byref(ns), C.byref(l2)) == h
            max_sym = int(np.nonzero(cnt)[0][-1])
            expect = np.where(nb > 0, lg.value + 1 - nb.astype(int), 0)[: max_sym + 1]
            assert ns.value == max_sym + 1 and l2.value == lg.value and np.array_equal(w[: max_sym + 1], expect)
    assert forms == {"fse", "nibble"}


def test_device_weight_parser_rejects_garbage():
    E = _emu()
    rng = np.random.default_rng(9)
    w = np.zeros(256, np.uint8)
    ns, lg = C.c_int(0), C.c_int(0)
    for _ in range(2000):
        n = int(rng.integers(1, 140))
        buf = rng.integers(0, 256, n + 8, dtype=np.uint8)
        r = E.emu_read_weights(buf.ctypes.data, n, w.ctypes.data, C.byref(ns), C.byref(lg))
        assert r == -1 or (0 < r <= n and 1 <= lg.value <= 12 and 2 <= ns.value <= 256)



def _device_decision(E, plane: np.ndarray, cap: int, thr: float) -> int:
    """What k_encode_table stores for one plane: its early-outs, then huf_block_decision (huf_serial.cuh)."""
    n = plane.size
    cnt = np.bincount(plane, minlength=256).astype(np.uint32)
    bits = np.zeros(4, np.uint32)
    thr64 = float(np.float32(thr))
    if cnt.max() == n:
        return int(E.emu_block_decision(1, bits.ctypes.data, 0, n, cap, thr64))
    if cnt.max() <= (n >> 7) + 4:
        return 0
    nb = np.zeros(256, np.uint8)
    val = np.zeros(256, np.uint16)
    hdr = np.zeros(512, np.uint8)
    lg = C.c_int(0)
    h = E.emu_table_from_counts(cnt.ctypes.data, n, nb.ctypes.data, val.ctypes.data, hdr.ctypes.data, C.byref(lg))
    seg = (n + 3) // 4
    for q in range(4):
        bits[q] = int(nb[plane[q * seg: min(n, (q + 1) * seg)]].astype(np.int64).sum())
    return int(E.emu_block_decision(0, bits.ctypes.data, h, n, cap, thr64))


def test_block_decision_matches_oracle_with_capacity():
    """huf_block_decision, the raw/RLE/coded rule the encoder runs per plane, against the oracle's HUF_compress
    with the same destination capacity and the threshold.  The capacity is the chunk: the plane itself for one
    byte group, 2x or 4x the plane for two or four; plus an unbounded one.  Every plane chunk_settings built on a
    capacity or threshold edge is included."""
    import chunk_settings as CS
    E = _emu()
    rng = np.random.default_rng(23)
    planes = []
    for it in range(3000):
        plen = int(rng.choice([2, 3, 8, 13, 14, 16, 17, 24, 32, 48, 64, 100, 128, 256, 512, 4096, int(rng.integers(2, 2049))]))
        k = int(rng.integers(1, 81))
        p = rng.dirichlet(np.ones(k) * rng.uniform(0.05, 2.0))
        planes.append((rng.choice(k, plen, p=p).astype(np.uint8), float(rng.choice(CS.THRESHOLDS))))
    edge = [(p, 0.95) for plen in CS.FLIP_PLENS for p in CS.capacity_flip_planes(plen)]
    edge.append((CS.slack_plane(), 1.0))
    edge += [(CS.exact_threshold_plane(plen, thr, s), thr) for thr in (0.5, 0.75) for plen in CS.EXACT_PLENS for s in range(3)]
    flips = 0
    for i, (plane, thr) in enumerate(planes + edge):
        caps = [plane.size, 2 * plane.size, 4 * plane.size, 1 << 20]
        got = [_device_decision(E, plane, cap, thr) for cap in caps]
        want = [CS.stored_size(plane, cap, thr) for cap in caps]
        assert got == want, (i, plane.size, thr, got, want)
        flips += got[0] != got[-1]
    for plane, thr in edge[: len(CS.FLIP_PLENS) * CS.FLIPS_PER_PLEN + 1]:
        assert _device_decision(E, plane, plane.size, thr) == 0 and _device_decision(E, plane, 1 << 20, thr) > 1
    assert flips >= len(CS.FLIP_PLENS) * CS.FLIPS_PER_PLEN + 1
