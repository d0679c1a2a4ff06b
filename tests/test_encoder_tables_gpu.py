"""The device encoder on the crafted cases of encoder_tables.py: every path writes the oracle's stream byte for byte.

Per layout, every case goes through zipnn_b200_compress (a regular, a ragged and a chunk < 64 * G case with d_out at
every offset 0-15 from a 256-byte-aligned base, the rest at offset 0), zipnn_b200_compress_batch (all cases of all
layouts in one call, at the default routing limit and with it lowered) and zipnn_b200_compress_host (a subset, in one
pass and in slabs of three chunks).  Outputs land in canary-filled buffers and inputs must come back unchanged.  Each
coded block is compared with HUF_compress of its plane first, so that a failure names the chunk and group.

The streams the device wrote are then parsed, and the test asserts what they covered: every residue mod 4 of each
bitstream's start address under both write kernels, every residue mod 32 of the bitstreams' bit totals, every
residue mod 16 of the raw planes' destinations, table logs 5-11, both weight-header forms and a full emission tile of
11-bit codes in both write kernels.  Every stream is decoded once by each decoder family as a round-trip check.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import encoder_tables as ET
from oracle import oracle as O
from zipnn_b200 import _native

pytestmark = pytest.mark.gpu

CANARY = 0xA5
PAD = 64
OFFSETS = range(16)
IDS = [f"G{G}b{b}" for G, b in ET.LAYOUTS]


def _stream():
    return torch.cuda.current_stream().cuda_stream


@functools.lru_cache(maxsize=None)
def layout_cases(G, bits):
    cs = ET.cases(G, bits)
    for c in cs:
        c.want = c.oracle()
    return cs


def _ref_block(plane, cap):
    L = O.ref_cdll()
    return O.ref_huf_compress(plane, cap) if L is not None else O.huf_compress(plane, cap)


def check_blocks(case, stream):
    """Each coded block of the device's stream against HUF_compress(plane, cap = chunk) (the reference's when built)."""
    for b in ET.parse(stream, case, 0):
        if b.kind != "huf":
            continue
        plane = case.planes[b.c][b.g]
        r, blk = _ref_block(plane, case.chunk)
        got = stream[b.off: b.off + len(blk)].tobytes()
        assert r > 1 and got == blk, f"{case.name}: chunk {b.c} group {b.g} ({case.names[b.c][b.g]}) differs from HUF_compress"


FACTS = {"start4": set(), "bits32": set(), "raw16": set(), "lg": set(), "form": set(), "full11": set()}


def record(case, stream, base):
    for b in ET.parse(stream, case, base):
        if b.kind == "raw" and b.kernel == "warp":
            plen = case.planes[b.c][b.g].size
            FACTS["raw16"] |= {(b.off + q * (plen // 4)) % 16 for q in range(4)}
        if b.kind != "huf":
            continue
        FACTS["start4"] |= {(b.kernel, q, s % 4) for q, s in enumerate(b.starts)}
        FACTS["bits32"] |= {x % 32 for x in b.bits}
        FACTS["lg"].add(b.lg)
        FACTS["form"].add(b.form)
        if b.lg == 11:
            lens = np.zeros(256, np.int64)
            lens[: b.lengths.size] = b.lengths
            tile = 512 if b.kernel == "warp" else 4096
            if ET.full_tiles_of(case.planes[b.c][b.g], lens, tile, 11):
                FACTS["full11"].add(b.kernel)


def compress(case, d_in, offset):
    """zipnn_b200_compress into a canary-filled buffer at 256-byte-aligned base + offset -> (stream, base address)."""
    n = case.data.size
    bound = _native.compress_bound(n, case.G, case.chunk, 32)
    buf = torch.full((256 + PAD + bound + PAD + 16,), CANARY, dtype=torch.uint8, device="cuda")
    lead = (-buf.data_ptr()) % 256 + 256
    at = lead + offset
    ws = torch.empty(_native.compress_workspace_size(n, case.G, case.chunk), dtype=torch.uint8, device="cuda")
    out_len = C.c_size_t(0)
    hb = C.create_string_buffer(ET.header(), 32)
    rc = _native.lib().zipnn_b200_compress(d_in.data_ptr(), n, hb, 32, case.G, case.bits, ET.bytes_mode(case.G), case.chunk,
                                           case.thr, buf.data_ptr() + at, bound, C.byref(out_len), ws.data_ptr(), ws.numel(),
                                           _stream())
    assert rc == 0, (case.name, rc)
    host = buf.cpu().numpy()
    ln = out_len.value
    assert np.all(host[:at] == CANARY) and np.all(host[at + ln:] == CANARY), f"{case.name}@{offset}: wrote outside the stream"
    return host[at: at + ln], buf.data_ptr() + at


@pytest.mark.parametrize("layout", ET.LAYOUTS, ids=IDS)
def test_compress_matches_oracle(layout):
    cases = layout_cases(*layout)
    aligned = {c.kind: c for c in cases[::-1]}   # one regular, one ragged, one chunk < 64 * G case at every offset
    for case in cases:
        d_in = torch.from_numpy(case.data.copy()).cuda()
        for off in (OFFSETS if aligned.get(case.kind) is case else (0,)):
            got, base = compress(case, d_in, off)
            if off == 0:
                check_blocks(case, got)
            assert np.array_equal(got, case.want), f"{case.name}@{off}: stream != oracle"
            record(case, got, base)
        assert np.array_equal(d_in.cpu().numpy(), case.data), f"{case.name}: the encoder changed its input"


def _batch(cases, max_chunks, monkeypatch):
    if max_chunks:
        monkeypatch.setenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", str(max_chunks))
    else:
        monkeypatch.delenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", raising=False)
    L = _native.lib()
    items = (_native.CompressItem * len(cases))()
    hb = C.create_string_buffer(ET.header(), 32)
    d_ins = [torch.from_numpy(c.data.copy()).cuda() for c in cases]
    offs, at = [], PAD
    for it, c, d in zip(items, cases, d_ins):
        it.d_in, it.n, it.h_hdr, it.hdr_len = d.data_ptr(), c.data.size, C.cast(hb, C.c_void_p), 32
        it.num_buf, it.bits_mode, it.bytes_mode, it.chunk, it.threshold = c.G, c.bits, ET.bytes_mode(c.G), c.chunk, c.thr
        it.out_cap = _native.compress_bound(c.data.size, c.G, c.chunk, 32)
        offs.append(at + (len(offs) % 16))
        at = offs[-1] + it.out_cap + PAD
    out = torch.full((at + 16,), CANARY, dtype=torch.uint8, device="cuda")
    for it, o in zip(items, offs):
        it.d_out = out.data_ptr() + o
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_compress_batch_workspace_size(items, len(cases), C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    lens = (C.c_size_t * len(cases))()
    before = _native.launch_count()
    assert L.zipnn_b200_compress_batch(items, len(cases), lens, ws.data_ptr(), ws.numel(), _stream()) == 0
    launches = _native.launch_count() - before
    host = out.cpu().numpy()
    prev = 0
    for c, o, ln, d in zip(cases, offs, lens, d_ins):
        assert np.all(host[prev: o] == CANARY), f"{c.name}: wrote before its stream"
        assert np.array_equal(host[o: o + ln], c.want), f"{c.name}: batch stream != oracle"
        assert np.array_equal(d.cpu().numpy(), c.data), f"{c.name}: the encoder changed its input"
        prev = o + ln
    assert np.all(host[prev:] == CANARY), "wrote past the last stream"
    return launches


def test_batch_matches_oracle(monkeypatch):
    cases = [c for G, b in ET.LAYOUTS for c in layout_cases(G, b)]
    # three byte-group classes, each with general-write work (the ragged and chunk < 64 * G cases): 5 launches each
    assert _batch(cases, 0, monkeypatch) == 3 * 5
    K = [-(-c.data.size // c.chunk) for c in cases]
    assert any(k > 4 for k in K) and any(k <= 4 for k in K)
    _batch(cases, 4, monkeypatch)   # tensors of more than 4 chunks take the single-tensor launches


@pytest.mark.parametrize("layout", [(1, 0), (2, 1), (4, 1)], ids=["G1b0", "G2b1", "G4b1"])
@pytest.mark.parametrize("slab", [None, 3])
def test_compress_host_matches_oracle(layout, slab, monkeypatch):
    cases = [c for c in layout_cases(*layout) if c.kind != "regular" or c.name.startswith("mid2")]
    for c in cases:
        if slab:
            monkeypatch.setenv("ZIPNN_B200_HOST_SLAB_BYTES", str(slab * c.chunk))
        else:
            monkeypatch.delenv("ZIPNN_B200_HOST_SLAB_BYTES", raising=False)
        data = np.ascontiguousarray(c.data.copy())
        cap = _native.compress_bound(data.size, c.G, c.chunk, 32)
        out = np.full(cap + PAD, CANARY, np.uint8)
        out_len = C.c_size_t(0)
        hb = C.create_string_buffer(ET.header(), 32)
        rc = _native.lib().zipnn_b200_compress_host(data.ctypes.data, data.size, hb, 32, c.G, c.bits, ET.bytes_mode(c.G),
                                                    c.chunk, c.thr, out.ctypes.data, cap, C.byref(out_len))
        assert rc == 0, (c.name, rc)
        assert np.array_equal(out[: out_len.value], c.want), f"{c.name}: host-path stream != oracle"
        assert np.all(out[cap:] == CANARY) and np.array_equal(data, c.data)


@pytest.mark.parametrize("layout", ET.LAYOUTS, ids=IDS)
@pytest.mark.parametrize("sync_max", ["0", "1000000000"])
def test_streams_round_trip(layout, sync_max, monkeypatch):
    monkeypatch.setenv("ZIPNN_B200_SYNC_MAX", sync_max)
    for c in layout_cases(*layout):
        n = c.data.size
        body = torch.from_numpy(c.want[32:].copy()).cuda()
        out = torch.full((n + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
        ws = torch.empty(_native.decompress_workspace_size(n, c.G, c.chunk), dtype=torch.uint8, device="cuda")
        rc = _native.lib().zipnn_b200_decompress(body.data_ptr(), body.numel(), c.G, c.bits, ET.bytes_mode(c.G), c.chunk, n,
                                                 out[PAD:].data_ptr(), ws.data_ptr(), ws.numel(), _stream(), 1)
        assert rc == 0, (c.name, rc)
        host = out.cpu().numpy()
        assert np.array_equal(host[PAD: PAD + n], c.data), c.name
        assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY)


def test_coverage():
    """What the device wrote in test_compress_matches_oracle covered every alignment and residue named above."""
    if not FACTS["lg"]:   # the compress test was deselected: run its cases here
        for layout in ET.LAYOUTS:
            test_compress_matches_oracle(layout)
    missing = {(k, q, r) for k in ("warp", "general") for q in range(4) for r in range(4)} - FACTS["start4"]
    assert not missing, f"bitstream start residues mod 4 never written: {sorted(missing)}"
    assert FACTS["bits32"] == set(range(32)), sorted(set(range(32)) - FACTS["bits32"])
    assert FACTS["raw16"] == set(range(16)), sorted(set(range(16)) - FACTS["raw16"])
    assert set(range(5, 12)) <= FACTS["lg"], sorted(FACTS["lg"])
    assert FACTS["form"] == {"fse", "nibble"}
    assert FACTS["full11"] == {"warp", "general"}, FACTS["full11"]
