"""The oracle (our C restatement) against the reference: committed golden streams, and what the
compiled reference returned on seeded blocks and streams (tests/golden/ref_checks.json, written by
tests/make_golden_ref_checks.py).  CPU only."""
import hashlib

import numpy as np
import pytest

import chunk_settings as CS
from conftest import golden_stream, load_manifest
from golden_inputs import load_ref_checks, make_input, raw_bytes
from oracle import oracle as O
from zipnn_b200 import ZipNN

CASES = load_manifest()


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.mark.parametrize("rec", CASES, ids=[c["name"] for c in CASES])
def test_port_reproduces_reference_stream(rec):
    data = make_input(rec["input"])
    raw = raw_bytes(data)
    if sha(raw) != rec["input_sha256"]:
        pytest.skip("input generator drifted on this machine (numpy/torch RNG or cast)")
    z = ZipNN(**rec["ctor"])
    plan = z.plan(data if rec["ctor"]["input_format"] == "torch" else raw)
    assert plan["header"][:24].hex() == rec["header_hex"][:48]
    stream = O.zipnn_compress(plan["header"], np.frombuffer(raw, dtype=np.uint8), plan["num_buf"], plan["bit_reorder"],
                              plan["byte_reorder"], plan["chunk"], plan["threshold"], threads=4).tobytes()
    assert len(stream) == rec["stream_len"]
    assert sha(stream) == rec["stream_sha256"]
    gold = golden_stream(rec)
    if gold is not None:
        assert stream == gold
    body = np.frombuffer(stream, dtype=np.uint8)[len(plan["header"]):]
    back = O.zipnn_decompress(body, plan["num_buf"], plan["bit_reorder"], plan["byte_reorder"], plan["chunk"], len(raw), threads=4)
    assert back.tobytes() == raw


def block_inputs():
    """-> [(src, dst capacity)]: the seeded HUF blocks compared with the reference's HUF_compress."""
    rng = np.random.default_rng(3)
    cases = []
    for it in range(300):
        size = int(rng.choice([12, 13, 64, 257, 1500, 4096, 65536, 131072, int(rng.integers(1, 131073))]))
        kind = it % 5
        if kind == 0:
            x = (rng.standard_normal(size) * 0.02).astype(np.float32)
            src = (x.view(np.uint32) >> 23).astype(np.uint8)
        elif kind == 1:
            src = rng.integers(0, 256, size, dtype=np.uint8)
        elif kind == 2:
            k = int(rng.integers(2, 256))
            src = rng.choice(k, size, p=rng.dirichlet(np.ones(k) * rng.uniform(0.01, 1))).astype(np.uint8)
        elif kind == 3:
            src = np.full(size, 7, dtype=np.uint8)
        else:
            src = np.minimum(rng.geometric(rng.uniform(0.02, 0.9), size), 255).astype(np.uint8)
        cases.append((src, 256 * 1024 if it % 2 else 128 * 1024))
    return cases


def stream_inputs():
    """-> [(header, data, G, bits, bytes_mode, chunk)]: the seeded streams compared with the reference's zipnn_core."""
    rng = np.random.default_rng(11)
    cases = []
    for it in range(40):
        G = [1, 2, 4][it % 3]
        bits = (it // 3) % 2
        bm = 220 if G == 4 else 10
        chunk = 128 * 1024 if G == 1 else int(rng.choice([256 * 1024, 65536, 4096]))
        nelem = int(rng.choice([1, 3, 13, 4096, chunk // G + 1, int(rng.integers(1, 200000))]))
        n = nelem * G
        if it % 4 == 3:
            data = rng.integers(0, 256, n, dtype=np.uint8)
        else:
            x = (rng.standard_normal(max(n // 2, 1) + 2) * 0.02).astype(np.float32)
            data = np.ascontiguousarray((x.view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)[:n])
        h = bytearray(32)
        h[0:2] = b"ZN"
        cases.append((h, data, G, bits, bm, chunk))
    return cases


def test_port_matches_compiled_reference_blocks():
    """HUF_compress of the port == the reference's: return code and output bytes."""
    want = load_ref_checks()["huf_blocks"]
    cases = block_inputs()
    assert len(cases) == len(want)
    for (src, cap), w in zip(cases, want):
        assert sha(src) == w["input_sha256"], "the seeded input generator drifted"
        r, out = O.huf_compress(src, cap)
        assert (int(r), sha(out)) == (w["ret"], w["out_sha256"])


def test_port_matches_compiled_reference_streams():
    """zipnn_core of the port == the reference's stream, and the port decodes it back to the input
    (the reference's combine_dtype did too when the golden data was written)."""
    want = load_ref_checks()["streams"]
    cases = stream_inputs()
    assert len(cases) == len(want)
    for (h, data, G, bits, bm, chunk), w in zip(cases, want):
        assert sha(data) == w["input_sha256"], "the seeded input generator drifted"
        o = O.zipnn_compress(h, data, G, bits, bm, chunk, 0.95, threads=2).tobytes()
        assert (len(o), sha(o)) == (w["stream_len"], w["stream_sha256"])
        assert O.zipnn_decompress(np.frombuffer(o[32:], dtype=np.uint8), G, bits, bm, chunk, data.size, threads=2).tobytes() == data.tobytes()


def test_port_matches_compiled_reference_settings():
    """zipnn_core of the port == the reference's stream at every chunk size from G to 2^12 and 2^19-2^21,
    thresholds 0-1.5, and the planes built to sit on the threshold and capacity edges; the port decodes each."""
    want = load_ref_checks()["settings"]
    cases = CS.settings_inputs()
    assert [c["name"] for c in cases] == [w["name"] for w in want]
    h = CS.header()
    for c, w in zip(cases, want):
        G, bits, chunk, data = c["G"], c["bits"], c["chunk"], c["data"]
        bm = 220 if G == 4 else 10
        assert sha(data) == w["input_sha256"], f"the seeded input generator drifted: {c['name']}"
        o = O.zipnn_compress(h, data, G, bits, bm, chunk, c["thr"], threads=4).tobytes()
        assert (len(o), sha(o)) == (w["stream_len"], w["stream_sha256"]), c["name"]
        back = O.zipnn_decompress(np.frombuffer(o[32:], dtype=np.uint8), G, bits, bm, chunk, data.size, threads=4)
        assert back.tobytes() == data.tobytes(), c["name"]


def _types(stream, G, chunk, n):
    K = -(-n // chunk)
    return np.frombuffer(stream, dtype=np.uint8)[32: 32 + G * K]


def test_settings_planes_sit_on_their_edges():
    """The searched planes are what chunk_settings says they are, in the reference's streams (same digests)."""
    h = CS.header()
    by_kind = {}
    for c in CS.settings_inputs(big=False):
        by_kind.setdefault(c["kind"], []).append(c)
    # capacity flips: raw in the stream (destination = plen); an unbounded destination would code every one
    for c in by_kind["capflip"] + [c for c in CS.settings_inputs() if c["kind"] == "capslack"]:
        plen, data = c["plen"], c["data"]
        planes = data.reshape(-1, plen)
        assert all(CS.stored_size(p, plen, c["thr"]) == 0 for p in planes)
        blind = [CS.stored_size(p, 1 << 20, c["thr"]) for p in planes]
        assert all(b > 1 for b in blind), c["name"]
        if c["kind"] == "capslack":
            assert plen - 9 <= blind[0] <= plen - 2
        s = O.zipnn_compress(h, data, 1, 0, 10, plen, c["thr"]).tobytes()
        assert not _types(s, 1, plen, data.size).any()
    # coded size exactly plen * thr: raw, and coded at any higher threshold
    for c in by_kind["exact"]:
        plen, planes = c["plen"], c["data"].reshape(-1, c["plen"])
        for p in planes:
            r, _ = O.huf_compress(p, plen)
            assert r == plen * c["thr"]
            assert CS.stored_size(p, plen, c["thr"]) == 0 and CS.stored_size(p, plen, c["thr"] + 0.01) == r
    # RLE at 2 and 3 bytes: kept exactly when 1 < plen * thr
    for c in by_kind["rle"]:
        G, chunk, data = c["G"], c["chunk"], c["data"]
        s = O.zipnn_compress(h, data, G, c["bits"], 220 if G == 4 else 10, chunk, c["thr"]).tobytes()
        t = _types(s, G, chunk, data.size).reshape(G, -1)
        plen = c["plen"]
        col = t[:, -1] if plen == 3 else t[:, 0]
        assert (col == (1 if 1 < plen * np.float32(c["thr"]) else 0)).all(), c["name"]
