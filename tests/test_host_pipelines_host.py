"""Host side of the host-memory pipeline tests (test_host_pipelines_gpu.py): models of the branches the host entry
points take, the plane-built inputs the GPU tests use, and the identity every one of those paths rests on, checked
on the oracle alone.

The paths that start in host memory all cut a stream into chunk ranges:
  * zipnn_b200_decompress_host decodes a large stream in slabs of `per` chunks on two CUDA streams (api_host.inc,
    decompress_host_slabs), rebasing each slab's size rows on the host;
  * zipnn_b200_compress_host compresses slab by slab and assembles the stream from the per-slab streams
    (compress_host_slabs); groups 1..G-1 leave for the caller's buffer early, on the bet that every group in front
    of them stays raw, and are copied again at the end when the bet is lost;
  * ZipNN streaming frames (`is_streaming=True`) are cut from the stream of the whole input
    (`_compress_frames_at_once`) and decoded by one batch call (`_decompress_frames_at_once`), or frame by frame.
The identity: a chunk range [c0, c1) of a stream, with its type rows cut and its cumulative size rows rebased to
the range, and its payload slices of each group, is the stream of the input bytes [c0*chunk, min(n, c1*chunk)).
The models here say which branch a GPU case takes, so that every case asserts it reaches the branch it was built
for.
"""
from __future__ import annotations

import numpy as np
import pytest

import plane_inputs as P
from oracle import oracle as O

KNOB = "ZIPNN_B200_HOST_SLAB_BYTES"
DEFAULT_SLABS = {"decode": 256 << 20, "encode": 128 << 20}   # HostKnobs in api_host.inc
DEFAULT_PIPELINE_MIN = 64 << 20
HUF_MAX_BLOCK = 128 * 1024
OK, E_CAPACITY, E_CORRUPT = 0, 2, 3
BYTES_MODE = {1: 10, 2: 10, 4: 220}


def header32(orig: int = 0) -> bytes:
    h = bytearray(32)
    h[0:2] = b"ZN"
    h[16:24] = int(orig).to_bytes(8, "little")
    return bytes(h)


# ------------------------------------------------------------------ slab partition (host_knobs, *_host_slabs)
class SlabPlan:
    __slots__ = ("piped", "per", "nslabs", "ragged_last", "bufset", "ranges", "K", "slab")

    def edges(self):
        """The first chunk of every slab but the first."""
        return [c0 for c0, _ in self.ranges[1:]]


def slab_plan(n: int, chunk: int, knob: int | None = None, kind: str = "decode") -> SlabPlan:
    """What the host call does for n input (compress) or output (decompress) bytes with ZIPNN_B200_HOST_SLAB_BYTES
    = knob (None or <= 0: the defaults).  bufset[i] is the buffer set / CUDA stream slab i uses (i & 1)."""
    if knob is not None and knob > 0:
        slab = pipeline_min = knob
    else:
        slab, pipeline_min = DEFAULT_SLABS[kind], DEFAULT_PIPELINE_MIN
    p = SlabPlan()
    p.slab = slab
    p.K = -(-n // chunk)
    p.piped = n >= pipeline_min and n > slab
    p.per = max(1, slab // chunk)
    p.nslabs = -(-p.K // p.per)
    p.ragged_last = p.K % p.per != 0
    p.bufset = [i & 1 for i in range(p.nslabs)]
    p.ranges = [(i * p.per, min(p.K, (i + 1) * p.per)) for i in range(p.nslabs)]
    return p


# ------------------------------------------------------------------ stream tables
def tables(stream: np.ndarray, hdr_len: int, G: int, K: int):
    """-> (types[G, K], cum[G, K] int64, payload0, group bases relative to payload0)."""
    s = np.asarray(stream, dtype=np.uint8)
    types = s[hdr_len: hdr_len + G * K].reshape(G, K)
    cum = s[hdr_len + G * K: hdr_len + 9 * G * K].copy().view("<u8").reshape(G, K).astype(np.int64)
    base = np.concatenate([[0], np.cumsum(cum[:, -1])[:-1]]).astype(np.int64)
    return types, cum, hdr_len + 9 * G * K, base


def sizes(cum: np.ndarray) -> np.ndarray:
    return np.diff(np.concatenate([np.zeros((cum.shape[0], 1), np.int64), cum], axis=1), axis=1)


def chunk_kinds(stream, hdr_len: int, G: int, chunk: int, n: int):
    """kind[g][c]: 'raw' (stored), 'rle' (one byte) or 'huf' (a HUF block), as the decoders read the stream."""
    K = -(-n // chunk)
    types, cum, _, _ = tables(stream, hdr_len, G, K)
    sz = sizes(cum)
    out = [[None] * K for _ in range(G)]
    for c in range(K):
        clen = min(chunk, n - c * chunk)
        for g in range(G):
            dec = P.plane_len(clen, G, g)
            out[g][c] = "raw" if types[g, c] == 0 or sz[g, c] == dec or dec == 0 else "rle" if sz[g, c] == 1 else "huf"
    return out


def chunk_class(kinds, c: int) -> str:
    """One word per chunk: raw (every group stored), rle (no group coded, one or more RLE), one / two (coded
    groups)."""
    col = [kinds[g][c] for g in range(len(kinds))]
    nh = col.count("huf")
    if nh:
        return "one" if nh == 1 else "two"
    return "rle" if "rle" in col else "raw"


# ------------------------------------------------------------------ the identity: a chunk range is a stream
def sub_stream(stream, hdr_len: int, G: int, chunk: int, n: int, c0: int, c1: int) -> np.ndarray:
    """The stream of chunks [c0, c1): header with the range's original length at [16:24] and its total length at
    [24:32], the cut type rows, the rebased size rows and each group's payload slice."""
    s = np.asarray(stream, dtype=np.uint8)
    K = -(-n // chunk)
    types, cum, payload0, base = tables(s, hdr_len, G, K)
    lo = cum[:, c0 - 1] if c0 else np.zeros(G, np.int64)
    hi = cum[:, c1 - 1]
    hdr = bytearray(s[:hdr_len].tobytes())
    hdr[16:24] = int(min(n, c1 * chunk) - c0 * chunk).to_bytes(8, "little")
    hdr[24:32] = int(hdr_len + 9 * G * (c1 - c0) + int((hi - lo).sum())).to_bytes(8, "little")
    parts = [bytes(hdr), np.ascontiguousarray(types[:, c0:c1]).tobytes(),
             (cum[:, c0:c1] - lo.reshape(G, 1)).astype("<u8").tobytes()]
    for g in range(G):
        a = payload0 + int(base[g])
        parts.append(s[a + int(lo[g]): a + int(hi[g])].tobytes())
    return np.frombuffer(b"".join(parts), dtype=np.uint8)


# ------------------------------------------------------------------ plane-built inputs
PLANE = {"raw": P.uniform, "rle": P.constant(3), "huf": P.geometric(0.5)}


def planned_bytes(pattern, G: int, bits: int, chunk: int, n: int, seed: int) -> np.ndarray:
    """Input bytes whose chunk c has, in group g, a plane of kind pattern[c % len(pattern)][g]."""
    rng = np.random.default_rng(seed)
    chunks = []
    for c in range(-(-n // chunk)):
        clen = min(chunk, n - c * chunk)
        kinds = pattern[c % len(pattern)]
        chunks.append([PLANE[kinds[g]](rng, P.plane_len(clen, G, g)) for g in range(G)])
    return P.tensor_from_planes(chunks, G, bits)


def intended(pattern, G: int, chunk: int, n: int):
    """kind[g][c] the pattern asks for.  A plane of under 64 bytes is not asked to code; one past 128 KiB (a HUF
    block's limit) is stored raw."""
    K = -(-n // chunk)
    out = [[None] * K for _ in range(G)]
    for c in range(K):
        clen = min(chunk, n - c * chunk)
        for g in range(G):
            k = pattern[c % len(pattern)][g]
            plen = P.plane_len(clen, G, g)
            out[g][c] = "raw" if plen > HUF_MAX_BLOCK else k if plen >= 64 else None
    return out


def realised(pattern, stream, hdr_len: int, G: int, chunk: int, n: int) -> bool:
    got = chunk_kinds(stream, hdr_len, G, chunk, n)
    want = intended(pattern, G, chunk, n)
    return all(w is None or w == k for gw, gk in zip(want, got) for w, k in zip(gw, gk))


# Chunk patterns for the slab decoder: raw, RLE, single-coded and two-coded-group chunks in an order that puts
# every class on both sides of a slab edge for per = 1, 2 and 3.
DECODE_PATTERN = {
    1: [("huf",), ("raw",), ("rle",), ("huf",), ("huf",), ("rle",), ("raw",), ("raw",), ("huf",), ("rle",), ("rle",)],
    2: [("raw", "huf"), ("huf", "huf"), ("raw", "raw"), ("rle", "huf"), ("raw", "rle"), ("huf", "raw"), ("rle", "rle"),
        ("huf", "huf"), ("raw", "raw"), ("raw", "huf"), ("rle", "raw")],
    4: [("raw", "raw", "raw", "huf"), ("rle", "rle", "huf", "huf"), ("raw", "raw", "raw", "raw"),
        ("raw", "huf", "raw", "huf"), ("rle", "raw", "rle", "raw"), ("huf", "raw", "raw", "raw"),
        ("rle", "rle", "rle", "rle"), ("huf", "raw", "huf", "raw"), ("raw", "raw", "raw", "raw"),
        ("raw", "rle", "raw", "huf"), ("rle", "rle", "huf", "rle")],
}


# The slab decoder's layouts: (G, bits_mode, chunk, n), each decoded with the knobs of decode_knobs(chunk).
DECODE_LAYOUTS = {
    "bf16": (2, 1, 65536, 10 * 65536 + 32768 + 6),
    "bf16_256k": (2, 1, 262144, 7 * 262144 + 1234),
    "fp16": (2, 0, 4096, 11 * 4096),
    "fp32": (4, 1, 262144, 9 * 262144 + 1000),
    "fp8": (1, 0, 131072, 10 * 131072 + 77),
}


def decode_knobs(chunk: int):
    """Slab knobs: below one chunk (per = 1), one chunk, 3*chunk - 1 (per = 2, not a multiple), 3*chunk."""
    return [chunk // 2, chunk, 3 * chunk - 1, 3 * chunk]


def edge_pairs(classes, plan: SlabPlan):
    """(class left of the edge, class right of it) for every slab edge."""
    return {(classes[e - 1], classes[e]) for e in plan.edges()}


# ------------------------------------------------------------------ decode: the host-side checks
def decode_host_check(body, G: int, chunk: int, orig: int, per: int):
    """Where decompress_host_slabs rejects the stream on the host: ('ok', None) when the host checks pass (the
    device then sees the rest), ('short' | 'room', None) before any work is enqueued, or ('row', i) when slab i's
    rows fail (a decreasing row, a slab larger than slab_max, planes larger than the slab) with slabs 0..i-1
    already enqueued."""
    b = np.asarray(body, dtype=np.uint8)
    K = -(-orig // chunk)
    if b.size < 9 * G * K:
        return "short", None
    _, cum, payload0, _ = tables(b, 0, G, K)
    u = cum.astype(np.uint64)
    room = b.size - payload0
    for g in range(G):
        tot = int(u[g, K - 1])
        if tot > room:
            return "room", None
        room -= tot
    slab_max, tables_max = per * chunk, 9 * G * per
    for i, c0 in enumerate(range(0, K, per)):
        c1 = min(K, c0 + per)
        total = 0
        for g in range(G):
            lo = int(u[g, c0 - 1]) if c0 else 0
            hi = int(u[g, c1 - 1])
            if hi < lo or hi - lo > slab_max:
                return "row", i
            total += hi - lo
        if total > slab_max + tables_max:
            return "row", i
    return "ok", None


# ------------------------------------------------------------------ encode: the early bet (compress_host_slabs)
def bet_model(stream, hdr_len: int, G: int, chunk: int, n: int, per: int, out_cap: int) -> dict:
    """Replays compress_host_slabs on the final stream's rows.  -> {
        status: OK / E_CAPACITY, site: None, 'payload0', ('g0', slab) or 'final',
        taken[g]: the group's early copy bet was taken at slab 0 (g >= 1),
        lost[g]: slab at which a taken bet was lost (a group in front turned non-raw), or None,
        skipped: [(g, slab)] early copies skipped because they would pass out_cap,
        copies: [(g, slab, dst, len, phase)] device-to-host payload copies in the order they are queued,
                phase "early" during the slab loop, "late" after it,
        late[g]: the group is copied again at the end (g >= 1), out_len }."""
    K = -(-n // chunk)
    types, cum, payload0, _ = tables(stream, hdr_len, G, K)
    sz = sizes(cum)
    res = dict(status=OK, site=None, taken={}, lost={g: None for g in range(1, G)}, skipped=[], copies=[], late={},
               out_len=None)
    if out_cap < payload0:
        return dict(res, status=E_CAPACITY, site="payload0")
    pred_base, at = [], payload0
    for g in range(G):
        pred_base.append(at)
        at += n // G + (1 if g < n % G else 0)
    all_raw = [True] * G
    early = [False] * G
    run = [0] * G
    nslabs = -(-K // per)
    before = []
    for i in range(nslabs):
        c0, c1 = i * per, min(K, (i + 1) * per)
        tot = [int(sz[g, c0:c1].sum()) for g in range(G)]
        before.append(list(run))
        for g in range(G):
            if types[g, c0:c1].any():
                all_raw[g] = False
        for g in range(G):
            front_raw = all(all_raw[:g])
            if g and not front_raw:
                if early[g] and res["lost"][g] is None:
                    res["lost"][g] = i
                early[g] = False
                continue
            a = pred_base[g] + run[g]
            if a + tot[g] > out_cap:
                if g == 0:
                    return dict(res, status=E_CAPACITY, site=("g0", i))
                res["skipped"].append((g, i))
                early[g] = False
                continue
            if i == 0:
                early[g] = True
                if g:
                    res["taken"][g] = True
            if tot[g] and (g == 0 or early[g]):
                res["copies"].append((g, i, a, tot[g], "early"))
        for g in range(G):
            run[g] += tot[g]
    base, total = [], payload0
    for g in range(G):
        base.append(total)
        total += run[g]
    for g in range(1, G):
        res["taken"].setdefault(g, False)
    if total > out_cap:
        return dict(res, status=E_CAPACITY, site="final")
    for g in range(1, G):
        res["late"][g] = not (early[g] and base[g] == pred_base[g])
        if res["late"][g]:
            for i in range(nslabs):
                c0, c1 = i * per, min(K, (i + 1) * per)
                t = int(sz[g, c0:c1].sum())
                if t:
                    res["copies"].append((g, i, base[g] + before[i][g], t, "late"))
    return dict(res, out_len=total)


# ------------------------------------------------------------------ streaming frames (zipnn.py)
def frame_paths(n: int, G: int, compression_chunk: int, streaming_chunk: int) -> dict:
    """{compress: 'at_once' | 'loop', decompress: 'batch' | 'fallback', frames: [(offset, length)]}: compress
    cuts frames from one stream of the whole input when a frame is a whole number of chunks; decompress decodes
    every frame by one batch call unless a frame's output would start off a 16-byte boundary (then frame by frame)."""
    chunk = compression_chunk if G != 1 else min(HUF_MAX_BLOCK, compression_chunk)
    comp = "at_once" if n and streaming_chunk % chunk == 0 and streaming_chunk >= chunk else "loop"
    frames = [(o, min(streaming_chunk, n - o)) for o in range(0, n, streaming_chunk)]
    dec = "fallback" if any(o % 16 for o, _ in frames) else "batch"
    return dict(compress=comp, decompress=dec, frames=frames, chunk=chunk)


# ================================================================== tests of the models
def test_slab_partition():
    p = slab_plan(7 * 4096 - 5, 4096, 2048)
    assert p.piped and p.per == 1 and p.nslabs == 7 and not p.ragged_last and p.bufset == [0, 1, 0, 1, 0, 1, 0]
    p = slab_plan(7 * 4096 - 5, 4096, 3 * 4096 - 1)
    assert p.piped and p.per == 2 and p.nslabs == 4 and p.ragged_last and p.ranges[-1] == (6, 7)
    p = slab_plan(6 * 4096, 4096, 3 * 4096)
    assert p.piped and p.per == 3 and p.nslabs == 2 and not p.ragged_last and p.bufset == [0, 1]
    # at the threshold: n == knob is not piped (n > slab), n == knob + 1 is
    assert not slab_plan(3 * 4096, 4096, 3 * 4096).piped
    assert slab_plan(3 * 4096 + 1, 4096, 3 * 4096).piped
    # defaults: 64 MiB minimum, slabs of 256 MiB (decode) / 128 MiB (encode)
    assert not slab_plan(200 << 20, 262144, None, "decode").piped
    assert slab_plan(200 << 20, 262144, None, "encode").piped
    assert not slab_plan(100 << 20, 262144, 0, "encode").piped


def test_bet_model_on_hand_built_rows():
    """bf16-like G=2 rows, per = 2, four slabs: group 0 turns coded in slab 2 -> group 1's bet is lost there."""
    G, chunk, K, hdr = 2, 4096, 8, 32
    n = K * chunk
    types = np.zeros((G, K), np.uint8)
    sz = np.full((G, K), chunk // 2, np.int64)
    types[1, :] = 1
    sz[1, :] = 700
    types[0, 5] = 1
    sz[0, 5] = 900
    cum = np.cumsum(sz, axis=1)
    body = types.tobytes() + cum.astype("<u8").tobytes()
    stream = np.frombuffer(header32(n) + body + bytes(int(sz.sum())), np.uint8)
    m = bet_model(stream, hdr, G, chunk, n, 2, stream.size)
    assert m["status"] == OK and m["taken"] == {1: True} and m["lost"] == {1: 2} and m["late"] == {1: True}
    assert m["out_len"] == stream.size
    # the early copies of slabs 0 and 1 went to the predicted base; the late ones to the real one
    payload0 = hdr + 9 * G * K
    early = [c for c in m["copies"] if c[0] == 1 and c[4] == "early"]
    assert [c[1] for c in early] == [0, 1] and all(c[2] >= payload0 + n // 2 for c in early)
    assert [c[1] for c in m["copies"] if c[0] == 1 and c[4] == "late"] == [0, 1, 2, 3]
    assert m["skipped"] == []
    assert bet_model(stream, hdr, G, chunk, n, 2, stream.size - 1)["site"] == "final"
    assert bet_model(stream, hdr, G, chunk, n, 2, payload0 - 1)["site"] == "payload0"
    assert bet_model(stream, hdr, G, chunk, n, 2, payload0 + 2 * chunk // 2 + 1)["site"] == ("g0", 1)
    # all raw in front: the bet holds and group 1 is not copied again
    types[0, 5], sz[0, 5] = 0, chunk // 2
    cum = np.cumsum(sz, axis=1)
    stream = np.frombuffer(header32(n) + types.tobytes() + cum.astype("<u8").tobytes() + bytes(int(sz.sum())), np.uint8)
    m = bet_model(stream, hdr, G, chunk, n, 2, stream.size)
    assert m["lost"] == {1: None} and m["late"] == {1: False}


def test_decode_host_check_model():
    G, chunk, n = 2, 4096, 7 * 4096 - 5
    data = planned_bytes(DECODE_PATTERN[2], G, 1, chunk, n, 3)
    s = O.zipnn_compress(header32(n), data, G, 1, 10, chunk)
    body = s[32:].copy()
    K = 7
    assert decode_host_check(body, G, chunk, n, 2) == ("ok", None)
    cum = body[G * K: 9 * G * K].view("<u8").reshape(G, K)
    bad = body.copy()
    bcum = bad[G * K: 9 * G * K].view("<u8").reshape(G, K)
    bcum[1, K - 1] = cum[1, 5] - 1        # decreases across the edge into the last slab (chunks 6..6)
    assert decode_host_check(bad, G, chunk, n, 2) == ("row", 3)
    assert decode_host_check(body[:-1], G, chunk, n, 2) == ("room", None)
    assert decode_host_check(body[: 9 * G * K - 1], G, chunk, n, 2) == ("short", None)


def test_frame_paths():
    assert frame_paths(3 << 20, 2, 262144, 1 << 20)["compress"] == "at_once"
    assert frame_paths(3 << 20, 2, 262144, 131072)["compress"] == "loop"
    assert frame_paths(3 << 20, 1, 262144, 131072)["compress"] == "at_once"     # fp8 codes 128 KiB chunks
    assert frame_paths(100, 2, 4096, 8)["decompress"] == "fallback"
    assert frame_paths(8, 2, 4096, 8)["decompress"] == "batch"                   # one frame starts at 0
    assert frame_paths(0, 2, 4096, 4096)["compress"] == "loop"
    f = frame_paths(5 * 4096 + 7, 4, 4096, 2 * 4096)
    assert f["frames"] == [(0, 8192), (8192, 8192), (16384, 4103)] and f["decompress"] == "batch"


def test_decode_cases_cover_the_slab_edges():
    """Across its four slab knobs, every decode layout has odd and even slab counts, a ragged last slab, and every
    chunk class on both sides of a slab edge; the layouts together have ragged and whole last chunks."""
    ragged_chunk = set()
    for name, (G, bits, chunk, n) in DECODE_LAYOUTS.items():
        K = -(-n // chunk)
        classes = [chunk_class(intended(DECODE_PATTERN[G], G, chunk, n), c) for c in range(K)]
        want = {"raw", "rle", "one"} | ({"two"} if G > 1 else set())
        pairs, counts, ragged = set(), set(), False
        for knob in decode_knobs(chunk):
            p = slab_plan(n, chunk, knob)
            assert p.piped, (name, knob)
            pairs |= edge_pairs(classes, p)
            counts.add(p.nslabs % 2)
            ragged |= p.ragged_last
        assert {a for a, _ in pairs} >= want and {b for _, b in pairs} >= want, name
        assert counts == {0, 1} and ragged, name
        assert [slab_plan(n, chunk, k).per for k in decode_knobs(chunk)] == [1, 1, 2, 3]
        ragged_chunk.add(n % chunk != 0)
    assert ragged_chunk == {True, False}


# ------------------------------------------------------------------ the identity on the oracle alone
IDENTITY = [(G, chunk) for G in (1, 2, 4) for chunk in sorted({G, 64, 512, 4096, 65536, 262144})]


@pytest.mark.parametrize("G,chunk", IDENTITY)
def test_chunk_range_is_a_stream(G, chunk):
    bits = 0 if G == 1 else 1
    K = 11
    n = K * chunk - (chunk // 2 if chunk >= 4 * G else 0)        # a ragged last chunk where the chunk allows one
    pattern = DECODE_PATTERN[G]
    data = planned_bytes(pattern, G, bits, chunk, n, seed=G * 1000 + chunk % 997)
    whole = O.zipnn_compress(header32(n), data, G, bits, BYTES_MODE[G], chunk)
    if chunk // G >= 64:
        assert realised(pattern, whole, 32, G, chunk, n), "the planes did not code as built"
    kinds = chunk_kinds(whole, 32, G, chunk, n)
    classes = [chunk_class(kinds, c) for c in range(K)]
    ranges = [(0, 1), (0, 3), (2, 5), (4, 9), (5, 6), (7, K), (K - 1, K), (0, K)]
    edge_classes = set()
    for c0, c1 in ranges:
        got = sub_stream(whole, 32, G, chunk, n, c0, c1)
        part = data[c0 * chunk: min(n, c1 * chunk)]
        want = O.zipnn_compress(header32(part.size), part, G, bits, BYTES_MODE[G], chunk)
        assert np.array_equal(got, want), (G, chunk, c0, c1)
        assert np.array_equal(O.zipnn_decompress(got[32:], G, bits, BYTES_MODE[G], chunk, part.size), part)
        edge_classes |= {classes[c0], classes[c1 - 1]}
    if 64 <= chunk // G <= HUF_MAX_BLOCK:
        assert edge_classes >= {"raw", "rle", "one"} | ({"two"} if G > 1 else set()), edge_classes
