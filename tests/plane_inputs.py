"""Inputs built from the contents of each byte plane, a test-side huff0 writer, and a host model of the
branches the decoders take on a stream.

The decoders' hard branches depend on the shape of the Huffman table and the length of the bitstreams, not on
the dtype.  So the tests here do not start from float values: they choose the byte planes of every chunk
(`tensor_from_planes` is the inverse of the split + sign-bit rotation) or write the HUF blocks themselves
(`huf_block`, `assemble_body`), and `predict` says from the stream alone what each chunk does in the fused
kernel (decode.cuh) and in the per-bitstream-CTA kernel (decode_sync.cuh), so that a test can assert that it
reaches the branch it was built for.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

LUT_LOG = 11             # kDecLutLog: the index space of the fused tables
POOL_CAP = {5: 1024, 0: 2048}  # fused_tail_cap(PB): tail entries shared by the 8 chunks of a warp
SYNC_STREAM_CAP = 28672  # kSyncStreamCap: longer bitstreams take the ring path of k_huf_decode_sync
SYNC_THREADS = 256
SYNC_MIN_SEGBITS = 192


# ---------------------------------------------------------------- planes <-> tensor bytes
def plane_len(chunk_len: int, G: int, g: int) -> int:
    return chunk_len // G + (1 if g < chunk_len % G else 0)


def _unrotate(buf: np.ndarray, G: int) -> None:
    """Inverse of the sign-bit rotation, on whole 32-bit words (a trailing len % 4 is left alone)."""
    words = buf.size // 4
    if not words:
        return
    u = buf[: 4 * words].view(np.uint32)
    if G == 2:
        u[:] = ((u << 8) & 0x80008000) | ((u >> 1) & 0x7F807F80) | (u & 0x7F007F)
    else:
        u[:] = ((u << 8) & 0x80000000) | ((u >> 1) & 0x7F800000) | (u & 0x7FFFFF)


def chunk_from_planes(planes, G: int, bits_mode: int) -> np.ndarray:
    """The chunk bytes whose split (O.split_chunk) is `planes`."""
    n = sum(int(p.size) for p in planes)
    out = np.empty(n, dtype=np.uint8)
    for g in range(G):
        assert planes[g].size == plane_len(n, G, g), (g, planes[g].size, n)
        out[g::G] = planes[g]
    if bits_mode == 1 and G > 1:
        _unrotate(out, G)
    return out


def tensor_from_planes(chunks, G: int, bits_mode: int) -> np.ndarray:
    """chunks: per chunk, the list of its G planes.  Every chunk but the last must have the same length."""
    return np.concatenate([chunk_from_planes(p, G, bits_mode) for p in chunks]) if chunks else np.zeros(0, np.uint8)


def planes_of(data: np.ndarray, G: int, bits_mode: int, chunk: int):
    """The planes of every chunk of `data` (the oracle's split)."""
    return [O.split_chunk(data[o: o + chunk], G, bits_mode) for o in range(0, data.size, chunk)]


# ---------------------------------------------------------------- plane families: f(rng, n) -> uint8[n]
def _choice(rng, p, n, offset=0):
    p = np.asarray(p, dtype=np.float64)
    return (rng.choice(p.size, n, p=p / p.sum()) + offset).astype(np.uint8)


def equiprobable(k: int, offset: int = 0):
    return lambda rng, n: (rng.integers(0, k, n) + offset).astype(np.uint8)


def geometric(p: float):
    return lambda rng, n: np.minimum(rng.geometric(p, n) - 1, 255).astype(np.uint8)


def fibonacci(rng, n):
    """Fibonacci counts over 14 symbols: the Huffman tree is as deep as it can be (the encoder caps it at 11)."""
    f = [1, 1]
    while len(f) < 14:
        f.append(f[-1] + f[-2])
    return _choice(rng, f[::-1], n)


def zipf256(rng, n):
    return _choice(rng, 1.0 / np.arange(1, 257) ** 1.1, n)


def dirichlet256(rng, n):
    return _choice(rng, rng.dirichlet(np.full(256, 0.5)), n)


def heavy256(rng, n):
    p = np.full(256, 0.87 / 255)
    p[37] = 0.13
    return _choice(rng, p, n)


def logexp_bf16(rng, n):
    """The exponent plane of bf16 values with log-uniform magnitudes over 2^-40 .. 2^40 (after the rotation)."""
    x = (2.0 ** rng.uniform(-40, 40, n)).astype(np.float32)
    return ((x.view(np.uint32) >> 23) & 0xFF).astype(np.uint8)


def with_rare(k: int):
    """16 equiprobable symbols and k rare ones seen once each: the rare codes are the longest the encoder allows,
    and k sets how much of the index space they take (the tail size x_cut)."""
    def f(rng, n):
        x = (rng.integers(0, 16, n) + 100).astype(np.uint8)
        x[rng.choice(n, k, replace=False)] = rng.choice(np.r_[0:100, 116:256], k, replace=False)
        return x
    return f


def constant(v: int = 0):
    return lambda rng, n: np.full(n, v, dtype=np.uint8)


def uniform(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8)


FAMILIES = {
    "eq2": equiprobable(2), "eq4": equiprobable(4), "eq8": equiprobable(8), "eq16": equiprobable(16, 100),
    "eq64": equiprobable(64, 60), "eq128": equiprobable(128),
    "geo5": geometric(0.5), "geo3": geometric(0.3), "fib": fibonacci,
    "zipf256": zipf256, "dirichlet256": dirichlet256, "heavy256": heavy256, "logexp": logexp_bf16,
    "const": constant(0), "raw": uniform,
}


def code_lengths(plane: np.ndarray) -> np.ndarray:
    """Code length per byte value of the table the reference encoder builds for this plane (0: absent)."""
    cnt = np.bincount(plane, minlength=256).astype(np.uint32)
    nb, _, _, _ = O.huf_table_from_counts(cnt, plane.size)
    return nb


def clustered(plane: np.ndarray) -> np.ndarray:
    """Each quarter of the plane (a huff0 bitstream) sorted by code length, longest first: long codes in runs."""
    nb = code_lengths(plane)
    seg = (plane.size + 3) // 4
    out = plane.copy()
    for q in range(4):
        part = out[q * seg: (q + 1) * seg]
        part[:] = part[np.argsort(-nb[part].astype(np.int32), kind="stable")]
    return out


# ---------------------------------------------------------------- a huff0 writer (any Kraft-complete lengths)
def canonical_values(lengths) -> np.ndarray:
    """Code values of the reference's canonical assignment (huf_compress.c:392-410): per length, from the
    longest down, consecutive values in symbol order."""
    nb = np.asarray(lengths, dtype=np.int64)
    log = int(nb.max())
    per_len = np.bincount(nb, minlength=log + 2)
    start = np.zeros(log + 2, dtype=np.int64)
    v = 0
    for length in range(log, 0, -1):
        start[length] = v
        v = (v + per_len[length]) >> 1
    val = np.zeros(256, dtype=np.uint16)
    for s in range(nb.size):
        if nb[s]:
            val[s] = start[nb[s]]
            start[nb[s]] += 1
    return val


def kraft_lengths(rng, nsym: int, max_len: int, min_len: int = 1, alphabet: int = 129) -> np.ndarray:
    """Random Kraft-complete code lengths of nsym codes, none longer than max_len, over random byte values below
    `alphabet` (raw 4-bit weights describe at most 129 symbols)."""
    assert 2 <= nsym <= alphabet <= 256 and nsym <= 1 << max_len
    if max_len == 12:
        min_len = max(min_len, 2)  # weights stop at 11: no 1-bit code under table log 12
    depth = [0]
    while len(depth) < nsym or min(depth) < min_len:
        ok = [i for i, d in enumerate(depth) if d < max_len]
        shallow = [i for i in ok if depth[i] < min_len]
        if shallow:
            i = shallow[0]
        elif max(depth) < max_len:  # one code of the longest length first: the table log is max_len
            i = int(np.argmax(depth))
        else:
            i = ok[int(rng.integers(0, len(ok)))]
        d = depth.pop(i)
        depth += [d + 1, d + 1]
    assert len(depth) == nsym, "min_len and nsym do not fit"
    nb = np.zeros(256, dtype=np.uint8)
    nb[np.sort(rng.choice(alphabet, nsym, replace=False))] = rng.permutation(depth)
    return nb


def plane_for_lengths(rng, nb, n: int, hot=None) -> np.ndarray:
    """A plane of n symbols whose frequencies follow 2^-length (so a block with these lengths compresses), every
    coded symbol present, optionally with one symbol `hot` drawn 3 % more often than its length says."""
    syms = np.nonzero(nb)[0]
    p = 2.0 ** -nb[syms].astype(np.float64)
    if hot is not None:
        p[np.searchsorted(syms, hot)] += 0.03 * p.sum()
    plane = syms[rng.choice(syms.size, n, p=p / p.sum())].astype(np.uint8)
    plane[: syms.size] = rng.permutation(syms)
    return plane


def _bitstream(plane: np.ndarray, nb: np.ndarray, val: np.ndarray) -> bytes:
    """huff0 bitstream (huf_compress.c:457-502): symbols from the last to the first, bits LSB first, then
    the end mark."""
    lens = nb[plane[::-1]].astype(np.int64)
    vals = val[plane[::-1]].astype(np.int64)
    pos = np.concatenate(([0], np.cumsum(lens)))
    total = int(pos[-1])
    bits = np.zeros(total + 1 + 7, dtype=np.uint8)
    for j in range(int(lens.max()) if lens.size else 0):
        m = lens > j
        bits[pos[:-1][m] + j] = (vals[m] >> j) & 1
    bits[total] = 1
    return np.packbits(bits[: (total + 8) // 8 * 8], bitorder="little").tobytes()


def raw_weight_header(nb: np.ndarray) -> bytes:
    """Table description with raw 4-bit weights (huf_compress.c:157-167): weights of symbols 0 .. max-1,
    the last symbol's weight implied."""
    nz = np.nonzero(nb)[0]
    max_sym = int(nz[-1])
    assert 1 <= max_sym <= 128, "raw weights describe at most 129 symbols"
    log = int(nb.max())
    w = np.zeros(max_sym + 1, dtype=np.uint8)
    w[nz] = log + 1 - nb[nz]
    w[max_sym] = 0
    hdr = bytearray([128 + max_sym - 1])
    for s in range(0, max_sym, 2):
        hdr.append((int(w[s]) << 4) | int(w[s + 1]))
    return bytes(hdr)


def huf_block(nb: np.ndarray, plane: np.ndarray) -> bytes:
    """A 4-stream HUF block of `plane` with code lengths nb (Kraft-complete, table log <= 12)."""
    nb = np.asarray(nb, dtype=np.uint8)
    assert np.all(nb[plane] > 0), "a symbol of the plane has no code"
    val = canonical_values(nb)
    seg = (plane.size + 3) // 4
    streams = [_bitstream(plane[q * seg: min((q + 1) * seg, plane.size)], nb, val) for q in range(4)]
    assert all(len(s) < 65536 for s in streams[:3])
    jump = b"".join(len(s).to_bytes(2, "little") for s in streams[:3])
    return raw_weight_header(nb) + jump + b"".join(streams)


def assemble_body(items, G: int) -> np.ndarray:
    """ZipNN stream body (after the python header): items[g][c] = (type, payload bytes).
    type 0 = stored raw, 1 = HUF block (1 byte: RLE)."""
    K = len(items[0])
    types = bytes(t for g in range(G) for t, _ in items[g])
    cums = []
    for g in range(G):
        cum = np.cumsum([len(p) for _, p in items[g]], dtype=np.uint64)
        cums.append(cum.astype("<u8").tobytes())
    payload = b"".join(p for g in range(G) for _, p in items[g])
    assert len(types) == G * K
    return np.frombuffer(types + b"".join(cums) + payload, dtype=np.uint8).copy()


def stream_items(planes, G: int, make_block):
    """items for assemble_body: make_block(g, c, plane) -> (type, bytes)."""
    return [[make_block(g, c, planes[c][g]) for c in range(len(planes))] for g in range(G)]


# ---------------------------------------------------------------- the host model of the decoders' branches
def tail_size(weights, lg: int, pb: int) -> int:
    """x_cut of lut_tail_size (pb = 5) / lut2_tail_size (pb = 0), or -1 where the fused kernel cannot take the
    table (table log > 11): the power of two (>= 64, >= 8) at or above the index bound of the codes longer than
    pb (8 for pb = 0) bits."""
    if lg > LUT_LOG:
        return -1
    cnt = np.bincount(np.asarray(weights, dtype=np.int64), minlength=16)
    long_bits = pb if pb else 8
    at = x_long = 0
    for w in range(1, lg + 1):
        at += (int(cnt[w]) << (w - 1)) << (LUT_LOG - lg)
        if lg + 1 - w > long_bits:
            x_long = at
    x_cut = 64 if pb else 8
    while x_cut < x_long:
        x_cut <<= 1
    return x_cut


class Item:
    __slots__ = ("g", "c", "kind", "src_off", "src_len", "dec_len", "lg", "nsym", "hsize", "lengths", "s_len", "counts",
                 "x_cut", "fixed_len", "segbits")


def predict(body, G: int, bits_mode: int, chunk: int, orig: int, body_addr_mod16: int = 0) -> dict:
    """What the stream makes the decoders do.  Returns {
        items[g][c]: Item (kind raw / rle / huf; for huf: table log, lengths, the 4 bitstream lengths s_len and
                     symbol counts, x_cut per PB, fixed code length and segbits per bitstream),
        mode[c]: 'plain' / 'general' / 'fused' as k_decode_meta sets it,
        pb: 5 or 0 (which fused instantiation the tensor gets),
        fused[c]: for fused-mode chunks, 'fused' or 'demoted' in k_huf_decode_fused (pool prefix per warp),
        pool_run[w]: tail entries the warp's fused chunks ask for,
        regular[w]: whether warp w takes the bulk-tensor side path (when the launch has the tensor maps),
        side_r0[g], k_full, K }."""
    b = np.asarray(body, dtype=np.uint8)
    K = (orig + chunk - 1) // chunk
    n_it = G * K
    types = b[:n_it]
    cum = b[n_it: 9 * n_it].view("<u8").reshape(G, K).astype(np.int64)
    payload0 = 9 * n_it
    base = [0] * 4
    for g in range(G - 1):
        base[g + 1] = base[g] + int(cum[g, -1])
    k_full = orig // chunk
    last_len = orig - k_full * chunk
    pb = 5 if (G >= 2 and bits_mode == 1) else 0
    items = [[None] * K for _ in range(G)]
    mode = []
    for c in range(K):
        clen = chunk if c < K - 1 or orig % chunk == 0 else orig - c * chunk
        nhuf, last_huf = 0, -1
        for g in range(G):
            it = Item()
            it.g, it.c = g, c
            lo = int(cum[g, c - 1]) if c else 0
            it.src_off = payload0 + base[g] + lo
            it.src_len = int(cum[g, c]) - lo
            it.dec_len = plane_len(clen, G, g)
            it.lg = it.hsize = -1
            if types[g * K + c] == 0 or it.src_len == it.dec_len or it.dec_len == 0:
                it.kind = "raw"
            elif it.src_len == 1:
                it.kind = "rle"
            else:
                it.kind = "huf"
                nhuf += 1
                last_huf = g
                blk = b[it.src_off: it.src_off + it.src_len]
                it.hsize, w, it.lg = O.huf_read_table(blk)
                it.nsym = w.size
                it.lengths = np.where(w > 0, it.lg + 1 - w.astype(np.int64), 0)
                it.x_cut = {5: tail_size(w, it.lg, 5), 0: tail_size(w, it.lg, 0)}
                p = blk[it.hsize:]
                l012 = [int(p[0]) | int(p[1]) << 8, int(p[2]) | int(p[3]) << 8, int(p[4]) | int(p[5]) << 8]
                it.s_len = l012 + [it.src_len - it.hsize - 6 - sum(l012)]
                seg = (it.dec_len + 3) // 4
                it.counts = [seg, seg, seg, it.dec_len - 3 * seg]
                present = np.unique(it.lengths[it.lengths > 0])
                it.fixed_len = int(present[0]) if present.size == 1 else 0
                it.segbits = []
                for q in range(4):
                    last = int(p[6 + sum(it.s_len[:q]) + it.s_len[q] - 1])
                    bits = 8 * (it.s_len[q] - 1) + last.bit_length() - 1
                    it.segbits.append(max((bits + SYNC_THREADS - 1) // SYNC_THREADS, SYNC_MIN_SEGBITS))
            items[g][c] = it
        if nhuf == 1 and last_huf == G - 1 and clen % 512 == 0:
            mode.append("fused")
        elif nhuf >= 1:
            mode.append("general")
        else:
            mode.append("plain")
    # k_huf_decode_fused: the 8 chunks of a warp share one tail pool (exclusive prefix over the slots; a chunk
    # whose running total passes the capacity is demoted, and so is every later chunk of the warp)
    fused, pool_run, regular = {}, [], []
    side_pred, at = [], 9 * n_it
    for g in range(3):
        side_pred.append(at)
        if g < G:
            at += k_full * (chunk // G) + plane_len(last_len, G, g)
    for w0 in range(0, K, 8):
        run = 0
        live_all = True
        for c in range(w0, w0 + 8):
            if c >= K or mode[c] != "fused":
                live_all = False
                continue
            x = items[G - 1][c].x_cut[pb]
            if x < 0:
                fused[c] = "demoted"
                live_all = False
                continue
            run += x
            fused[c] = "fused" if run <= POOL_CAP[pb] else "demoted"
            live_all = live_all and fused[c] == "fused"
            if c >= k_full:
                live_all = False
            for g in range(G - 1):
                t = items[g][c]
                live_all = live_all and t.kind == "raw" and t.src_off == side_pred[g] + c * (chunk // G)
        pool_run.append(run)
        regular.append(live_all)
    return dict(items=items, mode=mode, pb=pb, fused=fused, pool_run=pool_run, regular=regular, K=K, k_full=k_full,
                side_r0=[(body_addr_mod16 + p) & 15 for p in side_pred])


def misaligned_sync_guesses(it: Item) -> int:
    """Bitstreams of a fixed-length-code item whose CTA segment starts are not code boundaries
    (segbits % L != 0 and the stream spans more than one segment): those threads never resynchronise and are
    corrected only by the round loop of k_huf_decode_sync."""
    if not it.fixed_len:
        return 0
    n = 0
    for q in range(4):
        bits = it.counts[q] * it.fixed_len
        if it.segbits[q] % it.fixed_len and bits > it.segbits[q]:
            n += 1
    return n
