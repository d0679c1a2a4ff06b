"""A fixed corpus of corrupted streams and the verdict model every decode entry point must follow.

Streams come from files people download, so every decoder reads bytes from outside the program.  Each base stream
here is made by the oracle from the plane builders of test_decoder_tables_gpu and sends its chunks down one decoder
path (plane_inputs.predict says which); each mutant changes one field of one base at its first, a middle or its
last chunk.  Nothing is random at run time: the seeds are fixed and the corpus is the same on every run.

Mutants come in two kinds:
  * container mutants change a type byte, a cumulative size row, a group total or the body's length;
  * block mutants replace one Huffman item by a changed block through `replace_item`, which rewrites the size rows,
    so the container stays consistent and the verdict depends on the block alone.

`verdict(base, body)` is the contract: ('ok', bytes), ('corrupt', None) or ('unsupported', None), with a verdict per
chunk for the entry points that decode only some chunks.  Container rules are DESIGN §6; a block's verdict is that
of the reference's HUF_decompress4X1, which the port restates (tests/golden/corrupt_verdicts.json holds the
reference's own verdicts on every block mutant).  Where the model and the port part, the mutant's class is one of
DIVERGENCES, each pointing to its DESIGN entry.
"""
from __future__ import annotations

import functools

import numpy as np

import plane_inputs as P
from oracle import oracle as O

LAYOUT = {"bf16": (2, 1, 10), "fp16": (2, 0, 10), "fp32": (4, 1, 220), "fp8": (1, 0, 10)}
HUF_BLOCK_MAX = 128 * 1024
OK, CORRUPT, UNSUPPORTED = "ok", "corrupt", "unsupported"

# mutant classes where the model (and every decoder) parts from the port, with the reason
DIVERGENCES = {
    "raw_long": "DESIGN §7: a stored item longer than its plane is refused (the port, like the reference, reads "
                "the plane's length and ignores the rest)",
    "log12": "DESIGN §6: table log 12 is E_UNSUPPORTED (the port decodes it)",
}

CONTAINER = ("type", "row", "total", "cut", "trailing", "empty_huf", "raw_long")
BLOCK = ("table", "weights", "log12", "jump", "stream", "flip")


# ------------------------------------------------------------------ base streams
class Base:
    def __init__(self, name, dtype, chunk, data, body, path):
        self.name, self.dtype, self.chunk, self.data, self.body, self.path = name, dtype, chunk, data, body, path
        self.G, self.bits, self.bm = LAYOUT[dtype]
        self.orig = data.size
        self.K = -(-self.orig // chunk)
        self.pr = P.predict(body, self.G, self.bits, chunk, self.orig)
        self.targets = sorted({0, self.K // 2, self.K - 1})


def _planes_base(name, path, dtype, chunk, tops, seed, last=None, side=None):
    import test_decoder_tables_gpu as T
    c = T.planes_case(name, dtype, chunk, tops, seed, last=last, side=side)
    return Base(name, dtype, chunk, c.data, c.body, path)


@functools.lru_cache(maxsize=None)
def bases():
    import test_decoder_tables_gpu as T
    ring = [c for c in T.ring_cases() if c.name == "ring_bf16_heavy256"][0]
    out = [
        # 12 fused chunks (tail pool, bulk-tensor side plane) and a ragged last chunk (general)
        _planes_base("bf16_fused", "fused", "bf16", 262144, ["geo5"] * 13, 1, last=100000),
        # two coded groups in every chunk: the general kernels
        _planes_base("fp32_general", "general", "fp32", 65536, ["geo5"] * 5, 2, last=40000,
                     side=lambda c, g: "geo3" if g == 2 else "raw"),
        # 70 general chunks: 64 take a pool slot, the rest the overflow kernel
        _planes_base("fp16_overflow", "overflow", "fp16", 4096, ["geo5"] * 70, 3, side=lambda c, g: "geo3"),
        _planes_base("fp8_g1", "fused", "fp8", 131072, ["geo5"] * 4, 4, last=5000),
        # bitstreams past the sync decoder's shared-memory copy: its ring path
        Base("ring_bf16", "bf16", ring.chunk, ring.data, ring.body, "ring"),
        _planes_base("raw_only", "plain", "bf16", 4096, ["raw"] * 6, 5, last=1000),
        _planes_base("rle_only", "plain", "bf16", 4096, ["const"] * 6, 6, last=1002, side=lambda c, g: "const"),
        # a last chunk of one byte: group 1's plane there is empty
        _planes_base("empty_plane", "plain", "bf16", 4096, ["geo5"] * 3 + ["raw"], 7, last=1),
    ]
    return {b.name: b for b in out}


# ------------------------------------------------------------------ stream fields
def split(body, G, K):
    """-> (types[G, K], cum[G, K] as Python ints, payload0)."""
    b = np.asarray(body, dtype=np.uint8)
    types = b[: G * K].reshape(G, K)
    cum = [[int(v) for v in row] for row in b[G * K: 9 * G * K].view("<u8").reshape(G, K)]
    return types, cum, 9 * G * K


def items(body, G, K):
    """-> items[g][c] = (type, payload bytes) of a consistent body."""
    types, cum, payload0 = split(body, G, K)
    b = np.asarray(body, dtype=np.uint8)
    out, at = [], payload0
    for g in range(G):
        row, lo = [], 0
        for c in range(K):
            row.append((int(types[g, c]), b[at + lo: at + cum[g][c]].tobytes()))
            lo = cum[g][c]
        out.append(row)
        at += cum[g][K - 1]
    return out


def replace_item(body, G, K, g, c, payload, type_=None):
    """The body with item (g, c) replaced and the size rows rewritten to match."""
    it = items(body, G, K)
    t, _ = it[g][c]
    it[g][c] = (t if type_ is None else type_, bytes(payload))
    return P.assemble_body(it, G)


def row_at(G, K, g, c):
    return G * K + 8 * (g * K + c)


# ------------------------------------------------------------------ mutants
class Mutant:
    __slots__ = ("base", "id", "cls", "kind", "g", "c", "body", "field")

    def __init__(self, base, name, cls, g, c, body, field):
        self.base, self.cls, self.g, self.c, self.body, self.field = base, cls, g, c, np.asarray(body, np.uint8), field
        self.kind = "block" if cls in BLOCK else "container"
        self.id = f"{base.name}/{name}"


def _u64(body, at, v):
    b = body.copy()
    b[at: at + 8] = np.frombuffer(int(v % (1 << 64)).to_bytes(8, "little"), np.uint8)
    return b


def _huf_parts(blk):
    """-> (table description, [l0, l1, l2], [4 bitstreams])."""
    h, _, _ = O.huf_read_table(blk)
    p = blk[h:]
    ls = [int(p[0]) | int(p[1]) << 8, int(p[2]) | int(p[3]) << 8, int(p[4]) | int(p[5]) << 8]
    at, streams = 6, []
    for q in range(4):
        n = ls[q] if q < 3 else len(p) - at
        streams.append(bytearray(p[at: at + n]))
        at += n
    return bytes(blk[:h]), ls, streams


def _huf_join(hdr, ls, streams):
    return hdr + b"".join(int(v & 0xFFFF).to_bytes(2, "little") for v in ls) + b"".join(bytes(s) for s in streams)


def _direct_table(w):
    """Raw 4-bit weights (huf_compress.c:157-167) for weights w of symbols 0..len(w)-2 (the last one implied)."""
    n = len(w) - 1
    out = bytearray([128 + n - 1])
    ww = list(w[:n]) + [0]
    for s in range(0, n, 2):
        out.append((int(ww[s]) << 4) | int(ww[s + 1] if s + 1 < len(ww) else 0))
    return bytes(out)


def block_mutations(blk, dlen, rng):
    """(name, cls, new block) for one Huffman block of a dlen-byte plane."""
    blk = bytes(blk)
    hdr, ls, streams = _huf_parts(blk)
    out = []
    for v in sorted({0, 1, 127, 128, 255, (blk[0] + 1) & 255, (blk[0] - 1) & 255}):
        if v != blk[0]:
            out.append((f"table0={v}", "table", bytes([v]) + blk[1:]))
    _, w, lg = O.huf_read_table(np.frombuffer(blk, np.uint8))
    if w.size <= 129:
        ones = [s for s in range(w.size - 1) if w[s] == 1]
        if ones:
            bad = w.copy()
            bad[ones[0]] = 2
            out.append(("weights_sum", "weights", _direct_table(bad) + blk[len(hdr):]))
        for big in (12, 13, 15):
            bad = w.copy()
            bad[0] = big
            out.append((f"weight={big}", "weights", _direct_table(bad) + blk[len(hdr):]))
    nb = P.kraft_lengths(rng, 40, 12)
    out.append(("log12", "log12", P.huf_block(nb, P.plane_for_lengths(rng, nb, dlen))))
    rest = len(blk) - len(hdr) - 6
    for name, j in (("jump0", [0, ls[1], ls[2]]), ("jump_s3_empty", [ls[0], ls[1], rest - ls[0] - ls[1]]),
                    ("jump_past_rest", [ls[0], ls[1], rest - ls[0] - ls[1] + 1]), ("jump_ffff", [0xFFFF, ls[1], ls[2]])):
        out.append((name, "jump", _huf_join(hdr, j, streams)))
    for q in range(4):
        s = streams[q]
        last = s[-1]
        top = last.bit_length() - 1
        variants = [("last0", 0), ("mark_up", (last ^ (1 << top)) | (1 << min(top + 1, 7)) if top < 7 else last >> 1)]
        if top > 0:
            variants.append(("mark_down", (last ^ (1 << top)) | (1 << (top - 1))))
        for name, v in variants:
            t = [bytearray(x) for x in streams]
            t[q][-1] = v
            if bytes(t[q]) != bytes(s):
                out.append((f"s{q}_{name}", "stream", _huf_join(hdr, ls, t)))
        t = [bytearray(x) for x in streams]
        del t[q][-1]
        j = list(ls)
        if q < 3:
            j[q] -= 1
        out.append((f"s{q}_drop", "stream", _huf_join(hdr, j, t)))
        for where, pos in (("start", 0), ("mid", len(s) // 2), ("end", len(s) - 1)):
            t = [bytearray(x) for x in streams]
            t[q][pos] ^= 1 << int(rng.integers(0, 8))
            out.append((f"s{q}_flip_{where}", "stream", _huf_join(hdr, ls, t)))
    return out


@functools.lru_cache(maxsize=None)
def mutants(name):
    """Every mutant of base `name`, in a fixed order."""
    b = bases()[name]
    G, K, body = b.G, b.K, b.body
    rng = np.random.default_rng(sum(map(ord, name)))
    types, cum, payload0 = split(body, G, K)
    out = []

    def add(nm, cls, g, c, mb, field):
        out.append(Mutant(b, nm, cls, g, c, mb, field))

    # container
    for c in b.targets:
        for g in sorted({0, G - 1}):
            ti = g * K + c
            for v, nm in ((2, "2"), (0xFF, "ff"), (1 - min(int(body[ti]), 1), "swap")):
                m = body.copy()
                m[ti] = v
                add(f"type[{g},{c}]={nm}", "type", g, c, m, ("bytes", ti, ti + 1))
            at = row_at(G, K, g, c)
            prev = cum[g][c - 1] if c else 0
            for v, nm in ((cum[g][c] + 1, "+1"), (cum[g][c] - 1, "-1"), (prev - 1, "decreasing"), ((1 << 64) - 16, "near2^64")):
                add(f"row[{g},{c}]{nm}", "row", g, c, _u64(body, at, v), ("bytes", at, at + 8))
    room = body.size - payload0 - sum(cum[g][K - 1] for g in range(G - 1))
    at = row_at(G, K, G - 1, K - 1)
    add("total_past_payload", "total", G - 1, K - 1, _u64(body, at, room + 1), ("bytes", at, at + 8))
    for nm, n in (("cut_types", G * K // 2), ("cut_sizes", G * K + 4 * G * K + 3), ("cut_1", body.size - 1),
                  ("cut_payload", payload0 + (body.size - payload0) // 2)):
        add(nm, "cut", None, None, body[:n].copy(), ("prefix", n))
    add("trailing", "trailing", None, None, np.concatenate([body, np.arange(5, dtype=np.uint8)]), ("extend", 5))
    for c in range(K):
        for g in range(G):
            if P.plane_len(b.orig - c * b.chunk if c == K - 1 else b.chunk, G, g) == 0:
                ti = g * K + c
                m = body.copy()
                m[ti] = 1
                add(f"empty_huf[{g},{c}]", "empty_huf", g, c, m, ("bytes", ti, ti + 1))
    # block: the Huffman items at the target chunks (a stored item of the same chunk takes the raw_long mutant)
    huf_targets = [(g, c) for c in b.targets for g in range(G) if b.pr["items"][g][c].kind == "huf"]
    for c in b.targets:
        for g in range(G):
            it = b.pr["items"][g][c]
            if types[g, c] == 0 and it.dec_len:
                blk = body[it.src_off: it.src_off + it.src_len].tobytes()
                add(f"raw_long[{g},{c}]", "raw_long", g, c, replace_item(body, G, K, g, c, blk + b"\x00"), ("item", g, c))
                break
    for g, c in huf_targets:
        it = b.pr["items"][g][c]
        blk = body[it.src_off: it.src_off + it.src_len].tobytes()
        for nm, cls, nb in block_mutations(blk, it.dec_len, rng):
            add(f"{nm}[{g},{c}]", cls, g, c, replace_item(body, G, K, g, c, nb), ("item", g, c))
    # seeded single-bit flips inside the Huffman items at the targets (in place: the rows do not change)
    if huf_targets:
        for k in range(200):
            g, c = huf_targets[k % len(huf_targets)]
            it = b.pr["items"][g][c]
            pos = it.src_off + int(rng.integers(0, it.src_len))
            m = body.copy()
            m[pos] ^= 1 << int(rng.integers(0, 8))
            add(f"flip{k}@{pos}[{g},{c}]", "flip", g, c, m, ("item", g, c))
    return out


def all_mutants():
    return [m for name in bases() for m in mutants(name)]


# ------------------------------------------------------------------ the verdict model
class Verdict:
    __slots__ = ("status", "data", "chunks", "cls")

    def __repr__(self):
        return f"Verdict({self.status})"


_BLOCKS = {}


def block_verdict(blk, dlen):
    """A Huffman block's verdict, as HUF_decompress4X1 (restated by the port) gives it, with table log 12 refused
    as unsupported.  -> (status, plane or None)."""
    key = (np.asarray(blk, np.uint8).tobytes(), dlen)
    if key not in _BLOCKS:
        _BLOCKS[key] = _block_verdict(key[0], dlen)
    return _BLOCKS[key]


def _block_verdict(blk, dlen):
    try:
        _, _, lg = O.huf_read_table(blk)
    except ValueError:
        return CORRUPT, None
    if lg > P.LUT_LOG:
        return UNSUPPORTED, None
    try:
        return OK, O.huf_decompress(blk, dlen)
    except ValueError:
        return CORRUPT, None


def chunk_verdicts(base, body):
    """Per-chunk status (None when the body's tables cannot be read at all), following DESIGN §6."""
    G, K, chunk = base.G, base.K, base.chunk
    b = np.asarray(body, dtype=np.uint8)
    if b.size < 9 * G * K:
        return None
    types, cum, payload0 = split(b, G, K)
    payload_len = b.size - payload0
    base_g, room, totals_ok = [0] * 4, payload_len, True
    for g in range(G):
        tot = cum[g][K - 1]
        if tot > room:
            totals_ok = False
            break
        room -= tot
        if g + 1 < G:
            base_g[g + 1] = base_g[g] + tot
    out = []
    for c in range(K):
        clen = min(chunk, base.orig - c * chunk)
        st = OK if totals_ok else CORRUPT
        for g in range(G):
            if st == CORRUPT:
                break
            hi, lo = cum[g][c], (cum[g][c - 1] if c else 0)
            dlen = P.plane_len(clen, G, g)
            t = int(types[g, c])
            if hi < lo or hi > payload_len - base_g[g] or t > 1:
                st = CORRUPT
                break
            slen = hi - lo
            if t == 0:
                if slen != dlen:
                    st = CORRUPT
            elif dlen == 0 or slen == 0 or slen > dlen:
                st = CORRUPT
            elif 1 < slen < dlen:
                if dlen > HUF_BLOCK_MAX:
                    st = CORRUPT
                else:
                    off = payload0 + base_g[g] + lo
                    v, _ = block_verdict(b[off: off + slen], dlen)
                    if v != OK:
                        st = v
        out.append(st)
    return out


def verdict(base, body) -> Verdict:
    v = Verdict()
    v.chunks = chunk_verdicts(base, body)
    v.data = None
    if v.chunks is None or CORRUPT in v.chunks:
        v.status = CORRUPT
    elif UNSUPPORTED in v.chunks:
        v.status = UNSUPPORTED
    else:
        v.status = OK
        v.data = O.zipnn_decompress(body, base.G, base.bits, base.bm, base.chunk, base.orig, threads=8)
    return v


def port_status(base, body):
    """The port's verdict on the whole stream: (OK, bytes) or (CORRUPT, None)."""
    try:
        return OK, O.zipnn_decompress(body, base.G, base.bits, base.bm, base.chunk, base.orig, threads=8)
    except RuntimeError:
        return CORRUPT, None


def divergence(m: Mutant, v: Verdict):
    """The DIVERGENCES class of a mutant whose model verdict may part from the port's, or None."""
    if v.status == UNSUPPORTED:
        return "log12"
    return m.cls if m.cls in DIVERGENCES else None


def block_of(m: Mutant):
    """The mutated Huffman block of a block mutant and its plane length."""
    b = m.base
    types, cum, payload0 = split(m.body, b.G, b.K)
    base_g = sum(cum[h][b.K - 1] for h in range(m.g))
    lo = cum[m.g][m.c - 1] if m.c else 0
    off = payload0 + base_g + lo
    clen = min(b.chunk, b.orig - m.c * b.chunk)
    return m.body[off: payload0 + base_g + cum[m.g][m.c]], P.plane_len(clen, b.G, m.g)
