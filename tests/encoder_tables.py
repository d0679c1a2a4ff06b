"""Crafted inputs for the encoder's table build and emission pass, each of which names the branch it was built for.

The encoder's table build (huf_serial.cuh: huf_limit_depth, fse_pick_log, fse_normalize, huf_pack_weights,
huf_write_table; encode.cuh: warp_block_decision) and its emission kernels (k_encode_write_warp, k_encode_write) decide
the bytes of a stream on inputs that float weights rarely produce.  Here a case is a list of byte planes per chunk,
each plane built from an exact histogram and an order; `plane_inputs.tensor_from_planes` turns the planes of every
chunk into the tensor bytes for each layout.

Reaching a branch is proven on the project's own restatement: tests/host_emu defines huf_serial.cuh's ZB_HUF_TRACE
hook as a counter (`table`), and the restatement's lengths and headers are checked against the reference's for every
histogram here (test_encoder_tables_host.py), so a branch reached in the one is reached in the other.

`parse` reads a produced stream back into per-block facts (table log, header size and form, bitstream sizes,
absolute start offsets and bit totals), from which the GPU test asserts which alignments and residues the device
wrote.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np

import plane_inputs as P

HERE = os.path.dirname(os.path.abspath(__file__))

TRACE = ("limit", "limit_below11", "repay_break_total", "repay_break_nolow", "repay_step_up", "repay_largest",
         "repay_rank_emptied", "overshoot_no_rank1", "overshoot_rank1", "huf_log_floor", "fse_log_floor",
         "normalize_slow", "pack_distinct", "pack_rle", "table_fse", "table_nibble_lost", "table_nibble", "table_raw")
# the branches every run of the crafted histograms must reach (repay_break_nolow: the rank below the limit is empty,
# which the Kraft debt of a deep tree never allows; it is counted, not required)
REQUIRED = tuple(t for t in TRACE if t != "repay_break_nolow")

LAYOUTS = ((1, 0), (2, 0), (2, 1), (4, 0), (4, 1))
THRESHOLDS = (0.95, 1.0, 1.5)


def bytes_mode(G: int) -> int:
    return 220 if G == 4 else 10


def header() -> bytes:
    h = bytearray(32)
    h[0:2] = b"ZN"
    return bytes(h)


# ---------------------------------------------------------------- the restatement, with its branch counters
@functools.lru_cache(maxsize=None)
def emu() -> C.CDLL:
    E = C.CDLL(os.path.join(HERE, "host_emu", "libemu_serial.so"))
    E.emu_table_from_counts.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    E.emu_trace_take.argtypes = [C.c_void_p]
    E.emu_early_out.argtypes = [C.c_uint32, C.c_uint32]
    E.emu_block_decision.restype = C.c_uint32
    E.emu_block_decision.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_double]
    return E


class Table:
    __slots__ = ("nb", "val", "hdr", "lg", "trace")


def table(counts, n: int | None = None) -> Table:
    """huf_serial.cuh's table for a histogram: code lengths, values, header (None: -1, stored raw), table log, and the
    set of branches it took."""
    E = emu()
    cnt = np.ascontiguousarray(counts, dtype=np.uint32)
    n = int(cnt.sum()) if n is None else n
    t = Table()
    t.nb = np.zeros(256, np.uint8)
    t.val = np.zeros(256, np.uint16)
    hdr = np.zeros(512, np.uint8)
    lg = C.c_int(0)
    tr = np.zeros(64, np.uint32)
    E.emu_trace_take(tr.ctypes.data)
    h = E.emu_table_from_counts(cnt.ctypes.data, n, t.nb.ctypes.data, t.val.ctypes.data, hdr.ctypes.data, C.byref(lg))
    k = E.emu_trace_take(tr.ctypes.data)
    assert k == len(TRACE)
    t.hdr = hdr[:h].tobytes() if h > 0 else None
    t.lg = lg.value
    t.trace = {TRACE[i] for i in range(k) if tr[i]}
    return t


def decision(plane: np.ndarray, cap: int, thr: float) -> int:
    """What warp_block_decision stores for a plane, run on the host: huf_early_out, the table, huf_block_decision.
    0 = raw, 1 = RLE, else the coded block's size."""
    E = emu()
    n = plane.size
    cnt = np.bincount(plane, minlength=256).astype(np.uint32)
    bits = np.zeros(4, np.uint32)
    thr64 = float(np.float32(thr))
    early = E.emu_early_out(int(cnt.max()), n)
    if early == 0:
        return 0
    if early == 1:
        return int(E.emu_block_decision(1, bits.ctypes.data, 0, n, cap, thr64))
    t = table(cnt, n)
    h = len(t.hdr) if t.hdr is not None else -1
    if h <= 0 or h + 12 >= n:
        return 0
    seg = (n + 3) // 4
    for q in range(4):
        bits[q] = int(t.nb[plane[q * seg: min(n, (q + 1) * seg)]].astype(np.int64).sum())
    return int(E.emu_block_decision(0, bits.ctypes.data, h, n, cap, thr64))


# ---------------------------------------------------------------- histograms: (name, counts[256]) summing to plen
def _fit(counts: np.ndarray, plen: int):
    """Scale counts to sum to plen: a whole multiple, the rest on the most frequent symbol.  None if they do not fit."""
    c = counts.astype(np.int64)
    s = int(c.sum())
    if s > plen or s == 0:
        return None
    c = c * (plen // s)
    c[int(np.argmax(c))] += plen - int(c.sum())
    return c


def _place(c: np.ndarray, syms: np.ndarray) -> np.ndarray:
    out = np.zeros(256, np.int64)
    out[syms] = c
    return out


def _symbols(rng, k: int, how: str) -> np.ndarray:
    if how == "low":
        return np.arange(k)
    if how == "high":
        return np.arange(256 - k, 256)
    if how == "reversed":
        return np.arange(k)[::-1].copy()
    pool = np.arange(1 if k < 256 else 0, 256)   # scattered: symbol 0 absent when there is room
    return rng.choice(pool, k, replace=False)


def fib_counts(k: int, jitter: float, rng) -> np.ndarray:
    f = [1, 1]
    while len(f) < k:
        f.append(f[-1] + f[-2])
    c = np.array(f[::-1], np.float64)
    if jitter:
        c = c * rng.uniform(1 - jitter, 1 + jitter, k)
    return np.maximum(np.round(c), 1).astype(np.int64)


def geo_counts(k: int, ratio: float, top: float, rng, jitter: float = 0.0) -> np.ndarray:
    c = top * ratio ** np.arange(k, dtype=np.float64)
    if jitter:
        c = c * rng.uniform(1 - jitter, 1 + jitter, k)
    return np.maximum(np.round(c), 1).astype(np.int64)


def depth_histograms(plen: int, tries: int, seed: int):
    """Fibonacci counts over 13-26 symbols and geometric tails over 100-256, some jittered; seeded."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(tries):
        kind = i % 3
        if kind == 0:
            k = int(rng.integers(13, 27))
            c = fib_counts(k, float(rng.choice([0.0, 0.2, 0.5])), rng)
            name = f"fib{k}"
        elif kind == 1:
            k = int(rng.integers(100, 257))
            c = geo_counts(k, float(rng.uniform(0.9, 0.99)), plen * float(rng.uniform(0.02, 0.3)), rng,
                           float(rng.choice([0.0, 0.3])))
            name = f"geo{k}"
        else:   # a heavy head over a flat tail: many symbols pushed over the limit at once
            k = int(rng.integers(20, 257))
            head = int(rng.integers(1, 5))
            c = np.ones(k, np.int64) * int(rng.integers(1, 4))
            c[:head] = (plen * rng.dirichlet(np.ones(head)) * rng.uniform(0.5, 0.97)).astype(np.int64) + 1
            name = f"head{head}tail{k}"
        k = c.size
        c = _fit(c, plen) if kind != 2 else (c if c.sum() <= plen else None)
        if c is None:
            continue
        if kind == 2:
            c = c.copy()
            c[0] += plen - int(c.sum())
        syms = _symbols(rng, k, str(rng.choice(["low", "high", "reversed", "scattered"])))
        out.append((f"{name}-{i}", _place(c, syms)))
    return out


def tie_histograms(plen: int):
    """All counts equal over k symbols, several blocks of equal counts, scattered symbol sets."""
    out = []
    for k in (2, 3, 5, 7, 100, 129, 255, 256):
        if k > plen:
            continue
        c = np.full(k, plen // k, np.int64)
        c[: plen % k] += 1   # the first plen % k one higher: two tie blocks
        for how in ("low", "high", "scattered"):
            out.append((f"tie{k}-{how}", _place(c, _symbols(np.random.default_rng(k), k, how))))
    rng = np.random.default_rng(plen)
    for blocks in (2, 3, 6):
        sizes = rng.integers(2, 30, blocks)
        vals = np.sort(rng.choice(np.arange(1, 64), blocks, replace=False))[::-1]
        c = np.repeat(vals, sizes).astype(np.int64)
        c = _fit(c, plen)
        if c is not None:
            syms = np.sort(rng.choice(256, c.size, replace=False))
            syms[-1] = 255
            out.append((f"tieblocks{blocks}", _place(c, syms[rng.permutation(c.size)])))
    return out


def small_histograms(plen: int, tries: int, seed: int):
    """Planes of 13 bytes to a few KiB with many symbols: the table log drops below 11 (and the alphabet floor may
    raise it again)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(tries):
        k = int(rng.integers(2, min(plen, 256) + 1))
        p = rng.dirichlet(np.ones(k) * rng.uniform(0.05, 1.5))
        c = np.bincount(rng.choice(k, plen, p=p), minlength=k).astype(np.int64)
        syms = _symbols(rng, k, str(rng.choice(["low", "high", "scattered"])))
        out.append((f"small{k}-{i}", _place(c, syms)))
    return out


def header_histograms(plen: int, seed: int):
    """Weight headers: max_sym 127 / 128 / 129, pack returning 0 and 1, the two forms on both sides of
    hSize < maxSymbolValue / 2, fse_normalize_slow, and a description that cannot be written (stored raw)."""
    rng = np.random.default_rng(seed)
    out = []
    for ms in (127, 128, 129):
        for k in (2, 9, 40):   # k symbols up to max_sym, one of them max_sym
            syms = np.sort(rng.choice(ms, k - 1, replace=False))
            syms = np.append(syms, ms)
            p = rng.dirichlet(np.ones(k))
            c = np.maximum((p * plen).astype(np.int64), 1)
            c[0] += plen - int(c.sum())
            if c[0] > 0:
                out.append((f"maxsym{ms}-k{k}", _place(c, syms)))
    # pack returns 1: every weight equal -- max_sym + 1 symbols, all present, equal counts
    for k in (4, 16, 64):
        c = np.full(k, plen // k, np.int64)
        c[-1] += plen - int(c.sum())
        out.append((f"packrle{k}", _place(c, np.arange(k))))
    # pack returns 0: every weight at most once -- the weights of symbols 0..max_sym-1 all distinct (absent = 0)
    for k in (3, 4, 5):
        f = fib_counts(k, 0.0, rng)
        c = _fit(f, plen)
        if c is not None:
            out.append((f"packdistinct{k}", _place(c, np.arange(k))))
    # fse_normalize_slow: the weights of a small alphabet spread over many values, so that rounding hands out more
    # slots than the tANS table has.  Counts 2^(L - length) give a Huffman table of exactly those lengths.
    found = 0
    for _ in range(4000):
        L = int(rng.integers(6, 12))
        alphabet = int(rng.integers(8, 17))
        nsym = int(rng.integers(2, alphabet + 1))
        try:
            nb = P.kraft_lengths(rng, nsym, L, alphabet=alphabet)
        except AssertionError:
            continue
        c = np.where(nb > 0, 1 << (L - nb.astype(np.int64)), 0)
        c = _fit(c, plen)
        if c is not None and "normalize_slow" in table(c).trace:
            out.append((f"slow{alphabet}-{found}", c))
            found += 1
            if found == 3:
                break
    return out


def search(hists, want: set, per: int = 3):
    """The histograms whose table takes each branch in `want`, at most `per` per branch, in order."""
    hit = {b: 0 for b in want}
    out = []
    for name, c in hists:
        t = table(c)
        new = [b for b in t.trace if b in hit and hit[b] < per]
        if new:
            for b in t.trace:
                if b in hit:
                    hit[b] += 1
            out.append((name, c, t.trace))
    return out, hit


# A 4252-byte histogram over 205 symbols that a seeded search found: its weights spread over enough values that
# fse_normalize falls back to fse_normalize_slow, and the tANS header still wins over raw nibbles, so the slow path's
# output reaches the stream.  (On small alphabets the slow path's header always loses to the nibbles.)
SLOW_FSE = [3, 6, 13, 0, 66, 54, 1, 0, 3, 2, 2, 0, 5, 9, 0, 2, 6, 9, 1, 2, 50, 2, 0, 0, 33, 14, 19, 46, 29, 1, 28, 0,
            3, 17, 6, 6, 0, 13, 35, 32, 27, 86, 17, 2, 24, 7, 48, 3, 47, 10, 0, 20, 81, 5, 0, 54, 0, 7, 1, 12, 8, 17,
            17, 36, 4, 0, 0, 13, 1, 25, 11, 10, 12, 80, 2, 0, 22, 21, 3, 5, 50, 5, 21, 3, 19, 2, 0, 68, 25, 45, 4, 3,
            76, 21, 38, 24, 2, 0, 1, 2, 3, 9, 11, 11, 12, 11, 15, 3, 3, 0, 0, 2, 0, 20, 8, 1, 34, 2, 21, 4, 13, 9, 2,
            0, 11, 6, 0, 0, 3, 76, 3, 19, 37, 3, 9, 5, 9, 2, 0, 10, 0, 42, 1, 6, 61, 1, 8, 0, 0, 22, 30, 0, 1, 22, 2,
            0, 38, 0, 2, 65, 22, 6, 40, 4, 3, 88, 0, 68, 4, 0, 17, 0, 0, 40, 7, 3, 2, 2, 18, 0, 2, 32, 77, 2, 5, 77,
            19, 1, 17, 6, 2, 27, 0, 41, 4, 4, 56, 41, 3, 25, 90, 0, 2, 1, 72, 11, 0, 6, 28, 5, 0, 11, 26, 51, 94, 71,
            5, 14, 23, 17, 21, 7, 11, 83, 16, 71, 3, 5, 10, 3, 10, 1, 1, 10, 0, 2, 11, 4, 19, 18, 24, 5, 0, 4, 4, 30,
            85, 0, 63, 11, 54, 2, 11, 4, 1, 3]


def edge_histograms(plen: int, seed: int):
    """The histogram early-outs: the most frequent byte at plen (RLE), plen - 1, (plen >> 7) + 4 (raw by the
    heuristic) and + 5 (built), and small planes whose table description has hsize + 12 at plen - 1, plen, plen + 1."""
    out = [("rle", _place(np.array([plen]), np.array([7])))]
    if plen >= 2:
        out.append(("largest-plen-1", _place(np.array([plen - 1, 1]), np.array([3, 200]))))
    for d in (4, 5):
        top = (plen >> 7) + d
        if top >= plen:
            continue
        rest = plen - top
        k = -(-rest // top)   # other symbols of at most `top` each
        if k > 255:
            continue
        c = np.full(k, rest // k, np.int64)
        c[: rest % k] += 1
        out.append((f"largest-heur+{d}", _place(np.concatenate([[top], c]), np.arange(k + 1))))
    rng = np.random.default_rng(seed)
    want = {plen - 13: 0, plen - 12: 0, plen - 11: 0}   # hsize + 12 = plen - 1, plen, plen + 1
    for _ in range(20000):
        if all(v >= 2 for v in want.values()) or not 16 <= plen <= 48:
            break
        k = int(rng.integers(2, min(plen, 200)))
        if plen - k + 1 <= (plen >> 7) + 5:
            continue
        c = np.ones(k, np.int64)
        c[0] = int(rng.integers((plen >> 7) + 5, plen - k + 2))
        c[rng.integers(1, k, max(0, plen - int(c.sum())))] += 1
        c[0] += plen - int(c.sum())
        if c[0] < c[1:].max() or c[0] == plen:
            continue
        syms = np.sort(rng.choice(256, k, replace=False))
        h = table(_place(c, syms))
        hs = len(h.hdr) if h.hdr is not None else -1
        if hs in want and want[hs] < 2:
            want[hs] += 1
            out.append((f"hsize{hs}+12-vs-{plen}", _place(c, syms)))
    return out


# ---------------------------------------------------------------- planes: a histogram in an order
ORDERS = ("shuffled", "clustered", "short_first", "alternating")


def plane_from_counts(counts, order: str, rng, nb=None) -> np.ndarray:
    """A plane with exactly this histogram, in one of ORDERS or "long_quarter" (the longest codes fill the first
    stream quarter(s))."""
    plane = rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), np.asarray(counts, np.int64)))
    if order == "shuffled":
        return plane
    if order == "clustered":
        return P.clustered(plane)
    nb = table(counts).nb if nb is None else nb
    by_len = plane[np.argsort(-nb[plane].astype(np.int32), kind="stable")]   # longest first
    if order == "long_quarter":   # quarter 0 ends with the longest codes: full tiles of them in both write kernels
        seg = (plane.size + 3) // 4
        out = by_len.copy()
        out[:seg] = by_len[:seg][::-1]
        return out
    if order == "short_first":
        return by_len[::-1].copy()
    if order == "alternating":
        out = np.empty_like(by_len)
        half = (by_len.size + 1) // 2
        out[0::2] = by_len[:half]
        out[1::2] = by_len[half:][::-1]
        return out
    raise ValueError(order)


def quarter_bits(plane: np.ndarray, nb: np.ndarray):
    seg = (plane.size + 3) // 4
    return [int(nb[plane[q * seg: min(plane.size, (q + 1) * seg)]].astype(np.int64).sum()) for q in range(4)]


def tune_residues(plane: np.ndarray, nb: np.ndarray, targets) -> np.ndarray:
    """Swap symbols between stream quarters 0-2 and quarter 3, a code of length a against one of a + 1, until the
    code bits of quarter q are targets[q] mod 32 (q < 3).  The histogram, and so the table, does not change."""
    plane = plane.copy()
    n = plane.size
    seg = (n + 3) // 4
    if seg == 0 or 3 * seg >= n:
        return plane
    for q in range(3):
        lens = nb[plane].astype(np.int64)
        need = (targets[q] - int(lens[q * seg: (q + 1) * seg].sum())) % 32
        for _ in range(need):
            lens = nb[plane].astype(np.int64)
            mine, last = lens[q * seg: (q + 1) * seg], lens[3 * seg:]
            done = False
            for a in np.unique(mine):
                i = np.nonzero(mine == a)[0]
                j = np.nonzero(last == a + 1)[0]
                if i.size and j.size:
                    x, y = q * seg + int(i[0]), 3 * seg + int(j[0])
                    plane[x], plane[y] = plane[y], plane[x]
                    done = True
                    break
            if not done:
                return plane
    return plane


def eleven_bit_counts(plen: int, need: int, seed: int):
    """Three heavy symbols over a flat tail of 200-256 symbols: the tail sits three levels down, at 11 bits, and
    holds up to about an eighth of the plane.  -> counts with at least `need` bytes coded at 11 bits."""
    rng = np.random.default_rng(seed)
    for _ in range(2000):
        k = int(rng.integers(200, 253))
        t = max(1, int(plen * rng.uniform(0.8, 1.05) / (8 * k)))
        tail = t * k
        h3 = int(tail * rng.uniform(1.0, 1.3))
        h2 = int((h3 + tail) * rng.uniform(1.0, 1.3))
        h1 = plen - h2 - h3 - tail
        if h1 <= 0:
            continue
        c = _place(np.concatenate([[h1, h2, h3], np.full(k, t)]), np.arange(k + 3))
        tb = table(c)
        if tb.lg == 11 and int(c[tb.nb == 11].sum()) >= need:
            return c
    raise AssertionError(f"no 11-bit tail of {need} bytes at plen {plen}")


# ---------------------------------------------------------------- the cases: crafted planes packed into tensors
def catalog(plen: int, seed: int, depth_tries: int = 0):
    """(name, counts, order, branches) of every crafted plane of plen bytes: the searched depth-limited and small
    histograms (a few per limiter branch they reach), ties, weight headers and early-out edges, each in one of
    ORDERS in turn."""
    hists = []
    if depth_tries:
        picked, _ = search(depth_histograms(plen, depth_tries, seed), set(TRACE), per=2)
        hists += [(n, c) for n, c, _ in picked]
    if plen <= 8192:
        picked, _ = search(small_histograms(plen, 150, seed + 1), set(TRACE), per=2)
        hists += [(n, c) for n, c, _ in picked]
    hists += tie_histograms(plen)
    if plen >= 256:
        hists += header_histograms(plen, seed + 2)
    hists += edge_histograms(plen, seed + 3)
    return [(n, c, ORDERS[i % len(ORDERS)]) for i, (n, c) in enumerate(hists)]


class Case:
    """One tensor: `planes[c][g]` and their names, the stream settings, and the tensor bytes."""

    def __init__(self, name, G, bits, chunk, thr, planes, names):
        self.name, self.G, self.bits, self.chunk, self.thr = name, G, bits, chunk, thr
        self.planes, self.names = planes, names
        self.data = P.tensor_from_planes(planes, G, bits)
        self.kind = "small" if chunk % (64 * G) else ("ragged" if (self.data.size % chunk) % (64 * G) else "regular")

    def oracle(self) -> np.ndarray:
        from oracle import oracle as O
        return O.zipnn_compress(header(), self.data, self.G, self.bits, bytes_mode(self.G), self.chunk, self.thr, threads=2)


def _make_planes(specs, plen: int, rng, tune: bool):
    out, names = [], []
    for i, (name, c, order) in enumerate(specs):
        c = np.asarray(c, np.int64)
        assert int(c.sum()) == plen, (name, int(c.sum()), plen)
        nb = table(c).nb
        plane = plane_from_counts(c, order, rng, nb)
        if tune and order == "shuffled":
            plane = tune_residues(plane, nb, [(3 * i + q) % 32 for q in range(3)])
        out.append(plane)
        names.append(f"{name}/{order}")
    return out, names


def make_case(name, G, bits, chunk, thr, specs, last_plen=None, last_specs=(), seed=0, tune=True) -> Case:
    """Full chunks of chunk / G-byte planes from `specs` (cycled to fill whole chunks), then a last chunk of G planes
    of last_plen bytes from `last_specs` (cycled)."""
    rng = np.random.default_rng(seed)
    plen = chunk // G
    planes, names = _make_planes(specs, plen, rng, tune)
    k = -(-len(planes) // G)
    planes = [planes[(c * G + g) % len(planes)] for c in range(k) for g in range(G)]
    names = [names[(c * G + g) % len(names)] for c in range(k) for g in range(G)]
    chunks = [planes[c * G: (c + 1) * G] for c in range(k)]
    cnames = [names[c * G: (c + 1) * G] for c in range(k)]
    if last_plen:
        lp, ln = _make_planes(last_specs, last_plen, rng, tune)
        chunks.append([lp[g % len(lp)] for g in range(G)])
        cnames.append([ln[g % len(ln)] for g in range(G)])
    return Case(name, G, bits, chunk, thr, chunks, cnames)


@functools.lru_cache(maxsize=None)
def _catalogs():
    return {plen: catalog(plen, plen, depth_tries=300 if plen >= 2048 else 0)
            for plen in (32, 64, 1984, 2048, 2112, 4096, 32704, 40001, 131072)}


def cases(G: int, bits: int):
    """The tensors of one layout (all of them coded for one threshold each):
      big      131072-byte planes (warp kernel): depth-limited trees, ties, headers, edges, an 11-bit tail; last chunk
               of 32704-byte planes (stream quarters of 8176 bytes: the tile loop starts mid-tile)
      mid      2048-byte planes (table log 9-10) and a last chunk of 1984 (quarters of 512, then 496 bytes)
      mid2     4096-byte planes and a last chunk of 2112 (quarters of 528 bytes)
      ragged   65536-byte planes and a last chunk of 40001-byte planes (k_encode_write) with an 11-bit tail, at 1.5
      tiny64   64-byte planes (quarters of 16 bytes, warp kernel)
      tiny32   32-byte planes (chunk < 64 * G: k_encode_write writes every item), at 0.95, 1.0 and 1.5"""
    cat = _catalogs()
    s = 100 * G + bits
    eleven = lambda plen, need: [("eleven", eleven_bit_counts(plen, need, plen), "long_quarter")]   # noqa: E731
    out = [
        make_case(f"big-G{G}b{bits}", G, bits, 131072 * G, 0.95, cat[131072] + eleven(131072, 512),
                  32704, cat[32704] + eleven(32704, 512), seed=s),
        make_case(f"mid-G{G}b{bits}", G, bits, 2048 * G, 1.0, cat[2048], 1984, cat[1984], seed=s + 1),
        make_case(f"mid2-G{G}b{bits}", G, bits, 4096 * G, 0.95, cat[4096], 2112, cat[2112], seed=s + 2),
        make_case(f"ragged-G{G}b{bits}", G, bits, 65536 * G, 1.5, [("eleven65536", eleven_bit_counts(65536, 4096, 7),
                                                                    "long_quarter")] + list(depth_cases(65536)), 40001, eleven(40001, 4096) + cat[40001], seed=s + 3),
        make_case(f"tiny64-G{G}b{bits}", G, bits, 64 * G, 1.5, cat[64], seed=s + 4),
    ]
    for thr in THRESHOLDS:
        out.append(make_case(f"tiny32-G{G}b{bits}-{thr}", G, bits, 32 * G, thr, cat[32], seed=s + 5))
    return out


@functools.lru_cache(maxsize=None)
def depth_cases(plen: int):
    picked, _ = search(depth_histograms(plen, 200, plen), set(TRACE), per=1)
    return tuple((n, c, ORDERS[i % len(ORDERS)]) for i, (n, c, _) in enumerate(picked))


# ---------------------------------------------------------------- a produced stream, block by block
class Block:
    __slots__ = ("g", "c", "kind", "kernel", "off", "hsize", "form", "lg", "starts", "sbytes", "bits", "lengths")


def parse(stream: np.ndarray, case: Case, base_addr: int = 0):
    """Per (group, chunk): kind (raw / rle / huf), the kernel that wrote it ("warp" or "general"), its absolute
    address (base_addr + offset), and for coded blocks the table log, header size and form ("fse" / "nibble"),
    code lengths, the absolute address, byte size and code-bit total of each bitstream."""
    hl = len(header())
    pr = P.predict(stream[hl:], case.G, case.bits, case.chunk, case.data.size)
    out = []
    for g in range(case.G):
        for c in range(pr["K"]):
            it = pr["items"][g][c]
            b = Block()
            b.g, b.c, b.kind = g, c, it.kind
            clen = min(case.chunk, case.data.size - c * case.chunk)
            b.kernel = "warp" if clen % (64 * case.G) == 0 and case.kind != "small" else "general"
            b.off = base_addr + hl + it.src_off
            if it.kind == "huf":
                blk = stream[hl + it.src_off: hl + it.src_off + it.src_len]
                b.hsize, b.lg, b.lengths = it.hsize, it.lg, it.lengths
                b.form = "fse" if blk[0] < 128 else "nibble"
                b.sbytes = list(it.s_len)
                b.starts, b.bits, at = [], [], it.hsize + 6
                for q in range(4):
                    b.starts.append(b.off + at)
                    last = int(blk[at + b.sbytes[q] - 1])
                    b.bits.append(8 * (b.sbytes[q] - 1) + last.bit_length() - 1)
                    at += b.sbytes[q]
            out.append(b)
    return out


def full_tiles_of(plane: np.ndarray, lengths: np.ndarray, tile: int, L: int) -> int:
    """Full emission tiles (tile plane bytes from the end of a stream quarter) whose codes are all L bits."""
    seg = (plane.size + 3) // 4
    n = 0
    for q in range(4):
        part = lengths[plane[q * seg: min(plane.size, (q + 1) * seg)]]
        for end in range(part.size, tile - 1, -tile):
            n += bool(np.all(part[end - tile: end] == L))
    return n
