"""Host side of the box tests (test_boxes_gpu.py): a model of how the slice entry points split a box into pieces,
the box generator, and a classifier of which output store site and store class every box reaches.

The per-bitstream-CTA decoder writes a box through three store sites:
  merge   the fused-mode merge of sync_process (decode_sync.cuh): fused-mode chunks;
  regroup regroup_tile<G, true> (decode.cuh), from k_regroup_batch or the overflow kernel: plain, general and
          overflow chunks, 16 decoded bytes per store;
  put     box_put: the bytes of a chunk behind its last whole 16 bytes (a ragged last chunk, chunks under 16 bytes).
and each site has two store classes, fixed per piece: `fast` (base, pitch and len multiples of 16: one uint4 store)
and `bytes` (byte by byte).  The tests here check the piece model against the contract the C code documents
(zipnn_b200.cu, slice_pieces) and that the generated boxes reach every (site, class, chunk mode) the layouts allow.
"""
from __future__ import annotations

import functools
from math import gcd

import numpy as np

import test_decoder_tables_gpu as D
from test_slicing_host import cut_box

DEFAULT_LIMIT = 16384   # kSyncTablesMaxChunks: covering chunks above which a box is split (ZIPNN_B200_SLICE_PIECE_CHUNKS)
POOL_SLOTS, OVERFLOW_CTAS = 64, 32   # kDefaultSlots, kOverflowCtas
LIMITS = (2, 3, 7)      # the lowered piece limits the GPU tests run with
DEFAULT_CHUNK = {1: 131072, 2: 262144, 4: 262144}
DTYPE = {1: "fp8", 2: "bf16", 4: "fp32"}
CLASSES = ("fast", "bytes")


def round_up(v: int, a: int) -> int:
    return (v + a - 1) // a * a


# ------------------------------------------------------------------ the piece model (zipnn_b200.cu, slice_pieces)
class Piece:
    __slots__ = ("base", "rows", "pitch", "len", "out_off", "c0", "c1", "how")

    def __init__(self, base, rows, pitch, length, out_off, chunk, how):
        if rows == 1:
            pitch = round_up(length, 16)   # (one row: the pitch only keeps the store path's invariants)
        self.base, self.rows, self.pitch, self.len, self.out_off, self.how = base, rows, pitch, length, out_off, how
        self.c0 = base // chunk
        self.c1 = (base + (rows - 1) * pitch + length + chunk - 1) // chunk

    @property
    def box(self):
        return (self.base, self.rows, self.pitch, self.len)

    @property
    def fast(self) -> bool:
        return ((self.base | self.pitch | self.len) & 15) == 0


def valid_box(orig: int, box) -> bool:
    """What the host code accepts (E_ARG otherwise); empty boxes are valid."""
    base, rows, pitch, length = box
    if rows == 0 or length == 0:
        return True
    if base > orig or length > orig - base:
        return False
    return rows == 1 or (length <= pitch and rows - 1 <= (orig - base - length) // pitch)


def pieces_of(box, chunk: int, limit: int = DEFAULT_LIMIT) -> list:
    """The pieces of a valid box, in output order.  `how` says which rule made them: 'bytes' (one run, split at
    chunk boundaries when it covers more than `limit` chunks), 'rows' (groups of R rows, R a multiple of
    m = 16 / gcd(len, 16)), 'm_rows' (R raised to m: m rows of an odd length span more than the limit), 'each_row'
    (rows longer than a piece, each one a run)."""
    base, rows, pitch, length = box
    if rows == 0 or length == 0:
        return []
    out = []

    def run(b, e, off, how):
        unit = max(chunk, 16)
        per = limit * chunk // unit
        step = per - 1 if per > 1 else 1
        delta = b & 15
        while b < e:
            p = min(e, (b // unit + step) * unit + delta)
            out.append(Piece(b, 1, 0, p - b, off, chunk, how))
            off += p - b
            b = p

    if rows == 1 or pitch == length:
        run(base, base + rows * length, 0, "bytes")
    else:
        m = 16 // gcd(length, 16)
        span = (limit - 1) * chunk
        R = (span - length) // pitch + 1 if span >= length else 0
        R = R // m * m
        if R == 0 and m == 1:
            for r in range(rows):
                run(base + r * pitch, base + r * pitch + length, r * length, "each_row")
        else:
            how = "rows" if R else "m_rows"
            R = max(R, m)
            for r0 in range(0, rows, R):
                out.append(Piece(base + r0 * pitch, min(R, rows - r0), pitch, length, r0 * length, chunk, how))
    return out


def piece_overflows(piece: Piece, general: int, K: int, G: int, chunk: int) -> bool:
    """Does a piece send some of its `general` chunks to the overflow kernel?  Its plane pool is sized for
    min(kc, 64 + 32) slots of kc covering chunks (rounded up to 256 bytes); 32 of them belong to the overflow CTAs
    unless the pool holds the whole stream (fill_decode_cfg)."""
    kc = piece.c1 - piece.c0
    slots = kc if kc <= POOL_SLOTS else POOL_SLOTS + OVERFLOW_CTAS
    ps = round_up(chunk // G, 16) + 16
    have = round_up(slots * G * ps, 256) // (G * ps)
    if have >= K:
        return False
    max_slots = have - OVERFLOW_CTAS if have > OVERFLOW_CTAS else have
    assert general <= max_slots or have > OVERFLOW_CTAS, "a general chunk without a slot: the decode would fail"
    return general > max_slots


# ------------------------------------------------------------------ which store sites a box reaches
def box_meets(box, a: int, n: int) -> bool:
    """The kernels' rule (decode.cuh, box_meets): does the box hold a byte of [a, a + n)?"""
    base, rows, pitch, length = box
    e0 = base + length
    r = 0 if a < e0 else (a - e0) // pitch + 1
    return r < rows and base + r * pitch < a + n


def classify(case, box, limit: int = DEFAULT_LIMIT):
    """-> (pieces, {(site, class, chunk mode)}) for a box of a planes case."""
    pr, chunk, orig, G = case.pr, case.chunk, case.data.size, case.G
    K = pr["K"]
    pieces = pieces_of(box, chunk, limit)
    hit = set()
    for p in pieces:
        cls = "fast" if p.fast else "bytes"
        met = []
        for c in range(p.c0, p.c1):
            clen = min(chunk, orig - c * chunk)
            if box_meets(p.box, c * chunk, clen):
                met.append((c, clen))
        general = sum(1 for c, _ in met if pr["mode"][c] == "general")
        over = piece_overflows(p, general, K, G, chunk)
        for c, clen in met:
            mode = pr["mode"][c]
            if mode == "fused":
                hit.add(("merge", cls, "fused"))
                continue
            if mode == "general" and over:
                mode = "overflow"   # (which general chunks pass the pool is decided at run time: the piece's)
            vec = clen // 16 * 16
            if vec and box_meets(p.box, c * chunk, vec):
                hit.add(("regroup", cls, mode))
            if vec < clen and box_meets(p.box, c * chunk + vec, clen - vec):
                hit.add(("put", cls, mode))
    return pieces, hit


# Every combination the layouts allow.  Fused chunks are whole multiples of 512 bytes: only the merge writes them.
# box_put with the fast class needs chunks under 16 bytes (a fast box ends on a 16-byte boundary, in front of a
# ragged tail), and chunks that small never code a plane: they are plain.
ALLOWED = {("merge", cls, "fused") for cls in CLASSES} | \
    {("regroup", cls, mode) for cls in CLASSES for mode in ("plain", "general", "overflow")} | \
    {("put", "bytes", mode) for mode in ("plain", "general", "overflow")} | {("put", "fast", "plain")}


# ------------------------------------------------------------------ the streams
def _stream_specs(G: int):
    """(name, dtype, chunk, tops, side, last, modes it must have)."""
    dt = DTYPE[G]
    dflt = DEFAULT_CHUNK[G]
    specs = []
    for chunk in sorted({G, 8}):
        tops = ["raw" if c % 3 else "const" for c in range(150)]
        specs.append((f"tiny{chunk}", dt, chunk, tops, None, chunk - 1 if chunk > 1 else None, {"plain"}))
    # chunks of 64 bytes: coded planes make general chunks (not a multiple of 512), 400 of them: overflow
    tops = ["raw" if c % 11 == 5 else ("const" if c % 11 == 8 else "geo5") for c in range(400)]
    specs.append(("c64", dt, 64, tops, None, 37, {"plain", "general"}))
    # 512 bytes: fused chunks, a run of 100 general chunks (a second coded plane; fp8: none), plain ones
    tops = ["const" if c % 7 == 3 else "geo5" for c in range(300)]
    side = (lambda c, g: "geo5" if g == G - 2 and 100 <= c < 200 else "raw") if G > 1 else None
    specs.append(("c512", dt, 512, tops, side, 333, {"fused", "plain"} | ({"general"} if G > 1 else set())))
    # 4096 and the default chunk: every mode, a ragged last chunk of an odd length
    tops = ["raw" if c % 4 == 2 else ("const" if c % 4 == 3 else "geo5") for c in range(41)]
    side = (lambda c, g: "geo5" if g == G - 2 and c % 4 == 1 else "raw") if G > 1 else None
    specs.append(("c4096", dt, 4096, tops, side, 1001, {"fused", "plain", "general"}))
    if G == 2:
        specs.append(("c4096_fp16", "fp16", 4096, tops, side, 1001, {"fused", "plain", "general"}))
    specs.append(("cdef", dt, dflt, ["geo5", "geo5", "raw", "geo5"], side, 70001,
                  {"fused", "plain", "general"}))
    return specs


@functools.lru_cache(maxsize=None)
def box_streams(G: int) -> list:
    """The planes cases of one byte-group count, each asserted to hold the chunk modes it was built for."""
    out = []
    for i, (name, dtype, chunk, tops, side, last, modes) in enumerate(_stream_specs(G)):
        case = D.planes_case(f"{name}_G{G}", dtype, chunk, tops, seed=400 + 10 * G + i, last=last, side=side)
        got = set(case.pr["mode"])
        assert modes <= got, (case.name, modes, got)
        if last:
            assert last % 16 and (G == 1 or last % G), last   # a ragged last chunk: a tail for box_put
            assert case.pr["mode"][-1] != "fused"
        out.append(case)
    return out


# ------------------------------------------------------------------ the boxes
def _edge_lists(chunk: int, orig: int):
    bases = [0, 1, 15, 16, 17, chunk - 1, chunk, chunk + 1] + [4096 * k + d for k in (1, 2, 3) for d in (-1, 1)] + ["end"]
    lens = [1, 2, 15, 16, 17, 31, "pitch"]
    pitches = list(range(1, 16)) + [16, 48, 4080, 4095, 4096, 4097, 4112, chunk - 16, chunk + 16, 3 * chunk + 1]
    return bases, lens, [p for p in pitches if p >= 1], [1, 2, 3, "max"]


def gen_boxes(orig: int, chunk: int, seed: int, n: int = 28) -> list:
    """Seeded boxes drawn from the edge lists, then the whole tensor, its first and last byte and two empty boxes.
    Every box is valid; duplicates are dropped."""
    rng = np.random.default_rng(seed)
    bases, lens, pitches, rows_l = _edge_lists(chunk, orig)
    out = []
    tries = 0
    while len(out) < n and tries < 50 * n:
        tries += 1
        pitch = int(pitches[rng.integers(len(pitches))])
        ln = lens[rng.integers(len(lens))]
        ln = pitch if ln == "pitch" else min(int(ln), pitch)
        if ln > orig:
            continue
        want_rows = rows_l[rng.integers(len(rows_l))]
        b = bases[rng.integers(len(bases))]
        if b == "end":
            rows = (orig - ln) // pitch + 1 if want_rows == "max" else min(int(want_rows), (orig - ln) // pitch + 1)
            b = orig - ln - (rows - 1) * pitch
        else:
            b = int(b)
            if b + ln > orig:
                continue
            fit = (orig - b - ln) // pitch + 1
            rows = fit if want_rows == "max" else min(int(want_rows), fit)
        box = (b, rows, pitch, ln)
        assert valid_box(orig, box)
        if box not in out:
            out.append(box)
    o16 = orig // 16 * 16
    fixed = [(0, 1, orig, orig), (0, 1, 1, 1), (orig - 1, 1, 1, 1), (5, 0, 16, 16), (16, 3, 48, 0)]
    if o16 >= 64:   # the whole tensor up to its last 16-byte boundary, and a band of every 48-byte row: fast boxes
        fixed += [(0, 1, o16, o16), (16, (orig - 48) // 48 + 1, 48, 32)]
    return out + [b for b in fixed if b not in out]


def boxes_of(case) -> list:
    """The boxes of one stream (seeded by its name)."""
    return gen_boxes(case.data.size, case.chunk, seed=sum((i + 1) * ord(ch) for i, ch in enumerate(case.name)))


def expect(case, box) -> np.ndarray:
    """The box cut from the original bytes (cut_box; a strided view for boxes of many rows)."""
    base, rows, pitch, ln = box
    if rows * ln == 0:
        return np.zeros(0, np.uint8)
    if rows <= 256:
        return cut_box(case.data, box)
    view = np.lib.stride_tricks.as_strided(case.data[base:], (rows, ln), (pitch, 1), writeable=False)
    return np.ascontiguousarray(view).reshape(-1)


# ------------------------------------------------------------------ tests of the model
def _check_contract(box, chunk, limit, orig):
    pieces = pieces_of(box, chunk, limit)
    base, rows, pitch, ln = box
    if rows * ln == 0:
        assert pieces == []
        return pieces
    pos = np.arange(orig, dtype=np.int64)
    want = cut_box(pos, box)
    got = np.concatenate([cut_box(pos, p.box) for p in pieces])
    assert np.array_equal(got, want), (box, chunk, limit)
    at = 0
    for p in pieces:
        assert p.out_off == at and p.out_off % 16 == 0, (box, chunk, limit, p.out_off)
        assert p.rows >= 1 and p.len >= 1 and p.len <= p.pitch
        assert p.c0 * chunk <= p.base and p.c1 * chunk >= p.base + (p.rows - 1) * p.pitch + p.len
        at += p.rows * p.len
        if p.c1 - p.c0 > limit:
            # the two documented exceptions: m rows of an odd length span more than the limit, or, where `limit`
            # chunks are less than two 16-byte units, a run piece of one unit covers more than `limit` small chunks
            m = 16 // gcd(p.len, 16)
            assert (p.how == "m_rows" and p.rows <= m) or (limit * chunk < 32 and p.rows == 1 and p.len <= 16), \
                (box, chunk, limit, p.box, p.how)
    return pieces


def test_piece_model_tiles_every_box():
    """Random valid boxes at every chunk size and limit: the pieces tile the box in output order, every piece output
    is 16-byte aligned, and no piece covers more than `limit` chunks outside the documented exceptions."""
    rng = np.random.default_rng(1)
    hows = set()
    for chunk in (1, 2, 4, 8, 16, 64, 512, 4096):
        for limit in (2, 3, 5, 7, 64):
            orig = int(rng.integers(1, 60)) * max(chunk, 16) + int(rng.integers(0, 40))
            for _ in range(60):
                pitch = int(rng.integers(1, min(orig, 3 * max(chunk, 16) + 40) + 1))
                ln = int(rng.integers(1, pitch + 1))
                if ln > orig:
                    continue
                base = int(rng.integers(0, orig - ln + 1))
                rows = int(rng.integers(1, (orig - base - ln) // pitch + 2))
                pieces = _check_contract((base, rows, pitch, ln), chunk, limit, orig)
                if len(pieces) > 1:
                    hows.update(p.how for p in pieces)
    assert hows == {"bytes", "rows", "m_rows", "each_row"}, hows


def test_piece_model_at_the_real_limit():
    """A run of 16384 + 1 chunks splits in two; a multi-row box is grouped into rows of m."""
    chunk = 262144
    p = pieces_of((0, 1, 1 << 33, 1 << 33), chunk)
    assert len(p) == 3 and all(q.c1 - q.c0 <= DEFAULT_LIMIT for q in p) and p[0].c1 - p[0].c0 == DEFAULT_LIMIT - 1
    band = pieces_of((100, 262144, 32768, 2002), chunk)   # a column band of every row of 8 GiB
    assert [q.how for q in band] == ["rows"] * len(band) and len(band) == 3
    assert all(q.rows % 8 == 0 for q in band[:-1]) and all(q.c1 - q.c0 <= DEFAULT_LIMIT for q in band)


def test_rejections_model():
    orig = 1000
    assert not valid_box(orig, (orig - 9, 1, 16, 10))          # one byte past orig
    assert not valid_box(orig, (0, 2, 16, 17))                 # len > pitch with rows > 1
    fit = (orig - 3 - 5) // 16 + 1
    assert valid_box(orig, (3, fit, 16, 5)) and not valid_box(orig, (3, fit + 1, 16, 5))
    assert valid_box(orig, (orig + 5, 0, 1, 1)) and valid_box(orig, (0, 1, 1, 0))


def test_expect_matches_cut_box():
    rng = np.random.default_rng(2)
    data = rng.integers(0, 256, 50000, dtype=np.uint8)

    class C:
        pass
    c = C()
    c.data = data
    for box in ((3, 300, 100, 7), (0, 999, 50, 50), (17, 257, 3, 1), (5, 0, 4, 4)):
        assert np.array_equal(expect(c, box), cut_box(data, box)) if box[1] else expect(c, box).size == 0


def test_generated_boxes_reach_every_store_site_and_class():
    """The boxes of the GPU tests reach every (store site, store class, chunk mode) the layouts allow, every
    rule that splits a box under the lowered limits, and boxes of every kind (empty, whole, first and last byte,
    pitches around 4096 and below 16 and above a chunk, overflow chunks inside a multi-row box)."""
    hit, hows = set(), {lim: set() for lim in LIMITS}
    multi_row_overflow = 0
    kinds = set()
    for G in (1, 2, 4):
        for case in box_streams(G):
            for box in boxes_of(case):
                assert valid_box(case.data.size, box)
                pieces, h = classify(case, box)
                hit |= h
                if box[1] > 1 and any(k[2] == "overflow" for k in h):
                    multi_row_overflow += 1
                base, rows, pitch, ln = box
                if rows > 1:
                    kinds.add("pitch<16" if pitch < 16 else ("pitch~4096" if 4080 <= pitch <= 4112 else
                                                                ("pitch>chunk" if pitch > case.chunk else "other")))
                if rows * ln == 0:
                    kinds.add("empty")
                elif box == (0, 1, case.data.size, case.data.size):
                    kinds.add("whole")
                for lim in LIMITS:
                    split = pieces_of(box, case.chunk, lim)
                    if len(split) > 1:
                        hows[lim].update(p.how for p in split)
    assert hit == ALLOWED, (sorted(ALLOWED - hit), sorted(hit - ALLOWED))
    assert multi_row_overflow > 0
    assert {"pitch<16", "pitch~4096", "pitch>chunk", "empty", "whole"} <= kinds, kinds
    for lim in LIMITS:
        assert {"bytes", "rows", "m_rows", "each_row"} <= hows[lim], (lim, hows[lim])

