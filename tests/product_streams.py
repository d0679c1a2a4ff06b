"""Compressed weights for the product tests (test_product_streams_host.py, _gpu.py): streams of every kind the
decoder tests use, each one a matrix the matvec and the matmul must multiply by.  The builders also make the fp8
corpus (fp8_streams.py): a Case takes any weight dtype of the products, fp8 ones included.

A case is a tensor [out, in] of bf16, fp16 or fp32 in either byte layout (`bits`: 1 = the sign bit rotated next to
the mantissa, 0 = not; a stream's layout comes from its header, not from the dtype, so every dtype is built in
both), its dense bytes and an oracle-made stream body.  Every case is fused in every chunk (asserted here from the
stream with `plane_inputs.predict`), so no case multiplies by nothing.  The inventory:

  shapes      every fused chunk size from 512 B to 256 KiB on rows shorter than a quarter, rows spanning many
              chunks, in = 8, 24, 136 and 520, out = 1, a one-chunk tensor and a short last chunk; the weights are
              `exact_weights`, so the same cases carry the one-hot extraction and the exact sums
  families    a top plane from every plane_inputs family that stays fused, per chunk
  crafted     code tables of logs 1 to 11 that the reference encoder never writes, a hot 11-bit symbol, the tail
              pool warp mixes of the fused kernel, and fixed-length codes whose CTA segment guesses are misaligned
  ring        bitstreams longer than the 28 KiB the sync decoder keeps in shared memory, in whole chunks
  rle         low planes that are constant (RLE) in some chunks and raw in others
  special     inf, NaN, -0, bf16 exponent-0 and fp16 subnormal weights at known positions

Except in `special`, the top-plane symbols that could encode an all-ones exponent are remapped before the stream is
made (`safe_top`), and every weight is finite: one infinity would turn a whole product row into NaN and that row
would check nothing.
"""
from __future__ import annotations


import functools

import numpy as np
import torch

import plane_inputs as P
import test_decoder_tables_gpu as D
from oracle import oracle as O

TORCH = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32, "e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
ES = {"bf16": 2, "fp16": 2, "fp32": 4, "e4m3": 1, "e5m2": 1}
# the weights' code in their product call: ZIPNN_B200_MATVEC_BF16 / FP16 / FP32, ZIPNN_B200_FP8_E4M3 / E5M2
CODE = {"bf16": 0, "fp16": 1, "fp32": 2, "e4m3": 0, "e5m2": 1}
BYTES_MODE = {1: 10, 2: 10, 4: 220}
CHUNKS = tuple(512 << i for i in range(10))   # every chunk size a fused chunk can have: 512 B .. 256 KiB
LAYOUTS16 = (("bf16", 1), ("bf16", 0), ("fp16", 1), ("fp16", 0))
LAYOUTS = LAYOUTS16 + (("fp32", 1), ("fp32", 0))
MATMUL_NT, MATVEC_NT = 64, 8   # rows of x per call of a one-hot sweep


# ---------------------------------------------------------------- the top plane and the exponent
def exp_all_ones(dtype: str, bits: int, sym: np.ndarray) -> np.ndarray:
    """Which top-plane bytes can be part of an element whose exponent is all ones, in this layout."""
    s = np.asarray(sym, dtype=np.uint8)
    if dtype == "fp16":
        # rotated: the top byte is exponent(5) mantissa(3); not rotated: sign exponent(5) mantissa(2)
        return (s & 0xF8) == 0xF8 if bits else (s & 0x7C) == 0x7C
    # bf16 / fp32 rotated: the top byte is the exponent; not rotated: sign and the exponent's upper 7 bits
    return s == 0xFF if bits else (s & 0x7F) == 0x7F


def safe_top(dtype: str, bits: int, plane: np.ndarray) -> np.ndarray:
    """The plane with every symbol that could encode an all-ones exponent moved to one that cannot: an unused value
    where there is one (the histogram keeps its shape), else the value with bit 6 cleared (bit 6 is part of the
    exponent field in every layout, so the exponent is no longer all ones)."""
    out = np.asarray(plane, dtype=np.uint8).copy()
    present = np.zeros(256, dtype=bool)
    present[out] = True
    bad = np.nonzero(present & exp_all_ones(dtype, bits, np.arange(256)))[0]
    free = [v for v in range(256) if not present[v] and not exp_all_ones(dtype, bits, np.uint8(v))]
    for v in bad:
        to = free.pop(0) if free else v ^ 0x40
        out[out == v] = to
    return out


def safe_lengths(nb: np.ndarray, bad) -> np.ndarray:
    """Code lengths with every coded symbol that `bad` marks (one that could make a weight that is not finite, as
    `exp_all_ones` does) swapped with an uncoded one below 129 that it does not (raw 4-bit weights describe at most
    129 symbols)."""
    nb = np.asarray(nb, dtype=np.uint8).copy()
    free = [v for v in range(129) if nb[v] == 0 and not bad(np.uint8(v))]
    for v in np.nonzero((nb > 0) & bad(np.arange(256)))[0]:
        to = free.pop(0)
        nb[to], nb[v] = nb[v], 0
    return nb


# ---------------------------------------------------------------- a case
def tag(dtype: str, bits: int) -> str:
    """A layout in case names: dtype and bit order, or the dtype alone for one-byte weights (num_buf 1 has no bit order)."""
    return dtype if ES[dtype] == 1 else f"{dtype}b{bits}"


class Case:
    def __init__(self, name, dtype, bits, chunk, shape, data, body=None, special=False):
        self.name, self.dtype, self.bits, self.chunk, self.special = name, dtype, bits, chunk, special
        self.G, self.code = ES[dtype], CODE[dtype]
        self.bm = BYTES_MODE[self.G]
        self.data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        self.out, self.inn = shape
        assert self.out * self.inn * self.G == self.data.size, (name, shape, self.data.size)
        if body is None:
            body = O.zipnn_compress(bytes(32), self.data, self.G, bits, self.bm, chunk, 0.95, threads=8)[32:]
        self.body = np.ascontiguousarray(body, dtype=np.uint8)
        self.pr = P.predict(self.body, self.G, bits, chunk, self.data.size)
        assert self.pr["mode"] == ["fused"] * self.pr["K"], (name, self.pr["mode"])
        if not special:
            assert bool(torch.isfinite(self.weights().float()).all()), f"{name}: a weight that is not finite"

    @property
    def shape(self):
        return (self.out, self.inn)

    def weights(self) -> torch.Tensor:
        """W [out, in] on the host."""
        return torch.from_numpy(self.data.copy()).view(TORCH[self.dtype]).reshape(self.out, self.inn)

    def floats(self) -> np.ndarray:
        """W as float32 (exact)."""
        return self.weights().float().numpy()

    def top_items(self):
        return [self.pr["items"][self.G - 1][c] for c in range(self.pr["K"])]

    def layout_planes(self):
        """The planes of every chunk (the oracle's split): what the stream codes."""
        return P.planes_of(self.data, self.G, self.bits, self.chunk)


def from_planes(name, dtype, bits, chunk, tops, seed, shape_in, side=None, last=None, safe=None):
    """A tensor whose chunk c has the top plane tops[c] (a family name or an array; `safe`, default `safe_top`, is
    applied) and the other planes side(c, g), a family name or function (default: uniform bytes, stored raw); rows of
    `shape_in` elements."""
    G = ES[dtype]
    safe = safe or functools.partial(safe_top, dtype, bits)
    rng = np.random.default_rng(seed)
    chunks = []
    for c, top in enumerate(tops):
        n = last if (last and c == len(tops) - 1) else chunk
        planes = []
        for g in range(G):
            m = P.plane_len(n, G, g)
            if g == G - 1:
                planes.append(safe(top[:m] if isinstance(top, np.ndarray) else P.FAMILIES[top](rng, m)))
            else:
                fam = side(c, g) if side else "raw"
                planes.append((fam if callable(fam) else P.FAMILIES[fam])(rng, m))
        chunks.append(planes)
    data = P.tensor_from_planes(chunks, G, bits)
    n = data.size // G
    assert n % shape_in == 0, (name, n, shape_in)
    return Case(name, dtype, bits, chunk, (n // shape_in, shape_in), data)


def crafted(name, dtype, bits, chunk, blocks, seed, shape_in, last=None, bad=None):
    """test_decoder_tables_gpu.crafted_case in any layout: blocks[c] = code lengths of chunk c's top plane, or
    (lengths, a hot symbol), or a family name (the oracle's block).  Lengths go through `safe_lengths` with `bad`
    (default `exp_all_ones`) first.  `seed` may be a numpy Generator, which goes on drawing."""
    G = ES[dtype]
    bad = bad or functools.partial(exp_all_ones, dtype, bits)
    rng = np.random.default_rng(seed)
    chunks, items = [], [[] for _ in range(G)]
    for c, spec in enumerate(blocks):
        n = last if (last and c == len(blocks) - 1) else chunk
        planes = [P.FAMILIES["raw"](rng, P.plane_len(n, G, g)) for g in range(G - 1)]
        m = P.plane_len(n, G, G - 1)
        hot = None
        if isinstance(spec, tuple):
            spec, hot = spec
        if isinstance(spec, str):
            top = safe_top(dtype, bits, P.FAMILIES[spec](rng, m))
        else:
            nb = safe_lengths(spec, bad)
            if hot is not None and nb[hot] == 0:   # the hot symbol was moved: follow it
                hot = int(np.nonzero(nb == np.asarray(spec)[hot])[0][-1])
            top = P.plane_for_lengths(rng, nb, m, hot)
        planes.append(top)
        chunks.append(planes)
        for g in range(G):
            if g == G - 1 and not isinstance(spec, str):
                blk = P.huf_block(nb, top)
                assert len(blk) < m - 1, (name, c, len(blk), m)
                items[g].append((1, blk))
            else:
                items[g].append(D._oracle_block(g, c, planes[g]))
    data = P.tensor_from_planes(chunks, G, bits)
    body = P.assemble_body(items, G)
    n = data.size // G
    assert n % shape_in == 0
    return Case(name, dtype, bits, chunk, (n // shape_in, shape_in), data, body=body)


# ---------------------------------------------------------------- exact weights and the shapes
SIG_BITS = {"bf16": 8, "fp16": 11, "fp32": 24}
EXPS = {"bf16": (-9, -8, -7, -6), "fp16": (-20, -19), "fp32": (-30, -29)}


def exact_weights(dtype: str, shape, seed: int) -> torch.Tensor:
    """s * m * 2^e with a full-width significand m (8 bits bf16, 11 fp16, 24 fp32: the low planes stay raw) and at
    least two exponents e: every product with x in {-1, 0, 1} is a multiple of 2^min(e)."""
    rng = np.random.default_rng(seed)
    b = SIG_BITS[dtype]
    m = rng.integers(1 << (b - 1), 1 << b, shape).astype(np.float64)
    e = rng.choice(EXPS[dtype], shape).astype(np.float64)
    s = rng.choice([-1.0, 1.0], shape)
    w = torch.from_numpy(s * m * 2.0 ** e).to(TORCH[dtype])
    assert torch.equal(w.double(), torch.from_numpy(s * m * 2.0 ** e)), "exact in the dtype"
    return w


def unit(dtype: str) -> float:
    """The smallest product of exact_weights with x = +-1."""
    return 2.0 ** min(EXPS[dtype])


def max_units(dtype: str) -> int:
    """The largest |w| of exact_weights, in units."""
    return ((1 << SIG_BITS[dtype]) - 1) << (max(EXPS[dtype]) - min(EXPS[dtype]))


def exact_x(dtype: str, nt: int, inn: int, seed: int) -> torch.Tensor:
    """x in {-1, 0, 1} with few enough non-zeros per row that sum |x w| < 2^24 units for any exact_weights row plus a
    bias of at most max_units: every partial sum is exact in fp32, in any order."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-1, 2, (nt, inn)).astype(np.float32)
    cap = ((1 << 24) - 1) // max_units(dtype) - 1
    for t in range(nt):
        nz = np.nonzero(x[t])[0]
        if nz.size > cap:
            x[t, rng.choice(nz, nz.size - cap, replace=False)] = 0
    return torch.from_numpy(x).to(TORCH[dtype])


def shapes(dtype: str, chunk: int) -> list:
    """(name, out, in) of the shape inventory at one chunk size; every tensor is a multiple of 512 bytes, so its short
    last chunk (if any) stays fused."""
    es = ES[dtype]
    ce = chunk // es
    out = [("narrow24", 2048, 24), ("narrow8", 4096, 8), ("in136", 384, 136), ("in520", 128, 520),
           ("long_row", 4, 32768 if es == 2 else 16384), ("out1", 1, 16384 if es == 2 else 8192),
           ("one_chunk", max(1, ce // 128), 128)]
    # three full chunks and a short one of a multiple of 512 bytes (rows of 512 bytes)
    row = 512 // es
    short = 1536 if chunk > 1536 else 512
    out.append(("short_last", (3 * chunk + short) // 512, row))
    return out


def shape_cases(chunk: int, dtypes=("bf16", "fp16", "fp32")) -> list:
    """The shape inventory at one chunk size.  The 16-bit layouts take turns over the shapes, so every layout meets
    every chunk size; fp32 (the matvec's only) in both layouts on alternate shapes."""
    cases = []
    for k, (name, out, inn) in enumerate(shapes("bf16", chunk)):
        if "bf16" in dtypes or "fp16" in dtypes:
            dt, bits = LAYOUTS16[(k + CHUNKS.index(chunk)) % 4]
            w = exact_weights(dt, (out, inn), 1000 * CHUNKS.index(chunk) + k)
            cases.append(Case(f"{name}_{dt}b{bits}_c{chunk}", dt, bits, chunk, (out, inn), w.view(torch.uint8).numpy()))
    if "fp32" in dtypes:
        for k, (name, out, inn) in enumerate(shapes("fp32", chunk)):
            if k % 2 == CHUNKS.index(chunk) % 2:
                bits = (k // 2) % 2
                w = exact_weights("fp32", (out, inn), 5000 + 1000 * CHUNKS.index(chunk) + k)
                cases.append(Case(f"{name}_fp32b{bits}_c{chunk}", "fp32", bits, chunk, (out, inn), w.view(torch.uint8).numpy()))
    return cases


# ---------------------------------------------------------------- plane families, crafted tables, rings, RLE
def family_names(dtype: str, bits: int, chunk: int = 4096) -> list:
    """The plane_inputs families whose top plane the oracle codes at this chunk in this layout (after safe_top)."""
    G = ES[dtype]
    rng = np.random.default_rng(3)
    m = chunk // G
    out = []
    for fam in P.FAMILIES:
        plane = safe_top(dtype, bits, P.FAMILIES[fam](rng, m))
        r, blk = O.huf_compress(plane)
        if r not in (0, 1, O.ERR) and len(blk) < 0.95 * m:
            out.append(fam)
    return out


def family_case(dtype: str, bits: int) -> Case:
    fams = family_names(dtype, bits)
    return from_planes(f"families_{dtype}b{bits}", dtype, bits, 4096, fams + fams[::-1], seed=10 + 2 * CODE[dtype] + bits,
                       shape_in=256 if ES[dtype] == 2 else 128)


def kraft_blocks(rng) -> list:
    """`crafted` blocks: random Kraft-complete tables of every log from 1 to 11, each twice (once with a hot longest
    code), and a hot symbol on an 11-bit code."""
    blocks = []
    for lg in range(1, 12):
        for hot in (False, True):
            nb = P.kraft_lengths(rng, int(rng.integers(lg + 1 if lg < 12 else 2, min(100, 1 << lg) + 1)), lg)
            blocks.append((nb, int(np.nonzero(nb == nb.max())[0][0])) if hot else nb)
    nb = P.kraft_lengths(rng, 100, 11)
    blocks.append((nb, int(np.nonzero(nb == 11)[0][0])))
    return blocks


def crafted_case(dtype: str, bits: int) -> Case:
    """The `kraft_blocks` tables, one 4 KiB chunk each."""
    blocks = kraft_blocks(np.random.default_rng(20 + 2 * CODE[dtype] + bits))
    return crafted(f"crafted_{dtype}b{bits}", dtype, bits, 4096, blocks, seed=30 + bits, shape_in=128)


def log12_case(bits: int) -> Case:
    """A bf16 stream with one table-log-12 block among ordinary ones (valid, but beyond the decoders' tables)."""
    rng = np.random.default_rng(90 + bits)
    nb12 = P.kraft_lengths(rng, 90, 12, min_len=2)
    blocks = ["geo5"] * 8
    blocks[5] = nb12
    return crafted(f"log12_bf16b{bits}", "bf16", bits, 4096, blocks, seed=91, shape_in=256)


def warp_mix_case(dtype: str, bits: int) -> Case:
    """The tail-pool warp mixes of test_decoder_tables_gpu.warp_mix_case (a pool filled exactly, overflowed at slots
    0, 3 and 7, every chunk demoted) without its constant and raw top planes, which would not be fused."""
    G = ES[dtype]
    chunk = 4096
    m = chunk // G
    pb = 5 if bits == 1 else 0
    cap = P.POOL_CAP[pb]
    by = D._planes_by_cut(m, pb)
    cuts = sorted(x for x in by if 0 < x <= cap)
    small, big = cuts[0], max(by)
    rows = [D._exact_fill(cuts, cap)]
    for s in (0, 3, 7):
        if pb == 0 and s == 0:
            continue
        before, rem = [], cap
        for i in range(s):
            x = max(x for x in cuts if x <= rem - (s - 1 - i) * small)
            before.append(x)
            rem -= x
        rows.append(before + [min(x for x in by if x > rem)] + [small] * (7 - s))
    if pb == 5:
        rows.append([big] * 8)
    tops = [D._pick(by, x, i) for row in rows for i, x in enumerate(row)]
    return from_planes(f"warps_{dtype}b{bits}", dtype, bits, chunk, tops, seed=40 + bits, shape_in=128, last=chunk - 512)


def misaligned_quarter(L: int, lo: int, hi: int, step: int) -> int:
    """Symbols per bitstream s (a multiple of `step`: 64 for 16-bit weights and 128 for fp8, so that the chunk is a
    multiple of 512 bytes) with s * L > 192 * 256 bits and a CTA segment of ceil(s * L / 256) bits that is not a
    multiple of L."""
    s = -(-lo // step) * step
    while s <= hi:
        if s * L > 192 * 256 and (-(-s * L // 256)) % L:
            return s
        s += step
    raise AssertionError((L, lo, hi))


def fixed_length_cases(dtype: str, bits: int, safe=None) -> list:
    """2^L equiprobable symbols (fixed-length codes, which never resynchronise), L = 2, 4, 6: a full chunk (256 KiB for
    16-bit weights, 128 KiB for fp8: the largest) and a last chunk whose four quarters all start their CTA segments
    off a code boundary (not fp32: its top plane of a 256 KiB chunk is too short for L = 2).  `safe` as for
    `from_planes`."""
    G = ES[dtype]
    chunk = 131072 * G
    out = []
    for fam, L in (("eq4", 2), ("eq16", 4), ("eq64", 6)):
        s = misaligned_quarter(L, 12000, chunk // G // 4, 128 // G)
        out.append(from_planes(f"fixed{L}_{tag(dtype, bits)}", dtype, bits, chunk, [fam, fam], seed=60 + L, shape_in=64,
                               last=4 * s * G, safe=safe))
    return out


def ring_case(dtype: str, bits: int) -> Case:
    """Whole chunks whose top plane is 128 KiB, with quarter bitstreams of 28672 bytes (eq128) and about 30.8 KiB
    (heavy256): the second take the ring fallback of the sync decoder, whose rings alias the buffer the matmul adds up
    in.  (256 KiB chunks for 16-bit weights, 512 KiB for fp32.)"""
    G = ES[dtype]
    return from_planes(f"ring_{dtype}b{bits}", dtype, bits, 131072 * G, ["heavy256", "eq128", "heavy256"], seed=50 + bits,
                       shape_in=2048 // (G // 2))


def rle_case(dtype: str, bits: int) -> Case:
    """Low planes constant (RLE) in every third chunk and raw in the others; fp32: one low plane per chunk in turn.  The
    constant bytes are not zero and differ by chunk, so a fill of zeros or of another chunk's byte gives other weights."""
    G = ES[dtype]
    rle = lambda c: P.constant(0x5A + 3 * c)   # noqa: E731
    side = (lambda c, g: rle(c) if c % 3 == 0 else "raw") if G == 2 else (lambda c, g: rle(c) if g == c % 3 else "raw")
    return from_planes(f"rle_{dtype}b{bits}", dtype, bits, 4096, ["geo3", "eq16", "fib", "zipf256"] * 3, seed=70 + bits,
                       shape_in=512 // G, side=side)


def stream_cases(dtypes=("bf16", "fp16", "fp32")) -> list:
    """Every non-shape case, in every layout of the given dtypes."""
    out = []
    for dt, bits in LAYOUTS:
        if dt not in dtypes:
            continue
        out += [family_case(dt, bits), crafted_case(dt, bits), rle_case(dt, bits), ring_case(dt, bits)]
        if ES[dt] == 2:
            out += fixed_length_cases(dt, bits) + [warp_mix_case(dt, bits)]
    return out


# ---------------------------------------------------------------- special values
def special_case(dtype: str, bits: int) -> tuple:
    """Gaussian weights (std 0.02) with, at known positions: inf and NaN in rows 3, 10 and 11; -0; exponent-0 weights
    (bf16 / fp32 subnormals); fp16 subnormals; and for fp16 a few rows of weights near 2^14, which with x near 8 make
    sums past 65504.  -> (case, {what: [(row, column)]})."""
    out, inn = 64, 512
    g = torch.Generator().manual_seed(80 + 2 * CODE[dtype] + bits)
    w = (torch.randn(out, inn, generator=g) * 0.02).to(TORCH[dtype])
    at = {"inf": [(3, 7), (10, 100)], "-inf": [(10, 300), (11, 5)], "nan": [(11, 200)], "-0": [(0, 1), (5, 9), (20, 511)]}
    w[3, 7] = w[10, 100] = float("inf")
    w[10, 300] = w[11, 5] = float("-inf")
    w[11, 200] = float("nan")
    for r, c in at["-0"]:
        w[r, c] = -0.0
    bits16 = w.view(torch.int16) if ES[dtype] == 2 else w.view(torch.int32)
    rows = range(30, 40)
    sub = [(r, c) for r in rows for c in range(0, inn, 3)]
    at["subnormal"] = sub
    rng = np.random.default_rng(5)
    mant = torch.from_numpy(rng.integers(1, 1 << (7 if dtype == "bf16" else 10 if dtype == "fp16" else 23), len(sub)))
    sign = torch.from_numpy(rng.integers(0, 2, len(sub)))
    hi = {"bf16": 15, "fp16": 15, "fp32": 31}[dtype]
    for (r, c), m, s in zip(sub, mant.tolist(), sign.tolist()):
        bits16[r, c] = int((s << hi) | m) - (1 << (hi + 1) if s else 0)
    if dtype == "fp16":
        at["big"] = [(r, c) for r in (50, 51) for c in range(inn)]
        w[50] = torch.from_numpy(rng.uniform(2.0 ** 13, 2.0 ** 14, inn)).to(torch.float16)
        w[51] = -w[50]
    case = Case(f"special_{dtype}b{bits}", dtype, bits, 4096, (out, inn), w.contiguous().view(torch.uint8).numpy(), special=True)
    return case, at


# ---------------------------------------------------------------- the one-hot sweep
def sweep(inn: int, nt: int) -> list:
    """Calls of a one-hot sweep: (i0, rows).  Row t of call (i0, rows) is 2^k e_{i0 + t}."""
    return [(i0, min(nt, inn - i0)) for i0 in range(0, inn, nt)]


def edge_blocks(inn: int) -> list:
    """nt in {1, 16, 17, 33} on the first and the last columns (each MT of the matmul and masked token tiles); rows past
    the last column are zero."""
    return [(i0, nt) for nt in (1, 16, 17, 33) for i0 in sorted({0, max(0, inn - nt)})]


MAX_OUT = {"bf16": float(torch.finfo(torch.bfloat16).max), "fp16": 65504.0, "fp32": float(torch.finfo(torch.float32).max)}


def scales(dtype: str, w: torch.Tensor) -> list:
    """Exponents k of the x = 2^k sweeps: 0, and for bf16 / fp32 weights with exponent-0 values also 64, so that every
    weight meets a sweep in which w * 2^k is a normal fp32 and finite in the output type."""
    ks = [0]
    if dtype != "fp16" and not bool(valid(w, 0, dtype).all()):
        ks.append(64)
    return ks


def valid(w: torch.Tensor, k: int, dtype: str) -> torch.Tensor:
    """Where w * 2^k is zero, or a normal fp32 that the output type holds exactly and finitely."""
    v = w.double() * 2.0 ** k
    a = v.abs()
    ok = (a == 0) | ((a >= 2.0 ** -126) & (a <= MAX_OUT[dtype]))
    if dtype == "bf16":   # (a bf16 weight times a power of two keeps its 8 significant bits)
        return ok
    return ok & (v.to(TORCH[dtype]).double() == v)
