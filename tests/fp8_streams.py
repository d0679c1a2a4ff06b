"""fp8 weights for the fp8 matvec tests (test_matvec_fp8_host.py, _gpu.py), and a numpy model of its numerics.

A case is a product_streams.Case of an fp8 tensor [out, in] (float8_e4m3fn or float8_e5m2): its bytes and an
oracle-made stream body at num_buf 1 (one byte plane per element, the plane is the bytes), built by product_streams'
builders.  Every case is fused in every chunk (asserted from the stream with `plane_inputs.predict`).  The inventory:

  shapes      every fused chunk size from 512 B to 128 KiB (the largest fp8 chunk) on rows shorter than a quarter,
              rows spanning chunks, in = 16, 48, 144 and 528, out = 1, a one-chunk tensor and a short last chunk;
              the formats take turns over the shapes
  crafted     code tables of logs 1 to 11 that the reference encoder never writes, and a hot 11-bit symbol
  ring        bitstreams longer than the 28 KiB the sync decoder keeps in shared memory
  fixed       fixed-length codes (L = 2, 4, 6) whose CTA segment guesses are misaligned
  special     NaN, infinities, -0 and subnormal fp8 values at known positions

Outside `special` no weight is NaN or infinite: one would turn its whole product row into NaN or an infinity.
"""
from __future__ import annotations

import functools

import numpy as np
import torch

import product_streams as S

FORMATS = ("e4m3", "e5m2")
TORCH = {f: S.TORCH[f] for f in FORMATS}
CODE = {f: S.CODE[f] for f in FORMATS}        # ZIPNN_B200_FP8_E4M3 / _E5M2
XDTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
XCODE = {"bf16": 0, "fp16": 1}                # ZIPNN_B200_MATVEC_BF16 / _FP16
BITS = 1                                      # what ZipNN writes for fp8 (the bit order is ignored at num_buf 1)
CHUNKS = tuple(512 << i for i in range(9))    # every fused fp8 chunk size: 512 B .. 128 KiB


def not_finite(fmt: str, b) -> np.ndarray:
    """Which bytes are NaN or infinite in this format."""
    b = np.asarray(b, dtype=np.uint8)
    return (b & 0x7F) == 0x7F if fmt == "e4m3" else (b & 0x7C) == 0x7C


def safe(fmt: str, plane: np.ndarray) -> np.ndarray:
    """The plane with every NaN / infinity byte v replaced by v ^ 0x40 (bit 6 is an exponent bit in both formats)."""
    out = np.asarray(plane, dtype=np.uint8).copy()
    bad = not_finite(fmt, out)
    out[bad] ^= 0x40
    return out


# ---------------------------------------------------------------- shapes
def gauss_bytes(fmt: str, n: int, seed: int, std: float = 8.0) -> np.ndarray:
    """Gaussian weights in fp8 (std 8: normal and subnormal values of both formats, far from their largest)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, generator=g) * std).to(TORCH[fmt])
    return safe(fmt, w.view(torch.uint8).numpy())


def laplace_bytes(fmt: str, n: int, seed: int) -> np.ndarray:
    """Random signs and magnitude codes spread around 1.0 (Laplace, 4 codes): about 5 bits a byte, so every chunk
    codes (fused) even at 512 bytes, where Gaussian bytes sometimes stay raw."""
    rng = np.random.default_rng(seed)
    one, top = (0x38, 0x7E) if fmt == "e4m3" else (0x3C, 0x7B)
    mag = np.clip(np.round(one + rng.laplace(0, 4, n)), 0, top).astype(np.uint8)
    return mag | (rng.integers(0, 2, n, dtype=np.uint8) << 7)


def shapes(chunk: int) -> list:
    """(name, out, in) at one chunk size; every tensor is a multiple of 512 bytes, so a short last chunk stays fused."""
    short = 1536 if chunk > 1536 else 512
    return [("in16", 3072, 16), ("in48", 1024, 48), ("in144", 384, 144), ("in528", 128, 528), ("long_row", 4, 32768),
            ("out1", 1, 16384), ("one_chunk", max(1, chunk // 128), 128), ("short_last", (3 * chunk + short) // 512, 512)]


def shape_cases(chunk: int) -> list:
    k0 = CHUNKS.index(chunk)
    out = []
    for k, (name, o, i) in enumerate(shapes(chunk)):
        fmt = FORMATS[(k + k0) % 2]
        out.append(S.Case(f"{name}_{fmt}_c{chunk}", fmt, BITS, chunk, (o, i), laplace_bytes(fmt, o * i, 1000 * k0 + k)))
    return out


# ---------------------------------------------------------------- crafted tables, rings, fixed-length codes
def crafted_case(fmt: str) -> S.Case:
    """product_streams.kraft_blocks: one 4 KiB chunk per table, rows of 128."""
    rng = np.random.default_rng(20 + CODE[fmt])
    return S.crafted(f"crafted_{fmt}", fmt, BITS, 4096, S.kraft_blocks(rng), rng, 128, bad=functools.partial(not_finite, fmt))


def ring_case(fmt: str) -> S.Case:
    """128 KiB chunks whose quarter bitstreams are 28672 bytes (eq128) and about 30.8 KiB (heavy256): the second take
    the ring fallback of the sync decoder."""
    return S.from_planes(f"ring_{fmt}", fmt, BITS, 131072, ["heavy256", "eq128", "heavy256"], 50 + CODE[fmt], 2048,
                         safe=functools.partial(safe, fmt))


def stream_cases() -> list:
    out = []
    for fmt in FORMATS:
        out += [crafted_case(fmt), ring_case(fmt)] + S.fixed_length_cases(fmt, BITS, safe=functools.partial(safe, fmt))
    return out


# ---------------------------------------------------------------- special values
def special_case(fmt: str) -> tuple:
    """Gaussian weights with, at known positions, NaN (e4m3fn: 0x7F / 0xFF; e5m2: 0x7F), e5m2 infinities, -0 and
    subnormals.  -> (case, {what: [(row, column)]})."""
    out, inn = 64, 512
    w = gauss_bytes(fmt, out * inn, 80 + CODE[fmt], std=1.0).reshape(out, inn)
    at = {"nan": [(11, 200), (12, 3)], "-0": [(0, 1), (5, 9), (20, 511)]}
    w[11, 200], w[12, 3] = 0x7F, 0xFF
    if fmt == "e5m2":
        at["inf"], at["-inf"] = [(3, 7), (10, 100)], [(10, 300), (13, 5)]
        w[3, 7] = w[10, 100] = 0x7C
        w[10, 300] = w[13, 5] = 0xFC
    for r, c in at["-0"]:
        w[r, c] = 0x80
    rng = np.random.default_rng(5)
    at["subnormal"] = [(r, c) for r in range(30, 40) for c in range(0, inn, 3)]
    mant = 8 if fmt == "e4m3" else 4   # exponent field 0, mantissa not 0
    for r, c in at["subnormal"]:
        w[r, c] = int(rng.integers(1, mant)) | (0x80 if rng.integers(0, 2) else 0)
    return S.Case(f"special_{fmt}", fmt, BITS, 4096, (out, inn), w, special=True), at


# ---------------------------------------------------------------- integer weights for exact sums
def integer_case(fmt: str, chunk: int, shape, seed: int) -> S.Case:
    """Integer weights that both formats hold exactly: e4m3fn -16..16, e5m2 -7..7."""
    top = 16 if fmt == "e4m3" else 7
    rng = np.random.default_rng(seed)
    v = np.clip(np.round(rng.normal(0, top / 3, shape)), -top, top)
    w = torch.from_numpy(v).to(TORCH[fmt])
    assert torch.equal(w.double(), torch.from_numpy(v))
    return S.Case(f"int_{fmt}_{shape[0]}x{shape[1]}_c{chunk}", fmt, BITS, chunk, shape, w.view(torch.uint8).numpy())


# ---------------------------------------------------------------- scale grids
def layouts(out: int, inn: int) -> dict:
    """The scale layouts: name -> (bn, bk)."""
    return {"tensor": (out, inn), "row": (1, inn), "block128": (128, 128), "bk16": (3, 16)}


def grid_shape(out: int, inn: int, bn: int, bk: int) -> tuple:
    return (-(-out // bn), -(-inn // bk))


def random_scales(out: int, inn: int, bn: int, bk: int, seed: int) -> np.ndarray:
    """Positive fp32 scales of the size checkpoints have (around amax / 448 of 0.02-std weights), full significands."""
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.5, 2.0, grid_shape(out, inn, bn, bk)) * 2.0 ** -14).astype(np.float32)


def dequantized(w: np.ndarray, scale: np.ndarray, bn: int, bk: int) -> np.ndarray:
    """float(W) * S as fp64 [out, in]."""
    out, inn = w.shape
    s = np.repeat(np.repeat(scale.astype(np.float64), bn, 0)[:out], bk, 1)[:, :inn]
    return w.astype(np.float64) * s


# ---------------------------------------------------------------- the numerics, modelled
def _round_to(v: np.ndarray, xdt: str) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(XDTYPES[xdt]).float().numpy()


def model(w: np.ndarray, scale: np.ndarray, bn: int, bk: int, x: np.ndarray, chunk: int, xdt: str, bias=None) -> np.ndarray:
    """y [nt, out] as the kernels compute it, every fp32 operation in its order: per 16-weight vector an FMA chain in
    ascending columns and one multiply by the block's scale; per (block of a quarter plane, row, lane) the vectors'
    products added in step order from +0; the butterfly over the 32 lanes; per row the blocks' sums added in
    ascending element order from +0; the bias; one rounding to x's dtype.  w: float32 [out, in] (the fp8 values),
    scale: fp32 grid, x: float32 [nt, in] (values of xdt).  Products of an fp8 and a bf16 / fp16 value are exact in
    fp32 (at most 15 significant bits) unless they underflow, which the callers' x avoids."""
    out, inn = w.shape
    nt = x.shape[0]
    total = out * inn
    f32 = np.float32
    V = total // 16
    e = np.arange(V, dtype=np.int64) * 16
    rows, cols = e // inn, e % inn
    wv = w.reshape(V, 16)
    xv = x[:, cols[:, None] + np.arange(16)]                       # [nt, V, 16]
    s = np.zeros((nt, V), dtype=f32)
    for i in range(16):
        s = (s + (wv[None, :, i].astype(np.float64) * xv[:, :, i]).astype(f32)).astype(f32)
    sc = scale.reshape(-1)[(rows // bn) * scale.shape[1] + cols // bk].astype(f32)
    p = (s * sc[None, :]).astype(f32)
    # the block, lane and step of every vector
    c = e // chunk
    n = np.where(c == (total - 1) // chunk, total - c * chunk, chunk)
    q = n // 4
    r = e - c * chunk
    quarter = r // q
    u = (r - quarter * q) // 16
    vpw = ((q // 16 + 255) // 256) * 32
    warp = u // vpw
    j = u - warp * vpw
    lane, step = j % 32, j // 32
    block = (c * 4 + quarter) * 8 + warp
    # per (block, row, lane): the vectors' products in step order
    key = block * (out + 1) + rows                                  # (block, row) pairs in ascending element order
    uk, grp = np.unique(key, return_inverse=True)
    acc = np.zeros((nt, uk.size, 32), dtype=f32)
    for k in range(int(step.max()) + 1):
        at = step == k
        acc[:, grp[at], lane[at]] = (acc[:, grp[at], lane[at]] + p[:, at]).astype(f32)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, :, np.arange(32) ^ o]).astype(f32)
    slot = acc[:, :, 0]                                             # [nt, pairs]
    srow = uk % (out + 1)
    y = np.zeros((nt, out), dtype=f32)
    first = np.searchsorted(srow, np.arange(out), side="left") if np.all(np.diff(srow) >= 0) else None
    if first is not None:   # (rows ascend with the pairs: add each row's slots in order, position by position)
        count = np.bincount(srow, minlength=out)
        for k in range(int(count.max())):
            has = count > k
            y[:, has] = (y[:, has] + slot[:, first[has] + k]).astype(f32)
    else:   # pragma: no cover  (pairs always ascend by row: blocks cover ascending element ranges)
        raise AssertionError("pairs out of order")
    if bias is not None:
        y = (y + np.asarray(bias, dtype=f32)[None, :]).astype(f32)
    return _round_to(y, xdt)


def one_hot_model(w: np.ndarray, scale: np.ndarray, bn: int, bk: int, cols, k: int, xdt: str) -> np.ndarray:
    """y [len(cols), out] for x rows 2^k e_col: round(fl32(fl32(W[o][col] 2^k) * S[o / bn][col / bk]))."""
    out = w.shape[0]
    cols = np.asarray(cols)
    wc = (w[:, cols].T.astype(np.float64) * 2.0 ** k).astype(np.float32)
    sc = scale[(np.arange(out) // bn)[None, :], (cols // bk)[:, None]].astype(np.float32)
    return _round_to((wc * sc).astype(np.float32), xdt)
