"""The fp8 products, dequantizes and expert calls at their largest item and at real checkpoint shapes: the inventory and
the input builders of test_fp8_limits_host.py and test_fp8_limits_gpu.py.  Importable without a GPU.

The fp8 kernels find a weight's scale from 32-bit element, row and column indices (matvec_fp8_div, a multiply-high exact
for n, d < 2^31), and the experts form adds 32-bit slice and x-row offsets.  The host keeps them in range by refusing an
fp8 item of more than INT32_MAX elements or of more than one piece (16383 chunks: a run of 16384 is cut in two), and an
experts call whose x row offsets pass UINT32_MAX.  At the largest fp8 chunk (128 KiB) the largest item accepted has
16383 * 131072 = 2^31 - 2^17 elements.

Exact inputs (the main oracle): integer fp8 weights (fp8_streams.integer_case's: e4m3fn -16..16, e5m2 -7..7), x in
{-1, 0, 1} and a power of two 2^-s, s in 0..3, per scale block, drawn at random (a pattern periodic in the block number
would give a block read from a row 2^16 or 2^30 away the same scale).  Every product is exact, every partial sum is a
multiple of 2^-3 below 2^21 (`exact_sums`), so each result is the fp64 product rounded once to x's dtype, whatever the
order of the sums, and a scale read from the wrong block, or a partial sum dropped or doubled, changes it.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import fp8_streams as F

CHUNK = 131072                 # the largest fp8 chunk (zipnn.HUF_MAX_BLOCK)
MAX_CHUNKS = 16383             # chunks of the longest piece
INT32_MAX = 2 ** 31 - 1
UINT32_MAX = 2 ** 32 - 1
SMAX = 3                       # scales 2^-s, s in 0..SMAX
GIB = 2 ** 30
CEILING = 16 * GIB             # peak reserved device memory of any test in test_fp8_limits_gpu.py
TOP = {"e4m3": 16, "e5m2": 7}  # the integer weights' largest magnitude

# the largest item accepted and the first one refused: experts of 16383 rows, so expert boundaries fall inside chunks
LARGEST = (8, 16383, 16384)
REFUSED = (8, 16384, 16384)
LARGEST_IDS = ((7,), (0, 7))          # dequant_fp8_select
LARGEST_ROUTES = ([[7]], [[7, 0], [0, 7], [7, 0], [0, 7]])   # experts_matvec_fp8: T = 1 and 4
BIG_X_STRIDE = 2 ** 26                # x rows 2^26 elements apart: the x row offsets pass 2^27

# real checkpoint shapes: (name, fmt, shape, block); the formats take turns
DENSE = [
    ("dsv3_kv_a_proj_with_mqa", (576, 7168), (128, 128)),
    ("dsv3_q_a_proj", (1536, 7168), (128, 128)),
    ("dsv3_q_b_proj", (24576, 1536), (128, 128)),
    ("dsv3_kv_b_proj", (32768, 512), (128, 128)),
    ("dsv3_o_proj", (7168, 16384), (128, 128)),
    ("dsv3_mlp_gate", (18432, 7168), (128, 128)),
    ("dsv3_mlp_down", (7168, 18432), (128, 128)),
    ("llama405b_kv", (1024, 16384), "row"),
    ("llama405b_gate", (53248, 16384), "row"),
    ("llama405b_down", (16384, 53248), "row"),
]
EXPERTS = [
    ("qwen3_235b_gate_up", (128, 3072, 4096), (128, 128)),
    ("qwen3_235b_down", (128, 4096, 1536), (128, 128)),
]
TOP_K = 8
DENSE_MATVEC_ROWS = (1, 3, 8)
DENSE_MATMUL_ROWS = (9, 17, 33, 64)

# scale grids at their edges, on one mid-size tensor per format: dense [3000, 1216], selected 3 experts of 1000 rows (every tensor a whole
# number of 512-byte units, so its short last chunk decodes fused)
EDGE_SHAPE = (3, 1000, 1216)


def real_shapes() -> list:
    """(name, fmt, shape, (bn, bk)) of every real shape, the formats taking turns."""
    out = []
    for i, (name, shape, block) in enumerate(DENSE + EXPERTS):
        inn = shape[-1]
        out.append((name, F.FORMATS[i % 2], shape, (1, inn) if block == "row" else block))
    return out


def edge_blocks(out: int, inn: int) -> list:
    return [(1, 16), (1, inn), (3, 48), (127, 128), (128, 128), (129, 144), (out - 1, inn - 16), (out, inn),
            (out + 1, inn + 16), (2 ** 40, 2 ** 40)]


# ---------------------------------------------------------------- what the host accepts
def chunks(shape) -> int:
    return -(-math.prod(shape) // CHUNK)


def accepted(shape) -> bool:
    """product_item's rules for an fp8 item at 128 KiB chunks: one piece (at most 16383 chunks), at most INT32_MAX
    elements, rows of a multiple of 16 bytes."""
    return chunks(shape) <= MAX_CHUNKS and math.prod(shape) <= INT32_MAX and shape[-1] % 16 == 0


def x_offsets_fit(xrows: int, x_stride: int, inn: int) -> bool:
    """The experts call's guard on its 32-bit x row offsets (E_ARG when False)."""
    return xrows * max(x_stride, inn) <= UINT32_MAX


def grid(rows: int, inn: int, bn: int, bk: int) -> tuple:
    """The scale grid of a [rows, inn] matrix, blocks larger than it clamped to it (a one-element grid)."""
    return F.grid_shape(rows, inn, min(bn, rows), min(bk, inn))


def exact_sums(inn: int, fmt: str) -> bool:
    """Every partial sum of the exact inputs is exact in fp32: sum |x| |w| S <= inn * TOP * 1, a multiple of 2^-SMAX,
    stays below 2^(24 - SMAX); each product (an integer of at most 5 bits times +-1) and each dequantized weight
    (W * 2^-s, in bf16 and fp16 normal range) is exact."""
    top = TOP[fmt]
    return inn * top < 2 ** (24 - SMAX) and top * 2.0 ** -SMAX >= 2.0 ** -14 and top <= 2 ** 8


# ---------------------------------------------------------------- the divisions the kernels make
def recip(d: int) -> int:
    """matvec_fp8_recip: ceil(2^64 / (2 d)) as the kernels compute it."""
    return (2 ** 64 - 1) // (2 * d) + 1


def div(n, r: int) -> np.ndarray:
    """matvec_fp8_div: the high 64 bits of (2 n) * r, n uint32 (vectorised in 32-bit halves)."""
    a = 2 * np.asarray(n, dtype=np.uint64)
    rh, rl = np.uint64(r >> 32), np.uint64(r & 0xFFFFFFFF)
    return (a * rh + ((a * rl) >> np.uint64(32))) >> np.uint64(32)


def divisors() -> dict:
    """divisor -> the largest index it divides in the inventory's calls: `in` (the dequantize's element index), bn (row
    in the matrix or the slice), bk (column), the rows of a slice (row of the stacked experts) and top_k (pair number)."""
    out = {}

    def add(d, n):
        out[d] = max(out.get(d, 0), n)

    views = [(math.prod(LARGEST[:2]), LARGEST[2], LARGEST[0], (128, 128))]
    views += [(math.prod(s[:-1]), s[-1], s[0] if len(s) == 3 else 1, b) for _, _, s, b in real_shapes()]
    E, so, inn = EDGE_SHAPE
    views += [(E * so, inn, E, b) for b in edge_blocks(E * so, inn)] + [(E * so, inn, E, b) for b in edge_blocks(so, inn)]
    for rows, inn, E, (bn, bk) in views:
        so = rows // E
        add(inn, rows * inn - 1)
        add(min(bn, rows), rows - 1)
        add(min(bn, so), so - 1)
        add(min(bk, inn), inn - 1)
        add(so, rows - 1)
    for k in range(1, TOP_K + 1):
        add(k, 4 * k - 1)
    return out


# ---------------------------------------------------------------- device memory
def memory(test: str, shape=None) -> int:
    """Bytes of device memory a test of test_fp8_limits_gpu.py holds at its peak (an upper estimate)."""
    if test == "largest":
        n = math.prod(LARGEST)
        # dense fp8, stream (at most the dense bytes), bf16 out of one call, a fp64 row slab and its fp32 copy, x
        return n + n + 2 * n + 3 * (8192 * LARGEST[2] * 8) + 4 * BIG_X_STRIDE * 2 + GIB
    if test == "refused":
        n = math.prod(REFUSED)
        return 3 * n + GIB   # dense, stream, the plan's output
    if test == "real":
        n = math.prod(shape)
        # dense fp8, stream, the plan's output at create, bf16 out, fp64 row slabs
        return 3 * n + 2 * n + 2 * GIB
    if test == "edges":
        return GIB
    raise KeyError(test)


# ---------------------------------------------------------------- builders
def integer_weights(fmt: str, shape, seed: int, slab: int = 1 << 27) -> torch.Tensor:
    """fp8_streams.integer_case's weights (round(N(0, TOP / 3)) clipped to +-TOP) built on the device in slabs."""
    top = TOP[fmt]
    n = math.prod(shape)
    w = torch.empty(n, dtype=F.TORCH[fmt], device="cuda")
    g = torch.Generator("cuda").manual_seed(seed)
    for i in range(0, n, slab):
        m = min(slab, n - i)
        w[i: i + m] = (torch.randn(m, generator=g, device="cuda") * (top / 3)).round_().clamp_(-top, top).to(F.TORCH[fmt])
    return w.view(shape)


def pow2_scales(shape, seed: int) -> np.ndarray:
    """A power of two 2^-s, s in 0..SMAX at random, per scale block: fp32 of `shape`."""
    rng = np.random.default_rng(seed)
    return (2.0 ** -rng.integers(0, SMAX + 1, shape)).astype(np.float32)


def signs(shape, seed: int) -> np.ndarray:
    """x in {-1, 0, 1}."""
    return np.random.default_rng(seed).integers(-1, 2, shape).astype(np.float32)


def one_hot_torch(w: torch.Tensor, scale: torch.Tensor, bn: int, bk: int, cols: torch.Tensor, k: int, dtype) -> torch.Tensor:
    """fp8_streams.one_hot_model in torch, on w's device: y [len(cols), out] = round(fl32(fl32(W[o][col] 2^k) *
    S[o / bn][col / bk]))."""
    out = w.shape[0]
    wc = (w[:, cols].T.double() * 2.0 ** k).float()
    sc = scale[(torch.arange(out, device=w.device) // bn)[None, :], (cols // bk)[:, None]].float()
    return (wc * sc).to(dtype)
