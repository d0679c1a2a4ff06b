"""The inventory of test_fp8_limits_gpu.py checked without a GPU (tests/fp8_limits.py): which items the host accepts,
that the exact inputs give exact sums on every shape and block, the kernels' multiply-high division against Python's
`//` at every quotient boundary an inventory index meets, the experts call's x-offset guard at its boundary, and every
GPU test's device memory against its ceiling."""
import math

import numpy as np
import pytest
import torch

import fp8_limits as L
import fp8_streams as F


def test_chunk_counts_and_which_items_are_accepted():
    assert L.chunks(L.LARGEST) == L.MAX_CHUNKS and math.prod(L.LARGEST) == L.MAX_CHUNKS * L.CHUNK == 2 ** 31 - 2 ** 17
    assert L.chunks(L.REFUSED) == L.MAX_CHUNKS + 1 and math.prod(L.REFUSED) == 2 ** 31
    assert L.accepted(L.LARGEST) and not L.accepted(L.REFUSED)
    # the largest item's expert boundaries fall inside chunks, and its last 128-row block of each expert is ragged
    so = L.LARGEST[1] * L.LARGEST[2]
    assert all((e * so) % L.CHUNK for e in range(1, L.LARGEST[0])) and L.LARGEST[1] % 128
    # its last rows reach within 2^17 of 2^31
    assert 2 ** 31 - math.prod(L.LARGEST) == 2 ** 17
    for name, fmt, shape, block in L.real_shapes():
        assert L.accepted(shape), name
    # DeepSeek-V3's expert tensors ([256, 2048, 7168] and [256, 7168, 2048]) are past the limit and refused
    for shape in ((256, 2048, 7168), (256, 7168, 2048)):
        assert L.chunks(shape) > L.MAX_CHUNKS and not L.accepted(shape)
    # at 128 KiB chunks the piece limit alone keeps an item under INT32_MAX elements; rows need a multiple of 16 bytes
    assert L.MAX_CHUNKS * L.CHUNK <= L.INT32_MAX and not L.accepted((4, 24)) and L.accepted((4, 32))
    assert [f for _, f, _, _ in L.real_shapes()] == [F.FORMATS[i % 2] for i in range(len(L.real_shapes()))]


def test_exact_sums_on_every_shape_and_block():
    views = [(L.LARGEST[1] * L.LARGEST[0], L.LARGEST[2], "e4m3")]
    views += [(math.prod(s[:-1]), s[-1], f) for _, f, s, _ in L.real_shapes()]
    views += [(L.EDGE_SHAPE[0] * L.EDGE_SHAPE[1], L.EDGE_SHAPE[2], f) for f in F.FORMATS]
    for rows, inn, fmt in views:
        assert L.exact_sums(inn, fmt), (rows, inn, fmt)
    assert not L.exact_sums(2 ** 17, "e4m3"), "the bound binds"
    # the bound, computed: the worst x against the largest weights and scales
    for rows, inn, fmt in views:
        worst = inn * L.TOP[fmt] * 1.0
        assert worst < 2 ** (24 - L.SMAX) and float(np.float32(worst)) == worst
    # the dequantized weights of every scale are exact in both 16-bit types
    w = torch.arange(-16, 17, dtype=torch.float32)
    for s in range(L.SMAX + 1):
        for dt in (torch.bfloat16, torch.float16):
            assert torch.equal((w * 2.0 ** -s).to(dt).float(), w * 2.0 ** -s)
    # every scale grid of the edges has one element per block, clamped blocks a one-element grid
    E, so, inn = L.EDGE_SHAPE
    for rows in (E * so, so):
        for bn, bk in L.edge_blocks(rows, inn):
            gr, gc = L.grid(rows, inn, bn, bk)
            assert gr == -(-rows // min(bn, rows)) and gc == -(-inn // min(bk, inn)) and bk % 16 == 0
        assert L.grid(rows, inn, 2 ** 40, 2 ** 40) == (1, 1) == L.grid(rows, inn, rows + 1, inn + 16)


def test_scales_differ_between_blocks_a_power_of_two_apart():
    """A block read from a row 2^16 or an element 2^30 away gets another scale often enough to show."""
    s = L.pow2_scales((1024, 128), 1)
    assert set(np.unique(s).tolist()) == {1.0, 0.5, 0.25, 0.125}
    assert (s[512:] != s[:512]).mean() > 0.6


def test_one_hot_torch_is_the_model():
    rng = np.random.default_rng(2)
    for fmt in F.FORMATS:
        case = F.integer_case(fmt, 4096, (256, 160), 3)
        w = case.floats()
        for bn, bk in ((128, 32), (1, 160), (7, 16)):
            s = F.random_scales(256, 160, bn, bk, 4)
            cols = rng.integers(0, 160, 12)
            for k in (0, 3):
                want = F.one_hot_model(w, s, bn, bk, cols, k, "bf16")
                got = L.one_hot_torch(torch.from_numpy(w), torch.from_numpy(s), bn, bk, torch.from_numpy(cols), k, torch.bfloat16)
                assert np.array_equal(got.float().numpy().view(np.uint32), want.view(np.uint32)), (fmt, bn, bk, k)


def _boundaries(d: int, top: int) -> np.ndarray:
    q = np.arange(1, top // d + 2, dtype=np.uint64) * np.uint64(d)
    n = np.concatenate([q - np.uint64(1), q, np.array([0, top, 2 ** 31 - 1], dtype=np.uint64)])
    return n[n <= np.uint64(2 ** 31 - 1)]


def test_multiply_high_division_at_every_quotient_boundary():
    ds = L.divisors()
    assert {16384, 128, 16, 1, 3, 127, 129, 144, 1216, 1000, 3000, 16383, 3072, 4096}.issubset(ds)
    assert ds[16384] == math.prod(L.LARGEST) - 1
    for d, top in sorted(ds.items()):
        assert d < 2 ** 31 and top < 2 ** 31, d
        n = _boundaries(d, top)
        assert np.array_equal(L.div(n, L.recip(d)), n // np.uint64(d)), d
    # the model is the kernels' formula: Python's exact integers agree with the vectorised halves
    for d in (3, 127, 16383, 53248, 2 ** 31 - 1):
        for n in (0, 1, d - 1, d, 2 ** 31 - 2, 2 ** 31 - 1):
            assert int(L.div(n, L.recip(d))) == (2 * n * L.recip(d)) >> 64 == n // d, (d, n)


def test_float_division_would_fail_where_the_inventory_divides():
    """n times the fp32 reciprocal of d, truncated (a division a kernel might be tempted to use) is wrong at some
    boundary of most inventory divisors: the exact division is needed."""
    wrong = 0
    for d, top in L.divisors().items():
        n = _boundaries(d, top)
        f = np.floor(n.astype(np.float32) * np.float32(1.0 / d)).astype(np.uint64)
        wrong += int(np.any(f != n // np.uint64(d)))
    assert wrong >= 10


def test_experts_x_offset_guard_at_its_boundary():
    inn = 16384
    for xrows in (1, 2, 3, 4, 8, 32):
        s = (L.UINT32_MAX // xrows) // 8 * 8      # the largest stride (a multiple of 16 bytes of bf16) that fits
        assert L.x_offsets_fit(xrows, s, inn) and not L.x_offsets_fit(xrows, s + 8, inn) or xrows == 1, xrows
        assert L.x_offsets_fit(xrows, 0, inn)
    assert L.x_offsets_fit(1, L.UINT32_MAX, inn) and not L.x_offsets_fit(1, L.UINT32_MAX + 1, inn)
    assert not L.x_offsets_fit(2, 2 ** 31, inn) and L.x_offsets_fit(2, 2 ** 31 - 8, inn)
    # the largest item's call with x rows 2^26 elements apart fits, and passes 2^27
    T = len(L.LARGEST_ROUTES[1])
    assert L.x_offsets_fit(T, L.BIG_X_STRIDE, L.LARGEST[2]) and (T - 1) * L.BIG_X_STRIDE > 2 ** 27
    assert (T - 1) * L.BIG_X_STRIDE > 2 ** 24, "past the 24 bits a truncated offset keeps"


@pytest.mark.parametrize("test", ("largest", "refused", "real", "edges"))
def test_device_memory_estimates_under_the_ceiling(test):
    shapes = [s for _, _, s, _ in L.real_shapes()] if test == "real" else [None]
    for shape in shapes:
        need = L.memory(test, shape)
        assert 0 < need <= L.CEILING - 2 * L.GIB, (test, shape, need / L.GIB)
