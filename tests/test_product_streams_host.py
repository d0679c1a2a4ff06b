"""The product streams of tests/product_streams.py without a GPU: the matvec and matmul layouts (test_matvec_host /
test_matmul_host) at every fused chunk size and every new shape, what the builders claim about their streams, and the
one-hot sweep plan."""
import numpy as np
import pytest
import torch

import plane_inputs as P
import product_streams as S
import test_matmul_host as MMH
import test_matvec_host as MVH


def _layout_shapes():
    out = []
    for chunk in S.CHUNKS:
        for dt in ("bf16", "fp32"):
            for name, o, i in S.shapes(dt, chunk):
                out.append((chunk, S.ES[dt], o, i))
    return out


LAYOUT_SHAPES = _layout_shapes()


@pytest.mark.parametrize("chunk,es,out,inn", LAYOUT_SHAPES)
def test_matvec_layout(chunk, es, out, inn):
    L = MVH.Layout(out, inn, es, chunk)
    written = {}
    for c in range(L.K):
        for s in range(4):
            for w in range(8):
                for slot, vecs in L.warp_walk(c, s, w):
                    assert slot not in written and 0 <= slot < L.slots()
                    written[slot] = vecs
    read = set()
    for o in range(0, out, max(1, out // 64)):
        at = o * inn
        for slot, lo, hi in L.reduce_reads(o):
            assert lo == at and hi > lo and slot in written and slot not in read
            read.add(slot)
            vecs = sorted(written[slot])
            assert vecs[0][0] == lo and vecs[-1][0] + vecs[-1][1] == hi
            assert all(a[0] + a[1] == b[0] for a, b in zip(vecs, vecs[1:]))
            at = hi
        assert at == (o + 1) * inn


@pytest.mark.parametrize("chunk,es,out,inn", [s for s in LAYOUT_SHAPES if s[1] == 2])
def test_matmul_layout(chunk, es, out, inn):
    L = MMH.Layout(out, inn, chunk)
    firsts, written = [], {}
    for nt in (1, 17, 64):
        written.clear()
        for c in range(L.K):
            for s in range(4):
                e0, e1 = L.quarter(c, s)
                r_first = e0 // inn
                tiles = ((e1 - 1) // inn - r_first) // 8 + 1
                assert tiles <= L.rt, "the scratch formula bounds the tiles of every quarter"
                v = L.vectors(c, s)
                if nt == 1:
                    es_ = np.array(sorted(v.values()), dtype=np.int64)
                    assert np.all((es_ >= e0) & (es_ + 8 <= e1))
                    firsts.append(es_)
                rows = {}
                for (tile, _, _, g, _), e in v.items():
                    rows.setdefault((tile, g), []).append(e)
                for tile in range(tiles):
                    for row in range(8):
                        for t in {0, nt - 1}:
                            sl = L.slot(c, s, tile, t, row, nt)
                            assert sl not in written and 0 <= sl < L.slots() * nt
                            e = sorted(rows.get((tile, row), []))
                            written[sl] = (r_first + 8 * tile + row, (e[0], e[-1] + 8) if e else None)
        for o in range(0, out, max(1, out // 64)):
            for t in {0, nt - 1}:
                at = o * inn
                for sl, lo, hi in L.reduce_reads(o, t, nt):
                    row, rng = written[sl]
                    assert lo == at and row == o and rng == (lo, hi), (o, sl, rng, lo, hi)
                    at = hi
                assert at == (o + 1) * inn
    allv = np.sort(np.concatenate(firsts))
    assert np.array_equal(allv, np.arange(0, L.total, 8)), "every element in exactly one vector"


# ------------------------------------------------------------------ the builders' claims
@pytest.mark.parametrize("chunk", S.CHUNKS)
def test_shape_cases(chunk):
    cases = S.shape_cases(chunk)
    assert {(c.dtype, c.bits) for c in cases} >= set(S.LAYOUTS16) or len(cases) >= 8
    for c in cases:
        assert c.pr["mode"] == ["fused"] * c.pr["K"] and c.chunk == chunk
        assert torch.isfinite(c.weights()).all()
        assert all(it.kind == "raw" for row in c.pr["items"][: c.G - 1] for it in row), "full-width significands: raw low planes"
        w = c.weights().double()
        if c.G == 2:
            x = S.exact_x(c.dtype, 8, c.inn, 1).double()
            assert float((x.abs() @ w.abs().T).max()) / S.unit(c.dtype) + S.max_units(c.dtype) < 2 ** 24, "exact partial sums"
    names = {c.name.split("_")[0] for c in cases}
    assert {"narrow24", "narrow8", "in136", "in520", "long", "out1", "one", "short"} <= names
    one = [c for c in cases if c.name.startswith("one_chunk")]
    assert all(c.pr["K"] == 1 for c in one)
    long_row = [c for c in cases if c.name.startswith("long_row")]
    assert all(c.inn * c.G >= 4 * chunk for c in long_row) or chunk > 16384, "a row spans many chunks"
    if chunk > 1024:
        short = [c for c in cases if c.name.startswith("short_last")]
        assert all(0 < c.data.size % chunk and c.data.size % 512 == 0 for c in short)


def test_layouts_in_both_byte_orders():
    seen = set()
    for chunk in S.CHUNKS:
        seen |= {(c.dtype, c.bits, chunk) for c in S.shape_cases(chunk)}
    for dt, bits in S.LAYOUTS16:
        assert sum(1 for d, b, _ in seen if (d, b) == (dt, bits)) >= 2 * len(S.CHUNKS) // 4, (dt, bits)
    assert {(d, b) for d, b, _ in seen} == set(S.LAYOUTS)


@pytest.fixture(scope="module")
def stream_cases():
    return S.stream_cases()


def test_stream_cases_are_fused_finite_and_reach_their_branches(stream_cases):
    by = {}
    for c in stream_cases:
        assert c.pr["mode"] == ["fused"] * c.pr["K"], c.name
        assert torch.isfinite(c.weights()).all(), c.name
        top = c.layout_planes()
        assert not any(S.exp_all_ones(c.dtype, c.bits, p[c.G - 1]).any() for p in top), c.name
        by.setdefault(c.name.split("_")[0], []).append(c)
    for c in by["crafted"]:
        assert {it.lg for it in c.top_items()} == set(range(1, 12)), c.name
    for c in by["ring"]:
        lens = [s for it in c.top_items() for s in it.s_len]
        assert max(lens) > P.SYNC_STREAM_CAP and c.pr["k_full"] == c.pr["K"], c.name
    for c in by["rle"]:
        kinds = {it.kind for row in c.pr["items"][: c.G - 1] for it in row}
        assert kinds == {"rle", "raw"}, c.name
        fills = [int(c.body[it.src_off]) for row in c.pr["items"][: c.G - 1] for it in row if it.kind == "rle"]
        assert 0 not in fills and len(set(fills)) > 1, "RLE bytes that no zero or shared fill could stand in for"
    for name in ("fixed2", "fixed4", "fixed6"):
        for c in by[name]:
            it = c.top_items()[-1]
            assert it.fixed_len == int(name[-1]) and P.misaligned_sync_guesses(it) == 4, c.name
    for c in by["families"]:
        assert len(S.family_names(c.dtype, c.bits)) >= 12
    assert {(c.dtype, c.bits) for c in stream_cases} == set(S.LAYOUTS)


@pytest.mark.parametrize("dtype,bits", S.LAYOUTS)
def test_safe_top_removes_every_all_ones_exponent(dtype, bits):
    """Every byte value of the top plane, with random other planes: after safe_top no element is inf or NaN, and
    before it some are (the test of the layout is not vacuous)."""
    G = S.ES[dtype]
    rng = np.random.default_rng(1)
    top = np.repeat(np.arange(256, dtype=np.uint8), 4)
    chunks = [[rng.integers(0, 256, top.size, dtype=np.uint8) for _ in range(G - 1)] + [t] for t in (top, S.safe_top(dtype, bits, top))]
    for k, planes in enumerate(chunks):
        w = torch.from_numpy(P.chunk_from_planes(planes, G, bits)).view(S.TORCH[dtype])
        assert bool(torch.isfinite(w).all()) == (k == 1), (dtype, bits, k)


@pytest.mark.parametrize("dtype,bits", S.LAYOUTS)
def test_special_case(dtype, bits):
    case, at = S.special_case(dtype, bits)
    w = case.weights()
    for r, c in at["inf"]:
        assert w[r, c] == float("inf")
    for r, c in at["-inf"]:
        assert w[r, c] == float("-inf")
    assert all(torch.isnan(w[r, c]) for r, c in at["nan"])
    assert all(w[r, c] == 0 and torch.signbit(w[r, c]) for r, c in at["-0"])
    tiny = torch.finfo(S.TORCH[dtype]).tiny
    assert all(0 < abs(float(w[r, c])) < tiny for r, c in at["subnormal"])
    assert (~torch.isfinite(w)).sum() == 5


# ------------------------------------------------------------------ the one-hot sweep plan
@pytest.mark.parametrize("inn", (8, 24, 136, 520, 16384, 32768, 64, 65))
@pytest.mark.parametrize("nt", (S.MATMUL_NT, S.MATVEC_NT))
def test_sweep_reaches_every_column_once(inn, nt):
    cols = [i0 + t for i0, n in S.sweep(inn, nt) for t in range(n)]
    assert sorted(cols) == list(range(inn)) and all(1 <= n <= nt for _, n in S.sweep(inn, nt))
    edges = S.edge_blocks(inn)
    assert {n for _, n in edges} == {1, 16, 17, 33} and all(i0 == 0 or i0 + n == inn for i0, n in edges)


@pytest.mark.parametrize("dtype,bits", S.LAYOUTS)
def test_scales_check_every_element(dtype, bits):
    """Every (row, column) is checked in some sweep: its scaled value is a normal fp32 (or zero) and finite in the
    output type, for weights with every exponent the layout can hold."""
    G = S.ES[dtype]
    rng = np.random.default_rng(2)
    top = S.safe_top(dtype, bits, np.repeat(np.arange(256, dtype=np.uint8), 8))
    planes = [rng.integers(0, 256, top.size, dtype=np.uint8) for _ in range(G - 1)] + [top]
    w = torch.from_numpy(P.chunk_from_planes(planes, G, bits)).view(S.TORCH[dtype]).reshape(-1, 8)
    seen = torch.zeros_like(w, dtype=torch.bool)
    for k in S.scales(dtype, w):
        seen |= S.valid(w, k, dtype)
    assert bool(seen.all()), (dtype, bits, w[~seen][:4])
