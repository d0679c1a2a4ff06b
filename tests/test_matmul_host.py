"""The tensor-core matmul's fragments, element walk and partial-sum layout (csrc/matmul.cuh), restated in Python and
checked against brute force and the mma.m16n8k16 fragment tables of the PTX ISA, and the three-way forward dispatch of
resident.py with a fake plan.  No GPU.

Layout (16-bit weights): a chunk of n elements is four quarters (one per bitstream) of n / 4 elements.  A quarter is
cut into tiles of 8 W rows from its first row, a tile into groups of 128 columns, 4 steps of 32.  In load i of a group,
lane (g, j) forms the vector of row g, step (i + g) & 3, columns 8j .. 8j + 7.  Slot of (quarter, tile, token, row):
(((chunk * 4 + bitstream) * rt + tile) * n_tokens + token) * 8 + row, rt = ceil(rows a quarter may touch / 8).
"""
import numpy as np
import pytest
import torch

import test_matvec_host as MVH
from zipnn_b200 import resident as R

CHUNK = MVH.CHUNK


class Layout:
    def __init__(self, out: int, inn: int, chunk: int = CHUNK):
        self.out, self.inn = out, inn
        self.total = out * inn
        self.ce = chunk // 2
        self.K = (self.total + self.ce - 1) // self.ce
        rows = MVH.block_rows(min(self.ce, self.total) // 4, inn, out)
        self.rt = (rows + 7) // 8
        assert inn % 8 == 0
        assert all(self.chunk_elems(c) * 2 % 512 == 0 for c in range(self.K)), "every chunk must be fused"

    def slots(self) -> int:   # floats per token: zipnn_b200_decode_plan_matmul_scratch_size / (4 * n_tokens)
        return 4 * self.K * self.rt * 8

    def chunk_elems(self, c: int) -> int:
        return self.total - c * self.ce if c == self.K - 1 else self.ce

    def quarter(self, c: int, s: int) -> tuple:
        q = self.chunk_elems(c) // 4
        e0 = c * self.ce + s * q
        return e0, e0 + q

    def vectors(self, c: int, s: int) -> dict:
        """MatmulEp::quarter: -> {(tile, group, load i, g, j): first element} of every lane that forms a vector."""
        e0, e1 = self.quarter(c, s)
        inn = self.inn
        r_first = e0 // inn
        tiles = ((e1 - 1) // inn - r_first) // 8 + 1
        groups = (inn + 127) // 128
        t, grp, i, g, j = np.meshgrid(np.arange(tiles), np.arange(groups), np.arange(4), np.arange(8), np.arange(4), indexing="ij")
        col = grp * 128 + 32 * ((i + g) & 3) + 8 * j
        e = (r_first + 8 * t + g) * inn + col
        ok = (col < inn) & (e >= e0) & (e < e1)
        return {k: int(v) for k, v in zip(zip(*(a[ok].tolist() for a in (t, grp, i, g, j))), e[ok])}

    def slot(self, c: int, s: int, tile: int, token: int, row: int, nt: int) -> int:
        return (((c * 4 + s) * self.rt + tile) * nt + token) * 8 + row

    def reduce_reads(self, o: int, t: int, nt: int) -> list:
        """k_matmul_reduce for (token t, row o): [(slot, first element, end)] in the order it adds them."""
        reads, e = [], o * self.inn
        while e < (o + 1) * self.inn:
            c = e // self.ce
            q = self.chunk_elems(c) // 4
            s = (e - c * self.ce) // q
            qs = c * self.ce + s * q
            r = o - qs // self.inn
            reads.append((self.slot(c, s, r // 8, t, r % 8, nt), e, min(qs + q, (o + 1) * self.inn)))
            e = qs + q
        return reads


SHAPES = [(o, i) for o, i, es in MVH.SHAPES if es == 2] + [(8, 14336), (3, 28672), (40, 28672)]


# ---- fragments: a lane's registers against the PTX ISA's m16n8k16 tables (row-major A, column-major B) ------------------
def _mma(a_regs, b_regs):
    """D[16][8] of one mma.m16n8k16 from per-lane registers: a_regs[lane] = 8 values a0..a7, b_regs[lane] = b0..b3."""
    A, B = np.zeros((16, 16)), np.zeros((16, 8))
    for lane in range(32):
        g, j = lane >> 2, lane & 3
        a, b = a_regs[lane], b_regs[lane]
        for h in range(2):
            A[g, 2 * j + h], A[g + 8, 2 * j + h] = a[h], a[2 + h]
            A[g, 2 * j + 8 + h], A[g + 8, 2 * j + 8 + h] = a[4 + h], a[6 + h]
            B[2 * j + h, g], B[2 * j + 8 + h, g] = b[h], b[2 + h]
    return A @ B


def test_fragments_give_x_w_transposed():
    rng = np.random.default_rng(3)
    for _ in range(20):
        w = rng.standard_normal((8, 32))    # a tile: 8 W rows, one step of 32 columns
        x = rng.standard_normal((16, 32))   # one 16-token tile
        d = np.zeros((16, 8))
        for s in range(2):
            a_regs, b_regs = [], []
            for lane in range(32):
                g, j = lane >> 2, lane & 3
                v = w[g, 8 * j: 8 * j + 8]                                   # the lane's 16-byte vector: 4 registers
                xa, xc = x[g, 8 * j: 8 * j + 8], x[g + 8, 8 * j: 8 * j + 8]  # its two 16-byte loads of x
                word = lambda r, k: list(r[2 * k: 2 * k + 2])  # noqa: E731  register k: elements 2k, 2k + 1
                b_regs.append(word(v, 2 * s) + word(v, 2 * s + 1))
                a_regs.append(word(xa, 2 * s) + word(xc, 2 * s) + word(xa, 2 * s + 1) + word(xc, 2 * s + 1))
            d += _mma(a_regs, b_regs)
        assert np.allclose(d, x @ w.T), "D = x W^T: [token][row of the tile]"


def test_rotation_puts_steps_in_order():
    for g in range(8):
        rg = g & 3
        v = [(i + g) & 3 for i in range(4)]               # load i forms step (i + g) & 3
        u = [v[(t + 3) & 3] if rg & 1 else v[t] for t in range(4)]
        w = [u[(t + 2) & 3] if rg & 2 else u[t] for t in range(4)]
        assert w == [0, 1, 2, 3], g


@pytest.mark.parametrize("inn", (4096, 14336, 1024))
def test_plane_loads_are_free_of_bank_conflicts(inn):
    """The 16 lanes of a half warp read 8 bytes each of the quarter plane (one byte per element) at 16 different
    8-byte words of one 128-byte line modulo the banks, rows `inn` bytes apart."""
    for i in range(4):
        for half in range(2):
            words = set()
            for lane in range(16 * half, 16 * half + 16):
                g, j = lane >> 2, lane & 3
                off = g * inn + 32 * ((i + g) & 3) + 8 * j
                words.add((off % 128) // 8)
            assert len(words) == 16, (inn, i, half)


# ---- walk and slots ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out,inn", SHAPES)
def test_every_element_is_taken_once(out, inn):
    L = Layout(out, inn)
    firsts = []
    for c in range(L.K):
        for s in range(4):
            e0, e1 = L.quarter(c, s)
            v = L.vectors(c, s)
            es = np.array(sorted(v.values()), dtype=np.int64)
            assert len(es) == len(set(es.tolist())), "a vector formed twice"
            assert np.all((es >= e0) & (es + 8 <= e1)), "a vector outside its quarter"
            firsts.append(es)
            for (tile, grp, i, g, j), e in v.items():
                r, col = divmod(e, inn)
                assert col + 8 <= inn, "a vector never crosses a row"
                assert r == e0 // inn + 8 * tile + g and col == grp * 128 + 32 * ((i + g) & 3) + 8 * j
    allv = np.sort(np.concatenate(firsts))
    assert np.array_equal(allv, np.arange(0, L.total, 8)), "every element in exactly one vector"


@pytest.mark.parametrize("out,inn", SHAPES)
@pytest.mark.parametrize("nt", (1, 9, 64))
def test_slots_and_reduce_order_against_brute_force(out, inn, nt):
    L = Layout(out, inn)
    written = {}   # slot -> (row o, element range of the quarter in that row), from the vectors that feed it
    for c in range(L.K):
        for s in range(4):
            e0, e1 = L.quarter(c, s)
            r_first = e0 // inn
            tiles = ((e1 - 1) // inn - r_first) // 8 + 1
            assert tiles <= L.rt, "the scratch formula bounds the tiles of every quarter"
            rows = {}
            for (tile, _, _, g, _), e in L.vectors(c, s).items():
                rows.setdefault((tile, g), []).append(e)
            for tile in range(tiles):
                for row in range(8):
                    for t in range(0, nt, max(1, nt // 3)):
                        sl = L.slot(c, s, tile, t, row, nt)
                        assert sl not in written and 0 <= sl < L.slots() * nt
                        es = sorted(rows.get((tile, row), []))
                        written[sl] = (r_first + 8 * tile + row, (es[0], es[-1] + 8) if es else None)
    for o in range(out):
        for t in range(0, nt, max(1, nt // 3)):
            at = o * inn
            for sl, lo, hi in L.reduce_reads(o, t, nt):
                assert lo == at and hi > lo, "partials are added in ascending element order, without gaps"
                row, rng = written[sl]
                assert row == o and rng == (lo, hi), (o, sl, rng, lo, hi)
                at = hi
            assert at == (o + 1) * inn


# ---- the forward dispatch of resident.py ---------------------------------------------------------------------------
class FakePlan(MVH.FakePlan):
    def matmul(self, k, x, bias=None, scratch=None):
        self.calls.append(("matmul", k, tuple(x.shape), bias is not None, scratch))
        return torch.nn.functional.linear(x, self.weight, bias)


class FakeState:
    matvec_scratch, matmul_scratch = "mv", "mm"

    def __init__(self, matvec):
        self.matvec = matvec


def _linear(matvec, matmul, device=torch.device("cpu")):
    lin = torch.nn.Linear(16, 8)
    plan = FakePlan(lin.weight.detach().clone())
    del lin._parameters["weight"]
    lin.__dict__["forward"] = R._matvec_forward(lin, FakeState(matvec), plan, 0, [("weight", 0)], torch.float32, device, matmul)
    return lin, plan


@pytest.mark.parametrize("matvec,matmul", ((8, 16), (0, 16), (8, 0), (4, 64)))
def test_three_way_dispatch(matvec, matmul):
    lin, plan = _linear(matvec, matmul)
    with torch.no_grad():
        for rows in sorted({1, 8, 9, matmul, matmul + 1, 65} - {0}):
            plan.calls.clear()
            x = torch.randn(rows, 16)
            assert torch.equal(lin(x), torch.nn.functional.linear(x, plan.weight, lin.bias))
            if rows <= matvec:
                assert plan.calls == [("matvec", 0, (rows, 16), True, "mv")], (rows, plan.calls)
            elif rows <= matmul:
                assert plan.calls == [("matmul", 0, (rows, 16), True, "mm")], (rows, plan.calls)
            else:
                assert plan.calls == ["run"], (rows, plan.calls)
            assert "weight" not in lin.__dict__
        if matmul > 2:
            plan.calls.clear()
            lin(torch.randn(3, 1, 16))   # rows are the product of the leading dims
            assert plan.calls[0][0] == ("matvec" if 3 <= matvec else "matmul")
        # another dtype, an autocast region: the decode path whatever the size
        plan.calls.clear()
        with pytest.raises(RuntimeError):
            lin(torch.randn(9, 16).double())
        assert plan.calls == ["run"]
        plan.calls.clear()
        with torch.autocast("cpu", dtype=torch.bfloat16):
            lin(torch.randn(9, 16))
        assert plan.calls == ["run"]
    with pytest.raises(RuntimeError, match="no_grad"):
        lin(torch.randn(9, 16))


def test_another_device_decodes():
    lin, plan = _linear(8, 64, device=torch.device("cuda", 0))
    with torch.no_grad():
        for rows in (1, 9, 64):
            plan.calls.clear()
            lin(torch.randn(rows, 16))
            assert plan.calls == ["run"], rows


def test_prefetch_and_bad_counts_are_refused():
    model = torch.nn.Sequential(torch.nn.Linear(8, 8))
    with pytest.raises(ValueError, match="matmul and prefetch"):
        R.compress_module(model, prefetch=True, matmul=16)
    with pytest.raises(ValueError, match="matmul and prefetch"):
        R.load_module(model, [], prefetch=True, matmul=64)
    for bad in (-1, R.MATMUL_MAX_TOKENS + 1, 1.5, "4"):
        with pytest.raises(ValueError, match="matmul"):
            R.compress_module(model, matmul=bad)
    assert R._options(prefetch=True, matmul=0).matmul == 0
    assert R._options(matmul=R.MATMUL_MAX_TOKENS).matmul == R.MATMUL_MAX_TOKENS
