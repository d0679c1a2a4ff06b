"""The fp8 matmul's fragments, element walk and partial-sum layout (MatmulEp with FMT >= 0, csrc/matmul.cuh), restated
in Python and checked against the PTX ISA's mma.m16n8k16 tables and brute force, and the four-way forward dispatch of
resident fp8 modules with fp8_matmul=N on a fake plan.  No GPU.

Layout (fp8 weights, one byte per element): a chunk of n elements is four quarters of n / 4 elements.  A quarter is
cut into tiles of 8 W rows from its first row, a tile into groups of 256 columns, 4 steps of 64.  In load i of a group,
lane (g, j) forms the 16-byte vector of row g, step (i + g) & 3, columns 16j .. 16j + 15, and after the rotation
dequantizes it to 8 registers of bf16 / fp16 pairs: registers 2s and 2s + 1 are the B fragments of k step s = 0 .. 3.
Slots and the reduce are the 16-bit matmul's, in elements.
"""
import numpy as np
import pytest
import torch

import test_matmul_host as MMH
import test_matvec_host as MVH
from zipnn_b200 import resident as R
from zipnn_b200.resident import _Entry, _options, _Resident, _with_prefetch

CHUNK = 128 * 1024   # fp8 chunks are at most 128 KiB


class Layout(MMH.Layout):
    def __init__(self, out: int, inn: int, chunk: int = CHUNK):
        self.out, self.inn = out, inn
        self.total = out * inn
        self.ce = chunk
        self.K = (self.total + self.ce - 1) // self.ce
        rows = MVH.block_rows(min(self.ce, self.total) // 4, inn, out)
        self.rt = (rows + 7) // 8
        assert inn % 16 == 0
        assert all(self.chunk_elems(c) % 512 == 0 for c in range(self.K)), "every chunk must be fused"

    def vectors(self, c: int, s: int) -> dict:
        """MatmulEp<XDT, MT, FMT>::quarter: -> {(tile, group, load i, g, j): first element} of every lane that forms one."""
        e0, e1 = self.quarter(c, s)
        inn = self.inn
        r_first = e0 // inn
        tiles = ((e1 - 1) // inn - r_first) // 8 + 1
        groups = (inn + 255) // 256
        t, grp, i, g, j = np.meshgrid(np.arange(tiles), np.arange(groups), np.arange(4), np.arange(8), np.arange(4), indexing="ij")
        col = grp * 256 + 64 * ((i + g) & 3) + 16 * j
        e = (r_first + 8 * t + g) * inn + col
        ok = (col < inn) & (e >= e0) & (e < e1)
        return {k: int(v) for k, v in zip(zip(*(a[ok].tolist() for a in (t, grp, i, g, j))), e[ok])}


SHAPES = [(64, 4096), (16, 32768), (24, 14336), (40, 11008), (20000, 32), (8, 14336), (3, 57344), (128, 1040), (992, 1040)]


# ---- fragments ------------------------------------------------------------------------------------------------------
def test_fragments_give_x_d_transposed():
    """A lane's 16 dequantized weights (8 registers, register r = weights 2r, 2r + 1) are the B fragments of four k16
    steps; its two 16-byte loads of x per token row (columns 16j .. 16j + 7, then 16j + 8 .. 16j + 15) give the A
    fragments in the same k order: step s = 2h + s' takes words 2s', 2s' + 1 of load h."""
    rng = np.random.default_rng(3)
    for _ in range(20):
        d = rng.standard_normal((8, 64))    # a tile: 8 W rows, one step of 64 columns (dequantized)
        x = rng.standard_normal((16, 64))   # one 16-token tile
        acc = np.zeros((16, 8))
        for s in range(4):
            h, sp = divmod(s, 2)
            a_regs, b_regs = [], []
            for lane in range(32):
                g, j = lane >> 2, lane & 3
                v = d[g, 16 * j: 16 * j + 16]                                     # the lane's vector: 8 registers
                xa = x[g, 16 * j + 8 * h: 16 * j + 8 * h + 8]                     # load h of token g
                xc = x[g + 8, 16 * j + 8 * h: 16 * j + 8 * h + 8]                 # ... and of token g + 8
                word = lambda r, k: list(r[2 * k: 2 * k + 2])  # noqa: E731  register k: elements 2k, 2k + 1
                b_regs.append(word(v, 2 * s) + word(v, 2 * s + 1))
                a_regs.append(word(xa, 2 * sp) + word(xc, 2 * sp) + word(xa, 2 * sp + 1) + word(xc, 2 * sp + 1))
            acc += MMH._mma(a_regs, b_regs)
        assert np.allclose(acc, x @ d.T), "D = x W^T: [token][row of the tile]"


def test_rotation_puts_steps_in_order():
    MMH.test_rotation_puts_steps_in_order()   # the same two rounds of selects, on 4-register raw vectors


@pytest.mark.parametrize("inn", (1024, 4096, 14336))
def test_half_warp_plane_loads_take_two_wavefronts(inn):
    """The 16 lanes of a half warp read 16 bytes each of the quarter plane (one byte per element), rows `inn` bytes
    apart: 256 bytes, and each 16-byte bank group of a 128-byte line is hit by exactly 2 of them, the minimum.  Without
    the rotation all 4 rows would hit the same 64 bytes."""
    for i in range(4):
        for half in range(2):
            groups, plain = {}, {}
            for lane in range(16 * half, 16 * half + 16):
                g, j = lane >> 2, lane & 3
                off = g * inn + 64 * ((i + g) & 3) + 16 * j
                groups[(off % 128) // 16] = groups.get((off % 128) // 16, 0) + 1
                un = g * inn + 64 * i + 16 * j
                plain[(un % 128) // 16] = plain.get((un % 128) // 16, 0) + 1
            assert len(groups) == 8 and max(groups.values()) == 2, (inn, i, half, groups)
            assert max(plain.values()) == 4


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
            assert np.all((es >= e0) & (es + 16 <= e1)), "a vector outside its quarter"
            assert np.all((es - e0) % 16 == 0), "a vector starts on a 16-byte boundary of the quarter plane"
            firsts.append(es)
            for (tile, grp, i, g, j), e in v.items():
                r, col = divmod(e, inn)
                assert col + 16 <= inn, "a vector never crosses a row (so it lies in one scale block: bk % 16 == 0)"
                assert r == e0 // inn + 8 * tile + g and col == grp * 256 + 64 * ((i + g) & 3) + 16 * j
    allv = np.sort(np.concatenate(firsts))
    assert np.array_equal(allv, np.arange(0, L.total, 16)), "every element in exactly one vector"


@pytest.mark.parametrize("out,inn", SHAPES)
@pytest.mark.parametrize("nt", (1, 9, 64))
def test_slots_and_reduce_order_against_brute_force(out, inn, nt):
    L = Layout(out, inn)
    written = {}
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
                        written[sl] = (r_first + 8 * tile + row, (es[0], es[-1] + 16) if es else None)
    for o in range(0, out, max(1, out // 200)):
        for t in range(0, nt, max(1, nt // 3)):
            at = o * inn
            for sl, lo, hi in L.reduce_reads(o, t, nt):
                assert lo == at and hi > lo, "partials are added in ascending element order, without gaps"
                row, rng = written[sl]
                assert row == o and rng == (lo, hi), (o, sl, rng, lo, hi)
                at = hi
            assert at == (o + 1) * inn


# ---- the forward dispatch of resident fp8 modules ----------------------------------------------------------------------
class FakePlan:
    def __init__(self, wq, out_buf):
        self.wq, self.calls, self.device = wq, [], torch.device("cpu")
        self.outputs = [wq]
        self._out = out_buf

    def _d(self, scale, dtype):
        return R.dequantize_fp8(self.wq, scale, None, dtype)

    def run(self):
        self.calls.append("run")
        return [self.wq]

    def matvec_fp8(self, k, x, scale, block, scratch=None):
        self.calls.append(("matvec_fp8", tuple(x.shape), scratch))
        return torch.nn.functional.linear(x, self._d(scale, x.dtype))

    def matmul_fp8(self, k, x, scale, block, scratch=None):
        self.calls.append(("matmul_fp8", tuple(x.shape), scratch))
        return torch.nn.functional.linear(x, self._d(scale, x.dtype))

    def dequant_fp8(self, k, in_features, scale, block, dtype, out=None):
        self.calls.append(("dequant_fp8", in_features))
        out.copy_(self._d(scale, dtype))
        return out


class FakeState:
    fp8_scratch, fp8_matmul_scratch = "mv", "mm"

    def __init__(self, matvec, fp8_matmul):
        self.matvec, self.fp8_matmul = matvec, fp8_matmul


class Fp8Lin(torch.nn.Linear):
    """The attributes `_fp8_forward` reads of an FP8Linear."""

    def __init__(self):
        super().__init__(32, 8)
        self.block_size = None
        self.weight_scale_inv = torch.nn.Parameter(torch.tensor([0.5]), requires_grad=False)


def _fp8_linear(matvec, fp8_matmul, fast=True):
    lin = Fp8Lin()
    wq = (torch.randn(8, 32) * 4).to(torch.float8_e4m3fn)
    plan = FakePlan(wq, torch.empty(2 * 8 * 32, dtype=torch.uint8))
    del lin._parameters["weight"]
    lin.__dict__["forward"] = R._fp8_forward(lin, FakeState(matvec, fp8_matmul), plan, 0, [("weight", 0)], fast)
    return lin, plan


@pytest.mark.parametrize("matvec,fp8_matmul", ((8, 64), (0, 16), (8, 0), (4, 9), (8, 8)))
def test_four_way_dispatch(matvec, fp8_matmul):
    lin, plan = _fp8_linear(matvec, fp8_matmul)
    with torch.no_grad():
        for rows in sorted({1, 4, 8, 9, 16, 17, 64, 65} | ({fp8_matmul, fp8_matmul + 1} - {0})):
            plan.calls.clear()
            x = torch.randn(rows, 32).to(torch.bfloat16)
            y = lin(x)
            d = R.dequantize_fp8(plan.wq, lin.weight_scale_inv, None, torch.bfloat16)
            assert torch.equal(y, (torch.nn.functional.linear(x, d) + lin.bias).to(torch.bfloat16))
            if rows <= matvec:
                assert plan.calls == [("matvec_fp8", (rows, 32), "mv")], (rows, plan.calls)
            elif rows <= fp8_matmul:
                assert plan.calls == [("matmul_fp8", (rows, 32), "mm")], (rows, plan.calls)
            else:
                assert plan.calls == [("dequant_fp8", 32)], (rows, plan.calls)
        # a weight the products refuse: decoded and dequantized in torch at any size
        lin2, plan2 = _fp8_linear(matvec, fp8_matmul, fast=False)
        for rows in (1, 9, 65):
            plan2.calls.clear()
            lin2(torch.randn(rows, 32).to(torch.bfloat16))
            assert plan2.calls == ["run"], rows
        # another dtype: the decode, bind, forward, unbind path (the fp8 weight meets fp32 x in the module's forward)
        plan.calls.clear()
        with pytest.raises(RuntimeError):
            lin(torch.randn(9, 32))
        assert plan.calls == ["run"]
    with pytest.raises(RuntimeError, match="no_grad"):
        lin(torch.randn(9, 32).to(torch.bfloat16))


def test_options_and_report():
    model = torch.nn.Sequential(torch.nn.Linear(8, 8))
    for bad in (-1, R.MATMUL_MAX_TOKENS + 1, 1.5, "4"):
        with pytest.raises(ValueError, match="fp8_matmul"):
            R.compress_module(model, fp8=True, fp8_matmul=bad)
        with pytest.raises(ValueError, match="fp8_matmul"):
            R.load_module(model, [], fp8=True, fp8_matmul=bad)
    with pytest.raises(ValueError, match="fp8=True"):
        R.compress_module(model, fp8_matmul=16)
    with pytest.raises(ValueError, match="fp8=True"):
        R.load_module(model, [], matvec=8, fp8_matmul=64)
    with pytest.raises(ValueError, match="prefetch"):
        R.compress_module(model, fp8=True, prefetch=True, fp8_matmul=16)
    with pytest.raises(ValueError, match="prefetch"):
        _options(prefetch=True, fp8_matmul=16)
    assert _options(fp8=True, fp8_matmul=R.MATMUL_MAX_TOKENS).fp8_matmul == R.MATMUL_MAX_TOKENS
    assert _options().fp8_matmul == 0 and _options(fp8=True).fp8_matmul == 0
    state = _Resident()
    state.entries = [_Entry(None, None, [], mode) for mode in ("fp8", "fp8", "fp8_torch", "matmul")]
    state.fp8_scratch_bytes, state.fp8_matmul_scratch_bytes = 3, 5
    got = _with_prefetch({}, state, _options(fp8=True, matvec=8, fp8_matmul=64))
    assert got == {"matvec_modules": 1, "matvec_scratch_bytes": 0, "fp8_modules": 3, "fp8_scratch_bytes": 3,
                   "fp8_matmul_modules": 2, "fp8_matmul_scratch_bytes": 5}
    assert "fp8_matmul_modules" not in _with_prefetch({}, state, _options(fp8=True, matvec=8))
