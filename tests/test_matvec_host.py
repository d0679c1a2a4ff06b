"""The matvec's element walk and partial-sum layout (csrc/matvec.cuh), restated in Python and checked against brute
force, and the forward dispatch of resident.py with a fake plan.  No GPU.

Layout: a chunk of n elements is four quarters (one per bitstream) of n / 4 elements; a quarter's 16-byte vectors are
split over the 8 warps of its CTA in blocks of whole 32-vector steps.  Block (chunk, bitstream, warp) owns
rs = min(out, (block elements + in - 2) / in + 1) rows of slots, n_tokens floats each, from its first row on.
"""
import pytest
import torch

from zipnn_b200 import resident as R

CHUNK = 256 * 1024   # bytes (the codec's default)


def block_elems(n: int, esize: int) -> int:
    epv = 16 // esize
    nv = (n // 4) // epv
    return (nv + 255) // 256 * 32 * epv


def block_rows(be: int, inn: int, out: int) -> int:
    return min(out, (be + inn - 2) // inn + 1)


class Layout:
    def __init__(self, out: int, inn: int, esize: int, chunk: int = CHUNK):
        self.out, self.inn, self.esize = out, inn, esize
        self.total = out * inn
        self.ce = chunk // esize
        self.K = (self.total + self.ce - 1) // self.ce
        self.rs = block_rows(block_elems(min(self.ce, self.total), esize), inn, out)
        assert (inn * esize) % 16 == 0
        assert all(self.chunk_elems(c) * esize % 512 == 0 for c in range(self.K)), "every chunk must be fused"

    def slots(self) -> int:   # floats per token: zipnn_b200_decode_plan_matvec_scratch_size / (4 * n_tokens)
        return 32 * self.K * self.rs

    def chunk_elems(self, c: int) -> int:
        return self.total - c * self.ce if c == self.K - 1 else self.ce

    def block_of(self, e: int) -> tuple:
        """matvec_block_of: -> (id, start, end)."""
        c = e // self.ce
        n = self.chunk_elems(c)
        q, be = n // 4, block_elems(n, self.esize)
        r = e - c * self.ce
        s = r // q
        w = (r - s * q) // be
        start = c * self.ce + s * q + w * be
        return (c * 4 + s) * 8 + w, start, min(start + be, c * self.ce + (s + 1) * q)

    def warp_walk(self, c: int, s: int, w: int) -> list:
        """MatvecEp::quarter for one warp: -> [(slot, [(first element, elements) per vector added])] per flush."""
        epv = 16 // self.esize
        inn = self.inn
        count = self.chunk_elems(c) // 4
        nv = count // epv
        vpw = ((nv + 255) >> 8) << 5
        v0, v1 = w * vpw, min(nv, w * vpw + vpw)
        if v0 >= v1:
            return []
        e0 = c * self.ce + s * count + v0 * epv
        row0, col0 = divmod(e0, inn)
        base, first = ((c * 4 + s) * 8 + w) * self.rs, row0
        step_rows, step_cols = divmod(32 * epv, inn)
        flushes, acc, cur = [], [], row0
        for v in range(v0, v1, 32):
            nvalid = min(32, v1 - v)
            last = row0
            straddles = col0 + 32 * epv > inn
            if straddles:
                last += (col0 + nvalid * epv - 1) // inn
            lanes = []
            for lane in range(nvalid):
                lrow, lcol = row0, col0 + lane * epv
                if straddles:
                    q = lcol // inn
                    lrow, lcol = lrow + q, lcol - q * inn
                assert lcol + epv <= inn, "a vector never crosses a row"
                lanes.append((lrow, lrow * inn + lcol))
                assert lrow * inn + lcol == e0 + (v - v0 + lane) * epv
            for rr in range(row0, last + 1):
                if rr != cur:
                    flushes.append((base + cur - first, acc))
                    cur, acc = rr, []
                acc += [(e, epv) for lrow, e in lanes if lrow == rr]
            row0, col0 = row0 + step_rows, col0 + step_cols
            if col0 >= inn:
                row0, col0 = row0 + 1, col0 - inn
        flushes.append((base + cur - first, acc))
        return flushes

    def reduce_reads(self, o: int) -> list:
        """k_matvec_reduce for row o: the slots it adds, in order, with the element range each must hold."""
        reads, e = [], o * self.inn
        while e < (o + 1) * self.inn:
            bid, start, end = self.block_of(e)
            reads.append((bid * self.rs + o - start // self.inn, e, min(end, (o + 1) * self.inn)))
            e = end
        return reads


SHAPES = [
    (64, 4096, 2), (16, 32768, 2),            # rows divide a quarter plane, or are one
    (24, 14336, 2), (40, 11008, 2), (20000, 24, 2), (2048, 24, 4),   # rows straddle blocks and quarters
    (6, 49152, 2), (3, 49152, 4),             # a row spans several quarters
    (100, 4096, 2), (23, 11008, 4),           # a short last chunk
    (1, 16384, 2), (512, 8, 2), (4096, 8, 2), (1, 512, 4),   # one row; the narrowest rows
]


@pytest.mark.parametrize("out,inn,esize", SHAPES)
def test_walk_and_slots_against_brute_force(out, inn, esize):
    L = Layout(out, inn, esize)
    written = {}   # slot -> element ranges
    for c in range(L.K):
        for s in range(4):
            for w in range(8):
                for slot, vecs in L.warp_walk(c, s, w):
                    assert slot not in written, f"slot {slot} written twice"
                    assert 0 <= slot < L.slots()
                    assert vecs, "a flush with nothing in it"
                    written[slot] = vecs
    covered = 0
    read = set()
    for o in range(out):
        at = o * inn
        for slot, lo, hi in L.reduce_reads(o):
            assert lo == at and hi > lo, "partials are added in ascending element order, without gaps"
            assert slot in written and slot not in read, f"row {o} reads slot {slot}"
            read.add(slot)
            vecs = sorted(written[slot])
            assert vecs[0][0] == lo and vecs[-1][0] + vecs[-1][1] == hi
            assert all(a[0] + a[1] == b[0] for a, b in zip(vecs, vecs[1:])), "disjoint ranges whose union is the piece"
            covered += hi - lo
            at = hi
        assert at == (o + 1) * inn
    assert covered == L.total and read == set(written), "every written slot is read exactly once"


def test_block_of_matches_the_walk():
    L = Layout(100, 4096, 2)   # a short last chunk
    for c in range(L.K):
        for s in range(4):
            for w in range(8):
                fl = L.warp_walk(c, s, w)
                if fl:
                    first = min(v[0] for _, vecs in fl for v in vecs)
                    last = max(v[0] + v[1] for _, vecs in fl for v in vecs)
                    assert L.block_of(first) == ((c * 4 + s) * 8 + w, first, last) == L.block_of(last - 1)


# ---- the forward dispatch of resident.py ---------------------------------------------------------------------------
class FakePlan:
    def __init__(self, weight):
        self.weight, self.calls = weight, []

    def run(self):
        self.calls.append("run")
        return [self.weight]

    def matvec(self, k, x, bias=None, scratch=None):
        self.calls.append(("matvec", k, tuple(x.shape), bias is not None, scratch))
        return torch.nn.functional.linear(x, self.weight, bias)


class FakeState:
    matvec, matvec_scratch = 4, "scratch"


def _linear(bias=True):
    lin = torch.nn.Linear(16, 8, bias=bias)
    plan = FakePlan(lin.weight.detach().clone())
    want = lambda x: torch.nn.functional.linear(x, plan.weight, lin.bias)  # noqa: E731
    del lin._parameters["weight"]
    lin.__dict__["forward"] = R._matvec_forward(lin, FakeState(), plan, 0, [("weight", 0)], torch.float32, torch.device("cpu"))
    return lin, plan, want


@pytest.mark.parametrize("bias", (True, False))
def test_forward_dispatch(bias):
    lin, plan, want = _linear(bias)
    with torch.no_grad():
        for shape, small in (((16,), True), ((1, 16), True), ((4, 16), True), ((2, 2, 16), True), ((5, 16), False), ((3, 2, 16), False),
                             ((0, 16), True)):
            plan.calls.clear()
            x = torch.randn(shape)
            y = lin(x)
            assert torch.equal(y, want(x))
            if small:
                assert plan.calls == [("matvec", 0, shape, bias, "scratch")], (shape, plan.calls)
            else:
                assert plan.calls == ["run"], (shape, plan.calls)
            assert "weight" not in lin.__dict__, "the decoded weight stays bound after the forward"
        # another dtype than the weight's, or an autocast region: whatever F.linear does with it, through the decode path
        plan.calls.clear()
        with torch.autocast("cpu", dtype=torch.bfloat16):
            y = lin(torch.randn(2, 16))
        assert plan.calls == ["run"] and y.dtype == torch.bfloat16 and "weight" not in lin.__dict__
        plan.calls.clear()
        with pytest.raises(RuntimeError):
            lin(torch.randn(2, 16).double())
        assert plan.calls == ["run"] and "weight" not in lin.__dict__
    with pytest.raises(RuntimeError, match="no_grad"):
        lin(torch.randn(1, 16))
    with pytest.raises(RuntimeError, match="no_grad"):
        lin(torch.randn(9, 16))


def test_matvecs_and_dense_biases():
    class Mine(torch.nn.Linear):
        def forward(self, x):
            return super().forward(x) * 2

    a, b, c = torch.nn.Linear(8, 8), Mine(8, 8), torch.nn.Embedding(4, 8)
    assert R.matvecs(a) and not R.matvecs(b) and not R.matvecs(c)
    model = torch.nn.Sequential(a, b)
    _, groups = R.select(model)
    assert len(groups) == 4 and R.dense_biases(groups, 0) is groups
    kept = R.dense_biases(groups, 4)
    assert [id(p) for p, _ in kept] == [id(a.weight), id(b.weight), id(b.bias)]


def test_prefetch_and_bad_counts_are_refused():
    model = torch.nn.Sequential(torch.nn.Linear(8, 8))
    with pytest.raises(ValueError, match="prefetch"):
        R.compress_module(model, prefetch=True, matvec=4)
    with pytest.raises(ValueError, match="prefetch"):
        R.load_module(model, [], prefetch=True, matvec=1)
    for bad in (-1, R.MATVEC_MAX_TOKENS + 1, 1.5, "4"):
        with pytest.raises(ValueError, match="matvec"):
            R.compress_module(model, matvec=bad)
    assert R._options(prefetch=True, matvec=0).matvec == 0
    assert R._options(matvec=R.MATVEC_MAX_TOKENS).matvec == R.MATVEC_MAX_TOKENS
