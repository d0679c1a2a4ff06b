"""The matvec and the tensor-core matmul (zipnn_b200_decode_plan_matvec / _matmul, DecodePlan.matvec / .matmul) on every
kind of stream the decoder tests use (tests/product_streams.py), compared bit for bit with the dense bytes.

  * one-hot extraction: x[t] = 2^k e_{i0 + t}, so y[t][o] = W[o][i0 + t] * 2^k exactly whatever the order of the
    additions (every other product is an exact zero).  i0 sweeps every column (64 rows of x per matmul call, 8 per
    matvec call), so every element of W goes through each kernel once; 1, 16, 17 and 33 rows on the first and last
    columns reach each MT instantiation and the masked token tiles.  NaN where W is NaN, +0 == -0, everything else
    bit for bit;
  * exact sums: x in {-1, 0, 1} and weights whose every partial sum is exact in fp32, so y is the fp64 product
    rounded once, with and without bias, at every chunk size and shape;
  * a scratch poisoned with 0xFF (fp32 NaN) before every call: a slot the reduce reads but no CTA wrote shows as
    NaN.  One scratch shared by items of different shapes and chunk sizes, eagerly and in one captured graph;
  * every bf16 / fp16 target of the multi-item plan layouts (piece, segment base, decoys), in every rotation;
  * host threads calling matmul, matvec and run on one plan at once;
  * inf, NaN, -0, subnormal weights and fp16 overflow; the largest item the products take (16383 chunks).
"""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

import multi_item_plans as M
import product_streams as S
import test_decode_plan_gpu as DP
import test_matmul_gpu as MM
import test_matvec_gpu as MV
import test_multi_item_plans_gpu as MI
from zipnn_b200 import DecodePlan, ZipNN, _native

pytestmark = pytest.mark.gpu

POISON = 0xFF   # fp32 NaN in every scratch slot


def _st():
    return torch.cuda.current_stream().cuda_stream


class Scratch:
    """One scratch buffer for every call of this file, poisoned before each call."""

    def __init__(self):
        self.buf = None

    def get(self, need: int) -> torch.Tensor:
        if self.buf is None or self.buf.numel() < need + 256:
            self.buf = torch.empty(2 * need + 256, dtype=torch.uint8, device="cuda")
        self.buf[: need + 256].fill_(POISON)
        return self.buf[:need]


SCRATCH = Scratch()


def raw_plan(cases) -> DP.Plan:
    p = DP.Plan([DP.Item(c.name, c.body, c.G, c.bits, c.chunk, c.data.size, c.data) for c in cases])
    assert p.rc == 0, [c.name for c in cases]
    return p


def scratch_size(kind, p, item, code, inf, nt):
    """-> (status, bytes) of zipnn_b200_decode_plan_{kind}_scratch_size; `code` the weights' dtype, None for
    matvec_fp8, which takes none."""
    sz = C.c_size_t(0)
    codes = () if code is None else (code,)
    rc = getattr(_native.lib(), f"zipnn_b200_decode_plan_{kind}_scratch_size")(C.byref(p.plan), item, *codes, inf, nt, C.byref(sz))
    return rc, sz.value


def product(kind, p, item, code, x, y_ptr, ys, bias=None, scratch=None):
    """One raw call with a poisoned scratch: asserts success and two launches."""
    nt, inf = x.shape
    rc, need = scratch_size(kind, p, item, code, inf, nt)
    assert rc == 0, (kind, item, rc)
    s = SCRATCH.get(need) if scratch is None else scratch
    before = _native.launch_count()
    rc = getattr(_native.lib(), f"zipnn_b200_decode_plan_{kind}")(C.byref(p.plan), item, code, inf, x.data_ptr(), x.stride(0), nt,
                                                                   None if bias is None else bias.data_ptr(), y_ptr, ys, s.data_ptr(),
                                                                   need, _st())
    assert rc == 0 and _native.launch_count() - before == 2, (kind, item, rc)


def same_bits(got, want, mask=None):
    """Elementwise on float tensors: equal bits, or both zero (+0 == -0), or both NaN (where mask)."""
    it = {2: torch.int16, 4: torch.int32}[got.element_size()]
    ok = (got.view(it) == want.view(it)) | ((got == 0) & (want == 0)) | (torch.isnan(got) & torch.isnan(want))
    return ok if mask is None else ok | ~mask


def _first_bad(ok):
    bad = (~ok).nonzero()
    return None if bad.numel() == 0 else tuple(bad[0].tolist())


# ------------------------------------------------------------------ one-hot extraction
def one_hot(kind, p, item, case, W, blocks, k, dtype=None):
    """Run the one-hot blocks [(i0, rows)] at scale 2^k; -> (got, expected, where checked) as [sum rows, out].  y is
    strided inside a NaN canary buffer."""
    dt = S.TORCH[dtype or case.dtype]
    code = S.CODE[dtype or case.dtype]
    inn, out = case.inn, case.out
    rows = sum(n for _, n in blocks)
    ybuf = torch.full((rows + 2, out + 6), float("nan"), dtype=dt, device="cuda")
    nmax = max(n for _, n in blocks)
    x = torch.zeros(nmax, inn, dtype=dt, device="cuda")
    ar = torch.arange(nmax, device="cuda")
    cols = []
    r0 = 0
    for i0, n in blocks:
        m = max(0, min(n, inn - i0))   # rows whose column exists; the rest stay zero
        x.zero_()
        x.view(-1).index_fill_(0, ar[:m] * (inn + 1) + i0, 2.0 ** k)
        product(kind, p, item, code, x[:n], ybuf[1 + r0].data_ptr() + 3 * ybuf.element_size(), out + 6)
        cols += list(range(i0, i0 + n))
        r0 += n
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    mask[1: rows + 1, 3: 3 + out] = False
    assert torch.all(torch.isnan(ybuf[mask])), f"{case.name}: {kind} wrote outside y"
    got = ybuf[1: rows + 1, 3: 3 + out]
    col = torch.tensor(cols, device="cuda")
    have = col < inn
    Wd = W.cuda()
    w64 = torch.zeros(rows, out, dtype=torch.float64, device="cuda")
    w64[have] = Wd.double().T[col[have]] * 2.0 ** k
    want = w64.to(dt)
    where = torch.zeros(rows, out, dtype=torch.bool, device="cuda")
    where[have] = S.valid(Wd, k, dtype or case.dtype).T[col[have]]
    where[~have] = True
    return got, want, where


def check_one_hot(kind, p, item, case, W=None, edges=True):
    W = case.weights() if W is None else W
    nt = S.MATMUL_NT if kind == "matmul" else S.MATVEC_NT
    seen = torch.zeros(case.out, case.inn, dtype=torch.bool, device="cuda")
    for k in S.scales(case.dtype, W):
        got, want, where = one_hot(kind, p, item, case, W, S.sweep(case.inn, nt), k)
        ok = same_bits(got, want, where)
        assert bool(ok.all()), (case.name, kind, k, _first_bad(ok))
        seen |= where.T
        if edges:
            blocks = [b for b in S.edge_blocks(case.inn) if kind == "matmul" or b[1] <= S.MATVEC_NT]
            got, want, where = one_hot(kind, p, item, case, W, blocks, k)
            ok = same_bits(got, want, where)
            assert bool(ok.all()), (case.name, kind, "edges", k, _first_bad(ok))
    assert bool(seen.all()), f"{case.name}: an element no sweep checked"


def check_exact_sums(kind, p, item, case, seed):
    W = case.weights().cuda()
    dt = S.TORCH[case.dtype]
    nts = (1, 17, 64) if kind == "matmul" else (1, 3, 8)
    for nt in nts:
        for with_bias in (False, True):
            x = S.exact_x(case.dtype, nt, case.inn, seed + nt).cuda()
            bias = S.exact_weights(case.dtype, (case.out,), seed + 7).cuda() if with_bias else None
            y = torch.full((nt, case.out), float("nan"), dtype=dt, device="cuda")
            product(kind, p, item, case.code, x, y.data_ptr(), case.out, bias=bias)
            ref = x.double() @ W.double().T + (bias.double() if with_bias else 0)
            ok = same_bits(y, ref.to(dt))
            assert bool(ok.all()), (case.name, kind, nt, with_bias, _first_bad(ok))


def _kinds(case):
    return ("matmul", "matvec") if case.G == 2 else ("matvec",)


@pytest.mark.parametrize("chunk", S.CHUNKS)
def test_shapes_at_every_chunk_size(chunk):
    cases = S.shape_cases(chunk)
    p = raw_plan(cases)   # one plan: items of different shapes and dtypes share the scratch, in turn
    for i, case in enumerate(cases):
        for kind in _kinds(case):
            check_one_hot(kind, p, i, case)
            if case.G == 2:   # (fp32 weights have 24 significant bits: no sum of them is exact in fp32)
                check_exact_sums(kind, p, i, case, 100 * i)
    for it in p.items:
        it.check("products")   # (the outputs hold what create decoded: no product wrote them)
    assert p.status() == 0


def test_stream_kinds():
    cases = S.stream_cases()
    for case in cases:
        p = raw_plan([case])
        for kind in _kinds(case):
            check_one_hot(kind, p, 0, case)
        p.items[0].scribble()
        assert p.run() == 0 and p.status() == 0
        p.items[0].check("run after the products")


def test_table_log_12_is_refused_at_create():
    for bits in (1, 0):
        case = S.log12_case(bits)
        p = DP.Plan([DP.Item(case.name, case.body, 2, bits, case.chunk, case.data.size, case.data)])
        assert p.rc == _native.E_UNSUPPORTED, p.rc


# ------------------------------------------------------------------ one scratch, many items, a graph
def test_shared_scratch_eager_and_in_a_graph():
    """Items of different shapes and chunk sizes multiplied in turn through one scratch, eagerly and replayed from one
    captured graph; between replays the scratch is poisoned again."""
    cases = [c for ch in (512, 4096, 262144) for c in S.shape_cases(ch, dtypes=("bf16", "fp16"))[:4]]
    plans = [raw_plan([c]) for c in cases]
    calls = []
    need = 0
    for c, p in zip(cases, plans):
        for kind, nt in (("matmul", 33), ("matvec", 5), ("matmul", 64)):
            need = max(need, scratch_size(kind, p, 0, c.code, c.inn, nt)[1])
            x = S.exact_x(c.dtype, nt, c.inn, len(calls)).cuda()
            calls.append((kind, p, c, x, torch.full((nt, c.out), float("nan"), dtype=S.TORCH[c.dtype], device="cuda")))
    scratch = torch.full((need,), POISON, dtype=torch.uint8, device="cuda")

    def all_calls():
        for kind, p, c, x, y in calls:
            product(kind, p, 0, c.code, x, y.data_ptr(), c.out, scratch=scratch)

    def check(what):
        for kind, p, c, x, y in calls:
            ref = (x.double() @ c.weights().cuda().double().T).to(y.dtype)
            ok = same_bits(y, ref)
            assert bool(ok.all()), (what, c.name, kind, _first_bad(ok))
            y.fill_(float("nan"))

    all_calls()
    check("eager")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        all_calls()
    for r in range(3):
        scratch.fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        check(f"replay {r}")
    # two calls, same bits, each on a freshly poisoned scratch
    for kind, p, c, x, y in calls[:6]:
        product(kind, p, 0, c.code, x, y.data_ptr(), c.out)
        first = y.clone()
        product(kind, p, 0, c.code, x, y.data_ptr(), c.out)
        assert torch.equal(first.view(torch.uint8), y.view(torch.uint8)), (c.name, kind)


# ------------------------------------------------------------------ multi-item plans
def _refused_matmul(p, i, e):
    L = _native.lib()
    row = e.orig // e.shape[0] if len(e.shape) > 1 and e.orig else 0
    in_bytes = row if row and row % 16 == 0 else 16
    inf = in_bytes // 2
    x = torch.zeros(16, inf, dtype=torch.bfloat16, device="cuda")
    y = torch.full((16 * max(1, e.orig // in_bytes) * 2,), MV.CANARY, dtype=torch.uint8, device="cuda")
    scratch = SCRATCH.get(4 << 20)
    code = 1 if e.dtype == "fp16" else 0
    before = _native.launch_count()
    assert scratch_size("matmul", p, i, code, inf, 16)[0] == _native.E_UNSUPPORTED, e.name
    rc = L.zipnn_b200_decode_plan_matmul(C.byref(p.plan), i, code, inf, x.data_ptr(), inf, 16, None, y.data_ptr(), max(1, e.orig // in_bytes),
                                         scratch.data_ptr(), scratch.numel(), _st())
    assert rc == _native.E_UNSUPPORTED and _native.launch_count() == before, (e.name, rc)
    assert torch.all(y == MV.CANARY), e.name


def _matmul_ok_target(e):
    return e.eligible and e.dtype in ("bf16", "fp16")


@pytest.mark.parametrize("name", M.LAYOUTS)
def test_matmul_on_every_item_of_every_rotation(name, monkeypatch, dev_streams):
    entries, env = M.layout(name)
    MI._set_env(monkeypatch, env)
    limit = M.limit_of(env)
    n = 0
    for r in M.placements(entries):
        es = M.rotate(entries, r)
        model = M.Model(es, limit)
        p = DP.Plan([MI._item(e) for e in es])
        assert p.rc == 0
        for it in p.items:
            it.scribble()
        for i, e in enumerate(es):
            W = MI._weight(e)
            if model.piece[i] >= 0 and _matmul_ok_target(e):
                for nt in (1, 17, 64):
                    x = MI._x(e.dtype, (nt, e.shape[-1]), 31 * r + i + nt)
                    y = torch.full((nt, W.shape[0]), float("nan"), dtype=W.dtype, device="cuda")
                    product("matmul", p, i, S.CODE[e.dtype], x, y.data_ptr(), W.shape[0])
                    MM._check(y, x, W.reshape(W.shape[0], -1), None, (name, r, e.name, nt))
                    n += 1
            elif e.dtype in ("bf16", "fp16", "fp32", "fp8"):
                _refused_matmul(p, i, e)
        torch.cuda.synchronize()
        for it in p.items:
            host = it.out.cpu().numpy()
            assert np.all(host[DP.PAD: DP.PAD + it.want.size] == DP.CANARY ^ 0xFF), f"{it.name}: a matmul wrote a plan output"
        assert p.run() == 0 and p.status() == 0
        for it in p.items:
            it.check(f"run after the matmuls, rotation {r}")
        dp = M.without_boxes(es)
        dmodel = M.Model(dp, limit)
        plan = DecodePlan([dev_streams(e) for e in dp])
        for o in plan.outputs:
            o.view(torch.uint8).fill_(DP.CANARY)
        for k, e in enumerate(dp):
            if dmodel.piece[k] >= 0 and _matmul_ok_target(e):
                W = MI._weight(e)
                x = MI._x(e.dtype, (33, e.shape[-1]), 1000 * r + k)
                bias = MI._x(e.dtype, (e.shape[0],), 7 * k, std=0.5)
                MM._check(plan.matmul(k, x, bias=bias, scratch=SCRATCH.get(plan.matmul_scratch_bytes(k, e.shape[-1], 33))), x,
                          W.reshape(W.shape[0], -1), bias, (name, r, e.name))
            elif e.kind != "empty" and len(e.shape) > 1:
                assert not plan.matmul_ok(k, e.shape[-1]), e.name
        for o in plan.outputs:
            assert torch.all(o.view(torch.uint8) == DP.CANARY), "a matmul wrote a plan output"
        plan.run()
        for o, e in zip(plan.outputs, dp):
            assert torch.equal(o.view(torch.uint8).reshape(-1).cpu(), torch.from_numpy(e.data)), e.name
        plan.check()
    assert n > 0
    print(f"{name}: {n} matmuls")


@pytest.fixture(scope="module")
def dev_streams():
    cache = {}

    def get(e):
        if e.name not in cache:
            cache[e.name] = torch.from_numpy(e.stream.copy()).cuda()
        return cache[e.name]
    return get


# ------------------------------------------------------------------ threads
def test_products_and_runs_from_many_threads():
    """Four host threads, each on its own CUDA stream with its own scratch, call matmul and matvec on one plan in a
    shuffled order; runs of the plan (whose own scratch is one) take turns under a lock.  Every result equals what the
    same call gave from one thread, bit for bit."""
    import random
    ws = [S.exact_weights("bf16", (256, 1024), 1), S.exact_weights("fp16", (96, 520), 2), S.exact_weights("fp32", (64, 512), 3)]
    streams = [ZipNN(input_format="torch", compression_chunk=ch).compress(w.cuda()) for w, ch in zip(ws, (4096, 262144, 8192))]
    plan = DecodePlan(streams)
    calls = []
    g = torch.Generator("cuda").manual_seed(5)
    for k, w in enumerate(ws):
        for kind, nt in (("matmul", 64), ("matmul", 9), ("matvec", 8), ("matvec", 1)):
            if kind == "matmul" and w.dtype == torch.float32:
                continue
            calls.append((kind, k, (torch.randn(nt, w.shape[1], generator=g, device="cuda")).to(w.dtype)))
    want = [getattr(plan, kind)(k, x) for kind, k, x in calls]
    need = max(getattr(plan, f"{kind}_scratch_bytes")(k, x.shape[1], x.shape[0]) for kind, k, x in calls)
    torch.cuda.synchronize()
    lock = threading.Lock()
    W_THREADS, ROUNDS = 4, 4

    def body(i, at):
        rng = random.Random(i)
        scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
        for r in range(ROUNDS):
            order = list(range(len(calls))) + ["run"]
            rng.shuffle(order)
            for j in order:
                at(f"round {r} call {j}")
                if j == "run":
                    with lock:
                        outs = plan.run()
                        torch.cuda.current_stream().synchronize()
                        for o, w in zip(outs, ws):
                            assert torch.equal(o.cpu().view(torch.uint8), w.view(torch.uint8)), "run"
                    continue
                kind, k, x = calls[j]
                scratch.fill_(POISON)
                got = getattr(plan, kind)(k, x, scratch=scratch)
                assert torch.equal(got.view(torch.uint8), want[j].view(torch.uint8)), (kind, k, x.shape)

    from test_threads_gpu import run_workers
    run_workers(W_THREADS, body)
    plan.check()


# ------------------------------------------------------------------ special values
def _special_ref_check(y, x, w, what):
    """y against the fp64 product: NaN exactly where it is NaN, the same infinity where it is infinite, +-inf where an
    fp16 result is past the largest finite value, and within test_matmul_gpu's bound elsewhere."""
    x64, w64 = x.double(), w.double()
    ref = x64 @ w64.T
    y64 = y.double()
    assert torch.equal(torch.isnan(y64), torch.isnan(ref)), (what, "NaN", _first_bad(torch.isnan(y64) == torch.isnan(ref)))
    inf = torch.isinf(ref)
    assert torch.equal(y64[inf], ref[inf]), (what, "inf")
    fin = torch.isfinite(ref)
    mag = x64.abs() @ torch.where(torch.isfinite(w64), w64.abs(), 0).T
    bound = (x.shape[-1] + 1) * 2.0 ** -23 * mag + ref.abs() * MV.REL[y.dtype] + MV.TINY[y.dtype]
    top = S.MAX_OUT["fp16"] if y.dtype == torch.float16 else float("inf")
    over = fin & (ref.abs() - bound > top + 16)     # rounds past 65504 whatever the last bits
    under = fin & (ref.abs() + bound < top)
    assert torch.equal(y64[over], torch.sign(ref[over]) * float("inf")), (what, "overflow to inf")
    err = (y64 - ref).abs()
    ok = ~under | (err <= 2 * bound)
    assert bool(ok.all()), (what, _first_bad(ok))
    return int(over.sum())


@pytest.mark.parametrize("dtype,bits", S.LAYOUTS)
def test_special_values(dtype, bits):
    case, at = S.special_case(dtype, bits)
    p = raw_plan([case])
    W = case.weights().cuda()
    n_over = 0
    for kind in _kinds(case):
        nts = (1, 5, 17, 64) if kind == "matmul" else (1, 5, 8)
        for nt in nts:
            x = torch.randn(nt, case.inn, generator=torch.Generator("cuda").manual_seed(nt), device="cuda").to(W.dtype)
            if dtype == "fp16":
                x = x * 8
            y = torch.full((nt, case.out), 0.0, dtype=W.dtype, device="cuda")
            product(kind, p, 0, case.code, x, y.data_ptr(), case.out)
            n_over += _special_ref_check(y, x, W, (case.name, kind, nt))
        # one-hot over every column: the rows with inf / NaN give NaN except at their own infinities; -0 and
        # subnormals come back exactly (bf16 / fp32 exponent-0 weights at a scale that makes them normal)
        nt = S.MATMUL_NT if kind == "matmul" else S.MATVEC_NT
        for k in S.scales(dtype, W):
            got, want, where = one_hot(kind, p, 0, case, W, S.sweep(case.inn, nt), k)
            X = torch.eye(case.inn, dtype=torch.float64, device="cuda") * 2.0 ** k
            ref = (X @ W.double().T)
            bad_rows = ~torch.isfinite(W).all(1)
            want = torch.where(bad_rows[None, :], ref, want.double()).to(W.dtype)
            where = where | bad_rows[None, :]
            ok = same_bits(got, want, where)
            assert bool(ok.all()), (case.name, kind, k, _first_bad(ok))
    if dtype == "fp16":
        assert n_over > 0, "some fp16 sums must pass 65504"


# ------------------------------------------------------------------ subnormal products
def test_subnormal_products_at_x_1():
    """x = 1 times bf16 exponent-0 weights gives fp32-subnormal products.  The matvec (fp32 FMAs, no flush) keeps them;
    on an H100 80GB HBM3 mma.sync keeps them too, and decode + F.linear gives the same (DESIGN 3.12).  fp16 subnormal
    weights at x = 1 give normal fp32 products, bit for bit."""
    found = []
    for dtype, bits in S.LAYOUTS16:
        g = torch.Generator().manual_seed(7)
        w = (torch.randn(64, 256, generator=g) * 0.02).to(S.TORCH[dtype])
        iv = w.view(torch.int16)
        m = torch.randint(1, 1 << (7 if dtype == "bf16" else 10), (64, 128), generator=g, dtype=torch.int16)
        iv[:, ::2] = m | torch.where(torch.rand(64, 128, generator=g) < 0.5, -32768, 0).to(torch.int16)
        case = S.Case(f"sub_{dtype}b{bits}", dtype, bits, 4096, (64, 256), w.view(torch.uint8).numpy())
        p = raw_plan([case])
        wd = w.cuda()
        x = torch.zeros(64, 256, dtype=wd.dtype, device="cuda")
        x[torch.arange(64), torch.arange(64) * 2] = 1.0   # row t picks the subnormal at column 2t
        res = {}
        for kind in ("matmul", "matvec"):
            y = torch.full((64, 64), float("nan"), dtype=wd.dtype, device="cuda")
            for t0 in range(0, 64, 64 if kind == "matmul" else 8):
                n = 64 if kind == "matmul" else 8
                product(kind, p, 0, case.code, x[t0: t0 + n], y[t0].data_ptr(), 64)
            res[kind] = y
        res["linear"] = torch.nn.functional.linear(x, wd)
        want = wd[:, ::2][:, :64].T.contiguous()   # y[t][o] = W[o][2t]
        for name, y in res.items():
            ok = same_bits(y, want)
            kept = int(((y != 0) & (want != 0)).sum())
            print(f"{dtype} bits={bits} {name}: {int(ok.sum())} of {ok.numel()} exact, {kept} non-zero")
            found.append((dtype, bits, name, bool(ok.all()), _first_bad(ok)))
    assert all(f[3] for f in found), [f for f in found if not f[3]]


# ------------------------------------------------------------------ the largest item
BIG_CHUNKS = 16383   # the largest whole tensor that stays one piece: a run of 16384 chunks is cut into two


def _big_room(nbytes):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    need = 3 * nbytes + (4 << 30)   # dense, stream and the plan's output at create, and room for the rest
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{free / 2 ** 30:.1f} GiB of device memory free, {need / 2 ** 30:.1f} GiB needed")


def _big_weight(chunks, seed):
    n = chunks * 131072
    w = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    g = torch.Generator("cuda").manual_seed(seed)
    slab = 1 << 27
    for i in range(0, n, slab):
        m = min(slab, n - i)
        w[i: i + m] = (torch.randn(m, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    return w.view(-1, 16384)


def test_largest_item():
    """16383 chunks of 256 KiB (4 GiB - 256 KiB of bf16, element indices up to 2^31 - 2^17 - 1): every element through
    the matmul once and the first and last columns through the matvec.  16384 chunks are split into two pieces (a piece
    that starts on a chunk boundary covers at most 16383 of them), and both products refuse that item."""
    _big_room(BIG_CHUNKS * 262144)
    w = _big_weight(BIG_CHUNKS, 3)
    stream = ZipNN(input_format="torch").compress(w)
    plan = DecodePlan([stream])
    plan.release_out()
    out_f, inn = w.shape
    assert plan.matmul_ok(0, inn) and plan.matvec_ok(0, inn)
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    x = torch.zeros(64, inn, dtype=torch.bfloat16, device="cuda")
    ar = torch.arange(64, device="cuda")
    y = torch.empty(64, out_f, dtype=torch.bfloat16, device="cuda")
    scratch = SCRATCH.get(plan.matmul_scratch_bytes(0, inn, 64))
    for i0, n in S.sweep(inn, 64):
        x.zero_()
        x.view(-1).index_fill_(0, ar[:n] * (inn + 1) + i0, 1.0)
        scratch.fill_(POISON)
        plan.matmul(0, x[:n], out=y[:n], scratch=scratch)
        bad += (~same_bits(y[:n], w[:, i0: i0 + n].T)).sum()
    for i0, n in ((0, 8), (inn - 8, 8)):
        x.zero_()
        x.view(-1).index_fill_(0, ar[:n] * (inn + 1) + i0, 1.0)
        got = plan.matvec(0, x[:n], scratch=SCRATCH.get(plan.matvec_scratch_bytes(0, inn, n)))
        bad += (~same_bits(got, w[:, i0: i0 + n].T)).sum()
    assert int(bad) == 0, int(bad)
    plan.check()
    del plan, stream, w, x, y
    _big_room((BIG_CHUNKS + 1) * 262144)
    w = _big_weight(BIG_CHUNKS + 1, 4)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    plan.release_out()
    assert not plan.matmul_ok(0, 16384) and not plan.matvec_ok(0, 16384), "a split item"
    L = _native.lib()
    xs = torch.zeros(2, 16384, dtype=torch.bfloat16, device="cuda")
    ys = torch.full((2, 8), float("nan"), dtype=torch.bfloat16, device="cuda")
    scratch = SCRATCH.get(1 << 20)
    for kind in ("matmul", "matvec"):
        before = _native.launch_count()
        rc = getattr(L, f"zipnn_b200_decode_plan_{kind}")(plan._ref, 0, 0, 16384, xs.data_ptr(), 16384, 2, None, ys.data_ptr(), 8,
                                                           scratch.data_ptr(), scratch.numel(), _st())
        assert rc == _native.E_UNSUPPORTED and _native.launch_count() == before, (kind, rc)
    assert torch.all(torch.isnan(ys))
