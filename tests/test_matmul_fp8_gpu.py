"""The tensor-core fp8 matmul (zipnn_b200_decode_plan_matmul_fp8, DecodePlan.matmul_fp8) on every kind of fp8 stream
of tests/fp8_streams.py, and the resident fp8 modules' fp8_matmul=N.

Numerics: y[t][o] = x_dtype(sum_i x[t][i] * D[o][i] (+ bias[o])), D = x_dtype(float(W) * S) the weight dequant_fp8
writes, products and sums in fp32.
  * one-hot extraction: x[t] = 2^k e_{i0 + t} over every column of every case, at 1 to 64 rows per call, both formats,
    bf16 and fp16 x, the four scale layouts, y strided inside a NaN canary buffer and the scratch poisoned with NaN:
    y = D * 2^k bit for bit (NaN where another weight of the row is not finite, as 0 * inf);
  * exact sums: integer weights and x, power-of-two scales;
  * block-quantized Gaussian weights through the public API against fp64 x D^T: bias, `out` row views, misaligned x
    rows, determinism, per-tensor and per-row scales;
  * NaN and infinity positions against F.linear of torch's dequantize; a CUDA graph replayed with new x and scale;
  * every item of a multi-item plan, interleaved with runs, matvec_fp8 and dequant_fp8;
  * every host rejection; the corrupted fp8 streams of corrupt_streams.py;
  * resident modules with fp8_matmul=64: the tiny fp8 Llama of test_dequant_fp8_gpu and the every-mode model of
    test_resident_modes_gpu.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

import corrupt_streams as CS
import fp8_streams as F
import test_decode_plan_gpu as DP
import test_dequant_fp8_gpu as DQ
import test_resident_modes_gpu as RM
from test_dequant_fp8_host import model as dq_model
from test_product_streams_gpu import POISON, SCRATCH, _first_bad, _st, raw_plan, same_bits, scratch_size
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200 import resident as R
from zipnn_b200.plan import MATMUL_MAX_TOKENS

pytestmark = pytest.mark.gpu

LAYOUT_NAMES = ("tensor", "row", "block128", "bk16")
ROWS = (1, 8, 9, 15, 16, 17, 31, 32, 33, 48, 63, 64)


@pytest.fixture(scope="module", autouse=True)
def _release_cached_memory():
    """Whole models and captured F.linear calls here leave cuBLAS workspaces and cached blocks behind, which are
    released once the module is done (as test_dequant_fp8_gpu does)."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch._C._cuda_clearCublasWorkspaces()
    torch.cuda.empty_cache()


def call(p, item, fmt, xdt, x, scale, bn, bk, y_ptr, ys, bias=None):
    """One raw call on a scratch poisoned with NaN: asserts success and two launches."""
    nt, inf = x.shape
    rc, need = scratch_size("matmul_fp8", p, item, None, inf, nt)
    assert rc == 0, (item, rc)
    s = SCRATCH.get(need)
    before = _native.launch_count()
    rc = _native.lib().zipnn_b200_decode_plan_matmul_fp8(C.byref(p.plan), item, F.CODE[fmt], F.XCODE[xdt], inf, x.data_ptr(), x.stride(0),
                                                         nt, scale.data_ptr(), bn, bk, None if bias is None else bias.data_ptr(), y_ptr,
                                                         ys, s.data_ptr(), need, _st())
    assert rc == 0 and _native.launch_count() - before == 2, (item, rc)


def dequantized(case, s, bn, bk, xdt) -> np.ndarray:
    """D = xdt(fl32(W * S)) as float32, from the numpy model of dequant_fp8."""
    b = dq_model(case.data.reshape(case.out, case.inn), case.dtype, DQ.expanded(s, case.out, case.inn, bn, bk), xdt)
    if xdt == "fp16":
        return b.view(np.float16).astype(np.float32)
    return (b.astype(np.uint32) << 16).view(np.float32)


def one_hot_want(d: np.ndarray, k: int, xdt: str) -> np.ndarray:
    """[in, out]: column i of x = 2^k e_i -> xdt(D[o][i] * 2^k), NaN where another weight of row o is not finite."""
    bad = ~np.isfinite(d)
    other = (bad.sum(1, keepdims=True) - bad) > 0
    with np.errstate(invalid="ignore", over="ignore"):
        v = F._round_to(d * np.float32(2.0 ** k), xdt)
    return np.where(other, np.float32(np.nan), v).T


def _scale(case, layout, seed):
    bn, bk = F.layouts(case.out, case.inn)[layout]
    s = F.random_scales(case.out, case.inn, bn, bk, seed)
    return s, torch.from_numpy(s).cuda(), bn, bk


def check_one_hot(p, item, case, xdt, layout, k=0, first=0):
    """Every column through the kernel once, at the row counts of ROWS in turn (from ROWS[first])."""
    s, sd, bn, bk = _scale(case, layout, item + 17)
    dt = F.XDTYPES[xdt]
    inn, out = case.inn, case.out
    ybuf = torch.full((inn + 2, out + 6), float("nan"), dtype=dt, device="cuda")
    x = torch.zeros(MATMUL_MAX_TOKENS, inn, dtype=dt, device="cuda")
    ar = torch.arange(MATMUL_MAX_TOKENS, device="cuda")
    i0, r = 0, first
    while i0 < inn:
        n = min(ROWS[r % len(ROWS)], inn - i0)
        x.zero_()
        x.view(-1).index_fill_(0, ar[:n] * (inn + 1) + i0, 2.0 ** k)
        call(p, item, case.dtype, xdt, x[:n], sd, bn, bk, ybuf[1 + i0].data_ptr() + 3 * ybuf.element_size(), out + 6)
        i0, r = i0 + n, r + 1
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    mask[1: inn + 1, 3: 3 + out] = False
    assert torch.all(torch.isnan(ybuf[mask])), f"{case.name}: wrote outside y"
    got = ybuf[1: inn + 1, 3: 3 + out].float().cpu()
    want = torch.from_numpy(np.ascontiguousarray(one_hot_want(dequantized(case, s, bn, bk, xdt), k, xdt)))
    ok = same_bits(got, want)
    assert bool(ok.all()), (case.name, xdt, layout, _first_bad(ok))


@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_one_hot_at_every_chunk_size(chunk):
    cases = F.shape_cases(chunk)
    p = raw_plan(cases)   # one plan: items of different shapes and formats in turn
    k0 = F.CHUNKS.index(chunk)
    for i, case in enumerate(cases):
        for xdt in ("bf16", "fp16"):
            check_one_hot(p, i, case, xdt, LAYOUT_NAMES[(i + k0 + (xdt == "fp16")) % 4], first=i + k0)
    for it in p.items:
        it.check("after the products")   # (the outputs hold what create decoded: no product wrote them)
    assert p.status() == 0


def test_one_hot_on_every_stream_kind():
    for j, case in enumerate(F.stream_cases()):
        p = raw_plan([case])
        for xdt in ("bf16", "fp16"):
            for li, layout in enumerate(LAYOUT_NAMES):
                check_one_hot(p, 0, case, xdt, layout, k=(0, -2)[li % 2], first=j + li)
        p.items[0].scribble()
        assert p.run() == 0 and p.status() == 0
        p.items[0].check("run after the products")


# ------------------------------------------------------------------ exact sums
def test_exact_integer_sums():
    rng = np.random.default_rng(7)
    for j, (fmt, chunk, shape) in enumerate((("e4m3", 512, (160, 400)), ("e5m2", 4096, (5, 8192)), ("e4m3", 131072, (64, 4096)),
                                             ("e5m2", 2048, (48, 160)))):
        case = F.integer_case(fmt, chunk, shape, j)
        p = raw_plan([case])
        for layout in LAYOUT_NAMES:
            bn, bk = F.layouts(case.out, case.inn)[layout]
            s = (2.0 ** rng.integers(-2, 3, F.grid_shape(case.out, case.inn, bn, bk))).astype(np.float32)
            wd = F.dequantized(case.floats(), s, bn, bk)
            for xdt in ("bf16", "fp16"):
                for nt in (1, 9, 33, 64):
                    x = torch.from_numpy(rng.integers(-2, 3, (nt, case.inn)).astype(np.float32)).to(F.XDTYPES[xdt])
                    y = torch.full((nt, case.out), float("nan"), dtype=F.XDTYPES[xdt], device="cuda")
                    call(p, 0, fmt, xdt, x.cuda(), torch.from_numpy(s).cuda(), bn, bk, y.data_ptr(), case.out)
                    want = torch.from_numpy(x.double().numpy() @ wd.T).to(y.dtype)
                    assert torch.equal(y.cpu(), want), (case.name, layout, xdt, nt)


# ------------------------------------------------------------------ the public API on block-quantized weights
def check64(y, x, d, bias, what):
    """y against fp64 x D^T (+ bias): fp32 products and sums of `in` terms, then one rounding (two with a bias)."""
    d64 = d.double()
    x64 = x.double().reshape(-1, x.shape[-1])
    ref, mag = x64 @ d64.T, x64.abs() @ d64.abs().T
    bound = (x.shape[-1] + 2) * 2.0 ** -23 * mag
    rel = 2.0 ** -8 if y.dtype == torch.bfloat16 else 2.0 ** -11
    tol = bound + (ref.abs() + bound) * rel + (2.0 ** -24 if y.dtype == torch.float16 else 0)
    if bias is not None:
        ref = ref + bias.double()
        tol = tol + (ref.abs() + tol) * rel
    err = (y.double().reshape(ref.shape) - ref).abs()
    assert torch.all(err <= tol), (what, float((err - tol).max()))


@pytest.mark.parametrize("fmt", F.FORMATS)
def test_block_quantized_weights_through_the_api(fmt):
    out_f, in_f = 992, 1040   # ragged 128x128 blocks on both edges
    wq, scale = DQ._quantized(fmt, out_f, in_f, 3)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    assert plan.matmul_fp8_ok(0, in_f) and not plan.matmul_ok(0, in_f)
    need = plan.matmul_fp8_scratch_bytes(0, in_f, 64)
    for xdt in (torch.bfloat16, torch.float16):
        d = DQ.torch_dequant(wq, scale, (128, 128), xdt)
        assert torch.equal(d.view(torch.int16), plan.dequant_fp8(0, in_f, scale, (128, 128), xdt).view(torch.int16))
        g = torch.Generator("cuda").manual_seed(5)
        for shape in ((9, in_f), (2, 8, in_f), (64, in_f), (1, in_f)):
            x = torch.randn(shape, generator=g, device="cuda").to(xdt)
            bias = torch.randn(out_f, generator=g, device="cuda").to(xdt) * 0.1
            scratch = torch.full((need,), POISON, dtype=torch.uint8, device="cuda")
            y = plan.matmul_fp8(0, x, scale, block=(128, 128), bias=bias, scratch=scratch)
            assert y.shape == shape[:-1] + (out_f,) and y.dtype == xdt
            check64(y, x, d, bias, (fmt, xdt, shape))
            scratch.fill_(POISON)
            again = plan.matmul_fp8(0, x, scale, block=(128, 128), bias=bias, scratch=scratch)
            assert torch.equal(again.view(torch.int16), y.view(torch.int16)), "two calls, same bits"
        # out as a column slice of a wider buffer; x rows that are not 16-byte aligned (copied first)
        x = torch.randn(37, in_f, generator=g, device="cuda").to(xdt)
        wide = torch.full((37, out_f + 24), float("nan"), dtype=xdt, device="cuda")
        view = wide[:, 8: 8 + out_f]
        plan.matmul_fp8(0, x, scale, (128, 128), out=view)
        check64(view, x, d, None, (fmt, xdt, "out view"))
        assert torch.all(torch.isnan(wide[:, :8])) and torch.all(torch.isnan(wide[:, 8 + out_f:]))
        xbuf = torch.zeros(37 * in_f + 1, dtype=xdt, device="cuda")
        xm = xbuf[1:].view(37, in_f)
        xm.copy_(x)
        assert xm.data_ptr() % 16
        assert torch.equal(plan.matmul_fp8(0, xm, scale, (128, 128)).view(torch.int16), view.contiguous().view(torch.int16))
    # per tensor (block=None) and per row
    x = torch.randn(20, in_f, device="cuda").to(torch.bfloat16)
    one = torch.tensor([0.001], device="cuda")
    check64(plan.matmul_fp8(0, x, one), x, DQ.torch_dequant(wq, one, None, torch.bfloat16), None, "per tensor")
    rows = torch.rand(out_f, device="cuda") * 0.01
    check64(plan.matmul_fp8(0, x, rows, block=(1, in_f)), x, DQ.torch_dequant(wq, rows.view(-1, 1), (1, in_f), torch.bfloat16),
            None, "per row")
    plan.check()


def test_graph_capture_replays_with_new_x_and_scale():
    wq, scale = DQ._quantized("e4m3", 512, 2048, 11)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    x = torch.randn(40, 2048, device="cuda").to(torch.bfloat16)
    y = torch.empty(40, 512, dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(plan.matmul_fp8_scratch_bytes(0, 2048, 40), dtype=torch.uint8, device="cuda")
    plan.matmul_fp8(0, x, scale, (128, 128), out=y, scratch=scratch)   # first call outside: it reads the chunk modes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.matmul_fp8(0, x, scale, (128, 128), out=y, scratch=scratch)
    for r in range(3):
        x.copy_(torch.randn(40, 2048, device="cuda").to(torch.bfloat16))
        scale.mul_(1.5)
        scratch.fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        want = plan.matmul_fp8(0, x, scale, (128, 128))
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), r
        check64(y, x, DQ.torch_dequant(wq, scale, (128, 128), torch.bfloat16), None, ("replay", r))


def test_every_item_of_a_multi_item_plan_interleaved_with_other_calls():
    ws = [DQ._quantized("e4m3", 256, 1024, 1), DQ._quantized("e5m2", 96, 528, 2), DQ._quantized("e4m3", 1, 4096, 3)]
    other = (torch.randn(64, 512, device="cuda") * 0.02).to(torch.bfloat16)
    tensors = [ws[0][0], other, ws[1][0], ws[2][0]]
    streams = [ZipNN(input_format="torch", compression_chunk=ch).compress(t) for t, ch in zip(tensors, (65536, 262144, 131072, 131072))]
    plan = DecodePlan(streams)
    assert not plan.matmul_fp8_ok(1, 512), "a bf16 output"
    xs = {k: torch.randn(23, wq.shape[1], device="cuda").to(torch.float16) for k, (wq, _) in zip((0, 2, 3), ws)}
    alone = {}
    for k, (wq, scale) in zip((0, 2, 3), ws):
        single = DecodePlan([streams[k]])
        alone[k] = single.matmul_fp8(0, xs[k], scale, (128, 128))
        check64(alone[k], xs[k], DQ.torch_dequant(wq, scale, (128, 128), torch.float16), None, k)
    for r in range(2):
        for k, (wq, scale) in zip((0, 2, 3), ws):
            y = plan.matmul_fp8(k, xs[k], scale, (128, 128))
            assert torch.equal(y.view(torch.int16), alone[k].view(torch.int16)), (r, k)
            plan.matvec_fp8(k, xs[k][:8], scale, (128, 128))
            d = plan.dequant_fp8(k, wq.shape[1], scale, (128, 128), torch.float16)
            assert torch.equal(d.view(torch.int16), DQ.torch_dequant(wq, scale, (128, 128), torch.float16).view(torch.int16))
            outs = plan.run()
            torch.cuda.synchronize()
            for o, t in zip(outs, tensors):
                assert torch.equal(o.view(torch.uint8), t.view(torch.uint8)), (r, k)
    plan.check()


# ------------------------------------------------------------------ special values
@pytest.mark.parametrize("fmt", F.FORMATS)
def test_special_values_match_f_linear_of_the_dequantized_weight(fmt):
    """NaN and infinity positions are those of F.linear of the dequantized weight (the numpy model of dequant_fp8, bit
    for bit torch's dequantize), in fp64; scales 0.25 and 2^12 (fp16 overflow in D)."""
    case, _ = F.special_case(fmt)
    p = raw_plan([case])
    for sv in (0.25, 2.0 ** 12):
        s = np.full((1, 1), sv, dtype=np.float32)
        sd = torch.from_numpy(s).cuda()
        for xdt in ("bf16", "fp16"):
            dt = F.XDTYPES[xdt]
            d = torch.from_numpy(dequantized(case, s, case.out, case.inn, xdt)).cuda()
            for nt in (9, 64):
                xr = torch.randn(nt, case.inn, generator=torch.Generator("cuda").manual_seed(nt), device="cuda").to(dt)
                y = torch.zeros(nt, case.out, dtype=dt, device="cuda")
                call(p, 0, fmt, xdt, xr, sd, case.out, case.inn, y.data_ptr(), case.out)
                ref = xr.double() @ d.double().T
                assert torch.equal(torch.isnan(y), torch.isnan(ref)), (fmt, xdt, sv, "NaN")
                inf = torch.isinf(ref)
                assert torch.equal(y.double()[inf], ref[inf]), (fmt, xdt, sv, "inf")


# ------------------------------------------------------------------ rejections
def test_host_rejections_write_nothing(monkeypatch):
    L = _native.lib()
    wq, scale = DQ._quantized("e4m3", 64, 4096, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    need = plan.matmul_fp8_scratch_bytes(0, 4096, 20)
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    x = torch.randn(20, 4096, device="cuda").to(torch.bfloat16)
    y = torch.full((20, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    bad = [("tokens", dict(nt=MATMUL_MAX_TOKENS + 1), A), ("format", dict(fmt=2), A), ("format -1", dict(fmt=-1), A),
           ("x dtype fp32", dict(xdt=2), A), ("x dtype 3", dict(xdt=3), A), ("in 0", dict(inf=0), A),
           ("in not dividing", dict(inf=4112), A), ("item -1", dict(item=-1), A), ("item 1", dict(item=1), A),
           ("null x", dict(x=None), A), ("null y", dict(y=None), A), ("null scratch", dict(scratch=None), A),
           ("null scale", dict(scale=None), A), ("scale alignment", dict(scale=scale.data_ptr() + 2), A),
           ("block rows 0", dict(bn=0), A), ("block cols 0", dict(bk=0), A), ("block cols 8", dict(bk=8), A),
           ("block cols 140", dict(bk=140), A),
           ("x alignment", dict(x=x.data_ptr() + 2), A), ("x stride", dict(xs=4100), A), ("short x stride", dict(xs=2048), A),
           ("short y stride", dict(ys=32), A), ("y alignment", dict(y=y.data_ptr() + 1), A), ("bias alignment", dict(bias=bias.data_ptr() + 1), A),
           ("scratch alignment", dict(scratch=scratch.data_ptr() + 16), A), ("short scratch", dict(sb=need - 1), A),
           ("rows of 8 bytes", dict(inf=8), U)]
    for name, kw, want in bad:
        a = dict(item=0, fmt=0, xdt=0, inf=4096, x=x.data_ptr(), xs=4096, nt=20, scale=scale.data_ptr(), bn=128, bk=128,
                 bias=bias.data_ptr(), y=y.data_ptr(), ys=64, scratch=scratch.data_ptr(), sb=need)
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_matmul_fp8(plan._ref, a["item"], a["fmt"], a["xdt"], a["inf"], a["x"], a["xs"], a["nt"], a["scale"],
                                                 a["bn"], a["bk"], a["bias"], a["y"], a["ys"], a["scratch"], a["sb"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    assert torch.all(torch.isnan(y))
    out = C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_matmul_fp8_scratch_size(plan._ref, 0, 4096, MATMUL_MAX_TOKENS + 1, C.byref(out)) == A
    assert L.zipnn_b200_decode_plan_matmul_fp8_scratch_size(plan._ref, 0, 4096, 2, None) == A
    # the scratch is the matmul's formula: 4 quarters x row tiles x tokens x 8 rows of fp32 per chunk
    assert plan.matmul_fp8_scratch_bytes(0, 4096, 20) % (4 * 20 * 8 * 4) == 0
    # the 16-bit matmul still refuses fp8 items, and the fp8 one refuses 16-bit items
    assert L.zipnn_b200_decode_plan_matmul(plan._ref, 0, 0, 4096, x.data_ptr(), 4096, 20, None, y.data_ptr(), 64, scratch.data_ptr(),
                                           need, _st()) == U
    other = DecodePlan([ZipNN(input_format="torch").compress((torch.randn(64, 4096, device="cuda") * 0.02).to(torch.bfloat16))])
    assert not other.matmul_fp8_ok(0, 4096)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matmul_fp8(other._ref, 0, 0, 0, 4096, x.data_ptr(), 4096, 20, scale.data_ptr(), 128, 128, None,
                                               y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
    # Python-side refusals
    for kw, what in ((dict(block=None), "a grid scale without block"), (dict(block=(128, 8)), "bk 8"), (dict(block=(0, 128)), "bn 0"),
                     (dict(block=(32, 128)), "a grid of another block"), (dict(scale=scale.double()), "fp64 scale"),
                     (dict(x=x.float()), "fp32 x"), (dict(x=torch.zeros(65, 4096, dtype=torch.bfloat16, device="cuda")), "65 rows")):
        a = dict(x=x, scale=scale, block=(128, 128))
        a.update(kw)
        with pytest.raises(ValueError):
            plan.matmul_fp8(0, a["x"], a["scale"], block=a["block"])
    assert _native.launch_count() == before and torch.all(torch.isnan(y))
    # every item matvec_fp8_ok refuses: a plain (incompressible) fp8 item, a box, a plan without a segment index
    raw = torch.randint(0, 256, (64 * 4096,), dtype=torch.uint8, device="cuda")
    raw[(raw & 0x7F) == 0x7F] = 0
    pl = DecodePlan([ZipNN(input_format="torch").compress(raw.view(torch.float8_e4m3fn).view(64, 4096))])
    assert not pl.matvec_fp8_ok(0, 4096) and not pl.matmul_fp8_ok(0, 4096)
    case = F.shape_cases(4096)[0]
    boxed = DP.Plan([DP.Item(case.name, case.body, 1, case.bits, case.chunk, case.data.size, case.data[:4096 * 2],
                             box=(0, 2, 8192, 4096))])
    assert boxed.rc == 0
    for p_ref in (pl._ref, C.byref(boxed.plan)):
        before = _native.launch_count()
        assert L.zipnn_b200_decode_plan_matmul_fp8_scratch_size(p_ref, 0, 16, 1, C.byref(C.c_size_t(0))) == U
        assert L.zipnn_b200_decode_plan_matmul_fp8(p_ref, 0, 0, 0, 16, x.data_ptr(), 16, 1, scale.data_ptr(), 1, 16, None,
                                                   y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
        assert _native.launch_count() == before
    DP._set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    q = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    before = _native.launch_count()
    assert not q.matmul_fp8_ok(0, 4096)
    assert L.zipnn_b200_decode_plan_matmul_fp8(q._ref, 0, 0, 0, 4096, x.data_ptr(), 4096, 20, scale.data_ptr(), 128, 128, None,
                                               y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
    assert _native.launch_count() == before and torch.all(torch.isnan(y))


def test_corrupted_fp8_streams_follow_the_model():
    """Every mutant of the fp8 base of corrupt_streams.py: a plan whose create fails is refused (E_ARG, nothing
    launched); one that creates decodes to the verdict's bytes and is refused (E_UNSUPPORTED), as by matvec_fp8."""
    import test_corrupt_streams_gpu as T
    b = CS.bases()["fp8_g1"]
    assert b.pr["mode"][-1] != "fused"
    L = _native.lib()
    x = torch.zeros(9, 16, dtype=torch.bfloat16, device="cuda")
    y = torch.full((b.orig // 8,), float("nan"), dtype=torch.bfloat16, device="cuda")
    sc = torch.ones(1, device="cuda")
    small = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.empty(T.PAD + b.orig + T.PAD, dtype=torch.uint8, device="cuda")
    n = 0
    for m, v in T.cases("fp8_g1"):
        body = torch.from_numpy(m.body).cuda()
        out.fill_(T.CANARY)
        rc, plan, keep = T._plan_create(b, body.data_ptr(), m.body.size, out[T.PAD:])
        assert rc == T.STATUS[v.status], (m.id, rc, v.status)
        p = C.byref(plan)
        before = _native.launch_count()
        got = L.zipnn_b200_decode_plan_matmul_fp8(p, 0, 0, 0, 8, x.data_ptr(), 16, 9, sc.data_ptr(), 1, 16, None, y.data_ptr(), 1,
                                                  small.data_ptr(), small.numel(), _st())
        assert got == (_native.E_ARG if rc else _native.E_UNSUPPORTED), (m.id, got)
        assert _native.launch_count() == before, m.id
        if not rc:
            assert torch.equal(out[T.PAD: T.PAD + b.orig], torch.from_numpy(v.data).cuda()), m.id
            n += 1
    assert torch.all(torch.isnan(y))
    assert n > 0


# ------------------------------------------------------------------ resident fp8 models
FP8_CALLS = ("run", "matvec_fp8", "matmul_fp8", "dequant_fp8")


def within_bound_of_d(y, x, mod):
    """y against fp64 x D^T (+ bias, added as FP8Linear adds it), D torch's dequantize in x's dtype."""
    d = DQ.torch_dequant(mod.weight, mod.weight_scale_inv, mod.block_size, x.dtype).double()
    x64 = x.double().reshape(-1, x.shape[-1])
    ref, mag = x64 @ d.T, x64.abs() @ d.abs().T
    rel = 2.0 ** -8 if y.dtype == torch.bfloat16 else 2.0 ** -11
    bound = (x.shape[-1] + 2) * 2.0 ** -23 * mag
    tol = bound + (ref.abs() + bound) * rel
    if mod.bias is not None:
        ref = ref + mod.bias.double()
        tol = tol + (ref.abs() + tol) * rel
    return bool(torch.all((y.double().reshape(ref.shape) - ref).abs() <= tol))


def _record(monkeypatch, names):
    calls = []
    for name in names:
        orig = getattr(DecodePlan, name)

        def wrap(plan, *a, _orig=orig, _name=name, **kw):
            calls.append(_name)
            return _orig(plan, *a, **kw)
        monkeypatch.setattr(DecodePlan, name, wrap)
    return calls


def check_paths_and_bound(m, ref, monkeypatch, seed):
    """At 1, 8, 9, 64 and 65 rows each fast FP8Linear makes the expected plan call; over 64 rows its output is the
    reference's bits, at most 64 within the fp64 bound of the product with the dequantized weight (rounded to x's
    dtype for matmul_fp8, exact for matvec_fp8)."""
    state = getattr(m, R._ATTR)
    fast = {id(x): mode == "fp8" for x, _, _, mode in state.entries if mode in ("fp8", "fp8_torch")}
    calls = _record(monkeypatch, FP8_CALLS)
    g = torch.Generator("cuda").manual_seed(seed)
    with torch.no_grad():
        for rows in (1, 8, 9, 64, 65):
            lins = [x for x in m.modules() if type(x).__name__ == "FP8Linear"]
            for mod in lins:
                x = torch.randn(rows, mod.in_features, generator=g, device="cuda").to(torch.bfloat16)
                calls.clear()
                y = mod(x)
                r = DQ._ref_of(ref, m, mod)
                if not fast[id(mod)]:
                    assert calls == ["run"] and torch.equal(DQ.bits(y), DQ.bits(r(x))), rows
                    continue
                want = "matvec_fp8" if rows <= 8 else "matmul_fp8" if rows <= 64 else "dequant_fp8"
                assert calls == [want], (rows, calls)
                if rows > 64:
                    assert torch.equal(DQ.bits(y), DQ.bits(r(x))), rows
                elif rows > 8:
                    assert within_bound_of_d(y, x, r), (rows, want)
                else:   # matvec_fp8 multiplies by S * W unrounded
                    assert DQ.within_fp64_bound(y, x, r), (rows, want)
    monkeypatch.undo()


def test_compress_module_fp8_matmul(monkeypatch):
    m = DQ.tiny_fp8_llama(1, constant=True)
    ref = DQ.reference(m)
    before = DQ.dense_state(m)
    report = compress_module(m, fp8=True, matvec=8, fp8_matmul=64)
    assert report["fp8_modules"] == 15 and report["fp8_matmul_modules"] == 14, "the constant weight takes the fallback"
    state = getattr(m, R._ATTR)
    want = max(e.plan.matmul_fp8_scratch_bytes(0, e.module.in_features, 64) for e in state.entries if e.mode == "fp8")
    assert report["fp8_matmul_scratch_bytes"] == want
    assert state.fp8_matmul_scratch.numel() >= want
    check_paths_and_bound(m, ref, monkeypatch, 2)
    # a captured forward through matmul_fp8, replayed with new inputs
    mod = m.model.layers[1].mlp.up_proj
    with torch.no_grad():
        x = torch.randn(33, mod.in_features, device="cuda").to(torch.bfloat16)
        mod(x)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = mod(x)
        for r in range(2):
            x.copy_(torch.randn(33, mod.in_features, device="cuda").to(torch.bfloat16))
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(DQ.bits(y), DQ.bits(mod(x))), r
    decompress_module(m)
    after = DQ.dense_state(m)
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(DQ.raw(after[k]), DQ.raw(before[k])), k
    for name, x in m.named_modules():
        assert "forward" not in x.__dict__ and not x._forward_pre_hooks and not x._forward_hooks, name


def test_load_module_fp8_matmul_from_safetensors_and_znn(tmp_path, monkeypatch):
    src = DQ.tiny_fp8_llama(3)
    ref = DQ.reference(src)
    sd = {k: v.contiguous() for k, v in DQ.dense_state(src).items()}
    plain = str(tmp_path / "fp8.safetensors")
    save_file(sd, plain)
    kw = dict(fp8=True, matvec=8, fp8_matmul=64)
    a = DQ.tiny_fp8_llama(4)   # other values: every one must come from the file
    rep_a = load_module(a, plain, **kw)
    check_paths_and_bound(a, ref, monkeypatch, 5)
    znn = str(tmp_path / "fp8.znn.safetensors")
    save_module(a, znn)
    b = DQ.tiny_fp8_llama(5)
    rep_b = load_module(b, znn, **kw)
    assert rep_a == rep_b and rep_a["fp8_matmul_modules"] == 15
    with torch.no_grad():
        for rows in (9, 40):
            ids = torch.randint(0, 512, (1, rows), device="cuda")
            assert torch.equal(DQ.bits(a(ids, use_cache=False).logits), DQ.bits(b(ids, use_cache=False).logits)), rows
    decompress_module(b)
    for k, v in DQ.dense_state(b).items():
        assert torch.equal(DQ.raw(v), DQ.raw(sd[k])), k


def test_every_mode_with_fp8_matmul(monkeypatch):
    """The every-mode model of test_resident_modes_gpu with fp8_matmul=64 added: fp8_proj takes matmul_fp8 at 9 to 64
    rows, and every other module keeps its path and its bits."""
    dense = RM.make(1)
    base, model = copy.deepcopy(dense), copy.deepcopy(dense)
    rep_base = compress_module(base, **RM.ALL)
    rep = compress_module(model, **RM.ALL, fp8_matmul=64)
    assert rep["fp8_matmul_modules"] == 1 and rep["fp8_matmul_scratch_bytes"] > 0
    assert {k: v for k, v in rep.items() if not k.startswith("fp8_matmul")} == rep_base
    monkeypatch.setattr(RM, "PLAN_CALLS", RM.PLAN_CALLS + ("matmul_fp8",))
    paths = RM.Paths(monkeypatch)
    hs = paths.watch(model)
    g = torch.Generator("cuda").manual_seed(2)
    with torch.no_grad():
        for rows in RM.ROWS:
            ids = torch.randint(0, RM.VOCAB, (1, rows), device="cuda", generator=g)
            paths.calls.clear()
            paths.io.clear()
            model(ids)
            got = paths.by_module()
            product = "matvec" if rows <= 8 else "matmul" if rows <= 64 else "run"
            assert got["up_proj"] == got["down_proj"] == got["lm_head"] == [product], (rows, got)
            assert got["embed_tokens"] == ["gather"] and got["moe.experts"] == ["run_select"], rows
            assert got["fp8_proj"] == ["matvec_fp8" if rows <= 8 else "matmul_fp8" if rows <= 64 else "dequant_fp8"], rows
            for name, args, kwargs, out in list(paths.io):
                want = base.get_submodule(name)(*args, **kwargs)
                if name == "fp8_proj" and 8 < rows <= 64:
                    assert within_bound_of_d(out, args[0], dense.get_submodule(name)), rows
                else:
                    assert torch.equal(RM.bits(out), RM.bits(want)), (name, rows)
    for h in hs:
        h.remove()
