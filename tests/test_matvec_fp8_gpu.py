"""The fp8 matvec (zipnn_b200_decode_plan_matvec_fp8, DecodePlan.matvec_fp8) on every kind of fp8 stream of
tests/fp8_streams.py, bit for bit against the numpy model of its numerics there.

  * one-hot extraction: x[t] = 2^k e_{i0 + t} over every column of every case, both formats, bf16 and fp16 x, the scale
    layouts per tensor, per row, 128x128 with ragged edges and bk = 16 taking turns: y = round(fl32(W 2^k) S);
  * random x and bias against the model, every fp32 operation in the kernels' order;
  * exact sums: integer weights and x, power-of-two scales;
  * block-quantized Gaussian weights through the public API against fp64: bias, `out` row views, misaligned x rows, a
    scratch poisoned with NaN before each call, determinism and a captured graph replayed with new x;
  * every item of a multi-item plan, interleaved with runs that still decode every output exactly;
  * NaN, infinities, -0 and subnormal weights; every host rejection; the corrupted fp8 streams of corrupt_streams.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import corrupt_streams as CS
import fp8_streams as F
import test_decode_plan_gpu as DP
from test_product_streams_gpu import POISON, SCRATCH, _first_bad, _st, raw_plan, same_bits, scratch_size
from zipnn_b200 import DecodePlan, ZipNN, _native
from zipnn_b200.plan import MATVEC_MAX_TOKENS

pytestmark = pytest.mark.gpu

LAYOUT_NAMES = ("tensor", "row", "block128", "bk16")


def call(p, item, fmt, xdt, x, scale, bn, bk, y_ptr, ys, bias=None):
    """One raw call on a poisoned scratch: asserts success and two launches."""
    nt, inf = x.shape
    rc, need = scratch_size("matvec_fp8", p, item, None, inf, nt)
    assert rc == 0, (item, rc)
    s = SCRATCH.get(need)
    before = _native.launch_count()
    rc = _native.lib().zipnn_b200_decode_plan_matvec_fp8(C.byref(p.plan), item, F.CODE[fmt], F.XCODE[xdt], inf, x.data_ptr(), x.stride(0),
                                                         nt, scale.data_ptr(), bn, bk, None if bias is None else bias.data_ptr(), y_ptr,
                                                         ys, s.data_ptr(), need, _st())
    assert rc == 0 and _native.launch_count() - before == 2, (item, rc)


def _scale(case, layout, seed):
    bn, bk = F.layouts(case.out, case.inn)[layout]
    s = F.random_scales(case.out, case.inn, bn, bk, seed)
    return s, torch.from_numpy(s).cuda(), bn, bk


# ------------------------------------------------------------------ one-hot and the model
def check_one_hot(p, item, case, xdt, layout, k=0):
    """Every column through the kernel once, 8 rows of x per call, y strided inside a NaN canary buffer."""
    s, sd, bn, bk = _scale(case, layout, item + 17)
    dt = F.XDTYPES[xdt]
    inn, out = case.inn, case.out
    ybuf = torch.full((inn + 2, out + 6), float("nan"), dtype=dt, device="cuda")
    x = torch.zeros(MATVEC_MAX_TOKENS, inn, dtype=dt, device="cuda")
    ar = torch.arange(MATVEC_MAX_TOKENS, device="cuda")
    for i0 in range(0, inn, MATVEC_MAX_TOKENS):
        n = min(MATVEC_MAX_TOKENS, inn - i0)
        x.zero_()
        x.view(-1).index_fill_(0, ar[:n] * (inn + 1) + i0, 2.0 ** k)
        call(p, item, case.dtype, xdt, x[:n], sd, bn, bk, ybuf[1 + i0].data_ptr() + 3 * ybuf.element_size(), out + 6)
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    mask[1: inn + 1, 3: 3 + out] = False
    assert torch.all(torch.isnan(ybuf[mask])), f"{case.name}: wrote outside y"
    got = ybuf[1: inn + 1, 3: 3 + out].float().cpu()
    want = torch.from_numpy(F.one_hot_model(case.floats(), s, bn, bk, np.arange(inn), k, xdt))
    ok = same_bits(got, want)
    assert bool(ok.all()), (case.name, xdt, layout, _first_bad(ok))


def check_model(p, item, case, xdt, layout, nt, seed):
    """Random x (values near 1) and bias against the model, bit for bit."""
    s, sd, bn, bk = _scale(case, layout, seed)
    dt = F.XDTYPES[xdt]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(nt, case.inn, generator=g).to(dt)
    bias = torch.randn(case.out, generator=g).to(dt) * 2.0 ** -10
    y = torch.full((nt, case.out), float("nan"), dtype=dt, device="cuda")
    call(p, item, case.dtype, xdt, x.cuda(), sd, bn, bk, y.data_ptr(), case.out, bias=bias.cuda())
    want = F.model(case.floats(), s, bn, bk, x.float().numpy(), case.chunk, xdt, bias=bias.float().numpy())
    ok = same_bits(y.float().cpu(), torch.from_numpy(want))
    assert bool(ok.all()), (case.name, xdt, layout, nt, _first_bad(ok))


@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_shapes_at_every_chunk_size(chunk):
    cases = F.shape_cases(chunk)
    p = raw_plan(cases)   # one plan: items of different shapes and formats in turn
    k0 = F.CHUNKS.index(chunk)
    for i, case in enumerate(cases):
        xdt = ("bf16", "fp16")[(i + k0) % 2]
        layout = LAYOUT_NAMES[(i + k0 // 2) % 4]
        check_one_hot(p, i, case, xdt, layout)
        check_model(p, i, case, ("fp16", "bf16")[(i + k0) % 2], LAYOUT_NAMES[(i + 1) % 4], (1, 3, 8)[i % 3], 100 * k0 + i)
    for it in p.items:
        it.check("after the products")   # (the outputs hold what create decoded: no product wrote them)
    assert p.status() == 0


def test_stream_kinds():
    for j, case in enumerate(F.stream_cases()):
        p = raw_plan([case])
        for xdt in ("bf16", "fp16"):
            check_one_hot(p, 0, case, xdt, LAYOUT_NAMES[(j + (xdt == "fp16")) % 4])
        check_model(p, 0, case, "bf16", LAYOUT_NAMES[(j + 2) % 4], 8, j)
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
                for nt in (1, 3, 8):
                    x = torch.from_numpy(rng.integers(-2, 3, (nt, case.inn)).astype(np.float32)).to(F.XDTYPES[xdt])
                    y = torch.full((nt, case.out), float("nan"), dtype=F.XDTYPES[xdt], device="cuda")
                    call(p, 0, fmt, xdt, x.cuda(), torch.from_numpy(s).cuda(), bn, bk, y.data_ptr(), case.out)
                    want = torch.from_numpy(x.double().numpy() @ wd.T).to(y.dtype)
                    assert torch.equal(y.cpu(), want), (case.name, layout, xdt, nt)


# ------------------------------------------------------------------ the public API on block-quantized weights
def _quantized(fmt, out, inn, seed):
    """bf16 Gaussian weights (std 0.02), quantized per 128x128 block at amax / fp8 max -> (W fp8, scale) on the GPU."""
    g = torch.Generator("cuda").manual_seed(seed)
    w = (torch.randn(out, inn, generator=g, device="cuda") * 0.02).to(torch.bfloat16).float()
    gr, gc = F.grid_shape(out, inn, 128, 128)
    pad = torch.zeros(gr * 128, gc * 128, device="cuda")
    pad[:out, :inn] = w.abs()
    amax = pad.view(gr, 128, gc, 128).amax(dim=(1, 3))
    scale = (amax / float(torch.finfo(F.TORCH[fmt]).max)).clamp_min(2.0 ** -30).contiguous()
    full = scale.repeat_interleave(128, 0)[:out].repeat_interleave(128, 1)[:, :inn]
    return (w / full).to(F.TORCH[fmt]), scale


def _check64(y, x, wq, scale, bias, what, block=(128, 128)):
    """y against fp64 x (S W)^T (+ bias), S the grid of (bn, bk) blocks (a block larger than W is the whole of it)."""
    out, inn = wq.shape
    bn, bk = min(block[0], out), min(block[1], inn)
    s = scale.double().reshape(-(-out // bn), -(-inn // bk))
    wd = wq.double() * s.repeat_interleave(bn, 0)[:out].repeat_interleave(bk, 1)[:, :inn]
    x64 = x.double().reshape(-1, x.shape[-1])
    ref, mag = x64 @ wd.T, x64.abs() @ wd.abs().T
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    bound = (x.shape[-1] + 2) * 2.0 ** -24 * mag
    rel = 2.0 ** -8 if y.dtype == torch.bfloat16 else 2.0 ** -11
    tol = bound + (ref.abs() + bound) * rel + (2.0 ** -25 if y.dtype == torch.float16 else 0)
    err = (y.double().reshape(ref.shape) - ref).abs()
    assert torch.all(err <= tol), (what, float((err - tol).max()))


@pytest.mark.parametrize("fmt", F.FORMATS)
def test_block_quantized_weights_through_the_api(fmt):
    out_f, in_f = 992, 1040   # ragged 128x128 blocks on both edges (and whole 512-byte units in the last chunk)
    wq, scale = _quantized(fmt, out_f, in_f, 3)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    assert plan.matvec_fp8_ok(0, in_f) and not plan.matvec_ok(0, in_f)
    with pytest.raises(ValueError):
        plan.matvec(0, torch.zeros(1, in_f, dtype=torch.bfloat16, device="cuda"))
    need = plan.matvec_fp8_scratch_bytes(0, in_f, 8)
    for xdt in (torch.bfloat16, torch.float16):
        g = torch.Generator("cuda").manual_seed(5)
        for shape in ((in_f,), (3, in_f), (2, 4, in_f)):
            x = torch.randn(shape, generator=g, device="cuda").to(xdt)
            bias = torch.randn(out_f, generator=g, device="cuda").to(xdt) * 0.1
            scratch = torch.full((need,), POISON, dtype=torch.uint8, device="cuda")
            y = plan.matvec_fp8(0, x, scale, block=(128, 128), bias=bias, scratch=scratch)
            assert y.shape == shape[:-1] + (out_f,) and y.dtype == xdt
            _check64(y, x, wq, scale, bias, (fmt, xdt, shape))
            scratch.fill_(POISON)
            again = plan.matvec_fp8(0, x, scale, block=(128, 128), bias=bias, scratch=scratch)
            assert torch.equal(again.view(torch.int16), y.view(torch.int16)), "two calls, same bits"
        # out as a column slice of a wider buffer; x rows that are not 16-byte aligned (copied first)
        x = torch.randn(5, in_f, generator=g, device="cuda").to(xdt)
        wide = torch.full((5, out_f + 24), float("nan"), dtype=xdt, device="cuda")
        view = wide[:, 8: 8 + out_f]
        plan.matvec_fp8(0, x, scale, (128, 128), out=view)
        _check64(view, x, wq, scale, None, (fmt, xdt, "out view"))
        assert torch.all(torch.isnan(wide[:, :8])) and torch.all(torch.isnan(wide[:, 8 + out_f:]))
        xbuf = torch.zeros(5 * in_f + 1, dtype=xdt, device="cuda")
        xm = xbuf[1:].view(5, in_f)
        xm.copy_(x)
        assert xm.data_ptr() % 16
        assert torch.equal(plan.matvec_fp8(0, xm, scale, (128, 128)).view(torch.int16), view.contiguous().view(torch.int16))
    # per tensor (block=None) and per row
    x = torch.randn(4, in_f, device="cuda").to(torch.bfloat16)
    one = torch.tensor([0.001], device="cuda")
    _check64(plan.matvec_fp8(0, x, one), x, wq, torch.full((8, 9), 0.001, device="cuda"), None, "per tensor")
    rows = torch.rand(out_f, device="cuda") * 0.01
    got = plan.matvec_fp8(0, x, rows, block=(1, in_f))
    ref = (x.double() @ wq.double().T) * rows.double()
    assert torch.allclose(got.double(), ref, rtol=2 ** -7, atol=1e-6), "per row"
    plan.check()


def test_graph_capture_replays_with_new_x():
    wq, scale = _quantized("e4m3", 512, 2048, 11)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    x = torch.randn(8, 2048, device="cuda").to(torch.bfloat16)
    y = torch.empty(8, 512, dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(plan.matvec_fp8_scratch_bytes(0, 2048, 8), dtype=torch.uint8, device="cuda")
    plan.matvec_fp8(0, x, scale, (128, 128), out=y, scratch=scratch)   # first call outside: it reads the chunk modes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.matvec_fp8(0, x, scale, (128, 128), out=y, scratch=scratch)
    for r in range(3):
        x.copy_(torch.randn(8, 2048, device="cuda").to(torch.bfloat16))
        scratch.fill_(POISON)
        g.replay()
        torch.cuda.synchronize()
        want = plan.matvec_fp8(0, x, scale, (128, 128))
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), r
        _check64(y, x, wq, scale, None, ("replay", r))


# ------------------------------------------------------------------ multi-item plans
def test_every_item_of_a_multi_item_plan_interleaved_with_runs():
    ws = [_quantized("e4m3", 256, 1024, 1), _quantized("e5m2", 96, 528, 2), _quantized("e4m3", 1, 4096, 3)]
    other = (torch.randn(64, 512, device="cuda") * 0.02).to(torch.bfloat16)
    tensors = [ws[0][0], other, ws[1][0], ws[2][0]]
    streams = [ZipNN(input_format="torch", compression_chunk=ch).compress(t) for t, ch in zip(tensors, (65536, 262144, 131072, 131072))]
    plan = DecodePlan(streams)
    assert not plan.matvec_fp8_ok(1, 512), "a bf16 output"
    for r in range(2):
        for k, (wq, scale) in zip((0, 2, 3), ws):
            x = torch.randn(5, wq.shape[1], device="cuda").to(torch.float16)
            y = plan.matvec_fp8(k, x, scale, (128, 128))
            _check64(y, x, wq, scale, None, (r, k))
            outs = plan.run()
            torch.cuda.synchronize()
            for o, t in zip(outs, tensors):
                assert torch.equal(o.view(torch.uint8), t.view(torch.uint8)), (r, k)
    plan.check()


# ------------------------------------------------------------------ special values
@pytest.mark.parametrize("fmt", F.FORMATS)
def test_special_values(fmt):
    case, at = F.special_case(fmt)
    p = raw_plan([case])
    w = case.weights().double().cuda()
    bad_rows = ~torch.isfinite(w).all(1)
    assert int(bad_rows.sum()) == (2 if fmt == "e4m3" else 5)
    s = np.full((1, 1), 0.25, dtype=np.float32)
    sd = torch.from_numpy(s).cuda()
    for xdt in ("bf16", "fp16"):
        dt = F.XDTYPES[xdt]
        # one-hot over every column: the rows with NaN or infinities give what the dense product gives
        ybuf = torch.full((case.inn, case.out), float("nan"), dtype=dt, device="cuda")
        x = torch.zeros(8, case.inn, dtype=dt, device="cuda")
        for i0 in range(0, case.inn, 8):
            x.zero_()
            x[torch.arange(8), i0 + torch.arange(8)] = 1.0
            call(p, 0, fmt, xdt, x, sd, case.out, case.inn, ybuf[i0].data_ptr(), case.out)
        ref = (torch.eye(case.inn, dtype=torch.float64, device="cuda") @ (w * 0.25).T)   # NaN and inf where fp64 gives them
        want = torch.from_numpy(F.one_hot_model(case.floats(), s, case.out, case.inn, np.arange(case.inn), 0, xdt)).cuda()
        want = torch.where(bad_rows[None, :], ref.float(), want).to(dt)
        ok = same_bits(ybuf.float(), want.float())
        assert bool(ok.all()), (fmt, xdt, _first_bad(ok))
        # random x: NaN exactly where the fp64 product is NaN, the same infinity where it is infinite
        xr = torch.randn(5, case.inn, generator=torch.Generator("cuda").manual_seed(1), device="cuda").to(dt)
        y = torch.zeros(5, case.out, dtype=dt, device="cuda")
        call(p, 0, fmt, xdt, xr, sd, case.out, case.inn, y.data_ptr(), case.out)
        ref = xr.double() @ (w * 0.25).T
        assert torch.equal(torch.isnan(y), torch.isnan(ref)), (fmt, xdt, "NaN")
        inf = torch.isinf(ref)
        assert torch.equal(y.double()[inf], ref[inf]), (fmt, xdt, "inf")
        fin = torch.isfinite(ref)
        assert torch.allclose(y.double()[fin], ref[fin], rtol=2 ** -7, atol=1e-3), (fmt, xdt)


# ------------------------------------------------------------------ rejections
def test_host_rejections_write_nothing(monkeypatch):
    L = _native.lib()
    wq, scale = _quantized("e4m3", 64, 4096, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    need = plan.matvec_fp8_scratch_bytes(0, 4096, 2)
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    x = torch.randn(2, 4096, device="cuda").to(torch.bfloat16)
    y = torch.full((2, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    bad = [("tokens", dict(nt=MATVEC_MAX_TOKENS + 1), A), ("format", dict(fmt=2), A), ("format -1", dict(fmt=-1), A),
           ("x dtype fp32", dict(xdt=2), A), ("x dtype 3", dict(xdt=3), A), ("in 0", dict(inf=0), A),
           ("in not dividing", dict(inf=4112), A), ("item -1", dict(item=-1), A), ("item 1", dict(item=1), A),
           ("null x", dict(x=None), A), ("null y", dict(y=None), A), ("null scratch", dict(scratch=None), A),
           ("null scale", dict(scale=None), A), ("scale alignment", dict(scale=scale.data_ptr() + 2), A),
           ("block rows 0", dict(bn=0), A), ("block cols 0", dict(bk=0), A), ("block cols 8", dict(bk=8), A),
           ("block cols 136 + 4", dict(bk=140), A),
           ("x alignment", dict(x=x.data_ptr() + 2), A), ("x stride", dict(xs=4100), A), ("short x stride", dict(xs=2048), A),
           ("short y stride", dict(ys=32), A), ("y alignment", dict(y=y.data_ptr() + 1), A), ("bias alignment", dict(bias=bias.data_ptr() + 1), A),
           ("scratch alignment", dict(scratch=scratch.data_ptr() + 16), A), ("short scratch", dict(sb=need - 1), A),
           ("rows of 8 bytes", dict(inf=8), U)]
    for name, kw, want in bad:
        a = dict(item=0, fmt=0, xdt=0, inf=4096, x=x.data_ptr(), xs=4096, nt=2, scale=scale.data_ptr(), bn=128, bk=128,
                 bias=bias.data_ptr(), y=y.data_ptr(), ys=64, scratch=scratch.data_ptr(), sb=need)
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_matvec_fp8(plan._ref, a["item"], a["fmt"], a["xdt"], a["inf"], a["x"], a["xs"], a["nt"], a["scale"],
                                                 a["bn"], a["bk"], a["bias"], a["y"], a["ys"], a["scratch"], a["sb"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    assert torch.all(torch.isnan(y))
    out = C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_matvec_fp8_scratch_size(plan._ref, 0, 4096, MATVEC_MAX_TOKENS + 1, C.byref(out)) == A
    assert L.zipnn_b200_decode_plan_matvec_fp8_scratch_size(plan._ref, 0, 4096, 2, None) == A
    # the 16-bit entry points still refuse fp8 items, and the fp8 one refuses 16-bit items
    assert L.zipnn_b200_decode_plan_matvec(plan._ref, 0, 0, 4096, x.data_ptr(), 4096, 2, None, y.data_ptr(), 64, scratch.data_ptr(),
                                           need, _st()) == U
    assert not plan.matvec_ok(0, 4096)
    other = DecodePlan([ZipNN(input_format="torch").compress((torch.randn(64, 4096, device="cuda") * 0.02).to(torch.bfloat16))])
    assert not other.matvec_fp8_ok(0, 4096)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matvec_fp8(other._ref, 0, 0, 0, 4096, x.data_ptr(), 4096, 2, scale.data_ptr(), 128, 128, None,
                                               y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
    # Python-side refusals
    for kw, what in ((dict(block=None), "a grid scale without block"), (dict(block=(128, 8)), "bk 8"), (dict(block=(0, 128)), "bn 0"),
                     (dict(block=(32, 128)), "a grid of another block"), (dict(scale=scale.double()), "fp64 scale"),
                     (dict(scale=torch.ones(64, device="cuda")[::2]), "a non-contiguous scale"), (dict(x=x.float()), "fp32 x")):
        a = dict(x=x, scale=scale, block=(128, 128))
        a.update(kw)
        with pytest.raises(ValueError):
            plan.matvec_fp8(0, a["x"], a["scale"], block=a["block"])
    assert _native.launch_count() == before and torch.all(torch.isnan(y))
    # a plain (incompressible) fp8 item, a box, and a plan without a segment index
    raw = torch.randint(0, 256, (64 * 4096,), dtype=torch.uint8, device="cuda")
    raw[(raw & 0x7F) == 0x7F] = 0
    pl = DecodePlan([ZipNN(input_format="torch").compress(raw.view(torch.float8_e4m3fn).view(64, 4096))])
    assert not pl.matvec_fp8_ok(0, 4096)
    case = F.shape_cases(4096)[0]
    boxed = DP.Plan([DP.Item(case.name, case.body, 1, case.bits, case.chunk, case.data.size, case.data[:4096 * 2],
                             box=(0, 2, 8192, 4096))])
    assert boxed.rc == 0
    for p_ref in (pl._ref, C.byref(boxed.plan)):
        before = _native.launch_count()
        assert L.zipnn_b200_decode_plan_matvec_fp8_scratch_size(p_ref, 0, 16, 1, C.byref(C.c_size_t(0))) == U
        assert L.zipnn_b200_decode_plan_matvec_fp8(p_ref, 0, 0, 0, 16, x.data_ptr(), 16, 1, scale.data_ptr(), 1, 16, None,
                                                   y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
        assert _native.launch_count() == before
    DP._set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    q = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    before = _native.launch_count()
    assert not q.matvec_fp8_ok(0, 4096)
    assert L.zipnn_b200_decode_plan_matvec_fp8(q._ref, 0, 0, 0, 4096, x.data_ptr(), 4096, 2, scale.data_ptr(), 128, 128, None,
                                               y.data_ptr(), 64, scratch.data_ptr(), need, _st()) == U
    assert _native.launch_count() == before and torch.all(torch.isnan(y))


# ------------------------------------------------------------------ corrupted streams
def test_corrupted_fp8_streams_follow_the_model():
    """Every mutant of the fp8 base of corrupt_streams.py (verdicts held to tests/golden/corrupt_verdicts.json by
    test_corrupt_streams_host.py): a plan whose create fails is refused by the fp8 matvec (E_ARG, nothing launched),
    as by every other entry point; one that creates decodes to the verdict's bytes and is refused (E_UNSUPPORTED: its
    elements, 8 times an odd number, leave no rows of a multiple of 16 bytes, and its last chunk is not fused)."""
    import test_corrupt_streams_gpu as T
    b = CS.bases()["fp8_g1"]
    assert b.pr["mode"][-1] != "fused"
    L = _native.lib()
    x = torch.zeros(1, 16, dtype=torch.bfloat16, device="cuda")
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
        got = L.zipnn_b200_decode_plan_matvec_fp8(p, 0, 0, 0, 8, x.data_ptr(), 8, 1, sc.data_ptr(), 1, 16, None, y.data_ptr(), 1,
                                                  small.data_ptr(), small.numel(), _st())
        assert got == (_native.E_ARG if rc else _native.E_UNSUPPORTED), (m.id, got)
        assert _native.launch_count() == before, m.id
        if not rc:
            assert torch.equal(out[T.PAD: T.PAD + b.orig], torch.from_numpy(v.data).cuda()), m.id
            n += 1
    assert torch.all(torch.isnan(y))
    assert n > 0
