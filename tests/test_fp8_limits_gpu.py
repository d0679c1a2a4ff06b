"""The five fp8 entry points (matvec_fp8, matmul_fp8, dequant_fp8, dequant_fp8_select, experts_matvec_fp8) at their
largest item, at the first item they refuse, at real checkpoint shapes and on scale grids at their edges
(tests/fp8_limits.py holds the inventory; test_fp8_limits_host.py checks it without a GPU).

  * the main oracle: integer weights, x in {-1, 0, 1}, a random power of two per scale block, so every result is the
    fp64 product rounded once to x's dtype, compared bit for bit; the dequantizes bit for bit against torch's
    (W.float() * S_expanded).to(dtype), in row slabs;
  * the largest item, [8, 16383, 16384] e4m3fn at 128 KiB chunks (2^31 - 2^17 elements): every column through the
    matmul by one-hot x, exact sums at 1 to 64 rows, the selected dequantize and the experts matvec on the first and last
    experts, x rows 2^26 elements apart;
  * the first item refused, [8, 16384, 16384] (two pieces): every call refuses it, launches nothing and writes nothing,
    and the plan still decodes it;
  * DeepSeek-V3, Llama-3.1-405B and Qwen3-235B-A22B layer shapes, exact and Gaussian (within the fp64 bound);
  * blocks from (1, 16) to (2^40, 2^40) on one tensor per format.

Every test's peak reserved device memory stays under fp8_limits.CEILING (16 GiB), and is printed.
"""
import numpy as np
import pytest
import torch

import fp8_limits as L
import fp8_streams as F
from test_dequant_fp8_gpu import _quantized, torch_dequant
from test_experts_matvec_fp8_gpu import oracle
from test_fp8_experts_gpu import _experts_weight
from test_matmul_fp8_gpu import check64 as check64_d
from test_matvec_fp8_gpu import _check64
from test_product_streams_gpu import POISON, SCRATCH, _st, same_bits
from zipnn_b200 import DecodePlan, ZipNN, _native

pytestmark = pytest.mark.gpu

XDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
SLAB = 1 << 27   # elements of a row slab of the fp64 references


@pytest.fixture(autouse=True)
def device_memory_budget():
    """Every test here stays under fp8_limits.CEILING of reserved device memory at its peak, counted from what was
    reserved when it started (a failed test before it may still hold its tensors through its traceback)."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_reserved()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_reserved() - base
    torch.cuda.empty_cache()
    print(f"peak reserved device memory {peak / 2 ** 30:.2f} GiB")
    assert peak <= L.CEILING, f"the test reserved {peak / 2 ** 30:.2f} GiB of device memory at its peak"


def _room(need):
    """test_product_streams_gpu._big_room's pattern: skip when the shared device has less free memory than the test needs."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{free / 2 ** 30:.1f} GiB of device memory free, {need / 2 ** 30:.1f} GiB needed")


def bits(t):
    return t.view(torch.int16)


def slabs(rows, inn, bn):
    """Row slabs of at most about SLAB elements, each starting on a block row: (r0, r1, first and end block rows)."""
    step = max(bn, (max(1, SLAB // inn) // bn) * bn)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        yield r0, r1, r0 // bn, -(-r1 // bn)


def ref64(x, w, s, block):
    """fp64 x @ (W S)^T [n, rows] for W [rows, in] fp8 and S its grid of (bn, bk) blocks, in row slabs."""
    rows, inn = w.shape
    bn, bk = min(block[0], rows), min(block[1], inn)
    s = s.reshape(-(-rows // bn), -(-inn // bk))
    x64 = x.double()
    out = torch.empty(x.shape[0], rows, dtype=torch.float64, device="cuda")
    for r0, r1, g0, g1 in slabs(rows, inn, bn):
        e = s[g0:g1].double().repeat_interleave(bn, 0)[: r1 - r0].repeat_interleave(bk, 1)[:, :inn]
        out[:, r0:r1] = x64 @ (w[r0:r1].double() * e).T
    return out


def check_dequant(d, w, s, block, what):
    """d (the kernel's dequantize of W [rows, in]) bit for bit torch_dequant, in row slabs."""
    rows, inn = w.shape
    bn, bk = min(block[0], rows), min(block[1], inn)
    s = s.reshape(-(-rows // bn), -(-inn // bk))
    for r0, r1, g0, g1 in slabs(rows, inn, bn):
        assert torch.equal(bits(d[r0:r1]), bits(torch_dequant(w[r0:r1], s[g0:g1], (bn, bk), d.dtype))), (what, r0)


def signs(shape, seed):
    return torch.from_numpy(L.signs(shape, seed)).cuda()


def pow2(shape, seed):
    return torch.from_numpy(L.pow2_scales(shape, seed)).cuda()


def check_dense_exact(plan, k, w, s, block, what, mv_rows=L.DENSE_MATVEC_ROWS, mm_rows=L.DENSE_MATMUL_ROWS, seed=0):
    """matvec_fp8 and matmul_fp8 at every row count, both x dtypes, and dequant_fp8 in one dtype, on exact inputs."""
    rows, inn = w.shape
    x = signs((max(mv_rows + mm_rows), inn), seed)
    ref = ref64(x, w, s, block)
    for j, (xn, dt) in enumerate(XDT.items()):
        xd = x.to(dt)
        for n in mv_rows:
            y = plan.matvec_fp8(k, xd[:n], s, block)
            assert torch.equal(bits(y), bits(ref[:n].to(dt))), (what, "matvec_fp8", xn, n)
        for n in mm_rows:
            y = plan.matmul_fp8(k, xd[:n], s, block)
            assert torch.equal(bits(y), bits(ref[:n].to(dt))), (what, "matmul_fp8", xn, n)
    dt = XDT[("bf16", "fp16")[seed % 2]]
    check_dequant(plan.dequant_fp8(k, inn, s, block, dtype=dt), w, s, block, what)


def expert_refs(x, w, s, block, ids, per_pair):
    """fp64 y [T, k, so] of the exact experts call: each routed expert's slice times its pairs' x rows."""
    T, top_k = ids.shape
    so = w.shape[1]
    ref = torch.empty(T, top_k, so, dtype=torch.float64, device="cuda")
    idl = ids.tolist()
    for e in sorted({e for r in idl for e in r}):
        pairs = [(t, j) for t in range(T) for j in range(top_k) if idl[t][j] == e]
        xs = torch.stack([x[t, j] if per_pair else x[t] for t, j in pairs])
        r = ref64(xs, w[e], s[e], block)
        for i, (t, j) in enumerate(pairs):
            ref[t, j] = r[i]
    return ref


def check_select(plan, ids, w, s, block, dt, what):
    """dequant_fp8_select of one output: the routed slices bit for bit torch's; every other slice NaN (the fill) except
    in the chunks of the routed slices that straddle into it, which are correct there too."""
    E, so, inn = w.shape
    out = torch.full((E, so, inn), float("nan"), dtype=dt, device="cuda")
    plan.dequant_fp8_select(ids, [inn], [s], [block], dtype=dt, outs=[out])
    routed = sorted(set(ids.reshape(-1).tolist()))
    for e in routed:
        check_dequant(out[e], w[e], s[e], block, (what, e))
    bn, bk = min(block[0], so), min(block[1], inn)
    per = so * inn
    written = [((e * per) // L.CHUNK * L.CHUNK, -(-((e + 1) * per) // L.CHUNK) * L.CHUNK) for e in routed]
    flat = out.view(-1)
    for e in set(range(E)) - set(routed):
        lo, hi = e * per, (e + 1) * per
        keep = torch.ones(per, dtype=torch.bool, device="cuda")
        sg = s[e].reshape(-(-so // bn), -(-inn // bk))
        for a, b in written:
            a, b = max(a, lo), min(b, hi)
            if a < b:   # a chunk of a routed slice that straddles into this one: written, and correct
                keep[a - lo: b - lo] = False
                r0, r1 = (a - lo) // inn // bn * bn, -(-(b - lo) // inn)
                want = torch_dequant(w[e, r0:r1], sg[r0 // bn: -(-r1 // bn)], (bn, bk), dt).reshape(-1)
                base = lo + r0 * inn
                assert torch.equal(bits(flat[a:b]), bits(want[a - base: b - base])), (what, e, "straddle")
        assert bool(torch.isnan(flat[lo:hi][keep]).all()), (what, e, "an unrouted slice was written")
    return out


def _exact_plan(fmt, shape, seed):
    w = L.integer_weights(fmt, shape, seed)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    plan.release_out()
    return w, plan


# ------------------------------------------------------------------ 2. the largest item
def test_largest_item():
    """[8, 16383, 16384] e4m3fn, 16383 chunks of 128 KiB: element indices up to 2^31 - 2^17 - 1, expert boundaries
    inside chunks, the last 128-row block of each expert ragged."""
    _room(L.memory("largest"))
    E, so, inn = L.LARGEST
    rows = E * so
    w, plan = _exact_plan("e4m3", L.LARGEST, 1)
    w2 = w.view(rows, inn)
    ok = dict(matvec=plan.matvec_fp8_ok(0, inn), matmul=plan.matmul_fp8_ok(0, inn), dequant=plan.matvec_fp8_ok(0, inn),
              select=plan.dequant_fp8_select_ok([inn]), experts=plan.experts_matvec_fp8_ok(0, inn))
    assert all(ok.values()), ok
    blk = (128, 128)
    sd = pow2((-(-rows // 128), inn // 128), 2)            # the dense view [rows, in]
    se = pow2((E, -(-so // 128), inn // 128), 3)           # one grid per expert
    # matmul_fp8: every column once, 64 per call, against the one-hot model (the last rows sit within 2^17 of 2^31)
    x = torch.zeros(64, inn, dtype=torch.bfloat16, device="cuda")
    y = torch.empty(64, rows, dtype=torch.bfloat16, device="cuda")
    ar = torch.arange(64, device="cuda")
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    scratch = SCRATCH.get(plan.matmul_fp8_scratch_bytes(0, inn, 64))
    for i0 in range(0, inn, 64):
        x.zero_()
        x.view(-1).index_fill_(0, ar * (inn + 1) + i0, 1.0)
        scratch.fill_(POISON)
        plan.matmul_fp8(0, x, sd, blk, out=y, scratch=scratch)
        bad += (~same_bits(y, L.one_hot_torch(w2, sd, 128, 128, ar + i0, 0, torch.bfloat16))).sum()
    # matvec_fp8: one-hot at the first and last 8 columns (fp16)
    for i0 in (0, inn - 8):
        x.zero_()
        x.view(-1).index_fill_(0, ar[:8] * (inn + 1) + i0, 1.0)
        got = plan.matvec_fp8(0, x[:8].half(), sd, blk)
        bad += (~same_bits(got, L.one_hot_torch(w2, sd, 128, 128, ar[:8] + i0, 0, torch.float16))).sum()
    assert int(bad) == 0, int(bad)
    del x, y
    # exact sums: matvec at 1 and 8 rows, matmul at 9, 33 and 64; dequant_fp8 of the whole item, compared in row slabs
    check_dense_exact(plan, 0, w2, sd, blk, "largest", mv_rows=(1, 8), mm_rows=(9, 33, 64), seed=4)
    torch.cuda.empty_cache()
    # dequant_fp8_select with ids {7}, then {0, 7}
    for ids in L.LARGEST_IDS:
        check_select(plan, torch.tensor(ids, device="cuda"), w, se, blk, torch.bfloat16, ("select", ids))
        torch.cuda.empty_cache()
    # experts_matvec_fp8: T = 1 and 4, x per token and per pair; then x rows 2^26 elements apart (offsets past 2^27)
    for r, route in enumerate(L.LARGEST_ROUTES):
        ids = torch.tensor(route, device="cuda")
        T, k = ids.shape
        for per_pair in (False, True):
            x = signs((T, k, inn) if per_pair else (T, inn), 10 + 2 * r + per_pair)
            dt = XDT[("bf16", "fp16")[(r + per_pair) % 2]]
            got = plan.experts_matvec_fp8(0, ids, x.to(dt), se, blk)
            assert torch.equal(bits(got), bits(expert_refs(x, w, se, blk, ids, per_pair).to(dt))), (route, per_pair)
    ids = torch.tensor(L.LARGEST_ROUTES[1], device="cuda")
    T = ids.shape[0]
    buf = torch.zeros((T - 1) * L.BIG_X_STRIDE + inn, dtype=torch.bfloat16, device="cuda")
    xb = buf.as_strided((T, inn), (L.BIG_X_STRIDE, 1))
    x = signs((T, inn), 20)
    xb.copy_(x)
    got = plan.experts_matvec_fp8(0, ids, xb, se, blk)
    assert torch.equal(bits(got), bits(expert_refs(x, w, se, blk, ids, False).to(torch.bfloat16))), "x stride 2^26"
    plan.check()


def test_first_item_refused():
    """[8, 16384, 16384]: 2^31 elements, 16384 chunks, two pieces.  Every call refuses it (E_UNSUPPORTED), launches
    nothing and writes nothing, and a run still decodes it."""
    _room(L.memory("refused"))
    E, so, inn = L.REFUSED
    w = L.integer_weights("e5m2", L.REFUSED, 5)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    assert not plan.matvec_fp8_ok(0, inn) and not plan.matmul_fp8_ok(0, inn)
    assert not plan.dequant_fp8_select_ok([inn]) and not plan.experts_matvec_fp8_ok(0, inn)
    with pytest.raises(ValueError):
        plan.dequant_fp8(0, inn, torch.ones(1, device="cuda"))
    Lb = _native.lib()
    U, fmt = _native.E_UNSUPPORTED, F.CODE["e5m2"]
    x = torch.zeros(2, inn, dtype=torch.bfloat16, device="cuda")
    y = torch.full((2, 2, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    out = torch.full((4096,), float("nan"), dtype=torch.bfloat16, device="cuda")
    s = torch.ones(E * 128 * 128, device="cuda")
    ids = torch.tensor([[0, 7], [7, 1]], device="cuda")
    scratch = SCRATCH.get(64 << 20)
    item = (_native.Fp8SelectItem * 1)()
    item[0].in_features, item[0].d_scale, item[0].block_rows, item[0].block_cols, item[0].d_out = inn, s.data_ptr(), 128, 128, out.data_ptr()
    calls = {
        "matvec_fp8": lambda: Lb.zipnn_b200_decode_plan_matvec_fp8(plan._ref, 0, fmt, 0, inn, x.data_ptr(), inn, 2, s.data_ptr(), 128, 128,
                                                                   None, y.data_ptr(), 64, scratch.data_ptr(), scratch.numel(), _st()),
        "matmul_fp8": lambda: Lb.zipnn_b200_decode_plan_matmul_fp8(plan._ref, 0, fmt, 0, inn, x.data_ptr(), inn, 2, s.data_ptr(), 128, 128,
                                                                   None, y.data_ptr(), 64, scratch.data_ptr(), scratch.numel(), _st()),
        "dequant_fp8": lambda: Lb.zipnn_b200_decode_plan_dequant_fp8(plan._ref, 0, fmt, 0, inn, s.data_ptr(), 128, 128, out.data_ptr(), _st()),
        "dequant_fp8_select": lambda: Lb.zipnn_b200_decode_plan_dequant_fp8_select(plan._ref, E, ids.data_ptr(), 4, 8, fmt, 0, 1, item,
                                                                                   scratch.data_ptr(), scratch.numel(), _st()),
        "experts_matvec_fp8": lambda: Lb.zipnn_b200_decode_plan_experts_matvec_fp8(
            plan._ref, 0, E, ids.data_ptr(), 4, 8, 2, fmt, 0, inn, x.data_ptr(), inn, 0, s.data_ptr(), 128, 128, y.data_ptr(), 64,
            scratch.data_ptr(), scratch.numel(), _st()),
    }
    for name, call in calls.items():
        before = _native.launch_count()
        assert call() == U and _native.launch_count() == before, name
    torch.cuda.synchronize()
    assert torch.all(torch.isnan(y)) and torch.all(torch.isnan(out))
    got = plan.run()[0]
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.uint8), w.view(torch.uint8))
    plan.check()


# ------------------------------------------------------------------ 3. real checkpoint shapes
def _gaussian(fmt, shape, block, seed):
    """Gaussian weights quantized per block (test_dequant_fp8_gpu._quantized), built in row slabs of whole blocks."""
    rows, inn = shape
    step = max(block[0], (max(1, (1 << 26) // inn) // block[0]) * block[0])
    ws, ss = zip(*[_quantized(fmt, min(step, rows - r0), inn, seed + i, block) for i, r0 in enumerate(range(0, rows, step))])
    return torch.cat(ws), torch.cat([s.reshape(-1, s.shape[-1]) for s in ss])


@pytest.mark.parametrize("name,fmt,shape,block", [s for s in L.real_shapes() if len(s[2]) == 2], ids=lambda v: v if isinstance(v, str) else None)
def test_real_dense_shape(name, fmt, shape, block):
    _room(L.memory("real", shape))
    rows, inn = shape
    w, plan = _exact_plan(fmt, shape, 30)
    assert plan.matvec_fp8_ok(0, inn) and plan.matmul_fp8_ok(0, inn), name
    s = pow2(L.grid(rows, inn, *block), 31)
    check_dense_exact(plan, 0, w, s, block, name, seed=32)
    del w, plan
    torch.cuda.empty_cache()
    # Gaussian weights quantized per block, within the fp64 bound
    wq, sg = _gaussian(fmt, shape, block, 40)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    plan.release_out()
    assert plan.matvec_fp8_ok(0, inn), name
    x = torch.randn(8, inn, device="cuda").to(torch.bfloat16)
    y = plan.matvec_fp8(0, x, sg, block)
    for r0, r1, g0, g1 in slabs(rows, inn, block[0]):
        _check64(y[:, r0:r1], x, wq[r0:r1], sg[g0:g1], None, (name, r0), block=block)
    y = plan.matmul_fp8(0, x.half(), sg, block)
    for r0, r1, g0, g1 in slabs(rows, inn, block[0]):
        check64_d(y[:, r0:r1], x.half(), torch_dequant(wq[r0:r1], sg[g0:g1], block, torch.float16), None, (name, "matmul", r0))


@pytest.mark.parametrize("name,fmt,shape,block", [s for s in L.real_shapes() if len(s[2]) == 3], ids=lambda v: v if isinstance(v, str) else None)
def test_real_experts_shape(name, fmt, shape, block):
    """Top-8 routing at T = 1 to 4, x per token for gate_up and per pair for down; the selected dequantize of the same
    ids; per-pair matvec_fp8 as a second oracle at T = 1."""
    _room(L.memory("real", shape))
    E, so, inn = shape
    per_pair = "down" in name
    w, plan = _exact_plan(fmt, shape, 50)
    assert plan.experts_matvec_fp8_ok(0, inn) and plan.dequant_fp8_select_ok([inn]), name
    s = pow2((E,) + L.grid(so, inn, *block), 51)
    rng = np.random.default_rng(52)
    for T in range(1, 5):
        ids = torch.from_numpy(np.stack([rng.permutation(E)[:L.TOP_K] for _ in range(T)])).cuda()
        x = signs((T, L.TOP_K, inn) if per_pair else (T, inn), 53 + T)
        dt = XDT[("bf16", "fp16")[T % 2]]
        got = plan.experts_matvec_fp8(0, ids, x.to(dt), s, block)
        assert torch.equal(bits(got), bits(expert_refs(x, w, s, block, ids, per_pair).to(dt))), (name, T)
        if T == 1:
            assert torch.equal(bits(got), bits(oracle(plan, 0, ids, x.to(dt), s, so, *block))), (name, "per-pair matvec_fp8")
    check_select(plan, ids, w, s, block, torch.bfloat16, name)
    del w, plan
    torch.cuda.empty_cache()
    # Gaussian experts quantized per block, within the fp64 bound
    wq, sg = _experts_weight(fmt, E, so, inn, 60, block)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    plan.release_out()
    ids = torch.from_numpy(np.stack([rng.permutation(E)[:L.TOP_K] for _ in range(4)])).cuda()
    x = torch.randn((4, L.TOP_K, inn) if per_pair else (4, inn), device="cuda").to(torch.bfloat16)
    y = plan.experts_matvec_fp8(0, ids, x, sg, block)
    for t in range(4):
        for j in range(L.TOP_K):
            e = int(ids[t, j])
            _check64(y[t, j], (x[t, j] if per_pair else x[t])[None], wq[e], sg[e], None, (name, t, j), block=block)


# ------------------------------------------------------------------ 4. scale grids at their edges
@pytest.mark.parametrize("fmt", F.FORMATS)
def test_scale_grid_edges(fmt):
    """One tensor [3, 1000, 1216]: the dense calls see [3000, 1216], the selected ones 3 experts of 1000 rows; every
    block of fp8_limits.edge_blocks, blocks larger than the matrix a one-element grid."""
    _room(L.memory("edges"))
    E, so, inn = L.EDGE_SHAPE
    rows = E * so
    w = L.integer_weights(fmt, L.EDGE_SHAPE, 70 + F.CODE[fmt])
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    ok = dict(matvec=plan.matvec_fp8_ok(0, inn), matmul=plan.matmul_fp8_ok(0, inn), select=plan.dequant_fp8_select_ok([inn]),
              experts=plan.experts_matvec_fp8_ok(0, inn))
    assert all(ok.values()), ok
    w2 = w.view(rows, inn)
    for i, block in enumerate(L.edge_blocks(rows, inn)):
        s = pow2(L.grid(rows, inn, *block), 80 + i)
        check_dense_exact(plan, 0, w2, s, block, (fmt, "dense", block), mv_rows=(1, 5), mm_rows=(17,), seed=i)
    ids = torch.tensor([[2, 0], [1, 2]], device="cuda")
    for i, block in enumerate(L.edge_blocks(so, inn)):
        s = pow2((E,) + L.grid(so, inn, *block), 90 + i)
        for per_pair in (False, True):
            x = signs((2, 2, inn) if per_pair else (2, inn), 100 + i)
            dt = XDT[("bf16", "fp16")[(i + per_pair) % 2]]
            got = plan.experts_matvec_fp8(0, ids, x.to(dt), s, block)
            assert torch.equal(bits(got), bits(expert_refs(x, w, s, block, ids, per_pair).to(dt))), (fmt, block, per_pair)
        check_select(plan, ids[:1, :1], w, s, block, XDT[("bf16", "fp16")[i % 2]], (fmt, "select", block))
    outs = plan.run()
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.uint8), w.view(torch.uint8))
    plan.check()


# ------------------------------------------------------------------ 5. the experts x-offset guard
def test_experts_x_offset_guard_launches_nothing():
    """x row offsets are 32-bit: xrows * max(x_stride, in) past UINT32_MAX is E_ARG, before anything runs."""
    E, so, inn = 4, 64, 1024
    wq, s = _experts_weight("e4m3", E, so, inn, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    ids = torch.tensor([[0, 1], [2, 3]], device="cuda")
    x = torch.zeros(2, inn, dtype=torch.bfloat16, device="cuda")
    y = torch.full((2, 2, so), float("nan"), dtype=torch.bfloat16, device="cuda")
    need = plan.experts_matvec_fp8_scratch_bytes(0, inn, 2, 2)
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    for xrows, per_pair in ((2, 0), (4, 1)):
        stride = (L.UINT32_MAX // xrows) // 8 * 8 + 8
        assert not L.x_offsets_fit(xrows, stride, inn) and L.x_offsets_fit(xrows, stride - 8, inn)
        before = _native.launch_count()
        rc = _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8(
            plan._ref, 0, E, ids.data_ptr(), 4, 8, 2, F.CODE["e4m3"], 0, inn, x.data_ptr(), stride, per_pair, s.data_ptr(), 128, 128,
            y.data_ptr(), so, scratch.data_ptr(), need, _st())
        assert rc == _native.E_ARG and _native.launch_count() == before, (xrows, rc)
    torch.cuda.synchronize()
    assert torch.all(torch.isnan(y))
    plan.check()
