"""The selected experts matvec (zipnn_b200_decode_plan_experts_matvec_fp8, DecodePlan.experts_matvec_fp8) on an H100.

The oracle is matvec_fp8, tested on its own: for every pair p = (t, j) of ids [T, k], y[p] must equal, bit for bit, the
rows of expert ids[p] of matvec_fp8 on the same output seen as [E * out, in], with x = the pair's x row and the scale
expanded to one row per weight row ([E * out, ceil(in / bk)] with block (1, bk): every element gets the same fp32
scale, so ragged grids and one scale per expert are covered too).  The fp8 corpus of tests/fp8_streams.py at every
chunk size (both formats, special values included), bf16 and fp16 x, T = 1 to 4, k in {1, 2, 8}, x per token and per
pair, routings where tokens share experts; a Qwen3-30B-A3B-FP8-sized layer; five launches whatever the ids and none
for n = 0; bad ids; host rejections; graph replay; interleaving with the plan's other calls on one scratch.

Modules: transformers' tiny fp8 Qwen3-MoE and Mixtral under compress_module / load_module with fp8=True, experts=True,
experts_matvec=4: at up to 4 tokens each experts module's output is bit for bit the composition (gate, combine) of
per-pair matvec_fp8 calls; above, the model is bit for bit the one without experts_matvec.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import fp8_streams as F
from safetensors.torch import save_file
from test_fp8_experts_gpu import _experts_weight, dense_state, experts_of, layouts, raw, tiny_fp8_moe
from test_product_streams_gpu import _st, raw_plan
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200 import resident as R
from zipnn_b200.plan import EXPERTS_MATVEC_MAX_TOKENS

pytestmark = pytest.mark.gpu

LAUNCHES = 5   # index, pair tables, product, reduce, error pass
XDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
XNAME = {v: k for k, v in XDT.items()}


def expanded_rows(s: torch.Tensor, so: int, bn: int) -> torch.Tensor:
    """Per-expert grids [E, gr, gc] -> one scale row per weight row [E * so, gc] (the oracle's grid, block (1, bk))."""
    E = s.shape[0]
    return s.reshape(E, -1, s.shape[-1]).repeat_interleave(bn, dim=1)[:, :so].reshape(E * so, -1).contiguous()


def oracle(plan, k, ids, x, s, so, bn, bk):
    """y [T, top_k, so] from per-pair matvec_fp8 calls on output k seen as [E * so, in]."""
    T, top_k = ids.shape
    flat = expanded_rows(s, so, bn)
    out = torch.empty(T, top_k, so, dtype=x.dtype, device="cuda")
    for t in range(T):
        for j in range(top_k):
            e = int(ids[t, j])
            xr = x[t, j] if x.dim() == 3 else x[t]
            out[t, j] = plan.matvec_fp8(k, xr[None], flat, (1, bk))[0, e * so:(e + 1) * so]
    return out


def routing(E, T, k, rng, shared):
    """[T, k] distinct experts per token; `shared`: drawn from a pool of k + 1 experts, so tokens share most of them."""
    pool = rng.permutation(E)[:min(E, k + 1)] if shared else np.arange(E)
    return np.stack([rng.permutation(pool)[:k] for _ in range(T)])


def bits(t):
    return t.view(torch.int16)


def raw_experts(p, case, E, ids, x, s, bn, bk):
    """zipnn_b200_decode_plan_experts_matvec_fp8 on the corpus plan's item: -> y [T, k, so]; asserts five launches."""
    T, k = ids.shape
    so, inn = case.out // E, case.inn
    per_pair = x.dim() == 3
    need = C.c_size_t(0)
    assert _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size(C.byref(p.plan), 0, E, inn, T * k, k, C.byref(need)) == 0
    scratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    y = torch.full((T, k, so), float("nan"), dtype=x.dtype, device="cuda")
    before = _native.launch_count()
    rc = _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8(
        C.byref(p.plan), 0, E, ids.data_ptr(), T * k, ids.element_size(), k, F.CODE[case.dtype], F.XCODE[XNAME[x.dtype]], inn,
        x.data_ptr(), inn, int(per_pair), s.data_ptr(), bn, bk, y.data_ptr(), so, scratch.data_ptr(), need.value, _st())
    assert rc == 0 and _native.launch_count() - before == LAUNCHES, (case.name, rc)
    return y


def raw_oracle(p, case, E, ids, x, s, bn, bk):
    """Per-pair zipnn_b200_decode_plan_matvec_fp8 on the item seen as [E * so, in] with one scale row per weight row."""
    T, k = ids.shape
    so, inn = case.out // E, case.inn
    flat = expanded_rows(s, so, bn)
    need = C.c_size_t(0)
    assert _native.lib().zipnn_b200_decode_plan_matvec_fp8_scratch_size(C.byref(p.plan), 0, inn, 1, C.byref(need)) == 0
    scratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    y = torch.empty(case.out, dtype=x.dtype, device="cuda")
    out = torch.empty(T, k, so, dtype=x.dtype, device="cuda")
    for t in range(T):
        for j in range(k):
            xr = (x[t, j] if x.dim() == 3 else x[t]).contiguous()
            assert _native.lib().zipnn_b200_decode_plan_matvec_fp8(
                C.byref(p.plan), 0, F.CODE[case.dtype], F.XCODE[XNAME[x.dtype]], inn, xr.data_ptr(), inn, 1, flat.data_ptr(), 1, bk,
                None, y.data_ptr(), case.out, scratch.data_ptr(), need.value, _st()) == 0
            e = int(ids[t, j])
            out[t, j] = y[e * so:(e + 1) * so]
    return out


def check_case(case, seed):
    """The corpus case's own stream (raw_plan) seen as E experts, every k, T, both x dtypes and x layouts."""
    p = raw_plan([case])
    E = experts_of(case.out)
    so, inn = case.out // E, case.inn
    rng = np.random.default_rng(seed)
    names = list(layouts(so, inn))
    bn, bk = layouts(so, inn)[names[seed % len(names)]]
    s = torch.from_numpy(np.stack([F.random_scales(so, inn, bn, bk, seed + e) for e in range(E)])).cuda()
    for m, k in enumerate(kk for kk in (1, 2, 8) if kk <= E):
        for T in range(1, EXPERTS_MATVEC_MAX_TOKENS + 1):
            xdt = ("bf16", "fp16")[(T + m + seed) % 2]
            ids = torch.from_numpy(routing(E, T, k, rng, (T + m) % 2 == 0)).cuda()
            if T % 2:
                ids = ids.to(torch.int32)
            per_pair = (T + m) % 3 == 1
            x = torch.randn((T, k, inn) if per_pair else (T, inn), device="cuda").to(XDT[xdt])
            got = raw_experts(p, case, E, ids, x, s, bn, bk)
            want = raw_oracle(p, case, E, ids, x, s, bn, bk)
            assert torch.equal(bits(got), bits(want)), (case.name, k, T, xdt, per_pair, (bn, bk))
    assert p.status() == 0


@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_corpus_bit_for_bit_against_matvec_fp8(chunk):
    for i, case in enumerate(F.shape_cases(chunk)):
        check_case(case, 10 * F.CHUNKS.index(chunk) + i)


def test_stream_kinds_and_special_values():
    cases = F.stream_cases() + [F.special_case(f)[0] for f in F.FORMATS]
    for i, case in enumerate(cases):
        check_case(case, 500 + i)


def test_one_hot_x_gives_the_weights():
    """x = 2^3 e_col per token: y[p][o] = round(W[e][o][col] 2^3 * S[e][o / bn][col / bk]), fp8_streams.one_hot_model."""
    case = F.shape_cases(4096)[2]   # in144
    E = experts_of(case.out)
    wt = torch.from_numpy(case.data).view(F.TORCH[case.dtype]).reshape(E, case.out // E, case.inn)
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=4096).compress(wt.cuda())])
    so, inn = case.out // E, case.inn
    bn, bk = 5, 16
    s = np.stack([F.random_scales(so, inn, bn, bk, 7 + e) for e in range(E)])
    w = torch.from_numpy(case.data).view(F.TORCH[case.dtype]).float().numpy().reshape(E, so, inn)
    cols = [0, 17, 143, 64]
    x = torch.zeros(len(cols), inn, dtype=torch.bfloat16, device="cuda")
    for t, c in enumerate(cols):
        x[t, c] = 8.0
    ids = torch.tensor([[1, 0], [E - 1, 1], [1, 2], [0, E - 1]], device="cuda")
    got = plan.experts_matvec_fp8(0, ids, x, torch.from_numpy(s).cuda(), (bn, bk)).float().cpu().numpy()
    for t, c in enumerate(cols):
        for j in range(2):
            e = int(ids[t, j])
            want = F.one_hot_model(w[e], s[e], bn, bk, [c], 3, "bf16")[0]
            assert np.array_equal(got[t, j].view(np.uint32), want.view(np.uint32)), (t, j)


def test_qwen3_30b_a3b_fp8_layer_at_1_and_4_tokens():
    """Qwen3-30B-A3B-FP8: 128 experts, top-8, gate_up [128, 1536, 2048], down [128, 2048, 768], 128x128 blocks."""
    E, H, I, k = 128, 2048, 768, 8
    gu = _experts_weight("e4m3", E, 2 * I, H, 1000)
    dn = _experts_weight("e4m3", E, H, I, 2000)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w) for w, _ in (gu, dn)])
    assert plan.experts_matvec_fp8_ok(0, H) and plan.experts_matvec_fp8_ok(1, I)
    assert not plan.experts_matvec_fp8_ok(0, 40) and not plan.experts_matvec_fp8_ok(2, H)
    rng = np.random.default_rng(3)
    for T in (1, 4):
        ids = torch.from_numpy(routing(E, T, k, rng, False)).cuda()
        x = (torch.randn(T, H, device="cuda") * 0.5).to(torch.bfloat16)
        h = plan.experts_matvec_fp8(0, ids, x, gu[1], (128, 128))
        assert torch.equal(bits(h), bits(oracle(plan, 0, ids, x, gu[1], 2 * I, 128, 128))), T
        a = h[..., :I] * h[..., I:]
        d = plan.experts_matvec_fp8(1, ids, a, dn[1], (128, 128))
        assert torch.equal(bits(d), bits(oracle(plan, 1, ids, a, dn[1], H, 128, 128))), T
    plan.check()


def test_launch_count_n_zero_and_bad_ids():
    w, s = _experts_weight("e5m2", 16, 96, 512, 3)
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=16384).compress(w)])
    x = torch.randn(4, 512, device="cuda").to(torch.bfloat16)
    before = _native.launch_count()
    y = plan.experts_matvec_fp8(0, torch.zeros(0, 2, dtype=torch.int64, device="cuda"), x[:0], s, (128, 128))
    assert _native.launch_count() == before and y.shape == (0, 2, 96)
    for ids in ([[0, 1]], [[15, 0], [15, 1], [15, 2], [15, 3]], [[3, 4], [4, 3]]):
        idt = torch.tensor(ids, device="cuda")
        before = _native.launch_count()
        plan.experts_matvec_fp8(0, idt, x[:len(ids)], s, (128, 128))
        assert _native.launch_count() - before == LAUNCHES, ids
    plan.check()
    # out of range, and an expert repeated within a token (more pairs than slots), raise on check
    for ids in ([[2, -1]], [[16, 0]], [[5, 5]], [[3, 3], [3, 1]]):
        p2 = DecodePlan([ZipNN(input_format="torch", compression_chunk=16384).compress(w)])
        before = _native.launch_count()
        p2.experts_matvec_fp8(0, torch.tensor(ids, device="cuda"), x[:len(ids)], s, (128, 128))
        assert _native.launch_count() - before == LAUNCHES
        with pytest.raises(IndexError):
            p2.check()


def _scratch_size(ref, item, rows, inn, n_ids, top_k):
    out = C.c_size_t(0)
    rc = _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size(ref, item, rows, inn, n_ids, top_k, C.byref(out))
    return rc, out.value


def test_host_rejections_launch_nothing():
    E = 4
    w, s = _experts_weight("e4m3", E, 64, 1024, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    ref = plan._ref
    ids = torch.tensor([[0, 1], [2, 3]], device="cuda")
    x = torch.randn(2, 1024, device="cuda").to(torch.bfloat16)
    y = torch.empty(2, 2, 64, dtype=torch.bfloat16, device="cuda")
    rc, need = _scratch_size(ref, 0, E, 1024, 4, 2)
    assert rc == 0 and need > 0
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    good = dict(item=0, rows=E, ids=ids.data_ptr(), n=4, idb=8, top_k=2, fmt=F.CODE["e4m3"], xdt=0, inn=1024, x=x.data_ptr(),
                xs=1024, per_pair=0, scale=s.data_ptr(), bn=128, bk=128, y=y.data_ptr(), ys=64, scr=scratch.data_ptr(), sb=need)

    def call(**kw):
        a = dict(good, **kw)
        return _native.lib().zipnn_b200_decode_plan_experts_matvec_fp8(
            ref, a["item"], a["rows"], a["ids"], a["n"], a["idb"], a["top_k"], a["fmt"], a["xdt"], a["inn"], a["x"], a["xs"],
            a["per_pair"], a["scale"], a["bn"], a["bk"], a["y"], a["ys"], a["scr"], a["sb"], _st())

    assert call() == 0
    torch.cuda.synchronize()
    bad = [dict(item=1), dict(item=-1), dict(rows=3), dict(rows=0), dict(idb=2), dict(ids=None), dict(ids=ids.data_ptr() + 4),
           dict(n=3), dict(top_k=0), dict(n=10, top_k=2), dict(fmt=7), dict(xdt=2), dict(inn=1000), dict(inn=0), dict(x=None),
           dict(x=x.data_ptr() + 2), dict(xs=1000), dict(xs=1028), dict(scale=None), dict(scale=s.data_ptr() + 2), dict(bn=0),
           dict(bk=8), dict(bk=24), dict(y=None), dict(y=y.data_ptr() + 1), dict(ys=32), dict(scr=None),
           dict(scr=scratch.data_ptr() + 16), dict(sb=need - 1)]
    for kw in bad:
        before = _native.launch_count()
        assert call(**kw) != 0, kw
        assert _native.launch_count() == before, kw
    assert _scratch_size(ref, 0, E, 1024, 10, 2)[0] != 0    # 5 tokens
    assert _scratch_size(ref, 0, E, 1024, 3, 2)[0] != 0     # not whole tokens
    # the Python layer
    with pytest.raises(ValueError):
        plan.experts_matvec_fp8(0, torch.zeros(5, 2, dtype=torch.int64, device="cuda"), torch.zeros(5, 1024, dtype=torch.bfloat16, device="cuda"), s, (128, 128))
    with pytest.raises(ValueError):
        plan.experts_matvec_fp8(0, ids, x.float(), s, (128, 128))
    with pytest.raises(ValueError):
        plan.experts_matvec_fp8(0, ids, x, s[:2], (128, 128))
    with pytest.raises(ValueError):
        plan.experts_matvec_fp8(0, ids.reshape(-1), x, s, (128, 128))
    with pytest.raises(ValueError):
        plan.experts_matvec_fp8(0, ids, x, s, (128, 128), out=torch.empty(2, 2, 63, dtype=torch.bfloat16, device="cuda"))
    plan.check()


def test_graph_replays_new_ids_and_scales_and_interleaves_with_other_calls():
    E = 8
    gu = _experts_weight("e4m3", E, 704, 256, 11)   # ragged: 5.5 blocks of 128 rows per expert
    dn = _experts_weight("e4m3", E, 256, 352, 31)
    tensors = [w for w, _ in (gu, dn)]
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=65536).compress(w) for w in tensors])
    scales = [gu[1].clone(), dn[1].clone()]
    need = max(plan.select_scratch_bytes(), plan.experts_matvec_fp8_scratch_bytes(0, 256, 2), plan.experts_matvec_fp8_scratch_bytes(1, 352, 2),
               plan.matvec_fp8_scratch_bytes(0, 256, 1))
    shared = torch.empty(need, dtype=torch.uint8, device="cuda")
    ids = torch.tensor([[0, 1], [1, 2], [3, 1], [0, 2]], device="cuda")
    x = torch.randn(4, 256, device="cuda").to(torch.float16)
    a = torch.randn(4, 2, 352, device="cuda").to(torch.float16)
    ys = [torch.empty(4, 2, 704, dtype=torch.float16, device="cuda"), torch.empty(4, 2, 256, dtype=torch.float16, device="cuda")]

    def run():
        plan.experts_matvec_fp8(0, ids, x, scales[0], (128, 128), out=ys[0], scratch=shared)
        plan.experts_matvec_fp8(1, ids, a, scales[1], (128, 128), out=ys[1], scratch=shared)

    run()   # outside the capture: the first call reads the chunk modes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    rng = np.random.default_rng(4)
    dense = [w.view(torch.uint8).reshape(E, -1) for w in tensors]
    for r in range(3):
        ids.copy_(torch.from_numpy(routing(E, 4, 2, rng, r % 2 == 0)))
        scales[0].copy_(gu[1] * (r + 1.5))
        x.copy_(torch.randn(4, 256, device="cuda"))
        for y in ys:
            y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        replayed = [y.clone() for y in ys]
        eager = [plan.experts_matvec_fp8(0, ids, x, scales[0], (128, 128)), plan.experts_matvec_fp8(1, ids, a, scales[1], (128, 128))]
        for p, q in zip(replayed, eager):
            assert torch.equal(bits(p), bits(q)), r
        assert torch.equal(bits(eager[0]), bits(oracle(plan, 0, ids, x, scales[0], 704, 128, 128))), r
        # the other calls of the plan on the same scratch, in between
        sel = ids.reshape(-1).unique()
        coded = plan.run_select(ids, scratch=shared)
        for o, d in zip(coded, dense):
            assert torch.equal(o.view(torch.uint8).reshape(E, -1)[sel], d[sel]), r
        outs = plan.dequant_fp8_select(ids, [256, 352], scales, [(128, 128)] * 2, scratch=shared)
        assert not torch.isnan(outs[0][ids[0, 0]]).any()
        flat = expanded_rows(scales[0], 704, 128)
        y0 = plan.matvec_fp8(0, x[:1], flat, (1, 128), scratch=shared)
        e = int(ids[0, 0])
        assert torch.equal(bits(y0[0, e * 704:(e + 1) * 704]), bits(replayed[0][0, 0])), r
        if r == 1:
            for o, d in zip(plan.run(), dense):
                assert torch.equal(o.view(torch.uint8).reshape(E, -1), d)
        again = plan.experts_matvec_fp8(1, ids, a, scales[1], (128, 128), scratch=shared)
        assert torch.equal(bits(again), bits(replayed[1])), r
    plan.check()


# ------------------------------------------------------------------ resident modules
def composition(mod, plan, names, hidden, ids, weights):
    """The experts_matvec forward computed from per-pair matvec_fp8 calls: gate (or activation), combine."""
    where = dict(names)
    first, down = ("gate_up_proj" if "gate_up_proj" in where else "up_proj"), "down_proj"
    block = mod.block_size
    outs = []
    for name, x in ((first, hidden), (down, None)):
        k = where[name]
        s = getattr(mod, name + "_scale_inv")
        so, inn = plan.outputs[k].shape[1:]
        bn, bk = (so, inn) if block is None else block
        y = oracle(plan, k, ids, x if x is not None else a, s, so, min(bn, so), min(bk, inn))
        if x is not None:
            a = mod._apply_gate(y) if first == "gate_up_proj" else mod.act_fn(y)
        outs.append(y)
    d = outs[1]
    wd = (d * weights.to(d.dtype)[..., None]).to(torch.float32)
    acc = torch.zeros(wd.shape[0], wd.shape[2], dtype=torch.float32, device="cuda")
    for j in range(wd.shape[1]):
        acc += wd[:, j]
    return acc.to(hidden.dtype)


def check_experts_modules(m, seed):
    state = getattr(m, R._ATTR)
    entries = [e for e in state.entries if e.mode == "fp8_experts_matvec"]
    assert len(entries) == 2
    g = torch.Generator("cuda").manual_seed(seed)
    with torch.no_grad():
        for e in entries:
            E = e.module.num_experts
            for T in range(1, EXPERTS_MATVEC_MAX_TOKENS + 1):
                k = 2
                x = torch.randn(T, 256, generator=g, device="cuda").to(torch.bfloat16)
                ids = torch.stack([torch.randperm(E, generator=g, device="cuda")[:k] for _ in range(T)])
                w = torch.rand(T, k, generator=g, device="cuda").to(torch.bfloat16)
                got = e.module(x, ids, w)
                assert torch.equal(got, composition(e.module, e.plan, e.names, x, ids, w)), T
                assert torch.equal(e.module(hidden_states=x, top_k_index=ids, top_k_weights=w), got)


@pytest.mark.parametrize("which", ("qwen3", "mixtral"))
def test_resident_tiny_moe(which):
    m = tiny_fp8_moe(which, 1)
    base = copy.deepcopy(m)
    before = dense_state(m)
    want_rep = compress_module(base, fp8=True, experts=True, matvec=8)
    rep = compress_module(m, fp8=True, experts=True, matvec=8, experts_matvec=4)
    assert rep["experts_matvec_modules"] == 2 and rep["experts_matvec_scratch_bytes"] > 0
    assert {k: v for k, v in rep.items() if not k.startswith("experts_matvec")} == want_rep
    check_experts_modules(m, 2)
    state = getattr(m, R._ATTR)
    assert all(e.plan._scratches.get("experts_matvec_fp8") is None for e in state.entries)   # the shared scratch only
    g = torch.Generator("cuda").manual_seed(3)
    with torch.no_grad():
        # above the limit the experts take the "fp8_experts" forward: the model is the one without experts_matvec
        for impl in ("eager", "grouped_mm"):
            m.config._experts_implementation = base.config._experts_implementation = impl
            ids = torch.randint(0, 512, (1, 9), generator=g, device="cuda")
            assert torch.equal(m(ids, use_cache=False).logits, base(ids, use_cache=False).logits), impl
            # at most 4 tokens: the experts differ from the dense product only in the order of the fp32 sums
            ids = ids[:, :3]
            got, want = m(ids, use_cache=False).logits.double(), base(ids, use_cache=False).logits.double()
            assert torch.isfinite(got).all() and torch.allclose(got, want, rtol=0.05, atol=0.05 * want.abs().max().item()), impl
        # a graph-captured experts forward equals eager
        e = next(e for e in state.entries if e.mode == "fp8_experts_matvec")
        x = torch.randn(3, 256, device="cuda").to(torch.bfloat16)
        ids = torch.stack([torch.randperm(e.module.num_experts, device="cuda")[:2] for _ in range(3)])
        w = torch.rand(3, 2, device="cuda").to(torch.bfloat16)
        e.module(x, ids, w)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = e.module(x, ids, w)
        ids.copy_(torch.stack([torch.randperm(e.module.num_experts, device="cuda")[:2] for _ in range(3)]))
        x.copy_(torch.randn(3, 256, device="cuda"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, e.module(x, ids, w))
    with pytest.raises(RuntimeError, match="no_grad"):
        e.module(x, ids, w)
    decompress_module(m)
    after = dense_state(m)
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(raw(after[k]), raw(before[k])), k
    assert not any("forward" in x.__dict__ for x in m.modules())


def test_load_module_from_safetensors_and_znn(tmp_path):
    src = tiny_fp8_moe("qwen3", 3)
    sd = {k: v.contiguous() for k, v in dense_state(src).items()}
    want_rep = compress_module(tiny_fp8_moe("qwen3", 3), fp8=True, experts=True, matvec=8, experts_matvec=4)
    plain = str(tmp_path / "fp8_moe.safetensors")
    save_file(sd, plain)
    a = tiny_fp8_moe("qwen3", 4)   # other values: every one must come from the file
    assert load_module(a, plain, fp8=True, experts=True, matvec=8, experts_matvec=4) == want_rep
    check_experts_modules(a, 5)
    znn = str(tmp_path / "fp8_moe.znn.safetensors")
    save_module(a, znn)
    b = tiny_fp8_moe("qwen3", 5)
    assert load_module(b, znn, fp8=True, experts=True, matvec=8, experts_matvec=4) == want_rep
    check_experts_modules(b, 6)
    decompress_module(b)
    for k, v in dense_state(b).items():
        assert torch.equal(raw(v), raw(sd[k])), k
