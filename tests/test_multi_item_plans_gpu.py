"""Gathers and matvecs on every item of multi-item decode plans, against the dense bytes and an fp64 product.

The layouts of tests/multi_item_plans.py (6-12 items each: empty, constant, raw, general-mode, split and boxed items
around bf16 / fp16 / fp32 / fp8 targets, each with a decoy of equal geometry and other bytes), rotated so that every
target is first, in the middle and last:
  * the segment index holds every target's segments at the modelled seg_base, counting its coded symbols;
  * every whole item gathers through the raw ABI (canary-padded outputs, row sizes inside a chunk, straddling chunks
    and spanning several, duplicated / first-and-last / one-chunk / every-chunk / empty ids, int32 and int64) and
    through DecodePlan.gather; every eligible float item multiplies 1, 3 and 8 tokens, with and without bias, within
    the fp64 bound of test_matvec_gpu; box, split and empty items refuse both calls, constant, raw, general, ragged
    and fp8 items refuse the matvec, with no launch and nothing written;
  * gathers and matvecs write no plan output; a run after them decodes every item and the error word stays clean.
Also: two plans sharing one scratch buffer run, run_into, gather and multiply interleaved on one stream without a host
sync and in one captured graph; a plan created into the memory of an older plan follows its own items (the cached
"every chunk fused" answer included) while the stale struct is refused; a resident model whose tied embedding gathers
from item 1 of the head's plan; matvec bit for bit in fp16 and fp32, fp16 overflow to inf, and inf / NaN in W and x.
"""
import ctypes as C
import copy
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import multi_item_plans as M
import test_decode_plan_gpu as DP
import test_decoder_tables_gpu as D
import test_gather_gpu as GG
import test_matvec_gpu as MV
from test_resident_gather_gpu import graph_logits
from test_resident_gpu import H, VOCAB, Layer
from zipnn_b200 import DecodePlan, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200.resident import _ATTR

pytestmark = pytest.mark.gpu

CODE = {"bf16": 0, "fp16": 1, "fp32": 2}
ES = {"bf16": 2, "fp16": 2, "fp32": 4, "fp8": 1}
CANARY = DP.CANARY


def _st():
    return torch.cuda.current_stream().cuda_stream


def _set_env(monkeypatch, env):
    DP._set_env(monkeypatch, env)


def _item(e):
    return DP.Item(e.name, e.body, e.G, e.bits, e.chunk, e.orig, e.want, box=None if e.whole else e.box)


@pytest.fixture(scope="module")
def dev_streams():
    cache = {}

    def get(e):
        if e.name not in cache:
            cache[e.name] = torch.from_numpy(e.stream.copy()).cuda()
        return cache[e.name]
    return get


def _weight(e):
    return e.tensor.cuda()


def _x(dtype, shape, seed, std=1.0):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * std).to(M.TORCH[dtype])


def check_index(p, model, what):
    """The device's segment index against the model: its size, and every target's rows at the modelled seg_base."""
    ib, ci, seg = p.index()
    assert ci == model.coded_items and ib == ci * M.SEG_PER_ITEM * 8, what
    for i, e in enumerate(model.entries):
        if e.kind in ("target", "decoy"):
            first, n, sym = model.seg_rows(i)
            assert first > 0 or i == min(j for j, f in enumerate(model.entries) if f.coded(0, f.K)), (what, e.name)
            assert int(seg[first: first + n, 1].sum()) == sym, (what, e.name)


# ------------------------------------------------------------------ refusals
def _refused_gather(p, i):
    L = _native.lib()
    out = C.c_size_t(0)
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    o = torch.full((256,), CANARY, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_gather_scratch_size(C.byref(p.plan), i, 16, 1, C.byref(out)) == _native.E_UNSUPPORTED
    rc = L.zipnn_b200_decode_plan_gather(C.byref(p.plan), i, 16, ids.data_ptr(), 4, 8, o.data_ptr(), scratch.data_ptr(), scratch.numel(), _st())
    assert rc == _native.E_UNSUPPORTED and _native.launch_count() == before
    assert torch.all(o == CANARY)


def _refused_matvec(p, i, e):
    """Both matvec calls answer E_UNSUPPORTED for item i seen as rows of a multiple of 16 bytes that divides it."""
    L = _native.lib()
    code = CODE.get(e.dtype, 0)
    es = 4 if code == 2 else 2
    row = e.orig // e.shape[0] if len(e.shape) > 1 and e.orig else 0
    in_bytes = row if row and row % 16 == 0 else 16
    assert e.orig % in_bytes == 0 and e.orig % es == 0
    inf = in_bytes // es
    x = torch.zeros(inf, dtype=torch.float32, device="cuda")
    y = torch.full((max(1, e.orig // in_bytes) * 4,), CANARY, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(4 << 20, dtype=torch.uint8, device="cuda")
    out = C.c_size_t(0)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(p.plan), i, code, inf, 1, C.byref(out)) == _native.E_UNSUPPORTED, e.name
    rc = L.zipnn_b200_decode_plan_matvec(C.byref(p.plan), i, code, inf, x.data_ptr(), inf, 1, None, y.data_ptr(), y.numel() // 4,
                                         scratch.data_ptr(), scratch.numel(), _st())
    assert rc == _native.E_UNSUPPORTED and _native.launch_count() == before, (e.name, rc)
    assert torch.all(y == CANARY), e.name


def raw_matvec(p, i, e, x, bias=None):
    L = _native.lib()
    code = CODE[e.dtype]
    nt, inf = x.shape
    out_f = e.orig // ES[e.dtype] // inf
    sz = C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(p.plan), i, code, inf, nt, C.byref(sz)) == 0, e.name
    scratch = torch.empty(sz.value, dtype=torch.uint8, device="cuda")
    y = torch.full((nt, out_f), float("nan"), dtype=x.dtype, device="cuda")
    before = _native.launch_count()
    rc = L.zipnn_b200_decode_plan_matvec(C.byref(p.plan), i, code, inf, x.data_ptr(), inf, nt, bias.data_ptr() if bias is not None else None,
                                         y.data_ptr(), out_f, scratch.data_ptr(), sz.value, _st())
    assert rc == 0 and _native.launch_count() - before == 2, (e.name, rc)
    return y


# ------------------------------------------------------------------ every item of every rotation
def _raw_gathers(p, i, e, rng, full):
    n = 0
    for R in GG.row_sizes(e.orig, e.chunk):
        rows = e.orig // R
        sets = GG.id_sets(rows, R, e.chunk, rng)
        for k, ids in enumerate(sets if full else sets[:2] + sets[-1:]):
            t = torch.from_numpy(ids).to(torch.int32 if k % 2 else torch.int64).cuda()
            rc, out = GG.gather(p, i, R, t, 4 if k == 0 else 64)
            assert rc == 0, (e.name, R, k)
            GG.check_out(out, GG.expect(e.data, R, ids), f"{e.name} item {i} R={R} ids#{k}")
            n += 1
    return n


def _plan_gathers(plan, k, e, seed):
    rows = e.shape[0]
    W = _weight(e)
    g = torch.Generator("cuda").manual_seed(seed)
    for ids in (torch.randint(0, rows, (3, 17), device="cuda", generator=g), torch.tensor([rows - 1, 0, rows - 1], device="cuda", dtype=torch.int32),
                torch.zeros(0, dtype=torch.int64, device="cuda")):
        got = plan.gather(k, ids)
        assert got.shape == ids.shape + tuple(e.shape[1:]) and got.dtype == W.dtype
        want = W.view(torch.uint8).reshape(rows, -1).index_select(0, ids.reshape(-1).long())
        assert torch.equal(got.view(torch.uint8).reshape(want.shape), want), (e.name, k)


def _plan_matvecs(plan, k, e, seed):
    W = _weight(e)
    inf = e.shape[-1]
    assert plan.matvec_ok(k, inf), e.name
    out_f = e.orig // ES[e.dtype] // inf
    for nt in (1, 3, 8):
        for with_bias in (False, True):
            x = _x(e.dtype, (nt, inf), seed + 10 * nt + with_bias)
            bias = _x(e.dtype, (out_f,), seed + 7, std=0.5) if with_bias else None
            y = plan.matvec(k, x, bias=bias)
            MV._check(y, x, W.reshape(out_f, inf), bias, (e.name, k, nt, with_bias))


@pytest.mark.parametrize("name", M.LAYOUTS)
def test_every_item_of_every_rotation(name, monkeypatch, dev_streams):
    entries, env = M.layout(name)
    _set_env(monkeypatch, env)
    limit = M.limit_of(env)
    rng = np.random.default_rng(len(name))
    rots = M.placements(entries)
    n_gathers = 0
    for r in rots:
        es = M.rotate(entries, r)
        model = M.Model(es, limit)
        # the raw ABI: every item, boxes included
        p = DP.Plan([_item(e) for e in es])
        assert p.rc == 0, (name, r)
        for it in p.items:
            it.check("create")
        check_index(p, model, (name, r))
        for it in p.items:       # nothing the gathers and matvecs do may reach the outputs
            it.scribble()
        for i, e in enumerate(es):
            if model.piece[i] < 0:
                _refused_gather(p, i)
                _refused_matvec(p, i, e)
                continue
            n_gathers += _raw_gathers(p, i, e, rng, full=r == rots[0])
            if e.eligible:
                x = _x(e.dtype, (2, e.shape[-1]), 31 * r + i)
                MV._check(raw_matvec(p, i, e, x), x, _weight(e).reshape(-1, e.shape[-1]), None, (name, r, e.name))
            else:
                _refused_matvec(p, i, e)
        torch.cuda.synchronize()
        for it in p.items:
            host = it.out.cpu().numpy()
            assert np.all(host[:DP.PAD] == CANARY) and np.all(host[DP.PAD + it.want.size:] == CANARY), it.name
            assert np.all(host[DP.PAD: DP.PAD + it.want.size] == CANARY ^ 0xFF), f"{it.name}: a gather or matvec wrote a plan output"
        assert p.run() == 0 and p.status() == 0
        for it in p.items:
            it.check(f"run after the calls, rotation {r}")
        # DecodePlan: the whole items
        dp = M.without_boxes(es)
        dmodel = M.Model(dp, limit)
        plan = DecodePlan([dev_streams(e) for e in dp])
        assert plan.coded_items == dmodel.coded_items
        for o in plan.outputs:
            o.view(torch.uint8).fill_(CANARY)
        for k, e in enumerate(dp):
            if dmodel.piece[k] < 0:   # empty (no rows) or split: refused
                with pytest.raises(ValueError if e.kind == "empty" else _native.ZipNNNativeError) as err:
                    plan.gather(k, torch.zeros(1, dtype=torch.int64, device="cuda"))
                assert e.kind == "empty" or err.value.status == _native.E_UNSUPPORTED
                assert e.kind == "empty" or not plan.matvec_ok(k, 8)
                continue
            _plan_gathers(plan, k, e, 100 * r + k)
            if e.eligible:
                _plan_matvecs(plan, k, e, 1000 * r + 10 * k)
            elif e.dtype in CODE and len(e.shape) > 1:
                assert not plan.matvec_ok(k, e.shape[-1]), e.name
        for o in plan.outputs:
            assert torch.all(o.view(torch.uint8) == CANARY), "a gather or matvec wrote a plan output"
        plan.run()
        for o, e in zip(plan.outputs, dp):
            assert torch.equal(o.view(torch.uint8).reshape(-1).cpu(), torch.from_numpy(e.data)), e.name
        plan.check()
    print(f"{name}: {len(rots)} rotations, {n_gathers} raw gathers")


# ------------------------------------------------------------------ interleaved calls, eager and in one graph
def test_interleaved_calls_on_shared_scratch(dev_streams, monkeypatch):
    _set_env(monkeypatch, {})
    ea = M.without_boxes(M.layout("L1")[0])
    eb = M.without_boxes(M.layout("L3")[0])
    sa, sb = [dev_streams(e) for e in ea], [dev_streams(e) for e in eb]
    need = max(DecodePlan.sizes(sa)[1], DecodePlan.sizes(sb)[1], 8 << 20)
    shared = torch.empty(need, dtype=torch.uint8, device="cuda")
    pa, pb = DecodePlan(sa, scratch=shared), DecodePlan(sb, scratch=shared)
    names_a, names_b = [e.name for e in ea], [e.name for e in eb]
    a, b, d = names_a.index("A_bf16"), names_a.index("W_fp32"), names_a.index("emb_fp8")
    c = names_b.index("c4k_bf16")
    Wa, Wb, Wc, Wd = _weight(ea[a]), _weight(ea[b]), _weight(eb[c]), _weight(ea[d])
    assert pa.matvec_ok(b, Wb.shape[1]) and pb.matvec_ok(c, Wc.shape[1])   # (the first call synchronises: before the sequence)
    for plan, k, w in ((pa, a, Wa), (pa, d, Wd)):
        assert plan.gather_scratch_bytes(k, 1) <= need
    assert pa.matvec_scratch_bytes(b, Wb.shape[1]) <= need and pb.matvec_scratch_bytes(c, Wc.shape[1]) <= need
    ids_a = torch.zeros(24, dtype=torch.int64, device="cuda")
    ids_d = torch.zeros(40, dtype=torch.int32, device="cuda")
    xb = torch.zeros(8, Wb.shape[1], dtype=Wb.dtype, device="cuda")
    xc = torch.zeros(3, Wc.shape[1], dtype=Wc.dtype, device="cuda")
    oa = torch.empty(24, Wa.shape[1], dtype=Wa.dtype, device="cuda")
    od = torch.empty(40, Wd.shape[1], dtype=Wd.dtype, device="cuda")
    ob = torch.empty(8, Wb.shape[0], dtype=Wb.dtype, device="cuda")
    oc = torch.empty(3, Wc.shape[0], dtype=Wc.dtype, device="cuda")
    shifted = torch.empty(pa.nbytes["out"] + 4096, dtype=torch.uint8, device="cuda")
    sh = shifted[2048: 2048 + pa.nbytes["out"]]

    def sequence():
        pa.run()
        pa.gather(a, ids_a, out=oa, scratch=shared)
        pa.matvec(b, xb, out=ob, scratch=shared)
        pa.run_into(sh, max_ctas=3)
        pb.matvec(c, xc, out=oc, scratch=shared)
        pa.gather(d, ids_d, out=od, scratch=shared)
        pa.run()

    def feed(seed):
        g = torch.Generator("cuda").manual_seed(seed)
        ids_a.copy_(torch.randint(0, Wa.shape[0], (24,), device="cuda", generator=g))
        ids_d.copy_(torch.randint(0, Wd.shape[0], (40,), device="cuda", generator=g))
        xb.copy_(_x("fp32", tuple(xb.shape), seed + 1))
        xc.copy_(_x("bf16", tuple(xc.shape), seed + 2))
        for t in [o.view(torch.uint8) for o in pa.outputs] + [shifted, oa.view(torch.uint8), od.view(torch.uint8), ob.view(torch.uint8), oc.view(torch.uint8)]:
            t.fill_(CANARY)

    def verify(what):
        torch.cuda.synchronize()
        assert torch.equal(oa, Wa[ids_a]) and torch.equal(od.view(torch.uint8), Wd.view(torch.uint8)[ids_d.long()]), what
        MV._check(ob, xb, Wb, None, what)
        MV._check(oc, xc, Wc, None, what)
        assert torch.equal(ob, pa.matvec(b, xb.clone())) and torch.equal(oc, pb.matvec(c, xc.clone())), (what, "eager calls, own scratch")
        views = pa.views(sh)
        for o, v, e in zip(pa.outputs, views, ea):
            want = torch.from_numpy(e.data).cuda()
            assert torch.equal(o.view(torch.uint8).reshape(-1), want) and torch.equal(v.view(torch.uint8).reshape(-1), want), (what, e.name)
        assert torch.all(shifted[:2048] == CANARY) and torch.all(shifted[2048 + pa.nbytes["out"]:] == CANARY), what
        pa.check()
        pb.check()

    feed(1)
    sequence()
    verify("eager")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sequence()
    for rep in range(3):
        feed(10 + rep)
        g.replay()
        verify(f"replay {rep}")


# ------------------------------------------------------------------ a plan created into an older plan's memory
def _create_into(items, meta, scratch):
    L = _native.lib()
    arr = DP._array(items)
    plan = _native.DecodePlanStruct()
    rc = L.zipnn_b200_decode_plan_create(arr, len(items), meta.data_ptr(), meta.numel(), scratch.data_ptr(), scratch.numel(),
                                         C.byref(plan), _st())
    return rc, types.SimpleNamespace(plan=plan, items=items)


def _sizes(items):
    pb, sb = C.c_size_t(0), C.c_size_t(0)
    assert _native.lib().zipnn_b200_decode_plan_size(DP._array(items), len(items), None, C.byref(pb), C.byref(sb)) == 0
    return pb.value, sb.value


def test_plan_created_at_a_reused_address(monkeypatch):
    _set_env(monkeypatch, {})
    second = lambda c, g: "geo5"   # noqa: E731
    gen_p = M._planes_entry(D.planes_case("reuse_gen_p", "bf16", 4096, ["geo5"] * 4, seed=201, side=second), (64, 128), "general")
    gen_q = M._planes_entry(D.planes_case("reuse_gen_q", "bf16", 4096, ["geo5"] * 4, seed=202, side=second), (64, 128), "general")
    fus_p = M.pair("reuse_fus_p", "bf16", (64, 128), 4096, 203)[0]
    fus_q = M.pair("reuse_fus_q", "bf16", (64, 128), 4096, 205)[0]
    extra = M.pair("reuse_extra", "fp16", (32, 256), 4096, 207)[0]
    P_entries, Q_entries = [fus_p, gen_p], [gen_q, fus_q, extra]
    assert fus_p.fused and fus_q.fused and not gen_p.fused and not gen_q.fused
    P_items, Q_items = [_item(e) for e in P_entries], [_item(e) for e in Q_entries]
    (pp, ps), (qp, qs) = _sizes(P_items), _sizes(Q_items)
    meta = torch.empty(max(pp, qp), dtype=torch.uint8, device="cuda")
    scratch = torch.empty(max(ps, qs), dtype=torch.uint8, device="cuda")
    rc, P = _create_into(P_items, meta, scratch)
    assert rc == 0
    L = _native.lib()
    out = C.c_size_t(0)
    # P's record: item 0 fused (the answer is cached now), item 1 general
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(P.plan), 0, 0, 128, 1, C.byref(out)) == 0
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(P.plan), 1, 0, 128, 1, C.byref(out)) == _native.E_UNSUPPORTED
    x = _x("bf16", (2, 128), 5)
    MV._check(raw_matvec(P, 0, fus_p, x), x, _weight(fus_p), None, "P item 0")
    stale = _native.DecodePlanStruct.from_buffer_copy(P.plan)
    rc, Q = _create_into(Q_items, meta, scratch)
    assert rc == 0
    assert C.addressof(Q.plan) != C.addressof(stale)
    for it in Q.items:
        it.check("create Q")
    # Q follows its own items: item 0 general (refused although P's item 0 was fused), item 1 fused
    _refused_matvec(Q, 0, gen_q)
    MV._check(raw_matvec(Q, 1, fus_q, x), x, _weight(fus_q), None, "Q item 1")
    x16 = _x("fp16", (3, 256), 6)
    MV._check(raw_matvec(Q, 2, extra, x16), x16, _weight(extra), None, "Q item 2")
    rng = np.random.default_rng(7)
    for i, e in enumerate(Q_entries):
        _raw_gathers(Q, i, e, rng, full=False)
    # the stale struct: refused by every gather and matvec call, no launch
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    o = torch.full((4096,), CANARY, dtype=torch.uint8, device="cuda")
    big = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    before = _native.launch_count()
    for k in (0, 1, 2):
        assert L.zipnn_b200_decode_plan_gather_scratch_size(C.byref(stale), k, 256, 1, C.byref(out)) == _native.E_ARG
        assert L.zipnn_b200_decode_plan_gather(C.byref(stale), k, 256, ids.data_ptr(), 4, 8, o.data_ptr(), big.data_ptr(), big.numel(),
                                               _st()) == _native.E_ARG
        assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(stale), k, 0, 128, 1, C.byref(out)) == _native.E_ARG
        assert L.zipnn_b200_decode_plan_matvec(C.byref(stale), k, 0, 128, x.data_ptr(), 128, 2, None, o.data_ptr(), 64, big.data_ptr(),
                                               big.numel(), _st()) == _native.E_ARG
    assert _native.launch_count() == before and torch.all(o == CANARY)
    for it in Q.items:
        it.scribble()
    assert L.zipnn_b200_decode_plan_run(C.byref(Q.plan), _st()) == 0
    assert L.zipnn_b200_decode_plan_status(C.byref(Q.plan), _st()) == 0
    for it in Q.items:
        it.check("run Q")


# ------------------------------------------------------------------ a resident embedding that gathers from item 1
class NormHead(torch.nn.Module):
    """An lm_head with its own RMSNorm scale, registered in front of its weight."""

    def __init__(self):
        super().__init__()
        self.scale = torch.nn.Parameter(torch.ones(H))
        self.weight = torch.nn.Parameter(torch.empty(VOCAB, H))

    def forward(self, x):
        return F.linear(F.rms_norm(x, (H,), self.scale), self.weight)


class HeadModel(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.embed_tokens = torch.nn.Embedding(VOCAB, H)
        self.layers = torch.nn.ModuleList([Layer() for _ in range(2)])
        self.lm_head = NormHead()
        self.lm_head.weight = self.embed_tokens.weight

    def forward(self, ids):
        x = self.embed_tokens(ids)
        for layer in self.layers:
            x = layer(x)
        return self.lm_head(x)


def _head_model(dtype, seed):
    torch.manual_seed(seed)
    m = HeadModel()
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() > 1:
                p.normal_(0, 0.02)
            else:
                p.copy_(1 + 0.1 * torch.randn_like(p))
    return m.to(device="cuda", dtype=dtype).eval()


def _check_gathers_from_item_1(model):
    state = getattr(model, _ATTR)
    assert [m for m, _, _, _ in state.gathers] == [model.embed_tokens]
    _, plan, k, own = state.gathers[0]
    head = next(p for m, p, _, _ in state.entries if m is model.lm_head)
    assert plan is head and k == 1 and not own, "the tied embedding gathers output 1 of the head's plan"
    assert tuple(plan.outputs[0].shape) == (H,) and tuple(plan.outputs[1].shape) == (VOCAB, H)
    return plan


@pytest.mark.parametrize("how", ("compress", "load"))
def test_resident_gather_from_item_1(how, tmp_path):
    dtype = torch.bfloat16
    dense = _head_model(dtype, 21)
    assert dense.lm_head.weight is dense.embed_tokens.weight
    ids = torch.randint(0, VOCAB, (2, 13), device="cuda", generator=torch.Generator("cuda").manual_seed(22))
    with torch.inference_mode():
        want = dense(ids)
    if how == "compress":
        model = copy.deepcopy(dense)
        compress_module(model, gather=True)
    else:
        src = copy.deepcopy(dense)
        compress_module(src)
        path = os.path.join(tmp_path, "head.znn.safetensors")
        save_module(src, path)
        del src
        with torch.device("meta"):
            model = HeadModel().to(dtype).eval()
        load_module(model, path, gather=True)
    plan = _check_gathers_from_item_1(model)
    with torch.inference_mode():
        assert torch.equal(model(ids), want)
        assert torch.equal(model.embed_tokens(ids), dense.embed_tokens(ids))
    assert torch.equal(graph_logits(model, ids), want)
    plan.check()
    decompress_module(model)
    got, ref = dict(model.named_parameters()), dict(dense.named_parameters())
    assert set(got) == set(ref)
    for n, p in ref.items():
        assert torch.equal(got[n].view(torch.uint8), p.view(torch.uint8)), n
    assert model.lm_head.weight is model.embed_tokens.weight
    with torch.inference_mode():
        assert torch.equal(model(ids), want)


# ------------------------------------------------------------------ matvec: exact sums, overflow, inf and NaN
def _exact_weights(dtype, out_f, in_f, rng):
    """±m·2^e exact in the dtype whose every partial sum over in_f terms with x in {-1, 0, 1} is exact in fp32, and
    whose only Huffman-coded plane is the top one (fused chunks).  fp32: an 8-bit m leaves the low two planes zero
    (RLE) and the third one random.  fp16: an 8-bit m would leave three zero bits in the low byte, which then codes;
    an 11-bit m with two exponents keeps it random and the sums within 4096 * 2^11 * 2 < 2^24 units."""
    s = rng.choice([-1.0, 1.0], (out_f, in_f))
    if dtype == torch.float32:
        m, e = rng.integers(128, 256, (out_f, in_f)), rng.integers(-9, -5, (out_f, in_f))
    else:
        m, e = rng.integers(1024, 2048, (out_f, in_f)), rng.integers(-20, -18, (out_f, in_f))
    w64 = s * m.astype(np.float64) * 2.0 ** e.astype(np.float64)
    w = torch.from_numpy(w64).to(dtype)
    assert torch.equal(w.double(), torch.from_numpy(w64)), "the weights are exact in the dtype"
    return w.cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_exact_products_bit_for_bit(dtype):
    rng = np.random.default_rng(3 if dtype == torch.float16 else 4)
    for out_f, in_f, nt in ((64, 4096, 1), (192, 2048, 8), (1024, 256, 5), (24, 3072, 3)):
        w = _exact_weights(dtype, out_f, in_f, rng)
        x = torch.from_numpy(rng.integers(-1, 2, (nt, in_f)).astype(np.float32)).to(dtype).cuda()
        plan = MV._plan_of(w)
        assert plan.matvec_ok(0, in_f), "these weights must give fused chunks, or the case tests nothing"
        y = plan.matvec(0, x)
        want = (x.double() @ w.double().T).to(dtype)   # exact in fp32: one rounding, the same in any order
        assert torch.equal(y, want), (dtype, out_f, in_f, nt)
        plan.check()


def test_fp16_sums_past_65504_are_inf():
    rng = np.random.default_rng(5)
    out_f, in_f = 96, 1024
    m = rng.integers(1024, 2048, (out_f, in_f)).astype(np.float64) * 2.0 ** -4   # 64 <= |w| < 128, exact in fp16
    sign = np.ones((out_f, in_f))
    sign[1::3] = -1.0
    sign[2::3] = rng.choice([-1.0, 1.0], (out_f // 3, in_f))
    w = torch.from_numpy(sign * m).to(torch.float16).cuda()
    x = torch.from_numpy(np.stack([np.ones(in_f), -np.ones(in_f), rng.integers(-1, 2, in_f), (np.arange(in_f) < 600) * 1.0])
                         .astype(np.float32)).to(torch.float16).cuda()
    plan = MV._plan_of(w)
    assert plan.matvec_ok(0, in_f)
    y = plan.matvec(0, x)
    want = (x.double() @ w.double().T).to(torch.float16)   # sums of at most 1024 * 2^11 units of 2^-4: exact in fp32
    assert bool(torch.isposinf(want).any()) and bool(torch.isneginf(want).any()) and bool(torch.isfinite(want).any())
    assert torch.equal(torch.isposinf(y), torch.isposinf(want)) and torch.equal(torch.isneginf(y), torch.isneginf(want))
    assert torch.equal(y, want)
    plan.check()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_inf_and_nan_in_weights_and_activations(dtype):
    out_f, in_f, nt = 64, 512, 4
    w = MV._gauss((out_f, in_f), dtype, 40)
    inf, nan = float("inf"), float("nan")
    w[1, 5], w[2, 7], w[3, 9], w[4, 0], w[4, 100], w[5, 33] = inf, -inf, nan, inf, -inf, -inf
    x = MV._gauss((nt, in_f), dtype, 41, std=1.0)
    x[0, 11], x[1, 20], x[3, 5], x[3, 300] = inf, nan, -inf, inf
    plan = MV._plan_of(w)
    assert plan.matvec_ok(0, in_f), "the special values must leave the chunks fused"
    bias = MV._gauss((out_f,), dtype, 42, std=0.5)
    y = plan.matvec(0, x, bias=bias).double()
    prod = x.double()[:, None, :] * w.double()[None, :, :]
    has_nan = torch.isnan(prod).any(-1)
    pos, neg = torch.isposinf(prod).any(-1), torch.isneginf(prod).any(-1)
    want_nan = has_nan | (pos & neg)
    want_pinf, want_ninf = pos & ~want_nan, neg & ~want_nan
    assert bool(want_nan.any()) and bool(want_pinf.any()) and bool(want_ninf.any())
    finite = ~(want_nan | want_pinf | want_ninf)
    assert bool(finite[2, 6:].all()), "a token with finite x and rows with finite weights stay finite"
    assert torch.equal(torch.isnan(y), want_nan)
    assert torch.equal(torch.isposinf(y), want_pinf) and torch.equal(torch.isneginf(y), want_ninf)
    fin = torch.where(torch.isfinite(prod), prod, torch.zeros_like(prod))
    ref = fin.sum(-1) + bias.double()
    mag = fin.abs().sum(-1) + bias.double().abs()
    bound = (in_f + 1) * 2.0 ** -24 * mag
    tol = bound + (ref.abs() + bound) * MV.REL[dtype] + MV.TINY[dtype]
    err = (y - ref).abs()
    assert torch.all(err[finite] <= tol[finite]), float((err - tol)[finite].max())
    plan.check()
