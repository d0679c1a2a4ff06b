"""The selected fp8 dequantize (zipnn_b200_decode_plan_dequant_fp8_select, DecodePlan.dequant_fp8_select) and the fp8
experts module mode (compress_module / load_module with fp8=True and experts=True), on an H100.

Kernel: every case of the fp8 corpus of tests/fp8_streams.py (every fused chunk size, both formats) seen as E experts,
bf16 and fp16 out, per-expert grids that are one scale per expert, per row, 128x128, ragged (bn not dividing the expert's
rows) and bk = 16; ids single, duplicated, all, first and last, straddling chunks.  The outputs are poisoned with two
values in turn; then every element of a chunk that meets a selected slice equals the numpy model of
test_dequant_fp8_host.py with that element's own expert grid, and every other byte keeps the poison.  All ids give
dequant_fp8's bytes; n = 0 launches nothing; three launches whatever the ids; a bad id raises and selects nothing; a
graph replays with new ids and a new scale; two-item plans interleave with run, run_select, dequant_fp8 and matvec_fp8 on
one scratch; every host rejection launches nothing; the corrupted fp8 streams; a Qwen3-30B-A3B-FP8-sized layer.

Modules: transformers' tiny Qwen3-MoE and Mixtral, quantized to fp8 as a pre-quantized checkpoint loads, under
compress_module(fp8=True, experts=True, matvec=8), against a reference copy whose experts hold torch-dequantized bf16
weights and whose FP8Linears are compressed the same way: logits bit for bit under eager, batched_mm and grouped_mm.
"""
import copy
import ctypes as C
import inspect

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

import corrupt_streams as CS
import fp8_streams as F
from test_dequant_fp8_gpu import ODT, _quantized, expanded, torch_dequant
from test_dequant_fp8_host import model as dq_model
from test_dequant_fp8_host import same_bits as dq_same_bits
from test_product_streams_gpu import _st, raw_plan
from test_select_host import written_bytes
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200 import resident as R

pytestmark = pytest.mark.gpu

LAUNCHES = 3   # index, the replay decoder with the dequantizing stores, the error pass
POISONS = (0x00, 0xFF)


def select_scratch(p_ref, rows):
    out = C.c_size_t(0)
    assert _native.lib().zipnn_b200_decode_plan_select_scratch_size(p_ref, rows, C.byref(out)) == 0
    return torch.empty(out.value, dtype=torch.uint8, device="cuda")


def items(specs):
    """[(in_features, scale tensor or pointer, bn, bk, out pointer)] -> the ctypes array."""
    arr = (_native.Fp8SelectItem * max(1, len(specs)))()
    for it, (inn, scale, bn, bk, out) in zip(arr, specs):
        it.in_features, it.block_rows, it.block_cols, it.d_out = inn, bn, bk, out
        it.d_scale = scale.data_ptr() if isinstance(scale, torch.Tensor) else scale
    return arr


def call(p_ref, rows, ids, fmt, odt, specs, scratch, n_items=None):
    return _native.lib().zipnn_b200_decode_plan_dequant_fp8_select(
        p_ref, rows, ids.data_ptr() if ids is not None else None, 0 if ids is None else ids.numel(),
        8 if ids is None else ids.element_size(), F.CODE[fmt], ODT[odt][1], len(specs) if n_items is None else n_items,
        items(specs), scratch.data_ptr() if isinstance(scratch, torch.Tensor) else scratch,
        scratch.numel() if isinstance(scratch, torch.Tensor) else 0, _st())


def experts_of(out: int) -> int:
    return next(d for d in (8, 5, 3, 2, 1) if out % d == 0)


def layouts(so: int, inn: int) -> dict:
    """Per-expert grids: F.layouts and a ragged one (5 rows: most slices are not a multiple)."""
    return dict(F.layouts(so, inn), ragged=(5, 32))


def expert_scales(E, so, inn, bn, bk, seed) -> np.ndarray:
    return np.stack([F.random_scales(so, inn, bn, bk, seed + e) for e in range(E)])


def want_of(case, E, s, bn, bk, odt) -> np.ndarray:
    """The model's bits [E * so, in], each expert with its own grid."""
    so = case.out // E
    full = np.concatenate([expanded(s[e], so, case.inn, bn, bk) for e in range(E)])
    return dq_model(case.data.reshape(case.out, case.inn), case.dtype, full, odt)


def check_select(p_ref, case, E, odt, layout, ids_list, seed, scratch):
    so = case.out // E
    bn, bk = layouts(so, case.inn)[layout]
    s = expert_scales(E, so, case.inn, bn, bk, seed)
    sd = torch.from_numpy(s).cuda()
    n = case.out * case.inn
    want = want_of(case, E, s, bn, bk, odt)
    buf = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    for k, ids in enumerate(ids_list):
        idt = torch.from_numpy(np.asarray(ids)).to(torch.int32 if k % 2 else torch.int64).cuda()
        wb = written_bytes(n, case.chunk, E, np.asarray(ids))   # fp8: one byte per element
        for poison in POISONS:
            buf.fill_(poison)
            before = _native.launch_count()
            assert call(p_ref, E, idt, case.dtype, odt, [(case.inn, sd, bn, bk, buf.data_ptr())], scratch) == 0
            assert _native.launch_count() - before == LAUNCHES
            got = buf.cpu().numpy().view(np.uint16).reshape(-1)
            ok = dq_same_bits(got[wb], want.reshape(-1)[wb], odt)
            assert ok.all(), (case.name, E, odt, layout, ids, int(np.flatnonzero(wb)[np.argmin(ok)]))
            raw = buf.cpu().numpy().reshape(-1, 2)
            assert np.all(raw[~wb] == poison), (case.name, E, odt, layout, ids, "an element of an untouched chunk was written")
            for e in set(int(i) for i in ids):   # (every routed slice is in a touched chunk)
                assert wb[e * so * case.inn: (e + 1) * so * case.inn].all()


def id_sets(E, rng):
    return [[0], [E - 1], [E - 1, 0, 0, E - 1], list(range(E)), rng.integers(0, E, 3).tolist()]


@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_corpus_at_every_chunk_size(chunk):
    cases = F.shape_cases(chunk)
    rng = np.random.default_rng(chunk)
    k0 = F.CHUNKS.index(chunk)
    names = ("tensor", "row", "block128", "bk16", "ragged")
    for i, case in enumerate(cases):
        p = raw_plan([case])
        ref = C.byref(p.plan)
        E = experts_of(case.out)
        scratch = select_scratch(ref, E)
        ids = id_sets(E, rng)
        for j, odt in enumerate(("bf16", "fp16")):
            check_select(ref, case, E, odt, names[(i + k0 + 2 * j) % 5], ids[j::2], 100 * k0 + i, scratch)
        p.items[0].check("after the selected dequantizes")   # (create's bytes: nothing wrote the plan's outputs)
        assert p.status() == 0


def test_stream_kinds_and_all_ids_equal_dequant_fp8():
    """Crafted tables, ring bitstreams, fixed-length codes; all ids give dequant_fp8's bytes of the whole tensor."""
    for j, case in enumerate(F.stream_cases()):
        p = raw_plan([case])
        ref = C.byref(p.plan)
        E = experts_of(case.out)
        so = case.out // E
        scratch = select_scratch(ref, E)
        for odt in ("bf16", "fp16"):
            layout = ("block128", "ragged", "bk16", "row")[(j + (odt == "fp16")) % 4]
            bn, bk = layouts(so, case.inn)[layout]
            check_select(ref, case, E, odt, layout, [[E // 2], [0, E - 1]], j, scratch)
            # all ids, one grid per expert == dequant_fp8 of [E * so, in] when the grids tile the whole (bn | so)
            if so % bn == 0:
                s = torch.from_numpy(expert_scales(E, so, case.inn, bn, bk, j)).cuda()
                a = torch.empty(case.out, case.inn, dtype=ODT[odt][0], device="cuda")
                b = torch.full_like(a, float("nan"))
                assert call(ref, E, torch.arange(E, device="cuda"), case.dtype, odt, [(case.inn, s, bn, bk, a.data_ptr())], scratch) == 0
                assert _native.lib().zipnn_b200_decode_plan_dequant_fp8(ref, 0, F.CODE[case.dtype], ODT[odt][1], case.inn, s.data_ptr(),
                                                                        bn, bk, b.data_ptr(), _st()) == 0
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (case.name, odt)
        assert p.status() == 0


# ------------------------------------------------------------------ the public API
def _experts_weight(fmt, E, out, inn, seed, block=(128, 128)):
    """E experts quantized per block -> (W [E, out, in] fp8, S [E, gr, gc] fp32); block None: S [E, 1, 1]."""
    ws, ss = zip(*[_quantized(fmt, out, inn, seed + e, block) for e in range(E)])
    return torch.stack(ws), torch.stack([s.reshape(1, 1) if block is None else s for s in ss]).contiguous()


def ref_slices(w, s, block, dtype, ids):
    return {e: torch_dequant(w[e], s[e].reshape(()) if block is None else s[e], block, dtype) for e in set(ids.reshape(-1).tolist())}


def bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("block", [(128, 128), None, (64, 32)])
def test_api_ragged_grids_and_block_none(block):
    """Mixtral-tiny-like shapes: gate_up [8, 704, 256] (5.5 blocks of 128 rows), down [8, 256, 352]."""
    E = 8
    gu = _experts_weight("e4m3", E, 704, 256, 1, block)
    dn = _experts_weight("e4m3", E, 256, 352, 50, block)
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=65536).compress(w) for w, _ in (gu, dn)])
    assert plan.dequant_fp8_select_ok([256, 352]) and not plan.dequant_fp8_select_ok([256])
    assert not plan.dequant_fp8_select_ok([256, 48]) and not plan.dequant_fp8_select_ok([8, 352])
    for dt in (torch.bfloat16, torch.float16):
        for ids in (torch.tensor([[3, 5]], device="cuda"), torch.tensor([7, 7, 0], dtype=torch.int32, device="cuda")):
            outs = [torch.full(w.shape, float("nan"), dtype=dt, device="cuda") for w, _ in (gu, dn)]
            got = plan.dequant_fp8_select(ids, [256, 352], [gu[1], dn[1]], [block, block], dt, outs=outs)
            assert all(g is o for g, o in zip(got, outs))
            for (w, s), o in zip((gu, dn), got):
                for e, want in ref_slices(w, s, block, dt, ids).items():
                    assert torch.equal(bits(o[e]), bits(want)), (block, dt, e)
    plan.check()


def test_qwen3_30b_a3b_fp8_layer_is_exact_at_1_and_64_tokens():
    """One layer of Qwen3-30B-A3B-FP8: 128 experts, gate_up [128, 1536, 2048], down [128, 2048, 768], 128x128 blocks."""
    E, H, I = 128, 2048, 768
    g = torch.Generator("cuda").manual_seed(7)
    gu = _experts_weight("e4m3", E, 2 * I, H, 1000)
    dn = _experts_weight("e4m3", E, H, I, 2000)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w) for w, _ in (gu, dn)])
    assert plan.dequant_fp8_select_ok([H, I])
    outs = [torch.empty(w.shape, dtype=torch.bfloat16, device="cuda") for w, _ in (gu, dn)]
    for tokens in (1, 64):
        ids = torch.randint(0, E, (tokens, 8), generator=g, device="cuda")
        for o in outs:
            o.fill_(float("nan"))
        plan.dequant_fp8_select(ids, [H, I], [gu[1], dn[1]], [(128, 128)] * 2, outs=outs)
        for (w, s), o in zip((gu, dn), outs):
            for e, want in ref_slices(w, s, (128, 128), torch.bfloat16, ids).items():
                assert torch.equal(bits(o[e]), bits(want)), (tokens, e)
    plan.check()


def test_n_zero_launch_count_and_bad_ids():
    w, s = _experts_weight("e5m2", 16, 96, 512, 3)
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=16384).compress(w)])
    out = torch.full(w.shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    before = _native.launch_count()
    plan.dequant_fp8_select(torch.zeros(0, dtype=torch.int64, device="cuda"), [512], [s], [(128, 128)], outs=[out])
    assert _native.launch_count() == before and torch.isnan(out).all()
    for ids in ([0] * 5, [15] * 5, list(range(0, 15, 3)), [-1] * 5):
        before = _native.launch_count()
        plan.dequant_fp8_select(torch.tensor(ids, device="cuda"), [512], [s], [(128, 128)], outs=[out])
        assert _native.launch_count() - before == LAUNCHES, ids
        if ids[0] < 0:
            break
    with pytest.raises(IndexError):
        plan.check()
    # a bad id among good ones: the good ones are written, the bad one selects nothing
    plan2 = DecodePlan([ZipNN(input_format="torch", compression_chunk=16384).compress(w)])
    out.fill_(float("nan"))
    plan2.dequant_fp8_select(torch.tensor([[2, -1], [16, 9]], device="cuda"), [512], [s], [(128, 128)], outs=[out])
    with pytest.raises(IndexError):
        plan2.check()
    wb = written_bytes(w.numel(), 16384, 16, [2, 9]).reshape(16, -1)
    ref = R.dequantize_fp8(w, s, (128, 128), torch.bfloat16)
    for e in range(16):
        if wb[e].any():
            m = torch.from_numpy(wb[e]).cuda().reshape(96, 512)
            assert torch.equal(bits(out[e])[m], bits(ref[e])[m]), e
        assert torch.isnan(out[e][~torch.from_numpy(wb[e]).cuda().reshape(96, 512)]).all(), e


def test_graph_capture_replays_with_new_ids_and_a_new_scale():
    E = 16
    gu = _experts_weight("e4m3", E, 704, 256, 11)
    dn = _experts_weight("e4m3", E, 256, 352, 31)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w) for w, _ in (gu, dn)])
    scales = [gu[1].clone(), dn[1].clone()]
    outs = [torch.empty(w.shape, dtype=torch.bfloat16, device="cuda") for w, _ in (gu, dn)]
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    scratch = torch.empty(plan.select_scratch_bytes(), dtype=torch.uint8, device="cuda")
    run = lambda: plan.dequant_fp8_select(ids, [256, 352], scales, [(128, 128)] * 2, outs=outs, scratch=scratch)  # noqa: E731
    run()   # outside the capture: the first call reads the chunk modes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    for r in range(3):
        ids.copy_(torch.randint(0, E, (4,), device="cuda"))
        scales[0].copy_(gu[1] * (r + 1.5))
        for o in outs:
            o.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        replayed = [o.clone() for o in outs]
        eager = [torch.full_like(o, float("nan")) for o in outs]
        plan.dequant_fp8_select(ids, [256, 352], scales, [(128, 128)] * 2, outs=eager)
        for a, b, (w, _), s in zip(replayed, eager, (gu, dn), scales):
            assert torch.equal(bits(a), bits(b)), r
            for e, want in ref_slices(w, s, (128, 128), torch.bfloat16, ids).items():
                assert torch.equal(bits(a[e]), bits(want)), (r, e)
    plan.check()


def test_two_item_plan_interleaves_with_run_run_select_dequant_fp8_and_matvec_fp8():
    E = 8
    gu = _experts_weight("e4m3", E, 96, 512, 5)
    dn = _experts_weight("e4m3", E, 512, 48, 7)
    tensors = [w for w, _ in (gu, dn)]
    plan = DecodePlan([ZipNN(input_format="torch", compression_chunk=ch).compress(w) for w, ch in zip(tensors, (8192, 131072))])
    need = max(plan.select_scratch_bytes(), plan.matvec_fp8_scratch_bytes(0, 512, 1))
    shared = torch.empty(need, dtype=torch.uint8, device="cuda")
    dense = [w.view(torch.uint8).reshape(E, -1) for w in tensors]
    x = torch.randn(1, 512, device="cuda").to(torch.bfloat16)
    flat_scale = gu[1].reshape(E * 1, 4)   # gate_up: 96 rows per expert in one 128-row block -> the 2-D grid of [768, 512] by (96, 128)
    y0 = plan.matvec_fp8(0, x, flat_scale, (96, 128))
    for step in range(6):
        ids = torch.randint(0, E, (3, 2), device="cuda", dtype=torch.int32 if step % 2 else torch.int64)
        outs = plan.dequant_fp8_select(ids, [512, 48], [gu[1], dn[1]], [(128, 128)] * 2, scratch=shared)
        for (w, s), o in zip((gu, dn), outs):
            for e, want in ref_slices(w, s, (128, 128), torch.bfloat16, ids).items():
                assert torch.equal(bits(o[e]), bits(want)), step
        sel = ids.reshape(-1).unique()
        coded = plan.run_select(ids, scratch=shared)
        for o, d in zip(coded, dense):
            assert torch.equal(o.view(torch.uint8).reshape(E, -1)[sel], d[sel]), step
        assert torch.equal(plan.matvec_fp8(0, x, flat_scale, (96, 128), scratch=shared), y0), step
        whole = plan.dequant_fp8(0, 512, flat_scale, (96, 128))
        assert torch.equal(bits(whole), bits(R.dequantize_fp8(tensors[0], gu[1], (128, 128), torch.bfloat16).reshape(-1, 512)))
        if step % 3 == 2:
            for o, d in zip(plan.run(), dense):
                assert torch.equal(o.view(torch.uint8).reshape(E, -1), d)
    plan.check()


def test_host_rejections_launch_nothing():
    E = 4
    w, s = _experts_weight("e4m3", E, 64, 1024, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    ref = plan._ref
    out = torch.full(w.shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(plan.select_scratch_bytes(), dtype=torch.uint8, device="cuda")
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    L = _native.lib()
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    good = dict(plan=ref, rows=E, ids=ids.data_ptr(), n=4, ib=8, fmt=0, odt=0, n_items=1, inf=1024, scale=s.data_ptr(), bn=128, bk=128,
                out=out.data_ptr(), items=True, scratch=scratch.data_ptr(), sb=scratch.numel())
    bad = [("id bytes 2", dict(ib=2), A), ("rows 0", dict(rows=0), A), ("rows not dividing", dict(rows=3), A),
           ("rows whose slices are not whole rows", dict(rows=E * 64 * 2), A), ("null ids", dict(ids=None), A),
           ("misaligned ids", dict(ids=ids.data_ptr() + 4), A), ("null scratch", dict(scratch=None), A),
           ("misaligned scratch", dict(scratch=scratch.data_ptr() + 16), A), ("small scratch", dict(sb=scratch.numel() - 1), A),
           ("format 2", dict(fmt=2), A), ("out dtype fp32", dict(odt=2), A), ("out dtype 3", dict(odt=3), A), ("in 0", dict(inf=0), A),
           ("in not dividing", dict(inf=4112), A), ("null out", dict(out=None), A), ("out alignment 8", dict(out=out.data_ptr() + 8), A),
           ("null scale", dict(scale=None), A), ("scale alignment", dict(scale=s.data_ptr() + 2), A), ("block rows 0", dict(bn=0), A),
           ("block cols 8", dict(bk=8), A), ("n_items 0", dict(n_items=0), A), ("n_items 2", dict(n_items=2), A),
           ("null items", dict(items=False), A), ("null plan", dict(plan=None), A), ("rows of 8 bytes", dict(inf=8), U)]
    for name, kw, want in bad:
        a = dict(good)
        a.update(kw)
        arr = items([(a["inf"], a["scale"], a["bn"], a["bk"], a["out"])] * 2) if a["items"] else None
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_dequant_fp8_select(a["plan"], a["rows"], a["ids"], a["n"], a["ib"], a["fmt"], a["odt"], a["n_items"],
                                                         arr, a["scratch"], a["sb"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    # a bf16 item, a plain (incompressible) fp8 item, a plan of five items, a box-free plan without a segment index
    other = DecodePlan([ZipNN(input_format="torch").compress((torch.randn(E, 64, 1024, device="cuda") * 0.02).to(torch.bfloat16))])
    raw = torch.randint(0, 256, (E * 64 * 1024,), dtype=torch.uint8, device="cuda")
    raw[(raw & 0x7F) == 0x7F] = 0
    pl = DecodePlan([ZipNN(input_format="torch").compress(raw.view(torch.float8_e4m3fn).view(E, 64, 1024))])
    five = DecodePlan([ZipNN(input_format="torch").compress(w) for _ in range(5)])
    for p_, n_items in ((other, 1), (pl, 1), (five, 5)):
        sc = torch.empty(p_.select_scratch_bytes(), dtype=torch.uint8, device="cuda")
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_dequant_fp8_select(p_._ref, E, ids.data_ptr(), 4, 8, 0, 0, n_items,
                                                         items([(1024, s, 128, 128, out.data_ptr())] * n_items), sc.data_ptr(), sc.numel(), _st())
        assert rc == U and _native.launch_count() == before
        assert not p_.dequant_fp8_select_ok([1024] * n_items)
    # Python-side refusals
    before = _native.launch_count()
    for kw, what in ((dict(block=None), "a grid scale without block"), (dict(block=(128, 8)), "bk 8"), (dict(block=(32, 128)), "another grid"),
                     (dict(scale=s.double()), "fp64 scale"), (dict(scale=s[:, :, :1].expand(E, 1, 8)), "non-contiguous scale"),
                     (dict(dtype=torch.float32), "fp32 out"), (dict(out=out.float()), "fp32 out tensor"), (dict(out=out[:, :32]), "wrong shape"),
                     (dict(out=out.view(-1)), "flat out"), (dict(inf=4112), "in not dividing"), (dict(inf=8), "8-byte rows"),
                     (dict(ids=ids.cpu()), "CPU ids"), (dict(ids=ids.float()), "float ids")):
        a = dict(inf=1024, scale=s, block=(128, 128), dtype=torch.bfloat16, out=None, ids=ids)
        a.update(kw)
        with pytest.raises(ValueError):
            plan.dequant_fp8_select(a["ids"], [a["inf"]], [a["scale"]], [a["block"]], a["dtype"], outs=None if a["out"] is None else [a["out"]])
    assert _native.launch_count() == before and torch.isnan(out).all()


def test_corrupted_fp8_streams_are_refused():
    """Every mutant of the fp8 base of corrupt_streams.py: a plan whose create fails is refused (E_ARG, nothing launched),
    as by every other entry point; one that creates is refused too (E_UNSUPPORTED: its last chunk is not fused), and
    `status` keeps the verdict's."""
    import test_corrupt_streams_gpu as T
    b = CS.bases()["fp8_g1"]
    assert b.pr["mode"][-1] != "fused"
    L = _native.lib()
    sc = torch.ones(1, device="cuda")
    y = torch.full((b.orig,), float("nan"), dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty(T.PAD + b.orig + T.PAD, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    n = 0
    for m, v in T.cases("fp8_g1"):
        body = torch.from_numpy(m.body).cuda()
        out.fill_(T.CANARY)
        rc, plan, keep = T._plan_create(b, body.data_ptr(), m.body.size, out[T.PAD:])
        assert rc == T.STATUS[v.status], (m.id, rc, v.status)
        p = C.byref(plan)
        before = _native.launch_count()
        for inf in (8, 16):
            got = L.zipnn_b200_decode_plan_dequant_fp8_select(p, 1, ids.data_ptr(), 1, 8, 0, 0, 1, items([(inf, sc, 1, 16, y.data_ptr())]),
                                                              scratch.data_ptr(), scratch.numel(), _st())
            assert got in ((_native.E_ARG,) if rc else (_native.E_ARG, _native.E_UNSUPPORTED)), (m.id, got)
        assert _native.launch_count() == before, m.id
        if not rc:
            assert torch.equal(out[T.PAD: T.PAD + b.orig], torch.from_numpy(v.data).cuda()), m.id
            assert L.zipnn_b200_decode_plan_status(p, _st()) == 0, m.id
            n += 1
    assert torch.all(torch.isnan(y))
    assert n > 0


# ------------------------------------------------------------------ resident fp8 MoE models
def _tiny(which):
    import transformers as tf
    common = dict(hidden_size=256, intermediate_size=352, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                  num_hidden_layers=2, vocab_size=512)
    if which == "mixtral":
        return tf.MixtralForCausalLM, tf.MixtralConfig(num_local_experts=8, num_experts_per_tok=2, **common)
    return tf.Qwen3MoeForCausalLM, tf.Qwen3MoeConfig(num_experts=16, num_experts_per_tok=4, moe_intermediate_size=352,
                                                      decoder_sparse_step=1, mlp_only_layers=[], **common)


def tiny_fp8_moe(which, seed=0, constant=False):
    """transformers' tiny Mixtral / Qwen3-MoE on the GPU, bf16, every linear an FP8Linear and every experts module an
    FP8Experts, quantized per 128x128 block (layers[1]'s experts one scale per expert); constant=True: layers[1]'s
    down_proj experts are one value (no coded bitstream: dequant_fp8_select_ok refuses the plan)."""
    import transformers as tf
    from transformers.integrations.finegrained_fp8 import replace_with_fp8_linear
    pytest.importorskip("transformers")
    cls, cfg = _tiny(which)
    torch.manual_seed(seed)
    m = cls(cfg).to(torch.bfloat16)
    m = replace_with_fp8_linear(m, quantization_config=tf.FineGrainedFP8Config(weight_block_size=(128, 128)), pre_quantized=True)
    k = 0
    for name, mod in m.named_modules():
        if type(mod).__name__ == "FP8Linear":
            wq, scale = _quantized("e4m3", mod.out_features, mod.in_features, 100 * seed + k)
            mod.weight = torch.nn.Parameter(wq, requires_grad=False)
            mod.weight_scale_inv = torch.nn.Parameter(scale, requires_grad=False)
            k += 1
        elif type(mod).__name__ == "FP8Experts":
            block = None if name.startswith("model.layers.1.") else (128, 128)
            mod.block_size = block
            for pname in ("gate_up_proj", "down_proj"):
                E, out, inn = mod._parameters[pname].shape
                wq, scale = _experts_weight("e4m3", E, out, inn, 100 * seed + 10 * k, block)
                if constant and block is None and pname == "down_proj":
                    wq = torch.full_like(wq, 0.5)
                setattr(mod, pname, torch.nn.Parameter(wq, requires_grad=False))
                setattr(mod, pname + "_scale_inv", torch.nn.Parameter(scale, requires_grad=False))
                k += 1
    m = m.cuda().eval()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _impl(mod):
    from transformers.integrations.moe import ALL_EXPERTS_FUNCTIONS
    name = mod.config._experts_implementation
    return inspect.unwrap(type(mod).forward) if name == "eager" else ALL_EXPERTS_FUNCTIONS[name]


def reference(m):
    """A copy of `m` whose experts hold torch-dequantized bf16 weights and run transformers' bf16 implementation of
    `config._experts_implementation`, and whose FP8Linears are compressed as fp8=True, matvec=8 compresses them."""
    ref = copy.deepcopy(m)
    lins = []
    for mod in ref.modules():
        if type(mod).__name__ == "FP8Experts":
            for pname in ("gate_up_proj", "down_proj"):
                w = R.dequantize_fp8(getattr(mod, pname), getattr(mod, pname + "_scale_inv"), mod.block_size, torch.bfloat16)
                setattr(mod, pname, torch.nn.Parameter(w, requires_grad=False))
            mod.forward = (lambda mod: lambda *a, **k: _impl(mod)(mod, *a, **k))(mod)
        elif type(mod).__name__ == "FP8Linear":
            lins.append(mod)
    compress_module(ref, modules=lins, fp8=True, matvec=8)
    return ref


def _nan_forward(model, ids):
    for e in getattr(model, R._ATTR).entries:
        e.plan._out.fill_(0xFF)
    with torch.no_grad():
        return model(ids, use_cache=False).logits


IMPLS = ("eager", "batched_mm", "grouped_mm")


def check_logits(m, ref, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    for n in (1, 16):
        ids = torch.randint(0, 512, (1, n), generator=g, device="cuda")
        for impl in IMPLS:
            m.config._experts_implementation = ref.config._experts_implementation = impl
            want = _nan_forward(ref, ids)
            got = _nan_forward(m, ids)
            assert torch.equal(got, want), (impl, n)


def dense_state(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def raw(t):
    return t.reshape(-1).view(torch.uint8)


@pytest.mark.parametrize("which", ("qwen3", "mixtral"))
def test_resident_fp8_moe_logits_equal_the_dequantized_reference(which):
    torch.cuda.reset_peak_memory_stats()
    m = tiny_fp8_moe(which, 1, constant=True)
    ref = reference(m)
    before = dense_state(m)
    experts = [x for x in m.modules() if type(x).__name__ == "FP8Experts"]
    lins = [x for x in m.modules() if type(x).__name__ == "FP8Linear"]
    need = max(2 * (x.gate_up_proj.numel() + x.down_proj.numel()) for x in experts)
    rep = compress_module(m, fp8=True, experts=True, matvec=8)
    state = getattr(m, R._ATTR)
    mode = {id(e.module): e.mode for e in state.entries}
    assert [mode[id(x)] for x in experts] == ["fp8_experts", "fp8_experts_torch"], "the constant weight takes the fallback"
    assert rep["fp8_experts_modules"] == 2 and rep["experts_scratch_bytes"] > 0 and rep["fp8_modules"] == len(lins)
    assert rep["out_bytes"] >= need
    for x in experts:   # only the fp8 weights are compressed
        assert "gate_up_proj" not in x._parameters and "gate_up_proj_scale_inv" in x._parameters
    calls = {"select": 0}
    plan = next(e.plan for e in state.entries if e.module is experts[0])
    real = plan.dequant_fp8_select
    plan.dequant_fp8_select = lambda *a, **k: (calls.__setitem__("select", calls["select"] + 1), real(*a, **k))[1]
    check_logits(m, ref, 2)
    assert calls["select"] == 2 * len(IMPLS)
    # module calls, positional and by keyword; ids on the CPU take the whole decode and torch's dequantize, and give
    # what the reference gives them (an implementation that refuses CPU ids refuses them in both)
    x = torch.randn(5, 256, device="cuda").to(torch.bfloat16)
    idx = torch.randint(0, experts[0].num_experts, (5, 2), device="cuda")
    wts = torch.rand(5, 2, device="cuda").to(torch.bfloat16)
    rx = next(y for y in ref.modules() if type(y).__name__ == "FP8Experts")
    with torch.no_grad():
        for impl in IMPLS:
            m.config._experts_implementation = ref.config._experts_implementation = impl
            want = rx(x, idx, wts)
            assert torch.equal(experts[0](x, idx, wts), want), impl
            assert torch.equal(experts[0](hidden_states=x, top_k_index=idx, top_k_weights=wts), want), impl
            try:
                want_cpu = rx(x, idx.cpu(), wts)
            except Exception as err:   # noqa: BLE001  (transformers' own behaviour for CPU ids)
                with pytest.raises(type(err)):
                    experts[0](x, idx.cpu(), wts)
            else:
                assert torch.equal(experts[0](x, idx.cpu(), wts), want_cpu), impl
    assert calls["select"] == 2 * len(IMPLS) + 2 * len(IMPLS)
    with pytest.raises(RuntimeError, match="no_grad"):
        experts[0](x, idx, wts)
    assert torch.cuda.max_memory_allocated() < 16 << 30
    decompress_module(m)
    after = dense_state(m)
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(raw(after[k]), raw(before[k])), k
    assert not any("forward" in x.__dict__ for x in experts)


def test_load_module_fp8_moe_from_safetensors_and_znn(tmp_path):
    src = tiny_fp8_moe("qwen3", 3)
    ref = reference(src)
    sd = {k: v.contiguous() for k, v in dense_state(src).items()}
    want_rep = compress_module(tiny_fp8_moe("qwen3", 3), fp8=True, experts=True, matvec=8)
    plain = str(tmp_path / "fp8_moe.safetensors")
    save_file(sd, plain)
    a = tiny_fp8_moe("qwen3", 4)   # other values: every one must come from the file
    assert load_module(a, plain, fp8=True, experts=True, matvec=8) == want_rep
    check_logits(a, ref, 5)
    znn = str(tmp_path / "fp8_moe.znn.safetensors")
    save_module(a, znn)
    b = tiny_fp8_moe("qwen3", 5)
    assert load_module(b, znn, fp8=True, experts=True, matvec=8) == want_rep
    check_logits(b, ref, 6)
    decompress_module(b)
    for k, v in dense_state(b).items():
        assert torch.equal(raw(v), raw(sd[k])), k
