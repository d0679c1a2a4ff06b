"""The one-launch, CTA-budgeted replay of a decode plan (zipnn_b200_decode_plan_run_shifted, DecodePlan.run_into)
against the oracle.

The harness of test_decode_plan_gpu (Item: a device body and a canary-padded output) is laid out twice in one arena:
region A is where the plan is created, region B the same layout `shift` bytes further.  Every run into B must write
the oracle's bytes there, touch no canary and leave region A as it was; the same holds for a run back into A.  Each
set of items runs with CTA budgets of 1, 2, 3, 7 and the whole device, one after another (so the run's counters must
reset after every run).
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import test_decode_plan_gpu as DP
import test_decoder_tables_gpu as D
from oracle import oracle as O
import chunk_settings as CS
from zipnn_b200 import DecodePlan, ZipNN, _native

pytestmark = pytest.mark.gpu

CTAS = (1, 2, 3, 7, 0)
PAD, CANARY = DP.PAD, DP.CANARY


def run_shifted(plan, shift, ctas, stream=None):
    st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    return _native.lib().zipnn_b200_decode_plan_run_shifted(C.byref(plan), shift, ctas, st)


def laid_out(items):
    """Items in region A of one arena (256-byte aligned slots) -> (twins in region B, shift, arena)."""
    offs, at = [], 0
    for it in items:
        offs.append(at)
        at = (at + PAD + it.want.size + PAD + 255) // 256 * 256
    arena = torch.full((2 * at,), CANARY, dtype=torch.uint8, device="cuda")
    twins = []
    for it, o in zip(items, offs):
        it.out = arena[o: o + PAD + it.want.size + PAD]
        t = copy.copy(it)
        t.out = arena[at + o: at + o + PAD + it.want.size + PAD]
        twins.append(t)
    return twins, at, arena


def check_run_into(items, ctas_list=CTAS):
    twins, shift, _ = laid_out(items)
    p = DP.Plan(items)
    assert p.rc == 0, [it.name for it in items]
    for it in items:
        it.check("create")
    for ctas in ctas_list:
        for t in twins:
            t.scribble()
        assert run_shifted(p.plan, shift, ctas) == 0
        assert p.status() == 0
        for t in twins:
            t.check(f"run into B, {ctas} CTAs")
        for it in items:
            it.check(f"region A after a run into B, {ctas} CTAs")
    # back into A (shift 0), then B again: alternating buffers
    for it in items:
        it.scribble()
    assert run_shifted(p.plan, 0, 3) == 0
    for t in twins:
        t.scribble()
    assert run_shifted(p.plan, shift, 0) == 0
    assert p.status() == 0
    for it, t in zip(items, twins):
        it.check("run into A")
        t.check("run into B after A")
    return p


@pytest.mark.parametrize("G", [1, 2, 4])
def test_chunk_settings(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    check_run_into(DP._settings_items(G))


def test_ring_fallback_and_misaligned_guesses(monkeypatch):
    DP._set_env(monkeypatch, {})
    items = [DP._case_item(cs) for cs in D.ring_cases()]
    for fam, L in (("eq4", 2), ("eq16", 4), ("eq64", 6)):
        n = D._misaligned_len(L, 100000)
        items.append(DP._case_item(D.planes_case(f"fixed_{fam}", "fp8", 131072, [fam, fam], seed=60 + L, last=n)))
    check_run_into(items)


@pytest.mark.parametrize("dtype", ["bf16", "fp32", "fp16", "fp8"])
def test_tail_pool_and_tables(dtype, monkeypatch):
    DP._set_env(monkeypatch, {})
    case, _ = D.warp_mix_case(dtype)
    chunk = 131072 if dtype == "fp8" else 262144
    logs = D.planes_case(f"logs_{dtype}", dtype, chunk, ["eq2", "eq4", "eq8", "eq16", "zipf256", "heavy256"], seed=70)
    check_run_into([DP._case_item(case), DP._case_item(logs)])


def test_crafted_tables(monkeypatch):
    DP._set_env(monkeypatch, {})
    rng = np.random.default_rng(80)
    blocks = []
    for c in range(24):
        max_len = int(rng.integers(1, 12))
        blocks.append(D.P.kraft_lengths(rng, int(rng.integers(2, min(120, 1 << max_len) + 1)), max_len))
    check_run_into([DP._case_item(D.crafted_case("crafted_bf16", "bf16", 4096, blocks, seed=81)),
                    DP._case_item(D.crafted_case("crafted_fp16", "fp16", 4096, blocks, seed=83))])


def test_overflow_and_special_tensors(monkeypatch):
    """General chunks past the 64 pool slots (the overflow path: with 1, 2, 3 and 7 CTAs fewer CTAs than overflow
    slots take them), raw-only, RLE-only and empty tensors."""
    DP._set_env(monkeypatch, {})
    tops = ["eq128" if c % 3 == 1 else "geo5" for c in range(600)]
    over = D.planes_case("overflow_bf16", "bf16", 4096, tops, seed=12)
    fp32 = D.planes_case("fp32_general", "fp32", 4096, ["geo5"] * 100, seed=14, last=2052,
                         side=lambda c, g: "geo5" if g == 2 else "raw")
    items = [DP._case_item(over), DP._case_item(fp32)]
    rng = np.random.default_rng(5)
    for name, data in (("raw", rng.integers(0, 256, 100000, dtype=np.uint8)), ("rle", np.zeros(65536, np.uint8))):
        stream = O.zipnn_compress(CS.header(), data, 2, 1, 10, 4096, 0.95, threads=4)
        items.append(DP.Item(name, stream[32:], 2, 1, 4096, data.size, data))
    items.append(DP.Item("empty", b"", 2, 1, 4096, 0, np.zeros(0, np.uint8)))
    check_run_into(items)


def test_pieces_and_boxes(monkeypatch):
    DP._set_env(monkeypatch, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "5"})
    case = D.planes_case("pieces_bf16", "bf16", 4096, ["geo5"] * 37, seed=3, last=1000)
    box32 = D.planes_case("box_fp32", "fp32", 4096, ["geo5"] * 20, seed=8)
    check_run_into([DP._case_item(case)] + [DP._case_item(case, box) for box in D.slice_boxes(case)]
                   + [DP._case_item(box32, box) for box in D.slice_boxes(box32)])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2])
def test_every_dtype_through_decode_plan(dtype):
    torch.manual_seed(1)
    ts = [(torch.randn(1000, 700) * 0.02).to(dtype).cuda(), (torch.randn(333, 9) * 0.02).to(dtype).cuda()]
    z = ZipNN(input_format="torch")
    plan = DecodePlan([z.compress(t) for t in ts])
    bufs = [torch.full((plan.nbytes["out"] + 32,), CANARY, dtype=torch.uint8, device="cuda") for _ in range(2)]
    for r in range(4):
        buf = bufs[r % 2][16: 16 + plan.nbytes["out"]]
        buf.fill_(0)
        outs = plan.run_into(buf, max_ctas=(0, 5)[r % 2])
        torch.cuda.synchronize()
        assert all(torch.equal(o.view(torch.uint8), t.view(torch.uint8)) for o, t in zip(outs, ts))
        assert all(o.data_ptr() - buf.data_ptr() == p.data_ptr() - plan._out.data_ptr() for o, p in zip(outs, plan.outputs))
        assert torch.all(bufs[r % 2][:16] == CANARY) and torch.all(bufs[r % 2][16 + plan.nbytes["out"]:] == CANARY)
    plan.check()


def test_run_concurrent_with_matmuls():
    """A run on a side stream of a few CTAs next to a matmul loop on the current stream."""
    torch.manual_seed(2)
    ts = [(torch.randn(4096, 1024) * 0.02).to(torch.bfloat16).cuda() for _ in range(3)]
    z = ZipNN(input_format="torch")
    plan = DecodePlan([z.compress(t) for t in ts])
    buf = torch.empty(plan.nbytes["out"], dtype=torch.uint8, device="cuda")
    a = torch.randn(4096, 4096, device="cuda", dtype=torch.bfloat16)
    want = a @ a
    side = torch.cuda.Stream()
    for ctas in (4, 16, 0):
        buf.zero_()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            outs = plan.run_into(buf, max_ctas=ctas)
        ys = [a @ a for _ in range(8)]
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        assert all(torch.equal(o, t) for o, t in zip(outs, ts))
        assert all(torch.equal(y, want) for y in ys)
    plan.check()


def test_graph_with_runs_into_both_buffers():
    torch.manual_seed(3)
    ts = [(torch.randn(3, 700, 512) * 0.02).to(torch.bfloat16).cuda(), (torch.randn(5000) * 0.02).cuda()]
    z = ZipNN(input_format="torch")
    plan = DecodePlan([z.compress(t) for t in ts])
    b0, b1 = (torch.empty(plan.nbytes["out"], dtype=torch.uint8, device="cuda") for _ in range(2))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run_into(b0, 7)   # (warm-up on a side stream, as torch.cuda.graph wants)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        o0 = plan.run_into(b0, 7)
        o1 = plan.run_into(b1, 0)
    for _ in range(2):
        b0.zero_()
        b1.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(o, t) for o, t in zip(o0, ts)) and all(torch.equal(o, t) for o, t in zip(o1, ts))
    plan.check()


def test_errors_and_launch_count(monkeypatch):
    DP._set_env(monkeypatch, {})
    x = (torch.randn(2000, 300) * 0.02).to(torch.bfloat16).cuda()
    z = ZipNN(input_format="torch")
    plan = DecodePlan([z.compress(x)])
    buf = torch.empty(plan.nbytes["out"] + 64, dtype=torch.uint8, device="cuda")
    assert run_shifted(plan._plan, 8, 0) == _native.E_ARG
    assert run_shifted(plan._plan, -24, 0) == _native.E_ARG
    with pytest.raises(ValueError):
        plan.run_into(buf[8:])                      # unaligned
    with pytest.raises(ValueError):
        plan.run_into(buf[: plan.nbytes["out"] - 16])   # too short
    with pytest.raises(ValueError):
        plan.run_into(buf.view(torch.int8))
    before = _native.launch_count()
    for ctas in (1, 0, 3):
        plan.run_into(buf[16:], ctas)
    assert _native.launch_count() - before == 3
    torch.cuda.synchronize()
    assert torch.equal(buf[16: 16 + x.numel() * 2].view(torch.bfloat16).view(x.shape), x)
    plan.check()
    monkeypatch.setenv("ZIPNN_B200_PLAN_REPLAY", "0")
    noidx = DecodePlan([z.compress(x)])
    assert run_shifted(noidx._plan, 0, 0) == _native.E_UNSUPPORTED
