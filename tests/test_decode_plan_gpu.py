"""Decode plans (zipnn_b200_decode_plan_*, zipnn_b200.DecodePlan) against the oracle.

Every stream is decoded by the plan's create, then the outputs are overwritten with a canary and the plan is run
twice more: each time every output must be the oracle's bytes and the bytes around it untouched.  The inputs are the
chunk-size / threshold settings of tests/chunk_settings.py and the decoder-table cases of
test_decoder_tables_gpu.py (ring-fallback bitstreams, fixed-length codes with misaligned segment guesses, tail-pool
overflow, crafted tables), plus raw / RLE-only / empty tensors, general chunks past the 64 pool slots, items split
into pieces, and boxes, which must equal zipnn_b200_decompress_slices.

Create records the start and symbol count of every segment of the per-bitstream-CTA decoder (record mode); runs
decode each segment from its recorded start (replay mode).  For every plan the test reads the segment index back:
its size is 8 KiB per coded item of the type rows, its symbol counts add up to the coded planes' bytes (ring-fallback
bitstreams included), and it holds empty segments.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import chunk_settings as CS
import test_decoder_tables_gpu as D
from oracle import oracle as O
from zipnn_b200 import DecodePlan, ZipNN, _native

pytestmark = pytest.mark.gpu

PAD, CANARY = 64, 0xA5
RUN_LAUNCHES = 4   # sync decode, regroup, overflow, error OR
SEG_PER_ITEM = 4 * 256 * 8   # index bytes per coded item: 4 bitstreams x 256 threads x (u32 start, u32 count)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Item:
    """A body on the device and a canary-padded output for one slice item."""

    def __init__(self, name, body, G, bits, chunk, orig, want, box=None):
        self.name, self.G, self.bits, self.chunk, self.orig = name, G, bits, chunk, orig
        self.bm = 220 if G == 4 else 10
        self.dbody = torch.from_numpy(np.ascontiguousarray(body)).cuda() if len(body) else torch.zeros(16, dtype=torch.uint8, device="cuda")
        self.body_len = len(body)
        self.box = box or (0, 1, orig, orig)
        self.want = want
        self.out = torch.full((PAD + want.size + PAD,), CANARY, dtype=torch.uint8, device="cuda")

    def fill(self, it):
        base, rows, pitch, length = self.box
        it.d_body, it.body_len = self.dbody.data_ptr(), self.body_len
        it.num_buf, it.bits_mode, it.bytes_mode = self.G, self.bits, self.bm
        it.chunk, it.orig = self.chunk, self.orig
        it.base, it.rows, it.pitch, it.len = base, rows, pitch, length
        it.d_out = self.out[PAD:].data_ptr()

    def coded_items(self):
        """Type-1 entries of the stream's type rows: the coded items the plan sizes its index by."""
        if not self.orig:
            return 0
        K = -(-self.orig // self.chunk)
        return int(np.count_nonzero(self.dbody[: self.G * K].cpu().numpy() == 1))

    def coded_symbols(self):
        """-> (bytes of the Huffman-coded planes, whether some of them may be decoded by the overflow kernel).  The
        recorded segments of a whole tensor add up to the first unless general chunks outnumber the 64 pool slots:
        those past the pool go to k_decode_overflow, which has no segments (which ones is decided at run time)."""
        if not self.orig:
            return 0, False
        pr = D.P.predict(self.dbody[: self.body_len].cpu().numpy(), self.G, self.bits, self.chunk, self.orig)
        K = pr["K"]
        general = pr["mode"].count("general")
        return sum(it.dec_len for row in pr["items"] for it in row if it.kind == "huf"), K > 64 and general > 64

    def check(self, what):
        host = self.out.cpu().numpy()
        n = self.want.size
        assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY), f"{self.name}: {what} wrote outside its output"
        got = host[PAD: PAD + n]
        assert np.array_equal(got, self.want), (self.name, what, int(np.argmax(got != self.want)))

    def scribble(self):
        self.out[PAD: PAD + self.want.size].fill_(CANARY ^ 0xFF)


def _array(items):
    arr = (_native.SliceItem * max(1, len(items)))()
    for a, it in zip(arr, items):
        it.fill(a)
    return arr


class Plan:
    def __init__(self, items, scratch=None):
        L = _native.lib()
        self.items = items
        self.arr = _array(items)
        pb, sb = C.c_size_t(0), C.c_size_t(0)
        assert L.zipnn_b200_decode_plan_size(self.arr, len(items), None, C.byref(pb), C.byref(sb)) == 0
        self.plan_bytes, self.scratch_bytes = pb.value, sb.value
        self.meta = torch.empty(pb.value, dtype=torch.uint8, device="cuda")
        self.scratch = scratch if scratch is not None else torch.empty(max(1, sb.value), dtype=torch.uint8, device="cuda")
        self.plan = _native.DecodePlanStruct()
        self.rc = L.zipnn_b200_decode_plan_create(self.arr, len(items), self.meta.data_ptr(), pb.value, self.scratch.data_ptr(),
                                                  sb.value, C.byref(self.plan), _stream())

    def run(self):
        return _native.lib().zipnn_b200_decode_plan_run(C.byref(self.plan), _stream())

    def status(self):
        return _native.lib().zipnn_b200_decode_plan_status(C.byref(self.plan), _stream())

    def index(self):
        """-> (index bytes, coded items, the index as (start, count) rows)."""
        ib, ci = C.c_size_t(0), C.c_size_t(0)
        assert _native.lib().zipnn_b200_decode_plan_index(C.byref(self.plan), C.byref(ib), C.byref(ci)) == 0
        raw = self.meta[self.plan_bytes - ib.value:].cpu().numpy()
        return ib.value, ci.value, raw.view(np.uint32).reshape(-1, 2)


def check_plan(items, runs=2, whole=True, replay=True):
    """create, then `runs` runs after overwriting every output: all exact, nothing outside touched.  The segment
    index: 8 KiB per coded item; with whole tensors only (whole), its counts add up to the coded planes' bytes."""
    p = Plan(items)
    assert p.rc == 0, [it.name for it in items]
    for it in items:
        it.check("create")
    ib, ci, seg = p.index()
    assert ib == ci * SEG_PER_ITEM
    if not replay:
        assert ib == 0
    elif whole:
        assert ci == sum(it.coded_items() for it in items)
        sym = [it.coded_symbols() for it in items]
        got, want = int(seg[:, 1].sum()), sum(n for n, _ in sym)
        assert got == want if not any(o for _, o in sym) else 0 < got < want, (got, want)
    else:
        assert ci >= sum(it.coded_items() for it in items if it.box == (0, 1, it.orig, it.orig))
    p.seg = seg
    for r in range(runs):
        for it in items:
            it.scribble()
        assert p.run() == 0
        assert p.status() == 0
        for it in items:
            it.check(f"run {r}")
    return p


def _set_env(monkeypatch, env):
    for k in ("ZIPNN_B200_SLICE_PIECE_CHUNKS", "ZIPNN_B200_SYNC_MAX", "ZIPNN_B200_PLAN_REPLAY"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ------------------------------------------------------------------ every chunk size and threshold
def _settings_items(G):
    items = []
    for c in CS.settings_inputs(big=False):
        if c["G"] != G:
            continue
        stream = O.zipnn_compress(CS.header(), c["data"], c["G"], c["bits"], 220 if G == 4 else 10, c["chunk"], c["thr"], threads=8)
        items.append(Item(c["name"], stream[32:], c["G"], c["bits"], c["chunk"], c["data"].size, c["data"]))
    return items


@pytest.mark.parametrize("G", [1, 2, 4])
def test_chunk_settings(G, monkeypatch):
    """All settings of one byte-group count in one plan (items of every chunk size, raw / RLE / coded planes)."""
    _set_env(monkeypatch, {})
    items = _settings_items(G)
    assert len(items) > 20
    check_plan(items)


# ------------------------------------------------------------------ the decoder-table cases
def _case_item(case, box=None):
    if box is None:
        return Item(case.name, case.body, case.G, case.bits, case.chunk, case.data.size, case.data)
    return Item(case.name + f"-box{box}", case.body, case.G, case.bits, case.chunk, case.data.size, D.expect_box(case, *box), box=box)


def test_ring_fallback_bitstreams(monkeypatch):
    """Bitstreams longer than the sync decoder's shared-memory copy take the per-thread rings."""
    _set_env(monkeypatch, {})
    cases = D.ring_cases()
    assert max(max(cs.pr["items"][cs.G - 1][c].s_len) for cs in cases for c in range(cs.pr["K"])) > 28 * 1024
    for cs in cases:   # (each alone: the index's counts add up to this case's coded planes)
        check_plan([_case_item(cs)])


def test_misaligned_segment_guesses(monkeypatch):
    """Fixed-length codes never resynchronise: only the round loop puts the segment starts right."""
    _set_env(monkeypatch, {})
    items = []
    for fam, L in (("eq4", 2), ("eq16", 4), ("eq64", 6)):
        n = D._misaligned_len(L, 100000)
        case = D.planes_case(f"fixed_{fam}", "fp8", 131072, [fam, fam], seed=60 + L, last=n)
        assert D.P.misaligned_sync_guesses(case.pr["items"][0][1]) == 4
        items.append(_case_item(case))
    check_plan(items)


@pytest.mark.parametrize("dtype", ["bf16", "fp32", "fp16", "fp8"])
def test_tail_pool_mixes_and_tables(dtype, monkeypatch):
    """Warp mixes that fill and overflow the fused kernel's tail pool, chunks demoted to the general path, RLE and
    raw planes, table logs 1-4 and 256-symbol alphabets."""
    _set_env(monkeypatch, {})
    case, _ = D.warp_mix_case(dtype)
    chunk = 131072 if dtype == "fp8" else 262144
    logs = D.planes_case(f"logs_{dtype}", dtype, chunk, ["eq2", "eq4", "eq8", "eq16", "zipf256", "heavy256"], seed=70)
    check_plan([_case_item(case), _case_item(logs)])


def test_crafted_tables(monkeypatch):
    _set_env(monkeypatch, {})
    rng = np.random.default_rng(80)
    blocks = []
    for c in range(24):
        max_len = int(rng.integers(1, 12))
        blocks.append(D.P.kraft_lengths(rng, int(rng.integers(2, min(120, 1 << max_len) + 1)), max_len))
    check_plan([_case_item(D.crafted_case("crafted_bf16", "bf16", 4096, blocks, seed=81)),
                _case_item(D.crafted_case("crafted_fp16", "fp16", 4096, blocks, seed=83))])


def test_general_chunks_past_the_pool_and_special_tensors(monkeypatch):
    """More general chunks than the 64 + 32 plane slots (the overflow kernel takes the rest); a ragged fp32 tensor
    whose every chunk needs scratch; raw-only, RLE-only and empty tensors."""
    _set_env(monkeypatch, {})
    tops = ["eq128" if c % 3 == 1 else "geo5" for c in range(600)]
    over = D.planes_case("overflow_bf16", "bf16", 4096, tops, seed=12)
    assert sum(1 for v in over.pr["fused"].values() if v == "demoted") > 64 + 32
    fp32 = D.planes_case("fp32_general", "fp32", 4096, ["geo5"] * 100, seed=14, last=2052,
                         side=lambda c, g: "geo5" if g == 2 else "raw")
    assert fp32.pr["mode"].count("general") > 64 + 32
    items = [_case_item(over), _case_item(fp32)]
    rng = np.random.default_rng(5)
    for name, data in (("raw", rng.integers(0, 256, 100000, dtype=np.uint8)), ("rle", np.zeros(65536, np.uint8))):
        stream = O.zipnn_compress(CS.header(), data, 2, 1, 10, 4096, 0.95, threads=4)
        items.append(Item(name, stream[32:], 2, 1, 4096, data.size, data))
    items.append(Item("empty", b"", 2, 1, 4096, 0, np.zeros(0, np.uint8)))
    check_plan(items)


def test_pieces(monkeypatch):
    """Items split into pieces (the piece limit lowered to 5 chunks), whole tensors and boxes."""
    _set_env(monkeypatch, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "5"})
    case = D.planes_case("pieces_bf16", "bf16", 4096, ["geo5"] * 37, seed=3, last=1000)
    check_plan([_case_item(case)] + [_case_item(case, box) for box in D.slice_boxes(case)], whole=False)


def test_boxes_equal_the_slice_call(monkeypatch):
    _set_env(monkeypatch, {})
    cases = [D.planes_case("box_bf16", "bf16", 4096, ["geo5"] * 30, seed=7, last=2000),
             D.planes_case("box_fp32", "fp32", 4096, ["geo5"] * 20, seed=8)] + D.ring_cases()[:1]
    items = []
    for case in cases:
        for box in D.slice_boxes(case):
            rc, want = D.decode_slice(case, *box)
            assert rc == 0
            it = _case_item(case, box)
            assert np.array_equal(it.want, want)
            items.append(it)
    check_plan(items, whole=False)


# ------------------------------------------------------------------ host-free runs
@pytest.mark.parametrize("n", [1, 10, 300])
def test_run_launch_count_is_fixed(n):
    rng = np.random.default_rng(n)
    items = []
    for i in range(n):
        data = (torch.from_numpy(rng.standard_normal(4096 + 64 * (i % 7), dtype=np.float32) * np.float32(0.02))
                .to(torch.bfloat16).view(torch.uint8).numpy())
        stream = O.zipnn_compress(CS.header(), data, 2, 1, 10, 4096, 0.95, threads=4)
        items.append(Item(f"t{i}", stream[32:], 2, 1, 4096, data.size, data))
    p = check_plan(items, runs=1)
    before = _native.launch_count()
    for _ in range(3):
        assert p.run() == 0
    assert _native.launch_count() - before == 3 * RUN_LAUNCHES
    torch.cuda.synchronize()


def test_run_in_a_cuda_graph():
    x = (torch.randn(3, 700, 512) * 0.02).to(torch.bfloat16).cuda()
    y = (torch.randn(5000) * 0.02).cuda()
    z = ZipNN(input_format="torch")
    streams = [z.compress(x), z.compress(y)]
    plan = DecodePlan(streams)
    assert torch.equal(plan.outputs[0], x) and torch.equal(plan.outputs[1], y)
    assert plan.nbytes["index"] == plan.coded_items * SEG_PER_ITEM > 0 and plan.nbytes["plan"] > plan.nbytes["index"]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run()            # (warm-up on the side stream, as torch.cuda.graph wants)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = plan.run()
    for o in outs:
        o.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(plan.outputs[0], x) and torch.equal(plan.outputs[1], y)
    plan.check()


def test_plans_sharing_scratch():
    a = [(torch.randn(4096, 300) * 0.02).to(torch.bfloat16).cuda(), (torch.randn(9000) * 0.02).cuda()]
    b = [(torch.randn(2000, 513) * 0.02).to(torch.float16).cuda()]
    z = ZipNN(input_format="torch")
    sa, sb = [z.compress(t) for t in a], [z.compress(t) for t in b]
    need = max(DecodePlan.sizes(sa)[1], DecodePlan.sizes(sb)[1])
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    pa, pb = DecodePlan(sa, scratch=scratch), DecodePlan(sb, scratch=scratch)
    for _ in range(3):
        for o in pa.outputs + pb.outputs:
            o.view(torch.uint8).fill_(0xA5)
        pa.run()
        pb.run()
        assert all(torch.equal(o, t) for o, t in zip(pa.outputs, a))
        assert all(torch.equal(o, t) for o, t in zip(pb.outputs, b))
    pa.check()
    pb.check()


# ------------------------------------------------------------------ errors
def test_errors_at_create():
    case = D.planes_case("corrupt_bf16", "bf16", 4096, ["geo5"] * 8, seed=9)
    body = case.body.copy()
    G, K = 2, 8
    body[G * K + 8 * (K + 3): G * K + 8 * (K + 4)] = 255     # a size row of group 1 far past the payload
    p = Plan([Item("corrupt", body, 2, 1, 4096, case.data.size, case.data)])
    assert p.rc == _native.E_CORRUPT
    assert p.run() == _native.E_ARG and p.status() == _native.E_ARG

    rng = np.random.default_rng(90)
    nb12 = D.P.kraft_lengths(rng, 90, 12, min_len=2)
    blocks = [None] * 6
    blocks[3] = nb12
    log12 = D.crafted_case("log12_bf16", "bf16", 4096, blocks, seed=91)
    p = Plan([_case_item(log12)])
    assert p.rc == _native.E_UNSUPPORTED
    assert p.run() == _native.E_ARG

    stream = ZipNN(input_format="torch").compress((torch.randn(5000) * 0.02).to(torch.bfloat16).cuda()).clone()
    stream[-100:] = 0
    with pytest.raises(RuntimeError):
        DecodePlan([stream])


# ------------------------------------------------------------------ the index itself
def test_index_holds_empty_segments_and_runs_read_it(monkeypatch):
    """Short bitstreams leave most of the 256 segments empty: recorded with a start and no symbols.  A run decodes
    from the index alone: with the index cleared it writes other bytes (and no byte outside the outputs)."""
    _set_env(monkeypatch, {})
    case = D.planes_case("short_bf16", "bf16", 4096, ["geo5"] * 12, seed=21)
    it = _case_item(case)
    p = check_plan([it])
    starts, counts = p.seg[:, 0], p.seg[:, 1]
    assert np.count_nonzero((starts != 0) & (counts == 0)) > np.count_nonzero(counts)
    ib, _, _ = p.index()
    p.meta[p.plan_bytes - ib:].zero_()
    it.scribble()
    assert p.run() == 0
    host = it.out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + it.want.size:] == CANARY)
    assert not np.array_equal(host[PAD: PAD + it.want.size], it.want)


def test_plans_without_index_take_the_rounds(monkeypatch):
    """ZIPNN_B200_PLAN_REPLAY=0: no index, runs in decode mode, the same bytes."""
    _set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    cases = [D.planes_case("noidx_bf16", "bf16", 4096, ["geo5"] * 20, seed=22, last=3000)] + D.ring_cases()[:1]
    check_plan([_case_item(cs) for cs in cases], replay=False)
