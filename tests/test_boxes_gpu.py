"""Boxes of decoded bytes through the per-bitstream-CTA decoder family, against the dense bytes.

A. Box geometry: the seeded boxes of test_boxes_host.py (edges of base, len, pitch and rows, the whole tensor, its
   first and last byte, empty boxes) over planes cases of G = 1, 2, 4 that hold every chunk mode and chunk sizes from
   G bytes to the default.  Every (store site, store class, chunk mode) the layouts allow is asserted to be reached.
   Each box must equal the numpy cut of the input, with every canary untouched, through
     * zipnn_b200_decompress_slices, one call per box and one call for all boxes of a stream (outputs packed back
       to back at 16-byte aligned starts, canaries in the gaps), the latter also with the piece limit lowered to
       2, 3 and 7 chunks (splits by rows, by bytes, in groups of m rows, one row at a time);
     * a decode plan over the boxes (create and two runs), and its one-launch replay at 1, 3 and all CTAs.
   The plans' segment index counts the coded items of every piece's covering chunks: it must equal the piece
   model's count, so the model splits each box the way the library does.
B. Past 4 GiB: 9 GiB bf16 and 6 GiB fp32 tensors (payload offsets past 2^32, a box base past 2^32, pieces at the
   real limit of 16384 chunks, RLE, raw and general chunks beyond 4 GiB of decoded bytes) through the slices call,
   ZipNN.decompress_slice, the batch call and a decode plan, compared on the device with the dense tensor.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import test_boxes_host as H
import test_decode_plan_gpu as DP
import test_decoder_tables_gpu as D
import test_plan_run_into_gpu as RI
from tools.stream_windows import StreamTables
from zipnn_b200 import ZipNN, _native

pytestmark = pytest.mark.gpu

PAD, CANARY = DP.PAD, DP.CANARY
GS = (1, 2, 4)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _fill(it, dbody, body_len, G, bits, bm, chunk, orig, box, out_ptr):
    it.d_body, it.body_len = dbody, body_len
    it.num_buf, it.bits_mode, it.bytes_mode = G, bits, bm
    it.chunk, it.orig = chunk, orig
    it.base, it.rows, it.pitch, it.len = box
    it.d_out = out_ptr


def _slices(arr, n, check=1):
    L = _native.lib()
    wsz = C.c_size_t(0)
    rc = L.zipnn_b200_decompress_slices_workspace_size(arr, n, C.byref(wsz))
    if rc:
        return rc
    ws = torch.empty(max(wsz.value, 256), dtype=torch.uint8, device="cuda")
    return L.zipnn_b200_decompress_slices(arr, n, ws.data_ptr(), ws.numel(), _stream(), check)


def _cases(G):
    """(case, boxes, wants) of every stream of G; asserts that the boxes reach every store site and class."""
    out, hit = [], set()
    for case in H.box_streams(G):
        boxes = H.boxes_of(case)
        for box in boxes:
            hit |= H.classify(case, box)[1]
        out.append((case, boxes, [H.expect(case, b) for b in boxes]))
    assert hit == H.ALLOWED, sorted(H.ALLOWED ^ hit)
    return out


def _coded_in_pieces(case, boxes, limit):
    """Coded items (type-1 entries) over the covering chunks of every piece: what a plan's segment index holds."""
    K = case.pr["K"]
    types = case.body[: case.G * K].reshape(case.G, K)
    return sum(int(np.count_nonzero(types[:, p.c0: p.c1] == 1)) for b in boxes for p in H.pieces_of(b, case.chunk, limit))


# ------------------------------------------------------------------ A. box geometry
@pytest.mark.parametrize("G", GS)
def test_each_box_alone(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    n = 0
    for case, boxes, wants in _cases(G):
        for box, want in zip(boxes, wants):
            rc, got = D.decode_slice(case, *box)   # (asserts the canaries on both sides)
            assert rc == 0 and np.array_equal(got, want), (case.name, box, int(np.argmax(got != want)) if got.size == want.size else -1)
            n += 1
    print(f"G={G}: {n} boxes, one call each")


def _one_call(case, boxes, wants):
    """All boxes of a stream in one call, packed back to back at 16-byte aligned starts in one canary buffer."""
    body = torch.from_numpy(case.body.copy()).cuda()
    offs, at = [], PAD
    for w in wants:
        offs.append(at)
        at = H.round_up(at + w.size, 16)
    buf = torch.full((at + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    arr = (_native.SliceItem * len(boxes))()
    for it, box, o in zip(arr, boxes, offs):
        _fill(it, body.data_ptr(), case.body.size, case.G, case.bits, case.bm, case.chunk, case.data.size, box, buf.data_ptr() + o)
    rc = _slices(arr, len(boxes))
    expect = np.full(at + PAD, CANARY, dtype=np.uint8)
    for w, o in zip(wants, offs):
        expect[o: o + w.size] = w
    got = buf.cpu().numpy()
    bad = np.nonzero(got != expect)[0]
    where = ""
    if bad.size:
        i = int(np.searchsorted(offs, bad[0], side="right")) - 1
        where = f"first differing byte {int(bad[0])}: box {boxes[i] if i >= 0 else None} at {offs[i] if i >= 0 else None}"
    assert rc == 0 and not bad.size, (case.name, rc, where)


@pytest.mark.parametrize("limit", [None] + list(H.LIMITS))
@pytest.mark.parametrize("G", GS)
def test_all_boxes_of_a_stream_in_one_call(G, limit, monkeypatch):
    """With the piece limit lowered, also a plan per stream: its index must count the pieces the model makes."""
    DP._set_env(monkeypatch, {} if limit is None else {"ZIPNN_B200_SLICE_PIECE_CHUNKS": str(limit)})
    lim = limit or H.DEFAULT_LIMIT
    hows = set()
    for case, boxes, wants in _cases(G):
        for b in boxes:
            split = H.pieces_of(b, case.chunk, lim)
            if len(split) > 1:
                hows.update(p.how for p in split)
        _one_call(case, boxes, wants)
        if limit is not None:
            items = _items(case, boxes, wants)
            p = DP.Plan(items)
            assert p.rc == 0, case.name
            for it in items:
                it.check(f"create, limit {limit}")
            _, ci, _ = p.index()
            assert ci == _coded_in_pieces(case, boxes, lim), (case.name, limit)
    if limit is None:
        assert hows == set()    # nothing here covers 16384 chunks
    else:
        assert {"bytes", "rows", "m_rows", "each_row"} <= hows, hows


def _items(case, boxes, wants):
    return [DP.Item(f"{case.name}-{b}", case.body, case.G, case.bits, case.chunk, case.data.size, w, box=b)
            for b, w in zip(boxes, wants)]


def _plan_items(G):
    items, coded = [], 0
    for case, boxes, wants in _cases(G):
        coded += _coded_in_pieces(case, boxes, H.DEFAULT_LIMIT)
        items += _items(case, boxes, wants)
    return items, coded


@pytest.mark.parametrize("G", GS)
def test_plan_over_boxes(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    items, coded = _plan_items(G)
    p = DP.check_plan(items, whole=False)
    _, ci, _ = p.index()
    assert ci == coded
    print(f"G={G}: {len(items)} boxes in one plan")


@pytest.mark.parametrize("G", GS)
def test_run_shifted_over_boxes(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    items, _ = _plan_items(G)
    RI.check_run_into(items, ctas_list=(1, 3, 0))


def test_host_rejections_enqueue_nothing(monkeypatch):
    """A box one byte past orig, len > pitch with several rows, one row more than fits, a misaligned output: E_ARG
    from the workspace size, the call, the plan size and the plan create, with nothing launched or written (the
    valid box in front of the bad one included)."""
    DP._set_env(monkeypatch, {})
    case = next(c for c in H.box_streams(2) if c.name == "c4096_G2")
    orig = case.data.size
    fit = (orig - 3 - 5) // 16 + 1
    assert H.valid_box(orig, (3, fit, 16, 5))
    body = torch.from_numpy(case.body.copy()).cuda()
    out = torch.full((1 << 20,), CANARY, dtype=torch.uint8, device="cuda")
    good = (100, 4, 4096, 333)
    L = _native.lib()
    for bad, shift in (((orig - 9, 1, 16, 10), 0), ((0, 2, 16, 17), 0), ((3, fit + 1, 16, 5), 0), ((64, 2, 100, 50), 1)):
        assert not H.valid_box(orig, bad) or shift
        arr = (_native.SliceItem * 2)()
        _fill(arr[0], body.data_ptr(), case.body.size, 2, case.bits, case.bm, case.chunk, orig, good, out.data_ptr())
        _fill(arr[1], body.data_ptr(), case.body.size, 2, case.bits, case.bm, case.chunk, orig, bad, out.data_ptr() + 4096 + shift)
        torch.cuda.synchronize()
        before = _native.launch_count()
        wsz = C.c_size_t(0)
        assert L.zipnn_b200_decompress_slices_workspace_size(arr, 2, C.byref(wsz)) == _native.E_ARG
        ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        assert L.zipnn_b200_decompress_slices(arr, 2, ws.data_ptr(), ws.numel(), _stream(), 1) == _native.E_ARG
        pb, sb = C.c_size_t(0), C.c_size_t(0)
        assert L.zipnn_b200_decode_plan_size(arr, 2, _stream(), C.byref(pb), C.byref(sb)) == _native.E_ARG
        meta = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        plan = _native.DecodePlanStruct()
        assert L.zipnn_b200_decode_plan_create(arr, 2, meta.data_ptr(), meta.numel(), ws.data_ptr(), ws.numel(), C.byref(plan),
                                               _stream()) == _native.E_ARG
        assert L.zipnn_b200_decode_plan_run(C.byref(plan), _stream()) == _native.E_ARG
        assert _native.launch_count() == before, bad
        torch.cuda.synchronize()
        assert bool(torch.all(out == CANARY)), bad


# ------------------------------------------------------------------ B. past 4 GiB
CHUNK = 262144
ROW_ELEMS = 16384
LIM32 = 1 << 32


class Big:
    """A dense tensor on the device, its ZipNN stream and the stream's tables."""

    def __init__(self, name):
        dtype, gib = {"bf16": (torch.bfloat16, 9), "fp32": (torch.float32, 6)}[name]
        self.name, self.dtype = name, dtype
        self.esz = torch.empty(0, dtype=dtype).element_size()
        self.nbytes = gib << 30
        g = torch.Generator(device="cuda").manual_seed(91 + gib)
        t = torch.empty(self.nbytes // self.esz, dtype=dtype, device="cuda")
        slab = 1 << 27
        for i in range(0, t.numel(), slab):
            m = min(slab, t.numel() - i)
            t[i:i + m] = (torch.randn(m, generator=g, device="cuda", dtype=torch.float32) * 0.02).to(dtype)
        tb = t.view(torch.uint8)
        # past 4 GiB of decoded bytes: an RLE chunk, a raw chunk, and 120 chunks with two coded byte groups
        self.c_hi = LIM32 // CHUNK + 16
        c = self.c_hi
        tb[c * CHUNK: (c + 1) * CHUNK] = 0
        tb[(c + 2) * CHUNK: (c + 3) * CHUNK] = torch.randint(0, 256, (CHUNK,), dtype=torch.uint8, device="cuda", generator=g)
        self.run = (c + 8, c + 128)
        e0, e1 = self.run[0] * CHUNK // self.esz, self.run[1] * CHUNK // self.esz
        # values with 3 mantissa bits: the byte group of the sign and the top mantissa bits codes, and so does the
        # exponent's (fp32: the two low groups are zero, RLE)
        if dtype == torch.bfloat16:
            t.view(torch.int16)[e0:e1].bitwise_and_(-(1 << 4))
        else:
            t.view(torch.int32)[e0:e1].bitwise_and_(-(1 << 20))
        self.t, self.tb = t, tb
        self.t2d = t.view(-1, ROW_ELEMS)
        self.rowbytes = ROW_ELEMS * self.esz
        z = ZipNN(input_format="torch")
        self.stream = z.compress(self.t2d)   # (a 2-D stream: decompress_slice takes [rows, columns] indexes)
        plan = z._last_plan
        self.G, self.hdr = plan["num_buf"], len(plan["header"])
        self.bits, self.bm = plan["bit_reorder"], plan["byte_reorder"]
        assert plan["chunk"] == CHUNK
        self.K = -(-self.nbytes // CHUNK)
        self.tab = StreamTables(self.stream, self.hdr, self.G, self.K)
        self.body = self.stream[self.hdr:]
        self.body_base = [int(b) - self.hdr for b in self.tab.base]   # each group's payload, as offsets into the body
        self.tot = [int(x) for x in self.tab.cum[:, -1]]
        ty, cum = self.tab.types, self.tab.cum.astype(np.int64)
        size = lambda g, k: int(cum[g, k] - (cum[g, k - 1] if k else 0))
        assert all(ty[g, c] == 1 and size(g, c) == 1 for g in range(self.G)), "the zero chunk is RLE in every group"
        assert all(ty[g, c + 2] == 0 for g in range(self.G)), "the random chunk is raw"
        assert all(sum(ty[g, k] == 1 and size(g, k) > 1 for g in range(self.G)) >= 2 for k in range(*self.run))

    def crossings(self):
        """Chunks whose payload item lies across body offset 2^32, per group (first_chunk_past, as
        test_stream_windows does), and groups whose whole payload lies past it."""
        cross, past = [], []
        for g in range(self.G):
            b = self.body_base[g]
            if b >= LIM32:
                past.append(g)
            elif b + self.tot[g] > LIM32:
                cross.append((g, self.tab.first_chunk_past(g, LIM32 - b)))
        return cross, past


@pytest.fixture(scope="module")
def big():
    """One large tensor at a time: asking for the other one frees the first."""
    held = {}

    def get(name):
        if name not in held:
            held.clear()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            gib = {"bf16": 9, "fp32": 6}[name]
            need = (gib << 30) * (2 + (2 if name == "fp32" else 1)) + (4 << 30)   # dense + stream + outputs + 4 GiB
            free, total = torch.cuda.mem_get_info()
            print(f"{name}: {free / 2**30:.1f} GiB free of {total / 2**30:.1f} GiB, {need / 2**30:.1f} GiB needed")
            if free < need:
                pytest.skip(f"{name} {gib} GiB: {free / 2**30:.1f} GiB of device memory free, {need / 2**30:.1f} GiB needed")
            held[name] = Big(name)
        return held[name]

    yield get
    held.clear()
    torch.cuda.empty_cache()


def _box_of_index(bg, r0, r1, c0=0, c1=ROW_ELEMS):
    """t2d[r0:r1, c0:c1] -> (the box the slices call gets (whole rows: one run), the index, the box as rows of t2d)."""
    rows = (r0 * bg.rowbytes + c0 * bg.esz, r1 - r0, bg.rowbytes, (c1 - c0) * bg.esz)
    if c0 == 0 and c1 == ROW_ELEMS:
        n = (r1 - r0) * bg.rowbytes
        return (r0 * bg.rowbytes, 1, n, n), (slice(r0, r1),), rows
    return rows, (slice(r0, r1), slice(c0, c1)), rows


def _dense(bg, box):
    base, rows, pitch, ln = box
    return bg.tb.as_strided((rows, ln), (pitch, 1), base)


def _check_big_box(bg, box, index, rows_box, what):
    """The slices call (canaries around the output) and ZipNN.decompress_slice, against the dense bytes."""
    base, rows, pitch, ln = box
    n = rows * ln
    out = torch.full((n + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
    arr = (_native.SliceItem * 1)()
    _fill(arr[0], bg.body.data_ptr(), bg.body.numel(), bg.G, bg.bits, bg.bm, CHUNK, bg.nbytes, box, out.data_ptr() + PAD)
    assert _slices(arr, 1) == 0, what
    assert bool(torch.all(out[:PAD] == CANARY)) and bool(torch.all(out[PAD + n:] == CANARY)), what
    assert torch.equal(out[PAD: PAD + n].view(rows, ln), _dense(bg, box)), what
    del out
    got = ZipNN(input_format="torch").decompress_slice(bg.stream, index)
    assert got.is_cuda and got.dtype == bg.dtype
    assert torch.equal(got.reshape(rows_box[1], -1).view(torch.uint8), _dense(bg, rows_box)), what


def _big_cases(bg):
    """-> [(what, box, index)] with the branch each one targets asserted."""
    R = bg.nbytes // bg.rowbytes
    cases = []
    box, idx, rb = _box_of_index(bg, 0, R)
    p = H.pieces_of(box, CHUNK)
    assert box[3] // CHUNK > H.DEFAULT_LIMIT and len(p) >= 2, "the whole tensor splits at the real limit"
    assert all(q.c1 - q.c0 <= H.DEFAULT_LIMIT for q in p) and max(q.c1 - q.c0 for q in p) >= H.DEFAULT_LIMIT - 1
    cases.append(("whole", box, idx, rb))
    box, idx, rb = _box_of_index(bg, R - 5, R)
    assert box[0] > LIM32
    cases.append(("last rows", box, idx, rb))
    box, idx, rb = _box_of_index(bg, 0, R, 1001, 2000)
    p = H.pieces_of(box, CHUNK)
    assert box[1] == R and len(p) >= 2 and {q.how for q in p} == {"rows"}, "a column band of every row: pieces of rows"
    cases.append(("column band", box, idx, rb))
    r = LIM32 // bg.rowbytes
    box, idx, rb = _box_of_index(bg, r - 2, r + 2, 7, 16000)
    assert box[0] < LIM32 < box[0] + (box[1] - 1) * box[2] + box[3]
    cases.append(("rows across 2^32", box, idx, rb))
    box, idx, rb = _box_of_index(bg, r - 1, r + 1)
    assert box[0] < LIM32 < box[0] + box[3]
    cases.append(("run across 2^32", box, idx, rb))
    c = bg.c_hi
    box, idx, rb = _box_of_index(bg, c * CHUNK // bg.rowbytes - 3, bg.run[1] * CHUNK // bg.rowbytes + 3, 3, ROW_ELEMS - 5)
    assert box[0] > LIM32
    cases.append(("RLE, raw and general chunks past 4 GiB", box, idx, rb))
    cross, past = bg.crossings()
    assert cross and past, (bg.body_base, bg.tot)
    for g, cx in cross:
        assert 0 < cx < bg.K
        r0 = cx * CHUNK // bg.rowbytes
        box, idx, rb = _box_of_index(bg, r0 - 1, r0 + CHUNK // bg.rowbytes + 1, 1, ROW_ELEMS - 1)
        cases.append((f"group {g}'s payload across 2^32 (chunk {cx})", box, idx, rb))
    return cases


def _big_boxes(big, name):
    bg = big(name)
    cases = _big_cases(bg)
    for what, box, idx, rb in cases:
        _check_big_box(bg, box, idx, rb, f"{name}: {what}")
    cross, past = bg.crossings()
    print(f"{name}: {len(cases)} boxes; payload past 2^32 in groups {past}, across it in {[g for g, _ in cross]}")


def test_big_bf16_boxes(big, monkeypatch):
    DP._set_env(monkeypatch, {})
    bg = big("bf16")
    assert bg.body_base[1] > LIM32, "group 1's payload starts past 2^32"
    _big_boxes(big, "bf16")


def test_big_bf16_batch_with_small_streams(big, monkeypatch):
    DP._set_env(monkeypatch, {})
    bg = big("bf16")
    z = ZipNN(input_format="torch")
    small = [(torch.randn(3000, 77) * 0.02).to(torch.bfloat16).cuda(), (torch.randn(12345) * 0.02).cuda()]
    streams, plans = [], []
    for s in small:
        streams.append(z.compress(s))
        plans.append(z._last_plan)
    outs = [torch.empty(bg.nbytes, dtype=torch.uint8, device="cuda")] + \
        [torch.empty(s.numel() * s.element_size(), dtype=torch.uint8, device="cuda") for s in small]
    arr = (_native.BatchItem * 3)()
    srcs = [(bg.body, bg.G, bg.bits, bg.bm, bg.nbytes)] + [
        (st[len(p["header"]):], p["num_buf"], p["bit_reorder"], p["byte_reorder"], s.numel() * s.element_size())
        for st, p, s in zip(streams, plans, small)]
    for it, (body, G, bits, bm, n), o in zip(arr, srcs, outs):
        it.d_body, it.body_len = body.data_ptr(), body.numel()
        it.num_buf, it.bits_mode, it.bytes_mode, it.chunk, it.orig, it.d_out = G, bits, bm, CHUNK, n, o.data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(arr, 3, C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    assert L.zipnn_b200_decompress_batch(arr, 3, ws.data_ptr(), ws.numel(), _stream(), 1) == 0
    assert torch.equal(outs[0], bg.tb)
    for o, s in zip(outs[1:], small):
        assert torch.equal(o, s.view(torch.uint8).reshape(-1))


def test_big_fp32_boxes(big, monkeypatch):
    DP._set_env(monkeypatch, {})
    _big_boxes(big, "fp32")


class _DevItem:
    """A slice item over a device stream with its output in an arena (DP.Plan fills the C struct from it)."""

    def __init__(self, bg, box, arena, off):
        self.bg, self.box, self.arena, self.off = bg, box, arena, off
        self.n = box[1] * box[3]

    def fill(self, it):
        bg = self.bg
        _fill(it, bg.body.data_ptr(), bg.body.numel(), bg.G, bg.bits, bg.bm, CHUNK, bg.nbytes, self.box,
              self.arena.data_ptr() + self.off + PAD)

    def out(self, shift=0):
        return self.arena[shift + self.off + PAD: shift + self.off + PAD + self.n]

    def check(self, what, shift=0):
        a = self.arena
        o = shift + self.off
        assert bool(torch.all(a[o: o + PAD] == CANARY)) and bool(torch.all(a[o + PAD + self.n: o + 2 * PAD + self.n] == CANARY)), what
        assert torch.equal(self.out(shift).view(self.box[1], self.box[3]), _dense(self.bg, self.box)), what


def test_big_fp32_plan(big, monkeypatch):
    """A plan over the whole 6 GiB tensor and a column band: create, a run, and runs into a second buffer with
    0 (all) and 16 CTAs."""
    DP._set_env(monkeypatch, {})
    bg = big("fp32")
    R = bg.nbytes // bg.rowbytes
    boxes = [(0, 1, bg.nbytes, bg.nbytes), _box_of_index(bg, 0, R, 333, 4444)[0]]
    assert [len(H.pieces_of(b, CHUNK)) > 1 for b in boxes] == [True, True]
    offs, at = [], 0
    for b in boxes:
        offs.append(at)
        at = H.round_up(at + b[1] * b[3] + 2 * PAD, 256)
    arena = torch.full((2 * at,), CANARY, dtype=torch.uint8, device="cuda")
    items = [_DevItem(bg, b, arena, o) for b, o in zip(boxes, offs)]
    p = DP.Plan(items)
    assert p.rc == 0
    for it in items:
        it.check("create")
    assert bool(torch.all(arena[at:] == CANARY))
    for it in items:
        it.out().fill_(CANARY ^ 0xFF)
    assert p.run() == 0 and p.status() == 0
    for it in items:
        it.check("run")
    for ctas in (0, 16):
        for it in items:
            it.out(at).fill_(CANARY ^ 0xFF)
        assert RI.run_shifted(p.plan, at, ctas) == 0 and p.status() == 0
        for it in items:
            it.check(f"run into the second buffer, {ctas} CTAs", shift=at)
            it.check(f"first buffer after a run into the second, {ctas} CTAs")
