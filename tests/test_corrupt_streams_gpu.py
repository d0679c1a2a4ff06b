"""Every decode entry point on the corrupted-stream corpus (tests/corrupt_streams.py), held to the verdict model.

A refusal must be the model's status (E_CORRUPT / E_UNSUPPORTED); an acceptance must return the model's bytes, bit
for bit.  Every output sits between canaries that a call of either kind leaves intact.  Every device stream sits
inside an arena with guard bytes on both sides; the single-stream calls run with 0x00 and with 0xFF guards and must
give the same verdict and bytes, so no read outside [body, body + body_len) can affect a result.  After a refused
call, a clean stream decoded through the same workspace, plan scratch or host cache must be exact: no error state
sticks.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import corrupt_streams as CS
import test_decoder_tables_gpu as T
import test_host_pipelines_host as HM
from zipnn_b200 import ZipNN, _native

pytestmark = pytest.mark.gpu

STATUS = {CS.OK: 0, CS.CORRUPT: _native.E_CORRUPT, CS.UNSUPPORTED: _native.E_UNSUPPORTED}
CONFIGS = {k: T.CONFIGS[k] for k in ("sync", "fused", "fused_tma0", "fused_grid0")}
CANARY = 0xA5
PAD = 64
GUARD = 256
ALIGNS = (0, 5)
BASES = list(CS.bases())


def _st():
    return torch.cuda.current_stream().cuda_stream


_VERDICTS = {}


def cases(name):
    """[(mutant, model verdict)] of one base."""
    if name not in _VERDICTS:
        b = CS.bases()[name]
        _VERDICTS[name] = [(m, CS.verdict(b, m.body)) for m in CS.mutants(name)]
    return _VERDICTS[name]


class Rig:
    """One base's arena, output and workspace on the device, reused by every mutant of the base."""

    def __init__(self, b):
        self.b = b
        longest = max(m.body.size for m in CS.mutants(b.name))
        self.arena = torch.empty(GUARD + 16 + longest + GUARD, dtype=torch.uint8, device="cuda")
        self.out = torch.empty(PAD + b.orig + PAD, dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(_native.decompress_workspace_size(b.orig, b.G, b.chunk), dtype=torch.uint8, device="cuda")
        self.clean = torch.from_numpy(b.data).cuda()
        self.clean_body = torch.from_numpy(b.body).cuda()

    def place(self, body, align, guard):
        """The body at GUARD + align in the arena, guard bytes everywhere else -> its device address."""
        self.arena.fill_(guard)
        n = body.numel()
        self.arena[GUARD + align: GUARD + align + n].copy_(body)
        return self.arena.data_ptr() + GUARD + align

    def canaries_intact(self, out, n):
        return bool((out[:PAD] == CANARY).all()) and bool((out[PAD + n:] == CANARY).all())

    def decode(self, body, align, guard):
        b = self.b
        self.out.fill_(CANARY)
        ptr = self.place(body, align, guard)
        rc = _native.lib().zipnn_b200_decompress(ptr, body.numel(), b.G, b.bits, b.bm, b.chunk, b.orig, self.out[PAD:].data_ptr(),
                                                 self.ws.data_ptr(), self.ws.numel(), _st(), 1)
        assert self.canaries_intact(self.out, b.orig), "the decoder wrote outside its output"
        return rc, self.out[PAD: PAD + b.orig]

    def clean_decodes(self):
        rc, got = self.decode(self.clean_body, 0, 0x5A)
        return rc == 0 and torch.equal(got, self.clean)


def _expect(v, rc, got, want_dev, what):
    assert rc == STATUS[v.status], (what, rc, v.status)
    if v.status == CS.OK:
        assert torch.equal(got, want_dev), (what, int((got != want_dev).nonzero()[0]))


@pytest.mark.parametrize("name", BASES)
def test_decompress_follows_the_model(name, monkeypatch):
    b = CS.bases()[name]
    rig = Rig(b)
    for m, v in cases(name):
        body = torch.from_numpy(m.body).cuda()
        want = torch.from_numpy(v.data).cuda() if v.status == CS.OK else None
        for cfg, env in CONFIGS.items():
            T._set_env(monkeypatch, env)
            for align in ALIGNS:
                for guard in (0x00, 0xFF):
                    rc, got = rig.decode(body, align, guard)
                    _expect(v, rc, got, want, (m.id, cfg, align, guard))
                    if rc:
                        assert rig.clean_decodes(), (m.id, cfg, "an error stuck to the workspace")
    T._set_env(monkeypatch, {})


@pytest.mark.parametrize("name", BASES)
def test_batch_with_the_mutant_between_clean_streams(name):
    b = CS.bases()[name]
    L = _native.lib()
    clean = torch.from_numpy(b.body).cuda()
    want_clean = torch.from_numpy(b.data).cuda()
    outs = [torch.empty(PAD + b.orig + PAD, dtype=torch.uint8, device="cuda") for _ in range(3)]
    arena = torch.empty(GUARD + max(m.body.size for m in CS.mutants(name)) + GUARD, dtype=torch.uint8, device="cuda")
    ws = None
    for (m, v), guard in ((mv, gd) for mv in cases(name) for gd in (0x00, 0xFF)):
        arena.fill_(guard)
        arena[GUARD: GUARD + m.body.size].copy_(torch.from_numpy(m.body))
        arr = (_native.BatchItem * 3)()
        for i, (ptr, n) in enumerate(((clean.data_ptr(), b.body.size), (arena.data_ptr() + GUARD, m.body.size),
                                      (clean.data_ptr(), b.body.size))):
            outs[i].fill_(CANARY)
            arr[i].d_body, arr[i].body_len = ptr, n
            arr[i].num_buf, arr[i].bits_mode, arr[i].bytes_mode = b.G, b.bits, b.bm
            arr[i].chunk, arr[i].orig, arr[i].d_out = b.chunk, b.orig, outs[i][PAD:].data_ptr()
        wsz = C.c_size_t(0)
        assert L.zipnn_b200_decompress_batch_workspace_size(arr, 3, C.byref(wsz)) == 0
        if ws is None or ws.numel() < wsz.value:
            ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
        rc = L.zipnn_b200_decompress_batch(arr, 3, ws.data_ptr(), ws.numel(), _st(), 1)
        want = torch.from_numpy(v.data).cuda() if v.status == CS.OK else None
        _expect(v, rc, outs[1][PAD: PAD + b.orig], want, m.id)
        if v.chunks is None:
            # a body shorter than its own tables is refused before anything is enqueued: nothing is written
            assert all(bool((o == CANARY).all()) for o in outs), (m.id, "a batch refused on the host wrote")
            continue
        for i in (0, 2):
            assert torch.equal(outs[i][PAD: PAD + b.orig], want_clean), (m.id, "clean item", i)
        for o in outs:
            assert bool((o[:PAD] == CANARY).all()) and bool((o[PAD + b.orig:] == CANARY).all()), m.id


def _slices(b, body_dev, boxes, ws_cache):
    """boxes [(base, rows, pitch, len)] of one stream, one slice item each -> (status, [device outputs])."""
    L = _native.lib()
    its = (_native.SliceItem * len(boxes))()
    outs = []
    for i, (base, rows, pitch, length) in enumerate(boxes):
        o = torch.full((PAD + rows * length + PAD,), CANARY, dtype=torch.uint8, device="cuda")
        outs.append(o)
        it = its[i]
        it.d_body, it.body_len = body_dev[0], body_dev[1]
        it.num_buf, it.bits_mode, it.bytes_mode = b.G, b.bits, b.bm
        it.chunk, it.orig = b.chunk, b.orig
        it.base, it.rows, it.pitch, it.len, it.d_out = base, rows, pitch, length, o[PAD:].data_ptr()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_slices_workspace_size(its, len(boxes), C.byref(wsz)) == 0
    if ws_cache.get("ws") is None or ws_cache["ws"].numel() < wsz.value:
        ws_cache["ws"] = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    ws = ws_cache["ws"]
    rc = L.zipnn_b200_decompress_slices(its, len(boxes), ws.data_ptr(), ws.numel(), _st(), 1)
    for o, (_, rows, _, length) in zip(outs, boxes):
        assert bool((o[:PAD] == CANARY).all()) and bool((o[PAD + rows * length:] == CANARY).all())
    return rc, [o[PAD: -PAD] for o in outs]


def _far_chunks(b, m, v):
    """Chunks two or more away from the mutated one whose bytes the mutant cannot change: for block mutants, and for
    type bytes and size rows that leave every group total intact (a row of the last chunk is a total: it moves the
    payload of every later group)."""
    if m.c is None or v.chunks is None or m.cls not in CS.BLOCK + ("type", "row", "raw_long", "empty_huf"):
        return []
    if m.cls == "row" and m.c == b.K - 1:
        return []
    return [d for d in range(b.K) if abs(d - m.c) >= 2 and v.chunks[d] == CS.OK]


def _chunk_box(b, c):
    n = min(b.chunk, b.orig - c * b.chunk)
    return (c * b.chunk, 1, n, n)


@pytest.mark.parametrize("name", BASES)
def test_slices_follow_the_chunk_verdicts(name):
    """A box over the mutated chunk follows that chunk's verdict; a box two chunks or more away from it decodes
    exactly when the mutant leaves the group totals intact (block mutants, most rows); the whole stream as one box
    follows the stream's verdict."""
    b = CS.bases()[name]
    rig = Rig(b)
    cache = {}
    data = torch.from_numpy(b.data).cuda()
    whole = (0, 1, b.orig, b.orig)

    def clean_after(rc, what):
        if rc:
            rc2, (got2,) = _slices(b, (rig.place(rig.clean_body, 3, 0x5A), b.body.size), [whole], cache)
            assert rc2 == 0 and torch.equal(got2, data), (what, "an error stuck to the workspace")

    for (m, v), guard in ((mv, gd) for mv in cases(name) for gd in (0x00, 0xFF)):
        body = torch.from_numpy(m.body).cuda()
        want = torch.from_numpy(v.data).cuda() if v.status == CS.OK else None
        ptr = rig.place(body, 3, guard)
        rc, (got,) = _slices(b, (ptr, m.body.size), [whole], cache)
        _expect(v, rc, got, want, (m.id, "whole", guard))
        clean_after(rc, (m.id, "whole", guard))
        if m.c is None or v.chunks is None:
            continue
        box = _chunk_box(b, m.c)
        ptr = rig.place(body, 3, guard)
        rc, (got,) = _slices(b, (ptr, m.body.size), [box], cache)
        st = v.chunks[m.c]
        assert rc == STATUS[st], (m.id, "box over the chunk", guard, rc, st)
        if want is not None:
            assert torch.equal(got, want[box[0]: box[0] + box[3]]), (m.id, "box over the chunk", guard)
        clean_after(rc, (m.id, "box over the chunk", guard))
        far = _far_chunks(b, m, v)
        if far:
            d = far[len(far) // 2]
            box = _chunk_box(b, d)
            ptr = rig.place(body, 3, guard)
            rc, (got,) = _slices(b, (ptr, m.body.size), [box], cache)
            assert rc == 0 and torch.equal(got, data[box[0]: box[0] + box[3]]), (m.id, "box away from the chunk", d, guard)


def _plan_create(b, ptr, body_len, out, box=None):
    L = _native.lib()
    arr = (_native.SliceItem * 1)()
    it = arr[0]
    it.d_body, it.body_len = ptr, body_len
    it.num_buf, it.bits_mode, it.bytes_mode = b.G, b.bits, b.bm
    it.chunk, it.orig = b.chunk, b.orig
    base, rows, pitch, length = box or (0, 1, b.orig, b.orig)
    it.base, it.rows, it.pitch, it.len, it.d_out = base, rows, pitch, length, out.data_ptr()
    pb, sb = C.c_size_t(0), C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_size(arr, 1, None, C.byref(pb), C.byref(sb)) == 0
    meta = torch.empty(pb.value, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(max(1, sb.value), dtype=torch.uint8, device="cuda")
    plan = _native.DecodePlanStruct()
    rc = L.zipnn_b200_decode_plan_create(arr, 1, meta.data_ptr(), pb.value, scratch.data_ptr(), sb.value, C.byref(plan), _st())
    return rc, plan, (arr, meta, scratch)


@pytest.mark.parametrize("name", BASES)
def test_decode_plans_follow_the_model(name):
    b = CS.bases()[name]
    L = _native.lib()
    rig = Rig(b)
    data = torch.from_numpy(b.data).cuda()
    out = torch.empty(PAD + b.orig + PAD, dtype=torch.uint8, device="cuda")
    ids = torch.zeros(1, dtype=torch.int64, device="cuda")
    small = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    for (m, v), guard in ((mv, gd) for mv in cases(name) for gd in (0x00, 0xFF)):
        body = torch.from_numpy(m.body).cuda()
        ptr = rig.place(body, 7, guard)
        out.fill_(CANARY)
        rc, plan, keep = _plan_create(b, ptr, m.body.size, out[PAD:])
        assert rc == STATUS[v.status], (m.id, "create", rc, v.status)
        if rc:
            before = _native.launch_count()
            p = C.byref(plan)
            assert L.zipnn_b200_decode_plan_run(p, _st()) == _native.E_ARG, m.id
            assert L.zipnn_b200_decode_plan_run_shifted(p, 0, 1, _st()) == _native.E_ARG, m.id
            assert L.zipnn_b200_decode_plan_gather(p, 0, b.orig, ids.data_ptr(), 1, 8, out[PAD:].data_ptr(), small.data_ptr(),
                                                   small.numel(), _st()) == _native.E_ARG, m.id
            assert L.zipnn_b200_decode_plan_run_select(p, 1, ids.data_ptr(), 1, 8, small.data_ptr(), small.numel(), _st()) == _native.E_ARG, m.id
            assert L.zipnn_b200_decode_plan_status(p, _st()) == _native.E_ARG, m.id
            assert _native.launch_count() == before, (m.id, "a failed plan launched work")
            assert bool((out[:PAD] == CANARY).all()) and bool((out[PAD + b.orig:] == CANARY).all()), m.id
            # a clean plan in the same place decodes exactly
            rc2, plan2, keep2 = _plan_create(b, rig.place(rig.clean_body, 7, guard), b.body.size, out[PAD:])
            assert rc2 == 0 and L.zipnn_b200_decode_plan_run(C.byref(plan2), _st()) == 0
            assert torch.equal(out[PAD: PAD + b.orig], data), (m.id, "clean plan after a refused one")
        else:
            want = torch.from_numpy(v.data).cuda()
            p = C.byref(plan)
            for what, call in (("run", lambda: L.zipnn_b200_decode_plan_run(p, _st())),
                               ("shifted_1", lambda: L.zipnn_b200_decode_plan_run_shifted(p, 0, 1, _st())),
                               ("shifted_all", lambda: L.zipnn_b200_decode_plan_run_shifted(p, 0, 1 << 20, _st()))):
                out.fill_(CANARY)
                assert call() == 0, (m.id, what)
                assert L.zipnn_b200_decode_plan_status(p, _st()) == 0, (m.id, what)
                assert torch.equal(out[PAD: PAD + b.orig], want), (m.id, what)
                assert bool((out[:PAD] == CANARY).all()) and bool((out[PAD + b.orig:] == CANARY).all()), (m.id, what)
            if b.orig % 2 == 0:      # (gather and select see the item as rows of whole elements)
                gs = C.c_size_t(0)
                assert L.zipnn_b200_decode_plan_gather_scratch_size(p, 0, b.orig, 1, C.byref(gs)) == 0
                gscr = torch.empty(max(1, gs.value), dtype=torch.uint8, device="cuda")
                g_out = torch.full((PAD + b.orig + PAD,), CANARY, dtype=torch.uint8, device="cuda")
                assert L.zipnn_b200_decode_plan_gather(p, 0, b.orig, ids.data_ptr(), 1, 8, g_out[PAD:].data_ptr(), gscr.data_ptr(),
                                                       gscr.numel(), _st()) == 0, m.id
                assert torch.equal(g_out[PAD: PAD + b.orig], want), (m.id, "gather")
                ss = C.c_size_t(0)
                assert L.zipnn_b200_decode_plan_select_scratch_size(p, 1, C.byref(ss)) == 0
                sscr = torch.empty(max(1, ss.value), dtype=torch.uint8, device="cuda")
                out.fill_(CANARY)
                assert L.zipnn_b200_decode_plan_run_select(p, 1, ids.data_ptr(), 1, 8, sscr.data_ptr(), sscr.numel(), _st()) == 0, m.id
                assert torch.equal(out[PAD: PAD + b.orig], want), (m.id, "run_select")
        # a box plan away from the mutated chunk creates and runs exactly
        if m.c is not None and v.chunks is not None:
            ptr = rig.place(body, 7, guard)
            far = _far_chunks(b, m, v)
            if far:
                box = _chunk_box(b, far[0])
                bo = torch.full((PAD + box[3] + PAD,), CANARY, dtype=torch.uint8, device="cuda")
                rc, bplan, keep3 = _plan_create(b, ptr, m.body.size, bo[PAD:], box)
                assert rc == 0, (m.id, "box plan", far[0])
                assert L.zipnn_b200_decode_plan_run(C.byref(bplan), _st()) == 0, (m.id, "box plan run")
                assert torch.equal(bo[PAD: PAD + box[3]], data[box[0]: box[0] + box[3]]), (m.id, "box plan")


# ------------------------------------------------------------------ host memory
def _host_decode(b, body, knob, monkeypatch, tail=0):
    """zipnn_b200_decompress_host with the body at the start of a larger host array (tail bytes after it) ->
    (status, output with its canaries)."""
    if knob:
        monkeypatch.setenv(HM.KNOB, str(knob))
    else:
        monkeypatch.delenv(HM.KNOB, raising=False)
    src = np.full(body.size + tail, 0xEE, dtype=np.uint8)
    src[: body.size] = body
    out = np.full(PAD + b.orig + PAD, CANARY, dtype=np.uint8)
    rc = _native.lib().zipnn_b200_decompress_host(src.ctypes.data, body.size, b.G, b.bits, b.bm, b.chunk, b.orig,
                                                  out.ctypes.data + PAD)
    assert np.all(out[:PAD] == CANARY) and np.all(out[PAD + b.orig:] == CANARY)
    return rc, out[PAD: PAD + b.orig]


@pytest.mark.parametrize("name", BASES)
def test_host_pipelines_follow_the_model(name, monkeypatch):
    """One pass, and slabs of the most chunks (3, 2 or 1) that put the targets of the corpus (first, middle and last
    chunk) in the first, a middle and the last slab."""
    b = CS.bases()[name]
    per = next(p for p in (3, 2, 1) if len({c // p for c in b.targets}) == 3 and -(-b.K // p) >= 3)
    knob = per * b.chunk
    plan = HM.slab_plan(b.orig, b.chunk, knob)
    slabs = [c // plan.per for c in b.targets]
    assert plan.piped and slabs[0] == 0 and 0 < slabs[1] < plan.nslabs - 1 and slabs[2] == plan.nslabs - 1
    for m, v in cases(name):
        for k in (None, knob):
            rc, got = _host_decode(b, m.body, k, monkeypatch)
            assert rc == STATUS[v.status], (m.id, k, rc, v.status)
            if rc == 0:
                assert np.array_equal(got, v.data), (m.id, k)
            else:
                rc2, got2 = _host_decode(b, b.body, k, monkeypatch)
                assert rc2 == 0 and np.array_equal(got2, b.data), (m.id, k, "clean decode after a refused one")
    monkeypatch.delenv(HM.KNOB, raising=False)


def test_host_slabs_refuse_a_row_past_the_group_total_before_any_copy(monkeypatch):
    """A row of the last group that points past the group's total but within one slab of the row before it: the
    slab's payload copy would read past the end of the caller's buffer, and its output would reach the caller
    before the next slab's rows fail.  The host check refuses the stream at that slab, before any work: nothing of
    the output changes.  (The stream lies at the start of a larger host array, so a read past it stays in mapped
    memory.)"""
    b = CS.bases()["bf16_fused"]
    per = 3
    G, K = b.G, b.K
    body = b.body.copy()
    cum = body[G * K: 9 * G * K].view("<u8").reshape(G, K)
    i = 1                                                     # slab 1 holds chunks 3, 4 and 5
    cum[G - 1, 5] = cum[G - 1, K - 1] + 4096
    assert cum[G - 1, 5] - cum[G - 1, 2] <= per * b.chunk
    assert HM.decode_host_check(body, G, b.chunk, b.orig, per) == ("row", i)
    rc, got = _host_decode(b, body, per * b.chunk, monkeypatch, tail=2 * per * b.chunk)
    assert rc == _native.E_CORRUPT
    assert np.all(got == CANARY), "slab output reached the caller of a refused stream"
    rc, got = _host_decode(b, b.body, per * b.chunk, monkeypatch)
    assert rc == 0 and np.array_equal(got, b.data)
    monkeypatch.delenv(HM.KNOB, raising=False)


# ------------------------------------------------------------------ the Python surface
TORCH_DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32, "fp8": torch.float8_e4m3fn}


_HEADERS = {}


def _stream_of(b, body, shape=None):
    """The body behind a torch-format ZipNN header (with its packed shape, 1-D by default) for the base's layout."""
    es = torch.tensor([], dtype=TORCH_DT[b.dtype]).element_size()
    shape = tuple(shape or (b.orig // es,))
    if (b.name, shape) not in _HEADERS:
        s = ZipNN(input_format="torch").compress(torch.zeros(shape, dtype=TORCH_DT[b.dtype]).cuda()).cpu().numpy()
        start = ZipNN(input_format="torch")._retrieve_header(s.tobytes())
        h = bytearray(s[:start].tobytes())
        h[14] = b.chunk.bit_length() - 1
        _HEADERS[(b.name, shape)] = h
    h = bytearray(_HEADERS[(b.name, shape)])
    h[24:32] = (len(h) + body.size).to_bytes(8, "little")
    return np.concatenate([np.frombuffer(bytes(h), np.uint8), body])


@pytest.mark.parametrize("name", [n for n in BASES if n != "empty_plane"])
def test_zipnn_decompress_follows_the_model(name):
    b = CS.bases()[name]
    for m, v in cases(name):
        if m.cls == "flip":
            continue
        s = _stream_of(b, m.body)
        for where in ("cuda", "host"):
            src = torch.from_numpy(s).cuda() if where == "cuda" else s.tobytes()
            if v.status == CS.OK:
                got = ZipNN(input_format="torch").decompress(src)
                assert np.array_equal(got.cpu().contiguous().view(torch.uint8).numpy().reshape(-1), v.data), (m.id, where)
            elif v.status == CS.CORRUPT:
                with pytest.raises(RuntimeError, match="corrupt"):
                    ZipNN(input_format="torch").decompress(src)
            else:
                with pytest.raises(RuntimeError, match="unsupported|table log"):
                    ZipNN(input_format="torch").decompress(src)
    torch.cuda.synchronize()


def test_header_fields_out_of_range_are_refused_cleanly():
    """An `orig` the body cannot back, and dtype, chunk-exponent and byte-reorder codes out of range: ValueError or
    the corrupt RuntimeError, never a CUDA or out-of-memory error."""
    b = CS.bases()["bf16_fused"]
    s = _stream_of(b, b.body)
    assert np.array_equal(ZipNN(input_format="torch").decompress(torch.from_numpy(s).cuda()).cpu().view(torch.uint8).numpy(), b.data)
    for at, val, exc in ((slice(16, 24), (1 << 50).to_bytes(8, "little"), RuntimeError),
                         (slice(16, 24), (b.orig * 64).to_bytes(8, "little"), RuntimeError),
                         (15, 77, ValueError), (14, 40, ValueError), (14, 200, ValueError), (5, 220, ValueError), (5, 0, ValueError)):
        bad = bytearray(s.tobytes())
        bad[at] = val
        for where in ("cuda", "host"):
            src = torch.frombuffer(bytearray(bad), dtype=torch.uint8).cuda() if where == "cuda" else bytes(bad)
            with pytest.raises(exc) as e:
                ZipNN(input_format="torch").decompress(src)
            assert not isinstance(e.value, torch.OutOfMemoryError), (at, val, where)
            if exc is RuntimeError:
                assert "corrupt" in str(e.value), (at, val, where, str(e.value))
    torch.cuda.synchronize()


# ------------------------------------------------------------------ file loads and sliced reads
FILE_BASES = [n for n in BASES if n != "empty_plane"]      # (its byte length is not a whole number of elements)


def _representatives(name):
    """The first mutant of every class of a base (a file is written and read per mutant)."""
    seen, out = set(), []
    for m, v in cases(name):
        if m.cls not in seen:
            seen.add(m.cls)
            out.append((m, v))
    return out


def _matrix_shape(b):
    es = torch.tensor([], dtype=TORCH_DT[b.dtype]).element_size()
    numel = b.orig // es
    inf = next(k for k in (16, 4, 2, 1) if numel % k == 0)
    return (numel // inf, inf)


def _raises_as_verdict(v, fn, what):
    if v.status == CS.CORRUPT:
        with pytest.raises(RuntimeError, match="corrupt"):
            fn()
    else:
        with pytest.raises(RuntimeError, match="unsupported"):
            fn()
    torch.cuda.synchronize()


def _write(path, b, stream_np, shape):
    from zipnn_b200.safetensors_io import save_coded
    save_coded({}, {"weight": (torch.from_numpy(stream_np).cuda(), TORCH_DT[b.dtype], shape)}, path)


@pytest.mark.parametrize("name", FILE_BASES)
def test_file_loads_follow_the_model(name, tmp_path):
    """One .znn.safetensors entry per mutant through load_file (the batched decode), SafeOpen(device="cuda") without
    the batch (the per-tensor pipe) and load_module (the compressed residence), which must leave the module as it
    was when it raises."""
    from zipnn_b200 import SafeOpen, decompress_module, load_file, load_module
    b = CS.bases()[name]
    shape = _matrix_shape(b)
    dt = TORCH_DT[b.dtype]
    for k, (m, v) in enumerate(_representatives(name)):
        path = str(tmp_path / f"m{k}.znn.safetensors")
        _write(path, b, _stream_of(b, m.body, shape), shape)

        def via_load_file():
            return load_file(path, device="cuda")["weight"]

        def via_safe_open():
            with SafeOpen(path, "pt", device="cuda", batch=False) as f:
                t = f.get_tensor("weight")
            return t

        for what, fn in (("load_file", via_load_file), ("SafeOpen", via_safe_open)):
            if v.status == CS.OK:
                got = fn()
                assert got.dtype == dt and tuple(got.shape) == shape, (m.id, what)
                assert np.array_equal(got.cpu().contiguous().view(torch.uint8).numpy().reshape(-1), v.data), (m.id, what)
            else:
                _raises_as_verdict(v, fn, (m.id, what))
        if dt == torch.float8_e4m3fn:
            continue      # (no fp8 Linear)
        lin = torch.nn.Linear(shape[1], shape[0], bias=False, device="cuda", dtype=dt)
        with torch.no_grad():
            lin.weight.fill_(0.5)
        w0 = lin.weight
        if v.status == CS.OK:
            load_module(lin, path)
            decompress_module(lin)
            assert np.array_equal(lin.weight.detach().cpu().contiguous().view(torch.uint8).numpy().reshape(-1), v.data), m.id
        else:
            _raises_as_verdict(v, lambda: load_module(lin, path), (m.id, "load_module"))
            assert lin.weight is w0 and bool((lin.weight == 0.5).all()), (m.id, "load_module changed the module")


def test_file_header_fields_out_of_range_are_refused_cleanly(tmp_path):
    """The header mutants of an entry (an `orig` the body cannot back, chunk-exponent and byte-reorder codes out of
    range) through the file loads: ValueError or the corrupt RuntimeError, never a CUDA or out-of-memory error."""
    from zipnn_b200 import SafeOpen, load_file
    b = CS.bases()["bf16_fused"]
    shape = _matrix_shape(b)
    s = _stream_of(b, b.body, shape)
    for at, val, exc in ((slice(16, 24), (1 << 50).to_bytes(8, "little"), RuntimeError),
                         (slice(16, 24), (b.orig * 64).to_bytes(8, "little"), RuntimeError),
                         (14, 40, ValueError), (14, 200, ValueError), (5, 220, ValueError), (5, 0, ValueError)):
        bad = bytearray(s.tobytes())
        bad[at] = val
        path = str(tmp_path / "h.znn.safetensors")
        _write(path, b, np.frombuffer(bytes(bad), np.uint8).copy(), shape)
        for batch in (True, False):
            with pytest.raises(exc) as e:
                with SafeOpen(path, "pt", device="cuda", batch=batch) as f:
                    f.get_tensor("weight")
            assert not isinstance(e.value, torch.OutOfMemoryError), (at, val, batch)
            if exc is RuntimeError:
                assert "corrupt" in str(e.value), (at, val, batch, str(e.value))
        with pytest.raises(exc):
            load_file(path, device="cuda")
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", FILE_BASES)
def test_decompress_slice_follows_the_chunk_verdicts(name):
    """ZipNN.decompress_slice over the elements of the mutated chunk: that chunk's verdict, and the model's bytes
    when the stream is accepted.  A device stream for every mutant; a host stream (cut to the chunks on the host)
    for the block mutants, whose containers stay consistent."""
    b = CS.bases()[name]
    es = torch.tensor([], dtype=TORCH_DT[b.dtype]).element_size()
    for m, v in cases(name):
        if m.c is None or v.chunks is None or m.cls == "flip":
            continue
        s = _stream_of(b, m.body)
        a, n = m.c * b.chunk, min(b.chunk, b.orig - m.c * b.chunk)
        idx = slice(a // es, (a + n) // es)
        st = v.chunks[m.c]
        for where in ("cuda", "host") if m.kind == "block" else ("cuda",):
            src = torch.from_numpy(s).cuda() if where == "cuda" else s.tobytes()

            def fn():
                return ZipNN(input_format="torch").decompress_slice(src, idx)
            if st == CS.OK:
                got = fn()
                if v.status == CS.OK:
                    want = v.data[idx.start * es: idx.stop * es]
                    assert np.array_equal(got.cpu().contiguous().view(torch.uint8).numpy().reshape(-1), want), (m.id, where)
            else:
                _raises_as_verdict(_V(st), fn, (m.id, where))


class _V:
    def __init__(self, status):
        self.status = status
