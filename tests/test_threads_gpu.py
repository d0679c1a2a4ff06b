"""The library called from many host threads at once, each on its own CUDA stream with its own ZipNN objects, against
the oracle and against what the same calls give from one thread.

A checkpoint loader that opens shards from a thread pool calls the device codec, DecodePipe and SafeOpen from several
threads, and ctypes releases the GIL for the whole foreign call, so the library's process-wide host state -- launch
plans, pinned read-back blocks, wait events, the decode-plan registry, the host slab pipelines, DecodePipe's shared
streams, pool and slab cache -- is really used in parallel.  Every worker starts at a barrier, checks its own results
against its own input (inputs differ per worker, so a result handed to the wrong call shows), and a worker's exception
is raised in the main thread with the worker's name and the case it was on.  Rounds are few and fixed.

  1. device codec: every dtype, both decoders, ragged and empty tensors, through ZipNN and the raw ABI (with peeks on
     another worker's stream); the kernel launches of the concurrent run are those of the same calls run serially;
  2. corrupt streams raise in their own calls only;
  3. compress_batch / decompress_batch / decompress_slice;
  4. decode plans created at once, then run / gather / matvec interleaved, beside a worker that re-creates plans at
     one address;
  5. the host-memory pipelines, below and above the slab threshold;
  6. .znn.safetensors files loaded from a thread pool, DecodePipe's shared state created at once;
  7. a stream compressed on one thread and decoded on another after an event;
  8. the first calls of a fresh process, all made at once: through ZipNN, and through the raw ABI with nothing but the
     call after each thread's barrier, spread over every visible device.
Each test also keeps its peak reserved device memory under BUDGET.
"""
import ctypes as C
import hashlib
import os
import queue
import random
import subprocess
import sys
import threading
import traceback
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import test_matvec_gpu as MV
from oracle import oracle as O
from test_call_state import CASES, _bytes, _make, _oracle_stream
from zipnn_b200 import DecodePipe, DecodePlan, SafeOpen, ZipNN, _native, load_file, save_file
from zipnn_b200 import plan as PL

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SMALL = 8 << 20          # input bytes below which a case is checked against the oracle
LARGE_AT_ONCE = 2        # large cases (about 3 GB each at their peak) in flight at a time
BUDGET = 16 << 30        # peak reserved device memory of one test: the GPU is shared
CANARY = 0xA5


# ------------------------------------------------------------------ the harness
class Workers:
    """Run body(i, at) on n threads that start together at a barrier, each with its own CUDA stream made current.
    at(text) records what worker i is doing; the first exception of a worker is raised here with both."""

    def __init__(self, n: int, body, name: str = "worker"):
        self.n, self.body, self.name = n, body, name
        self.where = [""] * n
        self.errors = [None] * n
        self.barrier = threading.Barrier(n)
        self.failed = threading.Event()   # set when a worker fails: the others stop waiting for it

    def _main(self, i: int):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                self.barrier.wait(timeout=300)
                self.body(i, lambda text: self.where.__setitem__(i, text))
            st.synchronize()
        except BaseException as e:   # noqa: BLE001 -- re-raised in the main thread
            self.errors[i] = (e, traceback.format_exc())
            self.failed.set()
            self.barrier.abort()

    def run(self):
        threads = [threading.Thread(target=self._main, args=(i,), name=f"{self.name}-{i}") for i in range(self.n)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        failed = [i for i in range(self.n) if self.errors[i] is not None]
        # a worker that only saw the barrier break reports after the one that broke it
        failed.sort(key=lambda i: isinstance(self.errors[i][0], threading.BrokenBarrierError))
        if failed:
            i = failed[0]
            e, tb = self.errors[i]
            raise AssertionError(f"{self.name} {i} failed at [{self.where[i]}]: {e!r}\n{tb}") from e


def run_workers(n, body, name="worker"):
    Workers(n, body, name).run()


class LargeCases:
    """`with large:` around a large case: at most LARGE_AT_ONCE run at a time, and each gives its cached blocks back
    before the next starts.  The caching allocator keeps a freed block for later allocations on the stream that made it,
    so without that every worker stream that once ran a large case would keep its peak reserved to the end."""

    def __init__(self):
        self.sem = threading.Semaphore(LARGE_AT_ONCE)

    def __enter__(self):
        self.sem.acquire()

    def __exit__(self, *exc):
        try:
            torch.cuda.empty_cache()
        finally:
            self.sem.release()


@pytest.fixture(autouse=True)
def device_memory_budget():
    """Every test here stays under BUDGET of reserved device memory at its peak."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_reserved()
    torch.cuda.empty_cache()
    print(f"peak reserved device memory {peak / 2 ** 30:.2f} GiB")
    assert peak <= BUDGET, f"the test reserved {peak / 2 ** 30:.2f} GiB of device memory at its peak"


@pytest.fixture
def fast_switches():
    """Hand the GIL over ten times as often as by default, so Python-level check-then-act races show within a few rounds."""
    old = sys.getswitchinterval()
    sys.setswitchinterval(5e-4)
    yield
    sys.setswitchinterval(old)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _nbytes(dt, shape):
    return int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size()


def _layout(x):
    p = ZipNN(input_format="torch").plan(x)
    return p, len(p["header"])


# ------------------------------------------------------------------ 1. device codec, 8. counters
def _raw_compress(x, p):
    """zipnn_b200_compress with out_len, on the current stream -> the stream (the emission kernels may still run)."""
    flat = _bytes(x)
    n = flat.numel()
    hdr = p["header"]
    bound = _native.compress_bound(n, p["num_buf"], p["chunk"], len(hdr))
    wsz = _native.compress_workspace_size(n, p["num_buf"], p["chunk"])
    out = torch.empty(bound, dtype=torch.uint8, device=x.device)
    ws = torch.empty(wsz, dtype=torch.uint8, device=x.device)
    out_len = C.c_size_t(0)
    rc = _native.lib().zipnn_b200_compress(flat.data_ptr(), n, hdr, len(hdr), p["num_buf"], p["bit_reorder"], p["byte_reorder"],
                                           p["chunk"], p["threshold"], out.data_ptr(), bound, C.byref(out_len), ws.data_ptr(), wsz,
                                           _st())
    assert rc == 0, f"zipnn_b200_compress returned {rc}"
    return out[: out_len.value]


def _raw_decompress(s, p, n):
    """zipnn_b200_decompress with check=1 -> the decoded bytes."""
    h = len(p["header"])
    out = torch.empty(n, dtype=torch.uint8, device=s.device)
    for full in (False, True):
        wsz = _native.decompress_workspace_size(n, p["num_buf"], p["chunk"], full=full)
        ws = torch.empty(wsz, dtype=torch.uint8, device=s.device)
        rc = _native.lib().zipnn_b200_decompress(s.data_ptr() + h, s.numel() - h, p["num_buf"], p["bit_reorder"], p["byte_reorder"],
                                                 p["chunk"], n, out.data_ptr(), ws.data_ptr(), wsz, _st(), 1)
        if rc != _native.E_CAPACITY:
            break
    assert rc == 0, f"zipnn_b200_decompress returned {rc}"
    return out


def _digest(s):
    return hashlib.sha256(s.cpu().numpy()).hexdigest()


def _seed(w, ci):
    return 7000 + 100 * w + ci


def test_codec_from_many_threads():
    """8 workers, every case of test_call_state in a shuffled order per worker, two rounds.  Small streams equal the
    oracle's, large ones the stream the same call gave from one thread; every decode returns the input's bytes, dtype
    and shape.  Every other call goes through the raw ABI, and after each raw compress of a small case the worker
    peeks at a stream another worker published, on that worker's stream.  The concurrent run launches exactly the
    kernels the same calls launched one after another."""
    W, ROUNDS = 8, 2
    orders = []
    for w in range(W):
        o = list(range(len(CASES)))
        random.Random(w).shuffle(o)
        orders.append(o)
    small = [_nbytes(dt, sh) < SMALL for dt, sh in CASES]
    want = {}          # (w, ci) -> oracle stream (small cases)
    ref = {}           # (w, ci) -> sha256 of the serial run's stream (large cases)
    launches = {}      # (w, ci) -> launches of the serial run
    for w in range(W):
        for ci, (dt, sh) in enumerate(CASES):
            if small[ci]:
                want[(w, ci)] = _oracle_stream(_make(dt, sh, _seed(w, ci)))
    board = []         # (worker, stream object, stream tensor, its first bytes): what other workers may peek at
    big = LargeCases()

    def one(w, ci, record):
        dt, sh = CASES[ci]
        x = _make(dt, sh, _seed(w, ci))
        raw = x.numel() > 0 and (w + ci) % 2 == 1
        p, _ = _layout(x)
        before = _native.launch_count() if record else 0
        if raw:
            s = _raw_compress(x, p)
        else:
            s = ZipNN(input_format="torch").compress(x)
        if record and not small[ci]:
            ref[(w, ci)] = (s.numel(), _digest(s))
        if small[ci]:
            assert np.array_equal(s.cpu().numpy(), want[(w, ci)]), "stream != oracle"
        else:
            assert (s.numel(), _digest(s)) == ref[(w, ci)], "stream != the serial run's"
        if raw:
            y = _raw_decompress(s, p, x.numel() * x.element_size())
            assert torch.equal(y, _bytes(x)), "raw round trip"
        else:
            y = ZipNN(input_format="torch").decompress(s)
            assert y.is_cuda and y.dtype == x.dtype and tuple(y.shape) == tuple(x.shape) and y.is_contiguous()
            assert torch.equal(_bytes(y), _bytes(x)), "round trip"
        if record:
            torch.cuda.synchronize()
            launches[(w, ci)] = _native.launch_count() - before
        return s, raw

    # the serial run: reference streams of the large cases, launches per call
    for w in range(W):
        for ci in orders[w]:
            with big:
                one(w, ci, True)
    assert all(v > 0 for (w, ci), v in launches.items() if _nbytes(*CASES[ci])), launches

    def body(w, at):
        st = torch.cuda.current_stream()
        rng = random.Random(100 + w)
        for r in range(ROUNDS):
            for ci in orders[w]:
                at(f"round {r} case {ci} {CASES[ci]}")
                if small[ci]:
                    s, raw = one(w, ci, False)
                else:
                    with big:
                        s, raw = one(w, ci, False)
                        del s
                        continue
                if raw:
                    board.append((w, st, s, bytes(want[(w, ci)][:4096])))
                    others = [b for b in board[-16:] if b[0] != w]
                    if others:
                        ow, ost, os_, head = rng.choice(others)
                        at(f"round {r} case {ci}: peek at worker {ow}'s stream")
                        got = C.create_string_buffer(len(head))
                        rc = _native.lib().zipnn_b200_peek(os_.data_ptr(), len(head), got, ost.cuda_stream)
                        assert rc == 0 and got.raw == head, f"peek of worker {ow}'s stream"

    before = _native.launch_count()
    run_workers(W, body)
    torch.cuda.synchronize()
    assert _native.launch_count() - before == ROUNDS * sum(launches.values()), "launches dropped or doubled"
    board.clear()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ 2. errors stay with their call
def _corrupt(s, x, where):
    """The two corruptions of test_call_state.test_corrupt_stream_raises_and_the_next_call_is_clean."""
    bad = s.clone()
    _, hdr = _layout(x)
    G, K = 2, (x.numel() * 2 + 262143) // 262144
    cum = hdr + G * K
    if where == "size_table":
        bad[cum + 8 * (K + 7): cum + 8 * (K + 8)] = 0xFF
    else:
        bad[cum + 8 * (K - 1): cum + 8 * K] = 0x7F
    return bad


def test_corrupt_streams_fail_only_their_own_calls():
    """Two workers decode corrupt streams and must get "corrupt" every time, while four others decode good streams of
    both decoders (the large one is the corrupt streams' own source) and get their bytes."""
    x = _make(torch.bfloat16, (3200 * 131072,), 11)
    s = ZipNN(input_format="torch").compress(x)
    bads = [_corrupt(s, x, "size_table"), _corrupt(s, x, "total")]
    small_cases = [(ci, dt, sh) for ci, (dt, sh) in enumerate(CASES) if _nbytes(dt, sh) < SMALL]
    want = {(w, ci): _oracle_stream(_make(dt, sh, _seed(w, ci))) for w in range(2, 6) for ci, dt, sh in small_cases}
    big = LargeCases()
    ROUNDS = 3
    torch.cuda.synchronize()   # the streams above were written on this thread's stream

    def body(w, at):
        for r in range(ROUNDS):
            if w < 2:
                for k in (w, 1 - w):
                    at(f"round {r} corrupt stream {k}")
                    with big, pytest.raises(RuntimeError, match="corrupt"):
                        ZipNN(input_format="torch").decompress(bads[k])
                continue
            for ci, dt, sh in small_cases:
                at(f"round {r} case {ci}")
                xi = _make(dt, sh, _seed(w, ci))
                si = ZipNN(input_format="torch").compress(xi)
                assert np.array_equal(si.cpu().numpy(), want[(w, ci)]), "stream != oracle"
                assert torch.equal(_bytes(ZipNN(input_format="torch").decompress(si)), _bytes(xi))
            at(f"round {r} the good large stream")
            with big:
                y = ZipNN(input_format="torch").decompress(s)
                assert torch.equal(_bytes(y), _bytes(x)), "the good large stream"
                del y

    run_workers(6, body)
    del bads, s, x
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ 3. batches and slices
BATCH = [(torch.bfloat16, (3, 5, 7)), (torch.float32, (70001,)), (torch.float16, (257, 129)), (torch.float8_e4m3fn, (200000,)),
         (torch.bfloat16, (0,)), (torch.bfloat16, (2_500_000,)), (torch.float16, (4099,)), (torch.bfloat16, (600, 1000))]
BATCH_MAX_CHUNKS = 8     # ZIPNN_B200_ENC_BATCH_MAX_CHUNKS: the 2.5M-element tensor (20 chunks) takes the single-tensor launches
SLICED = len(BATCH) - 1  # 600 x 1000 bf16: 2000-byte rows, a chunk edge every 131.072 rows


def _decompress_batch_raw(streams, xs):
    """zipnn_b200_decompress_batch of every stream, check=1 -> the decoded bytes of each."""
    parsed = []
    for s, x in zip(streams, xs):
        p, h = _layout(x)
        parsed.append((s, p, h, x.numel() * x.element_size()))
    offs, at = [], 0
    for _, _, _, n in parsed:
        offs.append(at)
        at += (n + 15) // 16 * 16
    out = torch.full((max(at, 1),), CANARY, dtype=torch.uint8, device="cuda")
    arr = (_native.BatchItem * len(parsed))()
    for it, (s, p, h, n), o in zip(arr, parsed, offs):
        it.d_body, it.body_len = s.data_ptr() + h, s.numel() - h
        it.num_buf, it.bits_mode, it.bytes_mode = p["num_buf"], p["bit_reorder"], p["byte_reorder"]
        it.chunk, it.orig = p["chunk"], n
        it.d_out = out.data_ptr() + o if n else None
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(arr, len(parsed), C.byref(wsz)) == 0
    ws = torch.empty(max(wsz.value, 1), dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decompress_batch(arr, len(parsed), ws.data_ptr(), ws.numel(), _st(), 1)
    assert rc == 0, f"zipnn_b200_decompress_batch returned {rc}"
    return [out[o: o + n] for o, (_, _, _, n) in zip(offs, parsed)]


def _boxes(rng):
    """Boxes of the 600 x 1000 tensor that cross chunk edges (rows 131, 262, 393, 524), a row, a column and a tail."""
    r0 = int(rng.integers(100, 140))
    r1 = int(rng.integers(250, 600))
    c0 = int(rng.integers(0, 500))
    c1 = int(rng.integers(c0 + 1, 1001))
    return [(slice(r0, r1), slice(c0, c1)), (slice(0, 600), slice(c0, c0 + 1)), int(rng.integers(128, 136)),
            (Ellipsis, slice(c0, c1, 3)), slice(r1 - 1, None)]


def test_batches_and_slices_from_many_threads(monkeypatch):
    """Four workers batch-compress mixed lists (one tensor over the batch limit), batch-decode the streams through the
    raw ABI and read boxes across chunk edges with decompress_slice, two rounds."""
    monkeypatch.setenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", str(BATCH_MAX_CHUNKS))
    W, ROUNDS = 4, 2
    assert _nbytes(*BATCH[5]) > BATCH_MAX_CHUNKS * 262144
    xs = {w: [_make(dt, sh, 9000 + 100 * w + i) for i, (dt, sh) in enumerate(BATCH)] for w in range(W)}
    want = {w: [_oracle_stream(x) for x in xs[w]] for w in range(W)}
    torch.cuda.synchronize()

    def body(w, at):
        rng = np.random.default_rng(w)
        mine = xs[w]
        for r in range(ROUNDS):
            order = rng.permutation(len(mine))
            at(f"round {r} compress_batch order {order.tolist()}")
            streams = ZipNN(input_format="torch").compress_batch([mine[i] for i in order])
            for i, s in zip(order, streams):
                assert np.array_equal(s.cpu().numpy(), want[w][i]), f"batch stream of item {i} != oracle"
            at(f"round {r} decompress_batch")
            got = _decompress_batch_raw(streams, [mine[i] for i in order])
            for i, y in zip(order, got):
                assert torch.equal(y, _bytes(mine[i])), f"batch decode of item {i}"
            s = streams[int(np.nonzero(order == SLICED)[0][0])]
            for box in _boxes(rng):
                at(f"round {r} slice {box}")
                y = ZipNN(input_format="torch").decompress_slice(s, box)
                ref = mine[SLICED][box]
                assert y.is_cuda and y.dtype == ref.dtype and tuple(y.shape) == tuple(ref.shape), box
                assert torch.equal(_bytes(y), _bytes(ref)), box

    run_workers(W, body)


# ------------------------------------------------------------------ 4. decode plans
# (dtype, shape): outputs 0-2 multiply (whole chunks of one decode mode), output 3 is an embedding with a ragged tail
PLAN_ITEMS = [(torch.bfloat16, (256, 1024)), (torch.float16, (256, 512)), (torch.float32, (128, 512)), (torch.bfloat16, (300, 640))]


def _gauss(dt, shape, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * 0.02).to(dt)


class ChurnPlans:
    """Plans created again and again into one plan buffer: P = [fused, constant], Q = [constant, fused], with chunks
    of 4096 bytes.  The "every chunk fused" answer a matvec caches belongs to one create; a struct of an earlier create
    at the same address is refused."""

    SHAPE = (64, 128)

    def __init__(self):
        self.meta = self.scratch = None

    def _streams(self, seed, fused_first):
        fused = _gauss(torch.bfloat16, self.SHAPE, seed)
        const = torch.full(self.SHAPE, 0.25, dtype=torch.bfloat16, device="cuda")
        ws = [fused, const] if fused_first else [const, fused]
        z = ZipNN(input_format="torch", compression_chunk=4096)
        return ws, [z.compress(t) for t in ws]

    def create(self, seed, fused_first):
        ws, streams = self._streams(seed, fused_first)
        parsed = PL._parse(streams)
        offs, out_bytes = PL._offsets(parsed)
        pb, sb = C.c_size_t(0), C.c_size_t(0)
        L = _native.lib()
        assert L.zipnn_b200_decode_plan_size(PL._items(parsed, offs, 1 << 12), len(parsed), _st(), C.byref(pb), C.byref(sb)) == 0
        if self.meta is None:   # one plan buffer for every create: each plan is made at the same address
            self.meta = torch.empty(4 * pb.value, dtype=torch.uint8, device="cuda")
            self.scratch = torch.empty(4 * sb.value + 256, dtype=torch.uint8, device="cuda")
        assert self.meta.numel() >= pb.value and self.scratch.numel() >= sb.value
        out = torch.full((out_bytes,), CANARY, dtype=torch.uint8, device="cuda")
        plan = _native.DecodePlanStruct()
        rc = L.zipnn_b200_decode_plan_create(PL._items(parsed, offs, out.data_ptr()), len(parsed), self.meta.data_ptr(),
                                             self.meta.numel(), self.scratch.data_ptr(), self.scratch.numel(), C.byref(plan), _st())
        assert rc == 0, f"create returned {rc}"
        views = [out[o: o + p.nbytes].view(p.dtype).reshape(p.shape) for p, o in zip(parsed, offs)]
        return plan, ws, streams, out, views


def _raw_matvec(plan, k, x):
    L = _native.lib()
    need = C.c_size_t(0)
    rc = L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(plan), k, 0, x.shape[1], x.shape[0], C.byref(need))
    if rc:
        return rc, None
    out_f = ChurnPlans.SHAPE[0]
    y = torch.empty((x.shape[0], out_f), dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decode_plan_matvec(C.byref(plan), k, 0, x.shape[1], x.data_ptr(), x.shape[1], x.shape[0], None, y.data_ptr(),
                                         out_f, scratch.data_ptr(), scratch.numel(), _st())
    return rc, y


def _churn(at, rounds):
    """Drop and re-create plans at one address while other workers multiply."""
    L = _native.lib()
    cp = ChurnPlans()
    stale = None
    for r in range(rounds):
        fused_first = r % 2 == 0
        at(f"churn {r}: create ({'fused, constant' if fused_first else 'constant, fused'})")
        plan, ws, streams, out, views = cp.create(500 + r, fused_first)
        for v, w in zip(views, ws):
            assert torch.equal(_bytes(v), _bytes(w)), "create's decode"
        x = _gauss(torch.bfloat16, (3, ChurnPlans.SHAPE[1]), 600 + r)
        fk = 0 if fused_first else 1
        rc, y = _raw_matvec(plan, fk, x)
        assert rc == 0, f"matvec of the fused item returned {rc}"
        MV._check(y, x, ws[fk], None, f"churn {r} item {fk}")
        rc, _ = _raw_matvec(plan, 1 - fk, x)
        assert rc == _native.E_UNSUPPORTED, f"matvec of the constant item returned {rc}"
        if stale is not None:
            out_ = C.c_size_t(0)
            for k in (0, 1):
                assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(stale), k, 0, 128, 1, C.byref(out_)) == _native.E_ARG
                assert L.zipnn_b200_decode_plan_gather_scratch_size(C.byref(stale), k, 256, 1, C.byref(out_)) == _native.E_ARG
        out.fill_(CANARY)
        assert L.zipnn_b200_decode_plan_run(C.byref(plan), _st()) == 0
        assert L.zipnn_b200_decode_plan_status(C.byref(plan), _st()) == 0
        for v, w in zip(views, ws):
            assert torch.equal(_bytes(v), _bytes(w)), "run"
        stale = _native.DecodePlanStruct.from_buffer_copy(plan)


def test_decode_plans_from_many_threads():
    """Four workers create their plans at the same moment, then interleave run(), gather() and matvec() on fresh ids
    and activations for three rounds; a fifth re-creates plans at one address all the while."""
    W, ROUNDS = 4, 3
    dense = {w: [_gauss(dt, sh, 4000 + 10 * w + i) for i, (dt, sh) in enumerate(PLAN_ITEMS)] for w in range(W)}
    streams = {w: [ZipNN(input_format="torch").compress(t) for t in dense[w]] for w in range(W)}
    torch.cuda.synchronize()

    def worker(w, at):
        at("create")
        plan = DecodePlan(streams[w])
        for k in range(3):
            assert plan.matvec_ok(k, PLAN_ITEMS[k][1][1]), f"output {k} must multiply, or the case tests nothing"
        g = torch.Generator("cuda").manual_seed(w)
        rng = random.Random(w)
        for r in range(ROUNDS):
            steps = ["run", "gather0", "gather3", "matvec0", "matvec1", "matvec2"]
            rng.shuffle(steps)
            for step in steps:
                at(f"round {r} {step}")
                if step == "run":
                    for k, o in enumerate(plan.run()):
                        assert o.dtype == dense[w][k].dtype and torch.equal(_bytes(o), _bytes(dense[w][k])), f"run output {k}"
                elif step.startswith("gather"):
                    k = int(step[-1])
                    rows = PLAN_ITEMS[k][1][0]
                    ids = torch.randint(0, rows, (2, 5), generator=g, device="cuda", dtype=torch.int64 if r % 2 else torch.int32)
                    y = plan.gather(k, ids)
                    want = dense[w][k].index_select(0, ids.reshape(-1).long()).reshape(ids.shape + dense[w][k].shape[1:])
                    assert torch.equal(_bytes(y), _bytes(want)), f"gather of output {k}"
                else:
                    k = int(step[-1])
                    dt, (_, in_f) = PLAN_ITEMS[k]
                    nt = rng.choice((1, 3, 8))
                    x = (torch.randn((nt, in_f), generator=g, device="cuda") * 0.5).to(dt)
                    MV._check(plan.matvec(k, x), x, dense[w][k], None, f"worker {w} round {r} output {k}")
            plan.check()

    def body(i, at):
        if i == W:
            _churn(at, 8)
        else:
            worker(i, at)

    run_workers(W + 1, body)


# ------------------------------------------------------------------ 5. host pipelines
HOST_SLAB = 3 * 262144      # ZIPNN_B200_HOST_SLAB_BYTES: the slab paths at test sizes
HOST_CASES = [("numpy", np.float32, 70001), ("numpy", np.float16, 1_500_001), ("byte", "bfloat16", 200_000),
              ("byte", "bfloat16", 4_000_000)]


def _host_input(kind, dt, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "numpy":
        return (rng.standard_normal(n) * 0.02).astype(dt)
    return (torch.from_numpy(rng.standard_normal(n // 2).astype(np.float32) * 0.02).to(torch.bfloat16).view(torch.uint8).numpy().tobytes())


def _host_codec(kind, dt):
    return ZipNN(input_format="numpy") if kind == "numpy" else ZipNN(input_format="byte", bytearray_dtype=dt)


def test_host_pipelines_from_many_threads(monkeypatch):
    """Six workers code numpy arrays and bytes below and above the slab threshold through the host-memory calls
    (serialised inside the library), two rounds; every stream equals the oracle's and decodes to the input."""
    monkeypatch.setenv("ZIPNN_B200_HOST_SLAB_BYTES", str(HOST_SLAB))
    W, ROUNDS = 6, 2
    inputs, want = {}, {}
    for w in range(W):
        for ci, (kind, dt, n) in enumerate(HOST_CASES):
            x = _host_input(kind, dt, n, 300 + 10 * w + ci)
            p = _host_codec(kind, dt).plan(x)
            raw = np.frombuffer(x, dtype=np.uint8) if kind == "byte" else x.view(np.uint8)
            inputs[(w, ci)] = x
            want[(w, ci)] = O.zipnn_compress(p["header"], raw, p["num_buf"], p["bit_reorder"], p["byte_reorder"], p["chunk"],
                                             p["threshold"], threads=2)
    assert any(len(memoryview(x).cast("B")) > HOST_SLAB for x in inputs.values())
    assert any(len(memoryview(x).cast("B")) < HOST_SLAB for x in inputs.values())

    def body(w, at):
        order = list(range(len(HOST_CASES)))
        random.Random(w).shuffle(order)
        for r in range(ROUNDS):
            for ci in order:
                kind, dt, n = HOST_CASES[ci]
                at(f"round {r} case {HOST_CASES[ci]}")
                x = inputs[(w, ci)]
                s = _host_codec(kind, dt).compress(x)
                assert np.array_equal(np.frombuffer(s, dtype=np.uint8), want[(w, ci)]), "stream != oracle"
                y = _host_codec(kind, dt).decompress(bytes(s))
                if kind == "numpy":
                    assert y.dtype == x.dtype and y.shape == x.shape and np.array_equal(y.view(np.uint8), x.view(np.uint8))
                else:
                    assert bytes(y) == x

    run_workers(W, body)


# ------------------------------------------------------------------ 6. file loads in a thread pool
FILES = 6
SMALL_RING, SMALL_PIECE = 65536 + 48, 4096 + 16   # DecodePipe's slab ring shrunk: bodies span many slabs


def _file_tensors(f):
    g = torch.Generator().manual_seed(800 + f)
    return {
        "embed": (torch.randn(300, 700, generator=g) * 0.02).to(torch.bfloat16),
        "proj": torch.randn(50_001, generator=g) * 0.1,
        "norm": (torch.randn(64, 64, generator=g)).to(torch.float16),
        "tiny": (torch.randn(3, generator=g)).to(torch.bfloat16),
    }


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.cpu().contiguous().view(torch.uint8),
                                                                       b.cpu().contiguous().view(torch.uint8))


@pytest.fixture
def fresh_pipe_state(monkeypatch):
    """DecodePipe's process-wide streams, reader pool and slab cache as a new process has them, with a small ring; the
    pool made here is shut down afterwards."""
    monkeypatch.setattr(DecodePipe, "SLAB_BYTES", SMALL_RING)
    monkeypatch.setattr(DecodePipe, "COPY_PIECE", SMALL_PIECE)
    monkeypatch.setattr(DecodePipe, "_shared_streams", {})
    monkeypatch.setattr(DecodePipe, "_shared_pool", None)
    monkeypatch.setattr(DecodePipe, "_slab_cache", [])
    yield
    pool = DecodePipe._shared_pool
    if pool is not None:
        pool.shutdown(wait=True)


@pytest.mark.parametrize("cache", ["empty", "full"])
def test_file_loads_in_a_thread_pool(tmp_path, fresh_pipe_state, fast_switches, cache):
    """Six .znn.safetensors files loaded at once from a ThreadPoolExecutor, as a parallel shard loader does:
    load_file and SafeOpen(batch=False) to the GPU, and DecodePipe.submit of host streams.  Every tensor equals what
    was saved; the pipes built at once share one set of side streams and one reader pool; no cached slab is handed to
    two pipes."""
    saved = [_file_tensors(f) for f in range(FILES)]
    paths = [str(tmp_path / f"shard{f}.znn.safetensors") for f in range(FILES)]
    for t, p in zip(saved, paths):
        save_file({k: v.cuda() for k, v in t.items()}, p)
    host_streams = [ZipNN(input_format="torch").compress(t["embed"].cuda()).cpu().numpy() for t in saved]
    if cache == "full":
        DecodePipe._slab_cache.extend(torch.empty(SMALL_RING, dtype=torch.uint8, pin_memory=True) for _ in range(8))
    torch.cuda.synchronize()
    start, held = threading.Barrier(FILES), threading.Barrier(FILES)
    seen = [None] * FILES

    def load(f):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            try:
                start.wait(timeout=120)
                # every worker's first pipe is built at the same moment, and kept until all of them are done
                pipe = DecodePipe("cuda")
                seen[f] = (pipe._streams, pipe._pool, [sl for sl in pipe._stage if sl is not None])
                outs = [pipe.submit(host_streams[f]), pipe.submit(host_streams[f].tobytes())]
                got = load_file(paths[f], device="cuda")
                assert sorted(got) == sorted(saved[f]), f"shard {f}: keys"
                for k, v in saved[f].items():
                    assert got[k].is_cuda and _same(got[k], v), f"shard {f} load_file {k}"
                with SafeOpen(paths[f], "pt", device="cuda", batch=False) as so:
                    one = {k: so.get_tensor(k) for k in so.keys()}
                for k, v in saved[f].items():
                    assert _same(one[k], v), f"shard {f} SafeOpen {k}"
                pipe.finish()
                for y in outs:
                    assert _same(y, saved[f]["embed"]), f"shard {f} DecodePipe.submit"
                held.wait(timeout=120)
                pipe.release()
            except BaseException as e:
                start.abort()
                held.abort()
                raise AssertionError(f"shard {f} ({threading.current_thread().name}): {e!r}\n{traceback.format_exc()}") from e
            st.synchronize()

    with ThreadPoolExecutor(max_workers=FILES, thread_name_prefix="loader") as ex:
        futs = [ex.submit(load, f) for f in range(FILES)]
        errors = [e for e in (fu.exception() for fu in futs) if e is not None]
    errors.sort(key=lambda e: isinstance(e.__cause__, threading.BrokenBarrierError))   # the worker that broke a barrier first
    if errors:
        raise errors[0]
    streams = {id(s[0]) for s in seen}
    pools = {id(s[1]) for s in seen}
    assert len(streams) == 1 and seen[0][0] is DecodePipe._shared_streams[(torch.cuda.current_device(), 4)], "side streams made twice"
    assert len(pools) == 1 and seen[0][1] is DecodePipe._shared_pool, "reader pools made twice"
    handed = [id(sl) for s in seen for sl in s[2]]
    assert len(handed) == len(set(handed)), "one cached slab handed to two pipes"
    if cache == "full":
        assert handed, "the full cache handed nothing out"
    kept = [id(sl) for sl in DecodePipe._slab_cache]
    assert len(kept) == len(set(kept)) and len(kept) <= 8, "a slab cached twice"
    assert all(sl.numel() == SMALL_RING for sl in DecodePipe._slab_cache)


# ------------------------------------------------------------------ 7. a stream handed across threads
def test_stream_handed_across_threads():
    """A producer compresses on its stream and records an event; a consumer waits for the event on its own stream and
    decodes.  zipnn_b200_compress returns while its emission kernels run, so the event is what orders the decode."""
    ROUNDS = 2
    small = [_nbytes(dt, sh) < SMALL for dt, sh in CASES]
    want = {ci: _oracle_stream(_make(dt, sh, 6000 + ci)) for ci, (dt, sh) in enumerate(CASES) if small[ci]}
    q = queue.Queue(maxsize=2)    # at most two large cases in flight

    def put(item) -> bool:
        """False when the consumer failed: nothing takes items any more."""
        while not wk.failed.is_set():
            try:
                q.put(item, timeout=1)
                return True
            except queue.Full:
                pass
        return False

    def get():
        """The next item; None at the end or when the producer failed."""
        while not wk.failed.is_set():
            try:
                return q.get(timeout=1)
            except queue.Empty:
                pass
        return None

    def body(i, at):
        if i == 0:
            try:
                for r in range(ROUNDS):
                    for ci, (dt, sh) in enumerate(CASES):
                        at(f"produce round {r} case {ci}")
                        x = _make(dt, sh, 6000 + ci)
                        s = ZipNN(input_format="torch").compress(x)
                        done = torch.cuda.Event()
                        done.record()
                        if not put((r, ci, x, s, done)):
                            return
            finally:
                put(None)
            return
        while True:
            item = get()
            if item is None:
                return
            r, ci, x, s, done = item
            at(f"consume round {r} case {ci}")
            st = torch.cuda.current_stream()
            st.wait_event(done)
            s.record_stream(st)
            x.record_stream(st)
            if small[ci]:
                assert np.array_equal(s.cpu().numpy(), want[ci]), "stream != oracle"
            y = ZipNN(input_format="torch").decompress(s)
            assert y.dtype == x.dtype and tuple(y.shape) == tuple(x.shape) and torch.equal(_bytes(y), _bytes(x)), "round trip"
            del x, s, y

    wk = Workers(2, body, name="producer/consumer")
    wk.run()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ 8. the first calls of a process, all at once
_COLD = r"""
import threading, sys
import numpy as np, torch
sys.path[:0] = [{root!r}, {tests!r}]
from test_call_state import CASES, _make, _bytes
from zipnn_b200 import ZipNN, _native

torch.cuda.init()
W = len(CASES)
streams, launches_before, errors = [None] * W, None, []
barrier = threading.Barrier(W)
xs = [_make(dt, sh, 50 + i) for i, (dt, sh) in enumerate(CASES)]
torch.cuda.synchronize()

def work(i):
    try:
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            barrier.wait()
            s = ZipNN(input_format="torch").compress(xs[i])
            y = ZipNN(input_format="torch").decompress(s)
            assert torch.equal(_bytes(y), _bytes(xs[i])), f"case {{i}}: round trip"
            streams[i] = s.cpu()
        st.synchronize()
    except BaseException as e:
        errors.append(f"case {{i}}: {{e!r}}")

# the library is loaded, but no kernel has been launched and no launch plan, pinned block or event exists yet
_native.lib()
assert _native.launch_count() == 0
threads = [threading.Thread(target=work, args=(i,)) for i in range(W)]
for t in threads: t.start()
for t in threads: t.join()
assert not errors, errors
cold = _native.launch_count()
for i in range(W):
    s = ZipNN(input_format="torch").compress(xs[i])
    assert torch.equal(s.cpu(), streams[i]), f"case {{i}}: the cold concurrent stream differs from the warm serial one"
    y = ZipNN(input_format="torch").decompress(s)
    assert torch.equal(_bytes(y), _bytes(xs[i]))
torch.cuda.synchronize()
assert _native.launch_count() - cold == cold, (cold, _native.launch_count() - cold)
print("cold ok", cold)
"""


_COLD_RAW = r"""
import ctypes as C, threading, sys
import numpy as np, torch
sys.path[:0] = [{root!r}, {tests!r}]
from oracle import oracle as O
from test_call_state import CASES, _make, _bytes
from zipnn_b200 import ZipNN, _native

# Every case twice: a thread that compresses it and one that decodes the oracle's stream of it, spread over the visible
# devices.  Everything a call takes is made before the barrier, without calling the library, so the threads' first
# library calls -- and with them every launch plan, pinned block and wait event of the process -- start together.
ndev = torch.cuda.device_count()
L = _native.lib()
calls, checks, oracle = [], [], {{}}
for i, (dt, sh) in enumerate(CASES):
    if 0 in sh:
        continue
    for op in ("compress", "decompress"):
        d = len(calls) % ndev
        dev = torch.device("cuda", d)
        x = _make(dt, sh, 70 + i, device=dev)
        p = ZipNN(input_format="torch").plan(x.cpu())
        h, G, chunk = p["header"], p["num_buf"], p["chunk"]
        n = x.numel() * x.element_size()
        if i not in oracle:   # (the same seed gives the same tensor on every device)
            oracle[i] = O.zipnn_compress(h, _bytes(x).cpu().numpy(), G, p["bit_reorder"], p["byte_reorder"], chunk, p["threshold"],
                                         threads=8)
        want = oracle[i]
        with torch.cuda.device(dev):
            st = torch.cuda.Stream()
        if op == "compress":
            bound = _native.compress_bound(n, G, chunk, len(h))
            out = torch.empty(bound, dtype=torch.uint8, device=dev)
            ws = torch.empty(_native.compress_workspace_size(n, G, chunk), dtype=torch.uint8, device=dev)
            out_len = C.c_size_t(0)
            args = (x.data_ptr(), n, h, len(h), G, p["bit_reorder"], p["byte_reorder"], chunk, p["threshold"], out.data_ptr(), bound,
                    C.byref(out_len), ws.data_ptr(), ws.numel(), st.cuda_stream)
            calls.append((d, L.zipnn_b200_compress, args))
            checks.append((f"case {{i}} compress on cuda:{{d}}", lambda out=out, out_len=out_len, want=want:
                           np.array_equal(out[: out_len.value].cpu().numpy(), want), (x, out, ws)))
        else:
            body = torch.from_numpy(want[len(h):].copy()).to(dev)
            out = torch.empty(n, dtype=torch.uint8, device=dev)
            ws = torch.empty(_native.decompress_workspace_size(n, G, chunk), dtype=torch.uint8, device=dev)
            args = (body.data_ptr(), body.numel(), G, p["bit_reorder"], p["byte_reorder"], chunk, n, out.data_ptr(), ws.data_ptr(),
                    ws.numel(), st.cuda_stream, 1)
            calls.append((d, L.zipnn_b200_decompress, args))
            checks.append((f"case {{i}} decompress on cuda:{{d}}", lambda out=out, x=x: torch.equal(out, _bytes(x)), (body, out, ws)))
torch.cuda.synchronize()
assert _native.launch_count() == 0, "a library kernel ran before the threads"
W = len(calls)
rcs = [None] * W
barrier = threading.Barrier(W)

def work(i):
    d, fn, args = calls[i]
    torch.cuda.set_device(d)
    barrier.wait()
    rcs[i] = fn(*args)

def run_all(parallel):
    if parallel:
        threads = [threading.Thread(target=work, args=(i,)) for i in range(W)]
        for t in threads: t.start()
        for t in threads: t.join()
    else:
        for i, (d, fn, args) in enumerate(calls):
            torch.cuda.set_device(d)
            rcs[i] = fn(*args)
    torch.cuda.synchronize()
    for i in range(W):
        assert rcs[i] == 0, f"{{checks[i][0]}}: status {{rcs[i]}}"
        assert checks[i][1](), f"{{checks[i][0]}}: wrong result"

run_all(True)
cold = _native.launch_count()
run_all(False)
assert _native.launch_count() - cold == cold, (cold, _native.launch_count() - cold)
print("cold raw ok", W, "threads", ndev, "devices", cold, "launches")
"""


def test_first_raw_calls_of_a_process_at_once():
    """The process's first library calls made at once through the raw ABI, compresses and decodes of every non-empty
    case on as many threads, spread over the visible devices, with nothing but the call between each thread's barrier
    and its call: the launch-plan table is filled by concurrent inserts, and with two or more devices a plan taken for
    the wrong device shows as a failed launch.  Streams equal the oracle's, decodes the inputs, and the launches equal
    those of the same calls made afterwards one by one."""
    script = _COLD_RAW.format(root=ROOT, tests=HERE)
    r = subprocess.run([sys.executable, "-s", "-c", script], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "cold raw ok" in r.stdout, f"exit {r.returncode}\n{r.stdout}\n{r.stderr[-4000:]}"


def test_first_calls_of_a_process_at_once():
    """Every case of test_call_state on its own thread, all making the process's first library calls at once: the launch
    plans, pinned blocks and wait events are all created under contention.  The streams equal those of the same calls
    made afterwards one by one, and so do the kernel launches."""
    script = _COLD.format(root=ROOT, tests=HERE)
    r = subprocess.run([sys.executable, "-s", "-c", script], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "cold ok" in r.stdout, f"exit {r.returncode}\n{r.stdout}\n{r.stderr[-4000:]}"
