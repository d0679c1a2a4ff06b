"""Both Huffman decoders on table shapes, tail sizes, bitstream lengths and stream alignments that float weights
never produce.

Inputs are built plane by plane (tests/plane_inputs.py), and every case first asserts with the host model of the
decoders (`plane_inputs.predict`) that it reaches the branch it was built for: the tail pool of the fused kernel
filled exactly and overflowed, chunks demoted to the general kernels, the bulk-tensor side path broken by an
irregular chunk, all 16 side-plane alignments, bitstreams one byte either side of the sync decoder's shared-memory
copy, segment guesses that are never code boundaries, table logs 1 to 12.  Then:
  * the device encoder writes the oracle's stream byte for byte (oracle-made cases);
  * the ORACLE's stream (or a crafted one) decodes to the input under every decoder configuration, with the
    bytes in front of and behind the output untouched;
  * the batch and slice entry points agree.
"""
import ctypes as C
import functools
import re

import numpy as np
import pytest
import torch

import plane_inputs as P
from oracle import oracle as O
from zipnn_b200 import _native

pytestmark = pytest.mark.gpu

LAYOUT = {"bf16": (2, 1, 10), "fp16": (2, 0, 10), "fp32": (4, 1, 220), "fp8": (1, 0, 10)}
CONFIGS = {
    "default": {},
    "fused": {"ZIPNN_B200_SYNC_MAX": "0"},
    "sync": {"ZIPNN_B200_SYNC_MAX": "16384"},
    "fused_tma0": {"ZIPNN_B200_SYNC_MAX": "0", "ZIPNN_B200_TMA": "0"},
    "fused_tma1": {"ZIPNN_B200_SYNC_MAX": "0", "ZIPNN_B200_TMA": "1"},
    "fused_grid0": {"ZIPNN_B200_SYNC_MAX": "0", "ZIPNN_B200_GRID_MODE": "0"},
}
KNOBS = ("ZIPNN_B200_SYNC_MAX", "ZIPNN_B200_TMA", "ZIPNN_B200_GRID_MODE", "ZIPNN_B200_DEBUG")
CANARY = 0xA5
PAD = 64


def _set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Case:
    def __init__(self, name, dtype, chunk, data, body, crafted=False):
        self.name, self.dtype, self.chunk, self.data, self.body, self.crafted = name, dtype, chunk, data, body, crafted
        self.G, self.bits, self.bm = LAYOUT[dtype]
        self.pr = P.predict(body, self.G, self.bits, chunk, data.size)


def _oracle_block(g, c, plane):
    r, blk = O.huf_compress(plane)
    if r == 0:
        return 0, plane.tobytes()
    if r == 1:
        return 1, plane[:1].tobytes()
    return 1, blk


def planes_case(name, dtype, chunk, tops, seed, last=None, side=None):
    """A tensor whose chunk c has the top (coded) plane tops[c] (a family name or an array) and the other planes
    side(c, g) (default: uniform bytes, stored raw).  `last`: length of a ragged last chunk."""
    G, bits, bm = LAYOUT[dtype]
    rng = np.random.default_rng(seed)
    chunks = []
    for c, top in enumerate(tops):
        n = last if (last and c == len(tops) - 1) else chunk
        planes = []
        for g in range(G):
            m = P.plane_len(n, G, g)
            if g == G - 1:
                planes.append(top[:m] if isinstance(top, np.ndarray) else P.FAMILIES[top](rng, m))
            else:
                fam = side(c, g) if side else "raw"
                planes.append(P.FAMILIES[fam](rng, m))
        chunks.append(planes)
    data = P.tensor_from_planes(chunks, G, bits)
    body = O.zipnn_compress(bytes(32), data, G, bits, bm, chunk, 0.95, threads=8)[32:]
    return Case(name, dtype, chunk, data, body)


# ------------------------------------------------------------------ decoding, every way
def decode_single(case, body_off=PAD):
    """zipnn_b200_decompress on the case's body placed body_off bytes into a device buffer.
    -> (status, output bytes); asserts the canary around the output."""
    n = case.data.size
    buf = torch.zeros(body_off + case.body.size + 64, dtype=torch.uint8, device="cuda")
    buf[body_off: body_off + case.body.size] = torch.from_numpy(case.body)
    out = torch.full((PAD + n + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.decompress_workspace_size(n, case.G, case.chunk), dtype=torch.uint8, device="cuda")
    rc = _native.lib().zipnn_b200_decompress(buf[body_off:].data_ptr(), case.body.size, case.G, case.bits, case.bm, case.chunk, n,
                                             out[PAD:].data_ptr(), ws.data_ptr(), ws.numel(), _stream(), 1)
    host = out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY), f"{case.name}: wrote outside the output"
    return rc, host[PAD: PAD + n]


def decode_batch(cases):
    """All cases in one zipnn_b200_decompress_batch call -> (status, [output bytes])."""
    arr = (_native.BatchItem * len(cases))()
    keep = []
    for i, cs in enumerate(cases):
        b = torch.from_numpy(cs.body.copy()).cuda()
        out = torch.full((PAD + cs.data.size + PAD,), CANARY, dtype=torch.uint8, device="cuda")
        keep.append((b, out))
        arr[i].d_body, arr[i].body_len = b.data_ptr(), cs.body.size
        arr[i].num_buf, arr[i].bits_mode, arr[i].bytes_mode = cs.G, cs.bits, cs.bm
        arr[i].chunk, arr[i].orig, arr[i].d_out = cs.chunk, cs.data.size, out[PAD:].data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(arr, len(cases), C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decompress_batch(arr, len(cases), ws.data_ptr(), ws.numel(), _stream(), 1)
    outs = []
    for cs, (_, out) in zip(cases, keep):
        host = out.cpu().numpy()
        assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + cs.data.size:] == CANARY), f"{cs.name}: batch wrote outside"
        outs.append(host[PAD: PAD + cs.data.size])
    return rc, outs


def decode_slice(case, base, rows, pitch, length):
    """One box [base + r * pitch, + length) for r < rows through zipnn_b200_decompress_slices -> (status, bytes)."""
    it = (_native.SliceItem * 1)()
    b = torch.from_numpy(case.body.copy()).cuda()
    n_out = rows * length
    out = torch.full((PAD + n_out + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    it[0].d_body, it[0].body_len = b.data_ptr(), case.body.size
    it[0].num_buf, it[0].bits_mode, it[0].bytes_mode = case.G, case.bits, case.bm
    it[0].chunk, it[0].orig = case.chunk, case.data.size
    it[0].base, it[0].rows, it[0].pitch, it[0].len, it[0].d_out = base, rows, pitch, length, out[PAD:].data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_slices_workspace_size(it, 1, C.byref(wsz)) == 0
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")
    rc = L.zipnn_b200_decompress_slices(it, 1, ws.data_ptr(), ws.numel(), _stream(), 1)
    host = out.cpu().numpy()
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n_out:] == CANARY), f"{case.name}: slice wrote outside"
    return rc, host[PAD: PAD + n_out]


def slice_boxes(case):
    """A dim-0 box (whole rows) and a dim-1 box (a column band) of the tensor viewed as rows of ~1.5 chunks."""
    es = {1: 1, 2: 2, 4: 4}[case.G]
    pitch = max(es, (3 * case.chunk // 2 + 3 * es) // es * es)
    rows = max(1, case.data.size // pitch)
    if rows == 1:
        pitch = case.data.size // es * es
    r0, r1 = rows // 3, max(rows // 3 + 1, 2 * rows // 3)
    c0, c1 = (pitch // 5) // es * es, (4 * pitch // 5) // es * es
    return [(r0 * pitch, 1, pitch, (r1 - r0) * pitch), (c0, rows, pitch, c1 - c0)]


def expect_box(case, base, rows, pitch, length):
    return np.concatenate([case.data[base + r * pitch: base + r * pitch + length] for r in range(rows)])


def gpu_compress(case):
    L = _native.lib()
    n = case.data.size
    d_in = torch.from_numpy(case.data.copy()).cuda()
    bound = _native.compress_bound(n, case.G, case.chunk, 32)
    d_out = torch.zeros(bound, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.compress_workspace_size(n, case.G, case.chunk), dtype=torch.uint8, device="cuda")
    out_len = C.c_size_t(0)
    hbuf = (C.c_char * 32).from_buffer_copy(bytes(32))
    assert L.zipnn_b200_compress(d_in.data_ptr(), n, hbuf, 32, case.G, case.bits, case.bm, case.chunk, 0.95, d_out.data_ptr(), bound,
                                 C.byref(out_len), ws.data_ptr(), ws.numel(), _stream()) == 0
    return d_out[32: out_len.value].cpu().numpy()


def check_everywhere(case, monkeypatch, slices=True):
    """The stream decodes to the input under every configuration, and through the slice entry point."""
    if not case.crafted:
        assert np.array_equal(gpu_compress(case), case.body), f"{case.name}: device stream != oracle stream"
    assert np.array_equal(O.zipnn_decompress(case.body, case.G, case.bits, case.bm, case.chunk, case.data.size), case.data)
    for cfg, env in CONFIGS.items():
        _set_env(monkeypatch, env)
        rc, got = decode_single(case)
        assert rc == 0, (case.name, cfg, rc)
        assert np.array_equal(got, case.data), (case.name, cfg, int(np.argmax(got != case.data)))
    _set_env(monkeypatch, {})
    if slices:
        for box in slice_boxes(case):
            rc, got = decode_slice(case, *box)
            assert rc == 0 and np.array_equal(got, expect_box(case, *box)), (case.name, box)


# ------------------------------------------------------------------ warp mixes: the tail pool of the fused kernel
CUT_FAMILIES = [P.FAMILIES[f] for f in ("eq16", "geo5", "geo3", "fib", "zipf256", "dirichlet256", "heavy256", "eq128")] + \
    [P.with_rare(k) for k in (12, 24, 40, 100, 150, 220)] + \
    [lambda rng, n: P._choice(rng, np.r_[np.full(8, 0.05), np.full(200, 0.6 / 200)], n)]  # 200 codes of ~9 bits


@functools.lru_cache(maxsize=None)
def _planes_by_cut(m, pb):
    """Top planes of m bytes that the oracle codes, by the x_cut they get under PB = pb."""
    rng = np.random.default_rng(1000 + m + pb)
    by = {}
    for fam in CUT_FAMILIES:
        for _ in range(6):
            plane = fam(rng, m)
            r, blk = O.huf_compress(plane)
            if r in (0, 1, O.ERR) or len(blk) >= 0.95 * m:
                continue
            _, w, lg = O.huf_read_table(np.frombuffer(blk, dtype=np.uint8))
            by.setdefault(P.tail_size(w, lg, pb), []).append(plane)
    return by


def _pick(by, cut, k):
    lst = by[cut]
    return lst[k % len(lst)]


def _exact_fill(cuts, cap):
    """8 tail sizes from `cuts` that add up to exactly cap."""
    import itertools
    for combo in itertools.combinations_with_replacement(sorted(cuts), 8):
        if sum(combo) == cap:
            return list(combo)
    raise AssertionError(f"no 8 of {cuts} add up to {cap}")


def warp_mix_case(dtype, seed=0):
    G, bits, _ = LAYOUT[dtype]
    chunk = 2048 if dtype == "fp8" else 4096  # (fp8: larger planes get tails of at most 512 entries here)
    m = chunk // G
    pb = 5 if (G >= 2 and bits == 1) else 0
    cap = P.POOL_CAP[pb]
    by = _planes_by_cut(m, pb)
    cuts = sorted(x for x in by if 0 < x <= cap)
    small, big = cuts[0], max(by)
    warps = {"exact": [_pick(by, x, i) for i, x in enumerate(_exact_fill(cuts, cap))]}
    # the chunk at slot s is the first whose running total passes the capacity: s chunks that fill as much of the
    # pool as they can, then the smallest tail that does not fit any more
    for s in (0, 3, 7):
        if pb == 0 and s == 0:
            continue  # an x_cut is at most 2048 = the PB = 0 pool: one chunk never overflows it alone
        before, rem = [], cap
        for i in range(s):
            x = max(x for x in cuts if x <= rem - (s - 1 - i) * small)
            before.append(x)
            rem -= x
        over = min(x for x in by if x > rem)
        row = before + [over] + [small] * (7 - s)
        warps[f"over{s}"] = [_pick(by, x, i + s) for i, x in enumerate(row)]
    if pb == 5:
        warps["all_demoted"] = [_pick(by, big, i) for i in range(8)]
        mixed = [small, "const", big, "raw", small, big, "const", small]
    else:
        mixed = [cuts[-1], "const", cuts[-1], "raw", cuts[-1], cuts[-1], "const", small]
    warps["demoted_rle_raw"] = [x if isinstance(x, str) else _pick(by, x, i) for i, x in enumerate(mixed)]
    tops, names = [], []
    for name, row in warps.items():
        tops += row
        names.append(name)
    rng = np.random.default_rng(seed)
    tops += [P.FAMILIES["eq16"](rng, m) for _ in range(8 * 3)]  # plain fitting warps, and a ragged end
    case = planes_case(f"warps_{dtype}", dtype, chunk, tops, seed=seed + 1, last=chunk - 512)
    return case, names


@pytest.mark.parametrize("dtype", ["bf16", "fp32", "fp16", "fp8"])
def test_warp_mixes_fill_and_overflow_the_tail_pool(dtype, monkeypatch):
    case, names = warp_mix_case(dtype)
    pr = case.pr
    cap = P.POOL_CAP[pr["pb"]]
    status = lambda w: [pr["fused"].get(c) for c in range(8 * w, 8 * w + 8)]
    for w, name in enumerate(names):
        st = status(w)
        if name == "exact":
            assert pr["pool_run"][w] == cap and st == ["fused"] * 8, (name, st)
        elif name.startswith("over"):
            s = int(name[4:])
            assert st == ["fused"] * s + ["demoted"] * (8 - s), (name, st)
        elif name == "all_demoted":
            assert st == ["demoted"] * 8
        else:
            assert "fused" in st and "demoted" in st and None in st, (name, st)
            kinds = {case.pr["items"][case.G - 1][c].kind for c in range(8 * w, 8 * w + 8)}
            assert {"rle", "raw", "huf"} <= kinds
    assert any("fused" in status(w) and "demoted" in status(w) for w in range(len(names)))
    check_everywhere(case, monkeypatch)


def test_demotion_past_the_slot_pool_reaches_the_overflow_kernel(monkeypatch):
    """More than 4000 chunks, a third of them demoted at run time: far more general chunks than the 64 pool slots,
    so k_decode_overflow takes the rest (the tensor is past the sync threshold: the fused family by default)."""
    K = 4100
    tops = ["eq128" if c % 3 == 1 else "geo5" for c in range(K)]
    case = planes_case("overflow_bf16", "bf16", 4096, tops, seed=12)
    demoted = sum(1 for v in case.pr["fused"].values() if v == "demoted")
    assert case.pr["mode"].count("fused") == K and demoted > 64 + 32 + 1000, demoted
    check_everywhere(case, monkeypatch, slices=False)


# ------------------------------------------------------------------ side planes
@pytest.mark.parametrize("where", ["start", "middle", "end"])
def test_irregular_group0_breaks_the_bulk_side_path(where, monkeypatch):
    """bf16: one chunk's low plane is RLE or coded, which moves the predicted offset of every later chunk's side
    plane: warps from that chunk on leave the bulk-tensor path, the ones before keep it."""
    K = 64
    at = {"start": 0, "middle": 29, "end": K - 1}[where]
    for fam in ("const", "eq16"):
        case = planes_case(f"side_{where}_{fam}", "bf16", 4096, ["geo5"] * K, seed=20 + at,
                           side=lambda c, g, fam=fam: fam if c == at else "raw")
        reg = case.pr["regular"]
        assert reg[: at // 8] == [True] * (at // 8) and not any(reg[at // 8:]), (where, fam, reg)
        assert case.pr["mode"][at] == ("fused" if fam == "const" else "general")
        check_everywhere(case, monkeypatch)


def test_rle_side_planes(monkeypatch):
    """Side planes read with stride 0: bf16 powers of two (an all-zero low plane), and fp32 with each of groups
    0-2 RLE in turn."""
    case = planes_case("bf16_pow2", "bf16", 4096, ["geo5"] * 40, seed=30, side=lambda c, g: "const")
    assert all(case.pr["items"][0][c].kind == "rle" for c in range(40)) and case.pr["mode"] == ["fused"] * 40
    check_everywhere(case, monkeypatch)
    case = planes_case("fp32_rle_groups", "fp32", 4096, ["geo5"] * 48, seed=31, last=2048,
                       side=lambda c, g: "const" if g == c % 3 else "raw")
    for c in range(48):
        assert [case.pr["items"][g][c].kind for g in range(3)] == ["rle" if g == c % 3 else "raw" for g in range(3)]
    assert case.pr["mode"][:47] == ["fused"] * 47
    check_everywhere(case, monkeypatch)


# ------------------------------------------------------------------ alignment of the side plane
@pytest.mark.parametrize("chunk", [2048, 1024, 262144])
def test_every_side_plane_alignment(chunk, monkeypatch, capfd):
    """The body at offsets 0-15 of a device buffer: side_r0 takes all 16 values (the 4-way word switch of the
    bulk-tensor path times the byte shift).  2048 is the smallest chunk with the tensor maps, 1024 has none,
    262144 is the specialised flush."""
    K = 16 if chunk < 262144 else 8
    case = planes_case(f"align_{chunk}", "bf16", chunk, ["geo5"] * K, seed=40)
    assert all(case.pr["regular"]) and case.pr["mode"] == ["fused"] * K
    _set_env(monkeypatch, {"ZIPNN_B200_SYNC_MAX": "0", "ZIPNN_B200_DEBUG": "1"})
    seen = set()
    for off in range(16):
        want_r0 = P.predict(case.body, 2, 1, chunk, case.data.size, body_addr_mod16=off)["side_r0"][0]
        capfd.readouterr()
        rc, got = decode_single(case, body_off=PAD + off)
        err = capfd.readouterr().err
        m = re.findall(r"fused decode: K=(\d+) k_full=\d+ tma_flags=(\d+) side_r0=(\d+)", err)
        assert m, err
        k, flags, r0 = map(int, m[-1])
        assert k == K and r0 == want_r0 and flags == (2 if chunk >= 2048 else 0), (off, m[-1])
        assert rc == 0 and np.array_equal(got, case.data), (chunk, off)
        seen.add(r0)
    assert seen == set(range(16))


# ------------------------------------------------------------------ the ring path of the sync decoder
def ring_cases():
    out = []
    for dtype, chunk in (("fp8", 131072), ("bf16", 262144)):
        for fam in ("eq128", "heavy256"):
            case = planes_case(f"ring_{dtype}_{fam}", dtype, chunk, [fam, fam, fam], seed=50, last=chunk - 4 * LAYOUT[dtype][0])
            out.append(case)
    return out


def test_bitstreams_around_the_shared_memory_copy(monkeypatch):
    """fp8 and bf16 planes of 128 equiprobable symbols (quarters of exactly 28673 bytes, one over the copy; a
    131068-byte plane gives 28672, which stays in shared memory) and of 256 values with one heavy symbol (~30.8
    KiB): the window_frame / sync_scan / sync_emit path, single-tensor and batch."""
    cases = ring_cases()
    lens = set()
    for case in cases:
        top = case.G - 1
        for c in range(case.pr["K"]):
            lens.update(case.pr["items"][top][c].s_len)
    assert {28672, 28673} <= lens and max(lens) > 30000
    for case in cases:
        check_everywhere(case, monkeypatch)
    for env in ({}, CONFIGS["sync"]):
        _set_env(monkeypatch, env)
        rc, outs = decode_batch(cases)
        assert rc == 0 and all(np.array_equal(o, cs.data) for o, cs in zip(outs, cases))


# ------------------------------------------------------------------ codes that never resynchronise
def _misaligned_len(L, lo):
    """A plane length >= lo whose four quarters have segbits % L != 0."""
    s = lo // 4
    while True:
        if (-(-s * L // 256)) % L and s * L > 192 * 256:
            return 4 * s
        s += 1


def test_fixed_length_codes_with_misaligned_segment_guesses(monkeypatch):
    """2^L equiprobable symbols give fixed-length codes, which never resynchronise: a thread whose segment start
    is not a multiple of L from the end mark is put right only by the round loop.  Also runs of 11-bit codes
    (a Fibonacci plane, each quarter sorted by code length)."""
    cases = []
    for fam, L in (("eq4", 2), ("eq16", 4), ("eq64", 6)):
        n = _misaligned_len(L, 100000)
        case = planes_case(f"fixed_{fam}", "fp8", 131072, [fam, fam], seed=60 + L, last=n)
        it = case.pr["items"][0][1]
        assert it.fixed_len == L and P.misaligned_sync_guesses(it) == 4, (fam, it.segbits)
        cases.append(case)
    rng = np.random.default_rng(64)
    fib = [P.clustered(P.FAMILIES["fib"](rng, 131072)) for _ in range(2)]
    case = planes_case("fib_clustered", "fp8", 131072, fib, seed=65)
    it = case.pr["items"][0][0]
    assert it.lg == 11 and it.lengths.max() == 11
    cases.append(case)
    for case in cases:
        check_everywhere(case, monkeypatch)


# ------------------------------------------------------------------ table logs 1-4, 256-symbol alphabets
@pytest.mark.parametrize("dtype", ["fp8", "bf16", "fp16"])
def test_small_table_logs_and_full_alphabets(dtype, monkeypatch):
    fams = ["eq2", "eq4", "eq8", "eq16", "zipf256", "dirichlet256", "heavy256", "logexp"]
    chunk = 131072 if dtype == "fp8" else 262144
    case = planes_case(f"logs_{dtype}", dtype, chunk, fams, seed=70)
    top = case.G - 1
    logs = [case.pr["items"][top][c].lg for c in range(len(fams))]
    assert logs[:4] == [1, 2, 3, 4], logs
    for c in (4, 5, 6):  # 256-symbol alphabets; Zipf and Dirichlet have long tANS-coded table descriptions
        it = case.pr["items"][top][c]
        assert it.nsym > 200 and (c == 6 or 50 <= it.hsize <= 128), (c, it.nsym, it.hsize)
    check_everywhere(case, monkeypatch)


# ------------------------------------------------------------------ crafted streams
def crafted_case(name, dtype, chunk, blocks, seed, last=None):
    """blocks[c] = code lengths for the top plane of chunk c, or (lengths, a symbol drawn 3 % more often than its
    length says), or None (the oracle's block of a geo5 plane), or 'raw' / 'const' (that plane family).  The other planes are uniform bytes stored raw."""
    G, bits, bm = LAYOUT[dtype]
    rng = np.random.default_rng(seed)
    chunks, items = [], [[] for _ in range(G)]
    for c, spec in enumerate(blocks):
        n = last if (last and c == len(blocks) - 1) else chunk
        planes = [P.FAMILIES["raw"](rng, P.plane_len(n, G, g)) for g in range(G - 1)]
        m = P.plane_len(n, G, G - 1)
        hot = None
        if isinstance(spec, tuple):
            spec, hot = spec
        if isinstance(spec, str):
            top = P.FAMILIES[spec](rng, m)
        elif spec is None:
            top = P.FAMILIES["geo5"](rng, m)
        else:
            top = P.plane_for_lengths(rng, spec, m, hot)
        planes.append(top)
        chunks.append(planes)
        for g in range(G):
            if g == G - 1 and not isinstance(spec, str) and spec is not None:
                blk = P.huf_block(spec, top)
                assert len(blk) < m - 1, (name, c, len(blk), m)
                items[g].append((1, blk))
            else:
                items[g].append(_oracle_block(g, c, planes[g]))
    data = P.tensor_from_planes(chunks, G, bits)
    body = P.assemble_body(items, G)
    return Case(name, dtype, chunk, data, body, crafted=True)


def _lengths_with_tail(rng, x_cut, pb):
    """Kraft-complete lengths (table log 11) whose tail under PB = pb is exactly x_cut: codes of 1, 2, ... bits
    until x_cut of the 2048-entry index space is left, then codes longer than pb (8 for pb = 0) bits over more than
    half of it (the rest in codes one bit shorter), and one 11-bit pair."""
    long_len = 6 if pb == 5 else 9
    nb = np.zeros(256, dtype=np.uint8)
    syms = iter(rng.permutation(129))
    room, length = 2048, 1
    while room > x_cut:
        nb[next(syms)] = length
        room -= 2048 >> length
        length += 1
    long_amt = x_cut if pb == 5 else x_cut // 2 + 32
    nb[next(syms)] = nb[next(syms)] = 11
    for _ in range((long_amt - 2) // (2048 >> long_len)):
        nb[next(syms)] = long_len
    rest = long_amt - 2 - (long_amt - 2) // (2048 >> long_len) * (2048 >> long_len)
    for share_len in range(long_len + 1, 11):  # what is left of the long region, in codes of long_len+1 .. 10 bits
        if rest & (2048 >> share_len):
            nb[next(syms)] = share_len
            rest -= 2048 >> share_len
    assert rest == 0
    for _ in range((room - long_amt) // (2048 >> (long_len - 1))):
        nb[next(syms)] = long_len - 1
    assert sum(2.0 ** -nb[nb > 0].astype(np.float64)) == 1.0
    return nb


def test_crafted_suboptimal_codes(monkeypatch):
    """Valid code tables the reference encoder never chooses: random Kraft-complete lengths per chunk, a frequent
    symbol on an 11-bit code, and tails exactly at and one step over the pool of a warp."""
    rng = np.random.default_rng(80)
    for dtype in ("bf16", "fp16"):
        pb = 5 if dtype == "bf16" else 0
        cap = P.POOL_CAP[pb]
        big = 1024 if pb == 5 else 512
        blocks = []
        # warp 0: one chunk with a tail of the whole pool (bf16) / four that fill it (fp16); the rest plain
        at_cap = [_lengths_with_tail(rng, big, pb) for _ in range(cap // big)]
        blocks += at_cap + ["raw"] * (8 - len(at_cap))
        # warp 1: the same, then one more coded chunk: one step over
        blocks += [_lengths_with_tail(rng, big, pb) for _ in range(cap // big)] + [None] + ["const"] * (7 - cap // big)
        # warps 2-5: random lengths, some with a hot 11-bit symbol
        for c in range(32):
            max_len = int(rng.integers(1, 12))
            nb = P.kraft_lengths(rng, int(rng.integers(2, min(120, 1 << max_len) + 1)), max_len)
            blocks.append((nb, int(np.nonzero(nb == nb.max())[0][0])) if c % 4 == 0 else nb)
        case = crafted_case(f"crafted_{dtype}", dtype, 4096, blocks, seed=81)
        st = [case.pr["fused"].get(c) for c in range(16)]
        assert case.pr["pool_run"][0] == cap and st[: cap // big] == ["fused"] * (cap // big), st
        assert st[8: 8 + cap // big] == ["fused"] * (cap // big) and st[8 + cap // big] == "demoted", st
        check_everywhere(case, monkeypatch)
        # a frequent symbol on an 11-bit code
        nb = P.kraft_lengths(rng, 100, 11)
        hot = int(np.nonzero(nb == 11)[0][0])
        hot_case = crafted_case(f"hot11_{dtype}", dtype, 4096, [(nb, hot)] * 3 + [None] * 5, seed=82)
        top = P.planes_of(hot_case.data, 2, LAYOUT[dtype][1], 4096)[0][1]
        assert np.mean(top == hot) > 0.02 and hot_case.pr["items"][1][0].lengths[hot] == 11
        check_everywhere(hot_case, monkeypatch)


def test_table_log_12_is_unsupported_everywhere(monkeypatch):
    """A valid stream with one table-log-12 block (never written by the reference encoder, accepted by its
    decoder): every entry point reports E_UNSUPPORTED -- never E_CORRUPT, never wrong bytes -- and a slice whose
    box misses that chunk still decodes."""
    rng = np.random.default_rng(90)
    nb12 = P.kraft_lengths(rng, 90, 12, min_len=2)
    assert nb12.max() == 12
    K, bad = 24, 13
    blocks = [None] * K
    blocks[bad] = nb12
    case = crafted_case("log12_bf16", "bf16", 4096, blocks, seed=91)
    assert case.pr["items"][1][bad].lg == 12 and case.pr["items"][1][bad].x_cut == {5: -1, 0: -1}
    assert np.array_equal(O.zipnn_decompress(case.body, 2, 1, 10, 4096, case.data.size), case.data)
    for cfg, env in CONFIGS.items():
        _set_env(monkeypatch, env)
        rc, _ = decode_single(case)
        assert rc == _native.E_UNSUPPORTED, (cfg, rc)
    _set_env(monkeypatch, {})
    good = planes_case("log12_neighbour", "bf16", 4096, ["geo5"] * 8, seed=92)
    rc, outs = decode_batch([good, case])
    assert rc == _native.E_UNSUPPORTED
    assert np.array_equal(outs[0], good.data)
    rc, _ = decode_slice(case, bad * 4096 - 4096, 1, 0, 3 * 4096)
    assert rc == _native.E_UNSUPPORTED
    miss = (0, 1, 0, bad * 4096)  # every chunk in front of it
    rc, got = decode_slice(case, *miss)
    assert rc == 0 and np.array_equal(got, case.data[: bad * 4096])
    rc, got = decode_slice(case, (bad + 1) * 4096 + 16, 1, 0, 4096 * 5)
    assert rc == 0 and np.array_equal(got, case.data[(bad + 1) * 4096 + 16: (bad + 6) * 4096 + 16])
    # host buffers (pageable)
    out = np.zeros(case.data.size, dtype=np.uint8)
    body = case.body.copy()
    rc = _native.lib().zipnn_b200_decompress_host(body.ctypes.data, body.size, 2, 1, 10, 4096, case.data.size, out.ctypes.data)
    assert rc == _native.E_UNSUPPORTED
    torch.cuda.synchronize()


# ------------------------------------------------------------------ all cases of one dtype in one batch
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "fp8"])
def test_batch_of_every_case(dtype, monkeypatch):
    cases = [warp_mix_case(dtype)[0]]
    chunk = 131072 if dtype == "fp8" else 262144
    cases.append(planes_case(f"logs_{dtype}", dtype, chunk, ["eq2", "eq4", "eq8", "eq16", "zipf256", "heavy256"], seed=70))
    if dtype in ("fp8", "bf16"):
        cases += [c for c in ring_cases() if c.dtype == dtype]
    if dtype == "fp32":
        cases.append(planes_case("fp32_rle_groups", "fp32", 4096, ["geo5"] * 48, seed=31, last=2048,
                                 side=lambda c, g: "const" if g == c % 3 else "raw"))
    for env in ({}, CONFIGS["fused"], CONFIGS["sync"]):
        _set_env(monkeypatch, env)
        rc, outs = decode_batch(cases)
        assert rc == 0
        for cs, o in zip(cases, outs):
            assert np.array_equal(o, cs.data), cs.name
