"""The fused decoder's packed launch: one CTA of W warps per SM, each warp an independent decoder with its own
shared-memory region, against the one-warp-CTA launch (ZIPNN_B200_GRID_MODE=1) and the input.

Covered: every dtype class, both side-plane paths (ZIPNN_B200_TMA=0 / 2), tensors below one round of the machine,
exactly one full round (W x SMs x 8 chunks), one group more, chunk counts that are not a multiple of 8, a ragged
last chunk, chunks demoted at run time (tail-pool overflow, table log 12) and RLE side planes, CTAs of 1 and 3 warps
(warp regions 0 and 1 KiB past a 2 KiB boundary in one CTA), and a corrupt stream.  Every decode checks canaries
on both sides of its output.
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import plane_inputs as P
from oracle import oracle as O
from test_decoder_tables_gpu import LAYOUT, crafted_case, planes_case
from zipnn_b200 import _native

pytestmark = pytest.mark.gpu

KNOBS = ("ZIPNN_B200_SYNC_MAX", "ZIPNN_B200_TMA", "ZIPNN_B200_GRID_MODE", "ZIPNN_B200_WARPS_PER_SM", "ZIPNN_B200_DEBUG")
CANARY = 0xA5
PAD = 64
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32, "fp8": torch.float8_e4m3fn}
CHUNK = {"bf16": 4096, "fp16": 4096, "fp32": 4096, "fp8": 2048}
LAUNCH_RE = re.compile(r"fused launch: G=(\d+) PB=(\d+) mode=(\d+) warps_per_cta=(\d+) grid=(\d+) resident_warps_per_sm=(\d+)")


def _set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("ZIPNN_B200_SYNC_MAX", "0")  # always the fused family, whatever the size
    monkeypatch.setenv("ZIPNN_B200_GRID_MODE", "2")  # the packed launch unless the case asks for another
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Dev:
    """A stream body on the device and the tensor bytes it decodes to."""

    def __init__(self, name, dtype, chunk, data, body):
        self.name, self.dtype, self.chunk = name, dtype, chunk
        self.G, self.bits, self.bm = LAYOUT[dtype]
        self.data = data if torch.is_tensor(data) else torch.from_numpy(np.ascontiguousarray(data)).cuda()
        self.body = body if torch.is_tensor(body) else torch.from_numpy(np.ascontiguousarray(body)).cuda()
        self.K = -(-self.data.numel() // chunk)


def gpu_case(dtype, K, seed, ragged=0):
    """K chunks of weight-like values (K - 1 full chunks and a last one `ragged` bytes short), compressed on the
    device."""
    G, bits, bm = LAYOUT[dtype]
    chunk = CHUNK[dtype]
    n = K * chunk - ragged
    es = torch.tensor([], dtype=DTYPES[dtype]).element_size()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n // es, generator=g, device="cuda") * (0.5 if dtype == "fp8" else 0.02)
    data = x.to(DTYPES[dtype]).view(torch.uint8)
    L = _native.lib()
    bound = _native.compress_bound(n, G, chunk, 32)
    d_out = torch.zeros(bound, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.compress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
    out_len = C.c_size_t(0)
    hbuf = (C.c_char * 32).from_buffer_copy(bytes(32))
    assert L.zipnn_b200_compress(data.data_ptr(), n, hbuf, 32, G, bits, bm, chunk, 0.95, d_out.data_ptr(), bound, C.byref(out_len),
                                 ws.data_ptr(), ws.numel(), _stream()) == 0
    return Dev(f"{dtype}_K{K}_r{ragged}", dtype, chunk, data, d_out[32: out_len.value].clone())


def decode(case, capfd=None):
    """zipnn_b200_decompress into a buffer with canaries on both sides -> (status, output on the device, launch
    line of the debug log or None)."""
    n = case.data.numel()
    out = torch.full((PAD + n + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.decompress_workspace_size(n, case.G, case.chunk), dtype=torch.uint8, device="cuda")
    if capfd:
        capfd.readouterr()
    rc = _native.lib().zipnn_b200_decompress(case.body.data_ptr(), case.body.numel(), case.G, case.bits, case.bm, case.chunk, n,
                                             out[PAD:].data_ptr(), ws.data_ptr(), ws.numel(), _stream(), 1)
    launch = None
    if capfd:
        m = LAUNCH_RE.findall(capfd.readouterr().err)
        launch = tuple(map(int, m[-1])) if m else None
    assert bool((out[:PAD] == CANARY).all()) and bool((out[PAD + n:] == CANARY).all()), f"{case.name}: wrote outside the output"
    return rc, out[PAD: PAD + n], launch


def check_packed(case, monkeypatch, capfd, envs=({},), want_warps=None):
    """Under each env (plus both side-plane paths): the packed launch decodes to the input and to what the
    one-warp-CTA launch writes.  -> the packed launch lines."""
    seen = []
    for tma in ("2", "0"):
        _set_env(monkeypatch, {"ZIPNN_B200_TMA": tma, "ZIPNN_B200_GRID_MODE": "1"})
        rc, ref, _ = decode(case)
        assert rc == 0, (case.name, "grid1", tma, rc)
        assert torch.equal(ref, case.data), (case.name, "grid1", tma)
        for env in envs:
            _set_env(monkeypatch, {"ZIPNN_B200_TMA": tma, "ZIPNN_B200_DEBUG": "1", **env})
            rc, got, launch = decode(case, capfd)
            assert launch is not None and launch[2] == 2, (case.name, launch)
            if want_warps is not None and "ZIPNN_B200_WARPS_PER_SM" not in env:
                assert launch[3] == want_warps, (case.name, launch, want_warps)
            assert rc == 0, (case.name, env, tma, rc)
            assert torch.equal(got, ref) and torch.equal(got, case.data), (case.name, env, tma)
            seen.append(launch)
    return seen


def max_warps(dtype, monkeypatch, capfd):
    """(warps per CTA at the largest W the kernel variant holds, SM count), from the launch log."""
    case = gpu_case(dtype, 8, seed=1)
    _set_env(monkeypatch, {"ZIPNN_B200_DEBUG": "1", "ZIPNN_B200_WARPS_PER_SM": "64"})
    rc, got, launch = decode(case, capfd)
    assert rc == 0 and torch.equal(got, case.data)
    return launch[3], _native.lib().zipnn_b200_sm_count()


DEFAULT_WARPS = {"bf16": 13, "fp32": 10}  # fused_default_warps; the others take the most that fit in mode 2


def expected_warps(groups, W, sms):
    """launch_fused's choice in mode 2: W, but no more warps per SM than a round of the machine needs."""
    return min(W, -(-groups // sms))


# ------------------------------------------------------------------ chunk counts around the rounds
@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "fp8"])
def test_chunk_counts_around_one_round(dtype, monkeypatch, capfd):
    wmax, sms = max_warps(dtype, monkeypatch, capfd)
    assert wmax >= 8, (dtype, wmax)  # (the one-warp launch held 10-16)
    W = min(wmax, DEFAULT_WARPS.get(dtype, wmax))
    full = W * sms * 8
    for K, ragged in ((100, 0), (8 * sms + 3, 0), (full, 0), (full + 8, 0), (full + 5, CHUNK[dtype] - 512), (3 * full // 2 + 1, 0)):
        case = gpu_case(dtype, K, seed=K, ragged=ragged)
        groups = -(-K // 8)
        launches = check_packed(case, monkeypatch, capfd, want_warps=expected_warps(groups, W, sms))
        for lc in launches:
            assert lc[4] == min(-(-groups // lc[3]), sms), (case.name, lc)
        if K == full:
            assert launches[0][3] == W and launches[0][4] == sms


def test_default_launch_by_variant(monkeypatch, capfd):
    """Without the knobs, bf16 and fp32 take the packed launch and fp16 / fp8 one one-warp CTA per group."""
    for dtype, mode in (("bf16", 2), ("fp32", 2), ("fp16", 1), ("fp8", 1)):
        case = gpu_case(dtype, 4000, seed=3)
        _set_env(monkeypatch, {"ZIPNN_B200_DEBUG": "1"})
        monkeypatch.delenv("ZIPNN_B200_GRID_MODE")
        rc, got, launch = decode(case, capfd)
        assert rc == 0 and torch.equal(got, case.data) and launch[2] == mode, (dtype, launch)


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_small_ctas_hold_both_region_alignments(dtype, monkeypatch, capfd):
    """W = 1 and 3 (regions at 0, 13 and 26 KiB for bf16: both 2 KiB phases in one CTA), and W fixed at the maximum
    on a tensor that needs several rounds."""
    case = gpu_case(dtype, 2000, seed=7, ragged=CHUNK[dtype] // 2)
    launches = check_packed(case, monkeypatch, capfd, envs=({"ZIPNN_B200_WARPS_PER_SM": "1"}, {"ZIPNN_B200_WARPS_PER_SM": "3"},
                                                            {"ZIPNN_B200_WARPS_PER_SM": "64"}))
    assert {lc[3] for lc in launches} >= {1, 3}


# ------------------------------------------------------------------ demoted chunks and irregular side planes
def _big_tail_plane(rng, m, pb):
    """A top plane of m bytes whose tail table is more than an eighth of a warp's pool: eight of them overflow it."""
    fams = (P.with_rare(220), P.FAMILIES["zipf256"], P.FAMILIES["heavy256"],
            lambda rng, n: P._choice(rng, np.r_[np.full(8, 0.05), np.full(200, 0.6 / 200)], n))  # 200 codes of ~9 bits
    best = (0, None)
    for fam in fams:
        for _ in range(3):
            plane = fam(rng, m)
            r, blk = O.huf_compress(plane)
            if r in (0, 1, O.ERR) or len(blk) >= 0.95 * m:
                continue
            _, w, lg = O.huf_read_table(np.frombuffer(blk, dtype=np.uint8))
            cut = P.tail_size(w, lg, pb)
            if cut > best[0]:
                best = (cut, plane)
    assert 8 * best[0] > P.POOL_CAP[pb], best[0]
    return best[1]


@pytest.mark.parametrize("dtype", ["bf16", "fp16", "fp32", "fp8"])
def test_demoted_chunks_and_rle_side_planes(dtype, monkeypatch, capfd):
    G, bits, _ = LAYOUT[dtype]
    chunk = 4096
    rng = np.random.default_rng(5)
    m = chunk // G
    big = _big_tail_plane(rng, m, 5 if (G >= 2 and bits == 1) else 0)
    tops = []
    for w in range(13):  # 13 warps; with W = 3 they land in every warp slot of several CTAs
        if w % 3 == 1:
            tops += [big] * 8  # the pool overflows: the warp's last chunks are demoted
        else:
            tops += ["geo5" if G > 1 else "eq16"] * 8
    tops = tops[:-3]  # not a multiple of 8
    side = (lambda c, g: "const" if (c // 8) % 2 == 0 and g == 0 else "raw") if G > 1 else None
    pc = planes_case(f"demote_{dtype}", dtype, chunk, tops, seed=6, last=chunk - 1024, side=side)
    demoted = sum(1 for v in pc.pr["fused"].values() if v == "demoted")
    assert demoted > 0, pc.pr["fused"]
    case = Dev(pc.name, dtype, chunk, pc.data, pc.body)
    check_packed(case, monkeypatch, capfd, envs=({}, {"ZIPNN_B200_WARPS_PER_SM": "1"}, {"ZIPNN_B200_WARPS_PER_SM": "3"}))


def test_table_log_12_chunk_in_a_packed_cta(monkeypatch, capfd):
    """A table-log-12 block is demoted by the fused kernel and reported as E_UNSUPPORTED by every launch shape."""
    rng = np.random.default_rng(90)
    nb12 = P.kraft_lengths(rng, 90, 12, min_len=2)
    blocks = [None] * 40
    blocks[21] = nb12
    pc = crafted_case("log12_packed", "bf16", 4096, blocks, seed=91)
    case = Dev(pc.name, "bf16", 4096, pc.data, pc.body)
    for env in ({"ZIPNN_B200_GRID_MODE": "1"}, {}, {"ZIPNN_B200_WARPS_PER_SM": "3"}, {"ZIPNN_B200_TMA": "0"}):
        _set_env(monkeypatch, env)
        rc, _, _ = decode(case)
        assert rc == _native.E_UNSUPPORTED, (env, rc)


# ------------------------------------------------------------------ corrupt streams
def _item_offset(body, G, K, g, c):
    """Offset inside the body of item (g, c)'s payload."""
    cum = body[G * K: 9 * G * K].view(np.uint64).reshape(G, K)
    base = int(sum(int(cum[h, K - 1]) for h in range(g)))
    return 9 * G * K + base + (int(cum[g, c - 1]) if c else 0)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_corrupt_jump_table_is_reported(dtype, monkeypatch):
    """A coded item whose jump table points past its end, in a chunk decoded by the last warp of a late CTA."""
    case = gpu_case(dtype, 3000, seed=11)
    body = case.body.cpu().numpy().copy()
    G, K = case.G, case.K
    types = body[: G * K].reshape(G, K)
    c = max(i for i in range(K) if types[G - 1, i] == 1)
    off = _item_offset(body, G, K, G - 1, c)
    hb = int(body[off])
    hsize = 1 + (hb if hb < 128 else (hb - 127 + 1) // 2)
    body[off + hsize: off + hsize + 2] = 0xFF  # l0 = 65535 > the item
    bad = Dev(case.name + "_bad", dtype, case.chunk, case.data, body)
    for env in ({"ZIPNN_B200_GRID_MODE": "1"}, {}, {"ZIPNN_B200_WARPS_PER_SM": "3"}, {"ZIPNN_B200_TMA": "0"}):
        _set_env(monkeypatch, env)
        rc, _, _ = decode(bad)
        assert rc == _native.E_CORRUPT, (env, rc)
        rc, got, _ = decode(case)
        assert rc == 0 and torch.equal(got, case.data)
