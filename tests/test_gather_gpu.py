"""Gathers from decode plans (zipnn_b200_decode_plan_gather, DecodePlan.gather) against the dense bytes.

Every gathered row must equal the numpy row of the input bytes, with the canaries around the output untouched:
  * the streams of test_boxes_host.box_streams (fused, general, overflow and plain chunks, ragged last chunks, chunks
    from G bytes to the default) viewed as rows that divide chunks, straddle them and span many of them;
  * ids duplicated, unsorted, all in one chunk, covering every chunk, the first and last row, empty and 2-D, as int32
    and int64, with scratch slot counts that force one, two and many passes;
  * bf16, fp16, fp32 and both fp8 formats through DecodePlan.gather.
Also: the launch count does not depend on the ids; a captured graph replays with new ids; out-of-range ids give zero
rows and IndexError from check(); a corrupt stream is refused at create; host rejections launch and write nothing.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import test_boxes_host as H
import test_decode_plan_gpu as DP
from zipnn_b200 import DecodePlan, ZipNN, _native

pytestmark = pytest.mark.gpu

PAD, CANARY = 64, 0xA5


def _st():
    return torch.cuda.current_stream().cuda_stream


def scratch_size(p, item, R, slots):
    out = C.c_size_t(0)
    rc = _native.lib().zipnn_b200_decode_plan_gather_scratch_size(C.byref(p.plan), item, R, slots, C.byref(out))
    return rc, out.value


def gather(p, item, R, ids, slots):
    rc, sb = scratch_size(p, item, R, slots)
    assert rc == 0, rc
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
    n = ids.numel()
    out = torch.full((PAD + n * R + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    rc = _native.lib().zipnn_b200_decode_plan_gather(C.byref(p.plan), item, R, ids.data_ptr(), n, ids.element_size(),
                                                      out[PAD:].data_ptr(), scratch.data_ptr(), sb, _st())
    return rc, out


def expect(data: np.ndarray, R: int, ids: np.ndarray) -> np.ndarray:
    rows = data.reshape(-1, R)
    ids = ids.reshape(-1)
    good = (ids >= 0) & (ids < rows.shape[0])
    out = np.zeros((ids.size, R), dtype=np.uint8)
    out[good] = rows[ids[good]]
    return out.reshape(-1)


def check_out(out, want, what):
    host = out.cpu().numpy()
    n = want.size
    assert np.all(host[:PAD] == CANARY) and np.all(host[PAD + n:] == CANARY), f"{what}: wrote outside its output"
    got = host[PAD: PAD + n]
    assert np.array_equal(got, want), (what, int(np.argmax(got != want)))


def row_sizes(orig: int, chunk: int) -> list:
    """Divisors of orig: the smallest above 1, one inside a chunk, one about a chunk (straddling), one spanning
    several chunks, and the whole tensor."""
    divs = sorted({d for i in range(1, int(orig ** 0.5) + 1) if orig % i == 0 for d in (i, orig // i)})
    pick = [d for d in divs if d > 1][:1]
    pick += [d for d in divs if 2 < d < chunk][-1:]
    pick += [min(divs, key=lambda d: abs(d - (chunk + chunk // 2)))]
    pick += [d for d in divs if d > 3 * chunk][:1]
    pick += [orig]
    return sorted(set(pick))


def id_sets(rows: int, R: int, chunk: int, rng) -> list:
    in_one = max(1, chunk // R) if R < chunk else 1
    sets = [rng.integers(0, rows, 37),                                   # duplicated, unsorted
            np.array([0, rows - 1, rows - 1, 0]),                        # first and last row
            rng.integers(0, min(rows, in_one), 9),                       # all in one chunk (rows inside chunk 0)
            np.arange(rows)[::-1][:: max(1, rows // 20000)].copy(),     # every chunk (rows spread over all), backwards
            np.zeros(0, dtype=np.int64)]                                 # empty
    return sets


@pytest.mark.parametrize("G", (1, 2, 4))
def test_box_streams_every_row_shape(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    rng = np.random.default_rng(G)
    n_checks = 0
    for case in H.box_streams(G):
        orig = case.data.size
        item = DP.Item(case.name, case.body, case.G, case.bits, case.chunk, orig, case.data)
        p = DP.Plan([item])
        assert p.rc == 0
        for R in row_sizes(orig, case.chunk):
            rows = orig // R
            for k, ids in enumerate(id_sets(rows, R, case.chunk, rng)):
                dt = torch.int32 if k % 2 else torch.int64
                for slots in ((1, 2, 64) if k == 0 else (3,)):
                    t = torch.from_numpy(ids).to(dt).cuda()
                    rc, out = gather(p, 0, R, t, slots)
                    assert rc == 0
                    check_out(out, expect(case.data, R, ids), f"{case.name} R={R} ids#{k} slots={slots}")
                    n_checks += 1
        assert p.status() == 0
    print(f"G={G}: {n_checks} gathers")


def _plan_of(t: torch.Tensor) -> DecodePlan:
    s = ZipNN(input_format="torch").compress(t)
    return DecodePlan([s])


DTYPES = [torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2]


@pytest.mark.parametrize("dtype", DTYPES)
def test_dtypes_through_decode_plan(dtype):
    torch.manual_seed(5)
    w = (torch.randn(3000, 384, device="cuda") * 0.02).to(dtype)
    plan = _plan_of(w)
    for ids in (torch.randint(0, 3000, (2, 33), device="cuda"), torch.tensor([2999, 0, 7, 7], device="cuda", dtype=torch.int32),
                torch.arange(3000, device="cuda")):
        got = plan.gather(0, ids)
        assert got.shape == ids.shape + (384,) and got.dtype == dtype
        want = w.view(torch.uint8).index_select(0, ids.reshape(-1).long()).reshape(got.shape[:-1] + (-1,))
        assert torch.equal(got.view(torch.uint8), want)
    plan.check()
    # a 1-D output gathers elements
    v = w.reshape(-1)[:5000].contiguous()
    pv = _plan_of(v)
    ids = torch.randint(0, 5000, (100,), device="cuda")
    got = pv.gather(0, ids)
    assert got.shape == (100,)
    es = v.element_size()
    assert torch.equal(got.view(torch.uint8), v.view(torch.uint8).view(-1, es)[ids].reshape(-1))


def test_launch_count_does_not_depend_on_the_ids():
    torch.manual_seed(6)
    w = (torch.randn(8192, 256, device="cuda") * 0.02).to(torch.bfloat16)   # 4 MiB: 16 chunks of 512 rows
    plan = _plan_of(w)
    scratch = torch.empty(plan.gather_scratch_bytes(0, 4), dtype=torch.uint8, device="cuda")
    counts = []
    for ids in (torch.full((64,), 3, device="cuda"), torch.arange(0, 8192, 128, device="cuda")):
        before = _native.launch_count()
        got = plan.gather(0, ids, scratch=scratch)
        counts.append(_native.launch_count() - before)
        assert torch.equal(got, w[ids])
    assert counts[0] == counts[1] == 1 + 2 * 4, counts   # 64 ids x 1 chunk each may touch all 16 chunks: 4 passes of 4


def test_graph_replay_with_new_ids():
    torch.manual_seed(7)
    w = (torch.randn(4096, 512, device="cuda") * 0.02).to(torch.bfloat16)
    plan = _plan_of(w)
    ids = torch.zeros(48, dtype=torch.int64, device="cuda")
    scratch = torch.empty(plan.gather_scratch_bytes(0, 64), dtype=torch.uint8, device="cuda")
    out = torch.empty(48, 512, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.gather(0, ids, out=out, scratch=scratch)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.gather(0, ids, out=out, scratch=scratch)
    for seed in range(4):
        new = torch.randint(0, 4096, (48,), device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
        ids.copy_(new)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, w[new]), seed
    plan.check()


def test_out_of_range_ids():
    torch.manual_seed(8)
    w = (torch.randn(1000, 256, device="cuda") * 0.02).to(torch.bfloat16)
    plan = _plan_of(w)
    ids = torch.tensor([5, -1, 999, 1000, 1 << 40, 0, -(1 << 40)], device="cuda")
    got = plan.gather(0, ids)
    good = torch.tensor([True, False, True, False, False, True, False], device="cuda")
    assert torch.equal(got[good], w[ids[good]])
    assert torch.all(got[~good].view(torch.int16) == 0)
    with pytest.raises(IndexError):
        plan.check()


def test_corrupt_stream_refused_at_create():
    torch.manual_seed(9)
    w = (torch.randn(1000, 256, device="cuda") * 0.02).to(torch.bfloat16)
    s = ZipNN(input_format="torch").compress(w).clone()
    s[-40:] ^= 0x5A
    with pytest.raises(Exception, match="corrupt"):
        DecodePlan([s])


def test_host_rejections_launch_nothing(monkeypatch):
    DP._set_env(monkeypatch, {})
    case = next(c for c in H.box_streams(2) if c.name.startswith("c4096_"))   # whole item 0, a box item 1
    whole = DP.Item(case.name, case.body, case.G, case.bits, case.chunk, case.data.size, case.data)
    box = (16, 3, 4096, 100)
    boxed = DP.Item(case.name + "-box", case.body, case.G, case.bits, case.chunk, case.data.size, H.expect(case, box), box=box)
    p = DP.Plan([whole, boxed])
    assert p.rc == 0
    L = _native.lib()
    orig = case.data.size
    bad_r = next(r for r in range(2, orig) if orig % r)   # (the stream has a ragged, odd length)
    rc, sb = scratch_size(p, 0, 1, 4)
    assert rc == 0
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    out = torch.full((256,), CANARY, dtype=torch.uint8, device="cuda")
    bad = [("id_bytes", dict(id_bytes=2), _native.E_ARG), ("row 0", dict(R=0), _native.E_ARG),
           ("row not dividing", dict(R=bad_r), _native.E_ARG), ("null ids", dict(ids=0), _native.E_ARG),
           ("null out", dict(out=0), _native.E_ARG), ("null scratch", dict(scratch=0), _native.E_ARG),
           ("short scratch", dict(sb=scratch_size(p, 0, 1, 1)[1] - 1), _native.E_ARG), ("item -1", dict(item=-1), _native.E_ARG),
           ("item 2", dict(item=2), _native.E_ARG), ("box item", dict(item=1), _native.E_UNSUPPORTED)]
    for name, kw, want in bad:
        a = dict(item=0, R=1, ids=ids.data_ptr(), id_bytes=8, out=out.data_ptr(), scratch=scratch.data_ptr(), sb=sb)
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_gather(C.byref(p.plan), a["item"], a["R"], a["ids"], 4, a["id_bytes"], a["out"], a["scratch"],
                                             a["sb"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    assert torch.all(out == CANARY)
    assert scratch_size(p, 1, 1, 1)[0] == _native.E_UNSUPPORTED and scratch_size(p, 0, 1, 0)[0] == _native.E_ARG
    # a plan without a segment index
    DP._set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    q = DP.Plan([DP.Item(case.name, case.body, case.G, case.bits, case.chunk, orig, case.data)])
    assert q.rc == 0
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_gather(C.byref(q.plan), 0, 1, ids.data_ptr(), 4, 8, out.data_ptr(), scratch.data_ptr(), sb,
                                           _st()) == _native.E_UNSUPPORTED
    assert _native.launch_count() == before and torch.all(out == CANARY)
