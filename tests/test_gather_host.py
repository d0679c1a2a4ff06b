"""Host-side models of the decode plan gather (gather.cuh, zipnn_b200_decode_plan_gather), checked against numpy, and
the selection and report rules of resident gathers (no GPU).

  * the chunks a row covers and the bound on them (span), at every chunk size chunk_settings.py uses;
  * the pass partition: every touched chunk falls in exactly one pass, and the launch count is a function of n;
  * the scratch sizing;
  * which embeddings gather=True selects, tied and untied, with explicit selections;
  * the report arithmetic.
"""
import numpy as np
import pytest
import torch

import chunk_settings as CS
from zipnn_b200.resident import _Entry, _Resident, _options, _with_prefetch, gathers, select, split_gathers


def round_up(v, a):
    return (v + a - 1) // a * a


def span(row_bytes, chunk, K):
    """gather_span: the most chunks a row can touch, wherever it starts."""
    return min(K, (row_bytes + chunk - 2) // chunk + 1)


def cover(row_id, row_bytes, chunk):
    """Chunks row `row_id` covers (k_gather_index's marks)."""
    b = row_id * row_bytes
    return list(range(b // chunk, (b + row_bytes - 1) // chunk + 1))


def passes(n, row_bytes, chunk, K, slots):
    s = span(row_bytes, chunk, K)
    most = K if n > K // s else min(K, n * s)
    return (most + slots - 1) // slots


def launches(n, row_bytes, chunk, K, slots):
    return 0 if n == 0 else 1 + 2 * passes(n, row_bytes, chunk, K, slots)


def scratch_bytes(G, chunk, orig, slots):
    K = -(-orig // chunk)
    pstride = round_up(chunk // G, 16) + 16
    list_off = 256
    pos_off = round_up(list_off + 4 * K, 256)
    inv_off = round_up(pos_off + 4 * K, 256)
    planes_off = round_up(inv_off + 4 * G * K, 256)
    return planes_off + min(slots, K) * G * pstride


def chunk_sizes():
    out = set()
    for G in (1, 2, 4):
        out |= {1 << e for e in range(G.bit_length() - 1, 13)} | set(CS.BIG_CHUNKS)
    return sorted(out | {131072, 262144})


@pytest.mark.parametrize("chunk", chunk_sizes())
def test_cover_and_span(chunk):
    rng = np.random.default_rng(chunk)
    for row_bytes in sorted({1, 2, 3, 16, 17, chunk - 1 if chunk > 1 else 1, chunk, chunk + 1, 3 * chunk + 5, 2 * chunk}):
        rows = int(rng.integers(1, 300 if row_bytes < 65536 else 6))
        orig = rows * row_bytes
        K = -(-orig // chunk)
        s = span(row_bytes, chunk, K)
        worst = 0
        for r in range(rows):
            c = cover(r, row_bytes, chunk)
            b = r * row_bytes
            # numpy: the chunk index of every byte of the row
            want = np.unique(np.arange(b, b + row_bytes) // chunk)
            assert c == list(want)
            worst = max(worst, len(c))
        assert worst <= s <= K
        # the bound is reached by some start offset (it is the maximum over starts, not just these rows)
        assert max(len(cover(0, row_bytes, chunk)), (chunk - 1 + row_bytes - 1) // chunk + 1) >= min(s, K)


@pytest.mark.parametrize("seed", range(6))
def test_pass_partition(seed):
    rng = np.random.default_rng(seed)
    chunk = int(2 ** rng.integers(2, 18))
    row_bytes = int(rng.integers(1, 3 * chunk))
    rows = int(rng.integers(1, 5000))
    K = -(-rows * row_bytes // chunk)
    slots = int(rng.integers(1, 70))
    for n in (1, 2, 7, 64, 1000):
        ids = rng.integers(0, rows, n)
        touched = sorted({c for r in ids for c in cover(int(r), row_bytes, chunk)})
        P = passes(n, row_bytes, chunk, K, slots)
        pos = {c: i for i, c in enumerate(touched)}
        owner = [pos[c] // slots for c in touched]
        assert all(0 <= p < P for p in owner)                      # every touched chunk is in exactly one pass
        assert len(touched) <= min(n * span(row_bytes, chunk, K), K)
        # the launch count depends on n only: ids all in one chunk give the same count as spread ones
        assert launches(n, row_bytes, chunk, K, slots) == 1 + 2 * P


@pytest.mark.parametrize("G", (1, 2, 4))
def test_scratch_sizing(G):
    for chunk in (G, 64, 4096, 262144):
        for orig in (chunk * 3 + G, chunk * 40):
            one = scratch_bytes(G, chunk, orig, 1)
            K = -(-orig // chunk)
            per = round_up(chunk // G, 16) + 16
            assert scratch_bytes(G, chunk, orig, 2) - one == G * per
            assert scratch_bytes(G, chunk, orig, 10 ** 6) == scratch_bytes(G, chunk, orig, K)   # capped to K
            assert one % 16 == 0 and one >= 12 * K


class WithForward(torch.nn.Embedding):
    def forward(self, x):
        return super().forward(x) * 2


class Plain(torch.nn.Embedding):
    pass


class Net(torch.nn.Module):
    def __init__(self, tied=True):
        super().__init__()
        self.emb = torch.nn.Embedding(50, 8)
        self.sub = Plain(50, 8)
        self.fwd = WithForward(50, 8)
        self.norm_emb = torch.nn.Embedding(50, 8, max_norm=1.0)
        self.head = torch.nn.Linear(8, 50, bias=False)
        if tied:
            self.head.weight = self.emb.weight


def _split(model, modules=None, gather=True):
    modules, groups = select(model, modules)
    where = {id(p): i for i, (p, _) in enumerate(groups)}
    per = [(m, [(n, where[id(p)]) for n, p in m._parameters.items() if p is not None and id(p) in where]) for m in modules]
    per = [(m, names) for m, names in per if names]
    return split_gathers(per, gather), groups


def test_which_embeddings_gather():
    net = Net()
    assert gathers(net.emb) and gathers(net.sub)
    assert not gathers(net.fwd) and not gathers(net.norm_emb) and not gathers(net.head)
    (whole, looked, own), groups = _split(net)
    assert [m for m, _ in looked] == [net.emb, net.sub]
    assert {m for m, _ in whole} == {net.fwd, net.norm_emb, net.head}
    tied = next(i for i, (p, _) in enumerate(groups) if p is net.emb.weight)
    assert own == [i for m, i in looked if m is net.sub] and tied not in own   # the tied head holds the stream
    (whole, looked, own), _ = _split(Net(tied=False))
    assert len(own) == 2                                              # untied: each embedding needs a plan of its own
    (whole, looked, _), _ = _split(net, gather=False)
    assert looked == [] and len(whole) == 5
    # an explicit selection without the head: the tied weight is owned outside the selection and stays dense
    (whole, looked, own), _ = _split(net, modules=[net.emb, net.sub, net.fwd])
    assert [m for m, _ in looked] == [net.sub] and [m for m, _ in whole] == [net.fwd]


def test_report_arithmetic():
    state = _Resident()
    state.scratch = torch.empty(100, dtype=torch.uint8)
    state.gather_scratch = state.scratch
    state.gathers = [object(), object()]
    state.gather_plan_bytes = 4096
    base = {"plan_bytes": 1}
    assert _with_prefetch(base, state, _options()) == base
    assert _with_prefetch(base, state, _options(gather=True)) == dict(base, gather_modules=2, gather_bytes=4096)
    state.gather_scratch = torch.empty(300, dtype=torch.uint8)   # a scratch of its own counts
    assert _with_prefetch(base, state, _options(gather=True))["gather_bytes"] == 4096 + 300
    assert _with_prefetch(base, None, _options(gather=True)) == dict(base, gather_modules=0, gather_bytes=0)


def test_mode_report_counts():
    """Each mode's module count comes from the entries' modes: a "matmul" module is also a matvec module, an fp8 module
    counts whether its products take its weight or torch dequantizes it."""
    state = _Resident()
    state.entries = [_Entry(None, None, [], mode) for mode in ("matmul", "matvec", "fp8", "fp8_torch", "experts", "experts", "decode")]
    state.select_scratch = torch.empty(7, dtype=torch.uint8)
    state.matvec_scratch_bytes, state.matmul_scratch_bytes, state.fp8_scratch_bytes = 1, 2, 3
    got = _with_prefetch({}, state, _options(matvec=8, matmul=64, experts=True, fp8=True))
    assert got == {"matvec_modules": 2, "matvec_scratch_bytes": 1, "matmul_modules": 1, "matmul_scratch_bytes": 2,
                   "experts_modules": 2, "experts_scratch_bytes": 7, "fp8_modules": 2, "fp8_scratch_bytes": 3}
    assert _with_prefetch({}, None, _options(prefetch=True)) == {"prefetch_out_bytes": 0}
