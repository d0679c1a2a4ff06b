"""The corrupted-stream corpus and its verdict model, checked on the CPU (tests/corrupt_streams.py).

  * every base sends its chunks down the decoder path it is named for, and every mutant changes only its field;
  * the model agrees with the port on every mutant but the DIVERGENCES classes, and the port's block verdicts
    are the reference's HUF_decompress4X1 (tests/golden/corrupt_verdicts.json);
  * the reference's double-symbol decoder, which HUF_decompress picks for many planes, accepts blocks that 4X1
    rejects (DESIGN §7): counted here, and no mutant that every decoder accepts is decoded differently;
  * every path has rejected mutants of every field class and accepted mutants that change the output;
  * the slab decoder's host check refuses a row past its group's total at the slab that holds it.
"""
import hashlib
import json
import os
from collections import Counter, defaultdict

import numpy as np
import pytest

import corrupt_streams as CS
import plane_inputs as P
import test_host_pipelines_host as HM
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "corrupt_verdicts.json")
BASES = list(CS.bases())


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


def _digest(b):
    return None if b is None else hashlib.sha256(bytes(b)).hexdigest()[:16]


def test_bases_take_their_paths():
    for name, b in CS.bases().items():
        modes = Counter(b.pr["mode"])
        if b.path == "fused":
            assert modes["fused"] >= 3 and b.pr["mode"][-1] == "general", name
            assert any(b.pr["fused"].get(c) == "fused" for c in range(b.K)), name
        elif b.path == "general":
            assert modes["general"] == b.K <= 64, name
        elif b.path == "overflow":
            assert modes["general"] == b.K > 64, name
        elif b.path == "ring":
            assert max(max(b.pr["items"][b.G - 1][c].s_len) for c in range(b.K)) > P.SYNC_STREAM_CAP, name
        else:
            assert name in ("raw_only", "rle_only", "empty_plane"), name
    assert CS.bases()["bf16_fused"].pr["regular"][0], "the first warp of bf16_fused takes the bulk-tensor side path"
    kinds = {n: {it.kind for row in CS.bases()[n].pr["items"] for it in row} for n in ("raw_only", "rle_only")}
    assert kinds == {"raw_only": {"raw"}, "rle_only": {"rle"}}


@pytest.mark.parametrize("name", BASES)
def test_mutants_change_only_their_field(name):
    b = CS.bases()[name]
    base_items = CS.items(b.body, b.G, b.K)
    ids = set()
    for m in CS.mutants(name):
        assert m.id not in ids
        ids.add(m.id)
        f = m.field
        if f[0] == "bytes":
            assert m.body.size == b.body.size
            diff = np.nonzero(m.body != b.body)[0]
            assert diff.size and f[1] <= diff.min() and diff.max() < f[2], m.id
        elif f[0] == "prefix":
            assert m.body.size == f[1] < b.body.size and np.array_equal(m.body, b.body[: f[1]]), m.id
        elif f[0] == "extend":
            assert m.body.size == b.body.size + f[1] and np.array_equal(m.body[: b.body.size], b.body), m.id
        else:
            # block mutants (and stored items made longer) keep a consistent container: same type rows, rows
            # that add up to the payload, every other item unchanged
            _, g, c = f
            K, G = b.K, b.G
            assert np.array_equal(m.body[: G * K], b.body[: G * K]), m.id
            _, cum, payload0 = CS.split(m.body, G, K)
            assert payload0 + sum(cum[h][K - 1] for h in range(G)) == m.body.size, m.id
            got = CS.items(m.body, G, K)
            changed = [(h, d) for h in range(G) for d in range(K) if got[h][d] != base_items[h][d]]
            assert changed == [(g, c)], (m.id, changed)


@pytest.mark.parametrize("name", BASES)
def test_mutated_chunks_keep_their_decoder_path(name):
    """A block mutant's chunk takes the decoder path of the base's chunk (plane_inputs.predict on the mutant), so
    each path's own rejection is what the mutant exercises.  (Mutants whose table description no longer parses
    are refused before any path is chosen.)"""
    b = CS.bases()[name]
    n = 0
    for m in CS.mutants(name):
        if m.kind != "block":
            continue
        try:
            pr = P.predict(m.body, b.G, b.bits, b.chunk, b.orig)
        except (ValueError, IndexError):
            continue
        assert pr["mode"][m.c] == b.pr["mode"][m.c], (m.id, pr["mode"][m.c], b.pr["mode"][m.c])
        n += 1
    assert n or not any(it.kind == "huf" for row in b.pr["items"] for it in row), name


_VERDICTS = {}


def verdicts(name):
    """[(mutant, model verdict)] of one base, computed once per session."""
    if name not in _VERDICTS:
        b = CS.bases()[name]
        _VERDICTS[name] = [(m, CS.verdict(b, m.body)) for m in CS.mutants(name)]
    return _VERDICTS[name]


@pytest.mark.parametrize("name", BASES)
def test_model_matches_the_port(name):
    """The model is the port on every mutant, except the DIVERGENCES classes; each of those is cited in DESIGN."""
    b = CS.bases()[name]
    seen = Counter()
    for m, v in verdicts(name):
        st, data = CS.port_status(b, m.body)
        div = CS.divergence(m, v)
        if div:
            seen[div] += 1
            if div == "raw_long":
                assert v.status == CS.CORRUPT and st == CS.OK, m.id     # the port reads the plane's length only
            continue
        assert v.status == st, (m.id, v.status, st)
        if st == CS.OK:
            assert np.array_equal(v.data, data), m.id
    with open(os.path.join(os.path.dirname(HERE), "DESIGN.md")) as f:
        design = f.read()
    for div in seen:
        assert CS.DIVERGENCES[div].split(":")[0] in ("DESIGN §6", "DESIGN §7")
    assert "refused" in design and "stored item longer than its plane" in design


def test_port_is_the_reference_4x1_on_every_block_mutant():
    fx = _fixture()
    assert fx["decoders"] == ["HUF_decompress", "HUF_decompress4X1", "HUF_decompress4X2"]
    ref = fx["blocks"]
    n = 0
    clamp = 0
    for m in CS.all_mutants():
        if m.kind != "block":
            continue
        blk, dlen = CS.block_of(m)
        try:
            port = _digest(O.huf_decompress(blk, dlen))
        except ValueError:
            port = None
        huf, x1, x2 = ref[m.id]
        assert port == x1, m.id
        if huf is not None and x1 is not None:
            assert huf == x1 == x2, m.id      # accepted by every decoder: the same bytes
        if x1 is None and x2 is not None:
            clamp += 1
        n += 1
    assert n == len(ref)
    # the double-symbol decoder's clamp on the last symbol (DESIGN §7) accepts blocks the single-symbol one rejects
    assert clamp > 0


def test_fixture_regenerates_byte_identical():
    if O.ref_cdll() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    import make_golden_corrupt as MG
    with open(FIXTURE) as f:
        assert MG.render() == f.read()


def test_every_path_has_rejected_and_silent_mutants():
    """For each decoder path: a rejected mutant of every field class it has, and an accepted mutant whose output
    differs from the base's (wrong bytes that no check can see: the stream format has no checksum)."""
    rejected, silent = defaultdict(set), defaultdict(int)
    classes = defaultdict(set)
    for name, b in CS.bases().items():
        for m, v in verdicts(name):
            classes[b.path].add(m.cls)
            if v.status != CS.OK:
                rejected[b.path].add(m.cls)
            elif not np.array_equal(v.data, b.data):
                silent[b.path] += 1
    for path in ("fused", "general", "overflow", "ring"):
        # (the overflow base codes every plane: nothing is stored; the ring base's tables have more symbols than
        # the direct weight form can describe)
        want = set(CS.CONTAINER + CS.BLOCK) - {"trailing", "empty_huf"} - {"overflow": {"raw_long"}, "ring": {"weights"}}.get(path, set())
        assert classes[path] >= want, (path, want - classes[path])
        assert rejected[path] >= want, (path, want - rejected[path])
        assert silent[path] > 0, path
    assert "empty_huf" in rejected["plain"]


def test_host_slab_check_names_the_slab_of_a_row_past_the_total():
    """A row inside the last group that stays within one slab of its neighbour but points past the group's total:
    the slab decoder would copy from past the end of the caller's buffer.  Refused at that slab, before any work."""
    G, chunk, n, per = 2, 4096, 7 * 4096 - 5, 2
    data = HM.planned_bytes(HM.DECODE_PATTERN[2], G, 1, chunk, n, 3)
    body = O.zipnn_compress(HM.header32(n), data, G, 1, 10, chunk)[32:].copy()
    K = 7
    cum = body[G * K: 9 * G * K].view("<u8").reshape(G, K)
    i = 1                                          # slab 1 holds chunks 2 and 3
    cum[G - 1, 3] = cum[G - 1, K - 1] + 100        # past the group's total, < slab_max above its low row
    assert cum[G - 1, 3] - cum[G - 1, 1] <= per * chunk
    assert HM.decode_host_check(body, G, chunk, n, per) == ("row", i)
