"""CPU self-checks of tests/plane_inputs.py: the inverse split, the plane families, the huff0 writer and the
host model of the decoders' branches.  No GPU."""
import numpy as np
import pytest

import plane_inputs as P
from oracle import oracle as O

LAYOUTS = [(1, 0), (2, 0), (2, 1), (4, 0), (4, 1)]


@pytest.mark.parametrize("G,bits", LAYOUTS)
def test_inverse_split_matches_oracle_split(G, bits):
    rng = np.random.default_rng(40 + 10 * G + bits)
    for chunk in (1024, 4096, 262144):
        for last in (chunk, G, 3 * G + 1, chunk - 1, chunk // 2 + 5, 4 * G + 3):
            lens = [chunk] * 2 + [last]
            chunks = [[rng.integers(0, 256, P.plane_len(n, G, g), dtype=np.uint8) for g in range(G)] for n in lens]
            data = P.tensor_from_planes(chunks, G, bits)
            assert data.size == sum(lens)
            got = P.planes_of(data, G, bits, chunk)
            for want_c, got_c in zip(chunks, got):
                for g in range(G):
                    assert np.array_equal(want_c[g], got_c[g]), (chunk, last, g)
            # and the other way round: any bytes -> planes -> the same bytes
            raw = rng.integers(0, 256, data.size, dtype=np.uint8)
            assert np.array_equal(P.tensor_from_planes(P.planes_of(raw, G, bits, chunk), G, bits), raw)


def test_families_have_the_table_shapes_they_are_named_for():
    rng = np.random.default_rng(1)
    n = 131072
    for name, log in (("eq2", 1), ("eq4", 2), ("eq8", 3), ("eq16", 4), ("eq64", 6), ("eq128", 7)):
        nb = P.code_lengths(P.FAMILIES[name](rng, n))
        present = nb[nb > 0]
        assert present.size == 1 << log and np.all(present == log), name
    assert P.code_lengths(P.FAMILIES["fib"](rng, n)).max() == 11
    for name in ("zipf256", "dirichlet256", "heavy256"):
        plane = P.FAMILIES[name](rng, n)
        r, blk = O.huf_compress(plane)
        assert r not in (0, 1, O.ERR) and np.unique(plane).size > 200, name
        h, w, _ = O.huf_read_table(np.frombuffer(blk, dtype=np.uint8))
        assert blk[0] < 128 and (name == "heavy256" or 50 <= h <= 128), (name, h)  # tANS-coded weights
    assert np.unique(P.FAMILIES["logexp"](rng, n)).size > 75
    assert O.huf_compress(P.FAMILIES["const"](rng, n))[0] == 1
    assert O.huf_compress(P.FAMILIES["raw"](rng, n))[0] == 0
    c = P.clustered(P.FAMILIES["fib"](rng, n))
    nb = P.code_lengths(c)
    q = nb[c[: n // 4]]
    assert np.all(np.diff(q.astype(np.int32)) <= 0) and q[0] == 11


def test_writer_canonical_values_match_the_oracle_tables():
    rng = np.random.default_rng(2)
    for name in ("eq4", "eq16", "geo5", "geo3", "fib", "zipf256", "dirichlet256", "heavy256", "logexp"):
        for n in (2048, 32768, 131072):
            plane = P.FAMILIES[name](rng, n)
            cnt = np.bincount(plane, minlength=256).astype(np.uint32)
            nb, val, _, log = O.huf_table_from_counts(cnt, n)
            assert nb.max() == log
            mine = P.canonical_values(nb)
            assert np.array_equal(mine[nb > 0], val[nb > 0]), (name, n)


def test_writer_blocks_equal_the_oracle_where_it_writes_raw_weights():
    rng = np.random.default_rng(3)
    same = 0
    for it in range(60):
        k = int(rng.integers(2, 17))
        n = int(rng.choice([2048, 10000, 32768, 131072]))
        p = rng.dirichlet(np.ones(k) * float(rng.choice([0.3, 1.0, 5.0])))
        syms = np.sort(rng.choice(16 if it % 2 else k, k, replace=False))  # small alphabets: raw 4-bit weights
        plane = syms[rng.choice(k, n, p=p)].astype(np.uint8)
        r, blk = O.huf_compress(plane)
        if r in (0, 1, O.ERR) or blk[0] < 128:
            continue
        assert P.huf_block(P.code_lengths(plane), plane) == blk, it
        same += 1
    assert same >= 25


def test_writer_blocks_decode_with_the_oracle_and_the_reference():
    rng = np.random.default_rng(4)
    ref = O.ref_cdll()
    for it in range(80):
        max_len = int(rng.integers(1, 13))
        nsym = int(rng.integers(2, min(129, 1 << max_len) + 1))
        nb = P.kraft_lengths(rng, nsym, max_len)
        assert sum(2.0 ** -nb[nb > 0].astype(np.float64)) == 1.0
        n = int(rng.choice([2048, 5000, 32768, 131072]))
        long_syms = np.nonzero(nb == nb.max())[0]
        plane = P.plane_for_lengths(rng, nb, n, hot=int(long_syms[0]) if it % 3 == 0 else None)
        blk = P.huf_block(nb, plane)
        if len(blk) >= n:
            continue
        h, w, log = O.huf_read_table(np.frombuffer(blk, dtype=np.uint8))
        assert log == nb.max() and w.size == np.nonzero(nb)[0][-1] + 1
        assert np.array_equal(O.huf_decompress(blk, n), plane), it
        if ref is not None:
            dst = np.zeros(n + 64, dtype=np.uint8)
            src = np.frombuffer(blk, dtype=np.uint8).copy()
            r = ref.HUF_decompress(dst.ctypes.data, n, src.ctypes.data, src.size)
            assert not ref.HUF_isError(r) and np.array_equal(dst[:n], plane), it


def test_assembled_streams_decode_with_the_oracle():
    rng = np.random.default_rng(5)
    G, bits, chunk = 2, 1, 4096
    planes = [[P.FAMILIES["raw"](rng, 2048), P.FAMILIES[f](rng, 2048)] for f in ("eq16", "geo3", "const", "raw")]
    planes.append([P.FAMILIES["raw"](rng, 100), P.FAMILIES["eq4"](rng, 100)])
    data = P.tensor_from_planes(planes, G, bits)

    def make(g, c, plane):
        r, blk = O.huf_compress(plane)
        if r == 0:
            return 0, plane.tobytes()
        if r == 1:
            return 1, plane[:1].tobytes()
        return 1, blk

    body = P.assemble_body(P.stream_items(planes, G, make), G)
    want = O.zipnn_compress(bytes(32), data, G, bits, 10, chunk)[32:]
    assert np.array_equal(body, want)
    assert np.array_equal(O.zipnn_decompress(body, G, bits, 10, chunk, data.size), data)


def test_predictor_on_the_issue_numbers():
    """The bitstream lengths around the shared-memory cap of the sync decoder, table logs, tails and
    alignment, on oracle streams."""
    rng = np.random.default_rng(6)
    # fp8: a full plane of 128 equiprobable symbols -> quarters one byte over the cap; a 131068-byte last chunk -> at it
    full = P.FAMILIES["eq128"](rng, 131072)
    rag = P.FAMILIES["eq128"](rng, 131068)
    data = np.concatenate([full, rag])
    body = O.zipnn_compress(bytes(32), data, 1, 0, 10, 131072)[32:]
    pr = P.predict(body, 1, 0, 131072, data.size)
    assert pr["items"][0][0].s_len == [28673] * 4
    assert max(pr["items"][0][1].s_len) == P.SYNC_STREAM_CAP
    assert pr["mode"] == ["fused", "general"] and pr["pb"] == 0
    assert pr["items"][0][0].x_cut == {0: 8, 5: 2048} and pr["items"][0][0].fixed_len == 7
    # bf16 Gaussian: exponent plane coded, x_cut 64 under PB = 5, every warp regular
    x = (rng.standard_normal(131072 * 8) * 0.02).astype(np.float32)
    bf = (x.view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)
    body = O.zipnn_compress(bytes(32), bf, 2, 1, 10, 262144)[32:]
    pr = P.predict(body, 2, 1, 262144, bf.size, body_addr_mod16=5)
    assert pr["pb"] == 5 and pr["mode"] == ["fused"] * 8 and pr["regular"] == [True]
    assert all(pr["items"][1][c].x_cut[5] == 64 for c in range(8))
    assert pr["side_r0"][0] == (5 + 9 * 2 * 8) & 15


def test_predictor_pool_prefix_and_demotion():
    """Hand-computed pool prefixes: a chunk whose running total passes the capacity is demoted, and so is every
    later chunk of its warp."""
    rng = np.random.default_rng(7)
    G, bits, chunk = 2, 1, 4096
    fams = ["eq16"] * 3 + ["eq128"] + ["eq16"] * 4 + ["eq16"] * 8
    planes = [[P.FAMILIES["raw"](rng, 2048), P.FAMILIES[f](rng, 2048)] for f in fams]
    data = P.tensor_from_planes(planes, G, bits)
    body = O.zipnn_compress(bytes(32), data, G, bits, 10, chunk)[32:]
    pr = P.predict(body, G, bits, chunk, data.size)
    assert pr["mode"] == ["fused"] * 16
    assert [pr["items"][1][c].x_cut[5] for c in range(4)] == [64, 64, 64, 2048]
    assert [pr["fused"][c] for c in range(8)] == ["fused"] * 3 + ["demoted"] * 5
    assert pr["pool_run"] == [64 * 7 + 2048, 64 * 8] and pr["regular"] == [False, True]


def test_misaligned_sync_guesses_are_predicted():
    rng = np.random.default_rng(8)
    plane = P.FAMILIES["eq4"](rng, 4 * 25601)
    body = O.zipnn_compress(bytes(32), plane, 1, 0, 10, 131072)[32:]
    it = P.predict(body, 1, 0, 131072, plane.size)["items"][0][0]
    assert it.fixed_len == 2 and it.segbits == [201] * 4 and P.misaligned_sync_guesses(it) == 4
    plane = P.FAMILIES["eq4"](rng, 131072)
    body = O.zipnn_compress(bytes(32), plane, 1, 0, 10, 131072)[32:]
    it = P.predict(body, 1, 0, 131072, plane.size)["items"][0][0]
    assert it.segbits == [256] * 4 and P.misaligned_sync_guesses(it) == 0
