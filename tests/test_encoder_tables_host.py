"""The encoder's table build on crafted histograms (encoder_tables.py), on the host, against the reference.

  * huf_serial.cuh's restatement (code lengths, table log, header bytes) equals the reference's own
    HUF_optimalTableLog / HUF_buildCTable / HUF_writeCTable, and the oracle's, for every crafted histogram;
  * the oracle's HUF_compress equals the reference's on every crafted plane at the chunk's capacity, and the host run
    of warp_block_decision (encoder_tables.decision) stores what the reference stores;
  * the crafted histograms reach every named branch of the table build (one test names any that is never reached);
  * the oracle's stream of every crafted tensor equals the reference's zipnn_core stream.

The reference-backed tests skip only when the reference build (oracle/_ref) is absent.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import encoder_tables as ET
from oracle import oracle as O


class CElt(C.Structure):
    _fields_ = [("val", C.c_uint16), ("nbBits", C.c_uint8)]


@functools.lru_cache(maxsize=None)
def _ref():
    L = O.ref_cdll()
    if L is None:
        return None
    L.HUF_optimalTableLog.restype = C.c_uint
    L.HUF_optimalTableLog.argtypes = [C.c_uint, C.c_size_t, C.c_uint]
    L.HUF_buildCTable.restype = C.c_size_t
    L.HUF_buildCTable.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint]
    L.HUF_writeCTable.restype = C.c_size_t
    L.HUF_writeCTable.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint, C.c_uint]
    return L


def need_ref():
    L = _ref()
    if L is None or O.ref_core() is None:
        pytest.skip("the reference build (oracle/_ref) is absent")
    return L


def ref_table(L, counts):
    """The reference's table for a histogram: (nbBits[256], val[256], header bytes or None, table log)."""
    cnt = np.ascontiguousarray(counts, dtype=np.uint32)
    n = int(cnt.sum())
    max_sym = int(np.nonzero(cnt)[0][-1])
    log = L.HUF_optimalTableLog(11, n, max_sym)
    tree = (CElt * 256)()
    r = L.HUF_buildCTable(tree, cnt.ctypes.data, max_sym, log)
    assert not L.HUF_isError(r)
    nb = np.array([tree[s].nbBits if s <= max_sym else 0 for s in range(256)], np.uint8)
    val = np.array([tree[s].val if s <= max_sym else 0 for s in range(256)], np.uint16)
    dst = np.zeros(1024, np.uint8)
    h = L.HUF_writeCTable(dst.ctypes.data, dst.size, tree, max_sym, int(r))
    return nb, val, (None if L.HUF_isError(h) else dst[:h].tobytes()), int(r)


def crafted_histograms():
    """Every histogram the cases were built from, once."""
    seen, out = set(), []
    for plen, cat in ET._catalogs().items():
        for name, c, _ in cat:
            key = np.asarray(c, np.int64).tobytes()
            if key not in seen:
                seen.add(key)
                out.append((f"{plen}/{name}", np.asarray(c, np.int64)))
    for plen, need in ((131072, 512), (32704, 512), (65536, 4096), (40001, 4096)):
        out.append((f"{plen}/eleven", ET.eleven_bit_counts(plen, need, plen if plen != 65536 else 7)))
    for name, c, _ in ET.depth_cases(65536):
        out.append((f"65536/{name}", np.asarray(c, np.int64)))
    out.append(("4252/slow_fse", np.asarray(ET.SLOW_FSE, np.int64)))
    return out


def test_restatement_matches_reference_tables():
    L = need_ref()
    forms = set()
    for name, c in crafted_histograms():
        if (c > 0).sum() < 2:
            continue
        t = ET.table(c)
        nb, val, hdr, lg = ref_table(L, c)
        present = c > 0
        assert t.lg == lg, (name, t.lg, lg)
        assert np.array_equal(t.nb, nb), name
        assert np.array_equal(t.val[present], val[present]), name
        assert t.hdr == hdr, (name, t.hdr, hdr)
        onb, oval, ohdr, olog = O.huf_table_from_counts(c.astype(np.uint32), int(c.sum()))
        assert olog == lg and np.array_equal(onb, nb) and ohdr == hdr, name
        forms.add("raw" if hdr is None else ("fse" if hdr[0] < 128 else "nibble"))
    assert forms == {"fse", "nibble", "raw"}


def test_branches_reached():
    """Every named branch of the table build is taken by at least one crafted histogram."""
    reached = set()
    for _, c in crafted_histograms():
        if (c > 0).sum() >= 2:
            reached |= ET.table(c).trace
    missing = [b for b in ET.REQUIRED if b not in reached]
    assert not missing, f"branches never reached: {missing}"


def test_families_name_their_branches():
    """The family that was built for a branch reaches it: the limiter's on deep trees, the reduced log on small planes,
    the header forms on their histograms."""
    cat = ET._catalogs()
    names = lambda plen: {n.split("-")[0] for n, c, _ in cat[plen]}   # noqa: E731
    by = lambda plen, pre: [c for n, c, _ in cat[plen] if n.startswith(pre)]   # noqa: E731
    assert any("limit" in ET.table(c).trace for c in by(131072, "fib") + by(131072, "geo") + by(131072, "head"))
    assert all("limit_below11" not in ET.table(c).trace for c in by(131072, ""))
    assert any("limit_below11" in ET.table(c).trace for c in by(2048, "small") + by(2048, "fib") + by(2048, "geo"))
    assert all("pack_rle" in ET.table(c).trace for c in by(4096, "packrle"))
    assert all("pack_distinct" in ET.table(c).trace for c in by(4096, "packdistinct"))
    assert len(by(4096, "slow")) == 3 and all("normalize_slow" in ET.table(c).trace for c in by(4096, "slow"))
    assert {"normalize_slow", "table_fse"} <= ET.table(ET.SLOW_FSE).trace
    assert any("table_raw" in ET.table(c).trace for c in by(32, "small") + by(2048, "small"))
    assert {"tie2", "tie256", "maxsym127", "maxsym128", "maxsym129", "rle", "largest"} <= names(4096)
    # hsize + 12 one byte either side of the plane length
    hs = {n.split("+")[0] for n, c, _ in cat[32] if n.startswith("hsize")}
    assert hs == {"hsize19", "hsize20", "hsize21"}


def test_early_out_model():
    """huf_early_out on the edges of huf_compress.c:658, 673-674: the largest count at plen (RLE), plen - 1,
    (plen >> 7) + 4 (raw by the heuristic) and + 5 (the table is built); planes over 128 KiB are raw."""
    E = ET.emu()
    for plen, largest, want in ((0, 0, 0), (2, 2, 1), (2, 1, 0), (5, 4, 0), (6, 5, 2), (32, 32, 1), (32, 31, 2),
                                (32, 4, 0), (32, 5, 2), (2048, 20, 0), (2048, 21, 2), (2048, 2047, 2),
                                (2048, 2048, 1), (131072, 1028, 0), (131072, 1029, 2), (131072, 131072, 1),
                                (131073, 131073, 0), (131073, 5000, 0)):
        assert E.emu_early_out(largest, plen) == want, (plen, largest)


@pytest.mark.parametrize("layout", ET.LAYOUTS, ids=lambda x: f"G{x[0]}b{x[1]}")
def test_blocks_and_decisions_match_reference(layout):
    """Every crafted plane: the oracle's HUF_compress = the reference's at the chunk's capacity, and the host run of
    the device's block decision stores what the reference stores at the case's threshold."""
    need_ref()
    for case in ET.cases(*layout):
        for c, planes in enumerate(case.planes):
            for g, plane in enumerate(planes):
                where = (case.name, c, g, case.names[c][g])
                r, blk = O.huf_compress(plane, case.chunk)
                rr, rblk = O.ref_huf_compress(plane, case.chunk)
                assert (r, blk) == (rr, rblk), where
                stored = int(rr) if (rr != O.ERR and rr > 0 and rr < plane.size * np.float64(np.float32(case.thr))) else 0
                assert ET.decision(plane, case.chunk, case.thr) == stored, where


@pytest.mark.parametrize("layout", ET.LAYOUTS, ids=lambda x: f"G{x[0]}b{x[1]}")
def test_oracle_stream_matches_reference(layout):
    need_ref()
    ref = O.ref_core()
    G, bits = layout
    for case in ET.cases(G, bits):
        want = bytes(ref.zipnn_core(ET.header(), bytearray(case.data.tobytes()), G, bits, ET.bytes_mode(G), 0, case.chunk,
                                    case.thr, 10, 4))
        assert case.oracle().tobytes() == want, case.name
