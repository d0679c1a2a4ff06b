"""Host side of the multi-item plan tests (test_multi_item_plans_gpu.py): every layout, in every rotation the GPU tests
use, reaches what it is built for, so that a layout that stops reaching its branch fails here instead of passing
vacuously there.

  * every target is first, in the middle and last in some rotation, and in some rotation its piece index differs
    from its item index (an empty or split item in front of it);
  * every target behind the first one has a non-zero seg_base;
  * the split item has at least two pieces, the box and empty items none of their own, the general-mode item has
    general chunks, the constant item no Huffman-coded plane, the raw item no coded plane at all;
  * every matvec target is fused in every chunk, and every target has a decoy of equal geometry and other bytes.
"""
import numpy as np
import pytest

import multi_item_plans as M


@pytest.mark.parametrize("name", M.LAYOUTS)
def test_every_rotation_reaches_its_cases(name):
    entries, env = M.layout(name)
    assert 6 <= len(entries) <= 12
    limit = M.limit_of(env)
    rots = M.placements(entries)
    seen, shifted = {}, set()
    for r in rots:
        es = M.rotate(entries, r)
        m = M.Model(es, limit)
        targets = [i for i, e in enumerate(es) if e.kind == "target"]
        shifted |= {es[i].name for i in targets if m.piece[i] != i}
        assert all(m.seg_base[m.piece[i]] > 0 for i in targets[1:]), (name, r)
        for i, e in enumerate(es):
            if e.kind == "target":
                seen.setdefault(e.name, set()).add("first" if i == 0 else ("last" if i == len(es) - 1 else
                                                                           ("middle" if i == len(es) // 2 else "other")))
            if e.kind in ("box", "split", "empty"):
                assert m.piece[i] == -1
            else:
                assert m.piece[i] >= 0 and m.n_pieces(i) == 1, e.name
        # the plans of DecodePlan hold no boxes: their targets keep a non-zero seg_base behind the first
        dp = M.without_boxes(es)
        md = M.Model(dp, limit)
        assert all(md.seg_base[md.piece[i]] > 0 for i in [i for i, e in enumerate(dp) if e.kind == "target"][1:]), (name, r)
    for t, where in seen.items():
        assert {"first", "middle", "last"} <= where, (name, t, where)
    assert shifted == set(seen), ("targets never behind an empty or split item", set(seen) - shifted)


@pytest.mark.parametrize("name", M.LAYOUTS)
def test_kinds_and_decoys(name):
    entries, env = M.layout(name)
    by = {e.name: e for e in entries}
    limit = M.limit_of(env)
    m = M.Model(entries, limit)
    kinds = {e.kind for e in entries}
    for i, e in enumerate(entries):
        if e.kind == "target":
            d = by[e.decoy]
            assert d.kind == "decoy" and (d.dtype, d.shape, d.chunk, d.orig) == (e.dtype, e.shape, e.chunk, e.orig)
            assert not np.array_equal(d.data, e.data)
            assert np.all(np.any(d.rows() != e.rows(), axis=1)), "every row differs from the decoy's"
            assert e.coded(0, e.K) > 0
            assert e.eligible == e.matvec == d.eligible, e.name
            if e.matvec:
                assert e.dtype in M.MATVEC_DTYPES and e.fused, e.name
                assert e.shape[-1] * e.orig // int(np.prod(e.shape)) % 16 == 0, "rows of a multiple of 16 bytes"
            else:
                assert e.dtype not in M.MATVEC_DTYPES or not e.fused, "a float target that is not multiplied"
        elif e.kind == "split":
            assert m.n_pieces(i) >= 2 and e.coded(0, e.K) > 0
        elif e.kind == "general":
            assert "general" in e.pr["mode"] and "fused" not in e.pr["mode"]
        elif e.kind == "const":
            assert e.pr["mode"] == ["plain"] * e.K and all(it.kind == "rle" for row in e.pr["items"] for it in row)
        elif e.kind == "raw":
            assert e.coded(0, e.K) == 0 and e.pr["mode"] == ["plain"] * e.K
        elif e.kind == "empty":
            assert e.orig == 0 and m.n_pieces(i) == 0
        elif e.kind == "box":
            assert not e.whole and e.want.size == e.box[1] * e.box[3]
    want = {"L1": {"empty", "const", "target", "decoy"}, "L2": {"split", "general", "raw", "box", "empty", "target", "decoy"},
            "L3": {"empty", "target", "decoy"}}[name]
    assert want <= kinds, kinds
    if name == "L1":
        assert {e.dtype for e in entries if e.kind == "target"} == {"bf16", "fp8", "fp16", "fp32"}
        assert any(e.orig % e.chunk and e.kind == "target" for e in entries), "a ragged last chunk"
    if name == "L2":
        assert {e.dtype for e in entries if e.matvec} == set(M.MATVEC_DTYPES)
        assert all(e.K <= limit - 1 for e in entries if e.kind == "target")
    if name == "L3":
        assert {e.chunk for e in entries if e.kind == "target"} >= {512, 4096, 262144}


def test_seg_base_is_the_prefix_of_coded_items():
    """The model on a hand-checked case: L1 unrotated, where every item in front of a target is empty, constant (RLE:
    type-1 entries, sized like coded ones) or a 2-chunk tensor with one coded plane per chunk."""
    entries, _ = M.layout("L1")
    m = M.Model(entries)
    names = [e.name for e in entries]
    a = names.index("A_bf16")
    assert m.piece[a] == a - 1 and m.seg_base[m.piece[a]] == 2 * M.SEG_PER_ITEM
    w = names.index("W_fp32")
    assert m.piece[w] == w - 1 and m.seg_base[m.piece[w]] == (2 + 2 * 4) * M.SEG_PER_ITEM
    first, n, sym = m.seg_rows(w)
    assert n == 2 * M.SEG_PER_ITEM and sym == entries[w].orig // 4   # the exponent planes of two fp32 chunks
