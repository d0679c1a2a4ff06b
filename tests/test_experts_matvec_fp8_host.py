"""The selected experts matvec without a GPU: a numpy model of k_select_pairs (the per-expert pair tables), the scratch
formula, the experts_matvec option's refusals, the FP8Experts layouts it takes (transformers' own modules on the meta
device) and the report keys.
"""
import numpy as np
import pytest
import torch

from test_fp8_experts_host import _experts, experts_of, tiny_moe
from zipnn_b200 import resident as R
from zipnn_b200.plan import EXPERTS_MATVEC_MAX_TOKENS


# ------------------------------------------------------------------ k_select_pairs
def select_pairs(ids: np.ndarray, E: int, nt: int):
    """k_select_pairs: each pair counts the equal ids before and after it.  -> (cnt [E], tab [E, nt] (-1: unwritten),
    pos [n] (-1: unwritten), index error raised)."""
    ids = np.asarray(ids).reshape(-1)
    cnt = np.zeros(E, dtype=np.int64)
    tab = np.full((E, nt), -1, dtype=np.int64)
    pos = np.full(ids.size, -1, dtype=np.int64)
    err = False
    for p, e in enumerate(ids):
        if e < 0 or e >= E:
            err = True   # (k_select_index raises it)
            continue
        before, after = int(np.sum(ids[:p] == e)), int(np.sum(ids[p + 1:] == e))
        pos[p] = before
        if before < nt:
            tab[e, before] = p
        else:
            err = True
        if after == 0:
            cnt[e] = min(before + 1, nt)
    return cnt, tab, pos, err


def slots(T: int) -> int:
    return 1 if T <= 1 else 2 if T <= 2 else 4


def grouped(ids: np.ndarray, E: int):
    """The reference: per expert, its pair numbers in ascending order."""
    flat = np.asarray(ids).reshape(-1)
    return {e: [p for p in range(flat.size) if flat[p] == e] for e in range(E)}


@pytest.mark.parametrize("T,k,E", [(1, 1, 4), (1, 8, 128), (2, 2, 8), (3, 2, 8), (4, 8, 128), (4, 8, 9), (4, 1, 2)])
def test_pair_tables_of_top_k_routings(T, k, E):
    rng = np.random.default_rng(T * 100 + k * 10 + E)
    for _ in range(20):
        ids = np.stack([rng.permutation(E)[:k] for _ in range(T)])
        cnt, tab, pos, err = select_pairs(ids, E, slots(T))
        assert not err
        for e, ps in grouped(ids, E).items():
            assert cnt[e] == len(ps) <= T
            assert list(tab[e, :len(ps)]) == ps
            for j, p in enumerate(ps):
                assert pos[p] == j and tab[e, pos[p]] == p
        assert cnt.sum() == ids.size


def test_a_token_that_repeats_an_expert_raises_and_its_count_stops():
    # T = 1: one slot per expert; expert 5 twice
    cnt, tab, pos, err = select_pairs(np.array([[5, 5]]), 8, slots(1))
    assert err and cnt[5] == 1 and tab[5, 0] == 0 and list(pos) == [0, 1]
    # T = 2 (two slots): expert 3 three times
    cnt, tab, pos, err = select_pairs(np.array([[3, 3], [3, 1]]), 8, slots(2))
    assert err and cnt[3] == 2 and list(tab[3]) == [0, 1] and pos[2] == 2 and cnt[1] == 1
    # T = 3 has four slots: a repeat that fits raises nothing here (top-k never repeats)
    cnt, tab, pos, err = select_pairs(np.array([[3, 3], [3, 1], [0, 2]]), 8, slots(3))
    assert not err and cnt[3] == 3


def test_out_of_range_ids_mark_nothing():
    cnt, tab, pos, err = select_pairs(np.array([[2, -1], [8, 2]]), 8, slots(2))
    assert err and cnt[2] == 2 and list(tab[2]) == [0, 3] and pos[1] == -1 and pos[2] == -1
    assert cnt.sum() == 2


# ------------------------------------------------------------------ the scratch
def round_up(n, a=256):
    return (n + a - 1) // a * a


def block_rows(chunk_elems: int, inn: int, out: int) -> int:
    """matvec_block_elems / matvec_block_rows (matvec.cuh) for fp8 (16 elements per vector)."""
    nv = (chunk_elems // 4) // 16
    be = ((nv + 255) // 256) * 32 * 16
    return min((be + inn - 2) // inn + 1, out)


def scratch_bytes(select_bytes: int, E: int, n_ids: int, top_k: int, K: int, chunk_elems: int, inn: int, out: int) -> int:
    """The layout of zipnn_b200_decode_plan_experts_matvec_fp8: [select scratch][cnt E][tab E * nt][pos n][partials]."""
    nt = slots(n_ids // top_k)
    cnt = select_bytes
    tab = round_up(cnt + 4 * E)
    pos = round_up(tab + 4 * E * nt)
    part = round_up(pos + 4 * n_ids)
    return part + 32 * K * block_rows(chunk_elems, inn, E * out) * nt * 4


def test_scratch_formula_at_qwen3_30b_a3b_shapes():
    # gate_up_proj [128, 1536, 2048] in 128 KiB chunks: 3072 chunks, blocks of 4096 elements over rows of 2048: 3 rows
    assert block_rows(131072, 2048, 128 * 1536) == 3
    # down_proj [128, 2048, 768]: blocks of 4096 elements over rows of 768: 7 rows
    assert block_rows(131072, 768, 128 * 2048) == 7
    part = 32 * 3072 * 3 * 4 * 4
    assert scratch_bytes(0, 128, 32, 8, 3072, 131072, 2048, 1536) == round_up(round_up(round_up(512) + 4 * 128 * 4) + 4 * 32) + part
    assert part == 4718592
    # one token needs a quarter of the partial sums of four
    one = scratch_bytes(0, 128, 8, 8, 3072, 131072, 2048, 1536)
    assert one - round_up(round_up(round_up(512) + 512) + 32) == part // 4


# ------------------------------------------------------------------ the option
def test_options_refusals_and_messages():
    assert R._options().experts_matvec == 0
    assert R._options(fp8=True, experts=True, experts_matvec=EXPERTS_MATVEC_MAX_TOKENS).experts_matvec == EXPERTS_MATVEC_MAX_TOKENS
    for bad in (-1, EXPERTS_MATVEC_MAX_TOKENS + 1, 2.0, True, "4"):
        with pytest.raises(ValueError, match=f"experts_matvec must be an integer from 0 to {EXPERTS_MATVEC_MAX_TOKENS}"):
            R._options(fp8=True, experts=True, experts_matvec=bad)
    for kw in (dict(), dict(fp8=True), dict(experts=True)):
        with pytest.raises(ValueError, match="pass fp8=True and experts=True"):
            R._options(experts_matvec=1, **kw)
    # the existing checks come first, in their order
    with pytest.raises(ValueError, match="fp8=True and prefetch=True"):
        R._options(prefetch=True, fp8=True, experts_matvec=1)
    with pytest.raises(ValueError, match="fp8_matmul applies"):
        R._options(fp8_matmul=1, experts_matvec=1)
    with pytest.raises(ValueError, match="matvec must be an integer"):
        R._options(matvec=99, experts_matvec=99)


# ------------------------------------------------------------------ the layouts
@pytest.mark.parametrize("which", ("mixtral", "qwen3"))
@pytest.mark.parametrize("block", [(128, 128), None, (64, 32)])
def test_layout_of_transformers_fp8experts(which, block):
    """Even and ragged grids (gate_up_proj has 704 rows, 5.5 blocks of 128) and one scale per expert."""
    m = tiny_moe(which, block)
    ex = experts_of(m)
    assert len(ex) == 2 and all(R.experts_matvec_layout(x) == ("gate_up_proj", "down_proj") for x in ex)
    assert not any(R.experts_matvec_layout(x) for x in m.modules() if type(x).__name__ != "FP8Experts")


def test_layout_without_gate():
    pytest.importorskip("transformers")
    from transformers.integrations.finegrained_fp8 import FP8Experts
    m = tiny_moe("qwen3")
    with torch.device("meta"):
        x = FP8Experts(m.config, block_size=(128, 128), has_gate=False)
    assert R.experts_matvec_layout(x) == ("up_proj", "down_proj")


def test_layouts_that_are_refused():
    x = _experts()                        # fp8 experts, but not FP8Experts' projections
    assert R.fp8_experts(x) and R.experts_matvec_layout(x) is None
    x._apply_gate = lambda h: h
    assert R.experts_matvec_layout(x) is None
    m = tiny_moe("qwen3")
    ex = experts_of(m)[0]
    ex.__dict__["_apply_gate"] = None     # no gate to apply
    assert R.experts_matvec_layout(ex) is None
    ex = experts_of(m)[1]
    with torch.device("meta"):            # down_proj that does not take gate_up_proj's output
        ex.down_proj = torch.nn.Parameter(torch.empty(16, 256, 320, dtype=torch.float8_e4m3fn), requires_grad=False)
        ex.down_proj_scale_inv = torch.nn.Parameter(torch.empty(16, 2, 3))
    assert R.fp8_experts(ex) and R.experts_matvec_layout(ex) is None


# ------------------------------------------------------------------ the report
def test_report_keys_only_with_experts_matvec():
    state = R._Resident()
    state.entries = [R._Entry(None, None, [], "fp8_experts_matvec"), R._Entry(None, None, [], "fp8_experts")]
    state.experts_matvec_scratch_bytes = 1234
    without = R._with_prefetch({}, state, R._options(fp8=True, experts=True))
    assert "experts_matvec_modules" not in without and "experts_matvec_scratch_bytes" not in without
    assert without["fp8_experts_modules"] == 2
    got = R._with_prefetch({}, state, R._options(fp8=True, experts=True, experts_matvec=2))
    assert got["experts_matvec_modules"] == 1 and got["experts_matvec_scratch_bytes"] == 1234 and got["fp8_experts_modules"] == 2
