"""Host side of selected plan runs (zipnn_b200_decode_plan_run_select, DecodePlan.run_select, experts=True).

  * `touched_chunks`, the reference for the chunks a set of ids touches, which test_select_gpu.py takes as the exact
    write set of a selected run, against a byte-by-byte brute force: slices inside a chunk, aligned with chunks,
    straddling them and spanning many, one slice (E = 1), ids at both ends, duplicates and bad ids;
  * the experts-module rule (`experts_module`) on modules built on the meta device: a local experts class in the
    transformers convention, transformers' own MixtralExperts and Qwen3MoeExperts, and modules that must not qualify;
  * experts=True together with prefetch=True is a ValueError, before any device work.
"""
import numpy as np
import pytest
import torch

from zipnn_b200 import compress_module, load_module
from zipnn_b200.resident import experts_module, select


def touched_chunks(orig: int, chunk: int, rows: int, ids) -> np.ndarray:
    """-> bool [K]: the chunks of a tensor of `orig` bytes in `chunk`-byte chunks that meet slice e (bytes
    [e * S, (e + 1) * S), S = orig / rows) of an id e in [0, rows); other ids touch nothing."""
    assert orig % rows == 0
    S = orig // rows
    K = -(-orig // chunk)
    mask = np.zeros(K, dtype=bool)
    for e in np.asarray(ids).reshape(-1).tolist():
        if 0 <= e < rows:
            mask[e * S // chunk: (e * S + S - 1) // chunk + 1] = True
    return mask


def written_bytes(orig: int, chunk: int, rows: int, ids) -> np.ndarray:
    """-> bool [orig]: the bytes a selected run writes (every byte of every touched chunk)."""
    return np.repeat(touched_chunks(orig, chunk, rows, ids), chunk)[:orig]


def _brute(orig, chunk, rows, ids):
    S = orig // rows
    K = -(-orig // chunk)
    mask = np.zeros(K, dtype=bool)
    for e in ids:
        if 0 <= e < rows:
            for b in range(e * S, (e + 1) * S):
                mask[b // chunk] = True
    return mask


CASES = [
    # (orig, chunk, rows): slices inside a chunk, several per chunk, aligned with chunks, straddling, spanning many
    (4096, 512, 64),       # 64-byte slices, 8 per chunk
    (4096, 512, 8),        # one chunk per slice
    (4096, 512, 2),        # 4 chunks per slice
    (6000, 512, 3),        # 2000-byte slices straddling chunks, a ragged last chunk
    (6000, 512, 1),        # E = 1: every chunk
    (3 * 704, 256, 3),     # 704-byte slices: 2.75 chunks, every slice straddles
    (8 * 1536, 1024, 8),   # 1.5 chunks per slice
    (1000, 4096, 10),      # one chunk holds the whole tensor
]


@pytest.mark.parametrize("orig,chunk,rows", CASES)
def test_touched_chunks_match_brute_force(orig, chunk, rows):
    rng = np.random.default_rng(orig + chunk + rows)
    sets = [[0], [rows - 1], [0, rows - 1], [rows - 1, rows - 1, 0, 0], list(range(rows)),
            rng.integers(0, rows, 5).tolist(), [-1, rows, rows + 7, 0], []]
    for ids in sets:
        got = touched_chunks(orig, chunk, rows, ids)
        assert np.array_equal(got, _brute(orig, chunk, rows, ids)), (orig, chunk, rows, ids)
        wb = written_bytes(orig, chunk, rows, ids)
        assert wb.size == orig
        S = orig // rows
        for e in ids:   # every selected slice is inside the write set
            if 0 <= e < rows:
                assert wb[e * S: (e + 1) * S].all()


def test_all_ids_touch_every_chunk_and_bad_ids_nothing():
    for orig, chunk, rows in CASES:
        assert touched_chunks(orig, chunk, rows, range(rows)).all()
        assert not touched_chunks(orig, chunk, rows, [-5, -1, rows, 2 * rows]).any()


def test_straddling_slices_share_their_boundary_chunk():
    # 704-byte slices in 256-byte chunks: slice 1 is bytes [704, 1408), chunks 2 .. 5; chunk 2 also holds slice 0
    m = touched_chunks(3 * 704, 256, 3, [1])
    assert np.flatnonzero(m).tolist() == [2, 3, 4, 5]
    assert touched_chunks(3 * 704, 256, 3, [0])[2]


# ------------------------------------------------------------------ the experts-module rule
class Experts(torch.nn.Module):
    """The transformers convention: 3D weights [E, ...], biases [E, ...], `num_experts` = E."""

    def __init__(self, E=4, H=16, inter=8, bias=True, device="meta"):
        super().__init__()
        self.num_experts = E
        self.gate_up_proj = torch.nn.Parameter(torch.empty(E, 2 * inter, H, dtype=torch.bfloat16, device=device))
        self.down_proj = torch.nn.Parameter(torch.empty(E, H, inter, dtype=torch.bfloat16, device=device))
        if bias:
            self.gate_up_proj_bias = torch.nn.Parameter(torch.empty(E, 2 * inter, dtype=torch.bfloat16, device=device))
            self.down_proj_bias = torch.nn.Parameter(torch.empty(E, H, dtype=torch.bfloat16, device=device))


def test_local_experts_qualify():
    for bias in (False, True):
        m = Experts(bias=bias)
        assert experts_module(m)
        assert experts_module(m, ["gate_up_proj", "down_proj"])
        modules, _ = select(torch.nn.Sequential(torch.nn.Linear(16, 4, device="meta"), m))
        assert m in modules   # select() picks it by default: it owns its parameters directly


def test_modules_that_do_not_qualify():
    m = Experts()
    m.num_experts = 5                        # a wrong num_experts
    assert not experts_module(m)
    m = Experts()
    m.router = None
    m.extra = torch.nn.Parameter(torch.empty(3, 16, device="meta"))   # a 2D parameter whose shape[0] differs
    assert not experts_module(m)
    assert experts_module(m, ["gate_up_proj", "down_proj"])           # ... unless it is not compressed
    m = Experts()
    m.num_experts = 4.0                      # not an integer
    assert not experts_module(m)
    m = Experts()
    m.num_experts = True
    assert not experts_module(m)
    m = Experts()
    del m.num_experts                        # no num_experts at all
    assert not experts_module(m)
    assert not experts_module(torch.nn.Linear(4, 4, device="meta"))
    e = torch.nn.Module()
    e.num_experts = 4                        # no parameters
    assert not experts_module(e)


def _tiny(cls_config, **kw):
    cfg = cls_config(hidden_size=32, intermediate_size=48, moe_intermediate_size=48, num_attention_heads=2,
                     num_key_value_heads=1, head_dim=16, num_hidden_layers=1, vocab_size=64, **kw)
    return cfg


def test_transformers_experts_qualify():
    transformers = pytest.importorskip("transformers")
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts
    from transformers.models.qwen3_moe.modeling_qwen3_moe import Qwen3MoeExperts
    with torch.device("meta"):
        mix = MixtralExperts(_tiny(transformers.MixtralConfig, num_local_experts=8, num_experts_per_tok=2))
        qwen = Qwen3MoeExperts(_tiny(transformers.Qwen3MoeConfig, num_experts=16, num_experts_per_tok=4))
    for m, E in ((mix, 8), (qwen, 16)):
        assert m.num_experts == E
        assert experts_module(m), type(m).__name__
        for _, p in m.named_parameters():
            assert p.shape[0] == E


def test_experts_with_prefetch_is_a_value_error(tmp_path):
    m = torch.nn.Sequential(Experts(device="cpu"))
    with pytest.raises(ValueError, match="prefetch"):
        compress_module(m, prefetch=True, experts=True)
    with pytest.raises(ValueError, match="prefetch"):
        load_module(m, str(tmp_path / "none.safetensors"), prefetch=True, experts=True)
    assert all(p.device.type == "cpu" for p in m.parameters())   # untouched
