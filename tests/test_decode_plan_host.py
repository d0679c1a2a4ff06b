"""Decode plans and compressed-resident modules without a GPU: the ctypes view of the plan ABI against the header,
and the module selection rules of compress_module on CPU modules."""
import ctypes as C
import os
import re

import pytest
import torch

from zipnn_b200 import _native
from zipnn_b200.resident import select

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "zipnn_b200.h")) as f:
        return f.read()


def test_plan_struct_matches_header():
    m = re.search(r"typedef struct zipnn_b200_decode_plan \{\s*uint64_t opaque\[(\d+)\];\s*\} zipnn_b200_decode_plan;", _header())
    assert m, "zipnn_b200_decode_plan not found in the header"
    assert C.sizeof(_native.DecodePlanStruct) == 8 * int(m.group(1)) == 128
    assert C.alignment(_native.DecodePlanStruct) == 8


def test_plan_entry_points_are_declared_and_bound():
    h = _header()
    for name in ("zipnn_b200_decode_plan_size", "zipnn_b200_decode_plan_create", "zipnn_b200_decode_plan_run",
                 "zipnn_b200_decode_plan_status"):
        assert re.search(r"\bint " + name + r"\(", h), name
        assert name in _native.EXPORTS
    args = re.search(r"int zipnn_b200_decode_plan_create\(([^)]*)\)", h).group(1)
    assert len(args.split(",")) == 8
    args = re.search(r"int zipnn_b200_decode_plan_size\(([^)]*)\)", h).group(1)
    assert len(args.split(",")) == 5


class Block(torch.nn.Module):
    def __init__(self, h=8):
        super().__init__()
        self.norm = torch.nn.LayerNorm(h)
        self.q = torch.nn.Linear(h, h, bias=False)
        self.mlp = torch.nn.Sequential(torch.nn.Linear(h, 2 * h), torch.nn.Linear(2 * h, h))


class Model(torch.nn.Module):
    def __init__(self, h=8, vocab=16):
        super().__init__()
        self.embed = torch.nn.Embedding(vocab, h)
        self.blocks = torch.nn.ModuleList([Block(h), Block(h)])
        self.head = torch.nn.Linear(h, vocab, bias=False)
        self.head.weight = self.embed.weight       # tied
        self.counts = torch.nn.Parameter(torch.zeros(4, dtype=torch.int32), requires_grad=False)  # not a float type


def test_default_selection_takes_every_direct_owner():
    m = Model()
    mods, groups = select(m)
    want = [m.embed] + [x for b in m.blocks for x in (b.norm, b.q, b.mlp[0], b.mlp[1])] + [m.head]
    assert [id(x) for x in mods] == [id(x) for x in want]
    assert m not in mods          # owns only an int parameter
    assert len(groups) == 1 + 2 * (2 + 1 + 2 + 2)    # embedding/head once; norm w+b, q, two linears w+b per block


def test_tied_parameter_is_one_group_with_every_owner():
    m = Model()
    _, groups = select(m)
    tied = [g for g in groups if g[0] is m.embed.weight]
    assert len(tied) == 1
    assert sorted(n for _, n in tied[0][1]) == ["weight", "weight"]
    assert {id(o) for o, _ in tied[0][1]} == {id(m.embed), id(m.head)}


def test_tied_parameter_with_an_unselected_owner_stays_dense():
    m = Model()
    _, groups = select(m, [m.head, m.blocks[0].q])
    assert [g[0] for g in groups] == [m.blocks[0].q.weight]


def test_nested_selection_raises():
    m = Model()
    with pytest.raises(ValueError, match="contains"):
        select(m, [m.blocks[0], m.blocks[0].q])
    with pytest.raises(ValueError, match="contains"):
        select(m, [m.blocks[1].mlp[1], m.blocks[1]])


def test_explicit_selection_of_a_container():
    m = Model()
    mods, groups = select(m, [m.blocks[0].mlp])
    assert mods == [m.blocks[0].mlp] and groups == []   # a container owns no parameters directly


def test_default_selection_takes_innermost_owners():
    """MultiheadAttention owns in_proj_weight and contains its out_proj: the default takes out_proj, the container's
    own parameters stay dense, and nothing nests."""
    m = torch.nn.Sequential(torch.nn.MultiheadAttention(16, 2), torch.nn.Linear(16, 16))
    mods, groups = select(m)
    assert [id(x) for x in mods] == [id(m[0].out_proj), id(m[1])]
    assert all(p is not m[0].in_proj_weight for p, _ in groups)
