"""What load_module decides from a module and the files' headers alone (zipnn_b200.resident.plan_load), and the state
names save_module writes -- no GPU.

Modules are built on the meta device; the files are plain safetensors written on the CPU and the reference-made
tests/golden/ref_model.znn.safetensors.  Each state name becomes a "stream" (a compressed entry that stays
compressed), a "compress" candidate (a plain float entry of a selected parameter), "dense", or an "alias" (another
name of the same tied parameter is read instead).
"""
import os

import pytest
import torch
from safetensors.torch import save_file

from test_resident_gpu import Model
from zipnn_b200 import load_module
from zipnn_b200.resident import _ATTR, _Resident, first_names, plan_load, state_names

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_model.znn.safetensors")


def meta_model():
    with torch.device("meta"):
        return Model().to(torch.bfloat16)


def dense_state(dtype=torch.bfloat16):
    torch.manual_seed(0)
    m = Model().to(dtype)
    sd = m.state_dict()
    del sd["lm_head.weight"]
    return {k: v.contiguous() for k, v in sd.items()}


def write(tmp_path, tensors, name="model.safetensors"):
    path = str(tmp_path / name)
    save_file(tensors, path)
    return path


class RefModel(torch.nn.Module):
    """The parameters and buffer of the reference-made .znn file."""

    def __init__(self, fp16=torch.float16):
        super().__init__()
        P = lambda s, dt: torch.nn.Parameter(torch.empty(s, dtype=dt, device="meta"), requires_grad=False)  # noqa: E731
        self.w_bf16, self.w_fp16 = P((100, 100), torch.bfloat16), P((100, 100), fp16)
        self.w_fp32, self.w_fp8 = P((100, 100), torch.float32), P((100, 100), torch.float8_e4m3fn)
        self.big_bf16 = P((300, 257), torch.bfloat16)
        self.register_buffer("ids", torch.empty(10, 100, dtype=torch.int64, device="meta"))


def test_state_names_follow_state_dict_and_keep_the_first_tied_name():
    m = Model()
    names = state_names(m)
    assert [n for n, *_ in names] == list(m.state_dict())
    first, later = first_names(names)
    assert [n for n, *_ in later] == ["lm_head.weight"]
    assert "embed_tokens.weight" in [n for n, *_ in first]
    m.register_buffer("scratch", torch.zeros(3), persistent=False)
    m.layers[0].register_buffer("step", torch.zeros(1, dtype=torch.int64))
    assert [n for n, *_ in state_names(m)] == list(m.state_dict())


def test_default_selection_plain_file(tmp_path):
    path = write(tmp_path, dense_state())
    m = meta_model()
    plan = plan_load(m, path)
    assert plan.kinds.pop("lm_head.weight") == "alias"
    assert set(plan.kinds.values()) == {"compress"} and len(plan.kinds) == len(dense_state())
    assert not plan.streams and not plan.dense and len(plan.compress) == len(plan.groups)
    assert all(p.is_meta for p in m.parameters())


@pytest.mark.parametrize("present", [["embed_tokens.weight"], ["lm_head.weight"], ["embed_tokens.weight", "lm_head.weight"]])
def test_tied_weight_under_either_name_or_both(tmp_path, present):
    sd = dense_state()
    emb = sd.pop("embed_tokens.weight")
    for n in present:
        sd[n] = emb.clone()
    plan = plan_load(meta_model(), write(tmp_path, sd))
    read = present[0]
    other = "lm_head.weight" if read == "embed_tokens.weight" else "embed_tokens.weight"
    assert plan.kinds[read] == "compress" and plan.kinds[other] == "alias"
    assert len(plan.compress) == len(plan.groups)           # the tied parameter is one group, read once


def test_explicit_selection_and_a_weight_tied_to_an_unselected_owner(tmp_path):
    path = write(tmp_path, dense_state())
    m = meta_model()
    up = m.layers[0].mlp.up_proj
    plan = plan_load(m, path, modules=[up, m.embed_tokens])
    assert plan.kinds["layers.0.mlp.up_proj.weight"] == "compress"
    assert plan.kinds["embed_tokens.weight"] == "dense"      # lm_head, outside the selection, owns it too
    assert plan.kinds["lm_head.weight"] == "alias"
    assert sum(k == "compress" for k in plan.kinds.values()) == 1
    (e, owners, kind, requires_grad), = [d for d in plan.dense if d[0].shape == (1000, 256)]
    assert {id(o) for o, _ in owners} == {id(m.embed_tokens), id(m.lm_head)} and kind == "param" and requires_grad
    with pytest.raises(ValueError, match="contains"):
        plan_load(m, path, modules=[m.layers[0], up])


def test_reference_znn_file():
    m = RefModel()
    plan = plan_load(m, GOLDEN)
    assert plan.kinds == {"w_bf16": "stream", "w_fp16": "stream", "w_fp32": "stream", "w_fp8": "stream", "big_bf16": "stream",
                          "ids": "dense"}
    assert [e.compressed for _, e in plan.streams] == [True] * 5
    plan = plan_load(RefModel(), GOLDEN, modules=[])
    assert set(plan.kinds.values()) == {"dense"}


def test_checkpoint_split_over_two_files(tmp_path):
    sd = dense_state()
    keys = sorted(sd)
    a = write(tmp_path, {k: sd[k] for k in keys[::2]}, "a.safetensors")
    b = write(tmp_path, {k: sd[k] for k in keys[1::2]}, "b.safetensors")
    one = plan_load(meta_model(), write(tmp_path, sd))
    two = plan_load(meta_model(), [a, b])
    assert two.kinds == one.kinds
    assert {e.file for _, e in two.compress} == {a, b}
    with pytest.raises(ValueError, match="more than one file"):
        plan_load(meta_model(), [a, b, a])


def _refused(tmp_path, m, files, match):
    before = {n: p for n, p in m.named_parameters()}
    with pytest.raises(ValueError, match=match) as info:
        plan_load(m, files)
    assert {n: p for n, p in m.named_parameters()} == before
    return str(info.value)


def test_refusals(tmp_path):
    sd = dense_state()
    m = meta_model()
    missing = dict(sd)
    del missing["layers.1.mlp.down_proj.weight"]
    assert "layers.1.mlp.down_proj.weight" in _refused(tmp_path, m, write(tmp_path, missing, "m.safetensors"), "lack")
    extra = dict(sd, surplus=torch.zeros(2))
    assert "surplus" in _refused(tmp_path, m, write(tmp_path, extra, "x.safetensors"), "module lacks")
    wrong = dict(sd, **{"norm.weight": sd["norm.weight"].half()})
    assert "norm.weight" in _refused(tmp_path, m, write(tmp_path, wrong, "d.safetensors"), "dtype or shape")
    wrong = dict(sd, **{"layers.0.self_attn.q_proj.weight": torch.zeros(256, 255, dtype=torch.bfloat16)})
    assert "q_proj" in _refused(tmp_path, m, write(tmp_path, wrong, "s.safetensors"), "dtype or shape")
    path = write(tmp_path, sd)
    with torch.device("meta"):
        m.register_buffer("rope", torch.zeros(8), persistent=False)
    assert "rope" in _refused(tmp_path, m, path, "meta device")
    m.rope = torch.zeros(8)
    plan = plan_load(m, path)
    assert plan.moves == [(m, "rope")]
    setattr(m, _ATTR, _Resident())
    _refused(tmp_path, m, path, "already compressed")
    delattr(m, _ATTR)
    with pytest.raises(ValueError, match="CUDA"):
        load_module(m, path, device="cpu")


def test_compressed_entry_checked_against_metadata_and_module():
    assert "w_fp16" in _refused(None, RefModel(fp16=torch.bfloat16), GOLDEN, "dtype or shape")
