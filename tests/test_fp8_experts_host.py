"""The fp8 experts mode without a GPU: `fp8_experts` on transformers' own `FP8Experts` built on the meta device, the
parameters that stay dense under fp8=True and experts=True, `plan_load`, a numpy model of the selected dequantize's
per-slice scale index against torch's expanded grid, and the 3-D `dequantize_fp8` against a per-expert loop.

The index model is what k_select_dequant_fp8 computes per 16-byte vector (DequantEp with the per-slice grid): the slice
s = row / slice_rows by the multiply-high of matvec_fp8_div, then s * slice_grid + ((row - s * slice_rows) / bn) *
scols + col / bk.
"""
import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from zipnn_b200 import resident as R

COMMON = dict(hidden_size=256, intermediate_size=352, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
              num_hidden_layers=2, vocab_size=512)


def tiny_moe(which: str, block=(128, 128), scheme="dynamic", device="meta"):
    """transformers' tiny Mixtral or Qwen3-MoE on `device` with every linear an FP8Linear and every experts module an
    FP8Experts (`replace_with_fp8_linear`, as a pre-quantized checkpoint loads)."""
    tf = pytest.importorskip("transformers")
    from transformers.integrations.finegrained_fp8 import replace_with_fp8_linear
    if which == "mixtral":
        cls, cfg = tf.MixtralForCausalLM, tf.MixtralConfig(num_local_experts=8, num_experts_per_tok=2, **COMMON)
    else:
        cls, cfg = tf.Qwen3MoeForCausalLM, tf.Qwen3MoeConfig(num_experts=16, num_experts_per_tok=4, moe_intermediate_size=352,
                                                             decoder_sparse_step=1, mlp_only_layers=[], **COMMON)
    with torch.device(device):
        m = cls(cfg)
    q = tf.FineGrainedFP8Config(weight_block_size=block, activation_scheme=scheme)
    return replace_with_fp8_linear(m, quantization_config=q, pre_quantized=True)


def experts_of(m):
    return [x for x in m.modules() if type(x).__name__ == "FP8Experts"]


@pytest.mark.parametrize("which", ("mixtral", "qwen3"))
@pytest.mark.parametrize("block,scheme", [((128, 128), "dynamic"), ((128, 128), "static"), (None, "dynamic"), ((64, 32), "dynamic")])
def test_fp8_experts_accepts_transformers_fp8experts(which, block, scheme):
    """Divisible and ragged grids: gate_up_proj has 704 rows, 5.5 blocks of 128, and down_proj 352 columns."""
    m = tiny_moe(which, block, scheme)
    ex = experts_of(m)
    assert len(ex) == 2 and all(R.fp8_experts(x) for x in ex)
    assert not any(R.fp8_experts(x) for x in m.modules() if type(x).__name__ != "FP8Experts")
    assert all(not R.fp8_linears(x) for x in ex)


def test_fp8_experts_without_gate():
    pytest.importorskip("transformers")
    from transformers.integrations.finegrained_fp8 import FP8Experts
    m = tiny_moe("qwen3")
    with torch.device("meta"):
        x = FP8Experts(m.config, block_size=(128, 128), has_gate=False)
    assert "up_proj" in x._parameters and "gate_up_proj" not in x._parameters
    assert R.fp8_experts(x)


def _experts(block=(128, 128), E=4, out=192, inn=256):
    """A module of the FP8Experts attributes on meta: w [E, out, inn] and its scale grid."""
    x = torch.nn.Module()
    x.num_experts = E
    x.block_size = block
    gr, gc = (1, 1) if block is None else (-(-out // block[0]), -(-inn // block[1]))
    with torch.device("meta"):
        x.w = torch.nn.Parameter(torch.empty(E, out, inn, dtype=torch.float8_e4m3fn), requires_grad=False)
        x.w_scale_inv = torch.nn.Parameter(torch.empty(E, gr, gc))
    return x


def test_fp8_experts_refuses_what_is_not_one():
    assert R.fp8_experts(_experts()) and R.fp8_experts(_experts(None)) and R.fp8_experts(_experts((1, 16)))
    missing = _experts()
    del missing.w_scale_inv
    wrong_grid = _experts()
    wrong_grid.w_scale_inv = torch.nn.Parameter(torch.empty(4, 2, 3, device="meta"))
    flat_grid = _experts()
    flat_grid.w_scale_inv = torch.nn.Parameter(torch.empty(4 * 2 * 2, device="meta"))
    none_grid = _experts(None)
    none_grid.w_scale_inv = torch.nn.Parameter(torch.empty(4, device="meta"))
    fp64 = _experts()
    fp64.w_scale_inv = torch.nn.Parameter(torch.empty(4, 2, 2, dtype=torch.float64, device="meta"))
    bias = _experts()
    bias.w_bias = torch.nn.Parameter(torch.empty(4, 192, device="meta"))
    flat = _experts()
    flat.w = torch.nn.Parameter(torch.empty(192, 256, dtype=torch.float8_e4m3fn, device="meta"), requires_grad=False)
    flat.w_scale_inv = torch.nn.Parameter(torch.empty(2, 2, device="meta"))
    wrong_e = _experts()
    wrong_e.num_experts = 5
    no_block = _experts()
    del no_block.block_size
    bad_block = _experts()
    bad_block.block_size = (128, 0)
    bf16 = _experts()
    bf16.w = torch.nn.Parameter(torch.empty(4, 192, 256, dtype=torch.bfloat16, device="meta"))
    for x in (missing, wrong_grid, flat_grid, none_grid, fp64, bias, flat, wrong_e, no_block, bad_block, bf16):
        assert not R.fp8_experts(x)


def _kept(groups, **kw):
    return {(id(o), n) for _, owners in R.dense_biases(groups, 0, **kw) for o, n in owners}


@pytest.mark.parametrize("scheme", ("dynamic", "static"))
def test_dense_parameters_only_under_both_flags(scheme):
    m = tiny_moe("qwen3", scheme=scheme)
    ex = experts_of(m)
    _, groups = R.select(m)
    every = _kept(groups)
    both = _kept(groups, fp8=True, experts=True)
    fp8_only = _kept(groups, fp8=True)
    experts_only = _kept(groups, experts=True)
    assert experts_only == every   # (experts alone: dense_biases is not asked for anything)
    for x in ex:
        fp8 = {n for n, p in x._parameters.items() if p is not None and p.dtype in R._FP8}
        other = {n for n, p in x._parameters.items() if p is not None and p.dtype not in R._FP8}
        assert fp8 == {"gate_up_proj", "down_proj"} and "gate_up_proj_scale_inv" in other
        assert (scheme == "static") == ("down_proj_activation_scale" in other)
        assert all((id(x), n) in both for n in fp8) and not any((id(x), n) in both for n in other)
        assert all((id(x), n) in fp8_only for n in fp8 | other)   # fp8=True alone leaves the experts' groups as before
    # outside the experts, both flags keep what fp8=True keeps
    outside = {k for k in every if not any(k[0] == id(x) for x in ex)}
    assert both & outside == fp8_only & outside


def _checkpoint(tmp_path, which, block, scheme):
    m = tiny_moe(which, block, scheme)
    g = torch.Generator().manual_seed(0)
    sd = {}
    for name, t in m.state_dict().items():
        v = torch.randn(t.shape, generator=g) * 0.05
        sd[name] = (v * 8).to(t.dtype) if t.dtype in R._FP8 else v.to(t.dtype)
    path = str(tmp_path / "fp8_moe.safetensors")
    save_file({k: v.contiguous() for k, v in sd.items()}, path)
    return path


@pytest.mark.parametrize("block,scheme", [((128, 128), "static"), (None, "dynamic")])
def test_plan_load_reads_the_experts_scales_dense_under_both_flags(tmp_path, block, scheme):
    path = _checkpoint(tmp_path, "mixtral", block, scheme)
    experts_scale = (".experts.gate_up_proj_scale_inv", ".experts.down_proj_scale_inv", "_activation_scale")
    plan = R.plan_load(tiny_moe("mixtral", block, scheme, "cpu"), path, fp8=True, experts=True)
    for name, kind in plan.kinds.items():
        if name.endswith(experts_scale) or name.endswith(".weight_scale_inv"):
            assert kind == "dense", name
        elif name.endswith((".experts.gate_up_proj", ".experts.down_proj")):
            assert kind == "compress", name
    assert (scheme == "static") == any(n.endswith("_activation_scale") for n in plan.kinds)
    for kw in (dict(fp8=True), dict(experts=True), {}):   # either flag alone: the experts' scales compress as before
        off = R.plan_load(tiny_moe("mixtral", block, scheme, "cpu"), path, **kw)
        assert all(off.kinds[n] == "compress" for n in off.kinds if n.endswith(experts_scale[:2])), kw
        linear_scale = "dense" if kw.get("fp8") else "compress"   # (the FP8Linears' rule is fp8=True's alone)
        assert all(off.kinds[n] == linear_scale for n in off.kinds if n.endswith(".weight_scale_inv")), kw


# ------------------------------------------------------------------ the per-slice scale index
def _recip(d: int) -> int:
    return (2 ** 64 - 1) // (2 * d) + 1


def _div(n: np.ndarray, r: int) -> np.ndarray:
    """matvec_fp8_div: floor(2n * r / 2^64), in exact integers."""
    return np.array([(2 * int(v) * r) >> 64 for v in n.reshape(-1)], dtype=np.int64).reshape(n.shape)


def slice_index(E: int, out: int, inn: int, bn: int, bk: int) -> np.ndarray:
    """The scale index of every element of [E * out, inn], as the kernel forms it (bn, bk clamped as fp8_grid does)."""
    bn, bk = min(bn, out), min(bk, inn)
    scols, gr = -(-inn // bk), -(-out // bn)
    row = np.arange(E * out, dtype=np.int64)
    s = _div(row, _recip(out))
    r = row - s * out
    rowpart = s * (gr * scols) + _div(r, _recip(bn)) * scols
    colpart = _div(np.arange(inn, dtype=np.int64), _recip(bk))
    return rowpart[:, None] + colpart[None, :]


@pytest.mark.parametrize("E,out,inn,bn,bk", [(8, 704, 256, 128, 128), (16, 256, 352, 128, 128), (4, 96, 48, 32, 16),
                                              (3, 100, 64, 7, 16), (5, 1, 16, 1, 16), (4, 96, 48, 96, 48), (2, 50, 32, 500, 400)])
def test_slice_index_model_equals_torchs_expanded_grid(E, out, inn, bn, bk):
    gr, gc = -(-out // min(bn, out)), -(-inn // min(bk, inn))
    grid = torch.arange(E * gr * gc, dtype=torch.float64).reshape(E, gr, gc)
    want = grid.repeat_interleave(min(bn, out), 1)[:, :out].repeat_interleave(min(bk, inn), 2)[:, :, :inn]
    got = grid.reshape(-1)[torch.from_numpy(slice_index(E, out, inn, bn, bk))].reshape(E, out, inn)
    assert torch.equal(got, want)


def test_slice_index_at_the_largest_rows():
    """Rows near 2^31 (an fp8 item has at most INT32_MAX elements): the multiply-high still gives the exact quotient."""
    for out in (704, 1536, 4096, 28672, 3):
        rows = np.array([2 ** 31 - 1, 2 ** 31 - 2, 2 ** 30 + 12345, out * 1000 - 1, out * 1000], dtype=np.int64)
        assert np.array_equal(_div(rows, _recip(out)), rows // out), out


# ------------------------------------------------------------------ the 3-D torch dequantize
@pytest.mark.parametrize("block", [(128, 128), (64, 32), None, (1, 352)])
@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float16))
def test_dequantize_fp8_3d_equals_a_per_expert_loop(block, dtype):
    g = torch.Generator().manual_seed(1)
    E, out, inn = 5, 704, 352
    w = (torch.randn(E, out, inn, generator=g) * 40).to(torch.float8_e4m3fn)
    gr, gc = (1, 1) if block is None else (-(-out // block[0]), -(-inn // block[1]))
    s = torch.rand(E, gr, gc, generator=g) * 2.0 ** -6
    got = R.dequantize_fp8(w, s, block, dtype)
    assert got.shape == (E, out, inn) and got.dtype == dtype
    for e in range(E):
        want = R.dequantize_fp8(w[e], s[e].reshape(-1) if block is None else s[e], block, dtype)
        assert torch.equal(got[e].view(torch.int16), want.view(torch.int16)), e
