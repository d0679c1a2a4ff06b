"""The fp8 dequantize without a GPU: a numpy model of its numerics (one fp32 product, one rounding to bf16 / fp16)
against torch's `(W.to(float32) * S).to(dtype)` on every fp8 code, and the module rules of `fp8=True` --
`fp8_linears`, the parameters that stay dense, `plan_load` -- on transformers' own FP8Linear built on the meta device.

The model is what tests/test_dequant_fp8_gpu.py holds the kernel to, bit for bit.
"""
import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from zipnn_b200 import compress_module, load_module
from zipnn_b200 import resident as R

FORMATS = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
ODTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


# ------------------------------------------------------------------ the numpy model
def fp8_values(b, fmt: str) -> np.ndarray:
    """fp8 bytes -> their values as float64, decoded from the bit fields (e4m3fn: no infinities, S.1111.111 NaN;
    e5m2: IEEE-style)."""
    b = np.asarray(b, dtype=np.uint8).astype(np.int64)
    sign = np.where(b >> 7, -1.0, 1.0)
    if fmt == "e4m3":
        e, m = (b >> 3) & 15, b & 7
        v = np.where(e == 0, m * 2.0 ** -9, (1 + m / 8) * 2.0 ** (e - 7))
        v = np.where((e == 15) & (m == 7), np.nan, v)
    else:
        e, m = (b >> 2) & 31, b & 3
        v = np.where(e == 0, m * 2.0 ** -16, (1 + m / 4) * 2.0 ** (e - 15))
        v = np.where(e == 31, np.where(m == 0, np.inf, np.nan), v)
    return sign * v


def round_bits(f: np.ndarray, odt: str) -> np.ndarray:
    """fp32 values -> the bits of their round-to-nearest-even bf16 / fp16 values (uint16); NaN -> a quiet NaN."""
    f = np.ascontiguousarray(f, dtype=np.float32)
    if odt == "fp16":
        return f.astype(np.float16).view(np.uint16)
    u = f.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(f), (u >> 16).astype(np.uint16) | 0x7FC0, r).astype(np.uint16)


def model(b, fmt: str, s, odt: str) -> np.ndarray:
    """The dequantize of fp8 bytes b by fp32 scales s (same shape, the grid expanded): bits of odt(fl32(W * S))."""
    with np.errstate(over="ignore", invalid="ignore"):   # (inf * 0 and overflow are value classes under test)
        p = (fp8_values(b, fmt).astype(np.float32) * np.asarray(s, dtype=np.float32)).astype(np.float32)
        return round_bits(p, odt)


def same_bits(got: np.ndarray, want: np.ndarray, odt: str) -> np.ndarray:
    """Equal bits, or NaN in both (payloads may differ)."""
    dt = np.float16 if odt == "fp16" else None
    if dt is None:
        nan_g = ((got & 0x7F80) == 0x7F80) & ((got & 0x7F) != 0)
        nan_w = ((want & 0x7F80) == 0x7F80) & ((want & 0x7F) != 0)
    else:
        nan_g, nan_w = np.isnan(got.view(dt)), np.isnan(want.view(dt))
    return (got == want) | (nan_g & nan_w)


# scales for every value class: normal, full significands, products that overflow fp16 (and fp32), that are bf16 / fp16
# subnormals, fp32 subnormals, -0 and negative scales
SCALES = np.array([1.0, 0.25, 3.0, 1.0 + 2.0 ** -23, 2.0 ** -14 * 1.37, 2.0 ** 8, 2.0 ** 12, 2.0 ** -20, 2.0 ** -24, 2.0 ** -130,
                   2.0 ** -140, 2.0 ** -149, 3.0e38, -1.5, 0.0, -0.0], dtype=np.float32)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("odt", ODTYPES)
def test_model_matches_torch_on_every_code(fmt, odt):
    codes = np.arange(256, dtype=np.uint8)
    rng = np.random.default_rng(1)
    scales = np.concatenate([SCALES, (rng.uniform(0.5, 2.0, 48) * 2.0 ** rng.integers(-40, 20, 48)).astype(np.float32)])
    b = np.repeat(codes[None, :], scales.size, 0)
    s = np.repeat(scales[:, None], 256, 1)
    w = torch.from_numpy(b).view(FORMATS[fmt])
    assert np.array_equal(np.isnan(fp8_values(codes, fmt)), torch.isnan(w[0].float()).numpy())
    assert np.array_equal(np.nan_to_num(fp8_values(codes, fmt), posinf=1e300, neginf=-1e300),
                          np.nan_to_num(w[0].double().numpy(), posinf=1e300, neginf=-1e300))
    ref = (w.to(torch.float32) * torch.from_numpy(s)).to(ODTYPES[odt]).view(torch.int16).numpy().view(np.uint16)
    got = model(b, fmt, s, odt)
    ok = same_bits(got, ref, odt)
    assert ok.all(), [(float(scales[i]), int(codes[j])) for i, j in zip(*np.nonzero(~ok))][:8]
    # the classes were met: overflow to inf, subnormal results, -0, NaN
    vals = torch.from_numpy(got.view(np.int16)).view(ODTYPES[odt]).float()
    assert torch.isinf(vals).any() and torch.isnan(vals).any()
    tiny = torch.finfo(ODTYPES[odt]).tiny
    assert ((vals != 0) & (vals.abs() < tiny)).any()
    assert ((vals == 0) & torch.signbit(vals)).any()
    if odt == "fp16":
        assert torch.isinf(vals[(scales == 2.0 ** 12).nonzero()[0]]).any(), "fp16 overflow"


# ------------------------------------------------------------------ the module rules
def tiny_llama(block, scheme, device="meta"):
    """transformers' tiny Llama (2 layers, hidden 256) on `device` with every linear an FP8Linear."""
    transformers = pytest.importorskip("transformers")
    from transformers.integrations.finegrained_fp8 import replace_with_fp8_linear
    cfg = transformers.LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, head_dim=64, vocab_size=512)
    with torch.device(device):
        m = transformers.LlamaForCausalLM(cfg)
    q = transformers.FineGrainedFP8Config(weight_block_size=block, activation_scheme=scheme)
    return replace_with_fp8_linear(m, quantization_config=q, pre_quantized=True)


def fp8_modules(m):
    return [mod for mod in m.modules() if type(mod).__name__ == "FP8Linear"]


@pytest.mark.parametrize("block,scheme", [((128, 128), "dynamic"), ((128, 128), "static"), (None, "dynamic"), (None, "static")])
def test_fp8_linears_and_the_dense_parameters_on_transformers_fp8linear(block, scheme):
    m = tiny_llama(block, scheme)
    lins = fp8_modules(m)
    assert len(lins) == 15 and all(R.fp8_linears(x) for x in lins)
    assert not any(R.fp8_linears(x) for x in m.modules() if type(x).__name__ != "FP8Linear")
    modules, groups = R.select(m)
    kept = R.dense_biases(groups, 0, fp8=True)
    names = {(id(o), n) for _, owners in kept for o, n in owners}
    for x in lins:
        assert (id(x), "weight") in names
        assert (id(x), "weight_scale_inv") not in names and (id(x), "activation_scale") not in names
    assert len(kept) == len(groups) - sum(len(list(x.parameters())) - 1 for x in lins)
    assert R.dense_biases(groups, 0) is groups and len(R.dense_biases(groups, 0, fp8=False)) == len(groups)


def test_fp8_linears_refuses_what_is_not_an_fp8_linear():
    from transformers.integrations.finegrained_fp8 import FP8Linear
    with torch.device("meta"):
        plain = torch.nn.Linear(256, 128)
        bf16 = FP8Linear(256, 128, block_size=(128, 128), dtype=torch.bfloat16)
        ok = FP8Linear(256, 128, block_size=(128, 128), has_bias=True)
        e5 = FP8Linear(256, 128, block_size=(1, 256), dtype=torch.float8_e5m2)
        no_scale = torch.nn.Linear(256, 128)
        no_scale.weight = torch.nn.Parameter(torch.empty(128, 256, dtype=torch.float8_e4m3fn), requires_grad=False)
        no_scale.block_size = None
        wrong = FP8Linear(256, 128, block_size=(128, 128))
        wrong.weight_scale_inv = torch.nn.Parameter(torch.empty(2, 1))
        wrong_none = FP8Linear(256, 128, block_size=(128, 128))
        wrong_none.block_size = None
        fp64 = FP8Linear(256, 128, block_size=(128, 128))
        fp64.weight_scale_inv = torch.nn.Parameter(torch.empty(1, 2, dtype=torch.float64))
        no_block = FP8Linear(256, 128)
        del no_block.block_size
        flat = torch.nn.Module()
        flat.weight = torch.nn.Parameter(torch.empty(128, 256, dtype=torch.float8_e4m3fn), requires_grad=False)
        flat.weight_scale_inv = torch.nn.Parameter(torch.empty(()))
        flat.block_size = None
    assert R.fp8_linears(ok) and R.fp8_linears(e5) and R.fp8_linears(FP8Linear(256, 128).to("meta"))
    for x in (plain, bf16, no_scale, wrong, wrong_none, fp64, no_block, flat):
        assert not R.fp8_linears(x)
    # the bias and scales of an FP8Linear stay dense; those of a plain Linear only under matvec=N
    root = torch.nn.ModuleDict({"a": ok, "b": plain})
    _, groups = R.select(root)
    kept = {(id(o), n) for _, owners in R.dense_biases(groups, 0, fp8=True) for o, n in owners}
    assert kept == {(id(ok), "weight"), (id(plain), "weight"), (id(plain), "bias")}
    kept = {(id(o), n) for _, owners in R.dense_biases(groups, 4, fp8=True) for o, n in owners}
    assert kept == {(id(ok), "weight"), (id(plain), "weight")}


def _checkpoint(tmp_path, block, scheme):
    """A .safetensors file of the tiny fp8 Llama's full state, random values."""
    m = tiny_llama(block, scheme)
    g = torch.Generator().manual_seed(0)
    sd = {}
    for name, t in m.state_dict().items():
        v = torch.randn(t.shape, generator=g) * 0.05
        sd[name] = (v * 8).to(t.dtype) if t.dtype in R._FP8 else v.to(t.dtype)
    path = str(tmp_path / "fp8.safetensors")
    save_file({k: v.contiguous() for k, v in sd.items()}, path)
    return path


@pytest.mark.parametrize("block,scheme", [((128, 128), "static"), (None, "dynamic")])
def test_plan_load_reads_scales_and_biases_dense(tmp_path, block, scheme):
    path = _checkpoint(tmp_path, block, scheme)
    plan = R.plan_load(tiny_llama(block, scheme, "cpu"), path, fp8=True)   # (the rotary buffers are not in files)
    for name, kind in plan.kinds.items():
        if name.endswith((".weight_scale_inv", ".activation_scale")):
            assert kind == "dense", name
        elif name.endswith("_proj.weight") or name == "lm_head.weight":
            assert kind == "compress", name
    assert any(n.endswith(".weight_scale_inv") for n in plan.kinds)
    assert (scheme == "static") == any(n.endswith(".activation_scale") for n in plan.kinds)
    off = R.plan_load(tiny_llama(block, scheme, "cpu"), path)
    assert all(off.kinds[n] == "compress" for n in off.kinds if n.endswith(".weight_scale_inv"))


def test_fp8_and_prefetch_do_not_combine(tmp_path):
    m = tiny_llama((128, 128), "dynamic")
    with pytest.raises(ValueError, match="fp8=True and prefetch=True"):
        compress_module(m, fp8=True, prefetch=True)
    with pytest.raises(ValueError, match="fp8=True and prefetch=True"):
        load_module(m, str(tmp_path / "none.safetensors"), fp8=True, prefetch=True)
    assert getattr(m, R._ATTR, None) is None
