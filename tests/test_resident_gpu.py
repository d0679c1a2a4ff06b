"""Modules whose weights stay compressed in HBM (zipnn_b200.compress_module / decompress_module).

A small llama-like model (embedding, RMSNorm, attention-shaped and MLP linears, an lm_head tied to the embedding)
in bf16, fp16 and fp32, and a module that upcasts an fp8 weight in its forward: compressed, it computes exactly the
dense model's logits, directly and through a captured CUDA graph; it refuses to run with grad mode on; memory drops
by what compress_module reports; decompress_module gives back every parameter bit for bit.
"""
import copy
import gc

import pytest
import torch
import torch.nn.functional as F

from zipnn_b200 import compress_module, decompress_module

pytestmark = pytest.mark.gpu

H, HEADS, FFN, VOCAB, LAYERS = 256, 4, 704, 1000, 2


class Attention(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.q_proj = torch.nn.Linear(H, H, bias=False)
        self.k_proj = torch.nn.Linear(H, H // 2, bias=False)
        self.v_proj = torch.nn.Linear(H, H // 2, bias=False)
        self.o_proj = torch.nn.Linear(H, H, bias=False)

    def forward(self, x):
        b, t, _ = x.shape
        q = self.q_proj(x).view(b, t, HEADS, -1).transpose(1, 2)
        k = self.k_proj(x).view(b, t, HEADS // 2, -1).transpose(1, 2).repeat_interleave(2, dim=1)
        v = self.v_proj(x).view(b, t, HEADS // 2, -1).transpose(1, 2).repeat_interleave(2, dim=1)
        y = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        return self.o_proj(y.transpose(1, 2).reshape(b, t, H))


class MLP(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.gate_proj = torch.nn.Linear(H, FFN, bias=False)
        self.up_proj = torch.nn.Linear(H, FFN, bias=False)
        self.down_proj = torch.nn.Linear(FFN, H, bias=False)

    def forward(self, x):
        return self.down_proj(F.silu(self.gate_proj(x)) * self.up_proj(x))


class Layer(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.input_layernorm = torch.nn.RMSNorm(H)
        self.self_attn = Attention()
        self.post_attention_layernorm = torch.nn.RMSNorm(H)
        self.mlp = MLP()

    def forward(self, x):
        x = x + self.self_attn(self.input_layernorm(x))
        return x + self.mlp(self.post_attention_layernorm(x))


class Model(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.embed_tokens = torch.nn.Embedding(VOCAB, H)
        self.layers = torch.nn.ModuleList([Layer() for _ in range(LAYERS)])
        self.norm = torch.nn.RMSNorm(H)
        self.lm_head = torch.nn.Linear(H, VOCAB, bias=False)
        self.lm_head.weight = self.embed_tokens.weight

    def forward(self, ids):
        x = self.embed_tokens(ids)
        for layer in self.layers:
            x = layer(x)
        return self.lm_head(self.norm(x))


def make_model(dtype, seed=0):
    torch.manual_seed(seed)
    m = Model()
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() > 1:
                p.normal_(0, 0.02)
            else:
                p.copy_(1 + 0.1 * torch.randn_like(p))
    return m.to(device="cuda", dtype=dtype).eval()


def _snapshot(m):
    return {n: p.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_llama_like_exact(dtype):
    dense = make_model(dtype)
    model = copy.deepcopy(dense)
    assert model.lm_head.weight is model.embed_tokens.weight
    before = _snapshot(model)
    ids = torch.randint(0, VOCAB, (2, 17), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    rep = compress_module(model)
    # every matrix is compressed (a norm vector may not be: a stream has a fixed overhead); the tied one is stored once
    dense_left = dict(model.named_parameters())
    assert all(p.dim() == 1 for p in dense_left.values())
    assert rep["params"] + len(dense_left) == len(before) and rep["modules"] >= 3 + LAYERS * 7
    assert rep["stream_bytes"] < rep["dense_bytes"] == sum(t.numel() * t.element_size() for n, t in before.items() if n not in dense_left)
    for m in model.modules():
        assert "weight" not in m.__dict__
        assert "weight" in m._parameters or not hasattr(m, "weight")
    with torch.inference_mode():
        got = model(ids)
    assert torch.equal(got, want)
    with torch.no_grad():
        assert torch.equal(model(ids), want)
    for m in model.modules():
        assert "weight" not in m.__dict__          # unbound again after each forward
    with pytest.raises(RuntimeError, match="no_grad"):
        model(ids)
    decompress_module(model)
    after = dict(model.named_parameters())
    assert list(after) == list(before)          # in their original order (named_parameters, state_dict)
    assert list(model.state_dict()) == list(dense.state_dict())
    for n, t in before.items():
        assert torch.equal(after[n].view(torch.uint8), t.view(torch.uint8)), n
        assert after[n].requires_grad
    assert model.lm_head.weight is model.embed_tokens.weight
    with torch.inference_mode():
        assert torch.equal(model(ids), want)


def test_cuda_graph_of_a_compressed_forward():
    dense = make_model(torch.bfloat16, seed=1)
    model = copy.deepcopy(dense)
    compress_module(model)
    ids = torch.randint(0, VOCAB, (1, 9), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(ids)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = model(ids)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, want)


class Fp8Linear(torch.nn.Module):
    def __init__(self, w):
        super().__init__()
        self.weight = torch.nn.Parameter(w, requires_grad=False)

    def forward(self, x):
        return x @ self.weight.to(torch.bfloat16).t()


def test_fp8_weight_upcast_in_forward():
    torch.manual_seed(3)
    w = (torch.randn(512, 384) * 0.5).to(torch.float8_e4m3fn).cuda()
    dense = Fp8Linear(w.clone())
    mod = Fp8Linear(w.clone())
    x = torch.randn(5, 384, device="cuda", dtype=torch.bfloat16)
    rep = compress_module(mod)
    assert rep["params"] == 1
    with torch.inference_mode():
        assert torch.equal(mod(x), dense(x))
    decompress_module(mod)
    assert torch.equal(mod.weight.view(torch.uint8), w.view(torch.uint8)) and not mod.weight.requires_grad


def test_memory_drops_by_the_reported_bytes():
    model = make_model(torch.bfloat16, seed=2)
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    rep = compress_module(model)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    expect = rep["dense_bytes"] - (rep["stream_bytes"] + rep["plan_bytes"] + rep["scratch_bytes"] + rep["out_bytes"])
    slack = 512 * (rep["params"] + rep["modules"] + 4)   # the allocator rounds every block to 512 bytes
    assert abs((before - after) - expect) <= slack, (before - after, expect)
    assert 0 < rep["index_bytes"] < rep["plan_bytes"]   # the segment index is part of the plans' memory


def test_selection_rules():
    model = make_model(torch.bfloat16, seed=4)
    noise = torch.nn.Linear(H, H, bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        noise.weight.view(torch.int16).copy_(torch.randint(-(1 << 15), 1 << 15, (H, H), dtype=torch.int16, device="cuda"))
    model.noise = noise
    with pytest.raises(ValueError, match="contains"):
        compress_module(model, [model.layers[0], model.layers[0].mlp.up_proj])
    assert len(list(model.parameters())) > 0       # nothing was changed by the refused call
    rep = compress_module(model)
    kept = dict(model.named_parameters())
    assert "noise.weight" in kept                  # uniform random bits do not compress: it stays dense
    assert all(p.dim() == 1 for n, p in kept.items() if n != "noise.weight")
    assert rep["params"] + len(kept) == len(_snapshot(make_model(torch.bfloat16))) + 1
    ids = torch.randint(0, VOCAB, (1, 4), device="cuda")
    with torch.inference_mode():
        model(ids)
    decompress_module(model)
    assert model.noise.weight is noise.weight


class Failing(torch.nn.Linear):
    def forward(self, x):
        raise KeyError("boom")


def test_weights_are_unbound_when_forward_raises():
    mod = Failing(64, 64, bias=False, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        mod.weight.normal_(0, 0.02)
    compress_module(mod)
    with torch.inference_mode(), pytest.raises(KeyError):
        mod(torch.zeros(1, 64, device="cuda", dtype=torch.bfloat16))
    assert "weight" not in mod.__dict__
