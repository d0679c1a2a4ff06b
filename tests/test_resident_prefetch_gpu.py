"""Compressed-resident modules with prefetch (compress_module / load_module with prefetch=True).

The llama-like model of test_resident_gpu computes exactly the dense model's logits over several consecutive forwards
(so the learned successors are used), directly and through a captured CUDA graph of the root forward; so do models
whose forward order changes between calls, that call a module twice, and whose forward raises and then runs again;
so does the reference-made .znn file loaded with prefetch.  decompress_module gives back every parameter and leaves no
hook; the second output slot is the only memory prefetch adds; prefetch=False keeps the report as it was.
"""
import copy
import gc
import os

import pytest
import torch

from test_resident_gpu import VOCAB, Model, make_model
from test_resident_load_gpu import GOLDEN, graph_logits
from golden_safetensors_inputs import make_checkpoint
from zipnn_b200 import compress_module, decompress_module, load_module

pytestmark = pytest.mark.gpu


def _snapshot(m):
    return {n: p.detach().clone() for n, p in m.named_parameters()}


def _no_hooks(m):
    return all(not x._forward_pre_hooks and not x._forward_hooks for x in m.modules())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_llama_like_exact_over_forwards(dtype):
    dense = make_model(dtype)
    model = copy.deepcopy(dense)
    before = _snapshot(model)
    ids1 = torch.randint(0, VOCAB, (1, 1), device="cuda")
    ids8 = torch.randint(0, VOCAB, (2, 9), device="cuda")
    with torch.inference_mode():
        want1, want8 = dense(ids1), dense(ids8)
    rep = compress_module(model, prefetch=True)
    assert rep["prefetch_out_bytes"] == rep["out_bytes"]
    with torch.inference_mode():
        for _ in range(3):
            assert torch.equal(model(ids1), want1)
            assert torch.equal(model(ids8), want8)
    for _ in range(2):
        assert torch.equal(graph_logits(model, ids8), want8)
    decompress_module(model)
    assert _no_hooks(model)
    after = _snapshot(model)
    assert after.keys() == before.keys()
    assert all(torch.equal(after[n].view(torch.uint8), before[n].view(torch.uint8)) for n in before)


def test_graph_replayed_several_times():
    dense = make_model(torch.bfloat16)
    model = copy.deepcopy(dense)
    ids = torch.randint(0, VOCAB, (1, 4), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    compress_module(model, prefetch=True)
    with torch.inference_mode():
        model(ids)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(ids)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = model(ids)
        for _ in range(4):
            out.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, want)
        assert torch.equal(model(ids), want)


class Shuffled(Model):
    """Layers in an order given per call, one layer possibly twice, and an optional failure after the first layer."""

    def forward(self, ids, order=(0, 1), fail=False):
        x = self.embed_tokens(ids)
        for j, i in enumerate(order):
            x = self.layers[i](x)
            if fail and j == 0:
                raise RuntimeError("forward failed on purpose")
        return self.lm_head(self.norm(x))


def test_changed_order_repeated_module_and_raise():
    torch.manual_seed(0)
    dense = Shuffled()
    with torch.no_grad():
        for p in dense.parameters():
            p.copy_(0.02 * torch.randn_like(p) if p.dim() > 1 else 1 + 0.1 * torch.randn_like(p))
    dense = dense.to(device="cuda", dtype=torch.bfloat16).eval()
    model = copy.deepcopy(dense)
    compress_module(model, prefetch=True)
    ids = torch.randint(0, VOCAB, (1, 5), device="cuda")
    orders = [(0, 1), (0, 1), (1, 0), (0, 1), (1, 1), (0, 0, 1), (1, 1), (0, 1)]
    with torch.inference_mode():
        for k, order in enumerate(orders):
            if k == 4:
                with pytest.raises(RuntimeError, match="on purpose"):
                    model(ids, order, fail=True)
                for m in model.modules():
                    assert "weight" not in m.__dict__
            assert torch.equal(model(ids, order), dense(ids, order)), order
        # a submodule called directly, outside a root forward: serial and joined
        x = torch.randn(1, 5, 256, device="cuda", dtype=torch.bfloat16)
        assert torch.equal(model.layers[1](x), dense.layers[1](x))
        assert torch.equal(model(ids), dense(ids))


def test_reference_file_with_prefetch():
    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            want = make_checkpoint()
            for n, t in want.items():
                if n != "ids":
                    setattr(self, n, torch.nn.Parameter(torch.empty_like(t, device="meta"), requires_grad=False))
            self.register_buffer("ids", torch.empty_like(want["ids"], device="meta"))

        def forward(self):
            return {n: p.clone() for n, p in self.__dict__.items() if isinstance(p, torch.Tensor) and n != "ids"}

    want = make_checkpoint()
    model = Ref()
    rep = load_module(model, GOLDEN, prefetch=True)
    assert rep["params"] == 5 and rep["prefetch_out_bytes"] == rep["out_bytes"]
    with torch.inference_mode():
        for _ in range(3):
            got = model()
            assert got.keys() == {n for n in want if n != "ids"}
            for n, t in got.items():
                assert torch.equal(t.cpu().view(torch.uint8), want[n].view(torch.uint8)), n
    decompress_module(model)
    assert _no_hooks(model)
    for n, p in model.named_parameters():
        assert torch.equal(p.cpu().view(torch.uint8), want[n].view(torch.uint8)), n


def _settle():
    gc.collect()
    torch.cuda.synchronize()
    return torch.cuda.memory_allocated()


def test_memory_and_serial_report():
    dense = make_model(torch.bfloat16)
    a, b = copy.deepcopy(dense), copy.deepcopy(dense)
    del dense
    m0 = _settle()
    rep_a = compress_module(a)
    m1 = _settle()
    rep_b = compress_module(b, prefetch=True)
    m2 = _settle()
    assert "prefetch_out_bytes" not in rep_a
    assert {k: v for k, v in rep_b.items() if k != "prefetch_out_bytes"} == rep_a
    # both compressed b's dense weights away; b holds one more output buffer (rounded to the allocator's 512 bytes)
    slot = (rep_b["prefetch_out_bytes"] + 511) // 512 * 512
    assert (m2 - m1) - (m1 - m0) == slot
    decompress_module(a)
    decompress_module(b)
    assert _settle() == m0   # slot 1 is freed with the rest
