"""Resident models whose embedding runs as a gather (compress_module / load_module with gather=True).

The llama-like model of test_resident_gpu (lm_head tied to the embedding) and an untied variant, in bf16, fp16 and
fp32: logits equal the dense model's bit for bit, directly, through a captured CUDA graph and with prefetch; the
embedding is never decoded whole; the shared output buffer is sized by the largest module still decoded whole;
decompress_module restores the weights and save_module writes the gather=False file; load_module from a
.znn.safetensors file gives the same, within gather=False's peak device memory.
"""
import copy
import gc

import pytest
import torch

from test_resident_gpu import VOCAB, H, FFN, Model, make_model
from zipnn_b200 import DecodePlan, compress_module, decompress_module, load_module, save_module
from zipnn_b200.resident import _ATTR

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def untie(m):
    m.lm_head.weight = torch.nn.Parameter(m.embed_tokens.weight.detach().clone() * 0.5)
    return m


def make(dtype, tied, seed=0):
    m = make_model(dtype, seed)
    return m if tied else untie(m)


def graph_logits(model, ids):
    with torch.inference_mode():
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
    return out.clone()


class RunCounter:
    """Counts DecodePlan.run calls per plan."""

    def __init__(self, monkeypatch):
        self.calls = {}
        orig = DecodePlan.run
        counter = self

        def run(plan):
            counter.calls[id(plan)] = counter.calls.get(id(plan), 0) + 1
            return orig(plan)
        monkeypatch.setattr(DecodePlan, "run", run)


@pytest.mark.parametrize("tied", [True, False])
@pytest.mark.parametrize("dtype", DTYPES)
def test_logits_exact_and_embedding_never_decoded_whole(dtype, tied, monkeypatch):
    dense = make(dtype, tied)
    model = copy.deepcopy(dense)
    ids = torch.randint(0, VOCAB, (2, 17), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    rep = compress_module(model, gather=True)
    state = getattr(model, _ATTR)
    assert rep["gather_modules"] == 1 and [m for m, _, _, _ in state.gathers] == [model.embed_tokens]
    _, plan, k, own = state.gathers[0]
    assert own == (not tied)
    if tied:
        assert plan is next(p for m, p, _, _ in state.entries if m is model.lm_head) and rep["gather_bytes"] == 0
    else:
        assert plan.outputs is None and rep["gather_bytes"] == plan.nbytes["plan"]   # the plan of its own, no output
    assert all(m is not model.embed_tokens for m, _, _, _ in state.entries)
    counter = RunCounter(monkeypatch)
    with torch.inference_mode():
        got = model(ids)
    assert torch.equal(got, want)
    # every module decoded whole ran its plan once; the embedding ran none (a plan of its own would raise)
    assert sorted(counter.calls.values()) == [1] * len(state.entries)
    assert set(counter.calls) == {id(p) for _, p, _, _ in state.entries}
    with torch.inference_mode():
        emb = model.embed_tokens(ids)
    with torch.inference_mode():
        assert torch.equal(emb, dense.embed_tokens(ids))
    assert torch.equal(graph_logits(model, ids), want)
    with pytest.raises(RuntimeError, match="no_grad"):
        model.embed_tokens(ids)
    plan.check()
    decompress_module(model)
    for (n, a), (_, b) in zip(model.named_parameters(), dense.named_parameters()):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), n
    assert (model.lm_head.weight is model.embed_tokens.weight) == tied
    assert "forward" not in model.embed_tokens.__dict__
    with torch.inference_mode():
        assert torch.equal(model(ids), want)


@pytest.mark.parametrize("tied", [True, False])
@pytest.mark.parametrize("dtype", DTYPES)
def test_prefetch_with_gather(dtype, tied):
    dense = make(dtype, tied, seed=1)
    model = copy.deepcopy(dense)
    ids = torch.randint(0, VOCAB, (1, 9), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    rep = compress_module(model, prefetch=True, gather=True)
    state = getattr(model, _ATTR)
    assert state.gather_scratch is not state.scratch and rep["gather_bytes"] >= state.gather_scratch.numel()
    with torch.inference_mode():
        for _ in range(3):
            assert torch.equal(model(ids), want)
    assert torch.equal(graph_logits(model, ids), want)
    decompress_module(model)
    with torch.inference_mode():
        assert torch.equal(model(ids), want)


def test_out_bytes_is_the_largest_module_decoded_whole():
    dense = make(torch.bfloat16, tied=False, seed=2)
    selection = lambda m: [m.embed_tokens] + [lin for layer in m.layers for lin in layer.modules() if isinstance(lin, torch.nn.Linear)]
    a, b = copy.deepcopy(dense), copy.deepcopy(dense)
    rep_off = compress_module(a, modules=selection(a))
    rep_on = compress_module(b, modules=selection(b), gather=True)
    assert rep_off["out_bytes"] == VOCAB * H * 2                  # the embedding sets it without gathers
    assert rep_on["out_bytes"] == H * FFN * 2                     # the largest linear left (lm_head is not selected)
    assert rep_on["gather_modules"] == 1 and rep_on["modules"] == rep_off["modules"]
    ids = torch.randint(0, VOCAB, (3, 5), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
        assert torch.equal(a(ids), want) and torch.equal(b(ids), want)


@pytest.mark.parametrize("tied", [True, False])
def test_save_module_writes_the_gather_off_file(tmp_path, tied):
    dense = make(torch.bfloat16, tied, seed=3)
    a, b = copy.deepcopy(dense), copy.deepcopy(dense)
    compress_module(a)
    compress_module(b, gather=True)
    pa, pb = str(tmp_path / "a.znn.safetensors"), str(tmp_path / "b.znn.safetensors")
    save_module(a, pa)
    save_module(b, pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()


def _meta(dtype, tied):
    with torch.device("meta"):
        m = Model().to(dtype).eval()
    if not tied:
        m.lm_head.weight = torch.nn.Parameter(torch.empty(VOCAB, H, dtype=dtype, device="meta"))
    return m


def _peak_load(path, dtype, tied, **kw):
    model = _meta(dtype, tied)
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    rep = load_module(model, path, **kw)
    torch.cuda.synchronize()
    return model, rep, torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("tied", [True, False])
@pytest.mark.parametrize("dtype", DTYPES)
def test_load_module_gather(tmp_path, dtype, tied):
    dense = make(dtype, tied, seed=4)
    src = copy.deepcopy(dense)
    compress_module(src)
    path = str(tmp_path / "m.znn.safetensors")
    save_module(src, path)
    del src
    ids = torch.randint(0, VOCAB, (2, 11), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    m_off, rep_off, peak_off = _peak_load(path, dtype, tied)
    del m_off
    m_on, rep_on, peak_on = _peak_load(path, dtype, tied, gather=True)
    assert peak_on <= peak_off, (peak_on, peak_off)
    assert rep_on["gather_modules"] == 1
    with torch.inference_mode():
        assert torch.equal(m_on(ids), want)
    assert torch.equal(graph_logits(m_on, ids), want)
    again = str(tmp_path / "again.znn.safetensors")
    save_module(m_on, again)
    assert open(again, "rb").read() == open(path, "rb").read()
    decompress_module(m_on)
    for (n, a), (_, b) in zip(m_on.named_parameters(), dense.named_parameters()):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), n
