"""Loading models straight into compressed GPU residence (zipnn_b200.load_module) and saving them back from their
streams (zipnn_b200.save_module).

The llama-like model of test_resident_gpu (an lm_head tied to the embedding) is written by save_file / a plain
safetensors writer and loaded into a module built on meta, on the CPU and on CUDA: its logits equal the dense
model's bit for bit, directly and through a CUDA graph; the report and the streams equal compress_module's; device
memory stays within the documented bound and below the dense size; refused and corrupt loads leave memory and
module as they were; save_module writes save_file's bytes without decoding.
"""
import copy
import gc
import json
import os

import pytest
import torch
from safetensors.torch import save_file as plain_save_file

from golden_safetensors_inputs import make_checkpoint
from test_resident_gpu import VOCAB, H, Model, make_model
from zipnn_b200 import _native, compress_module, decompress_module, load_file, load_module, save_file, save_module
from zipnn_b200 import safetensors_io
from zipnn_b200.plan import _HEAD, _Stream
from zipnn_b200.resident import _ATTR, state_names

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_model.znn.safetensors")


def dealiased(model):
    sd = model.state_dict()
    del sd["lm_head.weight"]
    return sd


def build(where, dtype):
    if where == "meta":
        with torch.device("meta"):
            return Model().to(dtype).eval()
    torch.manual_seed(99)
    return Model().to(device=where, dtype=dtype).eval()


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


def resident_streams(model):
    """{name: stream bytes} of the compressed parameters, at their first names."""
    state = getattr(model, _ATTR)
    out = {}
    for name, _, _, kind, key in state_names(model):
        if kind == "resident" and key not in out.values():
            out[name] = key
    return {n: state.stream_of[k[1]].cpu() for n, k in out.items()}


def settle():
    gc.collect()
    torch.cuda.synchronize()
    return torch.cuda.memory_allocated()


@pytest.mark.parametrize("where", ["meta", "cpu", "cuda"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_znn_file_loads_exact(tmp_path, dtype, where):
    dense = make_model(dtype)
    path = str(tmp_path / "m.znn.safetensors")
    save_file(dealiased(dense), path)
    twin = copy.deepcopy(dense)
    want_rep = compress_module(twin)
    ids = torch.randint(0, VOCAB, (2, 11), device="cuda")
    with torch.inference_mode():
        want = dense(ids)
    model = build(where, dtype)
    requires = {n: p.requires_grad for n, p in model.named_parameters()}
    rep = load_module(model, path)
    for k in ("params", "modules", "dense_bytes", "stream_bytes"):
        assert rep[k] == want_rep[k], k
    got_streams, want_streams = resident_streams(model), resident_streams(twin)
    assert list(got_streams) == list(want_streams)
    assert all(torch.equal(got_streams[n], want_streams[n]) for n in want_streams)
    assert all(p.is_cuda for p in model.parameters()) and all(b.is_cuda for b in model.buffers())
    with torch.inference_mode():
        assert torch.equal(model(ids), want)
    assert torch.equal(graph_logits(model, ids), want)
    decompress_module(model)
    assert list(dict(model.named_parameters())) == list(dict(dense.named_parameters()))
    for (n, p), (_, q) in zip(model.named_parameters(), dense.named_parameters()):
        assert torch.equal(p.view(torch.uint8), q.view(torch.uint8)), n
        assert p.requires_grad == requires[n]
    assert model.lm_head.weight is model.embed_tokens.weight


class Noisy(Model):
    """The model plus a weight of uniform random bits, which does not compress."""

    def __init__(self):
        super().__init__()
        self.noise = torch.nn.Linear(H, H, bias=False)


def noisy_state(dtype):
    dense = make_model(dtype)
    sd = dealiased(dense)
    sd["noise.weight"] = torch.randint(-(1 << 15), 1 << 15, (H, H), dtype=torch.int16, device="cuda").view(dtype)
    return dense, sd


def test_plain_file_in_several_groups(tmp_path, monkeypatch):
    dense = make_model(torch.bfloat16, seed=5)
    path = str(tmp_path / "m.safetensors")
    plain_save_file({k: v.cpu() for k, v in dealiased(dense).items()}, path)
    twin = copy.deepcopy(dense)
    want_rep = compress_module(twin)
    group = 300_000
    monkeypatch.setattr(safetensors_io, "SAVE_GROUP_BYTES", group)
    model = build("meta", torch.bfloat16)
    base = settle()
    torch.cuda.reset_peak_memory_stats()
    rep = load_module(model, path)
    peak = torch.cuda.max_memory_allocated() - base
    assert len(getattr(model, _ATTR).streams) > 2            # one stream buffer per compressed group
    for k in ("params", "modules", "dense_bytes", "stream_bytes"):
        assert rep[k] == want_rep[k], k
    got_streams, want_streams = resident_streams(model), resident_streams(twin)
    assert all(torch.equal(got_streams[n], want_streams[n]) for n in want_streams)
    ids = torch.randint(0, VOCAB, (1, 7), device="cuda")
    with torch.inference_mode():
        assert torch.equal(model(ids), dense(ids))
    # what stays, plus one group: its input (at most the largest entry when that is over the budget), the streams'
    # bound and the workspace (both well under twice the input for these sizes), plus 16-byte stream alignment
    stays = _stays(model, rep)
    largest = max(t.numel() * t.element_size() for t in dealiased(dense).values())
    one_group = max(group, largest)
    assert peak <= stays + 3 * one_group + (1 << 20), (peak, stays, one_group)


def test_incompressible_weight_stays_dense(tmp_path):
    dense, sd = noisy_state(torch.bfloat16)
    path = str(tmp_path / "m.safetensors")
    plain_save_file({k: v.cpu() for k, v in sd.items()}, path)
    with torch.device("meta"):
        model = Noisy().to(torch.bfloat16).eval()
    rep = load_module(model, path)
    kept = dict(model.named_parameters())
    assert "noise.weight" in kept and torch.equal(kept["noise.weight"].view(torch.int16), sd["noise.weight"].view(torch.int16))
    assert rep["params"] > 0 and all(p.dim() == 1 for n, p in kept.items() if n != "noise.weight")
    ids = torch.randint(0, VOCAB, (1, 5), device="cuda")
    with torch.inference_mode():
        assert torch.equal(model(ids), dense(ids))


def _stays(model, rep):
    """Device bytes the loaded model keeps: streams (16-byte aligned), plans, scratch, output buffer, dense tensors."""
    state = getattr(model, _ATTR)
    streams = sum(b.numel() for b in state.streams)
    dense = sum(t.numel() * t.element_size() for t in {id(t): t for t in list(model.parameters()) + list(model.buffers())}.values())
    return streams + rep["plan_bytes"] + rep["scratch_bytes"] + rep["out_bytes"] + dense


def wide_stack():
    """Eight 2048 x 2048 linears: large enough that the shared output buffer and each stream's fixed costs (8 KiB of
    segment index per coded item) are small next to what compression saves, which they are not for the 2-layer model."""
    return torch.nn.Sequential(*[torch.nn.Linear(2048, 2048, bias=False) for _ in range(8)])


@pytest.mark.parametrize("kind", ["llama_like", "wide"])
def test_znn_load_peak_memory(tmp_path, kind):
    if kind == "llama_like":
        dense, new = make_model(torch.bfloat16, seed=6), lambda: build("meta", torch.bfloat16)
        sd = dealiased(dense)
    else:
        torch.manual_seed(6)
        dense = wide_stack().cuda().to(torch.bfloat16)
        with torch.no_grad():
            for p in dense.parameters():
                p.normal_(0, 0.02)
        sd = dense.state_dict()

        def new():
            with torch.device("meta"):
                return wide_stack().to(torch.bfloat16)
    path = str(tmp_path / "m.znn.safetensors")
    save_file(sd, path)
    dense_bytes = sum(t.numel() * t.element_size() for t in sd.values())
    del dense, sd
    model = new()
    base = settle()
    torch.cuda.reset_peak_memory_stats()
    rep = load_module(model, path)
    peak = torch.cuda.max_memory_allocated() - base
    state = getattr(model, _ATTR)
    blocks = len(list(model.parameters())) + 2 * rep["modules"] + len(state.streams) + 4
    heads = _HEAD * rep["params"]        # the plans' header peeks
    assert peak <= _stays(model, rep) + heads + 512 * blocks, (peak, _stays(model, rep))
    if kind == "wide":
        assert peak < dense_bytes, (peak, dense_bytes)


def test_reference_file():
    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            want = make_checkpoint()
            for n, t in want.items():
                if n != "ids":
                    setattr(self, n, torch.nn.Parameter(torch.empty_like(t, device="meta"), requires_grad=False))
            self.register_buffer("ids", torch.empty_like(want["ids"], device="meta"))

    want = make_checkpoint()
    model = Ref()
    rep = load_module(model, GOLDEN)
    assert rep["params"] == 5 and rep["modules"] == 1
    assert model.ids.is_cuda and torch.equal(model.ids.cpu(), want["ids"])
    decompress_module(model)
    for n, p in model.named_parameters():
        assert torch.equal(p.cpu().view(torch.uint8), want[n].view(torch.uint8)), n


def test_shards(tmp_path):
    dense = make_model(torch.float16, seed=7)
    sd = dealiased(dense)
    keys = sorted(sd)
    a, b = str(tmp_path / "a.znn.safetensors"), str(tmp_path / "b.safetensors")
    save_file({k: sd[k] for k in keys[::2]}, a)
    plain_save_file({k: sd[k].cpu() for k in keys[1::2]}, b)
    model = build("meta", torch.float16)
    rep = load_module(model, [a, b])
    assert rep["params"] == compress_module(copy.deepcopy(dense))["params"]
    ids = torch.randint(0, VOCAB, (1, 6), device="cuda")
    with torch.inference_mode():
        assert torch.equal(model(ids), dense(ids))


def _same_module(model, before):
    assert {n: p for n, p in model.named_parameters()} == before
    assert not hasattr(model, _ATTR)
    assert all(not m._forward_pre_hooks and not m._forward_hooks for m in model.modules())


def test_refusals_leave_memory_and_module(tmp_path):
    dense = make_model(torch.bfloat16, seed=8)
    sd = dealiased(dense)
    good = str(tmp_path / "m.znn.safetensors")
    save_file(sd, good)
    missing = str(tmp_path / "missing.znn.safetensors")
    save_file({k: v for k, v in sd.items() if k != "norm.weight"}, missing)
    wrong = str(tmp_path / "wrong.znn.safetensors")
    save_file(dict(sd, **{"layers.0.mlp.up_proj.weight": sd["layers.0.mlp.up_proj.weight"].half()}), wrong)
    # payload bytes of one compressed entry scrambled: the cumulative size of (byte group 1, chunk 0)
    name = "layers.1.mlp.gate_proj.weight"
    off, n = safetensors_io._safetensors_index(good)[name]
    blob = bytearray(open(good, "rb").read())
    s = _Stream(torch.empty(n, dtype=torch.uint8, device="meta"), bytes(blob[off: off + min(n, _HEAD)]))
    k = -(-s.nbytes // s.chunk)
    blob[off + s.after + s.num_buf * k + 8 * k + 3] ^= 0x40
    corrupt = str(tmp_path / "corrupt.znn.safetensors")
    open(corrupt, "wb").write(bytes(blob))
    for where in ("meta", "cuda"):
        model = build(where, torch.bfloat16)
        before = {n: p for n, p in model.named_parameters()}
        base = settle()
        for path, err, match in ((missing, ValueError, "norm.weight"), (wrong, ValueError, "up_proj"),
                                 (corrupt, RuntimeError, "corrupt")):
            with pytest.raises(err, match=match):
                load_module(model, path)
            assert settle() == base, path
            _same_module(model, before)
        load_module(model, good)
        with pytest.raises(ValueError, match="already compressed"):
            load_module(model, good)


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def test_save_module_writes_save_files_bytes(tmp_path):
    dense = make_model(torch.bfloat16, seed=9)
    want = str(tmp_path / "want.znn.safetensors")
    save_file(dealiased(dense), want)
    never = str(tmp_path / "never.znn.safetensors")
    save_module(dense, never)
    assert _bytes(never) == _bytes(want)
    comp = copy.deepcopy(dense)
    compress_module(comp)
    out = str(tmp_path / "compressed.znn.safetensors")
    save_module(comp, out)
    assert _bytes(out) == _bytes(want)
    loaded = build("meta", torch.bfloat16)
    load_module(loaded, want)
    again = str(tmp_path / "again.znn.safetensors")
    save_module(loaded, again)
    assert _bytes(again) == _bytes(want)


def test_save_module_launches_no_kernel_without_dense_floats(tmp_path):
    model = torch.nn.Module()
    want = make_checkpoint()
    for n, t in want.items():
        if n != "ids":
            setattr(model, n, torch.nn.Parameter(torch.empty_like(t, device="meta"), requires_grad=False))
    model.register_buffer("ids", torch.empty_like(want["ids"], device="meta"))
    load_module(model, GOLDEN)
    assert all(p.dtype == torch.int64 for p in list(model.parameters()) + list(model.buffers()))
    out = str(tmp_path / "saved.znn.safetensors")
    torch.cuda.synchronize()
    before = _native.launch_count()
    save_module(model, out)
    torch.cuda.synchronize()
    assert _native.launch_count() == before
    back = load_file(out, device="cuda")
    assert back.keys() == want.keys()
    for n, t in want.items():
        assert torch.equal(back[n].cpu().view(torch.uint8), t.view(torch.uint8)), n
    with open(out, "rb") as f:
        meta = json.loads(f.read(int.from_bytes(f.read(8), "little")))["__metadata__"]
    assert set(json.loads(meta["znn_compressed_vectors"])) == {n for n in want if n != "ids"}
