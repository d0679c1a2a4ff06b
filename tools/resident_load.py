#!/usr/bin/env python3
"""Loading a model straight into compressed GPU residence, and saving it back, on llama3-8b shapes.

The checkpoint has the tensors of tools/model_bench.py:llama_like (llama3-8b dims, --layers of them, an untied
lm_head), seeded bf16 with std 0.02 (norms 1.0), written as a plain .safetensors file and as a .znn.safetensors file
(zipnn_b200.save_file) under --dir (default /dev/shm, else the temporary directory).  In one process, with the ways
alternating over --reps rounds, it measures wall time (ending in a device synchronise) and the peak of
torch.cuda.max_memory_allocated over the starting allocation of:
  * dense:            zipnn_b200.load_file(.znn, device="cuda") + load_state_dict(assign=True) into a meta model;
  * dense+compress:   the same followed by compress_module;
  * load_module_znn:  load_module from the .znn file;
  * load_module_plain: load_module from the plain file;
and of saving the resident model: save_module against decompress_module + save_file.  It checks that the logits of
both resident models equal the dense model's at a few tokens.  Prints one JSON line with the card and its power limit.

usage: python tools/resident_load.py [--layers 8] [--reps 2] [--dir /dev/shm]
"""
import argparse
import gc
import json
import os
import shutil
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from safetensors.torch import save_file as plain_save_file  # noqa: E402

from tools.model_bench import llama_like  # noqa: E402
from tools.plan_bench import FFN, HEADS, KV, H, power_limit  # noqa: E402
from zipnn_b200 import compress_module, decompress_module, load_file, load_module, save_file, save_module  # noqa: E402

VOCAB = 128256


def lin(i, o):
    return torch.nn.Linear(i, o, bias=False)


class Attn(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.q_proj, self.k_proj, self.v_proj, self.o_proj = lin(H, H), lin(H, KV), lin(H, KV), lin(H, H)


class MLP(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.gate_proj, self.up_proj, self.down_proj = lin(H, FFN), lin(H, FFN), lin(FFN, H)


class Layer(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.self_attn, self.mlp = Attn(), MLP()
        self.input_layernorm, self.post_attention_layernorm = torch.nn.RMSNorm(H), torch.nn.RMSNorm(H)

    def forward(self, x):
        a, m = self.self_attn, self.mlp
        b, t, _ = x.shape
        h = self.input_layernorm(x)
        q = a.q_proj(h).view(b, t, HEADS, -1).transpose(1, 2)
        k = a.k_proj(h).view(b, t, KV // 128, -1).transpose(1, 2).repeat_interleave(HEADS * 128 // KV, dim=1)
        v = a.v_proj(h).view(b, t, KV // 128, -1).transpose(1, 2).repeat_interleave(HEADS * 128 // KV, dim=1)
        x = x + a.o_proj(F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(b, t, H))
        h = self.post_attention_layernorm(x)
        return x + m.down_proj(F.silu(m.gate_proj(h)) * m.up_proj(h))


class Inner(torch.nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.embed_tokens = torch.nn.Embedding(VOCAB, H)
        self.layers = torch.nn.ModuleList([Layer() for _ in range(layers)])
        self.norm = torch.nn.RMSNorm(H)


class Llama(torch.nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.model = Inner(layers)
        self.lm_head = lin(H, VOCAB)

    def forward(self, ids):
        x = self.model.embed_tokens(ids)
        for layer in self.model.layers:
            x = layer(x)
        return self.lm_head(self.model.norm(x))


def meta_model(layers):
    with torch.device("meta"):
        return Llama(layers).to(torch.bfloat16).eval()


def checkpoint(layers):
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {}
    for name, shape in llama_like(layers, H, FFN, VOCAB, KV).items():
        if len(shape) == 1:
            out[name] = torch.ones(shape, dtype=torch.bfloat16, device="cuda")
        else:
            out[name] = (torch.randn(shape, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    return out


def settle():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return torch.cuda.memory_allocated()


def measured(fn):
    """-> (fn's result, wall seconds, peak device bytes above the starting allocation)."""
    base = settle()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--dir", default="/dev/shm")
    a = ap.parse_args()
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "layers": a.layers}
    sd = checkpoint(a.layers)
    dense_bytes = sum(t.numel() * t.element_size() for t in sd.values())
    need = 2 * dense_bytes
    root = a.dir if os.path.isdir(a.dir) and shutil.disk_usage(a.dir).free > 1.2 * need else tempfile.gettempdir()
    work = tempfile.mkdtemp(prefix="resident_load_", dir=root)
    try:
        plain, znn = os.path.join(work, "m.safetensors"), os.path.join(work, "m.znn.safetensors")
        plain_save_file({k: v.cpu() for k, v in sd.items()}, plain)
        save_file(sd, znn)
        del sd
        res["dense_bytes"] = dense_bytes
        res["file_bytes"] = {"plain": os.path.getsize(plain), "znn": os.path.getsize(znn)}

        def dense():
            m = meta_model(a.layers)
            m.load_state_dict(load_file(znn, device="cuda"), assign=True)
            return m

        def dense_compress():
            m = dense()
            return m, compress_module(m)

        def resident(path):
            m = meta_model(a.layers)
            return m, load_module(m, path)

        ways = {"dense": dense, "dense+compress": dense_compress, "load_module_znn": lambda: resident(znn),
                "load_module_plain": lambda: resident(plain)}
        times = {k: [] for k in ways}
        peaks = {k: [] for k in ways}
        for _ in range(a.reps):
            for k, fn in ways.items():
                r, t, p = measured(fn)
                times[k].append(round(t, 3))
                peaks[k].append(p)
                if k == "load_module_znn":
                    res["report"] = r[1]
                del r
        res["load_s"] = times
        res["load_peak_bytes"] = {k: max(v) for k, v in peaks.items()}

        # logits of both resident models against the dense model at a few tokens
        ids = torch.randint(0, VOCAB, (1, 4), device="cuda")
        ref = dense()
        with torch.inference_mode():
            want = ref(ids)
        del ref
        settle()
        exact = {}
        for k, path in (("znn", znn), ("plain", plain)):
            m, _ = resident(path)
            with torch.inference_mode():
                exact[k] = bool(torch.equal(m(ids), want))
            del m
        res["logits_equal"] = exact

        # saving the resident model: from its streams, against decoding it first
        save_s = {"save_module": [], "decompress+save_file": []}
        save_peak = {k: 0 for k in save_s}
        out = os.path.join(work, "out.znn.safetensors")
        for _ in range(a.reps):
            m, _ = resident(znn)
            _, t, p = measured(lambda: save_module(m, out))
            save_s["save_module"].append(round(t, 3))
            save_peak["save_module"] = max(save_peak["save_module"], p)
            same = open(out, "rb").read() == open(znn, "rb").read()

            def decoded_save():
                decompress_module(m)
                save_file(m.state_dict(), out)
            _, t, p = measured(decoded_save)
            save_s["decompress+save_file"].append(round(t, 3))
            save_peak["decompress+save_file"] = max(save_peak["decompress+save_file"], p)
            del m
        res["save_s"] = save_s
        res["save_peak_bytes"] = save_peak
        res["save_module_reproduces_file"] = same
    finally:
        shutil.rmtree(work, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
