#!/usr/bin/env python3
"""The selected fp8 dequantize (DecodePlan.dequant_fp8_select) on real mixture-of-experts layer shapes, and the resident
fp8 experts mode (compress_module(fp8=True, experts=True)).

Layers: Qwen3-30B-A3B-FP8 (128 experts, top-8, H 2048, I 768) and a Mixtral-8x7B-shaped fp8 layer (8 experts, top-2,
H 4096, I 14336): gate_up_proj [E, 2I, H] and down_proj [E, H, I] from seeded bf16 Gaussian weights (std 0.02),
quantized to float8_e4m3fn per 128x128 block at amax / 448, one grid per expert.  Routings: uniform and Zipf (s = 1.2
over the experts, in a seeded random order), top-k distinct experts per token, at 1, 4, 16, 64 and 256 tokens.  In one
process, alternating and timed with CUDA events after warm-up, every output checked before it is timed; each point is the
median of --iters calls, repeated --repeats times (the spread is the range of those medians):
  * `dequant_fp8_select` of the routed experts into fixed outputs; `run_select` + torch's dequantize of the whole
    tensors (what could be written without it); `dequant_fp8` of the whole tensors; the chunks the routing touches, and
    the stream bytes of those chunks plus the bf16 bytes written per ms (GB/s);
  * the same call captured in a CUDA graph and replayed, at 1 token;
  * the experts module forward (transformers' FP8Experts, resident with fp8=True, experts=True) against a dense bf16
    copy with torch-dequantized weights, under the eager and grouped_mm experts implementations, outputs equal bit for bit.
Prints one JSON line with the card name and its power limit.

usage: python tools/fp8_experts_bench.py [--iters 20] [--warmup 5] [--repeats 3]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.fp8_linear_bench import spread  # noqa: E402
from tools.plan_bench import power_limit  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402
from zipnn_b200 import resident as R  # noqa: E402

LAYERS = {"qwen3-30b-a3b": dict(E=128, k=8, H=2048, I=768), "mixtral-8x7b": dict(E=8, k=2, H=4096, I=14336)}
TOKENS = (1, 4, 16, 64, 256)
B = 128
FP8_CHUNK = 131072   # the chunk of ZipNN's fp8 streams (one byte plane: 128 KiB)


def quantize_experts(E, out, inn, gen):
    """-> (W [E, out, in] e4m3fn, S [E, out / 128, in / 128] fp32), one expert at a time."""
    q = torch.empty(E, out, inn, dtype=torch.float8_e4m3fn, device="cuda")
    s = torch.empty(E, out // B, inn // B, device="cuda")
    for e in range(E):
        w = (torch.randn(out, inn, generator=gen, device="cuda") * 0.02).to(torch.bfloat16).float()
        blocks = w.view(out // B, B, inn // B, B)
        s[e] = (blocks.abs().amax(dim=(1, 3)) / 448.0).clamp_min(2.0 ** -30)
        q[e] = (blocks / s[e][:, None, :, None]).view(out, inn).to(torch.float8_e4m3fn)
    return q, s


def routing(kind, E, k, tokens, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        p = torch.ones(E)
    else:
        p = 1.0 / torch.arange(1, E + 1, dtype=torch.float64) ** 1.2
        p = p[torch.randperm(E, generator=g)]
    return torch.multinomial(p.expand(tokens, E), k, replacement=False, generator=g).cuda()


def touched(nbytes, chunk, E, ids):
    """Chunks a selection touches (whole-tensor item of E slices)."""
    S = nbytes // E
    mark = np.zeros(-(-nbytes // chunk), dtype=bool)
    for e in set(ids):
        mark[e * S // chunk: ((e + 1) * S - 1) // chunk + 1] = True
    return int(mark.sum()), mark.size


def layer_table(name, cfg, a, gen):
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    ws = [quantize_experts(E, 2 * I, H, gen), quantize_experts(E, H, I, gen)]
    streams = [ZipNN(input_format="torch").compress(q) for q, _ in ws]
    plan = DecodePlan(streams)
    inf, scales, blocks = [H, I], [s for _, s in ws], [(B, B)] * 2
    assert plan.dequant_fp8_select_ok(inf), name
    outs = [torch.empty(q.shape, dtype=torch.bfloat16, device="cuda") for q, _ in ws]
    whole = [torch.empty(q.shape, dtype=torch.bfloat16, device="cuda").view(-1, q.shape[-1]) for q, _ in ws]
    flat = [s.reshape(-1, s.shape[-1]) for s in scales]
    scratch = torch.empty(plan.select_scratch_bytes(), dtype=torch.uint8, device="cuda")
    chunk = FP8_CHUNK
    table = {"chunks": sum(-(-q.numel() // chunk) for q, _ in ws), "stream_bytes": plan.nbytes["streams"], "routings": {}}
    fns = [lambda ids: plan.dequant_fp8_select(ids, inf, scales, blocks, outs=outs, scratch=scratch),
           lambda ids: [R.dequantize_fp8(o, s, (B, B), torch.bfloat16) for o, s in zip(plan.run_select(ids, scratch=scratch), scales)],
           lambda ids: [plan.dequant_fp8(j, inf[j], flat[j], (B, B), out=whole[j]) for j in range(2)]]
    keys = ["dequant_fp8_select", "run_select_torch_dequant", "dequant_fp8_whole"]
    for kind in ("uniform", "zipf"):
        for tokens in TOKENS:
            ids = routing(kind, E, k, tokens, tokens + (kind == "zipf"))
            sel = sorted(set(ids.reshape(-1).tolist()))
            got = fns[0](ids)
            for (q, s), o in zip(ws, got):
                for e in sel[:4] + sel[-2:]:
                    want = R.dequantize_fp8(q[e], s[e], (B, B), torch.bfloat16)
                    assert torch.equal(o[e].view(torch.int16), want.view(torch.int16)), (name, kind, tokens, e)
            t = spread([lambda f=f: f(ids) for f in fns], a)
            n_touch = [touched(q.numel(), chunk, E, sel) for q, _ in ws]
            moved = sum(st.numel() * c / K for st, (c, K) in zip(streams, n_touch)) + sum(2 * q[0].numel() * len(sel) for q, _ in ws)
            table["routings"][f"{kind} {tokens}"] = dict(zip(keys, t), experts=len(sel), chunks=sum(c for c, _ in n_touch),
                                                         select_gbps=moved / t[0]["ms"] / 1e6)
    # a captured call at 1 token, replayed with new ids
    ids = routing("uniform", E, k, 1, 99)
    fns[0](ids)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fns[0](ids)
    ids.copy_(routing("uniform", E, k, 1, 100))
    g.replay()
    sel = sorted(set(ids.reshape(-1).tolist()))
    for (q, s), o in zip(ws, outs):
        assert torch.equal(o[sel[0]].view(torch.int16), R.dequantize_fp8(q[sel[0]], s[sel[0]], (B, B), torch.bfloat16).view(torch.int16))
    t = spread([g.replay, lambda: fns[0](ids)], a)
    table["graph_1_token"] = {"replay": t[0], "eager": t[1]}
    plan.check()
    print(json.dumps({name: table}), file=sys.stderr, flush=True)   # (progress: the layer's table so far)
    table["module"] = module_table(name, cfg, ws, a)
    return table


def module_table(name, cfg, ws, a):
    import transformers as tf
    from transformers.integrations.finegrained_fp8 import ALL_FP8_EXPERTS_FUNCTIONS, FP8Experts
    from transformers.integrations.moe import use_experts_implementation
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    # (a config that only sizes the experts module: FP8Experts reads hidden, intermediate, experts and the activation)
    conf = tf.Qwen3MoeConfig(hidden_size=H, moe_intermediate_size=I, num_experts=E, num_experts_per_tok=k)
    cls = use_experts_implementation(experts_class=type("FP8Experts", (FP8Experts,), {}), experts_interface=ALL_FP8_EXPERTS_FUNCTIONS)
    with torch.device("meta"):
        mod = cls(conf, block_size=(B, B))
    mod.gate_up_proj = torch.nn.Parameter(ws[0][0], requires_grad=False)
    mod.gate_up_proj_scale_inv = torch.nn.Parameter(ws[0][1], requires_grad=False)
    mod.down_proj = torch.nn.Parameter(ws[1][0], requires_grad=False)
    mod.down_proj_scale_inv = torch.nn.Parameter(ws[1][1], requires_grad=False)
    dense = copy.copy(mod)
    dense._parameters = dict(mod._parameters)
    for p in ("gate_up_proj", "down_proj"):
        dense._parameters[p] = torch.nn.Parameter(R.dequantize_fp8(getattr(mod, p), getattr(mod, p + "_scale_inv"), (B, B), torch.bfloat16),
                                                  requires_grad=False)
    root = torch.nn.ModuleDict({"experts": mod})
    report = compress_module(root, fp8=True, experts=True)
    assert report["fp8_experts_modules"] == 1, report
    table = {"report": report}
    for impl in ("eager", "grouped_mm"):
        conf._experts_implementation = impl
        for tokens in (1, 16, 64):
            x = (torch.randn(tokens, H, device="cuda") * 0.5).to(torch.bfloat16)
            ids = routing("uniform", E, k, tokens, 7 + tokens)
            w = torch.rand(tokens, k, device="cuda").to(torch.bfloat16)
            fns = [lambda: mod(x, ids, w), lambda: R._experts_impl(dense)(dense, x, ids, w)]
            assert torch.equal(fns[0]().view(torch.int16), fns[1]().view(torch.int16)), (name, impl, tokens)
            t = spread(fns, a)
            table[f"{impl} {tokens}"] = {"resident_fp8_experts": t[0], "dense_bf16": t[1]}
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--layers", default=",".join(LAYERS))
    a = ap.parse_args()
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "weights": "e4m3fn, 128x128 blocks per expert, amax / 448",
           "iters": a.iters, "repeats": a.repeats}
    gen = torch.Generator("cuda").manual_seed(0)
    with torch.no_grad():
        for name in a.layers.split(","):
            res[name] = layer_table(name, LAYERS[name], a, gen)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
