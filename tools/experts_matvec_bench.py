#!/usr/bin/env python3
"""The selected experts matvec (DecodePlan.experts_matvec_fp8) on real mixture-of-experts layer shapes, and the resident
"fp8_experts_matvec" mode (compress_module(fp8=True, experts=True, experts_matvec=4)).

Layers: those of tools/fp8_experts_bench.py, Qwen3-30B-A3B-FP8 (128 experts, top-8, H 2048, I 768) and a
Mixtral-8x7B-shaped fp8 layer (8 experts, top-2, H 4096, I 14336), float8_e4m3fn per 128x128 block.  Routings uniform
and Zipf at 1, 2 and 4 tokens (the most the kernel takes).  In one process, alternating and timed with CUDA events after
warm-up, every output checked first; each point is the median of --iters calls, repeated --repeats times (the spread is
the range of those medians):
  * plan level: the two experts_matvec_fp8 calls (first projection with x [T, H], down with x [T, k, I]) against
    dequant_fp8_select of both items, and that plus the bf16 grouped_mm the "fp8_experts" forward runs; a 1-token
    graph replay of the two calls;
  * module level: the resident FP8Experts forward with experts_matvec=4 against the same without it, and against a dense
    bf16 copy, under the grouped_mm and eager experts implementations.
Prints one JSON line with the card name and its power limit.

usage: python tools/experts_matvec_bench.py [--iters 20] [--warmup 5] [--repeats 3]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.fp8_experts_bench import LAYERS, B, quantize_experts, routing  # noqa: E402
from tools.fp8_linear_bench import spread  # noqa: E402
from tools.plan_bench import power_limit  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402
from zipnn_b200 import resident as R  # noqa: E402
from zipnn_b200.plan import EXPERTS_MATVEC_MAX_TOKENS  # noqa: E402

TOKENS = (1, 2, 4)


def experts_module(cfg, ws):
    import transformers as tf
    from transformers.integrations.finegrained_fp8 import ALL_FP8_EXPERTS_FUNCTIONS, FP8Experts
    from transformers.integrations.moe import use_experts_implementation
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    conf = tf.Qwen3MoeConfig(hidden_size=H, moe_intermediate_size=I, num_experts=E, num_experts_per_tok=k)
    cls = use_experts_implementation(experts_class=type("FP8Experts", (FP8Experts,), {}), experts_interface=ALL_FP8_EXPERTS_FUNCTIONS)
    with torch.device("meta"):
        mod = cls(conf, block_size=(B, B))
    for p, (q, s) in zip(("gate_up_proj", "down_proj"), ws):
        mod._parameters[p] = torch.nn.Parameter(q, requires_grad=False)
        mod._parameters[p + "_scale_inv"] = torch.nn.Parameter(s, requires_grad=False)
    return conf, mod


def layer_table(name, cfg, a, gen):
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    ws = [quantize_experts(E, 2 * I, H, gen), quantize_experts(E, H, I, gen)]
    plan = DecodePlan([ZipNN(input_format="torch").compress(q) for q, _ in ws])
    inf, scales, blocks = [H, I], [s for _, s in ws], [(B, B)] * 2
    assert plan.experts_matvec_fp8_ok(0, H) and plan.experts_matvec_fp8_ok(1, I), name
    need = max(plan.experts_matvec_fp8_scratch_bytes(j, inf[j], k) for j in range(2))
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    sel_scratch = torch.empty(plan.select_scratch_bytes(), dtype=torch.uint8, device="cuda")
    outs = [torch.empty(q.shape, dtype=torch.bfloat16, device="cuda") for q, _ in ws]
    conf, mod = experts_module(cfg, ws)
    conf._experts_implementation = "grouped_mm"
    table = {"routings": {}}

    def products(x, ids):
        h = plan.experts_matvec_fp8(0, ids, x, scales[0], (B, B), scratch=scratch)
        return plan.experts_matvec_fp8(1, ids, mod._apply_gate(h), scales[1], (B, B), scratch=scratch)

    def selected(ids):
        return plan.dequant_fp8_select(ids, inf, scales, blocks, outs=outs, scratch=sel_scratch)

    def selected_grouped(x, ids, w):
        selected(ids)
        mod.__dict__["gate_up_proj"], mod.__dict__["down_proj"] = outs
        try:
            return R._experts_impl(mod)(mod, x, ids, w)
        finally:
            del mod.__dict__["gate_up_proj"], mod.__dict__["down_proj"]

    for kind in ("uniform", "zipf"):
        for tokens in TOKENS:
            ids = routing(kind, E, k, tokens, tokens + (kind == "zipf"))
            x = (torch.randn(tokens, H, device="cuda") * 0.5).to(torch.bfloat16)
            w = torch.rand(tokens, k, device="cuda").to(torch.bfloat16)
            # check: pair (0, 0)'s first projection is matvec_fp8's rows of its expert
            e = int(ids[0, 0])
            h = plan.experts_matvec_fp8(0, ids, x, scales[0], (B, B), scratch=scratch)
            flat = scales[0].repeat_interleave(B, dim=1).reshape(E * 2 * I, -1).contiguous()
            want = plan.matvec_fp8(0, x[:1], flat, (1, B))[0, e * 2 * I:(e + 1) * 2 * I]
            assert torch.equal(h[0, 0].view(torch.int16), want.view(torch.int16)), (name, kind, tokens)
            fns = [lambda: products(x, ids), lambda: selected(ids), lambda: selected_grouped(x, ids, w)]
            t = spread(fns, a)
            table["routings"][f"{kind} {tokens}"] = dict(zip(["experts_matvec_fp8 x2", "dequant_fp8_select", "dequant_fp8_select+grouped_mm"], t),
                                                         experts=len(set(ids.reshape(-1).tolist())))
    ids = routing("uniform", E, k, 1, 99)
    x = (torch.randn(1, H, device="cuda") * 0.5).to(torch.bfloat16)
    y = products(x, ids)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = products(x, ids)
    ids.copy_(routing("uniform", E, k, 1, 100))
    g.replay()
    assert torch.equal(y.view(torch.int16), products(x, ids).view(torch.int16))
    table["graph_1_token"] = dict(zip(["replay", "eager"], spread([g.replay, lambda: products(x, ids)], a)))
    plan.check()
    del plan, outs, scratch, sel_scratch
    print(json.dumps({name: table}), file=sys.stderr, flush=True)
    table["module"] = module_table(name, cfg, ws, a)
    return table


def module_table(name, cfg, ws, a):
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    conf, mod = experts_module(cfg, ws)
    conf2, mod2 = experts_module(cfg, ws)
    dense = copy.copy(mod)
    dense._parameters = dict(mod._parameters)
    for p in ("gate_up_proj", "down_proj"):
        dense._parameters[p] = torch.nn.Parameter(R.dequantize_fp8(getattr(mod, p), getattr(mod, p + "_scale_inv"), (B, B), torch.bfloat16),
                                                  requires_grad=False)
    with_mv = compress_module(torch.nn.ModuleDict({"experts": mod}), fp8=True, experts=True, experts_matvec=EXPERTS_MATVEC_MAX_TOKENS)
    compress_module(torch.nn.ModuleDict({"experts": mod2}), fp8=True, experts=True)
    assert with_mv["experts_matvec_modules"] == 1, with_mv
    table = {"report": with_mv}
    for impl in ("eager", "grouped_mm"):
        conf._experts_implementation = conf2._experts_implementation = impl
        for tokens in TOKENS:
            x = (torch.randn(tokens, H, device="cuda") * 0.5).to(torch.bfloat16)
            ids = routing("uniform", E, k, tokens, 7 + tokens)
            w = torch.rand(tokens, k, device="cuda").to(torch.bfloat16)
            fns = [lambda: mod(x, ids, w), lambda: mod2(x, ids, w), lambda: R._experts_impl(dense)(dense, x, ids, w)]
            got, want = fns[0]().double(), fns[2]().double()
            assert torch.isfinite(got).all() and (got - want).abs().max() <= 0.02 * want.abs().max(), (name, impl, tokens)
            t = spread(fns, a)
            table[f"{impl} {tokens}"] = dict(zip(["experts_matvec", "fp8_experts", "dense_bf16"], t))
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
