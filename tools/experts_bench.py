#!/usr/bin/env python3
"""Decode only the routed experts of a compressed mixture-of-experts layer (DecodePlan.run_select, experts=True).

Seeded Gaussian bf16 weights (std 0.02) at two layer shapes: Qwen3-30B-A3B (128 experts, top-8, gate_up_proj
[128, 1536, 2048], down_proj [128, 2048, 768]) and Mixtral-8x7B (8 experts, top-2, [8, 28672, 4096], [8, 4096, 14336]).
In one process, alternating and timed with CUDA events after warm-up, medians, every output checked before it is
timed:
  * plan level: `run()` against `run_select(ids)` for the top-k routings of 1, 4, 16, 64 and 256 tokens, uniform and
    Zipf-skewed (expert e drawn with weight 1 / (e + 1)), with the distinct experts, the chunks decoded and the GB/s of
    decoded bytes; `run_select` of every expert against `run()` (the cost of the index and the compaction); the same
    calls captured as CUDA graphs at 1 token;
  * module level: a MoE block forward (router + experts module with the eager expert loop of transformers'
    MixtralExperts) at 1, 16 and 64 tokens three ways: dense, compressed with whole decode, compressed with
    experts=True.
Prints markdown tables and one JSON line, with the card name and its power limit.

usage: python tools/experts_bench.py [--iters 20] [--warmup 5] [--layers qwen3,mixtral]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.matvec_bench import graphed  # noqa: E402
from tools.plan_bench import power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module, decompress_module  # noqa: E402

LAYERS = {"qwen3": dict(E=128, k=8, H=2048, I=768), "mixtral": dict(E=8, k=2, H=4096, I=14336)}
TOKENS = (1, 4, 16, 64, 256)
MODULE_TOKENS = (1, 16, 64)


def routing(n, E, k, how, gen):
    """Top-k expert ids [n, k] (distinct per token), uniform or Zipf-skewed."""
    w = torch.ones(E) if how == "uniform" else 1.0 / torch.arange(1, E + 1, dtype=torch.float32)
    return torch.multinomial(w.expand(n, E), k, replacement=False, generator=gen).cuda()


def touched(orig, chunk, E, ids):
    S = orig // E
    m = np.zeros(-(-orig // chunk), dtype=bool)
    for e in np.unique(ids):
        m[e * S // chunk: (e * S + S - 1) // chunk + 1] = True
    return int(m.sum()), int(sum(min(chunk, orig - c * chunk) for c in np.flatnonzero(m)))


class Experts(torch.nn.Module):
    def __init__(self, E, H, I):
        super().__init__()
        self.num_experts = E
        self.gate_up_proj = torch.nn.Parameter(torch.empty(E, 2 * I, H, dtype=torch.bfloat16, device="cuda").normal_(0, 0.02))
        self.down_proj = torch.nn.Parameter(torch.empty(E, H, I, dtype=torch.bfloat16, device="cuda").normal_(0, 0.02))

    def forward(self, hidden_states, top_k_index, top_k_weights):   # transformers' MixtralExperts loop
        out = torch.zeros_like(hidden_states)
        mask = F.one_hot(top_k_index, num_classes=self.num_experts).permute(2, 1, 0)
        for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero():
            e = e[0]
            pos, tok = torch.where(mask[e])
            gate, up = F.linear(hidden_states[tok], self.gate_up_proj[e]).chunk(2, dim=-1)
            h = F.linear(F.silu(gate) * up, self.down_proj[e]) * top_k_weights[tok, pos, None]
            out.index_add_(0, tok, h.to(out.dtype))
        return out


class MoE(torch.nn.Module):
    def __init__(self, E, k, H, I):
        super().__init__()
        self.k = k
        self.gate = torch.nn.Linear(H, E, bias=False, device="cuda", dtype=torch.bfloat16)
        self.experts = Experts(E, H, I)

    def forward(self, x):
        w, idx = torch.topk(torch.softmax(self.gate(x).float(), -1), self.k, dim=-1)
        return self.experts(x, idx, w.to(x.dtype))


def plan_level(name, cfg, iters, warmup, gen):
    E, k, H, I = cfg["E"], cfg["k"], cfg["H"], cfg["I"]
    ws = [torch.empty(E, 2 * I, H, dtype=torch.bfloat16, device="cuda").normal_(0, 0.02),
          torch.empty(E, H, I, dtype=torch.bfloat16, device="cuda").normal_(0, 0.02)]
    plan = DecodePlan([ZipNN(input_format="torch").compress(w) for w in ws])
    assert plan.select_ok()
    chunk = 262144
    dense = [w.view(torch.uint8).reshape(E, -1) for w in ws]
    outs = plan.run()
    assert all(torch.equal(o.view(torch.uint8).reshape(E, -1), d) for o, d in zip(outs, dense))
    rows = []

    def check(ids):
        plan._out.fill_(0xFF)
        outs = plan.run_select(ids)
        sel = ids.reshape(-1).unique()
        assert all(torch.equal(o.view(torch.uint8).reshape(E, -1)[sel], d[sel]) for o, d in zip(outs, dense)), name

    all_ids = torch.arange(E, device="cuda")
    check(all_ids)
    t_run, t_all = timed([plan.run, lambda: plan.run_select(all_ids)], iters, warmup)
    dense_bytes = sum(w.numel() * 2 for w in ws)
    total_chunks = sum(-(-w.numel() * 2 // chunk) for w in ws)
    for how in ("uniform", "zipf"):
        for n in TOKENS:
            ids = routing(n, E, k, how, gen)
            check(ids)
            t_r, t_s = timed([plan.run, lambda: plan.run_select(ids)], iters, warmup)
            host = ids.cpu().numpy()
            ch = [touched(w.numel() * 2, chunk, E, host) for w in ws]
            nbytes = sum(b for _, b in ch)
            rows.append(dict(routing=how, tokens=n, experts=int(np.unique(host).size), chunks=sum(c for c, _ in ch),
                             run_ms=t_r, select_ms=t_s, select_gbps=nbytes / t_s / 1e6, run_gbps=dense_bytes / t_r / 1e6))
    ids1 = routing(1, E, k, "uniform", gen)
    check(ids1)
    g_run, g_sel = graphed(plan.run), graphed(lambda: plan.run_select(ids1))
    t_grun, t_gsel = timed([g_run, g_sel], iters, warmup)
    plan.check()
    res = dict(layer=name, dense_bytes=dense_bytes, stream_bytes=plan.nbytes["streams"], chunks=total_chunks,
               run_all_ms=t_run, select_all_ms=t_all, graph_1tok=dict(run_ms=t_grun, select_ms=t_gsel), rows=rows)
    del plan, outs, ws, dense
    torch.cuda.empty_cache()
    return res


def module_level(name, cfg, iters, warmup):
    torch.manual_seed(1)
    model = MoE(**cfg).eval()
    xs = {n: torch.randn(n, cfg["H"], device="cuda").to(torch.bfloat16) for n in MODULE_TOKENS}
    out = {}
    with torch.no_grad():
        want = {n: model(x) for n, x in xs.items()}
        for n, x in xs.items():
            out[n] = {"dense_ms": timed([lambda: model(x)], iters, warmup)[0]}
        for mode in ("whole", "experts"):
            compress_module(model, experts=mode == "experts")
            for n, x in xs.items():
                assert torch.equal(model(x), want[n]), (name, mode, n)
                out[n][mode + "_ms"] = timed([lambda: model(x)], iters, warmup)[0]
            decompress_module(model)
    del model
    torch.cuda.empty_cache()
    return {"layer": name, "rows": [dict(tokens=n, **v) for n, v in out.items()]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", default="qwen3,mixtral")
    a = ap.parse_args()
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "plan": [], "module": []}
    for name in a.layers.split(","):
        cfg = LAYERS[name]
        p = plan_level(name, cfg, a.iters, a.warmup, gen)
        res["plan"].append(p)
        print(f"\n{name}: run() {p['run_all_ms']:.3f} ms, run_select(all {cfg['E']}) {p['select_all_ms']:.3f} ms, "
              f"graph at 1 token: run {p['graph_1tok']['run_ms']:.3f} ms, select {p['graph_1tok']['select_ms']:.3f} ms")
        print("| routing | tokens | experts | chunks | run ms | select ms | select/run | select GB/s |")
        print("|---|---|---|---|---|---|---|---|")
        for r in p["rows"]:
            print(f"| {r['routing']} | {r['tokens']} | {r['experts']} | {r['chunks']}/{p['chunks']} | {r['run_ms']:.3f} | "
                  f"{r['select_ms']:.3f} | {r['select_ms'] / r['run_ms']:.2f} | {r['select_gbps']:.0f} |")
        m = module_level(name, cfg, a.iters, a.warmup)
        res["module"].append(m)
        print("| tokens | dense ms | whole decode ms | experts=True ms |")
        print("|---|---|---|---|")
        for r in m["rows"]:
            print(f"| {r['tokens']} | {r['dense_ms']:.3f} | {r['whole_ms']:.3f} | {r['experts_ms']:.3f} |")
    print(json.dumps(res))
    out = os.environ.get("EXPERTS_BENCH_OUT")
    if out:
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
