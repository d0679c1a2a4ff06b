#!/usr/bin/env python3
"""Prefetch for compressed-resident modules on llama3-8b layer shapes (the layer stack of tools/plan_bench.py).

Seeded Gaussian bf16 weights (std 0.02).  In one process, alternating and timed with CUDA events after warm-up:
  * the stack's forward at 1, 16 and 2048 tokens: dense, compressed serial (compress_module), and compressed with
    prefetch (compress_module(prefetch=True)) for a sweep of CTA budgets of the side-stream decode and for the side
    stream at default and at high priority; every output is checked against the dense one with torch.equal;
  * one layer's 7-matrix plan: run() against run_into(max_ctas=0), as enqueue time on the host and as device time,
    and run_into alternating between two output buffers.
Prints one JSON line, with the card name and its power limit.

usage: python tools/prefetch_bench.py [--layers 4] [--iters 20] [--warmup 5] [--ctas 16,33,66,132,0]
"""
import argparse
import copy
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tools.model_bench import llama_like  # noqa: E402
from tools.plan_bench import FFN, H, KV, Layer, power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402
from zipnn_b200.resident import _ATTR  # noqa: E402


def host_us(fn, n=200):
    """Median enqueue time of fn on the host, in microseconds (no synchronisation inside the window)."""
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e6)
    torch.cuda.synchronize()
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctas", default="16,33,66,132,0")
    ap.add_argument("--tokens", default="1,16,2048")
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit()}

    # ---- one layer's 7 matrices: run() against run_into()
    shapes = [s for n, s in llama_like(1, H, FFN, 128256, KV).items() if n.startswith("model.layers.0.") and len(s) == 2]
    ws = [(torch.randn(s, device="cuda") * 0.02).to(torch.bfloat16) for s in shapes]
    plan = DecodePlan(ZipNN(input_format="torch").compress_batch(ws))
    bufs = [torch.empty(plan.nbytes["out"], dtype=torch.uint8, device="cuda") for _ in range(2)]
    flip = [0]

    def into_two():
        flip[0] ^= 1
        plan.run_into(bufs[flip[0]])

    t_run, t_into, t_two = timed([plan.run, lambda: plan.run_into(bufs[0]), into_two], a.iters, a.warmup)
    for b in bufs:
        b.zero_()
        assert all(torch.equal(o, w) for o, w in zip(plan.run_into(b), ws))
    assert all(torch.equal(o, w) for o, w in zip(plan.run(), ws))
    plan.check()
    res["layer"] = {"run_ms": round(t_run, 4), "run_into_ms": round(t_into, 4), "run_into_two_buffers_ms": round(t_two, 4),
                    "run_call_us": round(host_us(plan.run), 1), "run_into_call_us": round(host_us(lambda: plan.run_into(bufs[0])), 1)}
    del ws, plan, bufs

    # ---- the stack: dense, serial, prefetch over budgets and priorities
    stack = torch.nn.Sequential(*[Layer() for _ in range(a.layers)])
    with torch.no_grad():
        for p in stack.parameters():
            p.normal_(0, 0.02) if p.dim() > 1 else p.fill_(1.0)
    stack = stack.to("cuda", torch.bfloat16).eval()
    serial, pre = copy.deepcopy(stack), copy.deepcopy(stack)
    compress_module(serial)
    rep = compress_module(pre, prefetch=True)
    ops = getattr(pre, _ATTR).prefetch[0].ops
    sides = {"default": ops.side, "high": torch.cuda.Stream(priority=torch.cuda.Stream.priority_range()[1])}
    ctas = [int(c) for c in a.ctas.split(",")]
    res["stack"] = {"layers": a.layers, "prefetch_out_bytes": rep["prefetch_out_bytes"], "forward_ms": {}}

    def prefetch_with(c, side):
        def f(x):
            ops.max_ctas, ops.side = c, side
            return pre(x)
        return f

    variants = {"dense": stack, "serial": serial}
    for prio, side in sides.items():
        for c in ctas:
            variants[f"prefetch_{prio}_{c or 'full'}"] = prefetch_with(c, side)
    with torch.inference_mode():
        for t in [int(x) for x in a.tokens.split(",")]:
            x = torch.randn(1, t, H, device="cuda", dtype=torch.bfloat16)
            want = stack(x)
            for name, f in variants.items():
                for _ in range(3):   # the first forward learns the order
                    assert torch.equal(f(x), want), (name, t)
            names = list(variants)
            ms = timed([lambda f=variants[n]: f(x) for n in names], a.iters, a.warmup)
            for name, f in variants.items():
                assert torch.equal(f(x), want), (name, t)
            res["stack"]["forward_ms"][f"{t}tok"] = {n: round(v, 3) for n, v in zip(names, ms)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
