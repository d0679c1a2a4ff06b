#!/usr/bin/env python3
"""x W^T for 8 to 64 rows straight from compressed weights on tensor cores (DecodePlan.matmul) on llama3-8b's shapes.

Seeded Gaussian bf16 weights (std 0.02).  In one process, alternating and timed with CUDA events after warm-up,
medians, every output checked before it is timed:
  * per matrix shape (4096x4096, 1024x4096, 14336x4096, 4096x14336) and for one layer's seven matrices in a row, at
    8, 16, 32 and 64 rows: `matmul`, `plan.run()` + F.linear and dense F.linear, and at 8 rows `matvec` as well;
  * the forward of `--layers` llama3-8b layers at 16, 32 and 64 rows: dense, compressed (serial) and compressed with
    matmul=64 and matvec=8, eager and as one captured CUDA graph.
Prints one JSON line, with the card name and its power limit.

usage: python tools/matmul_bench.py [--iters 20] [--warmup 5] [--layers 4]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.matvec_bench import LAYER, SHAPES, graphed  # noqa: E402
from tools.plan_bench import H, Layer, power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402
from zipnn_b200.plan import MATMUL_MAX_TOKENS, MATVEC_MAX_TOKENS  # noqa: E402

ROWS = (8, 16, 32, 64)


def close(y, x, w):
    """Within an ulp per fp32 addition of the fp64 product, plus the bf16 rounding."""
    ref = x.double() @ w.double().T
    mag = x.double().abs() @ w.double().abs().T
    return bool(torch.all((y.double() - ref).abs() <= (x.shape[-1] + 1) * 2.0 ** -23 * mag + (ref.abs() + 1e-30) * 2.0 ** -7))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", type=int, default=4)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "max_rows": MATMUL_MAX_TOKENS}

    mats = {}
    for name, (o, i) in SHAPES.items():
        w = (torch.randn(o, i, device="cuda") * 0.02).to(torch.bfloat16)
        plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
        assert plan.matmul_ok(0, i), name
        mats[name] = (w, plan, torch.empty(plan.matmul_scratch_bytes(0, i), dtype=torch.uint8, device="cuda"))
    table = {}
    for t in ROWS:
        row = {}
        mv_too = t <= MATVEC_MAX_TOKENS
        for name, (w, plan, scratch) in mats.items():
            x = torch.randn(t, w.shape[1], device="cuda").to(torch.bfloat16)
            assert close(plan.matmul(0, x, scratch=scratch), x, w), (name, t)
            assert torch.equal(F.linear(x, plan.run()[0]), F.linear(x, w)), (name, t)
            fns = [lambda: plan.matmul(0, x, scratch=scratch), lambda: F.linear(x, plan.run()[0]), lambda: F.linear(x, w)]
            if mv_too:
                assert close(plan.matvec(0, x, scratch=scratch), x, w), (name, t)
                fns.append(lambda: plan.matvec(0, x, scratch=scratch))
            ms = timed(fns, a.iters, a.warmup)
            row[name] = dict(zip(["matmul_ms", "decode_linear_ms", "dense_ms", "matvec_ms"], ms), stream_bytes=plan.nbytes["streams"])
        xs = {n: torch.randn(t, mats[n][0].shape[1], device="cuda").to(torch.bfloat16) for n in SHAPES}
        fns = [lambda: [mats[n][1].matmul(0, xs[n], scratch=mats[n][2]) for n in LAYER],
               lambda: [F.linear(xs[n], mats[n][1].run()[0]) for n in LAYER], lambda: [F.linear(xs[n], mats[n][0]) for n in LAYER]]
        if mv_too:
            fns.append(lambda: [mats[n][1].matvec(0, xs[n], scratch=mats[n][2]) for n in LAYER])
        ms = timed(fns, a.iters, a.warmup)
        row["layer (7 matrices)"] = dict(zip(["matmul_ms", "decode_linear_ms", "dense_ms", "matvec_ms"], ms),
                                         stream_bytes=sum(mats[n][1].nbytes["streams"] for n in LAYER))
        table[t] = row
    for _, plan, _ in mats.values():
        plan.check()
    res["matrices"] = table
    del mats

    torch.manual_seed(1)
    dense = torch.nn.Sequential(*[Layer() for _ in range(a.layers)])
    with torch.no_grad():
        for p in dense.parameters():
            p.normal_(0, 0.02) if p.dim() > 1 else p.fill_(1.0)
    dense = dense.to(device="cuda", dtype=torch.bfloat16).eval()
    serial, fused = copy.deepcopy(dense), copy.deepcopy(dense)
    compress_module(serial)
    rep = compress_module(fused, matvec=MATVEC_MAX_TOKENS, matmul=MATMUL_MAX_TOKENS)
    res["report"] = {k: rep[k] for k in ("matmul_modules", "matmul_scratch_bytes", "matvec_modules", "scratch_bytes", "out_bytes",
                                         "stream_bytes", "dense_bytes")}
    fwd = {}
    with torch.inference_mode():
        for t in (16, 32, MATMUL_MAX_TOKENS):
            x = torch.randn(1, t, H, device="cuda").to(torch.bfloat16)
            want = dense(x)
            assert torch.equal(serial(x), want)
            err = float((fused(x).double() - want.double()).abs().max() / want.double().abs().max())
            assert err < 0.05, err
            eager = [lambda: dense(x), lambda: serial(x), lambda: fused(x)]
            graphs = [graphed(f) for f in eager]
            ms = timed(eager + graphs, a.iters, a.warmup)
            fwd[t] = dict(zip(["dense", "compressed", "matmul", "dense_graph", "compressed_graph", "matmul_graph"], ms), matmul_max_rel_err=err)
    res["forward_ms"] = fwd
    print(json.dumps(res))


if __name__ == "__main__":
    main()
