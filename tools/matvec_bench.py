#!/usr/bin/env python3
"""x W^T straight from compressed weights (DecodePlan.matvec) on llama3-8b's matrix shapes.

Seeded Gaussian bf16 weights (std 0.02).  In one process, alternating and timed with CUDA events after warm-up,
medians, every output checked before it is timed:
  * per matrix shape (4096x4096, 1024x4096, 14336x4096, 4096x14336) and for one layer's seven matrices in a row, at
    1, 2, 4 and 8 tokens: `matvec`, `plan.run()` + F.linear, and dense F.linear; the stream bytes a call reads and the
    GB/s of stream bytes of the matvec;
  * the forward of `--layers` llama3-8b layers at 1 and at the maximum token count: dense, compressed (serial) and
    compressed with matvec=N, eager and as one captured CUDA graph.
Prints one JSON line, with the card name and its power limit.

usage: python tools/matvec_bench.py [--iters 20] [--warmup 5] [--layers 4]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.plan_bench import FFN, H, KV, Layer, power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402
from zipnn_b200.plan import MATVEC_MAX_TOKENS  # noqa: E402

SHAPES = {"q/o 4096x4096": (H, H), "k/v 1024x4096": (KV, H), "gate/up 14336x4096": (FFN, H), "down 4096x14336": (H, FFN)}
LAYER = ["q/o 4096x4096", "k/v 1024x4096", "k/v 1024x4096", "q/o 4096x4096", "gate/up 14336x4096", "gate/up 14336x4096", "down 4096x14336"]
TOKENS = (1, 2, 4, 8)


def close(y, x, w):
    ref = x.double() @ w.double().T
    mag = x.double().abs() @ w.double().abs().T
    return bool(torch.all((y.double() - ref).abs() <= (x.shape[-1] + 1) * 2.0 ** -24 * mag + (ref.abs() + 1e-30) * 2.0 ** -7))


def graphed(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", type=int, default=4)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "max_tokens": MATVEC_MAX_TOKENS}

    mats = {}
    for name, (o, i) in SHAPES.items():
        w = (torch.randn(o, i, device="cuda") * 0.02).to(torch.bfloat16)
        plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
        assert plan.matvec_ok(0, i), name
        mats[name] = (w, plan, torch.empty(plan.matvec_scratch_bytes(0, i), dtype=torch.uint8, device="cuda"))
    table = {}
    for t in TOKENS:
        row = {}
        for name, (w, plan, scratch) in mats.items():
            x = torch.randn(t, w.shape[1], device="cuda").to(torch.bfloat16)
            assert close(plan.matvec(0, x, scratch=scratch), x, w), (name, t)
            assert torch.equal(F.linear(x, plan.run()[0]), F.linear(x, w)), (name, t)
            mv, dec, dense = timed([lambda: plan.matvec(0, x, scratch=scratch), lambda: F.linear(x, plan.run()[0]), lambda: F.linear(x, w)],
                                   a.iters, a.warmup)
            row[name] = {"matvec_ms": mv, "decode_linear_ms": dec, "dense_ms": dense, "stream_bytes": plan.nbytes["streams"],
                         "dense_bytes": plan.nbytes["dense"], "matvec_stream_GBps": plan.nbytes["streams"] / mv / 1e6}
        xs = {n: torch.randn(t, mats[n][0].shape[1], device="cuda").to(torch.bfloat16) for n in SHAPES}
        fns = [lambda: [mats[n][1].matvec(0, xs[n], scratch=mats[n][2]) for n in LAYER],
               lambda: [F.linear(xs[n], mats[n][1].run()[0]) for n in LAYER], lambda: [F.linear(xs[n], mats[n][0]) for n in LAYER]]
        mv, dec, dense = timed(fns, a.iters, a.warmup)
        sb = sum(mats[n][1].nbytes["streams"] for n in LAYER)
        row["layer (7 matrices)"] = {"matvec_ms": mv, "decode_linear_ms": dec, "dense_ms": dense, "stream_bytes": sb,
                                     "dense_bytes": sum(mats[n][1].nbytes["dense"] for n in LAYER), "matvec_stream_GBps": sb / mv / 1e6}
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
    rep = compress_module(fused, matvec=MATVEC_MAX_TOKENS)
    res["report"] = {k: rep[k] for k in ("matvec_modules", "matvec_scratch_bytes", "scratch_bytes", "out_bytes", "stream_bytes", "dense_bytes")}
    fwd = {}
    with torch.inference_mode():
        for t in (1, MATVEC_MAX_TOKENS):
            x = torch.randn(1, t, H, device="cuda").to(torch.bfloat16)
            want = dense(x)
            assert torch.equal(serial(x), want)
            err = float((fused(x).double() - want.double()).abs().max() / want.double().abs().max())
            assert err < 0.05, err
            eager = [lambda: dense(x), lambda: serial(x), lambda: fused(x)]
            graphs = [graphed(f) for f in eager]
            ms = timed(eager + graphs, a.iters, a.warmup)
            fwd[t] = dict(zip(["dense", "compressed", "matvec", "dense_graph", "compressed_graph", "matvec_graph"], ms), matvec_max_rel_err=err)
    res["forward_ms"] = fwd
    print(json.dumps(res))


if __name__ == "__main__":
    main()
