#!/usr/bin/env python3
"""fp8 linear layers from compressed weights on llama3-8b's matrix shapes: DecodePlan.dequant_fp8 and the resident
fp8 module mode (compress_module(fp8=True, matvec=8)).

Weights: bf16 Gaussian weights (std 0.02, seeded) quantized to float8_e4m3fn per 128x128 block at amax / 448, the
layout of DeepSeek-V3's and the Qwen3 -FP8 checkpoints.  In one process, alternating and timed with CUDA events after
warm-up, every output checked against the torch reference before it is timed; each point is the median of --iters
calls, repeated --repeats times (the spread is the range of those medians):
  * per matrix shape (4096x4096, 1024x4096, 14336x4096, 4096x14336) and one layer's seven matrices in a row:
    `dequant_fp8` into a bf16 buffer, against `plan.run()` + torch's dequantize (fp32 cast, scale grid, multiply, bf16
    cast) and against `plan.run()` alone; GB/s of `dequant_fp8` counts the stream bytes read and the bf16 bytes
    written, and its share of the H100 SXM data-sheet 3.35 TB/s;
  * one layer of seven transformers FP8Linear modules resident with fp8=True, matvec=8, forward at 1, 8, 16, 64, 512
    and 2048 rows, against dense bf16 F.linear and against a dense fp8 weight + torch's dequantize + F.linear.
Prints one JSON line with the card name and its power limit.

usage: python tools/fp8_linear_bench.py [--iters 20] [--warmup 5] [--repeats 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.fp8_matvec_bench import LAYER, SHAPES, close, dequantize, quantize  # noqa: E402
from tools.plan_bench import power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data sheet
ROWS = (1, 8, 16, 64, 512, 2048)
B = 128


def spread(fns, a):
    """-> per callable {"ms": median of the repeats' medians, "range": [min, max]}."""
    reps = [timed(fns, a.iters, a.warmup) for _ in range(a.repeats)]
    out = []
    for k in range(len(fns)):
        v = sorted(r[k] for r in reps)
        out.append({"ms": v[len(v) // 2], "range": [v[0], v[-1]]})
    return out


def dequant_table(mats, a):
    table = {}
    for name in list(SHAPES) + ["layer (7 matrices)"]:
        names = LAYER if name.startswith("layer") else [name]
        m = [mats[n] for n in names]
        fns = [lambda: [d["plan"].dequant_fp8(0, d["q"].shape[1], d["scale"], (B, B), out=d["out"]) for d in m],
               lambda: [dequantize(d["plan"].run()[0], d["scale"]) for d in m],
               lambda: [d["plan"].run() for d in m]]
        for d in m:
            got = d["plan"].dequant_fp8(0, d["q"].shape[1], d["scale"], (B, B), out=d["out"])
            assert torch.equal(got.view(torch.int16), dequantize(d["q"], d["scale"]).view(torch.int16)), name
        t = spread(fns, a)
        sb = sum(d["plan"].nbytes["streams"] for d in m)
        ob = sum(d["out"].numel() * 2 for d in m)
        gbps = (sb + ob) / t[0]["ms"] / 1e6
        table[name] = {"dequant_fp8": t[0], "run_torch_dequant": t[1], "run": t[2], "stream_bytes": sb, "bf16_bytes": ob,
                       "dequant_fp8_GBps": gbps, "dequant_fp8_share_of_3.35TBps": gbps * 1e9 / HBM_BPS}
    return table


def layer_table(mats, a):
    from transformers.integrations.finegrained_fp8 import FP8Linear
    layer = torch.nn.ModuleList()
    for n in LAYER:
        o, i = SHAPES[n]
        lin = FP8Linear(i, o, block_size=(B, B)).cuda()
        lin.weight = torch.nn.Parameter(mats[n]["q"].clone(), requires_grad=False)
        lin.weight_scale_inv = torch.nn.Parameter(mats[n]["scale"].clone(), requires_grad=False)
        layer.append(lin)
    report = compress_module(layer, fp8=True, matvec=8)
    assert report["fp8_modules"] == 7, report
    table = {"report": report}
    for rows in ROWS:
        xs = [torch.randn(rows, SHAPES[n][1], device="cuda").to(torch.bfloat16) for n in LAYER]
        fns = [lambda: [lin(x) for lin, x in zip(layer, xs)],
               lambda: [F.linear(x, mats[n]["w"]) for n, x in zip(LAYER, xs)],
               lambda: [F.linear(x, dequantize(mats[n]["q"], mats[n]["scale"])) for n, x in zip(LAYER, xs)]]
        got, _, ref = (f() for f in fns)
        for n, x, y, r in zip(LAYER, xs, got, ref):
            if rows > 8:
                assert torch.equal(y.view(torch.int16), r.view(torch.int16)), (n, rows)
            else:
                assert close(y, x, mats[n]["q"], mats[n]["scale"]), (n, rows)
        t = spread(fns, a)
        table[rows] = {"resident_fp8": t[0], "dense_bf16_linear": t[1], "dense_fp8_dequant_linear": t[2]}
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "weights": "e4m3fn, 128x128 blocks, amax / 448",
           "iters": a.iters, "repeats": a.repeats}
    mats = {}
    with torch.no_grad():
        for name, (o, i) in SHAPES.items():
            w = (torch.randn(o, i, device="cuda") * 0.02).to(torch.bfloat16)
            q, scale = quantize(w)
            plan = DecodePlan([ZipNN(input_format="torch").compress(q)])
            assert plan.matvec_fp8_ok(0, i), name
            mats[name] = dict(w=w, q=q, scale=scale, plan=plan, out=torch.empty(o, i, dtype=torch.bfloat16, device="cuda"))
        res["dequant"] = dequant_table(mats, a)
        for d in mats.values():
            d["plan"].check()
        res["layer_forward"] = layer_table(mats, a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
