#!/usr/bin/env python3
"""The tensor-core fp8 matmul from compressed weights (DecodePlan.matmul_fp8) on llama3-8b's matrix shapes, and the
resident fp8 module mode with fp8_matmul=N.

Weights: bf16 Gaussian weights (std 0.02, seeded) quantized to float8_e4m3fn per 128x128 block at amax / 448, as in
tools/fp8_linear_bench.py.  In one process, alternating and timed with CUDA events after warm-up, every output checked
before it is timed; each point is the median of --iters calls, repeated --repeats times (the spread is the range of
those medians):
  * per matrix shape (4096x4096, 1024x4096, 14336x4096, 4096x14336) and one layer's seven matrices in a row, at 8, 16,
    32 and 64 rows: `matmul_fp8`, `dequant_fp8` + F.linear (what the resident layer does above `matvec` rows without
    fp8_matmul), `matvec_fp8` (8 rows only) and dense bf16 F.linear;
  * one layer of seven transformers FP8Linear modules resident with fp8=True, matvec=8, fp8_matmul=64 against the same
    layer with fp8=True, matvec=8, at the same rows.
Prints one JSON line with the card name and its power limit.

usage: python tools/fp8_matmul_bench.py [--iters 20] [--warmup 5] [--repeats 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.fp8_linear_bench import spread  # noqa: E402
from tools.fp8_matvec_bench import LAYER, SHAPES, close, dequantize, quantize  # noqa: E402
from tools.plan_bench import power_limit  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402

ROWS = (8, 16, 32, 64)
B = 128


def close_d(y, x, d):
    """y within the fp32-sum bound of fp64 x D^T, D the dequantized weight (bf16), rounded once to bf16."""
    x64, d64 = x.double(), d.double()
    ref, mag = x64 @ d64.T, x64.abs() @ d64.abs().T
    bound = (x.shape[-1] + 2) * 2.0 ** -23 * mag
    return bool(torch.all((y.double() - ref).abs() <= bound + (ref.abs() + bound) * 2.0 ** -8))


def product_table(mats, a):
    table = {}
    for name in list(SHAPES) + ["layer (7 matrices)"]:
        names = LAYER if name.startswith("layer") else [name]
        m = [mats[n] for n in names]
        table[name] = {}
        for rows in ROWS:
            xs = [torch.randn(rows, d["q"].shape[1], device="cuda").to(torch.bfloat16) for d in m]
            fns = [lambda: [d["plan"].matmul_fp8(0, x, d["scale"], (B, B), scratch=d["mm"]) for d, x in zip(m, xs)],
                   lambda: [F.linear(x, d["plan"].dequant_fp8(0, d["q"].shape[1], d["scale"], (B, B), out=d["out"])) for d, x in zip(m, xs)],
                   lambda: [F.linear(x, d["w"]) for d, x in zip(m, xs)]]
            keys = ["matmul_fp8", "dequant_fp8_linear", "dense_bf16_linear"]
            if rows <= 8:
                fns.append(lambda: [d["plan"].matvec_fp8(0, x, d["scale"], (B, B), scratch=d["mv"]) for d, x in zip(m, xs)])
                keys.append("matvec_fp8")
            for d, x in zip(m, xs):
                dq = dequantize(d["q"], d["scale"])
                assert close_d(d["plan"].matmul_fp8(0, x, d["scale"], (B, B), scratch=d["mm"]), x, dq), (name, rows)
                got = F.linear(x, d["plan"].dequant_fp8(0, d["q"].shape[1], d["scale"], (B, B), out=d["out"]))
                assert torch.equal(got.view(torch.int16), F.linear(x, dq).view(torch.int16)), (name, rows)
                if rows <= 8:
                    assert close(d["plan"].matvec_fp8(0, x, d["scale"], (B, B), scratch=d["mv"]), x, d["q"], d["scale"]), (name, rows)
            table[name][rows] = dict(zip(keys, spread(fns, a)))
    return table


def layer_table(mats, a):
    from transformers.integrations.finegrained_fp8 import FP8Linear

    def layer():
        mods = torch.nn.ModuleList()
        for n in LAYER:
            o, i = SHAPES[n]
            lin = FP8Linear(i, o, block_size=(B, B)).cuda()
            lin.weight = torch.nn.Parameter(mats[n]["q"].clone(), requires_grad=False)
            lin.weight_scale_inv = torch.nn.Parameter(mats[n]["scale"].clone(), requires_grad=False)
            mods.append(lin)
        return mods
    with_mm, without = layer(), layer()
    table = {"report": compress_module(with_mm, fp8=True, matvec=8, fp8_matmul=64)}
    assert table["report"]["fp8_matmul_modules"] == 7, table["report"]
    compress_module(without, fp8=True, matvec=8)
    for rows in ROWS:
        xs = [torch.randn(rows, SHAPES[n][1], device="cuda").to(torch.bfloat16) for n in LAYER]
        fns = [lambda: [lin(x) for lin, x in zip(with_mm, xs)], lambda: [lin(x) for lin, x in zip(without, xs)]]
        got, base = (f() for f in fns)
        for n, x, y, z in zip(LAYER, xs, got, base):
            if rows <= 8:
                assert torch.equal(y.view(torch.int16), z.view(torch.int16)), (n, rows)
            else:
                assert close_d(y, x, dequantize(mats[n]["q"], mats[n]["scale"])), (n, rows)
        t = spread(fns, a)
        table[rows] = {"resident_fp8_matmul_64": t[0], "resident_fp8": t[1]}
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
            assert plan.matmul_fp8_ok(0, i), name
            mats[name] = dict(w=w, q=q, scale=scale, plan=plan, out=torch.empty(o, i, dtype=torch.bfloat16, device="cuda"),
                              mm=torch.empty(plan.matmul_fp8_scratch_bytes(0, i, 64), dtype=torch.uint8, device="cuda"),
                              mv=torch.empty(plan.matvec_fp8_scratch_bytes(0, i, 8), dtype=torch.uint8, device="cuda"))
        res["products"] = product_table(mats, a)
        for d in mats.values():
            d["plan"].check()
        res["layer_forward"] = layer_table(mats, a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
