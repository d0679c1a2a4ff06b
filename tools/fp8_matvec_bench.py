#!/usr/bin/env python3
"""x (S . W)^T straight from compressed fp8 weights (DecodePlan.matvec_fp8) on llama3-8b's matrix shapes.

Weights: bf16 Gaussian weights (std 0.02, seeded) quantized to float8_e4m3fn per 128x128 block at amax / 448, the
layout of DeepSeek-V3's and the Qwen3 -FP8 checkpoints.  In one process, alternating and timed with CUDA events after
warm-up, medians, every output checked against fp64 before it is timed, per matrix shape (4096x4096, 1024x4096,
14336x4096, 4096x14336) and for one layer's seven matrices in a row, at 1, 2, 4 and 8 bf16 tokens:
  * `matvec_fp8`: the product from the compressed fp8 streams;
  * `plan.run()` + dequantize + F.linear: decode the fp8 weight, scale it to bf16 per block, multiply;
  * a dense resident fp8 weight + dequantize + F.linear: no compression;
  * the bf16 `matvec` on the same shape (bf16 weights, compressed), for reference;
and the fp8 stream ratio (stream bytes / fp8 bytes) and GB/s of stream of `matvec_fp8`.  Prints one JSON line, with the
card name and its power limit.

usage: python tools/fp8_matvec_bench.py [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.plan_bench import FFN, H, KV, power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN  # noqa: E402

SHAPES = {"q/o 4096x4096": (H, H), "k/v 1024x4096": (KV, H), "gate/up 14336x4096": (FFN, H), "down 4096x14336": (H, FFN)}
LAYER = ["q/o 4096x4096", "k/v 1024x4096", "k/v 1024x4096", "q/o 4096x4096", "gate/up 14336x4096", "gate/up 14336x4096", "down 4096x14336"]
TOKENS = (1, 2, 4, 8)
B = 128


def quantize(w):
    """bf16 [out, in] (multiples of 128) -> (e4m3fn weight, fp32 scale grid [out / 128, in / 128])."""
    o, i = w.shape
    blocks = w.float().view(o // B, B, i // B, B)
    scale = (blocks.abs().amax(dim=(1, 3)) / 448.0).clamp_min(2.0 ** -30)
    q = (blocks / scale[:, None, :, None]).view(o, i).to(torch.float8_e4m3fn)
    return q, scale.contiguous()


def dequantize(q, scale):
    o, i = q.shape
    return (q.float().view(o // B, B, i // B, B) * scale[:, None, :, None]).view(o, i).to(torch.bfloat16)


def close(y, x, q, scale):
    """Within the fp32 accumulation bound and a bf16 rounding of the fp64 product of the dequantized weight."""
    wd = q.double().view(q.shape[0] // B, B, q.shape[1] // B, B) * scale.double()[:, None, :, None]
    wd = wd.view(q.shape)
    ref, mag = x.double() @ wd.T, x.double().abs() @ wd.abs().T
    return bool(torch.all((y.double() - ref).abs() <= (x.shape[-1] + 2) * 2.0 ** -24 * mag + ref.abs() * 2.0 ** -8 + 1e-30))


def close_bf16(y, x, q, scale, tol=2.0 ** -6):
    """F.linear on the bf16-rounded dequantized weight: a looser check (the weight itself is rounded to bf16)."""
    wd = dequantize(q, scale).double()
    ref, mag = x.double() @ wd.T, x.double().abs() @ wd.abs().T
    return bool(torch.all((y.double() - ref).abs() <= tol * mag + 1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit(), "weights": "e4m3fn, 128x128 blocks, amax / 448"}
    mats = {}
    for name, (o, i) in SHAPES.items():
        w = (torch.randn(o, i, device="cuda") * 0.02).to(torch.bfloat16)
        q, scale = quantize(w)
        plan8 = DecodePlan([ZipNN(input_format="torch").compress(q)])
        plan16 = DecodePlan([ZipNN(input_format="torch").compress(w)])
        assert plan8.matvec_fp8_ok(0, i) and plan16.matvec_ok(0, i), name
        s8 = torch.empty(plan8.matvec_fp8_scratch_bytes(0, i), dtype=torch.uint8, device="cuda")
        s16 = torch.empty(plan16.matvec_scratch_bytes(0, i), dtype=torch.uint8, device="cuda")
        mats[name] = dict(w=w, q=q, scale=scale, plan8=plan8, plan16=plan16, s8=s8, s16=s16)
    table = {}
    for t in TOKENS:
        row = {}
        xs = {n: torch.randn(t, mats[n]["w"].shape[1], device="cuda").to(torch.bfloat16) for n in SHAPES}

        def fns(names):
            m = [mats[n] for n in names]
            x = [xs[n] for n in names]
            return [
                lambda: [d["plan8"].matvec_fp8(0, xx, d["scale"], (B, B), scratch=d["s8"]) for d, xx in zip(m, x)],
                lambda: [F.linear(xx, dequantize(d["plan8"].run()[0], d["scale"])) for d, xx in zip(m, x)],
                lambda: [F.linear(xx, dequantize(d["q"], d["scale"])) for d, xx in zip(m, x)],
                lambda: [d["plan16"].matvec(0, xx, scratch=d["s16"]) for d, xx in zip(m, x)],
            ]
        for name in SHAPES:
            d, x = mats[name], xs[name]
            mv8, dec, dense, mv16 = (f()[0] for f in fns([name]))
            assert close(mv8, x, d["q"], d["scale"]), (name, t, "matvec_fp8")
            assert close_bf16(dec, x, d["q"], d["scale"]) and torch.equal(dec, dense), (name, t, "decode + dequantize")
            ms = timed(fns([name]), a.iters, a.warmup)
            sb = d["plan8"].nbytes["streams"]
            row[name] = {"matvec_fp8_ms": ms[0], "decode_dequant_linear_ms": ms[1], "dense_fp8_dequant_linear_ms": ms[2],
                         "bf16_matvec_ms": ms[3], "fp8_stream_bytes": sb, "fp8_bytes": d["plan8"].nbytes["dense"],
                         "fp8_stream_ratio": sb / d["plan8"].nbytes["dense"], "matvec_fp8_stream_GBps": sb / ms[0] / 1e6}
        ms = timed(fns(LAYER), a.iters, a.warmup)
        sb = sum(mats[n]["plan8"].nbytes["streams"] for n in LAYER)
        db = sum(mats[n]["plan8"].nbytes["dense"] for n in LAYER)
        row["layer (7 matrices)"] = {"matvec_fp8_ms": ms[0], "decode_dequant_linear_ms": ms[1], "dense_fp8_dequant_linear_ms": ms[2],
                                     "bf16_matvec_ms": ms[3], "fp8_stream_bytes": sb, "fp8_bytes": db, "fp8_stream_ratio": sb / db,
                                     "matvec_fp8_stream_GBps": sb / ms[0] / 1e6}
        table[t] = row
    for d in mats.values():
        d["plan8"].check()
        d["plan16"].check()
    res["matrices"] = table
    print(json.dumps(res))


if __name__ == "__main__":
    main()
