#!/usr/bin/env python3
"""Embedding lookups straight from compressed weights (DecodePlan.gather) on llama3-8b's embedding shape.

A seeded Gaussian bf16 embedding (std 0.02) of 128256 x 4096 (1.05 GB, 4008 chunks of 256 KiB).  In one process,
alternating and timed with CUDA events after warm-up, medians:
  * dense F.embedding, DecodePlan.run() of the whole embedding, and DecodePlan.gather at n = 1, 8, 64, 512, 2048 and
    8192 ids, uniform and Zipf-distributed (exponent 1.1), each checked against the dense rows;
  * a resident llama-shaped model (the embedding, `--layers` llama3-8b layers, norm, untied lm_head) at 1 and 2048
    tokens: compress_module with gather off and on, serial and with prefetch; every output checked with torch.equal.
Prints one JSON line, with the card name and its power limit.

usage: python tools/gather_bench.py [--iters 20] [--warmup 5] [--layers 1] [--slots 64]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.plan_bench import FFN, H, KV, Layer, power_limit, timed  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, compress_module  # noqa: E402

VOCAB = 128256


def zipf_ids(n, seed):
    rng = np.random.default_rng(seed)
    return torch.from_numpy((rng.zipf(1.1, n) - 1) % VOCAB).cuda()


class Model(torch.nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.embed_tokens = torch.nn.Embedding(VOCAB, H)
        self.layers = torch.nn.ModuleList([Layer() for _ in range(layers)])
        self.norm = torch.nn.RMSNorm(H)
        self.lm_head = torch.nn.Linear(H, VOCAB, bias=False)

    def forward(self, ids):
        x = self.embed_tokens(ids)
        for layer in self.layers:
            x = layer(x)
        return self.lm_head(self.norm(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", type=int, default=1)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--ns", default="1,8,64,512,2048,8192")
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit()}

    w = (torch.randn(VOCAB, H, device="cuda") * 0.02).to(torch.bfloat16)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    scratch = torch.empty(plan.gather_scratch_bytes(0, a.slots), dtype=torch.uint8, device="cuda")
    res["embedding"] = {"dense_bytes": w.numel() * 2, "stream_bytes": plan.nbytes["streams"], "slots": a.slots,
                        "scratch_bytes": scratch.numel()}
    ids1 = torch.randint(0, VOCAB, (2048,), device="cuda")
    dense_ms, run_ms = timed([lambda: F.embedding(ids1, w), lambda: plan.run()], a.iters, a.warmup)
    res["dense_embedding_2048_ms"], res["plan_run_ms"] = dense_ms, run_ms
    gathers = {}
    for n in [int(x) for x in a.ns.split(",")]:
        uni = torch.randint(0, VOCAB, (n,), device="cuda")
        zipf = zipf_ids(n, n)
        outs = [torch.empty(n, H, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
        fns = [lambda: plan.gather(0, uni, out=outs[0], scratch=scratch), lambda: plan.gather(0, zipf, out=outs[1], scratch=scratch),
               lambda: F.embedding(uni, w)]
        t_uni, t_zipf, t_dense = timed(fns, a.iters, a.warmup)
        assert torch.equal(outs[0], w[uni]) and torch.equal(outs[1], w[zipf])
        touched = [len(torch.unique(ids * H * 2 // (256 * 1024))) for ids in (uni, zipf)]
        gathers[n] = {"uniform_ms": t_uni, "zipf_ms": t_zipf, "dense_ms": t_dense, "chunks_uniform": touched[0], "chunks_zipf": touched[1]}
    plan.check()
    res["gather"] = gathers
    del plan, scratch

    # ---- a resident model's forward, gather off and on, serial and with prefetch
    torch.manual_seed(1)
    dense = Model(a.layers)
    with torch.no_grad():
        for p in dense.parameters():
            p.normal_(0, 0.02) if p.dim() > 1 else p.fill_(1.0)
    dense = dense.to(device="cuda", dtype=torch.bfloat16).eval()
    models = {}
    for gather in (False, True):
        for prefetch in (False, True):
            m = copy.deepcopy(dense)
            rep = compress_module(m, prefetch=prefetch, gather=gather)
            models[f"gather={gather},prefetch={prefetch}"] = (m, rep)
    fwd = {}
    with torch.inference_mode():
        for t in (1, 2048):
            ids = torch.randint(0, VOCAB, (1, t), device="cuda")
            want = dense(ids)
            names = ["dense"] + list(models)
            fns = [lambda: dense(ids)] + [lambda m=m: m(ids) for m, _ in models.values()]
            ms = timed(fns, a.iters, a.warmup)
            for name, (m, _) in models.items():
                assert torch.equal(m(ids), want), name
            fwd[t] = dict(zip(names, ms))
    res["forward_ms"] = fwd
    res["reports"] = {k: {kk: v for kk, v in rep.items() if kk in ("out_bytes", "scratch_bytes", "gather_bytes", "prefetch_out_bytes")}
                      for k, (_, rep) in models.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
