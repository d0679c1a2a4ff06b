#!/usr/bin/env python3
"""Decode plans and compressed-resident modules on llama3-8b layer shapes (tools/model_bench.py:llama_like).

Seeded Gaussian bf16 weights (std 0.02).  In one process, alternating and timed with CUDA events after warm-up:
  * per layer: zipnn_b200_decompress_batch of the layer's 7 matrices against DecodePlan.run of the same streams, and
    a plan run in replay mode (segment starts from the plan's index) against one without an index
    (ZIPNN_B200_PLAN_REPLAY=0: the decode mode's rounds), as whole runs and as k_huf_decode_sync kernel time;
  * a stack of llama-like layers, dense against compress_module'd, at 1 and at 2048 tokens;
  * index bytes over stream bytes, and the HBM saved: dense - stream - plan - scratch - shared output buffer.
Prints one JSON line, with the card name and its power limit.

usage: python tools/plan_bench.py [--layers 4] [--iters 20] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.model_bench import llama_like  # noqa: E402
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module  # noqa: E402
from zipnn_b200.plan import _parse  # noqa: E402

H, FFN, KV, HEADS = 4096, 14336, 1024, 32


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def timed(fns, iters, warmup):
    """Alternate the callables; -> median ms of each."""
    for _ in range(warmup):
        for f in fns:
            f()
    times = [[] for _ in fns]
    for _ in range(iters):
        for k, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    return [sorted(t)[len(t) // 2] for t in times]


def sync_kernel_ms(fn, iters):
    """Mean time of the per-bitstream-CTA decode kernel over `iters` calls of fn (CUDA events around it)."""
    _native.timing_collect()
    _native.timing_enable(True)
    for _ in range(iters):
        fn()
    t = _native.timing_collect()
    _native.timing_enable(False)
    ms, n = t["k_huf_decode_sync"]
    return ms / max(n, 1)


def batch_decoder(streams):
    """zipnn_b200_decompress_batch of the streams into fresh outputs, unchecked (no synchronisation)."""
    parsed = _parse(streams)
    outs = [torch.empty(p.nbytes, dtype=torch.uint8, device="cuda") for p in parsed]
    arr = (_native.BatchItem * len(parsed))()
    for it, p, o in zip(arr, parsed, outs):
        it.d_body, it.body_len = p.stream.data_ptr() + p.after, p.stream.numel() - p.after
        it.num_buf, it.bits_mode, it.bytes_mode = p.num_buf, p.bits_mode, p.bytes_mode
        it.chunk, it.orig, it.d_out = p.chunk, p.nbytes, o.data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    _native.check(L.zipnn_b200_decompress_batch_workspace_size(arr, len(parsed), C.byref(wsz)))
    ws = torch.empty(wsz.value, dtype=torch.uint8, device="cuda")

    def run():
        L.zipnn_b200_decompress_batch(arr, len(parsed), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream, 0)
    return run, outs


class Layer(torch.nn.Module):
    def __init__(self):
        super().__init__()
        lin = lambda i, o: torch.nn.Linear(i, o, bias=False)  # noqa: E731
        self.input_layernorm, self.post_attention_layernorm = torch.nn.RMSNorm(H), torch.nn.RMSNorm(H)
        self.q_proj, self.k_proj, self.v_proj, self.o_proj = lin(H, H), lin(H, KV), lin(H, KV), lin(H, H)
        self.gate_proj, self.up_proj, self.down_proj = lin(H, FFN), lin(H, FFN), lin(FFN, H)

    def forward(self, x):
        b, t, _ = x.shape
        h = self.input_layernorm(x)
        q = self.q_proj(h).view(b, t, HEADS, -1).transpose(1, 2)
        k = self.k_proj(h).view(b, t, KV // 128, -1).transpose(1, 2).repeat_interleave(HEADS * 128 // KV, dim=1)
        v = self.v_proj(h).view(b, t, KV // 128, -1).transpose(1, 2).repeat_interleave(HEADS * 128 // KV, dim=1)
        y = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(b, t, H)
        x = x + self.o_proj(y)
        h = self.post_attention_layernorm(x)
        return x + self.down_proj(F.silu(self.gate_proj(h)) * self.up_proj(h))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": torch.cuda.get_device_name(), "power_limit": power_limit()}

    # ---- one layer's 7 matrices: batch decode against plan run
    shapes = [s for n, s in llama_like(1, H, FFN, 128256, KV).items() if n.startswith("model.layers.0.") and len(s) == 2]
    ws = [(torch.randn(s, device="cuda") * 0.02).to(torch.bfloat16) for s in shapes]
    streams = ZipNN(input_format="torch").compress_batch(ws)
    batch_run, batch_outs = batch_decoder(streams)
    plan = DecodePlan(streams)
    os.environ["ZIPNN_B200_PLAN_REPLAY"] = "0"
    try:
        plan_rounds = DecodePlan(streams)
    finally:
        del os.environ["ZIPNN_B200_PLAN_REPLAY"]
    batch_run()
    torch.cuda.synchronize()
    assert all(torch.equal(o.view(torch.bfloat16).view(w.shape), w) for o, w in zip(batch_outs, ws))
    assert all(torch.equal(o, w) for o, w in zip(plan.outputs, ws))
    t_batch, t_plan, t_rounds = timed([batch_run, plan.run, plan_rounds.run], a.iters, a.warmup)
    k_replay, k_decode = [], []
    for _ in range(3):   # alternating
        k_replay.append(sync_kernel_ms(plan.run, a.iters))
        k_decode.append(sync_kernel_ms(plan_rounds.run, a.iters))
    plan.check()
    plan_rounds.check()
    assert all(torch.equal(o, w) for o, w in zip(plan.outputs, ws)) and all(torch.equal(o, w) for o, w in zip(plan_rounds.outputs, ws))
    dense = sum(w.numel() * 2 for w in ws)
    sb = sum(s.numel() for s in streams)
    res["layer"] = {"dense_bytes": dense, "stream_bytes": sb, "plan_bytes": plan.nbytes["plan"], "scratch_bytes": plan.nbytes["scratch"],
                    "index_bytes": plan.nbytes["index"], "index_over_stream": plan.nbytes["index"] / sb,
                    "batch_decode_ms": round(t_batch, 4), "plan_run_ms": round(t_plan, 4), "plan_run_no_index_ms": round(t_rounds, 4),
                    "sync_kernel_replay_ms": [round(x, 4) for x in k_replay], "sync_kernel_decode_ms": [round(x, 4) for x in k_decode],
                    "plan_run_GBps": round(dense / t_plan / 1e6, 1)}
    del ws, streams, batch_outs, plan, plan_rounds, batch_run

    # ---- a stack of layers, dense against compressed
    stack = torch.nn.Sequential(*[Layer() for _ in range(a.layers)])
    with torch.no_grad():
        for p in stack.parameters():
            p.normal_(0, 0.02) if p.dim() > 1 else p.fill_(1.0)
    stack = stack.to("cuda", torch.bfloat16).eval()
    xs = {t: torch.randn(1, t, H, device="cuda", dtype=torch.bfloat16) for t in (1, 2048)}
    with torch.inference_mode():
        want = {t: stack(x) for t, x in xs.items()}
    import copy
    comp = copy.deepcopy(stack)
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    rep = compress_module(comp)
    torch.cuda.synchronize()
    m1 = torch.cuda.memory_allocated()
    res["stack"] = {"layers": a.layers, **rep, "index_over_stream": rep["index_bytes"] / rep["stream_bytes"], "allocated_drop": m0 - m1,
                    "net_saved": rep["dense_bytes"] - rep["stream_bytes"] - rep["plan_bytes"] - rep["scratch_bytes"] - rep["out_bytes"]}
    with torch.inference_mode():
        for t, x in xs.items():
            assert torch.equal(comp(x), want[t])
            td, tc = timed([lambda: stack(x), lambda: comp(x)], a.iters, a.warmup)
            res["stack"][f"forward_{t}tok_ms"] = {"dense": round(td, 3), "compressed": round(tc, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
