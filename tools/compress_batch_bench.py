#!/usr/bin/env python3
"""Batched against per-tensor compression of GPU-resident checkpoints, one JSON line per measurement.

Workloads (randn * 0.02 values in the real tensor shapes, as tools/model_bench.py):
  llama3-8b  32 layers, 291 bf16 tensors (~16 GB)
  gpt2       148 fp32 tensors
  synthetic  4096 tensors of 4-256 KiB, bf16 and fp32 mixed
For each: a `ZipNN.compress` loop against one `ZipNN.compress_batch`, alternating, reporting wall time (host clock
around work that ends in a synchronise), summed kernel time (the library's CUDA-event timing), kernel launches
(counted), host synchronisations (not counted: taken from the code, one per `compress` call and one per
`compress_batch` call) and whether the streams are identical.  `--large K,...` times a bf16 tensor of K chunks in a
batch of small tensors through the batch kernels and routed to the single-tensor launches; `--save DIR` times
`save_file` of llama3-8b from GPU tensors by phase, `--compress-file DIR` `compress_safetensors_file` by phase.

usage: python tools/compress_batch_bench.py [--reps 3] [--large 1024,4096,65536] [--save DIR] [--compress-file DIR]
       [--workloads llama3-8b,gpt2,synthetic]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from model_bench import MODELS  # noqa: E402
from zipnn_b200 import ZipNN, _native  # noqa: E402


def gpu_info():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:  # pragma: no cover
        return f"unknown ({exc})"


def workload(name, dev):
    g = torch.Generator(device=dev).manual_seed(1234)
    if name == "synthetic":
        sizes = torch.randint(4 * 1024, 256 * 1024 + 1, (4096,), generator=torch.Generator().manual_seed(7))
        out = []
        for i, nb in enumerate(sizes.tolist()):
            dt = torch.bfloat16 if i % 2 == 0 else torch.float32
            out.append((torch.randn(nb // dt.itemsize, generator=g, device=dev) * 0.02).to(dt))
        return out
    shapes, dtype = MODELS[name](0)
    return [(torch.randn(*s, generator=g, device=dev) * 0.02).to(dtype) for s in shapes.values()]


def timed(fn, per_kernel=None):
    _native.timing_enable(True)
    torch.cuda.synchronize()
    l0 = _native.launch_count()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    launches = _native.launch_count() - l0
    k = _native.timing_collect()
    _native.timing_enable(False)
    if per_kernel is not None:
        for name, (ms, cnt) in k.items():
            if cnt:
                per_kernel.setdefault(name, []).append(round(ms, 3))
    return res, wall, sum(ms for ms, _ in k.values()), launches


def compare(name, tensors, reps):
    nbytes = sum(t.numel() * t.element_size() for t in tensors)
    loop = lambda: [ZipNN(input_format="torch").compress(t) for t in tensors]  # noqa: E731
    batch = lambda: ZipNN(input_format="torch").compress_batch(tensors)  # noqa: E731
    ref = loop()
    got = batch()
    same = len(ref) == len(got) and all(torch.equal(a, b) for a, b in zip(ref, got))
    del ref, got
    rows = {"loop": [], "batch": []}
    order = (("loop", loop), ("batch", batch))
    for r in range(reps):
        for mode, fn in (order if r % 2 == 0 else order[::-1]):
            res, wall, kms, launches = timed(fn)
            del res
            rows[mode].append((wall, kms, launches))
    for mode, syncs in (("loop", len(tensors)), ("batch", 1)):   # from the code: compress() syncs once, compress_batch() once
        walls = [r[0] for r in rows[mode]]
        print(json.dumps(dict(workload=name, mode=mode, tensors=len(tensors), bytes=nbytes, identical=same,
                              wall_s=[round(w, 4) for w in walls], wall_median_s=round(statistics.median(walls), 4),
                              gbs=round(nbytes / statistics.median(walls) / 1e9, 2),
                              kernel_ms_median=round(statistics.median(r[1] for r in rows[mode]), 3),
                              launches=rows[mode][0][2], host_syncs_by_construction=syncs)), flush=True)


def large(dev, reps, chunk_counts):
    """Where to route: one bf16 tensor of K chunks (256 KiB) in a batch with 64 norm-sized tensors (8 KiB bf16), coded
    by the batch kernels (the routing limit lifted) and routed to the single-tensor launches (the limit just under K);
    `single` is the large tensor alone through zipnn_b200_compress.  ABBA order: the card's clock drifts over a run."""
    big = max(chunk_counts) * 262144
    base = (torch.randn(big // 8, device=dev) * 0.02).to(torch.bfloat16)
    full = base.repeat(4)
    del base
    g = torch.Generator(device=dev).manual_seed(5)
    small = [(torch.randn(4096, generator=g, device=dev) * 0.02).to(torch.bfloat16) for _ in range(64)]
    modes = ("single", "unrouted", "routed")

    def run(mode, t, K):
        if mode == "single":
            return [ZipNN(input_format="torch").compress(t)]
        os.environ["ZIPNN_B200_ENC_BATCH_MAX_CHUNKS"] = str(1 << 40) if mode == "unrouted" else str(K - 1)
        try:
            return ZipNN(input_format="torch").compress_batch([t] + small)
        finally:
            os.environ.pop("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", None)

    for K in chunk_counts:
        t = full[: K * 262144 // 2]
        ref = run("single", t, K)[0]
        outs = [run(m, t, K) for m in modes[1:]]
        same = all(torch.equal(ref, o[0]) for o in outs) and all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
        del ref, outs
        rows = {m: [] for m in modes}
        kernels = {m: {} for m in modes}
        for r in range(reps):
            for mode in (modes if r % 2 == 0 else modes[::-1]):
                res, wall, kms, launches = timed(lambda: run(mode, t, K), kernels[mode])
                del res
                rows[mode].append((wall, kms, launches))
        for mode in modes:
            print(json.dumps(dict(workload=f"one bf16 tensor of {K} chunks ({K * 262144 / 2**30:g} GiB)" +
                                  ("" if mode == "single" else " + 64 tensors of 8 KiB"), mode=mode, identical=same,
                                  wall_s=[round(r[0], 5) for r in rows[mode]], wall_median_ms=round(1e3 * statistics.median(r[0] for r in rows[mode]), 3),
                                  kernel_ms=[round(r[1], 3) for r in rows[mode]],
                                  kernel_ms_median=round(statistics.median(r[1] for r in rows[mode]), 3),
                                  per_kernel_ms=kernels[mode], launches=rows[mode][0][2])), flush=True)


def compress_file(dev, d, reps):
    """compress_safetensors_file of llama3-8b (32 layers) from a plain file in `d`, by phase: pread into pinned
    memory, H2D, kernels, D2H (device phases by CUDA events), and the rest (safetensors' writer, the index)."""
    from safetensors.torch import save_file as st_save
    from zipnn_b200 import compress_safetensors_file
    from zipnn_b200 import safetensors_io as SIO
    shapes, dtype = MODELS["llama3-8b"](0)
    g = torch.Generator(device=dev).manual_seed(1234)
    src = os.path.join(d, "llama3-8b-phases.safetensors")
    st_save({k: (torch.randn(*s, generator=g, device=dev) * 0.02).to(dtype).cpu() for k, s in shapes.items()}, src, {"format": "pt"})
    orig = SIO._compress_entries
    try:
        for rep in range(reps):
            timings = {}
            SIO._compress_entries = lambda entries, device, _t=None: orig(entries, device, timings)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            path, clen, olen = compress_safetensors_file(src)
            total = time.perf_counter() - t0
            print(json.dumps(dict(workload="compress_safetensors_file llama3-8b", rep=rep, bytes=olen, compressed=clen,
                                  total_s=round(total, 3), phases_s={k: round(v, 3) for k, v in timings.items()},
                                  rest_s=round(total - sum(timings.values()), 3), group_bytes=SIO.SAVE_GROUP_BYTES)), flush=True)
            os.remove(path)
    finally:
        SIO._compress_entries = orig
        os.remove(src)


def save(dev, d):
    from zipnn_b200 import safetensors_io as SIO
    shapes, dtype = MODELS["llama3-8b"](0)
    g = torch.Generator(device=dev).manual_seed(1234)
    tensors = {k: (torch.randn(*s, generator=g, device=dev) * 0.02).to(dtype) for k, s in shapes.items()}
    path = os.path.join(d, "llama3-8b-save.znn.safetensors")
    for rep in range(2):
        timings = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, infos, clen, olen = SIO._compress_entries(list(tensors.items()), dev, timings)
        t1 = time.perf_counter()
        SIO._write_compressed(out, infos, None, path)
        t2 = time.perf_counter()
        del out
        print(json.dumps(dict(workload="save_file llama3-8b from GPU", rep=rep, bytes=olen, compressed=clen,
                              total_s=round(t2 - t0, 3), compress_to_host_s=round(t1 - t0, 3),
                              phases_s={k: round(v, 3) for k, v in timings.items()}, safetensors_write_s=round(t2 - t1, 3),
                              group_bytes=SIO.SAVE_GROUP_BYTES)), flush=True)
        os.remove(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="llama3-8b,gpt2,synthetic")
    ap.add_argument("--large", default="", help="comma-separated chunk counts of single bf16 tensors, e.g. 1024,4096,65536")
    ap.add_argument("--save", default="")
    ap.add_argument("--compress-file", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    for name in [w for w in args.workloads.split(",") if w]:
        tensors = workload(name, dev)
        compare(name, tensors, args.reps)
        del tensors
        torch.cuda.empty_cache()
    if args.large:
        large(dev, args.reps, [int(k) for k in args.large.split(",")])
        torch.cuda.empty_cache()
    if args.save:
        save(dev, args.save)
        torch.cuda.empty_cache()
    if args.compress_file:
        compress_file(dev, args.compress_file, args.reps)


if __name__ == "__main__":
    main()
