#!/usr/bin/env python3
"""GPU time of the bench step that no kernel of ours accounts for.

usage: python tools/step_gaps.py [--size-gib 16] [--steps 10] [--warmup 3] [--out DIR (default: a temporary directory)]
                                [--mode both|events|trace]

The step is bench.py's: a bf16 tensor of size-gib GiB (randn * 0.02, seed 1234), compressed and decompressed through
ZipNN(input_format="torch"), with CUDA events between the two directions.

  events  profiler off, the library's kernel timing on as in bench.py.  Per direction: the path time between the
          events, the sum of the kernel times of the direction, and the difference (the gap), averaged over the steps.
  trace   torch.profiler with CPU and CUDA activities over one step after the warm-up, in a process of its own; the
          trace goes to DIR/step_gaps.pt.trace.json.  Every interval longer than 5 us inside the step in which the GPU
          runs none of its work, with the host call whose launch ended it and the host calls made during it, and the
          host duration of every runtime and driver call of the step.

Prints the card's name and power limit first, then one JSON line per mode.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GIB = 1 << 30
GPU_CATS = ("kernel", "gpu_memcpy", "gpu_memset")
HOST_CATS = ("cuda_runtime", "cuda_driver")
ENCODE_PREFIX = ("k_encode_",)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gib", type=float, default=16.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "step_gaps"))
    ap.add_argument("--mode", default="both", choices=["both", "events", "trace"])
    ap.add_argument("--min-gap-us", type=float, default=5.0)
    return ap.parse_args()


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(q[0])
        info["sm_clock_max_mhz"] = float(q[1])
    except Exception as exc:  # no nvidia-smi: say so rather than guess
        info["power_limit_w"] = f"unavailable ({str(exc)[:80]})"
    return info


def setup(args):
    import torch
    from bench import make_tensor
    from zipnn_b200 import ZipNN
    torch.cuda.set_device(0)
    t = make_tensor(int(args.size_gib * GIB), torch.bfloat16, torch.device("cuda", 0), 1234)

    def step():
        s = ZipNN(input_format="torch").compress(t)
        d = ZipNN(input_format="torch").decompress(s)
        return s, d
    s = d = None
    for _ in range(max(args.warmup, 1)):
        del s, d
        s, d = step()
    assert torch.equal(d.view(torch.uint8), t.view(torch.uint8)), "round trip is not exact"
    del s, d
    return t


def run_events(args):
    import torch
    from zipnn_b200 import ZipNN, _native
    t = setup(args)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.steps + 1)]
    _native.timing_enable(True)
    torch.cuda.synchronize()
    ev[0].record()
    for i in range(args.steps):
        s = ZipNN(input_format="torch").compress(t)
        ev[2 * i + 1].record()
        d = ZipNN(input_format="torch").decompress(s)
        ev[2 * i + 2].record()
        if i + 1 < args.steps:
            del s, d
    torch.cuda.synchronize()
    del s, d
    kt = _native.timing_collect()
    _native.timing_enable(False)
    K = args.steps
    tc = sum(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(K)) / K
    td = sum(ev[2 * i + 1].elapsed_time(ev[2 * i + 2]) for i in range(K)) / K
    kc = sum(ms for k, (ms, _) in kt.items() if k.startswith(ENCODE_PREFIX)) / K
    kd = sum(ms for k, (ms, _) in kt.items() if not k.startswith(ENCODE_PREFIX)) / K
    per_kernel = {k: {"ms_per_step": round(ms / K, 4), "launches_per_step": c / K} for k, (ms, c) in kt.items() if c}
    return {"mode": "events", "size_gib": args.size_gib, "steps": K,
            "compress": {"path_ms": round(tc, 4), "kernels_ms": round(kc, 4), "gap_ms": round(tc - kc, 4)},
            "decompress": {"path_ms": round(td, 4), "kernels_ms": round(kd, 4), "gap_ms": round(td - kd, 4)},
            "step_gap_ms": round(tc - kc + td - kd, 4), "step_ms": round(tc + td, 4), "kernels": per_kernel}


def idle_intervals(busy, lo, hi):
    """Gaps of [lo, hi) not covered by the (start, end) intervals in `busy`."""
    out, at = [], lo
    for a, b in sorted(busy):
        if b <= at:
            continue
        if a > at:
            out.append((at, min(a, hi)))
        at = max(at, b)
        if at >= hi:
            break
    if at < hi:
        out.append((at, hi))
    return [(a, b) for a, b in out if b > a]


def analyse_trace(path, min_gap_us):
    """Gaps and host calls of the step between the 'step' annotation's start and end (host clock, microseconds)."""
    with open(path) as f:
        evs = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X"]
    ann = [e for e in evs if e.get("name") == "step" and e.get("cat") == "user_annotation"]
    if not ann:
        raise RuntimeError("no 'step' annotation in the trace")
    lo, hi = ann[0]["ts"], ann[0]["ts"] + ann[0]["dur"]
    dirs = sorted((e["ts"], e["ts"] + e["dur"], e["name"]) for e in evs
                  if e.get("cat") == "user_annotation" and e.get("name") in ("compress", "decompress") and lo <= e["ts"] < hi)
    gpu = sorted((e for e in evs if e.get("cat") in GPU_CATS and e["ts"] + e["dur"] > lo and e["ts"] < hi), key=lambda e: e["ts"])
    host = sorted((e for e in evs if e.get("cat") in HOST_CATS and lo <= e["ts"] < hi), key=lambda e: e["ts"])
    by_corr = {e["args"].get("correlation"): e for e in host if "correlation" in e.get("args", {})}

    def direction(ts):
        for a, b, name in dirs:
            if a <= ts < b:
                return name
        return "between"
    # A direction starts when the host enters it: the GPU is idle from there until its first operation.  Idle time
    # is cut at the direction boundaries, as the bench's events cut it.
    bounds = sorted({lo, hi, *(a for a, _, _ in dirs), *(b for _, b, _ in dirs)})
    busy = [(e["ts"], e["ts"] + e["dur"]) for e in gpu]
    gaps = []
    for a, b in [iv for w0, w1 in zip(bounds, bounds[1:]) for iv in idle_intervals(busy, w0, w1)]:
        if b - a < min_gap_us:
            continue
        nxt = next((e for e in gpu if e["ts"] >= b - 0.5), None)
        prev = [e for e in gpu if e["ts"] + e["dur"] <= a + 0.5]
        launcher = by_corr.get(nxt["args"].get("correlation")) if nxt else None
        during = [e for e in host if e["ts"] < b and e["ts"] + e["dur"] > a]
        gaps.append({"start_us": round(a - lo, 1), "idle_us": round(b - a, 1), "direction": direction(a),
                     "after_gpu_op": prev[-1]["name"][:60] if prev else None,
                     "before_gpu_op": nxt["name"][:60] if nxt else None,
                     "ended_by_host_call": launcher["name"] if launcher else None,
                     "host_calls_during": [f'{e["name"]} {e["dur"]:.1f}us' for e in during][:12]})
    calls = [{"at_us": round(e["ts"] - lo, 1), "call": e["name"], "host_us": round(e["dur"], 1), "direction": direction(e["ts"])}
             for e in host]
    totals = {}
    for c in calls:
        k = (c["direction"], c["call"])
        n, us = totals.get(k, (0, 0.0))
        totals[k] = (n + 1, us + c["host_us"])
    return {"step_host_us": round(hi - lo, 1),
            "gpu_busy_us": round(sum(e["dur"] for e in gpu), 1),
            "idle_us_total": round(sum(g["idle_us"] for g in gaps), 1),
            "idle_us_by_direction": {d: round(sum(g["idle_us"] for g in gaps if g["direction"] == d), 1)
                                     for d in ("compress", "decompress", "between")},
            "gaps": gaps,
            "host_calls": calls,
            "host_call_totals": [{"direction": d, "call": c, "count": n, "host_us": round(us, 1)}
                                 for (d, c), (n, us) in sorted(totals.items(), key=lambda kv: -kv[1][1])]}


def run_trace(args):
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    from zipnn_b200 import ZipNN
    t = setup(args)
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "step_gaps.pt.trace.json")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(2):   # the first profiled step warms the profiler; the second is analysed
            torch.cuda.synchronize()
            with record_function("step" if i else "warm"):
                with record_function("compress"):
                    s = ZipNN(input_format="torch").compress(t)
                with record_function("decompress"):
                    d = ZipNN(input_format="torch").decompress(s)
            torch.cuda.synchronize()
            del s, d
    prof.export_chrome_trace(path)
    res = analyse_trace(path, args.min_gap_us)
    return {"mode": "trace", "size_gib": args.size_gib, "trace": os.path.relpath(path, ROOT), **res}


def report(args, res):
    """The whole result to DIR/step_gaps_<mode>.json; on stdout without the per-call list."""
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"step_gaps_{res['mode']}.json"), "w") as f:
        json.dump({"card": card(), **res}, f, indent=1)
    short = {k: v for k, v in res.items() if k not in ("host_calls", "kernels")}
    if "gaps" in short:
        short["gaps"] = sorted(short["gaps"], key=lambda g: -g["idle_us"])[:16]
        short["host_call_totals"] = short["host_call_totals"][:16]
    print(json.dumps(short), flush=True)


def main():
    args = parse()
    import torch
    assert torch.cuda.is_available(), "step_gaps measures on a GPU"
    if args.mode != "trace":
        print(json.dumps({"card": card()}), flush=True)
    if args.mode in ("both", "events"):
        report(args, run_events(args))
    if args.mode == "both":
        torch.cuda.empty_cache()
        cmd = [sys.executable, os.path.abspath(__file__), "--mode", "trace", "--size-gib", str(args.size_gib),
               "--warmup", str(args.warmup), "--out", args.out, "--min-gap-us", str(args.min_gap_us)]
        subprocess.check_call(cmd)
    elif args.mode == "trace":
        report(args, run_trace(args))


if __name__ == "__main__":
    main()
