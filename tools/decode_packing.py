#!/usr/bin/env python3
"""Warps per CTA of the fused decoder (k_huf_decode_fused): occupancy and kernel time of the packed launch
(ZIPNN_B200_GRID_MODE=2: one CTA of W warps per SM that claim chunk groups; the default for bf16 and fp32) against
one one-warp CTA per chunk group (ZIPNN_B200_GRID_MODE=1; the default for fp16 and fp8).

usage: python tools/decode_packing.py [--size-gib 16] [--reps 6] [--variant NAME=LIB ...] [--no-sweep]

Prints the card and its power limit, then JSON lines:
  * "occupancy": per <G, PB> variant and launch mode, the warps per CTA and the resident warps per SM;
  * "time": k_huf_decode_fused at size-gib bf16 (K = size / 256 KiB chunks), one-warp CTAs against the packed
    launch at its default W and at W = 8 .. 16 (ZIPNN_B200_WARPS_PER_SM), the configurations alternating;
  * "time_dtype": one-warp CTAs against the packed launch at W = 10 / 12 / 16 for fp16, fp32 and fp8, same size;
  * "sweep": the same two launches from 2048 to 65536 chunks (the round staircase).
A --variant (another build of the same sources, e.g. compiled with -DZB_FUSED_MAX_WARPS=17) runs its own
configurations in a process of its own, alternating with the default build's process.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KNOBS = ("ZIPNN_B200_GRID_MODE", "ZIPNN_B200_WARPS_PER_SM", "ZIPNN_B200_DEBUG", "ZIPNN_B200_SYNC_MAX")
ONE_WARP = {"ZIPNN_B200_GRID_MODE": "1"}
PACKED = {"ZIPNN_B200_GRID_MODE": "2"}
MAIN_CONFIGS = [ONE_WARP, PACKED] + [{**PACKED, "ZIPNN_B200_WARPS_PER_SM": str(w)} for w in (8, 10, 11, 12, 13, 14, 16)]
DTYPE_CONFIGS = [ONE_WARP] + [{**PACKED, "ZIPNN_B200_WARPS_PER_SM": str(w)} for w in (10, 12, 16)]
VARIANT_CONFIGS = [ONE_WARP, {**PACKED, "ZIPNN_B200_WARPS_PER_SM": "16"}, {**PACKED, "ZIPNN_B200_WARPS_PER_SM": "17"}]
# (dtype name, G, bits_mode, bytes_mode) -> the fused variant <G, PB> it runs
VARIANTS = [("bf16", 2, 1, 10, "<2,5>"), ("fp16", 2, 0, 10, "<2,0>"), ("fp32", 4, 1, 220, "<4,5>"), ("fp32_bits0", 4, 0, 220, "<4,0>"),
            ("fp8", 1, 0, 10, "<1,0>")]


def set_env(cfg):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ["ZIPNN_B200_SYNC_MAX"] = "0"  # the fused family at every size
    os.environ.update(cfg)


class Stderr:
    """Collects what the library writes to fd 2 (its debug lines)."""

    def __enter__(self):
        sys.stderr.flush()
        self.f = tempfile.TemporaryFile(mode="w+")
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *a):
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read()
        self.f.close()


def occupancy(lib_name):
    import ctypes as C
    import torch
    from zipnn_b200 import _native
    L = _native.lib()
    st = torch.cuda.current_stream().cuda_stream
    for name, G, bits, bm, var in VARIANTS:
        chunk, K = 4096, 64
        n = chunk * K
        x = (torch.randn(n // 4, device="cuda") * 0.02).view(torch.uint8) if G == 4 else \
            (torch.randn(n // 2, device="cuda") * 0.02).to(torch.bfloat16 if bits else torch.float16).view(torch.uint8) if G == 2 else \
            (torch.randn(n, device="cuda") * 0.5).to(torch.float8_e4m3fn).view(torch.uint8)
        bound = _native.compress_bound(n, G, chunk, 32)
        s = torch.zeros(bound, dtype=torch.uint8, device="cuda")
        ws = torch.empty(_native.compress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
        ln = C.c_size_t(0)
        hdr = (C.c_char * 32).from_buffer_copy(bytes(32))
        assert L.zipnn_b200_compress(x.data_ptr(), n, hdr, 32, G, bits, bm, chunk, 0.95, s.data_ptr(), bound, C.byref(ln), ws.data_ptr(), ws.numel(), st) == 0
        out = torch.empty(n, dtype=torch.uint8, device="cuda")
        dws = torch.empty(_native.decompress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
        for mode, cfg in (("one_warp_ctas", ONE_WARP), ("packed", {**PACKED, "ZIPNN_B200_WARPS_PER_SM": "64"})):
            set_env({**cfg, "ZIPNN_B200_DEBUG": "1"})
            with Stderr() as e:
                rc = L.zipnn_b200_decompress(s[32:].data_ptr(), ln.value - 32, G, bits, bm, chunk, n, out.data_ptr(), dws.data_ptr(), dws.numel(), st, 1)
            line = [ln_ for ln_ in e.text.splitlines() if "fused launch" in ln_][-1]
            kv = dict(t.split("=") for t in line.split()[3:])
            print(json.dumps({"occupancy": var, "lib": lib_name, "dtype": name, "mode": mode, "warps_per_cta": int(kv["warps_per_cta"]),
                              "resident_warps_per_sm": int(kv["resident_warps_per_sm"]), "exact": rc == 0 and torch.equal(out, x)}), flush=True)
    set_env({})


def fused_ms(z, s, reps=3):
    from zipnn_b200 import _native
    _native.timing_enable(True)
    for _ in range(reps):
        d = z.decompress(s)
        del d
    kt = _native.timing_collect()
    _native.timing_enable(False)
    ms, cnt = kt["k_huf_decode_fused"]
    return ms / max(cnt, 1)


def arm(lib_name, configs, size_gib, reps, sweep):
    import torch
    from bench import make_tensor
    from zipnn_b200 import ZipNN
    occupancy(lib_name)
    t = make_tensor(int(size_gib * (1 << 30)), torch.bfloat16, "cuda", 1234)
    z = ZipNN(input_format="torch")
    s = z.compress(t)
    for cfg in configs:  # warm-up and exactness of every configuration
        set_env(cfg)
        d = z.decompress(s)
        assert torch.equal(d.view(torch.uint8), t.view(torch.uint8)), cfg
        del d
    for r in range(reps):
        for cfg in configs:
            set_env(cfg)
            print(json.dumps({"time": cfg, "lib": lib_name, "rep": r, "fused_ms": round(fused_ms(z, s), 4)}), flush=True)
    del s
    if lib_name == "default":
        del t
        for dt in (torch.float16, torch.float32, torch.float8_e4m3fn):  # the other variants at the same size
            t = make_tensor(int(size_gib * (1 << 30)), dt, "cuda", 1234)
            s = z.compress(t)
            for r in range(reps):
                for cfg in DTYPE_CONFIGS:
                    set_env(cfg)
                    if r == 0:
                        d = z.decompress(s)
                        assert torch.equal(d.view(torch.uint8), t.view(torch.uint8)), (dt, cfg)
                        del d
                    print(json.dumps({"time_dtype": str(dt), "config": cfg, "rep": r, "fused_ms": round(fused_ms(z, s), 4)}), flush=True)
            del s, t
        t = make_tensor(int(size_gib * (1 << 30)), torch.bfloat16, "cuda", 1234)
    if sweep:
        chunk = 1 << 18
        K_all = t.numel() * 2 // chunk
        for K in [k for k in (2048, 3072, 4096, 6144, 8192, 12288, 16384, 16896, 17000, 20480, 24576, 32768, 33792, 34000, 49152, 50688, 51000, 65536)
                  if k <= K_all]:
            part = t[: K * chunk // 2]
            s = z.compress(part)
            row = {"sweep": K, "lib": lib_name}
            for name, cfg in (("one_warp_ctas", ONE_WARP), ("packed", PACKED)):
                set_env(cfg)
                d = z.decompress(s)
                assert torch.equal(d.view(torch.uint8), part.view(torch.uint8)), (K, name)
                del d
                row[name + "_ms"] = round(min(fused_ms(z, s, 2) for _ in range(3)), 4)
            set_env({**PACKED, "ZIPNN_B200_DEBUG": "1"})
            with Stderr() as e:
                d = z.decompress(s)
                torch.cuda.synchronize()
            del d
            line = [ln_ for ln_ in e.text.splitlines() if "fused launch" in ln_][-1]
            row["packed_launch"] = line.split("mode=2 ")[-1]
            print(json.dumps(row), flush=True)
            del s
    set_env({})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gib", type=float, default=16.0)
    ap.add_argument("--reps", type=int, default=6, help="timed runs per configuration and build")
    ap.add_argument("--variant", action="append", default=[], metavar="NAME=LIB")
    ap.add_argument("--arm", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--no-sweep", action="store_true")
    a = ap.parse_args()
    if a.arm is not None:  # one process per build
        name, reps, sweep = a.arm.split(":")
        arm(name, MAIN_CONFIGS if name == "default" else VARIANT_CONFIGS, a.size_gib, int(reps), sweep == "1")
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"}), flush=True)
    builds = [("default", None)] + [tuple(v.split("=", 1)) for v in a.variant]
    halves = [a.reps - a.reps // 2, a.reps // 2]
    for i, n in enumerate(halves):  # the builds alternate: two processes each
        for name, lib in builds:
            env = dict(os.environ)
            env.pop("ZIPNN_B200_LIB_VARIANT", None)
            if lib:
                env["ZIPNN_B200_LIB_VARIANT"] = os.path.abspath(lib)
            sweep = "1" if (i == 0 and name == "default" and not a.no_sweep) else "0"
            subprocess.run([sys.executable, os.path.abspath(__file__), "--size-gib", str(a.size_gib), "--arm", f"{name}:{n}:{sweep}"],
                           env=env, check=True)


if __name__ == "__main__":
    main()
