#!/usr/bin/env python3
"""Time k_huf_decode_fused under the library's tuning knobs (environment variables read per call).
usage: python tools/decode_probe.py [size_gib] [dtype]   -> one JSON line per configuration"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench import make_tensor  # noqa: E402
from zipnn_b200 import ZipNN, _native  # noqa: E402

CONFIGS = [
    {},
    {"ZIPNN_B200_GRID_MODE": "1", "ZIPNN_B200_SMEM_PAD": "1024"},    # fewer resident warps per SM (shared memory is what limits them; one-warp CTAs)
    {"ZIPNN_B200_GRID_MODE": "1", "ZIPNN_B200_SMEM_PAD": "3072"},
    {"ZIPNN_B200_GRID_MODE": "1", "ZIPNN_B200_SMEM_PAD": "6144"},
    {"ZIPNN_B200_GRID_MODE": "1", "ZIPNN_B200_SMEM_PAD": "12288"},
    {"ZIPNN_B200_TMA": "0"},            # side plane through cp.async slots instead of bulk tensor tiles
    {"ZIPNN_B200_TMA": "1"},            # ... and the output rows by bulk tensor stores
    {"ZIPNN_B200_GRID_MODE": "0"},      # persistent grid of one-warp CTAs
    {"ZIPNN_B200_GRID_MODE": "1"},      # one one-warp CTA per chunk group
    {"ZIPNN_B200_GRID_MODE": "2"},      # one CTA of several warps per SM that claim groups (tools/decode_packing.py has more)
]


def main():
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 16.0
    dtype = getattr(torch, sys.argv[2]) if len(sys.argv) > 2 else torch.bfloat16
    t = make_tensor(int(gib * (1 << 30)), dtype, "cuda", 1234)
    s = ZipNN(input_format="torch").compress(t)
    keys = sorted({k for c in CONFIGS for k in c})
    for cfg in CONFIGS:
        for k in keys:
            os.environ.pop(k, None)
        os.environ.update(cfg)
        ok = None
        try:
            for _ in range(2):
                d = ZipNN(input_format="torch").decompress(s)
            ok = bool(torch.equal(d.view(torch.uint8), t.view(torch.uint8)))
            del d
        except RuntimeError as exc:      # timing experiments that decode wrongly on purpose
            ok = f"raised: {exc}"[:60]
        _native.timing_enable(True)
        for _ in range(3):
            try:
                d = ZipNN(input_format="torch").decompress(s)
                del d
            except RuntimeError:
                pass
        kt = _native.timing_collect()
        _native.timing_enable(False)
        ms, cnt = kt["k_huf_decode_fused"]
        print(json.dumps({"config": cfg, "fused_ms": round(ms / max(cnt, 1), 4), "exact": ok}), flush=True)


if __name__ == "__main__":
    main()
