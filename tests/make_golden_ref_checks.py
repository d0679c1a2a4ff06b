#!/usr/bin/env python3
"""Write tests/golden/ref_checks.json: what the compiled reference (oracle/_ref, `make -C oracle ref`)
returns on the seeded cases of test_oracle.py and test_stream_windows.py, so that those tests compare
the port with the reference without needing the reference's sources or binary.

  huf_blocks  HUF_compress on each block of test_oracle.block_inputs(): return code, sha256 of the output
  streams     zipnn_core on each case of test_oracle.stream_inputs(): length and sha256 of the stream
              (checked here to decode back to the input with the reference's combine_dtype)
  windows     zipnn_core on the chunk windows of test_stream_windows.window_input()
  settings    zipnn_core on each case of chunk_settings.settings_inputs(): every chunk size from G to 2^12 and
              2^19-2^21, thresholds 0-1.5, planes at the threshold and capacity edges (checked to decode back)

usage:  python tests/make_golden_ref_checks.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    sys.path.insert(0, p)

from chunk_settings import header as settings_header, settings_inputs  # noqa: E402
from golden_inputs import REF_CHECKS  # noqa: E402
from oracle import oracle as O  # noqa: E402
from test_oracle import block_inputs, stream_inputs  # noqa: E402
from test_stream_windows import _hdr, window_input  # noqa: E402


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def main():
    ref = O.ref_core()
    if ref is None or O.ref_cdll() is None:
        sys.exit(f"the compiled reference is missing: build it first ({O.ref_path()})")
    blocks = []
    for src, cap in block_inputs():
        r, out = O.ref_huf_compress(src, cap)
        blocks.append({"input_sha256": sha(src), "ret": int(r), "out_sha256": sha(out)})
    streams = []
    for h, data, G, bits, bm, chunk in stream_inputs():
        r = bytes(ref.zipnn_core(bytes(h), bytearray(data.tobytes()), G, bits, bm, 0, chunk, 0.95, 10, 4))
        assert bytes(ref.combine_dtype(r[32:], G, bits, bm, chunk, data.size, 2)) == data.tobytes()
        streams.append({"input_sha256": sha(data), "stream_len": len(r), "stream_sha256": sha(r)})
    windows = []
    data, chunk, G, K, wins = window_input()
    for c0, c1 in wins:
        part = data[c0 * chunk: c1 * chunk]
        r = bytes(ref.zipnn_core(bytes(_hdr()), bytearray(part.tobytes()), G, 1, 10, 0, chunk, 0.95, 10, 4))
        windows.append({"c0": c0, "c1": c1, "input_sha256": sha(part), "stream_len": len(r), "stream_sha256": sha(r)})
    settings = []
    h = settings_header()
    for c in settings_inputs():
        G, bits, chunk, data = c["G"], c["bits"], c["chunk"], c["data"]
        bm = 220 if G == 4 else 10
        r = bytes(ref.zipnn_core(h, bytearray(data.tobytes()), G, bits, bm, 0, chunk, c["thr"], 10, 4))
        assert bytes(ref.combine_dtype(r[32:], G, bits, bm, chunk, data.size, 2)) == data.tobytes(), c["name"]
        settings.append({"name": c["name"], "input_sha256": sha(data), "stream_len": len(r), "stream_sha256": sha(r)})
    with open(REF_CHECKS, "w") as f:
        json.dump({"reference": "zipnn/zipnn v0.5.3 (0e9beed), C extension built -O3",
                   "huf_blocks": blocks, "streams": streams, "windows": windows, "settings": settings}, f, indent=0)
        f.write("\n")
    print(f"wrote {len(blocks)} blocks, {len(streams)} streams, {len(windows)} windows, {len(settings)} settings to {REF_CHECKS}")


if __name__ == "__main__":
    main()
