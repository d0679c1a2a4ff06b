#!/usr/bin/env python3
"""Write tests/golden/corrupt_verdicts.json: what the compiled reference (oracle/_ref, `make -C oracle ref`) makes
of the mutated Huffman block of every block mutant of tests/corrupt_streams.py, so that the tests compare the port
and the decoders with the reference without needing the reference's sources or binary.

  blocks  {mutant id: [HUF_decompress, HUF_decompress4X1, HUF_decompress4X2]}, each the first 16 hex digits of
          the sha256 of the decoded plane, or null when that decoder reports an error

usage:  python tests/make_golden_corrupt.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    sys.path.insert(0, p)

import corrupt_streams as CS  # noqa: E402
from oracle import oracle as O  # noqa: E402

PATH = os.path.join(HERE, "golden", "corrupt_verdicts.json")
DECODERS = ("HUF_decompress", "HUF_decompress4X1", "HUF_decompress4X2")


def digest(b):
    return None if b is None else hashlib.sha256(bytes(b)).hexdigest()[:16]


def render() -> str:
    if O.ref_cdll() is None:
        sys.exit(f"the compiled reference is missing: build it first ({O.ref_path()})")
    lines = []
    for m in CS.all_mutants():
        if m.kind != "block":
            continue
        blk, dlen = CS.block_of(m)
        got = O.ref_huf_decoders(blk, dlen)
        lines.append(f"    {json.dumps(m.id)}: {json.dumps([digest(got[d]) for d in DECODERS])}")
    return '{\n  "decoders": ' + json.dumps(list(DECODERS)) + ',\n  "blocks": {\n' + ",\n".join(lines) + "\n  }\n}\n"


def main():
    with open(PATH, "w") as f:
        f.write(render())
    print(f"wrote {PATH}")


if __name__ == "__main__":
    main()
