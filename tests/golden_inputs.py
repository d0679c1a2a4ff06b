"""Deterministic input generators shared by make_golden.py and the tests.

Inputs are regenerated from a seed rather than committed; each manifest record
carries the input sha256 so a test can tell "generator drifted" (skip) from
"codec wrong" (fail).
"""
import json
import os

import numpy as np
import torch

REF_CHECKS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_checks.json")

_TORCH_DT = {
    "bfloat16": torch.bfloat16, "float16": torch.float16, "float32": torch.float32,
    "float8_e4m3fn": torch.float8_e4m3fn, "float8_e5m2": torch.float8_e5m2, "uint8": torch.uint8,
}


def torch_dtype(name: str):
    return _TORCH_DT[name]


def make_input(spec: dict):
    """-> torch tensor for float dtypes, bytes for dtype == 'uint8'."""
    gen, n = spec["gen"], spec["n"]
    rng = np.random.default_rng(spec.get("seed", 1234))
    dt = _TORCH_DT[spec["dtype"]]
    if gen == "randn":
        x = rng.standard_normal(n, dtype=np.float32) * np.float32(spec["sigma"])
        t = torch.from_numpy(x).to(dt)
    elif gen == "rand_pm1":
        x = (rng.random(n, dtype=np.float32) * np.float32(2) - np.float32(1))
        t = torch.from_numpy(x).to(dt)
    elif gen == "randn_bf16_as_fp32":
        x = rng.standard_normal(n, dtype=np.float32) * np.float32(spec["sigma"])
        t = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32)
    elif gen == "zeros_ones":
        t = torch.cat([torch.zeros(n // 2, dtype=dt), torch.ones(n - n // 2, dtype=dt)])
    elif gen == "choice":
        p = np.asarray(spec["p"], dtype=np.float64)
        return rng.choice(len(p), n, p=p / p.sum()).astype(np.uint8).tobytes()
    elif gen == "bytes":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    elif gen == "half_zero":
        b = rng.integers(0, 256, n, dtype=np.uint8)
        b[rng.random(n) >= spec["frac"]] = 0
        return b.tobytes()
    else:
        raise ValueError(gen)
    if "shape" in spec:
        t = t.reshape(spec["shape"])
    return t


def raw_bytes(data) -> bytes:
    if isinstance(data, (bytes, bytearray)):
        return bytes(data)
    if data.numel() == 0:
        return b""
    return data.contiguous().reshape(-1).view(torch.uint8).numpy().tobytes()


def load_ref_checks() -> dict:
    """What the compiled reference returned on the seeded cases of test_oracle.py and
    test_stream_windows.py (written by make_golden_ref_checks.py)."""
    with open(REF_CHECKS) as f:
        return json.load(f)
