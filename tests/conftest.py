import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_manifest():
    with open(os.path.join(HERE, "golden", "manifest.json")) as f:
        return json.load(f)["cases"]


@pytest.fixture(scope="session")
def golden_cases():
    return load_manifest()


def golden_stream(rec):
    fn = rec.get("stream_file")
    if not fn:
        return None
    with open(os.path.join(HERE, "golden", fn), "rb") as f:
        return f.read()


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the oracle and the host-emulation shim are compiled (seconds, no GPU)."""
    import subprocess
    from oracle import oracle as O
    O.build(ref=True)
    emu = os.path.join(HERE, "host_emu")
    so = os.path.join(emu, "libemu_serial.so")
    src = os.path.join(emu, "emu_serial.cpp")
    hdr = os.path.join(ROOT, "zipnn_b200", "csrc", "huf_serial.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    yield
