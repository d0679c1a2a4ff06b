"""Host side of the batched encoder (no GPU): the save path's group planner, the per-item arguments that
`ZipNN.compress_batch` builds from `plan()`, and the ctypes layout of zipnn_b200_compress_item."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from zipnn_b200 import ZipNN, _native
from zipnn_b200 import zipnn as Z
from zipnn_b200.safetensors_io import _cuda_device, _plan_groups

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ group planner
@pytest.mark.parametrize("sizes,budget,want", [
    ([], 10, []),
    ([10], 10, [[0]]),                                   # exactly the budget
    ([5, 5], 10, [[0, 1]]),                              # adds up to exactly the budget
    ([5, 6], 10, [[0], [1]]),                            # one byte over
    ([4, 4, 4, 4], 10, [[0, 1], [2, 3]]),
    ([3, 11, 3], 10, [[0], [1], [2]]),                   # over the budget: a group on its own
    ([11], 10, [[0]]),
    ([11, 12], 10, [[0], [1]]),
    ([0, 0, 10, 0], 10, [[0, 1, 2, 3]]),                 # empty tensors cost nothing
    ([2, 9, 1, 1, 7, 25, 1], 10, [[0], [1, 2], [3, 4], [5], [6]]),
])
def test_plan_groups(sizes, budget, want):
    assert _plan_groups(sizes, budget) == want


def test_plan_groups_properties():
    rng = np.random.default_rng(7)
    for _ in range(300):
        sizes = [int(s) for s in rng.integers(0, 50, rng.integers(0, 40))]
        budget = int(rng.integers(1, 80))
        groups = _plan_groups(sizes, budget)
        assert [i for g in groups for i in g] == list(range(len(sizes)))   # every index once, in order
        for g in groups:
            assert len(g) == 1 or sum(sizes[i] for i in g) <= budget
        for a, b in zip(groups, groups[1:]):   # a group is cut only where the next tensor would not fit
            assert sum(sizes[i] for i in a) + sizes[b[0]] > budget


# ------------------------------------------------------------------ which device values take the batched file path
@pytest.mark.parametrize("device,want", [
    ("cuda", torch.device("cuda")), ("cuda:1", torch.device("cuda", 1)), (torch.device("cuda", 0), torch.device("cuda", 0)),
    (0, torch.device("cuda", 0)), (2, torch.device("cuda", 2)),
    (None, None), ("cpu", None), (torch.device("cpu"), None), ("meta", None), (False, None), (True, None), ("", None),
])
def test_cuda_device(device, want):
    assert _cuda_device(device) == want


# ------------------------------------------------------------------ per-item arguments
DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2)


def _tensors():
    g = torch.Generator().manual_seed(3)
    out = []
    for dt in DTYPES:
        for shape in ((0,), (1,), (3, 5), (1000, 7), (70000,)):
            out.append((torch.randn(shape, generator=g) * 0.02).to(dt))
    return out


@pytest.mark.parametrize("kw", [{}, {"compression_chunk": 4096, "compression_threshold": 0.5}, {"method": "HUFFMAN"}])
def test_items_match_single_calls(monkeypatch, kw):
    """Item i carries what ZipNN.compress(tensors[i]) hands to the native call."""
    seen = []

    def fake_host(flat_u8, header, num_buf, bits_mode, bytes_mode, chunk, threshold, out=None):
        seen.append(dict(n=flat_u8.numel(), header=header, num_buf=num_buf, bits_mode=bits_mode, bytes_mode=bytes_mode,
                         chunk=chunk, threshold=threshold))
        return memoryview(b"")

    monkeypatch.setattr(Z, "_compress_host", fake_host)
    tensors = _tensors()
    flats = [Z._torch_flat_u8(t) for t in tensors]
    z = ZipNN(input_format="torch", **kw)
    plans = [z.plan(t) for t in tensors]
    items, hdrs, offs, total = Z._batch_items(flats, plans)
    for t in tensors:
        ZipNN(input_format="torch", **kw).compress(t)
    assert len(seen) == len(items) == len(tensors)
    prev_end = 0
    for it, s, o, t in zip(items, seen, offs, tensors):
        assert it.n == s["n"] == t.numel() * t.element_size()
        assert C.string_at(it.h_hdr, it.hdr_len) == s["header"]
        assert (it.num_buf, it.bits_mode, it.bytes_mode, it.chunk) == (s["num_buf"], s["bits_mode"], s["bytes_mode"], s["chunk"])
        assert it.threshold == np.float32(s["threshold"])
        bound = C.c_size_t(0)
        assert _native.lib().zipnn_b200_compress_bound(it.n, it.num_buf, it.chunk, it.hdr_len, C.byref(bound)) == 0
        assert it.out_cap == bound.value
        assert o % 256 == 0 and o >= prev_end
        prev_end = o + it.out_cap
    assert total >= prev_end


def test_compress_batch_rejects():
    z = ZipNN(input_format="torch")
    with pytest.raises(ValueError):
        z.compress_batch([torch.zeros(4, dtype=torch.bfloat16)])            # not on a GPU
    with pytest.raises(ValueError):
        ZipNN(input_format="byte").compress_batch([])
    with pytest.raises(ValueError):
        ZipNN(input_format="torch", delta_compressed_type="byte").compress_batch([])
    assert z.compress_batch([]) == []


# ------------------------------------------------------------------ ctypes layout
def test_compress_item_offsets(tmp_path):
    src = tmp_path / "off.c"
    fields = [f for f, _ in _native.CompressItem._fields_]
    body = "".join(f'  printf("%zu ", offsetof(zipnn_b200_compress_item, {f}));\n' for f in fields)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "zipnn_b200.h"\nint main(void) {\n' + body +
                   '  printf("%zu\\n", sizeof(zipnn_b200_compress_item));\n  return 0;\n}\n')
    exe = tmp_path / "off"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [getattr(_native.CompressItem, f).offset for f in fields] + [C.sizeof(_native.CompressItem)]
    assert got == want
