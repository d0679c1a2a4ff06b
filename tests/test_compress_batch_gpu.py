"""zipnn_b200_compress_batch and what is built on it: ZipNN.compress_batch, save_file and the GPU path of
compress_safetensors_file.

Every stream of a batch must be byte for byte what zipnn_b200_compress writes for that item alone (and the
oracle's stream), whatever the other items are and in whatever order they come; files must be byte for byte
what per-tensor compression followed by safetensors' writer produces (the algorithm before the batch path,
restated here as `per_tensor_file`)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
from safetensors import safe_open
from safetensors.torch import save_file as st_save_file

import chunk_settings as CS
from golden_safetensors_inputs import make_checkpoint
from oracle import oracle as O
from zipnn_b200 import SafeOpen, ZipNN, _native, compress_safetensors_file, load_file, save_file
from zipnn_b200 import safetensors_io as SIO

pytestmark = pytest.mark.gpu

CANARY = 0xA5
PAD = 64


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bm(G):
    return 220 if G == 4 else 10


def _bound(n, G, chunk, hdr_len):
    return _native.compress_bound(n, G, chunk, hdr_len)


class Batch:
    """Items over one canary-filled output buffer: region i is exactly its bound, PAD canary bytes on each side."""

    def __init__(self, specs):
        # spec: dict(d_in tensor or None, n, hdr bytes, G, bits, chunk, thr)
        self.specs = specs
        self.items = (_native.CompressItem * len(specs))()
        self.hdrs, self.offs, at = [], [], PAD
        for it, s in zip(self.items, specs):
            hdr = C.create_string_buffer(s["hdr"], len(s["hdr"]))
            self.hdrs.append(hdr)
            it.d_in = s["ptr"] if s["n"] else None
            it.n = s["n"]
            it.h_hdr, it.hdr_len = C.cast(hdr, C.c_void_p), len(s["hdr"])
            it.num_buf, it.bits_mode, it.bytes_mode = s["G"], s["bits"], _bm(s["G"])
            it.chunk, it.threshold = s["chunk"], s["thr"]
            it.out_cap = s.get("cap", _bound(s["n"], s["G"], s["chunk"], len(s["hdr"])))
            self.offs.append(at)
            at += it.out_cap + PAD
        self.out = torch.full((at,), CANARY, dtype=torch.uint8, device="cuda")
        for it, o in zip(self.items, self.offs):
            it.d_out = self.out.data_ptr() + o

    def run(self, sync=True):
        L = _native.lib()
        n = len(self.specs)
        wsz = C.c_size_t(256)
        if L.zipnn_b200_compress_batch_workspace_size(self.items, n, C.byref(wsz)) != 0:   # (an invalid item: the call
            wsz.value = 256                                                                    #  must refuse it first)
        self.ws = torch.empty(max(wsz.value, 1), dtype=torch.uint8, device="cuda")
        lens = (C.c_size_t * n)()
        rc = L.zipnn_b200_compress_batch(self.items, n, lens if sync else None, self.ws.data_ptr(), self.ws.numel(), _stream())
        return rc, list(lens)

    def streams(self, lens):
        host = self.out.cpu().numpy()
        res = []
        for it, o, ln in zip(self.items, self.offs, lens):
            region = host[o - PAD: o + it.out_cap + PAD]
            assert np.all(region[:PAD] == CANARY), "wrote before the region"
            assert np.all(region[PAD + it.out_cap:] == CANARY), "wrote past the region"
            assert np.all(region[PAD + ln: PAD + it.out_cap] == CANARY), "wrote past the stream"
            res.append(host[o: o + ln].copy())
        return res


def single_compress(d_in, n, hdr, G, bits, chunk, thr):
    bound = _bound(n, G, chunk, len(hdr))
    d_out = torch.empty(bound, dtype=torch.uint8, device="cuda")
    ws = torch.empty(_native.compress_workspace_size(n, G, chunk), dtype=torch.uint8, device="cuda")
    out_len = C.c_size_t(0)
    hb = C.create_string_buffer(hdr, len(hdr))
    rc = _native.lib().zipnn_b200_compress(d_in.data_ptr() if n else None, n, hb, len(hdr), G, bits, _bm(G), chunk, thr,
                                           d_out.data_ptr(), bound, C.byref(out_len), ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, rc
    return d_out[: out_len.value].cpu().numpy()


# ------------------------------------------------------------------ every chunk size and threshold, one call
def test_settings_cases_in_one_call():
    cases = CS.settings_inputs()
    d_ins = [torch.from_numpy(c["data"].copy()).cuda() for c in cases]
    specs = [dict(ptr=d.data_ptr(), n=c["data"].size, hdr=CS.header(), G=c["G"], bits=c["bits"], chunk=c["chunk"], thr=c["thr"])
             for c, d in zip(cases, d_ins)]
    before = _native.launch_count()
    b = Batch(specs)
    rc, lens = b.run()
    assert rc == 0, rc
    launches = _native.launch_count() - before
    assert launches == 3 * 5, launches   # one of each kernel per byte-group class, each with general-write work
    got = b.streams(lens)
    for c, d, s in zip(cases, d_ins, got):
        want = O.zipnn_compress(CS.header(), c["data"], c["G"], c["bits"], _bm(c["G"]), c["chunk"], c["thr"], threads=2)
        assert np.array_equal(s, want), f"{c['name']}: batch stream != oracle stream"
        assert np.array_equal(s, single_compress(d, c["data"].size, CS.header(), c["G"], c["bits"], c["chunk"], c["thr"])), c["name"]
        assert np.array_equal(d.cpu().numpy(), c["data"]), "the encoder changed its input"
    rb = Batch(specs[::-1])
    rc, rlens = rb.run()
    assert rc == 0
    for s, r in zip(got, rb.streams(rlens)[::-1]):
        assert np.array_equal(s, r)


def test_settings_cases_routed(monkeypatch):
    """Tensors over the routing limit (lowered to 64 chunks) are coded by the single-tensor launches on the same
    stream, between and after batch tensors of every class; their streams and lengths are the same."""
    monkeypatch.setenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", "64")
    cases = CS.settings_inputs(big=False)[::3]
    d_ins = [torch.from_numpy(c["data"].copy()).cuda() for c in cases]
    specs = [dict(ptr=d.data_ptr(), n=c["data"].size, hdr=CS.header(), G=c["G"], bits=c["bits"], chunk=c["chunk"], thr=c["thr"])
             for c, d in zip(cases, d_ins)]
    assert any(-(-c["data"].size // c["chunk"]) > 64 for c in cases) and any(-(-c["data"].size // c["chunk"]) <= 64 for c in cases)
    b = Batch(specs)
    rc, lens = b.run()
    assert rc == 0, rc
    for c, s in zip(cases, b.streams(lens)):
        want = O.zipnn_compress(CS.header(), c["data"], c["G"], c["bits"], _bm(c["G"]), c["chunk"], c["thr"], threads=2)
        assert np.array_equal(s, want), c["name"]


# ------------------------------------------------------------------ a checkpoint-like mix
MIX_DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2)


def _mix():
    """Per dtype, coded with 4 KiB chunks: empty, one element, under 64*G bytes, a ragged last chunk, exact chunk
    multiples, several chunks; one fp8 tensor of 3100 chunks (past 3072, where the batch decoder hands a tensor to the
    single-tensor path), constant planes, and one input passed twice."""
    g = torch.Generator(device="cuda").manual_seed(11)
    out = []
    for dt in MIX_DTYPES:
        es = dt.itemsize
        for n in (0, 1, 60 // es, (3 * 4096 + 1000) // es, 4 * 4096 // es, 40000):
            out.append((torch.randn(n, generator=g, device="cuda") * 0.02).to(dt))
    out.append((torch.randn(3100 * 4096, generator=g, device="cuda") * 0.5).to(torch.float8_e4m3fn))
    out.append(torch.full((5000,), 0.25, device="cuda").to(torch.bfloat16))    # RLE planes
    out.append(out[3])                                                            # the same input twice
    return out


def decode_batch(streams, dtypes, shapes):
    """Streams -> tensors through zipnn_b200_decompress_batch (one call for all of them)."""
    L = _native.lib()
    items = (_native.BatchItem * len(streams))()
    outs = []
    for it, s, dt in zip(items, streams, dtypes):
        z = ZipNN(input_format="torch")
        head = s[: 4096].cpu().numpy().tobytes()
        off = z._retrieve_header(head)
        orig = z.original_len
        o = torch.empty(max(orig, 1), dtype=torch.uint8, device="cuda")
        outs.append(o[:orig])
        it.d_body, it.body_len = s.data_ptr() + off, s.numel() - off
        it.num_buf = dt.itemsize
        it.bits_mode, it.bytes_mode = head[6], head[5]
        chunk = z.compression_chunk if dt.itemsize != 1 else min(z.compression_chunk, 128 * 1024)
        it.chunk, it.orig, it.d_out = chunk, orig, o.data_ptr()
    wsz = C.c_size_t(0)
    assert L.zipnn_b200_decompress_batch_workspace_size(items, len(streams), C.byref(wsz)) == 0
    ws = torch.empty(max(wsz.value, 1), dtype=torch.uint8, device="cuda")
    assert L.zipnn_b200_decompress_batch(items, len(streams), ws.data_ptr(), ws.numel(), _stream(), 1) == 0
    return [o.view(dt).view(sh) for o, dt, sh in zip(outs, dtypes, shapes)]


# "2": every tensor of more than two chunks takes the single-tensor launches inside the batch call
@pytest.mark.parametrize("route", ["", "2"])
def test_checkpoint_mix_matches_compress_and_round_trips(monkeypatch, route):
    if route:
        monkeypatch.setenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", route)
    tensors = _mix()
    z = ZipNN(input_format="torch", compression_chunk=4096)
    got = z.compress_batch(tensors)
    assert len(got) == len(tensors)
    for t, s in zip(tensors, got):
        want = ZipNN(input_format="torch", compression_chunk=4096).compress(t)
        assert torch.equal(s, want), (t.dtype, t.shape)
    back = decode_batch(got, [t.dtype for t in tensors], [t.shape for t in tensors])
    for t, b in zip(tensors, back):
        assert torch.equal(b.view(torch.uint8), t.view(torch.uint8)), (t.dtype, t.shape)


def test_compress_batch_default_settings():
    g = torch.Generator(device="cuda").manual_seed(5)
    tensors = [(torch.randn(n, generator=g, device="cuda") * 0.02).to(dt)
               for dt in MIX_DTYPES for n in (0, 7, 100000, 3 * 131072 + 17)]
    tensors.append(tensors[2][1:])   # a view that is not 16-byte aligned
    got = ZipNN(input_format="torch").compress_batch(tensors)
    for t, s in zip(tensors, got):
        assert torch.equal(s, ZipNN(input_format="torch").compress(t))


# ------------------------------------------------------------------ launch count
def _launch_specs(reps, keep):
    g = torch.Generator(device="cuda").manual_seed(2)
    specs = []
    for r in range(reps):
        for dt, G, bits, n in ((torch.bfloat16, 2, 1, 3 * 262144 + 1000), (torch.float32, 4, 1, 70000 * 4), (torch.bfloat16, 2, 1, 262144)):
            t = torch.randn(n // dt.itemsize, generator=g, device="cuda").to(dt)
            keep.append(t)
            specs.append(dict(ptr=t.data_ptr(), n=n, hdr=CS.header(), G=G, bits=bits, chunk=262144, thr=0.95))
    return specs


def test_launch_count_does_not_depend_on_tensor_count():
    keep = []
    counts = []
    for reps in (1, 100):   # 3 and 300 tensors of the same two byte-group classes, each with a ragged last chunk
        b = Batch(_launch_specs(reps, keep))
        before = _native.launch_count()
        rc, _ = b.run()
        assert rc == 0
        counts.append(_native.launch_count() - before)
    # DESIGN 3.8: per class present, hist + table + scan + warp write, + general write when the class has general work
    assert counts == [2 * 5, 2 * 5]


# ------------------------------------------------------------------ invalid items
@pytest.mark.parametrize("bad", ["misaligned", "short", "chunk_below_G", "header_short"])
def test_invalid_item_writes_nothing(bad):
    keep = []
    specs = _launch_specs(2, keep)
    s = specs[3]
    want = 1   # E_ARG
    if bad == "misaligned":
        s["ptr"] += 8
        s["n"] -= 16
    elif bad == "short":
        s["cap"] = _bound(s["n"], s["G"], s["chunk"], 32) - 1
        want = 2   # E_CAPACITY
    elif bad == "chunk_below_G":
        s["chunk"] = 1
    else:
        s["hdr"] = bytes(31)
    b = Batch(specs)
    rc, _ = b.run()
    torch.cuda.synchronize()
    assert rc == want
    assert bool((b.out == CANARY).all())


# ------------------------------------------------------------------ asynchronous lengths
@pytest.mark.parametrize("route", ["", "2"])
def test_async_lengths_in_headers(monkeypatch, route):
    if route:
        monkeypatch.setenv("ZIPNN_B200_ENC_BATCH_MAX_CHUNKS", route)
    keep = []
    specs = _launch_specs(3, keep)
    specs.append(dict(ptr=0, n=0, hdr=CS.header() + b"\x01\x02", G=2, bits=1, chunk=262144, thr=0.95))   # header-only
    b1 = Batch(specs)
    rc, lens = b1.run(sync=True)
    assert rc == 0
    b2 = Batch(specs)
    rc, _ = b2.run(sync=False)
    assert rc == 0
    torch.cuda.current_stream().synchronize()
    host = b2.out.cpu().numpy()
    for o, ln in zip(b2.offs, lens):
        assert int.from_bytes(host[o + 24: o + 32].tobytes(), "little") == ln
    assert lens[-1] == 34
    assert all(np.array_equal(a, c) for a, c in zip(b1.streams(lens), b2.streams(lens)))


# ------------------------------------------------------------------ files
def per_tensor_file(src, dst):
    """The file writer before the batch path: one ZipNN.compress per floating-point tensor, safetensors' writer."""
    tensors, infos = {}, {}
    with safe_open(src, "pt", "cpu") as f:
        for name in f.keys():
            t = f.get_tensor(name)
            if not torch.is_floating_point(t):
                tensors[name] = t
                continue
            buf = ZipNN(input_format="torch", bytearray_dtype=t.dtype, method="HUFFMAN").compress(t.cuda())
            if buf.numel() >= t.numel() * t.element_size():
                tensors[name] = t
                continue
            tensors[name] = buf.cpu()
            infos[name] = {"dtype": str(t.dtype).replace("torch.", ""), "shape": str(list(t.shape))}
        md = f.metadata()
    md = dict(md) if md else {}
    md["znn_compressed_vectors"] = json.dumps(infos)
    st_save_file(tensors, dst, md)


def _file_bytes(p):
    with open(p, "rb") as f:
        return f.read()


def assert_same_file(a, b):
    """Byte for byte, except for the order of the metadata keys: safetensors writes a metadata dict of more than one
    key in hash order, which differs from one write to the next of the same dict."""
    x, y = _file_bytes(a), _file_bytes(b)
    if x == y:
        return
    hx, hy = int.from_bytes(x[:8], "little"), int.from_bytes(y[:8], "little")
    assert hx == hy and x[8 + hx:] == y[8 + hy:], "tensor data differ"
    jx, jy = json.loads(x[8: 8 + hx]), json.loads(y[8: 8 + hy])
    assert jx.pop("__metadata__") == jy.pop("__metadata__")
    assert list(jx.items()) == list(jy.items()), "tensor entries differ"


def _save_dict():
    d = make_checkpoint()
    g = torch.Generator().manual_seed(9)
    d["tiny_bf16"] = torch.tensor([0.5], dtype=torch.bfloat16)          # stream longer than the tensor: kept raw
    d["tiny_fp32"] = torch.randn(3, generator=g)
    d["empty_fp16"] = torch.zeros(0, 4, dtype=torch.float16)
    d["fp8_e5m2"] = (torch.randn(70000, generator=g) * 0.3).to(torch.float8_e5m2)
    d["big_fp32"] = torch.randn(300, 1000, generator=g) * 0.02
    d["mask"] = torch.ones(17, dtype=torch.bool)
    return d


@pytest.mark.parametrize("where", ["cuda", "cpu"])
@pytest.mark.parametrize("metadata", [None, {"format": "pt", "x": "y"}])
def test_save_file_matches_per_tensor_file(tmp_path, monkeypatch, where, metadata):
    monkeypatch.setattr(SIO, "SAVE_GROUP_BYTES", 64 * 1024)   # several groups, and tensors over the budget
    d = _save_dict()
    src = str(tmp_path / "m.safetensors")
    st_save_file(d, src, metadata)
    ref = str(tmp_path / "ref.znn.safetensors")
    per_tensor_file(src, ref)
    ours = str(tmp_path / "ours.znn.safetensors")
    save_file({k: (v.cuda() if where == "cuda" else v) for k, v in d.items()}, ours, metadata)
    assert_same_file(ours, ref)
    meta = json.loads(safe_open(ours, "pt", "cpu").metadata()["znn_compressed_vectors"])
    assert "tiny_bf16" not in meta and "w_bf16" in meta
    back = load_file(ours, "cuda")
    assert set(back) == set(d)
    for k, v in d.items():
        assert back[k].dtype == v.dtype and back[k].shape == v.shape
        assert torch.equal(back[k].cpu().view(torch.uint8) if v.numel() else back[k].cpu(), v.view(torch.uint8) if v.numel() else v), k
    with SafeOpen(ours, "pt", "cuda", slices=True) as f:
        for k, v in d.items():
            if v.dim() >= 1 and v.shape[0] > 1:
                got = f.get_slice(k)[1:]
                assert torch.equal(got.cpu().view(torch.uint8), v[1:].contiguous().view(torch.uint8)), k


def test_save_file_refuses_like_safetensors(tmp_path):
    base = torch.randn(10, 10).cuda()
    with pytest.raises(RuntimeError):
        save_file({"a": base, "b": base[2:]}, str(tmp_path / "x.znn.safetensors"))
    with pytest.raises(ValueError):
        save_file({"a": base.t()}, str(tmp_path / "x.znn.safetensors"))
    with pytest.raises(ValueError):
        save_file({"a": [1, 2]}, str(tmp_path / "x.znn.safetensors"))
    assert not os.path.exists(tmp_path / "x.znn.safetensors")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_save_file_refuses_two_devices(tmp_path):
    with pytest.raises(ValueError, match="one GPU"):
        save_file({"a": torch.randn(8, device="cuda:0"), "b": torch.randn(8, device="cuda:1")}, str(tmp_path / "x.znn.safetensors"))
    assert not os.path.exists(tmp_path / "x.znn.safetensors")


def test_compress_file_matches_per_tensor_file(tmp_path, monkeypatch):
    monkeypatch.setattr(SIO, "SAVE_GROUP_BYTES", 48 * 1024)
    src = str(tmp_path / "c.safetensors")
    st_save_file(make_checkpoint(), src)
    ref = str(tmp_path / "ref.znn.safetensors")
    per_tensor_file(src, ref)
    path, clen, olen = compress_safetensors_file(src)
    assert_same_file(path, ref)
    host_path = str(tmp_path / "h" / "c.safetensors")
    os.makedirs(os.path.dirname(host_path))
    st_save_file(make_checkpoint(), host_path)
    assert compress_safetensors_file(host_path, device=None)[1:] == (clen, olen)


@pytest.mark.parametrize("device", [None, "cpu", 0, "cuda", "cuda:0", torch.device("cuda", 0)])
def test_compress_file_device_values(tmp_path, monkeypatch, device):
    """A CUDA device (name, torch.device or index) takes the batched path; anything else the per-tensor path it took
    before, "cpu" included.  Both write the per-tensor algorithm's file."""
    calls = []
    orig = SIO._compress_entries
    monkeypatch.setattr(SIO, "_compress_entries", lambda *a, **k: calls.append(1) or orig(*a, **k))
    src = str(tmp_path / "c.safetensors")
    st_save_file(make_checkpoint(), src)   # (one metadata key: safetensors writes several in hash order)
    ref = str(tmp_path / "ref.znn.safetensors")
    per_tensor_file(src, ref)
    want = _file_bytes(ref)
    path, _, _ = compress_safetensors_file(src, device=device)
    assert _file_bytes(path) == want
    cuda = device is not None and device != "cpu"
    assert bool(calls) == cuda


def test_compress_file_llama_layers(tmp_path, monkeypatch):
    """Two decoder layers of llama3-8b's shapes (the embedding and head left out for size): tensors over the group
    budget, q/o projections within it, norms packed together."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from model_bench import MODELS
    monkeypatch.setattr(SIO, "SAVE_GROUP_BYTES", 64 << 20)
    shapes, dtype = MODELS["llama3-8b"](2)
    g = torch.Generator(device="cuda").manual_seed(1234)
    d = {k: (torch.randn(*s, generator=g, device="cuda") * 0.02).to(dtype).cpu() for k, s in shapes.items()
         if "embed" not in k and "lm_head" not in k}
    src = str(tmp_path / "l.safetensors")
    st_save_file(d, src, {"format": "pt"})
    ref = str(tmp_path / "ref.znn.safetensors")
    per_tensor_file(src, ref)
    path, _, _ = compress_safetensors_file(src)
    assert_same_file(path, ref)
