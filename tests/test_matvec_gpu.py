"""x W^T straight from compressed weights (zipnn_b200_decode_plan_matvec, DecodePlan.matvec, compress_module /
load_module with matvec=N) against the fp64 product of the decoded weights.

  * exact cases: weights and activations whose every partial sum is exact in fp32, so the result must be the fp64
    product rounded once, bit for bit, in any order of addition;
  * general cases: Gaussian weights and activations in bf16 / fp16 / fp32, rows that divide a quarter plane, straddle
    it and span several, a short last chunk, one row and the narrowest rows, every token count, strided x and y, with
    and without bias, under the bound of an fp32 accumulation plus one rounding; two calls give the same bits;
  * canaries around y and the scratch, 2 launches per call, none for no tokens, graph replay with new x;
  * host rejections write nothing; items with other chunk modes answer E_UNSUPPORTED;
  * a small llama-shaped model under compress_module(matvec=N) and load_module(matvec=N).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import test_boxes_host as H
import test_decode_plan_gpu as DP
import test_decoder_tables_gpu as D
import test_matvec_host as MH
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200.plan import MATVEC_MAX_TOKENS

pytestmark = pytest.mark.gpu

CANARY = 0xA5
CODE = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 2}
REL = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}   # half an ulp, relative, at most
TINY = {torch.bfloat16: 0.0, torch.float16: 2.0 ** -25, torch.float32: 0.0}              # half a subnormal step


def _st():
    return torch.cuda.current_stream().cuda_stream


def _plan_of(w: torch.Tensor) -> DecodePlan:
    return DecodePlan([ZipNN(input_format="torch").compress(w)])


def _gauss(shape, dtype, seed, std=0.02):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * std).to(dtype)


def _check(y, x, w, bias, what):
    """|y - fp64 product| <= in * 2^-24 * sum |x_i w_i| (fp32 accumulation) + half an ulp of the output type."""
    x64, w64 = x.double().reshape(-1, x.shape[-1]), w.double()
    ref = x64 @ w64.T
    mag = x64.abs() @ w64.abs().T
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    bound = (x.shape[-1] + 1) * 2.0 ** -24 * mag
    tol = bound + (ref.abs() + bound) * REL[y.dtype] + TINY[y.dtype]
    err = (y.double().reshape(ref.shape) - ref).abs()
    assert torch.all(err <= tol), (what, float((err - tol).max()))


def test_exact_products_bit_for_bit():
    rng = np.random.default_rng(1)
    for out_f, in_f, nt in ((64, 4096, 1), (192, 2048, 8), (1024, 256, 5), (24, 3072, 3)):
        m = rng.integers(128, 256, (out_f, in_f)).astype(np.float64)   # an 8-bit significand
        e = rng.integers(-9, -5, (out_f, in_f)).astype(np.float64)     # four exponents
        s = rng.choice([-1.0, 1.0], (out_f, in_f))
        w = torch.from_numpy(s * m * 2.0 ** e).to(torch.bfloat16).cuda()
        assert torch.equal(w.double().cpu(), torch.from_numpy(s * m * 2.0 ** e)), "the weights are exact in bf16"
        x = torch.from_numpy(rng.integers(-1, 2, (nt, in_f)).astype(np.float32)).to(torch.bfloat16).cuda()
        plan = _plan_of(w)
        assert plan.matvec_ok(0, in_f), "these weights must give fused chunks, or the case tests nothing"
        y = plan.matvec(0, x)
        want = (x.double() @ w.double().T).to(torch.bfloat16)   # sums of at most 4096 * 255 * 2^3 units: exact in fp32
        assert torch.equal(y, want), (out_f, in_f, nt)
        plan.check()


SHAPES = [s[:2] for s in MH.SHAPES if s[2] == 2]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_general_cases(dtype):
    es = torch.empty(0, dtype=dtype).element_size()
    shapes = [(o, i) for o, i in SHAPES if (i * es) % 16 == 0 and o * i * es <= 8 << 20] + [(3, 49152)]
    n_calls = 0
    for k, (out_f, in_f) in enumerate(shapes):
        w = _gauss((out_f, in_f), dtype, 100 + k)
        plan = _plan_of(w)
        assert plan.matvec_ok(0, in_f), (out_f, in_f)
        L = MH.Layout(out_f, in_f, es)
        for nt in range(1, MATVEC_MAX_TOKENS + 1):
            assert plan.matvec_scratch_bytes(0, in_f, nt) == L.slots() * nt * 4, "the layout the host test checks"
            bias = _gauss((out_f,), dtype, 7 * k + nt, std=0.5) if (k + nt) % 2 else None
            strided = nt % 3 == 0
            xbuf = _gauss((nt, in_f + (16 if strided else 0)), dtype, 1000 * k + nt, std=1.0)
            x = xbuf[:, 8: 8 + in_f] if strided else xbuf
            ybuf = torch.full((nt + 2, out_f + 6), float("nan"), dtype=dtype, device="cuda")
            y = ybuf[1: nt + 1, 3: 3 + out_f] if strided else None
            need = plan.matvec_scratch_bytes(0, in_f, nt)
            sbuf = torch.full((256 + need + 256,), CANARY, dtype=torch.uint8, device="cuda")
            off = -sbuf.data_ptr() % 256
            before = _native.launch_count()
            got = plan.matvec(0, x, bias=bias, out=y, scratch=sbuf[off: off + need])
            assert _native.launch_count() - before == 2, "two launches whatever the shape and token count"
            _check(got, x, w, bias, (dtype, out_f, in_f, nt))
            if strided:
                mask = torch.ones_like(ybuf, dtype=torch.bool)
                mask[1: nt + 1, 3: 3 + out_f] = False
                assert torch.all(torch.isnan(ybuf[mask])), "wrote outside y"
            assert torch.all(sbuf[:off] == CANARY) and torch.all(sbuf[off + need:] == CANARY), "wrote outside the scratch"
            again = plan.matvec(0, x, bias=bias)
            assert torch.equal(got.contiguous().view(torch.uint8), again.view(torch.uint8)), "two calls, two results"
            n_calls += 1
        plan.check()
    print(f"{dtype}: {n_calls} shapes x token counts")


def test_shapes_of_x_and_no_tokens():
    w = _gauss((64, 4096), torch.bfloat16, 3)
    plan = _plan_of(w)
    x = _gauss((2, 3, 4096), torch.bfloat16, 4, std=1.0)
    y = plan.matvec(0, x)
    assert y.shape == (2, 3, 64)
    _check(y, x, w, None, "3-D x")
    y1 = plan.matvec(0, x[0, 0])
    assert y1.shape == (64,) and torch.equal(y1, y[0, 0])
    odd = _gauss((4097,), torch.bfloat16, 5, std=1.0)[1:]   # a row that is not 16-byte aligned is copied first
    _check(plan.matvec(0, odd), odd, w, None, "misaligned x")
    before = _native.launch_count()
    assert plan.matvec(0, x[:0]).shape == (0, 3, 64) and _native.launch_count() == before, "no tokens, no launch"
    with pytest.raises(ValueError):
        plan.matvec(0, _gauss((9, 4096), torch.bfloat16, 6))
    with pytest.raises(ValueError):
        plan.matvec(0, x.float())
    with pytest.raises(ValueError):
        plan.matvec(0, _gauss((1, 4100), torch.bfloat16, 6))   # does not divide the tensor
    assert not plan.matvec_ok(0, 4100) and not plan.matvec_ok(0, 4) and plan.matvec_ok(0, 8)
    plan.check()


def test_graph_replay_with_new_x():
    w = _gauss((512, 1024), torch.bfloat16, 8)
    plan = _plan_of(w)
    x = torch.zeros(4, 1024, dtype=torch.bfloat16, device="cuda")
    out = torch.empty(4, 512, dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(plan.matvec_scratch_bytes(0, 1024, 4), dtype=torch.uint8, device="cuda")
    plan.matvec(0, x, out=out, scratch=scratch)   # (the first call for an output synchronises: not capturable)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.matvec(0, x, out=out, scratch=scratch)
    for seed in range(3):
        new = _gauss((4, 1024), torch.bfloat16, 20 + seed, std=1.0)
        x.copy_(new)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, plan.matvec(0, new)), seed
    plan.check()


def test_host_rejections_write_nothing(monkeypatch):
    L = _native.lib()
    w = _gauss((64, 4096), torch.bfloat16, 9)
    plan = _plan_of(w)
    need = plan.matvec_scratch_bytes(0, 4096, 2)
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    x = _gauss((2, 4096), torch.bfloat16, 10)
    y = torch.full((2, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    bad = [("tokens", dict(nt=MATVEC_MAX_TOKENS + 1), A), ("dtype", dict(dtype=3), A), ("in 0", dict(inf=0), A),
           ("in not dividing", dict(inf=4104), A), ("item -1", dict(item=-1), A), ("item 1", dict(item=1), A),
           ("null x", dict(x=None), A), ("null y", dict(y=None), A), ("null scratch", dict(scratch=None), A),
           ("x alignment", dict(x=x.data_ptr() + 2), A), ("x stride", dict(xs=4100), A), ("short x stride", dict(xs=2048), A),
           ("short y stride", dict(ys=32), A), ("y alignment", dict(y=y.data_ptr() + 1), A), ("bias alignment", dict(bias=bias.data_ptr() + 1), A),
           ("scratch alignment", dict(scratch=scratch.data_ptr() + 16), A), ("short scratch", dict(sb=need - 1), A),
           ("dtype of another size", dict(dtype=2, inf=2048), U), ("rows of 8 bytes", dict(inf=4), U)]
    for name, kw, want in bad:
        a = dict(item=0, dtype=0, inf=4096, x=x.data_ptr(), xs=4096, nt=2, bias=bias.data_ptr(), y=y.data_ptr(), ys=64,
                 scratch=scratch.data_ptr(), sb=need)
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_matvec(plan._ref, a["item"], a["dtype"], a["inf"], a["x"], a["xs"], a["nt"], a["bias"], a["y"],
                                             a["ys"], a["scratch"], a["sb"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    assert torch.all(torch.isnan(y))
    out = C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(plan._ref, 0, 0, 4096, MATVEC_MAX_TOKENS + 1, C.byref(out)) == A
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(plan._ref, 0, 0, 4096, 2, None) == A
    # a plan without a segment index
    DP._set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    q = _plan_of(w)
    before = _native.launch_count()
    assert not q.matvec_ok(0, 4096)
    assert L.zipnn_b200_decode_plan_matvec(q._ref, 0, 0, 4096, x.data_ptr(), 4096, 2, None, y.data_ptr(), 64, scratch.data_ptr(), need,
                                           _st()) == U
    assert _native.launch_count() == before and torch.all(torch.isnan(y))


# ---- items the matvec must refuse: the kernel skips a chunk that is not fused and the reduce would add whatever the
# scratch holds, so the host check is what stands between such an item and a wrong product -----------------------------
def _refused(pl, item, G, in_bytes, what):
    """Item `item` of the raw plan `pl`, seen as rows of in_bytes bytes (a multiple of 16 that divides it): both calls
    answer E_UNSUPPORTED, nothing is launched, y keeps its bytes."""
    L = _native.lib()
    code, inf = (0 if G == 2 else 2), in_bytes // G
    assert in_bytes % 16 == 0 and pl.items[item].orig % in_bytes == 0, "the shape itself must be acceptable"
    x = torch.zeros(inf, dtype=torch.uint8, device="cuda").repeat(G)
    y = torch.full((pl.items[item].orig // in_bytes * G,), CANARY, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(4 << 20, dtype=torch.uint8, device="cuda")
    out = C.c_size_t(0)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matvec_scratch_size(C.byref(pl.plan), item, code, inf, 1, C.byref(out)) == _native.E_UNSUPPORTED, what
    rc = L.zipnn_b200_decode_plan_matvec(C.byref(pl.plan), item, code, inf, x.data_ptr(), inf, 1, None, y.data_ptr(), y.numel() // G,
                                         scratch.data_ptr(), scratch.numel(), _st())
    assert rc == _native.E_UNSUPPORTED, (what, rc)
    assert _native.launch_count() == before, what
    assert torch.all(y == CANARY), what


def _raw_plan(case, box=None):
    want = case.data if box is None else H.expect(case, box)
    return DP.Plan([DP.Item(case.name, case.body, case.G, case.bits, case.chunk, case.data.size, want, box=box)])


def _decodes(pl, what):
    for it in pl.items:
        it.scribble()
    assert pl.run() == 0 and pl.status() == 0
    for it in pl.items:
        it.check(what)


@pytest.mark.parametrize("G", (2, 4))
def test_items_with_other_chunk_modes_boxes_and_split_items_are_unsupported(G, monkeypatch):
    DP._set_env(monkeypatch, {})
    dt = H.DTYPE[G]
    second = lambda c, g: "geo5" if g == G - 2 and c % 4 == 1 else "raw"  # noqa: E731  a second coded plane: general
    mixed = D.planes_case(f"mv_mixed_G{G}", dt, 4096, ["geo5"] * 16, seed=700 + G, side=second)
    assert mixed.pr["mode"][0] == "fused" and set(mixed.pr["mode"]) == {"fused", "general"}
    many = D.planes_case(f"mv_overflow_G{G}", dt, 512, ["geo5"] * 300, seed=710 + G,
                         side=lambda c, g: "geo5" if g == G - 2 and c >= 1 else "raw")
    assert many.pr["mode"][0] == "fused" and many.pr["mode"].count("general") > 64 + 32, "general chunks past the pool: overflow"
    ragged = D.planes_case(f"mv_ragged_G{G}", dt, 4096, ["geo5"] * 5, seed=720 + G, last=3840)
    assert ragged.pr["mode"][:-1] == ["fused"] * 4 and ragged.pr["mode"][-1] != "fused" and 3840 % 512
    plain = D.planes_case(f"mv_plain_G{G}", dt, 4096, ["geo5"] * 7 + ["const"], seed=730 + G)
    assert plain.pr["mode"] == ["fused"] * 7 + ["plain"], "only the last chunk differs"
    for case, in_bytes in ((mixed, 512), (many, 128), (ragged, 256), (plain, 1024)):
        pl = _raw_plan(case)
        assert pl.rc == 0
        _refused(pl, 0, G, in_bytes, case.name)
        _decodes(pl, case.name)
    # an eligible tensor: accepted whole (so the refusals above and below are about modes and pieces, nothing else),
    # refused as a box and when it was split into pieces
    good = D.planes_case(f"mv_fused_G{G}", dt, 4096, ["geo5"] * 8, seed=740 + G)
    assert good.pr["mode"] == ["fused"] * 8
    pl = _raw_plan(good)
    out = C.c_size_t(0)
    assert pl.rc == 0
    assert _native.lib().zipnn_b200_decode_plan_matvec_scratch_size(C.byref(pl.plan), 0, 0 if G == 2 else 2, 512 // G, 1, C.byref(out)) == 0
    assert out.value > 0
    boxed = _raw_plan(good, box=(0, 2, 8192, 4096))
    assert boxed.rc == 0
    _refused(boxed, 0, G, 512, "a box")
    _decodes(boxed, "a box")
    DP._set_env(monkeypatch, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "5"})
    split = _raw_plan(good)
    assert split.rc == 0
    _refused(split, 0, G, 512, "a split item")
    _decodes(split, "a split item")


def test_ineligible_outputs_of_a_decode_plan_still_decode():
    """DecodePlan.matvec_ok is False and run() gives the dense bytes for: a last chunk that is not a multiple of 512
    bytes, an fp32 tensor with three mantissa bits (two coded planes in every chunk) and a constant tensor (no coded
    plane)."""
    ragged = _gauss((1039, 128), torch.bfloat16, 30)   # 256 KiB + 3840 bytes
    coarse = (_gauss((512, 256), torch.float32, 31).view(torch.int32) & -(1 << 20)).view(torch.float32)
    const = torch.full((256, 256), 2.0 ** -6, dtype=torch.bfloat16, device="cuda")
    for name, w in (("ragged", ragged), ("coarse", coarse), ("const", const)):
        plan = _plan_of(w)
        before = _native.launch_count()
        assert not plan.matvec_ok(0, w.shape[1]), name
        with pytest.raises(ValueError):
            plan.matvec(0, torch.zeros(1, w.shape[1], dtype=w.dtype, device="cuda"))
        assert _native.launch_count() == before, name
        plan.outputs[0].zero_()
        assert torch.equal(plan.run()[0].view(torch.uint8), w.view(torch.uint8)), name
        plan.check()


# ---- resident models ------------------------------------------------------------------------------------------------
class Block(torch.nn.Module):
    def __init__(self, d, f):
        super().__init__()
        self.q = torch.nn.Linear(d, d, bias=False)
        self.up = torch.nn.Linear(d, f, bias=False)
        self.down = torch.nn.Linear(f, d, bias=False)

    def forward(self, x):
        return x + self.down(torch.nn.functional.silu(self.up(self.q(x))))


class Llamaish(torch.nn.Module):
    def __init__(self, tied, vocab=1000, d=256, f=512):
        super().__init__()
        self.emb = torch.nn.Embedding(vocab, d)
        self.blocks = torch.nn.Sequential(Block(d, f), Block(d, f))
        self.proj = torch.nn.Linear(d, d, bias=True)
        self.const = torch.nn.Linear(d, d, bias=False)   # a constant weight: RLE planes, no fused chunk
        self.head = torch.nn.Linear(d, vocab, bias=False)
        if tied:
            self.head.weight = self.emb.weight

    def forward(self, ids):
        x = self.blocks(self.emb(ids))
        return self.head(self.proj(x) + self.const(x))


def _model(tied, dtype, device="cuda"):
    torch.manual_seed(11)
    m = Llamaish(tied)
    with torch.no_grad():
        for p in m.parameters():   # Gaussian weights: one coded byte plane per chunk in every dtype
            p.normal_(0, 0.05)
        m.const.weight.fill_(2.0 ** -6)
    return m.to(dtype).to(device).eval()


N = 4


@pytest.mark.parametrize("tied", (False, True))
@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16))
@pytest.mark.parametrize("how", ("compress", "load"))
def test_resident_model(how, dtype, tied, tmp_path):
    dense = _model(tied, dtype)
    params = {n: p.detach().clone() for n, p in dense.named_parameters()}
    ids = torch.randint(0, 1000, (N + 1,), device="cuda", generator=torch.Generator("cuda").manual_seed(12))
    with torch.no_grad():
        want = [dense(ids[:t]).double() for t in range(1, N + 2)]
    plain = _model(tied, dtype)
    compress_module(plain)
    f0, f1 = os.path.join(tmp_path, "plain.znn.safetensors"), os.path.join(tmp_path, "matvec.znn.safetensors")
    save_module(plain, f0)
    if how == "compress":
        model = _model(tied, dtype)
        rep = compress_module(model, matvec=N)
    else:
        with torch.device("meta"):
            model = Llamaish(tied).to(dtype).eval()
        rep = load_module(model, f0, matvec=N)
    # q, up, down of two blocks, proj and the head multiply from the stream; the constant weight does not
    assert rep["matvec_modules"] == 8 and rep["matvec_scratch_bytes"] > 0
    assert "forward" not in model.const.__dict__ and "forward" in model.head.__dict__
    assert isinstance(model.proj.bias, torch.nn.Parameter) and "weight" not in model.proj._parameters
    tol = 1e-4 if dtype == torch.float32 else 4e-2
    with torch.no_grad():
        for t in range(1, N + 1):
            got = model(ids[:t]).double()
            assert (got - want[t - 1]).abs().max() <= tol * want[t - 1].abs().max(), (t, float((got - want[t - 1]).abs().max()))
        before = _native.launch_count()
        model.head(want[0].to(dtype)[:, :256].contiguous())
        assert _native.launch_count() - before == 2, "a matvec module decodes nothing for a small input"
        assert torch.equal(model(ids), plain(ids)), "more rows than N: the decode path, bit for bit"
        assert torch.equal(model(ids).double(), want[N])
    save_module(model, f1)
    with open(f0, "rb") as a, open(f1, "rb") as b:
        assert a.read() == b.read(), "the saved file does not depend on matvec"
    decompress_module(model)
    assert "forward" not in model.head.__dict__
    got = dict(model.named_parameters())
    assert set(got) == set(params)
    for n, p in params.items():
        assert torch.equal(got[n], p), n
    assert (model.head.weight is model.emb.weight) == tied
    with torch.no_grad():
        assert torch.equal(model(ids).double(), want[N])
