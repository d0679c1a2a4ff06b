"""x W^T for up to 64 rows on tensor cores, straight from compressed weights (zipnn_b200_decode_plan_matmul,
DecodePlan.matmul, compress_module / load_module with matmul=N) against the fp64 product of the decoded weights.

  * exact cases: weights and activations whose every partial sum is exact in fp32, bit for bit;
  * Gaussian bf16 / fp16 cases over test_matvec_gpu's shapes at 1 to 64 rows, strided x and y, with and without bias,
    under the bound of an fp32 accumulation that may round by up to an ulp at each addition; two calls, same bits;
  * canaries around y and the scratch, 2 launches per call, none for no rows, graph replay with new x;
  * host rejections write nothing; fp32 and items with other chunk modes, boxes and split items are E_UNSUPPORTED;
  * test_matvec_gpu's small llama-shaped model under compress_module(matmul=64) and load_module(matmul=64).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import test_decode_plan_gpu as DP
import test_decoder_tables_gpu as D
import test_matmul_host as MMH
import test_matvec_gpu as MV
from zipnn_b200 import _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200.plan import MATMUL_MAX_TOKENS

pytestmark = pytest.mark.gpu

ROWS = (1, 8, 9, 15, 16, 17, 31, 32, 33, 48, 63, 64)


def _check(y, x, w, bias, what):
    """|y - fp64 product| <= (in + 1) * 2^-23 * sum |x_i w_i| (an ulp per fp32 addition) + half an ulp of the output."""
    x64, w64 = x.double().reshape(-1, x.shape[-1]), w.double()
    ref = x64 @ w64.T
    mag = x64.abs() @ w64.abs().T
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    bound = (x.shape[-1] + 1) * 2.0 ** -23 * mag
    tol = bound + (ref.abs() + bound) * MV.REL[y.dtype] + MV.TINY[y.dtype]
    err = (y.double().reshape(ref.shape) - ref).abs()
    assert torch.all(err <= tol), (what, float((err - tol).max()))


def test_exact_products_bit_for_bit():
    rng = np.random.default_rng(2)
    for out_f, in_f in ((64, 4096), (192, 2048), (24, 3072)):
        m = rng.integers(128, 256, (out_f, in_f)).astype(np.float64)   # an 8-bit significand
        e = rng.integers(-9, -5, (out_f, in_f)).astype(np.float64)     # four exponents
        s = rng.choice([-1.0, 1.0], (out_f, in_f))
        w = torch.from_numpy(s * m * 2.0 ** e).to(torch.bfloat16).cuda()
        plan = MV._plan_of(w)
        assert plan.matmul_ok(0, in_f), "these weights must give fused chunks, or the case tests nothing"
        for nt in (1, 8, 9, 16, 17, 33, 64):
            x = torch.from_numpy(rng.integers(-1, 2, (nt, in_f)).astype(np.float32)).to(torch.bfloat16).cuda()
            y = plan.matmul(0, x)
            want = (x.double() @ w.double().T).to(torch.bfloat16)   # sums of at most 4096 * 255 * 2^3 units: exact in fp32
            assert torch.equal(y, want), (out_f, in_f, nt)
        plan.check()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_general_cases(dtype):
    shapes = [(o, i) for o, i in MV.SHAPES if o * i * 2 <= 8 << 20] + [(3, 49152)]
    for k, (out_f, in_f) in enumerate(shapes):
        w = MV._gauss((out_f, in_f), dtype, 200 + k)
        plan = MV._plan_of(w)
        assert plan.matmul_ok(0, in_f), (out_f, in_f)
        L = MMH.Layout(out_f, in_f)
        for nt in ROWS:
            assert plan.matmul_scratch_bytes(0, in_f, nt) == L.slots() * nt * 4, "the layout the host test checks"
            bias = MV._gauss((out_f,), dtype, 7 * k + nt, std=0.5) if (k + nt) % 2 else None
            strided = nt % 3 == 0
            xbuf = MV._gauss((nt, in_f + (16 if strided else 0)), dtype, 1000 * k + nt, std=1.0)
            x = xbuf[:, 8: 8 + in_f] if strided else xbuf
            ybuf = torch.full((nt + 2, out_f + 6), float("nan"), dtype=dtype, device="cuda")
            y = ybuf[1: nt + 1, 3: 3 + out_f] if strided else None
            need = plan.matmul_scratch_bytes(0, in_f, nt)
            sbuf = torch.full((256 + need + 256,), MV.CANARY, dtype=torch.uint8, device="cuda")
            off = -sbuf.data_ptr() % 256
            before = _native.launch_count()
            got = plan.matmul(0, x, bias=bias, out=y, scratch=sbuf[off: off + need])
            assert _native.launch_count() - before == 2, "two launches whatever the shape and row count"
            _check(got, x, w, bias, (dtype, out_f, in_f, nt))
            if strided:
                mask = torch.ones_like(ybuf, dtype=torch.bool)
                mask[1: nt + 1, 3: 3 + out_f] = False
                assert torch.all(torch.isnan(ybuf[mask])), "wrote outside y"
            assert torch.all(sbuf[:off] == MV.CANARY) and torch.all(sbuf[off + need:] == MV.CANARY), "wrote outside the scratch"
            again = plan.matmul(0, x, bias=bias)
            assert torch.equal(got.contiguous().view(torch.uint8), again.view(torch.uint8)), "two calls, two results"
        plan.check()


def test_shapes_of_x_and_no_rows():
    w = MV._gauss((64, 4096), torch.bfloat16, 3)
    plan = MV._plan_of(w)
    x = MV._gauss((4, 5, 4096), torch.bfloat16, 4, std=1.0)
    y = plan.matmul(0, x)
    assert y.shape == (4, 5, 64)
    _check(y, x, w, None, "3-D x")
    before = _native.launch_count()
    assert plan.matmul(0, x[:0]).shape == (0, 5, 64) and _native.launch_count() == before, "no rows, no launch"
    with pytest.raises(ValueError):
        plan.matmul(0, MV._gauss((65, 4096), torch.bfloat16, 6))
    with pytest.raises(ValueError):
        plan.matmul(0, x.float())
    assert not plan.matmul_ok(0, 4100) and not plan.matmul_ok(0, 4) and plan.matmul_ok(0, 8)
    f32 = MV._plan_of(MV._gauss((64, 1024), torch.float32, 5))
    assert f32.matvec_ok(0, 1024) and not f32.matmul_ok(0, 1024), "fp32 weights: the matvec, not the matmul"
    plan.check()


def test_graph_replay_with_new_x():
    w = MV._gauss((512, 1024), torch.bfloat16, 8)
    plan = MV._plan_of(w)
    x = torch.zeros(40, 1024, dtype=torch.bfloat16, device="cuda")
    out = torch.empty(40, 512, dtype=torch.bfloat16, device="cuda")
    scratch = torch.empty(plan.matmul_scratch_bytes(0, 1024, 40), dtype=torch.uint8, device="cuda")
    plan.matmul(0, x, out=out, scratch=scratch)   # (the first call for an output synchronises: not capturable)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.matmul(0, x, out=out, scratch=scratch)
    for seed in range(3):
        new = MV._gauss((40, 1024), torch.bfloat16, 20 + seed, std=1.0)
        x.copy_(new)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, plan.matmul(0, new)), seed
    plan.check()


def test_host_rejections_write_nothing(monkeypatch):
    L = _native.lib()
    w = MV._gauss((64, 4096), torch.bfloat16, 9)
    plan = MV._plan_of(w)
    need = plan.matmul_scratch_bytes(0, 4096, 2)
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    x = MV._gauss((2, 4096), torch.bfloat16, 10)
    y = torch.full((2, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    bad = [("rows", dict(nt=MATMUL_MAX_TOKENS + 1), A), ("dtype", dict(dtype=3), A), ("in 0", dict(inf=0), A),
           ("in not dividing", dict(inf=4104), A), ("item -1", dict(item=-1), A), ("item 1", dict(item=1), A),
           ("null x", dict(x=None), A), ("null y", dict(y=None), A), ("null scratch", dict(scratch=None), A),
           ("x alignment", dict(x=x.data_ptr() + 2), A), ("x stride", dict(xs=4100), A), ("short x stride", dict(xs=2048), A),
           ("short y stride", dict(ys=32), A), ("y alignment", dict(y=y.data_ptr() + 1), A), ("bias alignment", dict(bias=bias.data_ptr() + 1), A),
           ("scratch alignment", dict(scratch=scratch.data_ptr() + 16), A), ("short scratch", dict(sb=need - 1), A),
           ("fp32", dict(dtype=2, inf=2048), U), ("rows of 8 bytes", dict(inf=4), U)]
    for name, kw, want in bad:
        a = dict(item=0, dtype=0, inf=4096, x=x.data_ptr(), xs=4096, nt=2, bias=bias.data_ptr(), y=y.data_ptr(), ys=64,
                 scratch=scratch.data_ptr(), sb=need)
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_matmul(plan._ref, a["item"], a["dtype"], a["inf"], a["x"], a["xs"], a["nt"], a["bias"], a["y"],
                                             a["ys"], a["scratch"], a["sb"], MV._st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    assert torch.all(torch.isnan(y))
    out = C.c_size_t(0)
    assert L.zipnn_b200_decode_plan_matmul_scratch_size(plan._ref, 0, 0, 4096, MATMUL_MAX_TOKENS + 1, C.byref(out)) == A
    assert L.zipnn_b200_decode_plan_matmul_scratch_size(plan._ref, 0, 0, 4096, 2, None) == A
    w32 = MV._gauss((64, 1024), torch.float32, 11)
    f32 = MV._plan_of(w32)
    assert L.zipnn_b200_decode_plan_matmul_scratch_size(f32._ref, 0, 2, 1024, 2, C.byref(out)) == U
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matmul(f32._ref, 0, 2, 1024, x.data_ptr(), 1024, 2, None, y.data_ptr(), 64, scratch.data_ptr(), need,
                                           MV._st()) == U
    assert _native.launch_count() == before and torch.all(torch.isnan(y))
    assert torch.equal(f32.run()[0], w32), "an fp32 plan still decodes"
    f32.check()
    # a plan without a segment index
    DP._set_env(monkeypatch, {"ZIPNN_B200_PLAN_REPLAY": "0"})
    q = MV._plan_of(w)
    assert not q.matmul_ok(0, 4096)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matmul(q._ref, 0, 0, 4096, x.data_ptr(), 4096, 2, None, y.data_ptr(), 64, scratch.data_ptr(), need,
                                           MV._st()) == U
    assert _native.launch_count() == before and torch.all(torch.isnan(y))
    assert torch.equal(plan.run()[0], w), "the plan still decodes"


def _refused(pl, item, in_bytes, what):
    L = _native.lib()
    inf = in_bytes // 2
    x = torch.zeros(16, inf, dtype=torch.bfloat16, device="cuda")
    y = torch.full((16 * (pl.items[item].orig // in_bytes) * 2,), MV.CANARY, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(4 << 20, dtype=torch.uint8, device="cuda")
    out = C.c_size_t(0)
    before = _native.launch_count()
    assert L.zipnn_b200_decode_plan_matmul_scratch_size(C.byref(pl.plan), item, 0, inf, 16, C.byref(out)) == _native.E_UNSUPPORTED, what
    rc = L.zipnn_b200_decode_plan_matmul(C.byref(pl.plan), item, 0, inf, x.data_ptr(), inf, 16, None, y.data_ptr(),
                                         pl.items[item].orig // in_bytes, scratch.data_ptr(), scratch.numel(), MV._st())
    assert rc == _native.E_UNSUPPORTED and _native.launch_count() == before, (what, rc)
    assert torch.all(y == MV.CANARY), what


def test_items_with_other_chunk_modes_boxes_and_split_items_are_unsupported(monkeypatch):
    DP._set_env(monkeypatch, {})
    dt = MV.H.DTYPE[2]
    second = lambda c, g: "geo5" if g == 0 and c % 4 == 1 else "raw"  # noqa: E731  a second coded plane: general
    mixed = D.planes_case("mm_mixed", dt, 4096, ["geo5"] * 16, seed=800, side=second)
    assert set(mixed.pr["mode"]) == {"fused", "general"}
    plain = D.planes_case("mm_plain", dt, 4096, ["geo5"] * 7 + ["const"], seed=830)
    assert plain.pr["mode"] == ["fused"] * 7 + ["plain"], "a constant (RLE) last chunk"
    for case, in_bytes in ((mixed, 512), (plain, 1024)):
        pl = MV._raw_plan(case)
        assert pl.rc == 0
        _refused(pl, 0, in_bytes, case.name)
        MV._decodes(pl, case.name)
    good = D.planes_case("mm_fused", dt, 4096, ["geo5"] * 8, seed=840)
    assert good.pr["mode"] == ["fused"] * 8
    boxed = MV._raw_plan(good, box=(0, 2, 8192, 4096))
    assert boxed.rc == 0
    _refused(boxed, 0, 512, "a box")
    MV._decodes(boxed, "a box")
    DP._set_env(monkeypatch, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "5"})
    split = MV._raw_plan(good)
    assert split.rc == 0
    _refused(split, 0, 512, "a split item")
    MV._decodes(split, "a split item")
    const = MV._plan_of(torch.full((256, 256), 2.0 ** -6, dtype=torch.bfloat16, device="cuda"))
    assert not const.matmul_ok(0, 256)


@pytest.mark.parametrize("matvec", (0, 8))
@pytest.mark.parametrize("how", ("compress", "load"))
def test_resident_model(how, matvec, tmp_path):
    dtype = torch.bfloat16
    dense = MV._model(False, dtype)
    params = {n: p.detach().clone() for n, p in dense.named_parameters()}
    ids = torch.randint(0, 1000, (65,), device="cuda", generator=torch.Generator("cuda").manual_seed(13))
    plain = MV._model(False, dtype)
    compress_module(plain)
    f0, f1 = os.path.join(tmp_path, "plain.znn.safetensors"), os.path.join(tmp_path, "matmul.znn.safetensors")
    save_module(plain, f0)
    if how == "compress":
        model = MV._model(False, dtype)
        rep = compress_module(model, matvec=matvec, matmul=MATMUL_MAX_TOKENS)
    else:
        with torch.device("meta"):
            model = MV.Llamaish(False).to(dtype).eval()
        rep = load_module(model, f0, matvec=matvec, matmul=MATMUL_MAX_TOKENS)
    assert rep["matmul_modules"] == 8 and rep["matmul_scratch_bytes"] > 0
    assert ("matvec_modules" in rep) == bool(matvec)
    assert "forward" not in model.const.__dict__ and "forward" in model.head.__dict__
    with torch.no_grad():
        for t in (9, 16, 33, 64):
            want = dense(ids[:t]).double()
            got = model(ids[:t]).double()
            assert (got - want).abs().max() <= 4e-2 * want.abs().max(), (t, float((got - want).abs().max()))
        before = _native.launch_count()
        model.head(MV._gauss((16, 256), dtype, 14, std=1.0))
        assert _native.launch_count() - before == 2, "a matmul module decodes nothing for an input in range"
        assert torch.equal(model(ids), plain(ids)), "65 rows: the decode path, bit for bit"
    save_module(model, f1)
    with open(f0, "rb") as a, open(f1, "rb") as b:
        assert a.read() == b.read(), "the saved file does not depend on matmul"
    decompress_module(model)
    assert "forward" not in model.head.__dict__
    got = dict(model.named_parameters())
    assert set(got) == set(params)
    for n, p in params.items():
        assert torch.equal(got[n], p), n


def test_fp32_model_decodes():
    dense = MV._model(False, torch.float32)
    model = MV._model(False, torch.float32)
    plain = MV._model(False, torch.float32)
    compress_module(plain)
    rep = compress_module(model, matvec=8, matmul=MATMUL_MAX_TOKENS)
    assert rep["matmul_modules"] == 0 and rep["matvec_modules"] == 8
    ids = torch.randint(0, 1000, (16,), device="cuda", generator=torch.Generator("cuda").manual_seed(15))
    with torch.no_grad():
        assert torch.equal(model(ids), plain(ids)), "fp32 weights at 16 rows: the decode path, bit for bit"
        assert torch.equal(model(ids), dense(ids))
