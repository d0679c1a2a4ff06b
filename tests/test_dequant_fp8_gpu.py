"""The fp8 dequantize (zipnn_b200_decode_plan_dequant_fp8, DecodePlan.dequant_fp8) and the fp8 module mode
(compress_module / load_module with fp8=True).

  * every case of the fp8 corpus of tests/fp8_streams.py, both formats, bf16 and fp16 out, the scale layouts per
    tensor, per row, 128x128 with ragged edges and bk = 16, bit for bit against the numpy model of
    test_dequant_fp8_host.py (NaN positions aside), out between guard bytes poisoned with two values;
  * multi-item plans interleaved with runs, matvec_fp8 and gathers; a captured graph replayed with a new scale; two
    launches per call; every host rejection with no launch; the corrupted fp8 streams of corrupt_streams.py;
  * transformers' tiny Llama with every linear an FP8Linear, resident through compress_module and load_module (from
    .safetensors and from the .znn.safetensors save_module writes), against a reference copy whose FP8Linear forward
    is torch's dequantize + F.linear: bit for bit over 8 rows, within the fp64 bound at 1 and 8 rows.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as TF
from safetensors.torch import save_file

import corrupt_streams as CS
import fp8_streams as F
from test_dequant_fp8_host import model as dq_model
from test_dequant_fp8_host import same_bits as dq_same_bits
from test_product_streams_gpu import _st, raw_plan
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200 import resident as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _release_cached_memory():
    """This module builds whole models and captures F.linear in CUDA graphs, which gives the capture stream cuBLAS
    workspaces of its own that torch keeps for the life of the process.  Once it is done, those workspaces and the
    allocator's cached blocks are released, so that it leaves no long-lived blocks behind: between them a later test
    that accounts device memory can be handed a free block larger than it asked for, not split, counted as
    allocated."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch._C._cuda_clearCublasWorkspaces()
    torch.cuda.empty_cache()

LAYOUT_NAMES = ("tensor", "row", "block128", "bk16")
ODT = {"bf16": (torch.bfloat16, 0), "fp16": (torch.float16, 1)}   # ZIPNN_B200_MATVEC_BF16 / _FP16
GUARD = 64


def call(p_ref, item, fmt, odt, inn, scale, bn, bk, out_ptr):
    """One raw call: asserts success and two launches."""
    before = _native.launch_count()
    rc = _native.lib().zipnn_b200_decode_plan_dequant_fp8(p_ref, item, F.CODE[fmt], ODT[odt][1], inn, scale.data_ptr(), bn, bk, out_ptr, _st())
    assert rc == 0 and _native.launch_count() - before == 2, (item, rc)


def expanded(s: np.ndarray, out: int, inn: int, bn: int, bk: int) -> np.ndarray:
    return np.repeat(np.repeat(s, bn, 0)[:out], bk, 1)[:, :inn]


def check_case(p_ref, item, case, odt, layout, seed, scales=None):
    """The dequantize of one item into a buffer with guards, poisoned with 0x00 and then 0xFF: exactly [out, in] is
    written, bit for bit the model's."""
    bn, bk = F.layouts(case.out, case.inn)[layout]
    s = F.random_scales(case.out, case.inn, bn, bk, seed) if scales is None else scales
    sd = torch.from_numpy(s).cuda()
    n = case.out * case.inn
    want = dq_model(case.data.reshape(case.out, case.inn), case.dtype, expanded(s, case.out, case.inn, bn, bk), odt)
    for poison in (0x00, 0xFF):
        buf = torch.full((2 * GUARD + 2 * n,), poison, dtype=torch.uint8, device="cuda")
        call(p_ref, item, case.dtype, odt, case.inn, sd, bn, bk, buf.data_ptr() + GUARD)
        host = buf.cpu().numpy()
        assert np.all(host[:GUARD] == poison) and np.all(host[GUARD + 2 * n:] == poison), (case.name, "wrote outside out")
        got = host[GUARD: GUARD + 2 * n].view(np.uint16).reshape(case.out, case.inn)
        ok = dq_same_bits(got, want, odt)
        assert ok.all(), (case.name, odt, layout, tuple(np.argwhere(~ok)[0]))


@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_shapes_at_every_chunk_size(chunk):
    cases = F.shape_cases(chunk)
    p = raw_plan(cases)
    k0 = F.CHUNKS.index(chunk)
    for i, case in enumerate(cases):
        check_case(C.byref(p.plan), i, case, ("bf16", "fp16")[(i + k0) % 2], LAYOUT_NAMES[(i + k0 // 2) % 4], 100 * k0 + i)
    for it in p.items:
        it.check("after the dequantizes")   # (the outputs hold what create decoded: no dequantize wrote them)
    assert p.status() == 0


def test_stream_kinds():
    for j, case in enumerate(F.stream_cases()):
        p = raw_plan([case])
        for odt in ("bf16", "fp16"):
            check_case(C.byref(p.plan), 0, case, odt, LAYOUT_NAMES[(j + (odt == "fp16")) % 4], j)
        p.items[0].scribble()
        assert p.run() == 0 and p.status() == 0
        p.items[0].check("run after the dequantizes")


@pytest.mark.parametrize("fmt", F.FORMATS)
def test_special_values(fmt):
    """NaN, infinities, -0 and subnormal weights, times scales that overflow fp16, give fp16 / bf16 subnormals, fp32
    subnormals, and are negative."""
    case, _ = F.special_case(fmt)
    p = raw_plan([case])
    for odt in ("bf16", "fp16"):
        for v in (0.25, 2.0 ** 12, 2.0 ** -20, 2.0 ** -130, 2.0 ** -149, -3.0):
            check_case(C.byref(p.plan), 0, case, odt, "tensor", 0, scales=np.full((1, 1), v, dtype=np.float32))
        rng = np.random.default_rng(3)
        s = (rng.uniform(0.5, 2.0, (22, 32)) * 2.0 ** rng.integers(-140, 12, (22, 32))).astype(np.float32)
        check_case(C.byref(p.plan), 0, case, odt, "bk16", 0, scales=s)   # (bk16 of [64, 512]: (3, 16), a [22, 32] grid)
    assert p.status() == 0


# ------------------------------------------------------------------ the public API
def _quantized(fmt, out, inn, seed, block=(128, 128)):
    """bf16 Gaussian weights (std 0.02) quantized per block at amax / fp8 max -> (W fp8, fp32 scale) on the GPU;
    block None: one scale, a 0-d tensor."""
    g = torch.Generator("cuda").manual_seed(seed)
    w = (torch.randn(out, inn, generator=g, device="cuda") * 0.02).to(torch.bfloat16).float()
    top = float(torch.finfo(F.TORCH[fmt]).max)
    if block is None:
        scale = (w.abs().max() / top).clamp_min(2.0 ** -30)
        return (w / scale).to(F.TORCH[fmt]), scale.contiguous()
    bn, bk = block
    gr, gc = F.grid_shape(out, inn, bn, bk)
    pad = torch.zeros(gr * bn, gc * bk, device="cuda")
    pad[:out, :inn] = w.abs()
    scale = (pad.view(gr, bn, gc, bk).amax(dim=(1, 3)) / top).clamp_min(2.0 ** -30).contiguous()
    full = scale.repeat_interleave(bn, 0)[:out].repeat_interleave(bk, 1)[:, :inn]
    return (w / full).to(F.TORCH[fmt]), scale


def torch_dequant(wq, scale, block, dtype):
    """The reference: (W.to(float32) * S_expanded).to(dtype)."""
    if block is None:
        return (wq.to(torch.float32) * scale.reshape(())).to(dtype)
    out, inn = wq.shape
    s = scale.repeat_interleave(block[0], 0)[:out].repeat_interleave(block[1], 1)[:, :inn]
    return (wq.to(torch.float32) * s).to(dtype)


def bits(t):
    return t.view(torch.int16)


def test_api_multi_item_plan_interleaved_with_runs_matvecs_and_gathers():
    ws = [_quantized("e4m3", 256, 1024, 1), _quantized("e5m2", 96, 528, 2), _quantized("e4m3", 1, 4096, 3)]
    other = (torch.randn(64, 512, device="cuda") * 0.02).to(torch.bfloat16)
    tensors = [ws[0][0], other, ws[1][0], ws[2][0]]
    streams = [ZipNN(input_format="torch", compression_chunk=ch).compress(t) for t, ch in zip(tensors, (65536, 262144, 131072, 131072))]
    plan = DecodePlan(streams)
    with pytest.raises(ValueError):
        plan.dequant_fp8(1, 512, torch.ones(1, device="cuda"))
    ids = torch.tensor([3, 0, 200, 255], device="cuda")
    for r in range(2):
        for k, (wq, scale) in zip((0, 2, 3), ws):
            inn = wq.shape[1]
            for dt in (torch.bfloat16, torch.float16):
                before = _native.launch_count()
                got = plan.dequant_fp8(k, inn, scale, (128, 128), dtype=dt)
                assert _native.launch_count() - before == 2
                assert got.shape == wq.shape and got.dtype == dt
                assert torch.equal(bits(got), bits(torch_dequant(wq, scale, (128, 128), dt))), (r, k, dt)
            y = plan.matvec_fp8(k, torch.randn(3, inn, device="cuda").to(torch.bfloat16), scale, (128, 128))
            assert torch.isfinite(y).all()
            outs = plan.run()
            torch.cuda.synchronize()
            for o, t in zip(outs, tensors):
                assert torch.equal(o.view(torch.uint8), t.view(torch.uint8)), (r, k)
        assert torch.equal(plan.gather(0, ids).view(torch.uint8), ws[0][0][ids].view(torch.uint8))
    # per tensor, per row, an out of the caller's, and without the plan's output buffer
    wq, scale = ws[0]
    one = torch.tensor(0.001, device="cuda")
    assert torch.equal(bits(plan.dequant_fp8(0, 1024, one)), bits(torch_dequant(wq, one, None, torch.bfloat16)))
    rows = torch.rand(256, device="cuda") * 0.01
    assert torch.equal(bits(plan.dequant_fp8(0, 1024, rows, (1, 1024), torch.float16)),
                       bits((wq.float() * rows[:, None]).to(torch.float16)))
    out = torch.empty(256, 1024, dtype=torch.bfloat16, device="cuda")
    plan.release_out()
    assert plan.dequant_fp8(0, 1024, scale, (128, 128), out=out) is out
    assert torch.equal(bits(out), bits(torch_dequant(wq, scale, (128, 128), torch.bfloat16)))
    plan.check()


def test_graph_capture_replays_with_a_new_scale():
    wq, scale = _quantized("e4m3", 512, 2048, 11)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    out = torch.empty(512, 2048, dtype=torch.bfloat16, device="cuda")
    s = scale.clone()
    plan.dequant_fp8(0, 2048, s, (128, 128), out=out)   # first call outside: it reads the chunk modes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.dequant_fp8(0, 2048, s, (128, 128), out=out)
    for r in range(3):
        s.copy_(scale * (r + 1.5))
        out.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(out), bits(torch_dequant(wq, s, (128, 128), torch.bfloat16))), r
    plan.check()


def test_host_rejections_launch_nothing():
    L = _native.lib()
    wq, scale = _quantized("e4m3", 64, 4096, 9)
    plan = DecodePlan([ZipNN(input_format="torch").compress(wq)])
    out = torch.full((64, 4096), float("nan"), dtype=torch.bfloat16, device="cuda")
    A, U = _native.E_ARG, _native.E_UNSUPPORTED
    bad = [("format", dict(fmt=2), A), ("format -1", dict(fmt=-1), A), ("out dtype fp32", dict(odt=2), A), ("out dtype 3", dict(odt=3), A),
           ("out dtype -1", dict(odt=-1), A), ("in 0", dict(inf=0), A), ("in not dividing", dict(inf=4112), A), ("item -1", dict(item=-1), A),
           ("item 1", dict(item=1), A), ("null out", dict(out=None), A), ("out alignment 8", dict(out=out.data_ptr() + 8), A),
           ("out alignment 2", dict(out=out.data_ptr() + 2), A), ("null scale", dict(scale=None), A),
           ("scale alignment", dict(scale=scale.data_ptr() + 2), A), ("block rows 0", dict(bn=0), A), ("block cols 0", dict(bk=0), A),
           ("block cols 8", dict(bk=8), A), ("block cols 140", dict(bk=140), A), ("null plan", dict(plan=None), A),
           ("rows of 8 bytes", dict(inf=8), U)]
    for name, kw, want in bad:
        a = dict(plan=plan._ref, item=0, fmt=0, odt=0, inf=4096, scale=scale.data_ptr(), bn=128, bk=128, out=out.data_ptr())
        a.update(kw)
        before = _native.launch_count()
        rc = L.zipnn_b200_decode_plan_dequant_fp8(a["plan"], a["item"], a["fmt"], a["odt"], a["inf"], a["scale"], a["bn"], a["bk"], a["out"], _st())
        assert rc == want and _native.launch_count() == before, (name, rc)
    # a bf16 item, a plain (incompressible) fp8 item, and a plan without a segment index
    other = DecodePlan([ZipNN(input_format="torch").compress((torch.randn(64, 4096, device="cuda") * 0.02).to(torch.bfloat16))])
    raw = torch.randint(0, 256, (64 * 4096,), dtype=torch.uint8, device="cuda")
    raw[(raw & 0x7F) == 0x7F] = 0
    pl = DecodePlan([ZipNN(input_format="torch").compress(raw.view(torch.float8_e4m3fn).view(64, 4096))])
    for p_ in (other, pl):
        before = _native.launch_count()
        assert L.zipnn_b200_decode_plan_dequant_fp8(p_._ref, 0, 0, 0, 4096, scale.data_ptr(), 128, 128, out.data_ptr(), _st()) == U
        assert _native.launch_count() == before
    # Python-side refusals
    before = _native.launch_count()
    for kw, what in ((dict(block=None), "a grid scale without block"), (dict(block=(128, 8)), "bk 8"), (dict(block=(0, 128)), "bn 0"),
                     (dict(block=(32, 128)), "a grid of another block"), (dict(scale=scale.double()), "fp64 scale"),
                     (dict(scale=torch.ones(64, device="cuda")[::2]), "a non-contiguous scale"), (dict(dtype=torch.float32), "fp32 out"),
                     (dict(out=out.float()), "an fp32 out"), (dict(out=out[:, :2048]), "a non-contiguous out"),
                     (dict(out=out[:32]), "a wrong shape"), (dict(out=out.view(-1)), "a flat out"),
                     (dict(inf=4112), "in_features not dividing"), (dict(inf=8), "rows of 8 bytes")):
        a = dict(inf=4096, scale=scale, block=(128, 128), dtype=torch.bfloat16, out=None)
        a.update(kw)
        with pytest.raises(ValueError):
            plan.dequant_fp8(0, a["inf"], a["scale"], block=a["block"], dtype=a["dtype"], out=a["out"])
    misaligned = torch.empty(64 * 4096 + 8, dtype=torch.bfloat16, device="cuda")[4:4 + 64 * 4096].view(64, 4096)
    with pytest.raises(ValueError):
        plan.dequant_fp8(0, 4096, scale, (128, 128), out=misaligned)
    assert _native.launch_count() == before and torch.all(torch.isnan(out))


def test_corrupted_fp8_streams_are_refused():
    """Every mutant of the fp8 base of corrupt_streams.py: a plan whose create fails is refused by the dequantize (E_ARG,
    nothing launched), as by every other entry point; one that creates decodes to the verdict's bytes and is refused
    (E_UNSUPPORTED: its rows cannot be a multiple of 16 bytes and its last chunk is not fused), and `status` keeps the
    verdict's."""
    import test_corrupt_streams_gpu as T
    b = CS.bases()["fp8_g1"]
    assert b.pr["mode"][-1] != "fused"
    L = _native.lib()
    sc = torch.ones(1, device="cuda")
    y = torch.full((b.orig,), float("nan"), dtype=torch.bfloat16, device="cuda")
    out = torch.empty(T.PAD + b.orig + T.PAD, dtype=torch.uint8, device="cuda")
    n = 0
    for m, v in T.cases("fp8_g1"):
        body = torch.from_numpy(m.body).cuda()
        out.fill_(T.CANARY)
        rc, plan, keep = T._plan_create(b, body.data_ptr(), m.body.size, out[T.PAD:])
        assert rc == T.STATUS[v.status], (m.id, rc, v.status)
        p = C.byref(plan)
        before = _native.launch_count()
        for inf in (8, 16):
            got = L.zipnn_b200_decode_plan_dequant_fp8(p, 0, 0, 0, inf, sc.data_ptr(), 1, 16, y.data_ptr(), _st())
            assert got in ((_native.E_ARG,) if rc else (_native.E_ARG, _native.E_UNSUPPORTED)), (m.id, got)
        assert _native.launch_count() == before, m.id
        if not rc:
            assert torch.equal(out[T.PAD: T.PAD + b.orig], torch.from_numpy(v.data).cuda()), m.id
            assert L.zipnn_b200_decode_plan_status(p, _st()) == 0, m.id
            n += 1
    assert torch.all(torch.isnan(y))
    assert n > 0


# ------------------------------------------------------------------ resident fp8 models
def _config():
    import transformers
    return transformers.LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                    num_key_value_heads=2, head_dim=64, vocab_size=512)


def tiny_fp8_llama(seed=0, constant=False):
    """transformers' tiny Llama on the GPU, bf16, every linear an FP8Linear with 128x128 blocks but layers[0]'s o_proj,
    per tensor; layers[1]'s up_proj has an fp32 bias.  constant=True: layers[1]'s down_proj weight is one value (its
    stream holds no coded bitstream, so matvec_fp8_ok refuses it)."""
    import transformers
    from transformers.integrations.finegrained_fp8 import replace_with_fp8_linear
    torch.manual_seed(seed)
    m = transformers.LlamaForCausalLM(_config()).to(torch.bfloat16)
    m = replace_with_fp8_linear(m, quantization_config=transformers.FineGrainedFP8Config(weight_block_size=(128, 128)), pre_quantized=True)
    for i, (name, mod) in enumerate([(n, x) for n, x in m.named_modules() if type(x).__name__ == "FP8Linear"]):   # (on meta)
        block = None if name == "model.layers.0.self_attn.o_proj" else (128, 128)
        wq, scale = _quantized("e4m3", mod.out_features, mod.in_features, 100 * seed + i, block)
        if constant and name == "model.layers.1.mlp.down_proj":
            wq = torch.full_like(wq, 0.5)
        mod.block_size = block
        mod.weight = torch.nn.Parameter(wq, requires_grad=False)
        mod.weight_scale_inv = torch.nn.Parameter(scale, requires_grad=False)
        if name == "model.layers.1.mlp.up_proj":
            mod.bias = torch.nn.Parameter(torch.randn(mod.out_features, device="cuda") * 0.01)
    m = m.cuda().eval()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def reference(m):
    """A copy of `m` whose FP8Linear forward is torch's dequantize + F.linear, the bias added as FP8Linear adds it."""
    ref = copy.deepcopy(m)

    def fwd(mod):
        def forward(x):
            y = TF.linear(x, torch_dequant(mod.weight, mod.weight_scale_inv, mod.block_size, x.dtype))
            return y if mod.bias is None else (y + mod.bias).to(x.dtype)
        return forward
    for mod in ref.modules():
        if type(mod).__name__ == "FP8Linear":
            mod.forward = fwd(mod)
    return ref


def lin_io(m):
    """Forward hooks that record every FP8Linear's (input, output) in call order -> (the list, the handles)."""
    rec, hs = [], []
    for mod in m.modules():
        if type(mod).__name__ == "FP8Linear":
            hs.append(mod.register_forward_hook(lambda mod, a, out: rec.append((mod, a[0].clone(), out.clone()))))
    return rec, hs


def within_fp64_bound(y, x, mod):
    """matvec_fp8's bound against fp64 (test_matvec_fp8_gpu._check64), for any block."""
    wd = torch_dequant(mod.weight, mod.weight_scale_inv, mod.block_size, torch.float64)
    x64 = x.double().reshape(-1, x.shape[-1])
    ref, mag = x64 @ wd.T, x64.abs() @ wd.abs().T
    if mod.bias is not None:
        ref = ref + mod.bias.double()
    bound = (x.shape[-1] + 2) * 2.0 ** -24 * mag
    rel = 2.0 ** -8 if y.dtype == torch.bfloat16 else 2.0 ** -11
    if mod.bias is None:
        tol = bound + (ref.abs() + bound) * rel
    else:   # the product is rounded once, then the sum with the bias once more
        t1 = bound + ((ref - mod.bias.double()).abs() + bound) * rel
        tol = t1 + (ref.abs() + t1) * rel
    return bool(torch.all((y.double().reshape(ref.shape) - ref).abs() <= tol))


def check_against_reference(m, ref, seed):
    """Over 8 rows every FP8Linear output and the logits equal the reference's bits; at 1 and 8 rows every output is
    within the fp64 bound of the product with the dequantized weight."""
    g = torch.Generator("cuda").manual_seed(seed)
    with torch.no_grad():
        for rows in (1, 8, 9, 64, 300):
            ids = torch.randint(0, 512, (1, rows), generator=g, device="cuda")
            got_rec, h1 = lin_io(m)
            want_rec, h2 = lin_io(ref)
            got = m(ids, use_cache=False).logits
            want = ref(ids, use_cache=False).logits
            for h in h1 + h2:
                h.remove()
            assert len(got_rec) == len(want_rec) == 15
            if rows > 8:
                assert torch.equal(bits(got), bits(want)), rows
                for (_, _, a), (_, _, b) in zip(got_rec, want_rec):
                    assert torch.equal(bits(a), bits(b)), rows
            else:   # matvec_fp8 within the bound; the fallback is the reference's forward on the same input
                fast = {id(x): mode == "fp8" for x, _, _, mode in getattr(m, R._ATTR).entries if mode in ("fp8", "fp8_torch")}
                for mod, x, y in got_rec:
                    r = _ref_of(ref, m, mod)
                    if fast[id(mod)]:
                        assert within_fp64_bound(y, x, r), (rows, type(r).__name__)
                    else:
                        assert torch.equal(bits(y), bits(r(x))), rows


def _ref_of(ref, m, mod):
    """The reference's module at `mod`'s name."""
    name = next(n for n, x in m.named_modules() if x is mod)
    return ref.get_submodule(name)


def raw(t):
    return t.reshape(-1).view(torch.uint8)


def dense_state(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def check_resident(m, ref, report, seed):
    lins = [x for x in m.modules() if type(x).__name__ == "FP8Linear"]
    assert report["fp8_modules"] == len(lins) == 15
    assert report["out_bytes"] >= 2 * max(x.out_features * x.in_features for x in lins)
    assert report["fp8_scratch_bytes"] > 0
    for x in lins:   # only the weight is compressed
        assert "weight" not in x._parameters and "weight_scale_inv" in x._parameters
    check_against_reference(m, ref, seed)


def test_compress_module_fp8_against_the_reference():
    m = tiny_fp8_llama(1, constant=True)
    ref = reference(m)
    before = dense_state(m)
    report = compress_module(m, fp8=True, matvec=8)
    state = getattr(m, R._ATTR)
    fast = {id(x): mode == "fp8" for x, _, _, mode in state.entries if mode in ("fp8", "fp8_torch")}
    down = m.model.layers[1].mlp.down_proj
    assert fast[id(down)] is False and sum(fast.values()) == 14, "the constant weight takes the fallback"
    assert report["out_bytes"] == 2 * 512 * 256   # (twice the largest fp8 weight; the bf16 embedding decodes to as many)
    check_resident(m, ref, report, 2)
    # one captured forward per path (matvec_fp8, dequant_fp8 + F.linear, the fallback), replayed with new inputs
    with torch.no_grad():
        for mod, rows in ((m.model.layers[1].mlp.up_proj, 8), (m.model.layers[1].mlp.up_proj, 64), (down, 8), (down, 64),
                          (m.model.layers[0].self_attn.o_proj, 9)):
            x = torch.randn(rows, mod.in_features, device="cuda").to(torch.bfloat16)
            mod(x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y = mod(x)
            for r in range(2):
                x.copy_(torch.randn(rows, mod.in_features, device="cuda").to(torch.bfloat16))
                g.replay()
                torch.cuda.synchronize()
                assert torch.equal(bits(y), bits(mod(x))), (rows, r)
    decompress_module(m)
    after = dense_state(m)
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(raw(after[k]), raw(before[k])), k


def test_load_module_fp8_from_safetensors_and_znn(tmp_path):
    src = tiny_fp8_llama(3)
    ref = reference(src)
    sd = {k: v.contiguous() for k, v in dense_state(src).items()}
    plain = str(tmp_path / "fp8.safetensors")
    save_file(sd, plain)
    a = tiny_fp8_llama(4)   # other values: every one must come from the file
    report = load_module(a, plain, fp8=True, matvec=8)
    check_resident(a, ref, report, 5)
    znn = str(tmp_path / "fp8.znn.safetensors")
    save_module(a, znn)
    b = tiny_fp8_llama(5)
    report = load_module(b, znn, fp8=True, matvec=8)
    check_resident(b, ref, report, 6)
    decompress_module(b)
    for k, v in dense_state(b).items():
        assert torch.equal(raw(v), raw(sd[k])), k
