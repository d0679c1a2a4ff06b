"""Selected plan runs (zipnn_b200_decode_plan_run_select, DecodePlan.run_select) and experts=True against the dense
bytes, on an H100.

Plan level: every output is poisoned (guard bytes on both sides included) with two different poison bytes in turn, then
a selected run must write exactly the chunks test_select_host.touched_chunks names, with the dense bytes, and leave
every other byte poisoned.  Streams: the plain, general and overflow chunks of test_boxes_host.box_streams (fp8, bf16,
fp16, fp32), the fused streams of every chunk size and the crafted tables of product_streams, and the multi-item
layouts of multi_item_plans; slices inside chunks, aligned with them and straddling them.  All ids give run()'s bytes;
duplicates, int32 / int64 and n = 0; bad ids raise from check() and select nothing; run_select interleaved with run,
gather and matvec on one shared scratch; a captured graph replayed with new ids; a fixed launch count; rejections.

Module level: a MoE block (top-k router + experts module in the transformers convention, expert slices straddling
256 KiB chunks) under compress_module / load_module(experts=True) equals the dense block bit for bit, with the shared
output buffer filled with NaN before every forward; decompress_module / save_module round trips; the grad-mode error.
With transformers: tiny Mixtral and Qwen3-MoE logits under the eager, batched_mm and grouped_mm experts
implementations equal the dense model's.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import multi_item_plans as M
import product_streams as PS
import test_boxes_host as H
import test_decode_plan_gpu as DP
import test_gather_gpu as GG
from test_select_host import written_bytes
from zipnn_b200 import DecodePlan, ZipNN, _native, compress_module, decompress_module, load_module, save_module
from zipnn_b200.resident import _ATTR

pytestmark = pytest.mark.gpu

PAD = DP.PAD
POISONS = (0xA5, 0x5A)
SELECT_LAUNCHES = 5   # index, replay decoder, regroup, overflow, error OR


def _st():
    return torch.cuda.current_stream().cuda_stream


def scratch_size(p, rows):
    out = C.c_size_t(0)
    rc = _native.lib().zipnn_b200_decode_plan_select_scratch_size(C.byref(p.plan), rows, C.byref(out))
    return rc, out.value


def run_select(p, rows, ids, scratch=None):
    rc, sb = scratch_size(p, rows)
    assert rc == 0, rc
    if scratch is None:
        scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
    return _native.lib().zipnn_b200_decode_plan_run_select(C.byref(p.plan), rows, ids.data_ptr(), ids.numel(), ids.element_size(),
                                                           scratch.data_ptr(), scratch.numel(), _st())


def check_selected(p, rows, ids, what, scratch=None):
    """Poison, select, compare: the touched chunks hold the dense bytes, every other byte the poison."""
    ids_host = ids.cpu().numpy().reshape(-1)
    for poison in POISONS:
        for it in p.items:
            it.out.fill_(poison)
        assert run_select(p, rows, ids, scratch) == 0
        for it in p.items:
            host = it.out.cpu().numpy()
            n = it.want.size
            assert np.all(host[:PAD] == poison) and np.all(host[PAD + n:] == poison), f"{it.name} {what}: wrote outside its output"
            body = host[PAD: PAD + n]
            wb = written_bytes(it.orig, it.chunk, rows, ids_host)
            bad = np.flatnonzero(body[wb] != it.want[wb])
            assert bad.size == 0, (it.name, what, "touched chunk byte differs", int(np.flatnonzero(wb)[bad[0]]))
            stray = np.flatnonzero(body[~wb] != poison)
            assert stray.size == 0, (it.name, what, "untouched byte written", int(np.flatnonzero(~wb)[stray[0]]))


def id_sets(rows, rng):
    return [np.array([0]), np.array([rows - 1]), np.array([rows - 1, 0, 0, rows - 1]),
            rng.integers(0, rows, 3), np.arange(rows)[::2].copy()]


def _ids(a, k):
    return torch.from_numpy(np.asarray(a)).to(torch.int32 if k % 2 else torch.int64).cuda()


def _case(G: int, prefix: str):
    return next(c for c in H.box_streams(G) if c.name.startswith(prefix + "_"))


def _item(case):
    return DP.Item(case.name, case.body, case.G, case.bits, case.chunk, case.data.size, case.data)


def rows_of(orig: int, chunk: int) -> list:
    """Slice counts: slices inside a chunk, about a chunk and straddling, spanning many chunks, and one slice."""
    return sorted({orig // R for R in GG.row_sizes(orig, chunk)} | {1})


@pytest.mark.parametrize("G", (1, 2, 4))
def test_box_streams_write_exactly_the_touched_chunks(G, monkeypatch):
    """Plain, general and overflow chunks (c64: 400 general chunks, past the 64 pool slots), fused ones, ragged
    last chunks; fp8, bf16, fp16 and fp32."""
    DP._set_env(monkeypatch, {})
    rng = np.random.default_rng(G)
    for case in H.box_streams(G):
        orig = case.data.size
        item = DP.Item(case.name, case.body, case.G, case.bits, case.chunk, orig, case.data)
        p = DP.Plan([item])
        assert p.rc == 0
        for rows in rows_of(orig, case.chunk):
            for k, ids in enumerate(id_sets(rows, rng)):
                check_selected(p, rows, _ids(ids, k), f"rows={rows} ids#{k}")
        assert p.status() == 0


def _stream_items():
    cases = []
    for chunk in PS.CHUNKS:
        sc = PS.shape_cases(chunk, ("bf16",))
        cases += [sc[0], sc[-1]]   # 48-byte rows (many per chunk) and a short last chunk
    return cases + PS.stream_cases(("bf16", "fp16", "fp32"))


def test_fused_streams_every_chunk_size_and_crafted_tables():
    rng = np.random.default_rng(7)
    for case in _stream_items():
        orig = case.data.size
        item = DP.Item(case.name, case.body, case.G, case.bits, case.chunk, orig, case.data)
        p = DP.Plan([item])
        assert p.rc == 0
        for rows in sorted({case.out, 1} | set(rows_of(orig, case.chunk)[:2])):
            ids = rng.integers(0, rows, 2).tolist() + [0, rows - 1]
            check_selected(p, rows, _ids(ids, rows), f"rows={rows}")
        assert p.status() == 0


def _layout_items(name):
    entries, env = M.layout(name)
    model = M.Model(entries, M.limit_of(env))
    keep = [e for i, e in enumerate(entries) if model.piece[i] >= 0 and e.orig]
    return keep, env


@pytest.mark.parametrize("name", M.LAYOUTS)
def test_multi_item_layouts(name, monkeypatch):
    keep, env = _layout_items(name)
    DP._set_env(monkeypatch, env)
    g = 0
    for e in keep:
        g = math.gcd(g, e.orig)
    items = [DP.Item(e.name, e.body, e.G, e.bits, e.chunk, e.orig, e.data) for e in keep]
    p = DP.Plan(items)
    assert p.rc == 0
    rng = np.random.default_rng(len(name))
    divs = [d for d in range(1, g + 1) if g % d == 0]
    for rows in sorted({1, divs[len(divs) // 2], g}):
        for k, ids in enumerate(id_sets(rows, rng)):
            check_selected(p, rows, _ids(ids, k), f"{name} rows={rows} ids#{k}")
    assert p.status() == 0


def test_all_ids_equal_run_and_n_zero_writes_nothing():
    case = _case(2, "c4096")   # fused, plain and general chunks, a ragged last chunk
    orig = case.data.size
    item = _item(case)
    p = DP.Plan([item])
    assert p.rc == 0
    assert p.run() == 0
    by_run = item.out.clone()
    for rows in rows_of(orig, case.chunk):
        item.out.fill_(POISONS[0])
        assert run_select(p, rows, _ids(np.arange(rows), rows)) == 0
        assert torch.equal(item.out[PAD: PAD + orig], by_run[PAD: PAD + orig]), rows
        assert bool((item.out[:PAD] == POISONS[0]).all()) and bool((item.out[PAD + orig:] == POISONS[0]).all())
    item.out.fill_(POISONS[1])
    before = _native.launch_count()
    assert run_select(p, 1, torch.zeros(0, dtype=torch.int64, device="cuda")) == 0
    assert _native.launch_count() == before
    assert bool((item.out == POISONS[1]).all())


def test_launch_count_does_not_depend_on_the_ids():
    case = _case(2, "c64")   # overflow chunks
    orig = case.data.size
    p = DP.Plan([_item(case)])
    rows = orig // GG.row_sizes(orig, case.chunk)[0]
    for ids in (np.zeros(9, np.int64), np.arange(9) * (rows // 9), np.array([rows - 1] * 9), np.array([-1] * 9)):
        before = _native.launch_count()
        assert run_select(p, rows, _ids(ids, 0)) == 0
        assert _native.launch_count() - before == SELECT_LAUNCHES


def test_bad_ids_raise_and_select_nothing():
    torch.manual_seed(3)
    w = (torch.randn(64, 300, 200, device="cuda") * 0.02).to(torch.bfloat16)
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    out = plan._out
    out.fill_(POISONS[0])
    ids = torch.tensor([[5, -1], [64, 9]], device="cuda")
    plan.run_select(ids)
    with pytest.raises(IndexError):
        plan.check()
    host = out[: plan.nbytes["dense"]].cpu().numpy()
    wb = written_bytes(w.numel() * 2, 262144, 64, [5, 9])
    dense = w.view(torch.uint8).reshape(-1).cpu().numpy()
    assert np.array_equal(host[wb], dense[wb]) and np.all(host[~wb] == POISONS[0])


def test_decode_plan_interleaved_with_run_gather_and_matvec_on_one_scratch():
    torch.manual_seed(4)
    E = 16
    ws = [(torch.randn(E, 96, 512, device="cuda") * 0.02).to(torch.bfloat16),
          (torch.randn(E, 512, 48, device="cuda") * 0.02).to(torch.bfloat16)]
    plan = DecodePlan([ZipNN(input_format="torch").compress(w) for w in ws])
    assert plan.select_ok()
    need = max(plan.select_scratch_bytes(), plan.gather_scratch_bytes(0, 4), plan.matvec_scratch_bytes(1, 48, 1))
    shared = torch.empty(need, dtype=torch.uint8, device="cuda")
    dense = [w.view(torch.uint8).reshape(E, -1) for w in ws]
    x = (torch.randn(1, 48, device="cuda")).to(torch.bfloat16)
    y0 = plan.matvec(1, x)   # on the plan's own matvec scratch: the same bits every time
    for step in range(6):
        ids = torch.randint(0, E, (3, 2), device="cuda", dtype=torch.int32 if step % 2 else torch.int64)
        outs = plan.run_select(ids, scratch=shared)
        sel = ids.reshape(-1).unique()
        for o, d in zip(outs, dense):
            assert torch.equal(o.view(torch.uint8).reshape(E, -1)[sel], d[sel]), step
        g = plan.gather(0, ids, scratch=shared)
        assert torch.equal(g.view(torch.uint8).reshape(-1, dense[0].shape[1]), dense[0][ids.reshape(-1).long()])
        assert torch.equal(plan.matvec(1, x, scratch=shared), y0)
        if step % 3 == 2:
            outs = plan.run()
            for o, d in zip(outs, dense):
                assert torch.equal(o.view(torch.uint8).reshape(E, -1), d)
    plan.check()


def test_graph_capture_replays_with_new_ids():
    torch.manual_seed(5)
    E = 32
    w = (torch.randn(E, 700, 300, device="cuda") * 0.02).to(torch.bfloat16)   # 420000-byte slices: straddling
    plan = DecodePlan([ZipNN(input_format="torch").compress(w)])
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    plan.run_select(ids)   # warm up (kernel attributes) outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run_select(ids)
    dense = w.view(torch.uint8).reshape(-1).cpu().numpy()
    for step in range(4):
        new = torch.randint(0, E, (4,), device="cuda")
        ids.copy_(new)
        plan._out.fill_(POISONS[step % 2])
        g.replay()
        torch.cuda.synchronize()
        host = plan._out[: dense.size].cpu().numpy()
        wb = written_bytes(dense.size, 262144, E, new.cpu().numpy())
        assert np.array_equal(host[wb], dense[wb]) and np.all(host[~wb] == POISONS[step % 2]), step
    plan.check()


def test_rejections_launch_nothing(monkeypatch):
    DP._set_env(monkeypatch, {})
    case = _case(2, "c4096")
    orig = case.data.size
    item = _item(case)
    p = DP.Plan([item])
    rows = orig // GG.row_sizes(orig, case.chunk)[0]
    rc, sb = scratch_size(p, rows)
    assert rc == 0
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    L = _native.lib()
    before = _native.launch_count()
    call = lambda r=rows, d=ids.data_ptr(), n=4, ib=8, s=scratch.data_ptr(), b=sb: L.zipnn_b200_decode_plan_run_select(  # noqa: E731
        C.byref(p.plan), r, d, n, ib, s, b, _st())
    assert call(r=orig + 1) == _native.E_ARG                  # rows does not divide
    assert call(r=0) == _native.E_ARG
    assert call(ib=2) == _native.E_ARG
    assert call(d=None) == _native.E_ARG
    assert call(d=ids.data_ptr() + 4) == _native.E_ARG        # misaligned ids
    assert call(s=scratch.data_ptr() + 16) == _native.E_ARG   # misaligned scratch
    assert call(b=sb - 1) == _native.E_ARG
    assert scratch_size(p, orig + 1)[0] == _native.E_ARG
    assert _native.launch_count() == before
    assert p.status() == 0
    # a box, an empty item and a split item are not one whole-tensor piece
    box = DP.Item(case.name, case.body, case.G, case.bits, case.chunk, orig, H.expect(case, (16, 3, 4096, 100)), box=(16, 3, 4096, 100))
    empty = DP.Item("empty", np.zeros(0, np.uint8), 2, 0, 4096, 0, np.zeros(0, np.uint8))
    for items in ([item, box], [item, empty]):
        q = DP.Plan(items)
        assert q.rc == 0
        assert scratch_size(q, 1)[0] == _native.E_UNSUPPORTED
    DP._set_env(monkeypatch, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": "5"})
    q = DP.Plan([item])
    assert q.rc == 0 and scratch_size(q, 1)[0] == _native.E_UNSUPPORTED


# ------------------------------------------------------------------ module level
class Experts(torch.nn.Module):
    """The transformers convention, with the eager loop of MixtralExperts."""

    def __init__(self, E, H_, inter, dtype):
        super().__init__()
        self.num_experts = E
        self.gate_up_proj = torch.nn.Parameter(torch.randn(E, 2 * inter, H_, dtype=torch.float32).mul_(0.02).to(dtype))
        self.down_proj = torch.nn.Parameter(torch.randn(E, H_, inter, dtype=torch.float32).mul_(0.02).to(dtype))

    def forward(self, hidden_states, top_k_index, top_k_weights):
        out = torch.zeros_like(hidden_states)
        for e in top_k_index.unique().tolist():
            pos, tok = torch.where(top_k_index.T == e)
            gate, up = torch.nn.functional.linear(hidden_states[tok], self.gate_up_proj[e]).chunk(2, dim=-1)
            h = torch.nn.functional.linear(torch.nn.functional.silu(gate) * up, self.down_proj[e])
            out.index_add_(0, tok, h * top_k_weights[tok, pos, None])
        return out


class MoE(torch.nn.Module):
    def __init__(self, E=8, H_=1024, inter=352, k=2, dtype=torch.bfloat16, kw=False):
        super().__init__()
        self.k, self.kw = k, kw
        self.router = torch.nn.Linear(H_, E, bias=False, dtype=dtype)
        self.experts = Experts(E, H_, inter, dtype)

    def forward(self, x):
        w, idx = torch.topk(torch.softmax(self.router(x).float(), -1), self.k, dim=-1)
        w = w.to(x.dtype)
        if self.kw:
            return self.experts(x, top_k_index=idx, top_k_weights=w)
        return self.experts(x, idx, w)


def _moe(kw=False):
    torch.manual_seed(11)
    return MoE(kw=kw).cuda().eval()


def _nan_forward(model, x):
    state = getattr(model, _ATTR)
    for _, plan, _, _ in state.entries:
        plan._out.fill_(0xFF)   # NaN in every bf16 element of the shared output buffer
    with torch.no_grad():
        return model(x)


@pytest.mark.parametrize("kw", (False, True))
def test_compressed_moe_block_is_exact(kw):
    model = _moe(kw)
    xs = [torch.randn(n, 1024, device="cuda").to(torch.bfloat16) for n in (1, 3, 16, 64)]
    idx16 = torch.tensor([[3, 6]], dtype=torch.int16, device="cuda")
    w16 = torch.tensor([[0.75, 0.25]], dtype=torch.bfloat16, device="cuda")
    with torch.no_grad():
        want = [model(x) for x in xs]
        y16 = model.experts(xs[0], idx16, w16)
    rep = compress_module(model, experts=True)
    assert rep["experts_modules"] == 1 and rep["experts_scratch_bytes"] > 0
    state = getattr(model, _ATTR)
    plan = next(p for m, p, _, _ in state.entries if m is model.experts)
    calls = {"select": 0, "run": 0}
    real_sel, real_run = plan.run_select, plan.run
    plan.run_select = lambda *a, **k: (calls.__setitem__("select", calls["select"] + 1), real_sel(*a, **k))[1]
    plan.run = lambda *a, **k: (calls.__setitem__("run", calls["run"] + 1), real_run(*a, **k))[1]
    for x, w in zip(xs, want):
        got = _nan_forward(model, x)
        assert torch.equal(got, w)
    assert calls == {"select": len(xs), "run": 0}
    with torch.no_grad():   # ids of another dtype fall back to the whole decode
        y = model.experts(xs[0], idx16, w16)
    assert calls["run"] == 1 and torch.equal(y, y16)
    with pytest.raises(RuntimeError, match="no_grad"):
        model(xs[0])
    decompress_module(model)
    with torch.no_grad():
        assert all(torch.equal(model(x), w) for x, w in zip(xs, want))


def test_load_module_experts(tmp_path):
    from safetensors.torch import save_file as plain_save_file
    model = _moe()
    x = torch.randn(5, 1024, device="cuda").to(torch.bfloat16)
    with torch.no_grad():
        want = model(x)
    plain = str(tmp_path / "plain.safetensors")
    plain_save_file({k: v.contiguous() for k, v in model.state_dict().items()}, plain)
    compress_module(model, experts=True)
    znn = str(tmp_path / "m.znn.safetensors")
    save_module(model, znn)
    for path in (znn, plain):
        with torch.device("meta"):
            fresh = MoE()
        rep = load_module(fresh, path, experts=True)
        assert rep["experts_modules"] == 1
        assert torch.equal(_nan_forward(fresh, x), want), path
        decompress_module(fresh)
        for k, v in _moe().state_dict().items():
            assert torch.equal(fresh.state_dict()[k], v), k


# ------------------------------------------------------------------ transformers models
def _tiny_models():
    tf = pytest.importorskip("transformers")
    common = dict(hidden_size=256, intermediate_size=352, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                  num_hidden_layers=2, vocab_size=512)
    return [(tf.MixtralForCausalLM, tf.MixtralConfig(num_local_experts=8, num_experts_per_tok=2, **common)),
            (tf.Qwen3MoeForCausalLM, tf.Qwen3MoeConfig(num_experts=16, num_experts_per_tok=4, moe_intermediate_size=352,
                                                        decoder_sparse_step=1, mlp_only_layers=[], **common))]


@pytest.mark.parametrize("which", (0, 1))
def test_transformers_moe_logits_are_exact(which):
    cls, cfg = _tiny_models()[which]
    torch.manual_seed(21)
    model = cls(cfg).to(torch.bfloat16).cuda().eval()
    ids = {n: torch.randint(0, cfg.vocab_size, (1, n), device="cuda") for n in (1, 16)}
    impls = ("eager", "batched_mm", "grouped_mm")
    want = {}
    with torch.no_grad():
        for impl in impls:
            model.config._experts_implementation = impl
            for n, t in ids.items():
                want[impl, n] = model(t).logits
    rep = compress_module(model, experts=True)
    # the experts modules, and the routers (weight [E, H], num_experts = E: they pass no ids, so they decode whole)
    experts = [m for m in model.modules() if type(m).__name__.endswith("Experts")]
    mode = {id(m): mode for m, _, _, mode in getattr(model, _ATTR).entries}
    assert len(experts) == cfg.num_hidden_layers and all(mode.get(id(m)) == "experts" for m in experts)
    assert rep["experts_modules"] == 2 * cfg.num_hidden_layers
    for impl in impls:
        model.config._experts_implementation = impl
        for n, t in ids.items():
            got = _nan_forward(model, t).logits
            assert torch.equal(got, want[impl, n]), (cls.__name__, impl, n)
    assert torch.cuda.max_memory_allocated() < 16 << 30
