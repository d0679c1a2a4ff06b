"""Every run mode on one model: compress_module / load_module with gather=True, matvec=8, matmul=64, experts=True and
fp8=True together.

The model has an embedding tied to a bf16 lm_head, bf16 linears (one with a bias), the mixture-of-experts block of
test_select_gpu and an FP8Linear built as test_dequant_fp8_gpu builds them.  At 1, 8, 64 and 65 rows each module
takes the path of its mode (the DecodePlan calls made while it runs) and gives bit for bit the output the same module
gives in a copy of the model compressed with its own mode alone.  compress_module and load_module, from .safetensors
and from .znn.safetensors, give the same report and logits; decompress_module gives back every parameter, hook and
forward.
"""
import copy

import pytest
import torch
import torch.nn.functional as F
from safetensors.torch import save_file as plain_save_file

from test_dequant_fp8_gpu import _quantized
from test_select_gpu import MoE
from zipnn_b200 import DecodePlan, compress_module, decompress_module, load_module, save_module
from zipnn_b200.resident import _ATTR

pytestmark = pytest.mark.gpu

H, FFN, VOCAB = 256, 512, 1024
ROWS = (1, 8, 64, 65)
ALL = dict(gather=True, matvec=8, matmul=64, experts=True, fp8=True)
# each mode alone; fp8 with matvec=8, the row limit of its matvec_fp8
ALONE = {"gather": dict(gather=True), "matvec": dict(matvec=8), "matmul": dict(matmul=64), "experts": dict(experts=True),
         "fp8": dict(fp8=True, matvec=8)}
LEAVES = ("embed_tokens", "up_proj", "down_proj", "moe.router", "moe.experts", "fp8_proj", "lm_head")
PLAN_CALLS = ("run", "run_select", "gather", "matvec", "matmul", "matvec_fp8", "dequant_fp8")


class Model(torch.nn.Module):
    def __init__(self):
        from transformers.integrations.finegrained_fp8 import FP8Linear
        super().__init__()
        self.embed_tokens = torch.nn.Embedding(VOCAB, H)
        self.up_proj = torch.nn.Linear(H, FFN)
        self.down_proj = torch.nn.Linear(FFN, H, bias=False)
        self.moe = MoE(E=8, H_=H, inter=FFN // 2)
        self.fp8_proj = FP8Linear(H, H, block_size=(128, 128))
        self.lm_head = torch.nn.Linear(H, VOCAB, bias=False)
        self.lm_head.weight = self.embed_tokens.weight

    def forward(self, ids):
        x = self.embed_tokens(ids)
        x = x + self.down_proj(F.silu(self.up_proj(x)))
        x = x + self.moe(x.reshape(-1, H)).view(x.shape)
        x = x + self.fp8_proj(x)
        return self.lm_head(x)


def _with_fp8_weight(m, seed):
    """`m` with an e4m3 weight and its 128x128-block scales in fp8_proj (after the bf16 cast, which would take them)."""
    if seed is None:
        wq, scale = torch.empty(H, H, dtype=torch.float8_e4m3fn, device="meta"), torch.empty(2, 2, device="meta")
    else:
        wq, scale = _quantized("e4m3", H, H, seed)
    m.fp8_proj.weight = torch.nn.Parameter(wq, requires_grad=False)
    m.fp8_proj.weight_scale_inv = torch.nn.Parameter(scale, requires_grad=False)
    return m.eval()


def make(seed):
    torch.manual_seed(seed)
    m = Model()
    with torch.no_grad():
        for p in (m.embed_tokens.weight, m.up_proj.weight, m.up_proj.bias, m.down_proj.weight):
            p.normal_(0, 0.02)
    return _with_fp8_weight(m.to(device="cuda", dtype=torch.bfloat16), seed)


def meta():
    with torch.device("meta"):
        m = Model().to(torch.bfloat16)
    return _with_fp8_weight(m, None)


class Paths:
    """The DecodePlan calls made while each leaf module runs (outermost calls only), and each leaf's inputs and output."""

    def __init__(self, monkeypatch):
        self.calls, self.io, self.stack, self.depth = [], [], [], 0
        for name in PLAN_CALLS:
            monkeypatch.setattr(DecodePlan, name, self._wrap(name, getattr(DecodePlan, name)))

    def _wrap(self, name, orig):
        def call(plan, *args, **kwargs):
            if self.depth == 0:
                self.calls.append((self.stack[-1] if self.stack else None, name))
            self.depth += 1
            try:
                return orig(plan, *args, **kwargs)
            finally:
                self.depth -= 1
        return call

    def watch(self, model) -> list:
        """Hooks on the leaves of `model` that keep the running one on the stack and record its calls -> handles."""
        def done(name):
            def hook(mod, args, kwargs, out):
                self.stack.pop()
                self.io.append((name, [a.clone() for a in args], {k: v.clone() for k, v in kwargs.items()}, out.clone()))
            return hook
        hs = []
        for name in LEAVES:
            mod = model.get_submodule(name)
            hs.append(mod.register_forward_pre_hook(lambda mod, args, name=name: self.stack.append(name), prepend=True))
            hs.append(mod.register_forward_hook(done(name), with_kwargs=True))
        return hs

    def by_module(self) -> dict:
        out = {}
        for name, call in self.calls:
            out.setdefault(name, []).append(call)
        return out


def own_mode(name, rows):
    """The option that sets the path of leaf `name` at `rows` rows."""
    if name == "embed_tokens":
        return "gather"
    if name == "moe.experts":
        return "experts"
    if name == "fp8_proj":
        return "fp8"
    return "matmul" if 8 < rows <= 64 else "matvec"


def bits(t):
    return t.view(torch.int16)


def test_each_module_takes_its_path_and_gives_its_own_modes_bits(monkeypatch):
    dense = make(1)
    model = copy.deepcopy(dense)
    alone = {mode: copy.deepcopy(dense) for mode in ALONE}
    rep = compress_module(model, **ALL)
    assert rep["gather_modules"] == 1 and rep["experts_modules"] == 1 and rep["fp8_modules"] == 1
    assert rep["matvec_modules"] >= 3 and rep["matmul_modules"] >= 3   # up_proj, down_proj, lm_head; the router if it takes them
    for mode, kw in ALONE.items():
        compress_module(alone[mode], **kw)
    paths = Paths(monkeypatch)
    hs = paths.watch(model)
    g = torch.Generator("cuda").manual_seed(2)
    with torch.no_grad():
        for rows in ROWS:
            ids = torch.randint(0, VOCAB, (1, rows), device="cuda", generator=g)
            paths.calls.clear()
            paths.io.clear()
            model(ids)
            got = paths.by_module()
            assert None not in got and sorted(got) == sorted(LEAVES), got
            product = "matvec" if rows <= 8 else "matmul" if rows <= 64 else "run"
            assert got["embed_tokens"] == ["gather"], rows
            assert got["up_proj"] == got["down_proj"] == got["lm_head"] == [product], (rows, got)
            assert got["moe.experts"] == ["run_select"], rows
            assert got["fp8_proj"] == ["matvec_fp8" if rows <= 8 else "dequant_fp8"], rows
            assert sorted(n for n, _, _, _ in paths.io) == sorted(LEAVES)
            for name, args, kwargs, out in list(paths.io):
                paths.calls.clear()
                want = alone[own_mode(name, rows)].get_submodule(name)(*args, **kwargs)
                assert [c for _, c in paths.calls] == got[name], (name, rows)
                assert torch.equal(bits(out), bits(want)), (name, rows)
    for h in hs:
        h.remove()


def test_load_module_reaches_compress_modules_report_and_logits(tmp_path):
    dense = make(3)
    model = copy.deepcopy(dense)
    want_rep = compress_module(model, **ALL)
    sd = dense.state_dict()
    del sd["lm_head.weight"]   # tied: one name is enough
    plain = str(tmp_path / "m.safetensors")
    plain_save_file({k: v.contiguous().cpu() for k, v in sd.items()}, plain)
    znn = str(tmp_path / "m.znn.safetensors")
    save_module(model, znn)
    ids = {rows: torch.randint(0, VOCAB, (1, rows), device="cuda") for rows in ROWS}
    with torch.no_grad():
        want = {rows: model(t) for rows, t in ids.items()}
    for path in (plain, znn):
        m = meta()
        rep = load_module(m, path, **ALL)
        assert rep == want_rep, path
        with torch.no_grad():
            for rows, t in ids.items():
                assert torch.equal(bits(m(t)), bits(want[rows])), (path, rows)
        decompress_module(m)
        for (n, p), (_, q) in zip(m.named_parameters(), dense.named_parameters()):
            assert torch.equal(p.view(torch.uint8), q.view(torch.uint8)), (path, n)


def test_decompress_module_restores_every_parameter_hook_and_forward():
    dense = make(4)
    model = copy.deepcopy(dense)
    compress_module(model, **ALL)
    with torch.no_grad():
        for rows in ROWS:
            model(torch.randint(0, VOCAB, (1, rows), device="cuda"))
    decompress_module(model)
    assert not hasattr(model, _ATTR)
    assert [n for n, _ in model.named_parameters()] == [n for n, _ in dense.named_parameters()]
    for (n, p), (_, q) in zip(model.named_parameters(), dense.named_parameters()):
        assert type(p) is torch.nn.Parameter and p.requires_grad == q.requires_grad, n
        assert p.dtype == q.dtype and torch.equal(p.view(torch.uint8), q.view(torch.uint8)), n
    assert model.lm_head.weight is model.embed_tokens.weight
    for name, mod in model.named_modules():
        assert "forward" not in mod.__dict__ and not mod._forward_pre_hooks and not mod._forward_hooks, name
