"""Keep a model's weights compressed in GPU memory and decode each module's weights just before it runs.

`compress_module(model)` replaces the floating-point parameters of the selected modules with ZipNN streams in HBM
(about 0.66 of the bytes for bf16 weights).  Each compressed module gets a `DecodePlan` (plan.py); a forward
pre-hook runs it and binds the decoded weights as plain attributes, a forward hook removes them again.  The codec
is lossless, so the module computes bit for bit what it computed with dense weights.

Rules:
  * inference only: the decoded weights live in a buffer shared by every compressed module, so autograd could not
    keep them; a compressed module raises RuntimeError when it runs with grad mode on (use torch.no_grad() or
    torch.inference_mode());
  * the selected modules must not contain one another (they would overwrite each other's weights in the shared
    buffer): the default selection takes the innermost parameter owners, an explicit one that nests raises
    ValueError; all their runs go to one CUDA stream at a time;
  * the decoded weights are views of the shared buffer, valid only during the module's own forward: a forward that
    returns (a view of) its weight returns memory the next compressed module overwrites -- such a module must not be
    selected;
  * a parameter shared by several modules (tied weights) is stored once; a parameter also owned by a module outside
    the selection stays dense, as does one whose stream is not smaller than its bytes;
  * with `prefetch=True` the next module's weights are decoded on a side stream while the current module computes
    (prefetch.py); to capture a CUDA graph, capture the root module's forward, not a submodule's: the root's
    forward hook is what joins the side stream;
  * with `gather=True` a selected `torch.nn.Embedding` (its class's own forward, no max_norm) looks its rows up
    straight from the stream (`DecodePlan.gather`: only the chunks the ids touch are decoded) and is never decoded
    whole; its output is an ordinary tensor the caller owns;
  * with `matvec=N` a selected `torch.nn.Linear` (its class's own forward) multiplies inputs of at most N rows
    straight from the stream (`DecodePlan.matvec`: the dense weight is neither written nor read) and decodes as
    before for larger inputs; its bias stays a dense parameter;
  * with `matmul=N` such a Linear with a bf16 / fp16 weight multiplies inputs of more rows than the matvec takes and
    at most N on tensor cores (`DecodePlan.matmul`), again without a dense weight;
  * with `fp8=True` a selected fp8 linear layer (`fp8_linears`: transformers' `FP8Linear`) keeps its scales and bias
    dense and runs W8A16 from its stream at any number of rows: `DecodePlan.matvec_fp8` for at most `matvec` rows,
    `DecodePlan.dequant_fp8` + F.linear for more; it needs no downloaded kernel;
  * with `fp8=True` and `experts=True` together, an fp8 experts module (`fp8_experts`: transformers' `FP8Experts`)
    keeps its scales dense and runs W8A16: `DecodePlan.dequant_fp8_select` writes only its routed experts' weights,
    dequantized to bf16 / fp16, and the bf16 experts implementation its config names runs on them;
  * with `experts=True` the experts module of a mixture-of-experts layer (`experts_module`: 3D weights [E, ...] called
    as experts(hidden_states, top_k_index, top_k_weights)) decodes only the slices [e] of the experts its router
    picked (`DecodePlan.run_select`); its own forward then runs unchanged and reads only those slices;
  * `state_dict()` does not see compressed parameters; `decompress_module(model)` restores them as dense
    `Parameter`s, bit for bit, and removes the hooks and plans.

`load_module(model, files)` reaches the same state straight from safetensors / .znn.safetensors files, with no dense
copy of the compressed weights on the GPU, and `save_module(model, file)` writes a compressed model back to a
.znn.safetensors file from its streams, with no decode.
"""
from __future__ import annotations

import inspect
import math
import os
import traceback
from typing import NamedTuple

import torch
import torch.nn.functional as F

from . import prefetch as _prefetch
from .plan import _HEAD, EXPERTS_MATVEC_MAX_TOKENS, MATMUL_MAX_TOKENS, MATVEC_MAX_TOKENS, DecodePlan, _Stream
from .safetensors_io import _FileRange, _cuda_device, compress_groups, file_entries, save_coded
from .util_safetensors import COMPRESSION_METHOD
from .zipnn import DecodePipe, ZipNN

_DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2)
_FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)
_ATTR = "_zipnn_resident"


def _own_params(m: torch.nn.Module):
    return [(n, p) for n, p in m._parameters.items() if p is not None and p.dtype in _DTYPES]


def select(module: torch.nn.Module, modules=None):
    """The selection rules without compressing anything (no GPU needed).

    -> (modules, groups): the selected modules, and one group per distinct parameter to compress:
    (parameter, [(module, name), ...] every place it is bound).  Default selection: every submodule that directly
    owns parameters of the codec's dtypes and contains no other such module (an owner that contains one, e.g.
    torch.nn.MultiheadAttention with its out_proj, keeps its own parameters dense).  ValueError when one module of an
    explicit selection contains another."""
    if modules is None:
        owners = [m for m in module.modules() if _own_params(m)]
        owned = {id(m) for m in owners}
        modules = [m for m in owners if not any(id(sub) in owned for sub in m.modules() if sub is not m)]
    else:
        modules = list(dict.fromkeys(modules))
    chosen = {id(m) for m in modules}
    for m in modules:
        for sub in m.modules():
            if sub is not m and id(sub) in chosen:
                raise ValueError(f"compress_module: selected module {type(m).__name__} contains selected module {type(sub).__name__}")
    places = {}   # id(param) -> (param, [(module, name)]) over the whole model, to find ties
    for m in module.modules():
        for n, p in m._parameters.items():
            if p is not None:
                places.setdefault(id(p), (p, []))[1].append((m, n))
    groups, seen = [], set()
    for m in modules:
        for _, p in _own_params(m):
            if id(p) in seen:
                continue
            seen.add(id(p))
            owners = places.get(id(p), (p, [(m, n) for n, q in m._parameters.items() if q is p]))[1]
            if all(id(o) in chosen for o, _ in owners):
                groups.append((p, owners))
    return modules, groups


class _Options(NamedTuple):
    """The run modes of compress_module / load_module, as `_options` checked them."""
    prefetch: bool
    gather: bool
    matvec: int    # the most input rows a matvec module multiplies without decoding (0: none)
    matmul: int    # the most input rows a matmul module multiplies without decoding (0: none)
    experts: bool
    fp8: bool
    fp8_matmul: int  # the most input rows an "fp8" module multiplies on tensor cores without dequantizing (0: none)
    experts_matvec: int  # the most tokens an "fp8_experts_matvec" module multiplies from its streams (0: none)


def _options(prefetch=False, gather=False, matvec=0, matmul=0, experts=False, fp8=False, fp8_matmul=0,
             experts_matvec=0) -> _Options:
    """ValueError for a row count out of range, for fp8_matmul without fp8=True, for experts_matvec without fp8=True
    and experts=True, and for a mode that does not combine with prefetch=True."""
    for name, n, limit in (("matvec", matvec, MATVEC_MAX_TOKENS), ("matmul", matmul, MATMUL_MAX_TOKENS),
                           ("fp8_matmul", fp8_matmul, MATMUL_MAX_TOKENS)):
        if not (isinstance(n, int) and 0 <= n <= limit):
            raise ValueError(f"{name} must be an integer from 0 to {limit}, not {n!r}")
        if n and prefetch:
            raise ValueError(f"{name} and prefetch=True do not combine yet: the prefetch schedule decodes every module")
    if experts and prefetch:
        raise ValueError("experts=True and prefetch=True do not combine: the prefetch schedule decodes every module "
                         "before its router has picked the experts")
    if fp8 and prefetch:
        raise ValueError("fp8=True and prefetch=True do not combine yet: the prefetch schedule decodes every module")
    if fp8_matmul and not fp8:
        raise ValueError("fp8_matmul applies to the fp8 modules of fp8=True: pass fp8=True with it")
    if not (isinstance(experts_matvec, int) and not isinstance(experts_matvec, bool) and 0 <= experts_matvec <= EXPERTS_MATVEC_MAX_TOKENS):
        raise ValueError(f"experts_matvec must be an integer from 0 to {EXPERTS_MATVEC_MAX_TOKENS}, not {experts_matvec!r}")
    if experts_matvec and not (fp8 and experts):
        raise ValueError("experts_matvec applies to the fp8 experts modules of fp8=True with experts=True: pass fp8=True and "
                         "experts=True with it")
    return _Options(bool(prefetch), bool(gather), matvec, matmul, bool(experts), bool(fp8), fp8_matmul, experts_matvec)


class _Entry(NamedTuple):
    """A module decoded whole and how it runs, as `_resident_state` decided it."""
    module: torch.nn.Module
    plan: DecodePlan
    names: list   # [(name, index into the plan's outputs)]
    mode: str     # hooks: "decode", "prefetch", "experts"; a forward of its own: "matvec", "matmul", "fp8", "fp8_torch",
                  # "fp8_experts", "fp8_experts_torch", "fp8_experts_matvec"


class _Resident:
    """What compress_module leaves on the root module: per compressed module its plan and parameter names."""

    def __init__(self):
        self.entries = []     # _Entry per module decoded whole
        self.hooks = []       # the entries' hook handles
        self.params = {}      # parameter index -> (requires_grad, dtype, shape, [(module, name)] where it was bound)
        self.stream_of = {}   # parameter index -> its stream (a view of `streams`)
        self.streams = []     # the buffers that hold the streams (one per load group)
        self.order = {}       # id(module) -> (module, its parameter names in their original order)
        self.prefetch = None  # prefetch=True: (Prefetcher, slot 1 buffer, root hook handles)
        self.gathers = []     # gather=True: (embedding module, plan, index into the plan's outputs, own plan?)
        self.scratch = None   # the plans' shared scratch
        self.gather_scratch = None  # the gathers' scratch: the plans' one, or a buffer of its own (prefetch)
        self.gather_plan_bytes = 0  # memory of the plans that only serve gathers
        self.matvec = 0       # matvec=N: the most input rows a "matvec" / "matmul" / "fp8" module multiplies by a matvec
        self.matvec_scratch = None     # the matvecs' scratch and what the largest of them needs of it
        self.matvec_scratch_bytes = 0
        self.matmul_scratch = None     # the "matmul" modules' matmul scratch and what the largest needs of it
        self.matmul_scratch_bytes = 0
        self.select_scratch = None     # the "experts" and "fp8_experts" modules' selected-run scratch, sized for the largest
        self.fp8_scratch = None        # the "fp8" modules' matvec_fp8 scratch and what the largest needs of it
        self.fp8_scratch_bytes = 0
        self.fp8_matmul = 0            # fp8_matmul=N: the most input rows an "fp8" module multiplies by matmul_fp8
        self.fp8_matmul_scratch = None  # the "fp8" modules' matmul_fp8 scratch and what the largest needs of it
        self.fp8_matmul_scratch_bytes = 0
        self.experts_matvec = 0        # experts_matvec=N: the most tokens an "fp8_experts_matvec" module multiplies from its streams
        self.experts_matvec_scratch = None  # their experts_matvec_fp8 scratch and what the largest needs of it
        self.experts_matvec_scratch_bytes = 0


def _grad_mode_error(mod, shared: bool = False):
    raise RuntimeError(f"{type(mod).__name__} holds compressed weights and runs only under torch.no_grad() or "
                       "torch.inference_mode()" + (" (its decoded weights live in a shared buffer)" if shared else ""))


def _bind(mod, names, outs) -> None:
    for name, k in names:
        object.__setattr__(mod, name, outs[k])


def _pre_hook(plan, names):
    def hook(mod, args):
        if torch.is_grad_enabled():
            _grad_mode_error(mod, shared=True)
        _bind(mod, names, plan.run())
    return hook


def _pre_hook_experts(plan, names, state):
    # the ids: experts(hidden_states, top_k_index, top_k_weights), positional or by keyword
    def hook(mod, args, kwargs):
        if torch.is_grad_enabled():
            _grad_mode_error(mod, shared=True)
        ids = args[1] if len(args) > 1 else kwargs.get("top_k_index")
        if (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.device == plan.device
                and ids.dtype in (torch.int32, torch.int64)):
            _bind(mod, names, plan.run_select(ids, scratch=state.select_scratch))
        else:
            _bind(mod, names, plan.run())
    return hook


def _pre_hook_prefetch(sched, key, names, views):
    def hook(mod, args):
        if torch.is_grad_enabled():
            _grad_mode_error(mod, shared=True)
        _bind(mod, names, views[sched.before(key)])
    return hook


def gathers(module: torch.nn.Module) -> bool:
    """Does `gather=True` look `module` up by a gather instead of decoding its weight whole?  A torch.nn.Embedding
    (or subclass) whose class does not override forward and that has no max_norm (which renormalises the weight)."""
    return isinstance(module, torch.nn.Embedding) and type(module).forward is torch.nn.Embedding.forward and module.max_norm is None


def _gather_forward(mod, state, plan, k):
    # padding_idx, scale_grad_by_freq and sparse only shape gradients, which a compressed module never has
    def forward(input):
        if torch.is_grad_enabled():
            _grad_mode_error(mod)
        return plan.gather(k, input, scratch=state.gather_scratch)
    return forward


def matvecs(module: torch.nn.Module) -> bool:
    """Does `matvec=N` multiply small inputs of `module` from its compressed weight?  A torch.nn.Linear (or subclass)
    whose class does not override forward."""
    return isinstance(module, torch.nn.Linear) and type(module).forward is torch.nn.Linear.forward


def experts_module(module: torch.nn.Module, names=None) -> bool:
    """Does `experts=True` decode only the routed experts of `module`?  A module whose integer attribute `num_experts`
    equals shape[0] of every parameter in `names` (default: every parameter of the codec's dtypes it owns directly;
    there must be one): the convention of transformers' `*Experts` modules (gate_up_proj [E, 2I, H], down_proj
    [E, H, I], biases [E, ...]).  Once its streams exist, its plan must also pass `DecodePlan.select_ok`."""
    n = getattr(module, "num_experts", None)
    if not isinstance(n, int) or isinstance(n, bool) or n <= 0:
        return False
    params = [p for name, p in _own_params(module) if names is None or name in names]
    return bool(params) and all(p.dim() >= 1 and p.shape[0] == n for p in params)


def fp8_linears(module: torch.nn.Module) -> bool:
    """Does `fp8=True` run `module` from its compressed fp8 weight?  A torch.nn.Linear (or subclass) with a 2-D
    float8_e4m3fn / float8_e5m2 `weight`, an fp32 `weight_scale_inv` and a `block_size` that is None (a one-element
    scale) or (bn, bk) with the grid's shape [ceil(out / bn), ceil(in / bk)]: transformers' `FP8Linear`, found by these
    attributes."""
    w, scale = getattr(module, "weight", None), getattr(module, "weight_scale_inv", None)
    if not (isinstance(module, torch.nn.Linear) and isinstance(w, torch.Tensor) and w.dim() == 2 and w.dtype in _FP8
            and isinstance(scale, torch.Tensor) and scale.dtype == torch.float32 and hasattr(module, "block_size")):
        return False
    block = module.block_size
    if block is None:
        return scale.numel() == 1
    if not (isinstance(block, (tuple, list)) and len(block) == 2 and all(isinstance(b, int) and b >= 1 for b in block)):
        return False
    return tuple(scale.shape) == (-(-w.shape[0] // block[0]), -(-w.shape[1] // block[1]))


def fp8_experts(module: torch.nn.Module) -> bool:
    """Does `fp8=True, experts=True` run `module` from its compressed fp8 expert weights?  A module of the
    `experts_module` convention (integer `num_experts` = E) with a `block_size` that is None or (bn, bk), at least one
    float8_e4m3fn / float8_e5m2 parameter, each of them 3-D [E, out, in] with an fp32 `<name>_scale_inv` of the grid
    the block implies, [E, ceil(out / bn), ceil(in / bk)] (None: [E, 1, 1]), and no bias parameter: transformers'
    `FP8Experts` (gate_up_proj or up_proj, down_proj), found by these attributes."""
    if not (experts_module(module) and hasattr(module, "block_size")):
        return False
    block, n = module.block_size, module.num_experts
    if block is not None and not (isinstance(block, (tuple, list)) and len(block) == 2
                                  and all(isinstance(b, int) and not isinstance(b, bool) and b >= 1 for b in block)):
        return False
    params = {name: p for name, p in module._parameters.items() if p is not None}
    fp8 = [(name, p) for name, p in params.items() if p.dtype in _FP8]
    if not fp8 or any("bias" in name for name in params):
        return False
    for name, w in fp8:
        s = params.get(name + "_scale_inv")
        if w.dim() != 3 or not (isinstance(s, torch.Tensor) and s.dtype == torch.float32):
            return False
        grid = (n, 1, 1) if block is None else (n, -(-w.shape[1] // block[0]), -(-w.shape[2] // block[1]))
        if tuple(s.shape) != grid:
            return False
    return True


def experts_matvec_layout(module: torch.nn.Module):
    """The projections of an `fp8_experts` module in one of transformers' `FP8Experts` layouts, which experts_matvec=N
    multiplies from the streams: -> (first, "down_proj"), first = "gate_up_proj" [E, 2I, H], gated by the module's
    `_apply_gate`, or "up_proj" [E, I, H] (an FP8Experts built with has_gate=False), activated by its `act_fn`, and
    down_proj [E, H, I]; None for any other module.  The parameters decide, not the `has_gate` attribute: transformers
    sets it True whatever the constructor was given."""
    if not fp8_experts(module):
        return None
    params = {name: p for name, p in module._parameters.items() if p is not None and p.dtype in _FP8}
    gate = "gate_up_proj" in params
    first = "gate_up_proj" if gate else "up_proj"
    if sorted(params) != sorted([first, "down_proj"]) or not callable(getattr(module, "_apply_gate" if gate else "act_fn", None)):
        return None
    f, d = params[first].shape, params["down_proj"].shape
    inter = f[1] // 2 if gate else f[1]
    if (gate and f[1] % 2) or f[0] != d[0] or d[1] != f[2] or d[2] != inter:
        return None
    return first, "down_proj"


def dequantize_fp8(weight: torch.Tensor, scale: torch.Tensor, block, dtype: torch.dtype) -> torch.Tensor:
    """torch's dequantize of an fp8 weight [..., out, in]: (W.to(float32) * S_expanded).to(dtype), S expanded over its
    (bn, bk) blocks (block None: one scale per [out, in] matrix), one grid [ceil(out / bn), ceil(in / bk)] per leading
    index (an experts weight [E, out, in] has one per expert).  `DecodePlan.dequant_fp8` and `dequant_fp8_select` give
    the same bits."""
    w = weight.to(torch.float32)
    lead = tuple(weight.shape[:-2])
    if block is None:
        return (w * scale.reshape(lead + (1, 1))).to(dtype)
    (out, inn), (bn, bk) = weight.shape[-2:], block
    s = scale.reshape(lead + (-(-out // bn), -(-inn // bk))).repeat_interleave(bn, -2)[..., :out, :]
    s = s.repeat_interleave(bk, -1)[..., :inn]
    return (w * s).to(dtype)


def dense_biases(groups, matvec: int, fp8: bool = False, experts: bool = False) -> list:
    """`select`'s groups without the parameters that stay dense: under matvec=N the biases owned by `matvecs` modules
    only (the matvec adds them after the sum, so they must not need a decode); under fp8=True every parameter but the
    weight of `fp8_linears` modules (scales, bias, activation scale: the products read them as they are); under
    fp8=True and experts=True together every parameter but the fp8 ones of `fp8_experts` modules (scales, static
    activation scales)."""
    if not (matvec or fp8):
        return groups

    def dense(o, n):
        return ((matvec and n == "bias" and matvecs(o)) or (fp8 and n != "weight" and fp8_linears(o))
                or (fp8 and experts and o._parameters[n].dtype not in _FP8 and fp8_experts(o)))
    return [(p, owners) for p, owners in groups if not all(dense(o, n) for o, n in owners)]


def _fp8_block(mod) -> tuple:
    return None if mod.block_size is None else tuple(mod.block_size)


def _rows(input) -> int:
    """The rows of an input [..., in_features]: the product of its leading dims (None without a last dim to divide by)."""
    width = input.shape[-1] if input.dim() else 0
    return input.numel() // width if width else None


def _decoded(mod, plan, names, forward):
    """-> f(input): the decode, bind, `forward(mod, input)`, unbind of the hooks every other compressed module has."""
    pre, post = _pre_hook(plan, names), _unbind(names)

    def run(input):
        pre(mod, (input,))
        try:
            return forward(mod, input)
        finally:
            post(mod, (input,), None)
    return run


def _fp8_forward(mod, state, plan, k, names, fast: bool):
    """The forward of an fp8 linear module (W8A16: the activations are not quantized).  A bf16 / fp16 input on the plan's
    device, outside autocast, is multiplied with the dequantized weight S * W: at most `state.matvec` rows by
    `plan.matvec_fp8`, more and at most `state.fp8_matmul` by `plan.matmul_fp8`, more by `plan.dequant_fp8` into the
    shared output buffer and F.linear; the bias is added as FP8Linear.forward adds it.  A module whose weight `fast` is False for (`matvec_fp8_ok` refuses it) decodes it and
    dequantizes in torch into a fresh tensor instead (the fp8 bytes occupy the shared buffer), with the same result.
    Any other input takes the decode, bind, module's own forward, unbind of the other compressed modules."""
    decoded = _decoded(mod, plan, names, type(mod).forward)
    block = _fp8_block(mod)
    shape = tuple(plan.outputs[k].shape)
    nbytes = 2 * shape[0] * shape[1]

    def forward(input):
        if (input.dtype in (torch.bfloat16, torch.float16) and input.device == plan.device
                and not torch.is_autocast_enabled(plan.device.type)):
            if torch.is_grad_enabled():
                _grad_mode_error(mod)
            rows = _rows(input)
            scale = mod.weight_scale_inv
            if fast and rows is not None and rows <= state.matvec:
                y = plan.matvec_fp8(k, input, scale, block, scratch=state.fp8_scratch)
            elif fast and rows is not None and rows <= state.fp8_matmul:
                y = plan.matmul_fp8(k, input, scale, block, scratch=state.fp8_matmul_scratch)
            else:
                if fast:
                    w = plan.dequant_fp8(k, shape[1], scale, block, input.dtype, out=plan._out[:nbytes].view(input.dtype).view(shape))
                else:
                    w = dequantize_fp8(plan.run()[k], scale, block, input.dtype)
                y = F.linear(input, w)
            return y if mod.bias is None else (y + mod.bias).to(input.dtype)
        return decoded(input)
    return forward


def _experts_impl(mod):
    """The experts function `mod.config._experts_implementation` names, for bf16 / fp16 weights: transformers'
    `ALL_EXPERTS_FUNCTIONS` entry ("batched_mm", "grouped_mm"), else the class's own loop under the dispatcher that
    transformers puts on `forward` (which would pick the fp8 functions)."""
    name = getattr(getattr(mod, "config", None), "_experts_implementation", None)
    if name not in (None, "eager"):
        from transformers.integrations.moe import ALL_EXPERTS_FUNCTIONS
        if name in ALL_EXPERTS_FUNCTIONS:
            return ALL_EXPERTS_FUNCTIONS[name]
    return inspect.unwrap(type(mod).forward)


def _fp8_experts_forward(mod, state, plan, names, fast: bool):
    """The forward of an fp8 experts module (W8A16: the activations are not quantized), called as experts(hidden_states,
    top_k_index, top_k_weights), positional or by keyword.  For bf16 / fp16 hidden_states on the plan's device, outside
    autocast, with CUDA int32 / int64 ids there: `plan.dequant_fp8_select` writes the routed experts' weights S * W in
    the input's dtype into the shared output buffer, they are bound as the weights, and `_experts_impl` runs on them.
    A module `fast` is False for (`dequant_fp8_select_ok` refuses it), and any other input, takes a selected run (the ids
    as above; else the whole decode) and torch's dequantize into fresh tensors instead, with the same result."""
    block = _fp8_block(mod)
    shapes = [tuple(o.shape) for o in plan.outputs]
    inf = [sh[-1] for sh in shapes]
    blocks = [block] * len(names)
    sizes = [2 * math.prod(sh) for sh in shapes]
    offs = [0]
    for n in sizes[:-1]:
        offs.append(offs[-1] + (n + 15) // 16 * 16)
    unbind = _unbind(names)

    def forward(*args, **kwargs):
        if torch.is_grad_enabled():
            _grad_mode_error(mod, shared=True)
        hidden = args[0] if args else kwargs.get("hidden_states")
        ids = args[1] if len(args) > 1 else kwargs.get("top_k_index")
        scales = [getattr(mod, name + "_scale_inv") for name, _ in names]
        on_device = (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.device == plan.device
                     and ids.dtype in (torch.int32, torch.int64))
        if (fast and on_device and isinstance(hidden, torch.Tensor) and hidden.dtype in (torch.bfloat16, torch.float16)
                and hidden.device == plan.device and not torch.is_autocast_enabled(plan.device.type)):
            outs = [plan._out[o: o + n].view(hidden.dtype).view(sh) for o, n, sh in zip(offs, sizes, shapes)]
            ws = plan.dequant_fp8_select(ids, inf, scales, blocks, hidden.dtype, outs=outs, scratch=state.select_scratch)
        else:
            dt = hidden.dtype if isinstance(hidden, torch.Tensor) and hidden.dtype in (torch.bfloat16, torch.float16, torch.float32) else torch.bfloat16
            coded = plan.run_select(ids, scratch=state.select_scratch) if on_device and plan.select_ok() else plan.run()
            ws = [dequantize_fp8(coded[k], s, block, dt) for (_, k), s in zip(names, scales)]
        _bind(mod, names, ws)
        try:
            return _experts_impl(mod)(mod, *args, **kwargs)
        finally:
            unbind(mod, args, None)
    return forward


def _fp8_experts_matvec_forward(mod, state, plan, names):
    """The forward of an "fp8_experts_matvec" module: the inputs the fast path of `_fp8_experts_forward` takes, with at
    most `state.experts_matvec` rows of hidden_states [T, H] and ids [T, k], are multiplied by the routed experts
    straight from the streams, nothing bound and the shared output buffer untouched: h = experts_matvec_fp8 of the first
    projection with x [T, H]; the gate (`_apply_gate`) or the activation; d = experts_matvec_fp8 of down_proj with x
    [T, k, I]; then FP8Experts.forward's combine, d times the routing weights in d's dtype, in fp32 summed over the k
    slots in ascending order, back to the input's dtype.  Every other input goes to `_fp8_experts_forward` as before."""
    fallback = _fp8_experts_forward(mod, state, plan, names, True)
    block = _fp8_block(mod)
    first, down = experts_matvec_layout(mod)
    where = dict(names)
    kf, kd = where[first], where[down]

    def forward(*args, **kwargs):
        hidden = args[0] if args else kwargs.get("hidden_states")
        ids = args[1] if len(args) > 1 else kwargs.get("top_k_index")
        weights = args[2] if len(args) > 2 else kwargs.get("top_k_weights")
        if not (not torch.is_grad_enabled() and isinstance(ids, torch.Tensor) and ids.is_cuda and ids.device == plan.device
                and ids.dtype in (torch.int32, torch.int64) and ids.dim() == 2 and isinstance(hidden, torch.Tensor)
                and hidden.dtype in (torch.bfloat16, torch.float16) and hidden.device == plan.device and hidden.dim() == 2
                and hidden.shape[0] == ids.shape[0] <= state.experts_matvec and isinstance(weights, torch.Tensor)
                and not torch.is_autocast_enabled(plan.device.type)):
            return fallback(*args, **kwargs)
        scratch = state.experts_matvec_scratch
        h = plan.experts_matvec_fp8(kf, ids, hidden, getattr(mod, first + "_scale_inv"), block, scratch=scratch)
        a = mod._apply_gate(h) if first == "gate_up_proj" else mod.act_fn(h)
        d = plan.experts_matvec_fp8(kd, ids, a, getattr(mod, down + "_scale_inv"), block, scratch=scratch)
        wd = (d * weights.to(d.dtype)[..., None]).to(torch.float32)
        acc = torch.zeros(wd.shape[0], wd.shape[2], dtype=torch.float32, device=wd.device)
        for j in range(wd.shape[1]):
            acc += wd[:, j]
        return acc.to(hidden.dtype)
    return forward


def _matvec_forward(mod, state, plan, k, names, dtype, device, matmul: int = 0):
    """The forward of a matvec module: an input of at most `state.matvec` rows (a host-side test of its shape) that has
    the weight's `dtype` and `device`, outside autocast, goes to `plan.matvec`; one of more rows and at most `matmul`
    (the module's limit: `matmul` for a "matmul" module, 0 for a "matvec" one) goes to `plan.matmul`.  Then nothing is
    decoded or bound.  Any other input (a larger one, another dtype, an autocast region: whatever F.linear accepts)
    takes the decode, bind, forward, unbind of the hooks every other compressed module has."""
    decoded = _decoded(mod, plan, names, torch.nn.Linear.forward)

    def forward(input):
        rows = _rows(input)
        if (rows is not None and rows <= max(state.matvec, matmul) and input.dtype == dtype and input.device == device
                and not torch.is_autocast_enabled(device.type)):
            if torch.is_grad_enabled():
                _grad_mode_error(mod)
            if rows <= state.matvec:
                return plan.matvec(k, input, bias=mod.bias, scratch=state.matvec_scratch)
            return plan.matmul(k, input, bias=mod.bias, scratch=state.matmul_scratch)
        return decoded(input)
    return forward


def _unbind(names):
    def hook(mod, args, output):
        for name, _ in names:
            mod.__dict__.pop(name, None)
    return hook


_EMPTY_REPORT = {"dense_bytes": 0, "stream_bytes": 0, "plan_bytes": 0, "index_bytes": 0, "scratch_bytes": 0, "out_bytes": 0,
                 "params": 0, "modules": 0}


def split_gathers(per_module, gather: bool) -> tuple:
    """[(module, [(name, stream index)])] -> (modules decoded whole, [(embedding, stream index)] looked up by gathers,
    the gathers' stream indexes no whole-decoded module holds: each needs a plan of its own)."""
    whole, looked = [], []
    for m, names in per_module:
        if gather and gathers(m) and [n for n, _ in names] == ["weight"]:
            looked.append((m, names[0][1]))
        else:
            whole.append((m, names))
    held = {i for _, names in whole for _, i in names}
    own = list(dict.fromkeys(i for _, i in looked if i not in held))
    return whole, looked, own


def _aligned_views(sizes: list, dev) -> tuple:
    """Byte sizes -> (one uint8 buffer, a view of each size in it): back to back, each at a 16-byte aligned offset,
    since the plans' recorded segment starts depend on a stream's address modulo 16."""
    offs, at = [], 0
    for n in sizes:
        offs.append(at)
        at = (at + n + 15) // 16 * 16
    buf = torch.empty(max(at, 1), dtype=torch.uint8, device=dev)
    return buf, [buf[o: o + n] for o, n in zip(offs, sizes)]


def _pack(streams: dict, dev) -> tuple:
    """{group index: CUDA uint8 stream} -> (one tight buffer holding them at 16-byte aligned offsets, {index: its
    view}); the sources are only read."""
    buf, views = _aligned_views([s.numel() for s in streams.values()], dev)
    for v, s in zip(views, streams.values()):
        v.copy_(s)
    return buf, dict(zip(streams, views))


def _resident_state(modules, groups, streams: dict, buffers: list, dev, opts: _Options) -> tuple:
    """The back half of compress_module and load_module: streams {group index: CUDA stream} -> per selected module
    one DecodePlan over its parameters' streams, all sharing one output and one scratch buffer.  Raises like
    `decompress` on a corrupt stream; nothing outside is touched until `_commit`.  -> (_Resident, report).

    gather=True: embeddings (`gathers`) get no output space.  One whose weight a whole-decoded module also holds (a
    tied lm_head) gathers through that module's plan; any other gets a plan of its own, created first, into a
    transient buffer that is freed before the shared output buffer exists (so the peak stays that of gather=False).

    Every other module is an `_Entry`, its plan and its room in the shared output buffer kept (larger inputs decode),
    in the first mode that applies: "matmul" for a `matvecs` module whose one compressed parameter is a weight that
    `DecodePlan.matmul_ok` accepts (matmul=N), "matvec" for one that only `DecodePlan.matvec_ok` accepts (matvec=N);
    "fp8" for an `fp8_linears` module whose one compressed parameter is its weight and which `DecodePlan.matvec_fp8_ok`
    accepts, "fp8_torch" for one it refuses (fp8=True; the shared output buffer holds at least twice such a weight's
    bytes, its dequantized weight); "fp8_experts" for an `fp8_experts` module whose compressed parameters are its fp8
    ones and whose plan `DecodePlan.select_ok` and `DecodePlan.dequant_fp8_select_ok` accept, "fp8_experts_torch" for
    one they refuse (fp8=True and experts=True; the shared output buffer holds at least 2 bytes per fp8 element of such
    a module, its dequantized weights); "experts" for an `experts_module` whose plan passes `DecodePlan.select_ok`
    (experts=True); else "prefetch" with prefetch=True, "decode" without."""
    where = {id(groups[i][0]): i for i in streams}
    per_module = []
    for m in modules:
        names = [(n, where[id(p)]) for n, p in _own_params(m) if id(p) in where]
        if names:
            per_module.append((m, names))
    whole, looked, own = split_gathers(per_module, opts.gather)
    sizes = [DecodePlan.sizes([streams[i] for _, i in names]) for _, names in whole]
    own_sizes = [DecodePlan.sizes([streams[i]]) for i in own]
    fp8_mods = {id(m) for m, names in whole if opts.fp8 and fp8_linears(m) and [n for n, _ in names] == ["weight"]}
    # fp8 experts whose fp8 parameters, and only those, are compressed; their dequantized weights go to the shared buffer
    fp8_exp = {id(m) for m, names in whole if opts.fp8 and opts.experts and fp8_experts(m)
               and sorted(n for n, _ in names) == sorted(n for n, p in _own_params(m) if p.dtype in _FP8)}
    out_need = max([s[0] for s in sizes] + [2 * m.weight.numel() for m, _ in whole if id(m) in fp8_mods]
                   + [sum((2 * groups[i][0].numel() + 15) // 16 * 16 for _, i in names) for m, names in whole if id(m) in fp8_exp]
                   + [1])
    out = None if own else torch.empty(out_need, dtype=torch.uint8, device=dev)
    scratch = torch.empty(max([s[1] for s in sizes + own_sizes] + [1]), dtype=torch.uint8, device=dev)
    state = _Resident()
    state.streams = buffers
    state.scratch = scratch
    plan_bytes = index_bytes = 0
    by_stream = {}   # stream index -> (plan, output index) a gather reads
    for i, (out_bytes, _) in zip(own, own_sizes):
        transient = torch.empty(max(out_bytes, 1), dtype=torch.uint8, device=dev)
        plan = DecodePlan([streams[i]], out=transient, scratch=scratch)
        plan.release_out()
        del transient
        by_stream[i] = (plan, 0)
        state.gather_plan_bytes += plan.nbytes["plan"]
        index_bytes += plan.nbytes["index"]
    if out is None:
        out = torch.empty(out_need, dtype=torch.uint8, device=dev)
    for m, names in whole:
        plan = DecodePlan([streams[i] for _, i in names], out=out, scratch=scratch)
        plan_bytes += plan.nbytes["plan"]
        index_bytes += plan.nbytes["index"]
        local = [(n, k) for k, (n, _) in enumerate(names)]
        for k, (_, i) in enumerate(names):
            by_stream.setdefault(i, (plan, k))
        linear = matvecs(m) and local == [("weight", 0)]
        mm = bool(opts.matmul) and linear and plan.matmul_ok(0, m.in_features)
        if mm or (opts.matvec and linear and plan.matvec_ok(0, m.in_features)):
            mode = "matmul" if mm else "matvec"
        elif id(m) in fp8_mods:
            block = _fp8_block(m)
            mode = "fp8" if plan.matvec_fp8_ok(0, m.in_features) and (block is None or block[1] % 16 == 0) else "fp8_torch"
        elif id(m) in fp8_exp:
            block = _fp8_block(m)
            fast = plan.select_ok() and plan.dequant_fp8_select_ok([o.shape[-1] for o in plan.outputs])
            mode = "fp8_experts" if fast and (block is None or block[1] % 16 == 0) else "fp8_experts_torch"
            if mode == "fp8_experts" and opts.experts_matvec and experts_matvec_layout(m) is not None and all(
                    plan.experts_matvec_fp8_ok(k, plan.outputs[k].shape[-1]) for _, k in local):
                mode = "fp8_experts_matvec"
        elif opts.experts and experts_module(m, [n for n, _ in local]) and plan.select_ok():
            mode = "experts"
        else:
            mode = "prefetch" if opts.prefetch else "decode"
        state.entries.append(_Entry(m, plan, local, mode))
    for m, i in looked:
        plan, k = by_stream[i]
        state.gathers.append((m, plan, k, i in own))
    dense = 0
    for i in streams:
        p, owners = groups[i]
        dense += p.numel() * p.element_size()
        state.params[i] = (p.requires_grad, p.dtype, tuple(p.shape), owners)
    state.stream_of = dict(streams)
    return state, {"dense_bytes": dense, "stream_bytes": sum(s.numel() for s in streams.values()), "plan_bytes": plan_bytes,
                   "index_bytes": index_bytes, "scratch_bytes": scratch.numel(), "out_bytes": out.numel(),
                   "params": len(streams), "modules": len(per_module)}


def _plans_scratch_or_own(state: _Resident, need: int):
    """The plans' scratch if it holds `need` bytes, else a buffer of `need` bytes."""
    return state.scratch if need <= state.scratch.numel() else torch.empty(need, dtype=torch.uint8, device=state.scratch.device)


def _commit(module: torch.nn.Module, state: _Resident, opts: _Options) -> None:
    """Hooks and forwards on, compressed parameters out: after this the model runs from its streams."""
    sched = None
    if opts.prefetch and state.entries:
        plans = [e.plan for e in state.entries]
        slot1 = torch.empty_like(plans[0]._out)
        slots = [plans[0]._out, slot1]
        sched = _prefetch.Prefetcher(_prefetch.CudaOps(plans[0].device, plans, slots, _prefetch.prefetch_ctas()))
        roots = [module.register_forward_pre_hook(lambda mod, args: sched.root_begin(), prepend=True),
                 module.register_forward_hook(lambda mod, args, output: sched.root_end(), always_call=True)]
        state.prefetch = (sched, slot1, roots)
    if state.gathers:
        # the plans' scratch, whose runs share the forward's stream; with prefetch those runs move to the side stream,
        # so the gathers get a buffer of their own, of the plans' scratch's size at least.  One slot at least.
        need = max(plan.gather_scratch_bytes(k, 1) for _, plan, k, _ in state.gathers)
        if opts.prefetch or need > state.scratch.numel():
            state.gather_scratch = torch.empty(max(need, state.scratch.numel()), dtype=torch.uint8, device=state.scratch.device)
        else:
            state.gather_scratch = state.scratch
        for m, plan, k, _ in state.gathers:
            m.__dict__["forward"] = _gather_forward(m, state, plan, k)
    state.matvec = opts.matvec
    matvec = [e for e in state.entries if e.mode in ("matvec", "matmul")]
    matmul = [e for e in state.entries if e.mode == "matmul"]
    experts = [e for e in state.entries if e.mode == "experts" or (e.mode.startswith("fp8_experts") and e.plan.select_ok())]
    fp8 = [e for e in state.entries if e.mode == "fp8"]
    if matvec and opts.matvec:
        state.matvec_scratch_bytes = max(e.plan.matvec_scratch_bytes(0, e.module.in_features, opts.matvec) for e in matvec)
        state.matvec_scratch = _plans_scratch_or_own(state, state.matvec_scratch_bytes)
    if matmul:
        state.matmul_scratch_bytes = max(e.plan.matmul_scratch_bytes(0, e.module.in_features, opts.matmul) for e in matmul)
        state.matmul_scratch = _plans_scratch_or_own(state, state.matmul_scratch_bytes)
    if experts:
        # always a buffer of its own: run_select and dequant_fp8_select must not be given the plans' scratch
        need = max(e.plan.select_scratch_bytes() for e in experts)
        state.select_scratch = torch.empty(need, dtype=torch.uint8, device=state.scratch.device)
    if fp8 and opts.matvec:
        state.fp8_scratch_bytes = max(e.plan.matvec_fp8_scratch_bytes(0, e.module.in_features, opts.matvec) for e in fp8)
        state.fp8_scratch = _plans_scratch_or_own(state, state.fp8_scratch_bytes)
    state.fp8_matmul = opts.fp8_matmul
    if fp8 and opts.fp8_matmul:
        state.fp8_matmul_scratch_bytes = max(e.plan.matmul_fp8_scratch_bytes(0, e.module.in_features, opts.fp8_matmul) for e in fp8)
        state.fp8_matmul_scratch = _plans_scratch_or_own(state, state.fp8_matmul_scratch_bytes)
    state.experts_matvec = opts.experts_matvec
    em = [e for e in state.entries if e.mode == "fp8_experts_matvec"]
    if em:   # (top_k = E bounds the pair tables of any routing)
        state.experts_matvec_scratch_bytes = max(e.plan.experts_matvec_fp8_scratch_bytes(k, e.plan.outputs[k].shape[-1], e.module.num_experts,
                                                                                           opts.experts_matvec)
                                                 for e in em for _, k in e.names)
        state.experts_matvec_scratch = _plans_scratch_or_own(state, state.experts_matvec_scratch_bytes)
    for key, (m, plan, names, mode) in enumerate(state.entries):
        if mode in ("matvec", "matmul"):   # no hooks: its forward decides per input whether anything is decoded
            m.__dict__["forward"] = _matvec_forward(m, state, plan, 0, names, plan.outputs[0].dtype, plan.device,
                                                    opts.matmul if mode == "matmul" else 0)
        elif mode in ("fp8", "fp8_torch"):   # no hooks either: its forward multiplies from the stream, or decodes
            m.__dict__["forward"] = _fp8_forward(m, state, plan, 0, names, mode == "fp8")
        elif mode in ("fp8_experts", "fp8_experts_torch"):   # its forward binds the dequantized weights itself
            m.__dict__["forward"] = _fp8_experts_forward(m, state, plan, names, mode == "fp8_experts")
        elif mode == "fp8_experts_matvec":   # no binding at all for a few tokens; more take the "fp8_experts" forward
            m.__dict__["forward"] = _fp8_experts_matvec_forward(m, state, plan, names)
        else:
            if mode == "experts":
                pre = m.register_forward_pre_hook(_pre_hook_experts(plan, names, state), with_kwargs=True)
            elif mode == "prefetch":
                pre = m.register_forward_pre_hook(_pre_hook_prefetch(sched, key, names, [plan.views(b) for b in sched.ops.slots]))
            else:
                pre = m.register_forward_pre_hook(_pre_hook(plan, names))
            state.hooks += [pre, m.register_forward_hook(_unbind(names), always_call=True)]
    # the dense parameters go: nothing here keeps their storage alive
    for _, _, _, owners in state.params.values():
        for o, n in owners:
            state.order.setdefault(id(o), (o, list(o._parameters)))
            del o._parameters[n]
    setattr(module, _ATTR, state)


def compress_module(module: torch.nn.Module, modules=None, prefetch: bool = False, gather: bool = False, matvec: int = 0,
                    matmul: int = 0, experts: bool = False, fp8: bool = False, fp8_matmul: int = 0, experts_matvec: int = 0) -> dict:
    """Compress the weights of `modules` (default: every submodule that directly owns bf16 / fp16 / fp32 / fp8
    parameters) into streams kept in HBM, decoded just before each module's forward.  All parameters are compressed
    in one `compress_batch` call and must be on one CUDA device.

    -> {"dense_bytes", "stream_bytes", "plan_bytes", "index_bytes", "scratch_bytes", "out_bytes", "params",
        "modules"}: bytes of the parameters now compressed, of their streams, of the plans' memory, of the segment
    index (the recorded segment starts, part of the plans' memory), of the shared plane scratch and of the shared output buffer
    (the size of the largest module's decoded weights).

    prefetch=True: decode each module's weights on a side stream while the module before it computes (prefetch.py),
    into a second output buffer of the shared one's size; the report gains "prefetch_out_bytes", that buffer's bytes.

    gather=True: a selected embedding whose weight is compressed (`gathers`) runs its forward as
    `DecodePlan.gather` and is never decoded whole.  A tied lm_head keeps its whole decode and the embedding gathers
    through the same plan; an untied one gets a plan of its own.  Embeddings take no room in the shared output buffer
    ("out_bytes": the largest module decoded whole), and their plans are not in "plan_bytes" (their indexes are in
    "index_bytes").  The gathers use the plans' scratch (they run on the forward's stream, as the plans do), or with
    prefetch=True a buffer of its own.  The report gains "gather_modules" and "gather_bytes": memory that exists only
    for gathers, i.e. the plans of their own plus a scratch of their own.

    matvec=N (1 .. MATVEC_MAX_TOKENS; 0, the default, changes nothing): a selected `torch.nn.Linear` (`matvecs`) whose
    weight `DecodePlan.matvec_ok` accepts computes inputs of at most N rows (product of the leading dims) as
    `DecodePlan.matvec` -- two launches, the weight neither decoded nor bound -- and larger inputs as before.  The
    results of the small inputs are fp32 sums rounded once, so they differ from the dense model's in the last bits.
    The bias of every `matvecs` module stays a dense parameter, whether or not its weight turns out eligible (that is
    known only once the streams exist): against matvec=0 the report's "params", "dense_bytes" and "stream_bytes" lack
    those biases, which stay resident dense.  Inputs of another dtype or device than the weight, and inputs inside an
    autocast region, take the decode path whatever their size.  A tied weight keeps one stream; each owner has its
    plan as before.  The shared output buffer stays, since larger inputs (prefill) decode into it.  The report gains
    "matvec_modules" and "matvec_scratch_bytes" (one scratch for all of them, sized for the largest; the plans'
    scratch when that is large enough).  ValueError together with prefetch=True.

    matmul=N (0 .. MATMUL_MAX_TOKENS; 0, the default, changes nothing): a `matvecs` module whose bf16 / fp16 weight
    `DecodePlan.matmul_ok` accepts computes inputs of more than `matvec` rows and at most N as `DecodePlan.matmul`
    (tensor cores, two launches, the weight neither decoded nor bound); inputs of at most `matvec` rows still take the
    matvec, larger ones, other dtypes or devices and autocast regions the decode.  The biases stay dense as for
    matvec.  The report gains "matmul_modules" and "matmul_scratch_bytes" (one scratch for all of them, as for the
    matvec).  ValueError together with prefetch=True.

    experts=True (default False, which changes nothing): a selected module that `experts_module` accepts, and whose
    plan `DecodePlan.select_ok` accepts, decodes through a forward pre-hook that takes the ids from its forward's second
    positional argument or keyword `top_k_index` (transformers' `experts(hidden_states, top_k_index, top_k_weights)`).
    For CUDA int32 / int64 ids on the plan's device the hook runs `DecodePlan.run_select`: only the chunks of the
    experts those ids name are decoded; any other call decodes the whole module.  The module's own forward then reads
    only the slices [e] of the routed experts, so its outputs equal the dense module's bit for bit, whichever experts
    implementation it uses; the other slices of the shared buffer hold stale bytes.  The report gains
    "experts_modules" and "experts_scratch_bytes" (one run_select scratch shared by them all, sized for the largest).
    ValueError together with prefetch=True.

    fp8=True (default False, which changes nothing): the W8A16 reading of fp8 checkpoints.  A selected `fp8_linears`
    module (transformers' `FP8Linear`) compresses only its weight; `weight_scale_inv`, `bias` and `activation_scale`
    stay dense parameters.  Its forward multiplies bf16 / fp16 inputs on the weight's device, outside autocast, with the
    dequantized weight S * W in the input's dtype -- it does not quantize the activations, so it is not FP8Linear's own
    W8A8 forward, and it needs no downloaded kernel: inputs of at most `matvec` rows go to `DecodePlan.matvec_fp8`
    (fp32 sums rounded once), larger ones to `DecodePlan.dequant_fp8` into the shared output buffer and F.linear (bit for
    bit F.linear of torch's dequantize), then the bias is added as FP8Linear adds it.  So fp8=True, matvec=8 is the
    decode-time setting.  A weight that `DecodePlan.matvec_fp8_ok` refuses (a constant one, say) is decoded and
    dequantized in torch instead, with the same result.  Other inputs decode and run the module's own forward.  The
    shared output buffer holds at least twice the largest such weight's bytes.  `matmul` does not apply to fp8 weights;
    `fp8_matmul` (below) is their tensor-core path.
    The report gains "fp8_modules" and "fp8_scratch_bytes" (the matvec_fp8 scratch, the plans' one when it is large
    enough).  ValueError together with prefetch=True.

    fp8=True and experts=True together (either alone changes nothing here): a selected `fp8_experts` module
    (transformers' `FP8Experts`) compresses only its fp8 weights; the `*_scale_inv` grids and static activation scales
    stay dense parameters.  Its forward takes bf16 / fp16 hidden_states on the weights' device, outside autocast, with
    CUDA int32 / int64 `top_k_index` there: `DecodePlan.dequant_fp8_select` writes only the routed experts' weights,
    dequantized to the input's dtype (bit for bit torch's dequantize), into the shared output buffer, and the experts
    implementation `config._experts_implementation` names runs on them -- the class's own loop for "eager",
    transformers' bf16 `batched_mm` / `grouped_mm` functions for those -- so it needs no downloaded kernel and does not
    quantize the activations.  A module whose plan `dequant_fp8_select_ok` refuses, and any other input, takes a
    selected run (or the whole decode) and torch's dequantize instead, with the same result.  The shared output buffer
    holds at least 2 bytes per fp8 element of such a module; the selected-run scratch ("experts_scratch_bytes") serves
    both kinds of experts modules.  The report of a model with such modules gains "fp8_experts_modules".

    fp8_matmul=N (0 .. MATMUL_MAX_TOKENS; 0, the default, changes nothing): with fp8=True, an fp8 module whose weight
    `DecodePlan.matvec_fp8_ok` accepts computes bf16 / fp16 inputs of more than `matvec` rows and at most N as
    `DecodePlan.matmul_fp8` (tensor cores, two launches, the weight neither dequantized into the shared buffer nor
    read back): F.linear of the same dequantized weight, with the fp32 sums in another order.  Inputs of at most
    `matvec` rows still take matvec_fp8, larger ones dequant_fp8 + F.linear.  The report gains "fp8_matmul_modules" and
    "fp8_matmul_scratch_bytes" (one scratch for all of them, the plans' one when it is large enough).  ValueError
    without fp8=True and together with prefetch=True.

    experts_matvec=N (0 .. EXPERTS_MATVEC_MAX_TOKENS; 0, the default, changes nothing): with fp8=True and experts=True,
    an "fp8_experts" module in one of transformers' `FP8Experts` layouts (`experts_matvec_layout`) whose plan
    `DecodePlan.experts_matvec_fp8_ok` accepts for both projections runs as "fp8_experts_matvec": bf16 / fp16 inputs of
    at most N tokens are multiplied by the routed experts straight from the streams (`DecodePlan.experts_matvec_fp8`,
    no weight written or bound), then gated and combined as FP8Experts.forward does; larger inputs take the
    "fp8_experts" forward.  The report gains "experts_matvec_modules" and "experts_matvec_scratch_bytes" (one scratch
    for all of them, the plans' one when it is large enough).  ValueError without both fp8=True and experts=True."""
    opts = _options(prefetch, gather, matvec, matmul, experts, fp8, fp8_matmul, experts_matvec)
    if getattr(module, _ATTR, None) is not None:
        raise ValueError("compress_module: this module is already compressed")
    modules, groups = select(module, modules)
    groups = dense_biases(groups, max(opts.matvec, opts.matmul), opts.fp8, opts.experts)
    params = [p for p, _ in groups]
    if not params:
        setattr(module, _ATTR, None)
        return dict(_EMPTY_REPORT)
    if not all(p.is_cuda for p in params) or len({p.device for p in params}) > 1:
        raise ValueError("compress_module: the selected parameters must lie on one CUDA device")
    dev = params[0].device
    with torch.no_grad():   # the .znn files' method byte: the streams are the ones save_file writes, byte for byte
        coded = ZipNN(input_format="torch", method=COMPRESSION_METHOD).compress_batch([p.detach() for p in params])
    # the streams move into one tight buffer; the batch's output buffer (sized by the bound) is dropped
    buf, streams = _pack({i: s for i, (p, s) in enumerate(zip(params, coded)) if s.numel() < p.numel() * p.element_size()}, dev)
    del coded, params
    state, report = _resident_state(modules, groups, streams, [buf], dev, opts)
    _commit(module, state, opts)
    return _with_prefetch(report, state, opts)


def _with_prefetch(report: dict, state, opts: _Options) -> dict:
    """`report` with the keys of every mode `opts` turns on, prefetch's and the others'; all 0 for a model with nothing
    compressed (state None)."""
    state = _Resident() if state is None else state
    modes = [e.mode for e in state.entries]
    report = dict(report)
    if opts.prefetch:
        report.update(prefetch_out_bytes=state.prefetch[1].numel() if state.prefetch else 0)
    if opts.gather:
        own = state.gather_scratch is not None and state.gather_scratch is not state.scratch
        report.update(gather_modules=len(state.gathers), gather_bytes=state.gather_plan_bytes + (state.gather_scratch.numel() if own else 0))
    if opts.matvec:
        report.update(matvec_modules=modes.count("matvec") + modes.count("matmul"), matvec_scratch_bytes=state.matvec_scratch_bytes)
    if opts.matmul:
        report.update(matmul_modules=modes.count("matmul"), matmul_scratch_bytes=state.matmul_scratch_bytes)
    if opts.experts:
        report.update(experts_modules=modes.count("experts"),
                      experts_scratch_bytes=0 if state.select_scratch is None else state.select_scratch.numel())
    if opts.fp8:
        report.update(fp8_modules=modes.count("fp8") + modes.count("fp8_torch"), fp8_scratch_bytes=state.fp8_scratch_bytes)
    fp8_experts_modules = modes.count("fp8_experts") + modes.count("fp8_experts_torch") + modes.count("fp8_experts_matvec")
    if fp8_experts_modules:   # (only fp8=True with experts=True makes them; a model without one keeps its report)
        report.update(fp8_experts_modules=fp8_experts_modules)
    if opts.fp8_matmul:
        report.update(fp8_matmul_modules=modes.count("fp8"), fp8_matmul_scratch_bytes=state.fp8_matmul_scratch_bytes)
    if opts.experts_matvec:
        report.update(experts_matvec_modules=modes.count("fp8_experts_matvec"),
                      experts_matvec_scratch_bytes=state.experts_matvec_scratch_bytes)
    return report


def decompress_module(module: torch.nn.Module) -> None:
    """Undo `compress_module`: every compressed parameter becomes a dense `Parameter` again (tied ones one shared
    object again), bit for bit; the hooks, plans and streams are released."""
    state = getattr(module, _ATTR, None)
    if state is None:
        if hasattr(module, _ATTR):
            delattr(module, _ATTR)
            return
        raise ValueError("decompress_module: this module was not compressed by compress_module")
    if state.prefetch is not None:
        sched, _, roots = state.prefetch
        torch.cuda.current_stream(sched.ops.dev).wait_stream(sched.ops.side)
        for h in roots:
            h.remove()
        sched.ops.slots = None   # slot 1 goes with the state
        state.prefetch = None
    for h in state.hooks:
        h.remove()
    for m, _, _, mode in state.entries:
        if mode in ("matvec", "matmul", "fp8", "fp8_torch", "fp8_experts", "fp8_experts_torch", "fp8_experts_matvec"):   # the modes whose forward _commit replaced
            m.__dict__.pop("forward", None)
    for m, _, _, _ in state.gathers:
        m.__dict__.pop("forward", None)
    # each module's plan decodes into the shared buffer once more; its parameters are copied out of it, so the
    # model needs its dense size plus that buffer, not twice its dense size
    dense = {}
    idx_of = {id(t): i for i, t in state.stream_of.items()}
    with torch.no_grad():
        for m, plan, local, _ in state.entries:
            outs = plan.run()
            for (name, k), s_ in zip(local, plan._streams):
                i = idx_of[id(s_)]
                if i not in dense:
                    dense[i] = outs[k].clone()
        for m, plan, k, _ in state.gathers:   # an embedding of its own plan: every row, gathered
            i = idx_of[id(plan._streams[k])]
            if i not in dense:
                rows = state.params[i][2][0]
                dense[i] = plan.gather(k, torch.arange(rows, device=plan.device), scratch=state.gather_scratch)
    for i, t in dense.items():
        requires_grad, _, _, owners = state.params[i]
        p = torch.nn.Parameter(t, requires_grad=requires_grad)
        for o, n in owners:
            o.__dict__.pop(n, None)
            o._parameters[n] = p
    # the parameters go back to where they were in each module's _parameters (named_parameters / state_dict order)
    for o, names in state.order.values():
        params = o._parameters
        reordered = {n: params[n] for n in names if n in params}
        reordered.update((n, v) for n, v in params.items() if n not in reordered)
        params.clear()
        params.update(reordered)
    state.entries.clear()
    state.gathers.clear()
    delattr(module, _ATTR)


def state_names(module: torch.nn.Module) -> list:
    """`module`'s full dense state in `state_dict()` order, compressed parameters at their owners' names (where
    `decompress_module` would put them back): [(name, owner module, attribute, kind, key)], kind "param" (a dense
    Parameter), "resident" (a compressed one) or "buffer" (a persistent buffer); every name of one tensor has the
    same key."""
    state = getattr(module, _ATTR, None)
    resident = {}
    if state is not None:
        for i, (_, _, _, owners) in state.params.items():
            for o, n in owners:
                resident[(id(o), n)] = i
    out = []

    def walk(m, prefix):
        names = list(m._parameters)
        if state is not None and id(m) in state.order:
            first = state.order[id(m)][1]
            names = first + [n for n in names if n not in first]
        for n in names:
            p = m._parameters.get(n)
            if p is not None:
                out.append((prefix + n, m, n, "param", id(p)))
            elif (id(m), n) in resident:
                out.append((prefix + n, m, n, "resident", ("resident", resident[(id(m), n)])))
        for n, b in m._buffers.items():
            if b is not None and n not in m._non_persistent_buffers_set:
                out.append((prefix + n, m, n, "buffer", id(b)))
        for n, c in m._modules.items():
            if c is not None:
                walk(c, prefix + n + ".")

    walk(module, "")
    return out


def first_names(entries) -> tuple:
    """`state_names` -> (the first name of every tensor, the later names of tied tensors)."""
    seen, first, later = set(), [], []
    for e in entries:
        (later if e[4] in seen else first).append(e)
        seen.add(e[4])
    return first, later


class LoadPlan:
    """What `load_module` does with each key, decided from the module and the files' headers alone."""

    def __init__(self, modules, groups):
        self.modules, self.groups = modules, groups   # as `select` gives them
        self.streams = []   # (group index, FileEntry): compressed entries that stay compressed, read as they are
        self.compress = []  # (group index, FileEntry): plain floating-point entries, compressed on the device
        self.dense = []     # (FileEntry, [(module, attribute)], kind, requires_grad): read (and decoded) to dense
        self.moves = []     # (module, name): non-persistent buffers, moved to the device
        self.kinds = {}     # every state name -> "stream", "compress", "dense" or "alias" (not read)


def _stream_header(e) -> _Stream:
    """The header of a compressed entry, checked as DecodePlan checks it, read from the file (no device work)."""
    with open(e.file, "rb") as f:
        f.seek(e.offset)
        head = f.read(min(e.nbytes, _HEAD))
    return _Stream(torch.empty(e.nbytes, dtype=torch.uint8, device="meta"), head)


def _files(filenames) -> list:
    if isinstance(filenames, (str, os.PathLike)):
        return [os.fspath(filenames)]
    return [os.fspath(f) for f in filenames]


def plan_load(module: torch.nn.Module, filenames, modules=None, matvec: int = 0, fp8: bool = False, experts: bool = False) -> LoadPlan:
    """The checks and choices of `load_module`, from the files' headers: ValueError naming the keys for a missing or
    unexpected key, a dtype or shape that differs, a non-persistent buffer on the meta device, and for a module that
    is already compressed."""
    if getattr(module, _ATTR, None) is not None:
        raise ValueError("load_module: this module is already compressed")
    found = file_entries(_files(filenames))
    modules, groups = select(module, modules)
    groups = dense_biases(groups, matvec, fp8, experts)   # (matvec=N, fp8=True: the parameters that stay dense are read so)
    plan = LoadPlan(modules, groups)
    group_of = {id(p): gi for gi, (p, _) in enumerate(groups)}
    by_key = {}
    for name, m, attr, kind, key in state_names(module):
        by_key.setdefault(key, []).append((name, m, attr, kind))
    missing = [names[0][0] for names in by_key.values() if not any(n in found for n, _, _, _ in names)]
    known = {n for names in by_key.values() for n, _, _, _ in names}
    unexpected = sorted(k for k in found if k not in known)
    if missing or unexpected:
        raise ValueError(f"load_module: keys the files lack: {missing}; keys the module lacks: {unexpected}")
    meta = []
    for prefix, m in module.named_modules():
        for n in m._non_persistent_buffers_set:
            b = m._buffers.get(n)
            if b is not None:
                if b.is_meta:
                    meta.append(prefix + ("." if prefix else "") + n)
                else:
                    plan.moves.append((m, n))
    if meta:
        raise ValueError(f"load_module: non-persistent buffers on the meta device (no file holds them): {meta}")
    wrong = []
    for key, names in by_key.items():
        name, m, attr, kind = next(n for n in names if n[0] in found)
        for n in names:
            plan.kinds[n[0]] = "alias"
        e = found[name]
        t = m._parameters[attr] if kind == "param" else m._buffers[attr]
        if e.dtype != t.dtype or e.shape != tuple(t.shape):
            wrong.append(f"{name}: {e.dtype} {list(e.shape)} in the file, {t.dtype} {list(t.shape)} in the module")
            continue
        if e.compressed:
            try:
                s = _stream_header(e)
            except (ValueError, RuntimeError) as err:
                wrong.append(f"{name}: {err}")
                continue
            if s.dtype != e.dtype or s.shape != e.shape or s.nbytes != t.numel() * t.element_size():
                wrong.append(f"{name}: its stream holds {s.dtype} {list(s.shape)}, the metadata says {e.dtype} {list(e.shape)}")
                continue
        gi = group_of.get(key) if kind == "param" else None
        if gi is not None and e.compressed:
            plan.streams.append((gi, e))
            plan.kinds[name] = "stream"
        elif gi is not None and e.floating and not e.znn_file:   # a .znn file stored it raw: it does not compress
            plan.compress.append((gi, e))
            plan.kinds[name] = "compress"
        else:
            plan.dense.append((e, [(n[1], n[2]) for n in names], kind, kind == "param" and t.requires_grad))
            plan.kinds[name] = "dense"
    if wrong:
        raise ValueError(f"load_module: dtype or shape differs (no casting): {wrong}")
    plan.streams.sort(key=lambda g: g[0])
    plan.compress.sort(key=lambda g: g[0])
    return plan


def _load_device(plan: LoadPlan, dev, opts: _Options) -> tuple:
    """Every device step of load_module; the module is not touched.  -> (_Resident or None, report, dense tensors of
    plan.dense, {group index: dense tensor} of plain entries that did not compress, moved buffers of plan.moves)."""
    pipe = DecodePipe(dev)
    fds = {}

    def fd(fn):
        if fn not in fds:
            fds[fn] = os.open(fn, os.O_RDONLY)
        return fds[fn]

    def upload(dst, e):   # file bytes -> device through the pipe's pinned slab ring
        if e.nbytes:
            pipe._upload(dst, e.nbytes, lambda d, a, b: pipe._fill_from_file(d, fd(e.file), e.offset + a), cur)

    try:
        with torch.cuda.device(dev), torch.no_grad():
            cur = torch.cuda.current_stream()
            # compressed entries of selected parameters: one buffer, each stream at a 16-byte aligned offset, never
            # decoded but by plan create
            buffers, streams = [], {}
            if plan.streams:
                buf, views = _aligned_views([e.nbytes for _, e in plan.streams], dev)
                buffers.append(buf)
                for (gi, e), v in zip(plan.streams, views):
                    streams[gi] = v
                    upload(v, e)
            # plain floating-point entries of selected parameters: compressed a group at a time, compress_module's rule
            entries = [(gi, _FileRange(fd(e.file), e.offset, e.nbytes, e.dtype, e.shape)) for gi, e in plan.compress]
            stayed = {}
            for g in compress_groups(entries, dev):
                small = {}
                for k, i in enumerate(g.grp):
                    gi = entries[i][0]
                    if g.streams[k].numel() < entries[i][1].nbytes:
                        small[gi] = g.streams[k]
                    else:
                        stayed[gi] = g.flats[k].clone()
                if small:
                    buf, views = _pack(small, dev)
                    buffers.append(buf)
                    streams.update(views)
                del g, small
            # everything else becomes dense; compressed entries through the batched decode, one call per run of
            # entries that lie back to back in a file (a call reads the span from its first to its last entry)
            dense, runs = [None] * len(plan.dense), {}
            for j, (e, _, _, _) in enumerate(plan.dense):
                if e.compressed:
                    runs.setdefault(e.file, []).append(j)
                else:
                    dense[j] = torch.empty(e.shape, dtype=e.dtype, device=dev)
                    upload(dense[j].view(-1).view(torch.uint8), e)
            for fn, js in runs.items():
                js.sort(key=lambda j: plan.dense[j][0].offset)
                run = []
                for j in js + [None]:
                    e = plan.dense[j][0] if j is not None else None
                    if run and (e is None or plan.dense[run[-1]][0].offset + plan.dense[run[-1]][0].nbytes != e.offset):
                        got = pipe.submit_file_batch(fd(fn), [(plan.dense[r][0].offset, plan.dense[r][0].nbytes) for r in run])
                        for r, t in zip(run, got):
                            er = plan.dense[r][0]
                            dense[r] = t if t is not None else pipe.submit_file(fd(fn), er.offset, er.nbytes)
                        run = []
                    if j is not None:
                        run.append(j)
            pipe.finish()
            moved = [m._buffers[n].to(dev) for m, n in plan.moves]
            if plan.groups:
                state, report = _resident_state(plan.modules, plan.groups, dict(sorted(streams.items())), buffers, dev, opts)
            else:
                state, report = None, dict(_EMPTY_REPORT)
        return state, report, dense, stayed, moved
    finally:
        pipe.release()
        for f in fds.values():
            os.close(f)


def load_module(module: torch.nn.Module, filenames, device="cuda", modules=None, prefetch: bool = False,
                gather: bool = False, matvec: int = 0, matmul: int = 0, experts: bool = False, fp8: bool = False,
                fp8_matmul: int = 0, experts_matvec: int = 0) -> dict:
    """Load a checkpoint into `module` with the weights of `modules` kept compressed on `device`: the state
    `compress_module` leaves (same selection rules, hooks, plans and report), reached without a dense copy of those
    weights on the GPU.

    filenames: one path or a list of paths, the shards of one checkpoint, .safetensors and .znn.safetensors mixed (the
    index JSON is not read).  The module's parameters and buffers may be on the meta device, the CPU or `device`.

    Keys follow `load_state_dict(strict=True)`: every key of the module's dense `state_dict()` must be in the files
    and every key of the files in the module, but for tied parameters: one name of a tied parameter is enough (as
    `save_module`, `safetensors.torch.save_model` and Hugging Face checkpoints store them); if several are present the
    first in `state_dict()` order is read and the others are not.  Dtypes and shapes must match (no casting); for a
    compressed entry both the `znn_compressed_vectors` metadata and the stream's header are checked.  Each violation,
    a non-persistent buffer on the meta device and an already compressed module raise ValueError naming the keys,
    from the headers, before any device allocation.

    Where each entry goes:
      * a compressed entry of a selected parameter: its stream is read from the file (through DecodePipe's pinned slab
        ring) into one device buffer at a 16-byte aligned offset and stays compressed;
      * a plain floating-point entry of a selected parameter (plain .safetensors files): compressed on the device in
        groups of SAVE_GROUP_BYTES input bytes; it stays compressed when its stream is smaller, else dense;
      * everything else (unselected parameters, ones tied to an unselected owner, entries a .znn file stored raw,
        non-float tensors, buffers): a dense tensor on `device`; compressed ones through the batched decode.  A
        parameter becomes a new Parameter with the old one's requires_grad, shared by every owner of a tied one.
      Non-persistent buffers move to `device`.

    Atomic: the module is changed only after every plan exists (plan create finds a corrupt stream and raises as
    `decompress` does); on any error the module keeps its tensors, hooks and attributes and the device memory this
    call allocated is released.

    Device memory: what stays (streams, plans, shared scratch and output buffer, dense tensors) plus transients -- the
    plans' header peeks (up to 2.3 KB per stream), and for compressed entries that become dense their compressed bytes
    and the batched decode's workspace; plain entries add one group at a time: its input, its streams' bound and the
    compress workspace.  A model loaded from .znn files never has its compressed weights dense on the device.

    prefetch, gather, matvec, matmul, experts, fp8, fp8_matmul, experts_matvec: as for `compress_module`.

    -> the report of `compress_module`."""
    opts = _options(prefetch, gather, matvec, matmul, experts, fp8, fp8_matmul, experts_matvec)
    dev = _cuda_device(device)
    if dev is None:
        raise ValueError(f"load_module: {device!r} is not a CUDA device")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    plan = plan_load(module, filenames, modules, max(opts.matvec, opts.matmul), opts.fp8, opts.experts)
    try:
        state, report, dense, stayed, moved = _load_device(plan, dev, opts)
    except BaseException as e:
        traceback.clear_frames(e.__traceback__)   # the frames' locals would keep the call's device memory alive
        raise

    def assign(owners, kind, requires_grad, t):
        if kind == "param":
            t = torch.nn.Parameter(t, requires_grad=requires_grad)
        for o, n in owners:
            (o._parameters if kind == "param" else o._buffers)[n] = t

    for (_, owners, kind, requires_grad), t in zip(plan.dense, dense):
        assign(owners, kind, requires_grad, t)
    for gi, t in stayed.items():
        p, owners = plan.groups[gi]
        assign(owners, "param", p.requires_grad, t)
    for (m, n), b in zip(plan.moves, moved):
        m._buffers[n] = b
    if state is None:
        setattr(module, _ATTR, None)
    else:
        _commit(module, state, opts)
    return _with_prefetch(report, state, opts)


def save_module(module: torch.nn.Module, filename, metadata=None) -> None:
    """Write `module`'s full state -- its dense `state_dict()` and its compressed parameters at their owners' names --
    as a .znn.safetensors file, one name per tied parameter (the first in `state_dict()` order).

    Compressed parameters are written from their streams (one device-to-host copy, no decode or encode); dense
    floating-point tensors are compressed as `save_file` compresses them, adding at most one compress group to the
    device memory.  The file is byte for byte `save_file` of the dense model's state dict without the later tied names
    (with `save_file`'s caveat: at most one metadata key)."""
    state = getattr(module, _ATTR, None)
    tensors, coded = {}, {}
    for name, m, attr, kind, key in first_names(state_names(module))[0]:
        if kind == "resident":
            _, dtype, shape, _ = state.params[key[1]]
            coded[name] = (state.stream_of[key[1]], dtype, shape)
        else:
            tensors[name] = (m._parameters if kind == "param" else m._buffers)[attr].detach()
    save_coded(tensors, coded, filename, metadata)
