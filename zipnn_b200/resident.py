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
  * `state_dict()` does not see compressed parameters; `decompress_module(model)` restores them as dense
    `Parameter`s, bit for bit, and removes the hooks and plans.
"""
from __future__ import annotations

import torch

from .plan import DecodePlan
from .zipnn import ZipNN

_DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2)
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


class _Resident:
    """What compress_module leaves on the root module: per compressed module its plan and parameter names."""

    def __init__(self):
        self.entries = []     # (module, plan, [(name, index into the plan's outputs)], [hook handles])
        self.params = {}      # parameter index -> (requires_grad, dtype, shape, [(module, name)] where it was bound)
        self.stream_of = {}   # parameter index -> its stream (a view of `streams`)
        self.streams = None   # the one buffer that holds every stream
        self.order = {}       # id(module) -> (module, its parameter names in their original order)


def _pre_hook(plan, names):
    def hook(mod, args):
        if torch.is_grad_enabled():
            raise RuntimeError(f"{type(mod).__name__} holds compressed weights and runs only under torch.no_grad() or "
                               "torch.inference_mode() (its decoded weights live in a shared buffer)")
        outs = plan.run()
        for name, k in names:
            object.__setattr__(mod, name, outs[k])
    return hook


def _unbind(names):
    def hook(mod, args, output):
        for name, _ in names:
            mod.__dict__.pop(name, None)
    return hook


def compress_module(module: torch.nn.Module, modules=None) -> dict:
    """Compress the weights of `modules` (default: every submodule that directly owns bf16 / fp16 / fp32 / fp8
    parameters) into streams kept in HBM, decoded just before each module's forward.  All parameters are compressed
    in one `compress_batch` call and must be on one CUDA device.

    -> {"dense_bytes", "stream_bytes", "plan_bytes", "index_bytes", "scratch_bytes", "out_bytes", "params",
        "modules"}: bytes of the parameters now compressed, of their streams, of the plans' memory, of the segment
    index (the recorded segment starts, part of the plans' memory), of the shared plane scratch and of the shared output buffer
    (the size of the largest module's decoded weights)."""
    if getattr(module, _ATTR, None) is not None:
        raise ValueError("compress_module: this module is already compressed")
    modules, groups = select(module, modules)
    params = [p for p, _ in groups]
    if not params:
        setattr(module, _ATTR, None)
        return {"dense_bytes": 0, "stream_bytes": 0, "plan_bytes": 0, "index_bytes": 0, "scratch_bytes": 0, "out_bytes": 0,
                "params": 0, "modules": 0}
    if not all(p.is_cuda for p in params) or len({p.device for p in params}) > 1:
        raise ValueError("compress_module: the selected parameters must lie on one CUDA device")
    dev = params[0].device
    with torch.no_grad():
        coded = ZipNN(input_format="torch").compress_batch([p.detach() for p in params])
    keep = [i for i, (p, s) in enumerate(zip(params, coded)) if s.numel() < p.numel() * p.element_size()]
    # the streams move into one tight buffer; the batch's output buffer (sized by the bound) is dropped
    offs, at = [], 0
    for i in keep:
        offs.append(at)
        at = (at + coded[i].numel() + 15) // 16 * 16
    buf = torch.empty(max(at, 1), dtype=torch.uint8, device=dev)
    streams = {}
    for i, o in zip(keep, offs):
        n = coded[i].numel()
        buf[o: o + n].copy_(coded[i])
        streams[i] = buf[o: o + n]
    del coded
    # per module, the streams of its parameters
    where = {id(params[i]): i for i in keep}
    per_module = []
    for m in modules:
        names = [(n, where[id(p)]) for n, p in _own_params(m) if id(p) in where]
        if names:
            per_module.append((m, names))
    sizes = [DecodePlan.sizes([streams[i] for _, i in names]) for _, names in per_module]
    out = torch.empty(max([s[0] for s in sizes] + [1]), dtype=torch.uint8, device=dev)
    scratch = torch.empty(max([s[1] for s in sizes] + [1]), dtype=torch.uint8, device=dev)
    state = _Resident()
    state.streams = buf
    plan_bytes = index_bytes = 0
    for m, names in per_module:
        idx = [i for _, i in names]
        plan = DecodePlan([streams[i] for i in idx], out=out, scratch=scratch)
        plan_bytes += plan.nbytes["plan"]
        index_bytes += plan.nbytes["index"]
        local = [(n, k) for k, (n, _) in enumerate(names)]
        state.entries.append((m, plan, local, [m.register_forward_pre_hook(_pre_hook(plan, local)),
                                               m.register_forward_hook(_unbind(local), always_call=True)]))
    # the dense parameters go: nothing here keeps their storage alive
    dense = 0
    restore = {}
    for i in keep:
        p, owners = groups[i]
        dense += p.numel() * p.element_size()
        restore[i] = (p.requires_grad, p.dtype, tuple(p.shape), owners)
        for o, n in owners:
            state.order.setdefault(id(o), (o, list(o._parameters)))
            del o._parameters[n]
    state.params = restore
    state.stream_of = {i: streams[i] for i in keep}
    del params, groups
    setattr(module, _ATTR, state)
    return {"dense_bytes": dense, "stream_bytes": sum(s.numel() for s in state.stream_of.values()), "plan_bytes": plan_bytes,
            "index_bytes": index_bytes, "scratch_bytes": scratch.numel(), "out_bytes": out.numel(), "params": len(keep),
            "modules": len(per_module)}


def decompress_module(module: torch.nn.Module) -> None:
    """Undo `compress_module`: every compressed parameter becomes a dense `Parameter` again (tied ones one shared
    object again), bit for bit; the hooks, plans and streams are released."""
    state = getattr(module, _ATTR, None)
    if state is None:
        if hasattr(module, _ATTR):
            delattr(module, _ATTR)
            return
        raise ValueError("decompress_module: this module was not compressed by compress_module")
    for _, _, _, hooks in state.entries:
        for h in hooks:
            h.remove()
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
    delattr(module, _ATTR)
