#!/usr/bin/env python3
"""Model-shaped load-path benchmark (BASELINE.json configs 1-3).

No network: the checkpoints are synthesised with the real tensor shapes and randn*0.02 values
(SURVEY.md section 8d), written as .safetensors to --dir (default /dev/shm), compressed to
.znn.safetensors with zipnn_b200.compress_safetensors_file, and then loaded the way vLLM's weight
iterator does it (`with safe_open(f, framework="pt") as f: for name in f.keys(): f.get_tensor(name)`)
through zipnn_b200.SafeOpen(device="cuda") -- compressed bytes H2D, decode on the GPU.

With --tp N the same file is loaded the way each rank of tensor-parallel N would load it (all ranks in turn on one
GPU): column-parallel weights (q, k, v, gate, up, embedding, lm_head) by dim 0, row-parallel ones (o, down) by dim 1,
through SafeOpen(slices=True) and through get_tensor + narrow, one JSON line per rank.

usage: python tools/model_bench.py [gpt2|llama3-8b|granite-8b] [--layers N] [--dir /dev/shm] [--tp N]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from safetensors import safe_open  # noqa: E402
from safetensors.torch import save_file  # noqa: E402

from zipnn_b200 import SafeOpen, compress_safetensors_file  # noqa: E402


def gpt2_shapes(layers=12):
    h = 768
    s = {"wte.weight": (50257, h), "wpe.weight": (1024, h), "ln_f.weight": (h,), "ln_f.bias": (h,)}
    for i in range(layers):
        p = f"h.{i}."
        s.update({p + "ln_1.weight": (h,), p + "ln_1.bias": (h,), p + "attn.c_attn.weight": (h, 3 * h),
                  p + "attn.c_attn.bias": (3 * h,), p + "attn.c_proj.weight": (h, h), p + "attn.c_proj.bias": (h,),
                  p + "ln_2.weight": (h,), p + "ln_2.bias": (h,), p + "mlp.c_fc.weight": (h, 4 * h),
                  p + "mlp.c_fc.bias": (4 * h,), p + "mlp.c_proj.weight": (4 * h, h), p + "mlp.c_proj.bias": (h,)})
    return s, torch.float32


def llama_like(layers, h, ffn, vocab, kv):
    s = {"model.embed_tokens.weight": (vocab, h), "model.norm.weight": (h,), "lm_head.weight": (vocab, h)}
    for i in range(layers):
        p = f"model.layers.{i}."
        s.update({p + "self_attn.q_proj.weight": (h, h), p + "self_attn.k_proj.weight": (kv, h),
                  p + "self_attn.v_proj.weight": (kv, h), p + "self_attn.o_proj.weight": (h, h),
                  p + "mlp.gate_proj.weight": (ffn, h), p + "mlp.up_proj.weight": (ffn, h),
                  p + "mlp.down_proj.weight": (h, ffn), p + "input_layernorm.weight": (h,),
                  p + "post_attention_layernorm.weight": (h,)})
    return s


MODELS = {
    "gpt2": lambda L: gpt2_shapes(L or 12),
    "llama3-8b": lambda L: (llama_like(L or 32, 4096, 14336, 128256, 1024), torch.bfloat16),
    "granite-8b": lambda L: (llama_like(L or 40, 4096, 12800, 49155, 1024), torch.float16),
}


def load_chunk_sharded(path, rank, world, dev):
    """BASELINE.json config 4: every tensor of the file is partitioned by CHUNK RANGE over the ranks.  A rank reads
    only what it needs -- header + tables of each entry, then the payload byte ranges of its chunks -- assembles a
    self-contained local stream per tensor (rows rebased, as zipnn_b200.sharded.scatter_stream does between GPUs),
    uploads them in one buffer and decodes all of them with one batched call.  -> {name: flat local slice}"""
    import ctypes as C
    import numpy as np
    from zipnn_b200 import ZipNN, _native
    from zipnn_b200.safetensors_io import _safetensors_index
    from zipnn_b200.sharded import byte_range, chunk_range
    from zipnn_b200.util_torch import torch_dtype_of_code
    from zipnn_b200.zipnn import HEADER_LEN, HUF_MAX_BLOCK
    idx = _safetensors_index(path)
    fd = os.open(path, os.O_RDONLY)
    plans, total = [], 0
    for name, (off, nbytes) in idx.items():
        head = os.pread(fd, min(nbytes, HEADER_LEN + 1 + 9 * 255), off)
        z = ZipNN(input_format="torch")
        after = z._retrieve_header(head)
        G = z._num_buf_of_dtype()
        chunk = z.compression_chunk if G != 1 else min(HUF_MAX_BLOCK, z.compression_chunk)
        n = z.original_len
        K = (n + chunk - 1) // chunk
        c0, c1 = chunk_range(K, rank, world)
        b0, b1 = byte_range(n, chunk, rank, world)
        if c1 <= c0:
            plans.append((name, None))
            continue
        tab = np.frombuffer(os.pread(fd, 9 * G * K, off + after), dtype=np.uint8)
        types = tab[: G * K].reshape(G, K)
        cum = np.frombuffer(tab[G * K:].tobytes(), dtype="<u8").reshape(G, K).astype(np.int64)
        payload0 = off + after + 9 * G * K
        base = payload0 + np.concatenate([[0], np.cumsum(cum[:, -1])[:-1]])
        lo = cum[:, c0 - 1] if c0 else np.zeros(G, dtype=np.int64)
        hi = cum[:, c1 - 1]
        Kl = c1 - c0
        local_len = 9 * G * Kl + int((hi - lo).sum())
        plans.append((name, dict(G=G, chunk=chunk, bits=z._bit_reorder, bm=z._byte_reorder, n_local=b1 - b0, Kl=Kl, at=total,
                                 types=types[:, c0:c1], cum=cum[:, c0:c1] - lo.reshape(G, 1), spans=[(int(base[g] + lo[g]), int(hi[g] - lo[g])) for g in range(G)],
                                 local_len=local_len, dtype=torch_dtype_of_code(z.dtype))))
        total += (local_len + 64 + 15) // 16 * 16
    host = torch.empty(total + 64, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for name, p in plans:
        if p is None:
            continue
        at = p["at"] + 64
        G, Kl = p["G"], p["Kl"]
        hv[at: at + G * Kl] = np.ascontiguousarray(p["types"]).reshape(-1)
        hv[at + G * Kl: at + 9 * G * Kl] = p["cum"].astype("<u8").reshape(-1).view(np.uint8)
        w = at + 9 * G * Kl
        for foff, ln in p["spans"]:
            if ln:
                os.preadv(fd, [memoryview(hv[w: w + ln])], foff)
            w += ln
    os.close(fd)
    dbuf = host.to(dev, non_blocking=True)
    items = [(name, p) for name, p in plans if p is not None]
    arr = (_native.BatchItem * len(items))()
    outs = {}
    for i, (name, p) in enumerate(items):
        out = torch.empty(p["n_local"], dtype=torch.uint8, device=dev)
        outs[name] = out.view(p["dtype"])
        arr[i].d_body = dbuf.data_ptr() + p["at"] + 64
        arr[i].body_len = p["local_len"]
        arr[i].num_buf, arr[i].bits_mode, arr[i].bytes_mode = p["G"], p["bits"], p["bm"]
        arr[i].chunk, arr[i].orig = p["chunk"], p["n_local"]
        arr[i].d_out = out.data_ptr()
    L = _native.lib()
    wsz = C.c_size_t(0)
    _native.check(L.zipnn_b200_decompress_batch_workspace_size(arr, len(items), C.byref(wsz)))
    ws = torch.empty(wsz.value, dtype=torch.uint8, device=dev)
    _native.check(L.zipnn_b200_decompress_batch(arr, len(items), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream, 1))
    return outs


COLUMN_PARALLEL = ("q_proj", "k_proj", "v_proj", "gate_proj", "up_proj", "embed_tokens", "lm_head")   # sharded by dim 0
ROW_PARALLEL = ("o_proj", "down_proj")                                                               # sharded by dim 1


def tp_shard(name, shape, rank, world):
    """(dim, start, stop) of rank's shard as transformers' get_tensor_shard cuts it (torch.chunk), or None for a
    replicated tensor."""
    kind = name.split(".")[-2]
    dim = 0 if kind in COLUMN_PARALLEL else 1 if kind in ROW_PARALLEL else None
    if dim is None or len(shape) < 2:
        return None
    size = -(-shape[dim] // world)
    start = min(rank * size, shape[dim])
    return dim, start, min(start + size, shape[dim])


def load_tp_rank(path, rank, world, dev, slices):
    """Every tensor of the file as rank `rank` of tensor-parallel `world` needs it: through CompressedSlice
    (slices=True), or get_tensor + narrow.  -> ({name: tensor}, bytes read from the file, bytes copied H2D)."""
    from zipnn_b200 import slicing
    from zipnn_b200.safetensors_io import _safetensors_index
    counted = [0]
    orig_read, orig_into = slicing.FileSource.read, slicing.FileSource.read_into

    def read(self, off, n):
        counted[0] += n
        return orig_read(self, off, n)

    def read_into(self, off, mv):
        counted[0] += len(mv)
        return orig_into(self, off, mv)

    got, plain = {}, 0
    idx = _safetensors_index(path)
    slicing.FileSource.read, slicing.FileSource.read_into = read, read_into
    try:
        with SafeOpen(path, "pt", str(dev), slices=slices) as f:
            comp = f.compressed_tensors_metadata
            for name in f.keys():
                shape = json.loads(comp[name]["shape"]) if name in comp else f.get_slice(name).get_shape()
                sh = tp_shard(name, shape, rank, world)
                if name not in comp:
                    plain += idx[name][1]
                if slices:
                    sl = f.get_slice(name)
                    ix = (slice(None),) * sh[0] + (slice(sh[1], sh[2]),) if sh else slice(None)
                    got[name] = sl[ix] if name in comp else sl[ix].to(dev)
                elif sh is None:
                    got[name] = f.get_tensor(name)
                else:
                    dim, a, b = sh
                    got[name] = f.get_tensor(name).narrow(dim, a, b - a).contiguous()
        torch.cuda.synchronize()
    finally:
        slicing.FileSource.read, slicing.FileSource.read_into = orig_read, orig_into
    if not slices:   # the batched load path reads and uploads every compressed entry whole
        counted[0] = sum(idx[k][1] for k in idx if k in comp)
    return got, counted[0] + plain, counted[0] + plain


def tp_bench(path, world, dev, model):
    """One JSON line per rank of TP=world, all ranks in turn on one GPU: sliced reads next to get_tensor + narrow."""
    from zipnn_b200 import _native
    load_tp_rank(path, 0, world, dev, True)                  # warm-up (page cache, allocator, kernels)
    load_tp_rank(path, 0, world, dev, False)
    for rank in range(world):
        row = dict(model=model, mode=f"tp rank {rank} of {world}", device=torch.cuda.get_device_name(dev))
        outs = {}
        for key, slices in (("slices", True), ("get_tensor_narrow", False)):
            t0 = time.perf_counter()
            got, nread, nh2d = load_tp_rank(path, rank, world, dev, slices)
            wall = time.perf_counter() - t0
            _native.timing_collect()
            _native.timing_enable(True)
            load_tp_rank(path, rank, world, dev, slices)
            ker = _native.timing_collect()
            _native.timing_enable(False)
            row[key] = dict(wall_s=round(wall, 4), file_bytes_read=nread, h2d_bytes=nh2d,
                            decode_kernel_ms=round(sum(ms for ms, _ in ker.values()), 3),
                            decode_launches=sum(n for _, n in ker.values()))
            outs[key] = got
        row["exact"] = all(torch.equal(outs["slices"][k].view(torch.uint8), outs["get_tensor_narrow"][k].view(torch.uint8))
                           for k in outs["slices"])
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("model", nargs="?", default="gpt2", choices=sorted(MODELS))
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--dir", default="/dev/shm")
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--sharded", action="store_true", help="under torchrun: every tensor partitioned by chunk range over the ranks")
    ap.add_argument("--tp", type=int, default=0, help="load as each rank of tensor-parallel N would (one GPU, ranks in turn): "
                                                      "sliced reads vs get_tensor + narrow, one JSON line per rank")
    args = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    shapes, dtype = MODELS[args.model](args.layers)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    src = os.path.join(args.dir, f"{args.model}.safetensors")
    path = src[: -len(".safetensors")] + ".znn.safetensors"
    tensors = {}
    nbytes = t_comp = 0
    if rank == 0:
        g = torch.Generator(device=dev).manual_seed(1234)
        for name, shp in shapes.items():
            n = 1
            for d in shp:
                n *= d
            tensors[name] = (torch.randn(n, generator=g, device=dev) * 0.02).to(dtype).reshape(shp).cpu()
        nbytes = sum(t.numel() * t.element_size() for t in tensors.values())
        save_file(tensors, src, {"format": "pt"})
        t0 = time.perf_counter()
        path, clen, olen = compress_safetensors_file(src)
        torch.cuda.synchronize()
        t_comp = time.perf_counter() - t0
    if world > 1:
        box = [nbytes]
        dist.broadcast_object_list(box, 0)
        nbytes = box[0]
        dist.barrier()

    def load(opener, p):
        t0 = time.perf_counter()
        got = {}
        with opener(p, "pt", f"cuda:{local}") as f:
            for name in f.keys():
                got[name] = f.get_tensor(name)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, got

    if args.tp and rank == 0:
        tp_bench(path, args.tp, dev, args.model)
    elif args.sharded and world > 1:
        from zipnn_b200.sharded import byte_range
        load_chunk_sharded(path, rank, world, dev)          # warm-up
        torch.cuda.synchronize(); dist.barrier()
        t0 = time.perf_counter()
        got = load_chunk_sharded(path, rank, world, dev)
        torch.cuda.synchronize()
        t_local = time.perf_counter() - t0
        tt = torch.tensor([t_local], device=dev, dtype=torch.float64)
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        # exactness: rank 0 holds the originals; every rank sends a checksum of its slices
        ok = True
        if rank == 0:
            for k, t in tensors.items():
                esz = t.element_size()
                chunk = 131072 if esz == 1 else 262144
                b0, b1 = byte_range(t.numel() * esz, chunk, 0, world)
                ok = ok and torch.equal(got[k].view(torch.uint8).cpu(), t.reshape(-1).view(torch.uint8)[b0:b1]) if k in got else ok
        if rank == 0:
            row = dict(model=args.model, mode=f"chunk-sharded over {world} GPUs", dtype=str(dtype).replace("torch.", ""), tensors=len(shapes), bytes=nbytes,
                       rank0_slices_exact=bool(ok), load_s=round(float(tt.item()), 3), load_gbs=round(nbytes / float(tt.item()) / 1e9, 2),
                       compress_file_s=round(t_comp, 3))
            print(json.dumps(row), flush=True)
    elif rank == 0:
        load(SafeOpen, path)                       # warm-up (page cache, allocator, kernels)
        t_znn, got = load(SafeOpen, path)
        ok = all(torch.equal(got[k].view(torch.uint8).cpu(), tensors[k].view(torch.uint8)) for k in tensors)
        del got
        t_seq, _ = load(lambda p, fw, d: SafeOpen(p, fw, d, batch=False), path)
        load(safe_open, src)
        t_raw, _ = load(safe_open, src)
        row = dict(model=args.model, dtype=str(dtype).replace("torch.", ""), tensors=len(tensors), bytes=nbytes,
                   file_ratio=round(os.path.getsize(path) / os.path.getsize(src), 4), exact=ok,
                   compress_file_s=round(t_comp, 3), compress_file_gbs=round(nbytes / t_comp / 1e9, 2),
                   load_znn_to_cuda_s=round(t_znn, 3), load_znn_gbs=round(nbytes / t_znn / 1e9, 2),
                   load_znn_per_tensor_s=round(t_seq, 3),
                   load_plain_safetensors_to_cuda_s=round(t_raw, 3), load_plain_gbs=round(nbytes / t_raw / 1e9, 2),
                   speedup_vs_plain=round(t_raw / t_znn, 2))
        print(json.dumps(row), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0 and not args.keep:
        os.remove(src)
        os.remove(path)


if __name__ == "__main__":
    main()
