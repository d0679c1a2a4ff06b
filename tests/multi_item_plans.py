"""Decode plans of many items for the gather and matvec tests (test_multi_item_plans_host.py, _gpu.py).

A gather or a matvec finds its item through two numbers that plan create records on the host: the item's piece (its
control block, `s.B.cfgs + piece`) and the piece's first segment index entry (`s.X.seg + seg_base`).  The piece differs
from the item once an earlier item is empty or was split into pieces; seg_base is non-zero once an earlier item has
coded chunks.  The layouts here reach both for every target (the first with some rotation), place every target first,
in the middle and last by rotating the layout, and give every target a decoy: an item
of the same dtype, shape and chunk size with other bytes.  A call that read the wrong piece or the wrong segment base
would return the decoy's rows or multiply by the decoy's matrix: plausible values, no fault, and the comparisons with
the dense bytes reject them.

Every item is a torch-format stream made by the oracle (the header `ZipNN.plan` gives the tensor), so the same bytes
feed `DecodePlan` and the raw slice-item ABI.  `Model` restates what create records: the pieces (test_boxes_host's
piece model), each item's piece index (-1 for a box, a split item or an empty one) and each piece's seg_base (the
coded items of the type rows of the pieces in front of it, 4 x 256 entries each).
"""
from __future__ import annotations

import functools

import numpy as np
import torch

import plane_inputs as P
import test_boxes_host as H
import test_decoder_tables_gpu as D
from oracle import oracle as O
from test_slicing_host import cut_box
from zipnn_b200 import ZipNN

SEG_PER_ITEM = 4 * 256   # segment index entries per coded item: 4 bitstreams x 256 threads
TORCH = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32, "fp8": torch.float8_e4m3fn}
MATVEC_DTYPES = ("bf16", "fp16", "fp32")
SPLIT_LIMIT = 5          # ZIPNN_B200_SLICE_PIECE_CHUNKS of layout L2: whole items of at most 4 chunks stay one piece


class Entry:
    """One item: a tensor's bytes, its oracle-made torch-format stream and the fields of its slice item.

    kind:  'target' (gathered and, when `matvec`, multiplied; `decoy` names its decoy), 'decoy', 'const', 'raw',
           'general', 'empty', 'split' or 'box'."""

    def __init__(self, name, dtype, shape, data, chunk, kind="target", decoy=None, matvec=False, box=None):
        self.name, self.dtype, self.shape, self.kind, self.decoy, self.matvec = name, dtype, tuple(shape), kind, decoy, matvec
        self.data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        if self.data.size:
            self.tensor = torch.from_numpy(self.data.copy()).view(TORCH[dtype]).reshape(self.shape)
        else:
            self.tensor = torch.empty(self.shape, dtype=TORCH[dtype])
        z = ZipNN(input_format="torch", compression_chunk=chunk)
        pl = z.plan(self.tensor)
        self.G, self.bits, self.bm, self.chunk = pl["num_buf"], pl["bit_reorder"], pl["byte_reorder"], pl["chunk"]
        self.stream = O.zipnn_compress(pl["header"], self.data, self.G, self.bits, self.bm, self.chunk, pl["threshold"], threads=4)
        self.after = ZipNN(input_format="torch")._retrieve_header(self.stream[:32 + 1 + 9 * 255].tobytes())
        self.body = self.stream[self.after:]
        self.orig = self.data.size
        self.box = box if box is not None else (0, 1, self.orig, self.orig)
        self.whole = box is None
        self.want = self.data if self.whole else cut_box(self.data, box)
        self.K = -(-self.orig // self.chunk) if self.orig else 0

    @functools.cached_property
    def pr(self):
        """plane_inputs.predict of the stream (None for an empty tensor)."""
        return P.predict(self.body, self.G, self.bits, self.chunk, self.orig) if self.orig else None

    @property
    def types(self) -> np.ndarray:
        return self.body[: self.G * self.K].reshape(self.G, self.K)

    def coded(self, c0: int, c1: int) -> int:
        """Type-1 entries of the type rows over chunks [c0, c1): the coded items a piece sizes its index by."""
        return int(np.count_nonzero(self.types[:, c0:c1] == 1)) if self.orig else 0

    def symbols(self, c0: int, c1: int) -> int:
        """Bytes of the Huffman-coded planes of chunks [c0, c1): what the piece's segments count."""
        if not self.orig:
            return 0
        return sum(self.pr["items"][g][c].dec_len for g in range(self.G) for c in range(c0, c1) if self.pr["items"][g][c].kind == "huf")

    @property
    def fused(self) -> bool:
        return bool(self.orig) and set(self.pr["mode"]) == {"fused"}

    @property
    def eligible(self) -> bool:
        """Can the matvec multiply by it: a bf16 / fp16 / fp32 whole tensor, fused in every chunk, rows of a multiple
        of 16 bytes (targets with `matvec` and their decoys)."""
        return (self.whole and self.dtype in MATVEC_DTYPES and len(self.shape) > 1 and self.fused
                and (self.orig // self.shape[0]) % 16 == 0)

    def rows(self) -> np.ndarray:
        """The tensor's bytes as rows along dim 0."""
        return self.data.reshape(self.shape[0], -1)


class Model:
    """What plan create records for a list of items under a piece limit."""

    def __init__(self, entries, limit: int = H.DEFAULT_LIMIT):
        self.entries = list(entries)
        self.pieces = []   # (item index, test_boxes_host.Piece)
        for i, e in enumerate(self.entries):
            self.pieces += [(i, p) for p in H.pieces_of(e.box, e.chunk, limit)]
        self.seg_base = [0]
        for i, p in self.pieces:
            self.seg_base.append(self.seg_base[-1] + self.entries[i].coded(p.c0, p.c1) * SEG_PER_ITEM)
        self.piece = []
        for i, e in enumerate(self.entries):
            mine = [j for j, (k, _) in enumerate(self.pieces) if k == i]
            self.piece.append(mine[0] if len(mine) == 1 and e.whole else -1)
        self.coded_items = self.seg_base[-1] // SEG_PER_ITEM

    def n_pieces(self, i: int) -> int:
        return sum(1 for k, _ in self.pieces if k == i)

    def seg_rows(self, i: int) -> tuple:
        """-> (first index entry, entries, coded symbols) of whole item i's one piece."""
        j = self.piece[i]
        _, p = self.pieces[j]
        return self.seg_base[j], self.seg_base[j + 1] - self.seg_base[j], self.entries[i].symbols(p.c0, p.c1)


def rotate(entries, r: int) -> list:
    return list(entries[r:]) + list(entries[:r])


def placements(entries) -> list:
    """Rotations that put every target first, in the middle and last."""
    n = len(entries)
    out = set()
    for i, e in enumerate(entries):
        if e.kind == "target":
            out |= {i % n, (i - n // 2) % n, (i + 1) % n}
    return sorted(out)


# ------------------------------------------------------------------ tensors
def gauss(dtype: str, shape, seed: int) -> np.ndarray:
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(shape, generator=g) * (0.5 if dtype == "fp8" else 0.02)
    return t.to(TORCH[dtype]).view(torch.uint8).numpy().reshape(-1)


def pair(name, dtype, shape, chunk, seed, matvec=True) -> list:
    """A target and its decoy."""
    return [Entry(name, dtype, shape, gauss(dtype, shape, seed), chunk, decoy=name + "~", matvec=matvec),
            Entry(name + "~", dtype, shape, gauss(dtype, shape, seed + 1), chunk, kind="decoy")]


def empty(name, dtype, shape, chunk=262144) -> Entry:
    return Entry(name, dtype, shape, np.zeros(0, np.uint8), chunk, kind="empty")


def _planes_entry(case, shape, kind, box=None) -> Entry:
    return Entry(case.name, case.dtype, shape, case.data, case.chunk, kind=kind, box=box)


# ------------------------------------------------------------------ the layouts
@functools.lru_cache(maxsize=None)
def layout(name: str) -> tuple:
    """-> (entries, env): the items in their unrotated order and the environment the plan is made under."""
    if name == "L1":
        const = torch.full((256, 256), 2.0 ** -6, dtype=torch.bfloat16).view(torch.uint8).numpy().reshape(-1)
        ragged = (1039, 128)   # 256 KiB + 3840 bytes: a ragged last chunk
        entries = ([empty("empty_bf16", "bf16", (0, 256)), Entry("const_bf16", "bf16", (256, 256), const, 262144, kind="const")]
                   + pair("A_bf16", "bf16", (512, 512), 262144, 10)
                   + pair("emb_fp8", "fp8", (2048, 128), 262144, 20, matvec=False)
                   + pair("W_fp32", "fp32", (256, 512), 262144, 30)
                   + pair("W_fp16", "fp16", (512, 512), 262144, 40)
                   + pair("ragged_bf16", "bf16", ragged, 262144, 50, matvec=False))
        return entries, {}
    if name == "L2":
        split = D.planes_case("split_bf16", "bf16", 4096, ["geo5"] * 13, seed=60, last=1008)
        second = lambda c, g: "geo5"   # noqa: E731  a second coded plane in every chunk: general mode
        general = D.planes_case("general_bf16", "bf16", 4096, ["geo5"] * 4, seed=61, side=second)
        boxed = D.planes_case("boxed_bf16", "bf16", 4096, ["geo5", "const", "geo5", "raw", "geo5"], seed=63, last=1008)
        raw = np.random.default_rng(62).integers(0, 256, 4 * 4096, dtype=np.uint8)
        entries = ([_planes_entry(split, (split.data.size // 2,), "split"), _planes_entry(general, (64, 128), "general"),
                    Entry("raw_bf16", "bf16", (64, 128), raw, 4096, kind="raw")]
                   + pair("T_fp16", "fp16", (64, 128), 4096, 70)
                   + [_planes_entry(boxed, (boxed.data.size // 2,), "box", box=(16, 3, 4096, 100)),
                      empty("empty_fp16", "fp16", (0, 64), 4096)]
                   + pair("T_fp32", "fp32", (32, 128), 4096, 80)
                   + pair("T_bf16", "bf16", (32, 256), 4096, 90))
        return entries, {"ZIPNN_B200_SLICE_PIECE_CHUNKS": str(SPLIT_LIMIT)}
    if name == "L3":
        entries = (pair("c4k_bf16", "bf16", (256, 256), 4096, 100)
                   + [empty("empty_fp8", "fp8", (0, 32), 4096)]
                   + pair("c512_fp16", "fp16", (64, 128), 512, 110)
                   + pair("dflt_bf16", "bf16", (512, 512), 262144, 120)
                   + [empty("empty_bf16", "bf16", (0,), 512)]
                   + pair("c4k_fp32", "fp32", (128, 128), 4096, 130))
        return entries, {}
    raise KeyError(name)


LAYOUTS = ("L1", "L2", "L3")


def limit_of(env: dict) -> int:
    return int(env.get("ZIPNN_B200_SLICE_PIECE_CHUNKS", H.DEFAULT_LIMIT))


def without_boxes(entries) -> list:
    """The items a DecodePlan can hold (whole tensors only)."""
    return [e for e in entries if e.whole]
