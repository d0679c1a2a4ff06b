"""Seeded streams at every chunk size and threshold the stream format accepts.

`settings_inputs()` is shared by make_golden_ref_checks.py (what the compiled reference writes for each case),
test_oracle.py (the oracle against those digests) and test_chunk_sizes_gpu.py (the device codec against the
oracle).  The cases:

  chunks      G in {1, 2, 4} x bits_mode (0 only for G = 1) x every power-of-two chunk from G to 2^12, and
              2^19-2^21, at threshold 0.95; ragged tails of 0, G and 64*G - G bytes past the last full chunk
  thresholds  0.0, 0.5, 0.75, 0.95, 1.0 and 1.5 at two chunk sizes per G, and 2- and 3-byte planes around
              the RLE rule `1 < plen * thr`
  exact       one-group planes whose coded size is exactly plen * thr at the binary-exact thresholds 0.5 and
              0.75: the comparison is strict, so they stay raw
  capacity    one-group planes of 16-128 bytes that the reference keeps raw only because HUF_compress's
              destination is the chunk (= the plane), and one 2^17-byte plane at threshold 1.0 whose coded
              size lies in the last bytes below the plane length, where a bitstream's 8-byte slack refuses it

The searches use the oracle's HUF_compress; they are seeded, so every run builds the same planes.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import oracle as O

THRESHOLDS = (0.0, 0.5, 0.75, 0.95, 1.0, 1.5)
BIG_CHUNKS = (1 << 19, 1 << 20, 1 << 21)
FLIP_PLENS = (16, 32, 64, 128)
FLIPS_PER_PLEN = 6
SLACK_PLEN = 1 << 17
EXACT_PLENS = (256, 4096)


def layouts():
    """(G, bits_mode) pairs the format has: bits_mode only changes anything for G > 1."""
    return [(1, 0), (2, 0), (2, 1), (4, 0), (4, 1)]


def stored_size(plane: np.ndarray, cap: int, thr: float) -> int:
    """What the reference stores for one plane: 0 = raw, 1 = RLE, else the coded size (zipnn_core.c:365-373)."""
    r, _ = O.huf_compress(plane, cap)
    if r == O.ERR or r == 0:
        return 0
    return int(r) if r < plane.size * np.float64(np.float32(thr)) else 0


def _coded(plane: np.ndarray, cap: int) -> int:
    r, _ = O.huf_compress(plane, cap)
    return 0 if (r == O.ERR or r <= 1) else int(r)


# ---------------------------------------------------------------- element data
def _gauss(rng, n: int, G: int, chunk: int) -> np.ndarray:
    x = rng.standard_normal(n // G, dtype=np.float32)
    if G == 1:
        t = torch.from_numpy(x * np.float32(0.5)).to(torch.float8_e4m3fn)
    elif G == 2:
        t = torch.from_numpy(x * np.float32(0.02)).to(torch.bfloat16 if chunk.bit_length() % 2 else torch.float16)
    else:
        t = torch.from_numpy(x * np.float32(0.02))
    return t.view(torch.uint8).numpy().copy()


def _two_symbol(rng, n: int, G: int) -> np.ndarray:
    """Elements drawn from two values: every plane has at most two symbols (RLE or one-bit codes)."""
    vals = rng.integers(0, 256, (2, G), dtype=np.uint8)
    pick = rng.random(n // G) < 0.2
    return np.where(pick[:, None], vals[0], vals[1]).astype(np.uint8).reshape(-1)


def family_data(family: str, rng, n: int, G: int, chunk: int) -> np.ndarray:
    if family == "gauss":
        return _gauss(rng, n, G, chunk)
    if family == "const":
        return np.tile(rng.integers(0, 256, G, dtype=np.uint8), n // G)
    if family == "two":
        return _two_symbol(rng, n, G)
    if family == "bytes":
        return rng.integers(0, 256, n, dtype=np.uint8)
    raise ValueError(family)


FAMILIES = ("gauss", "const", "two", "bytes")


def _tails(G: int, chunk: int):
    return [t for t in (0, G, 64 * G - G) if t < chunk]


# ---------------------------------------------------------------- searched planes
def capacity_flip_planes(plen: int, count: int = FLIPS_PER_PLEN, seed: int = 0):
    """Dirichlet planes over symbols 0..k-1, k = 2-80, that the reference keeps raw with a destination of plen bytes (one
    group: the chunk is the plane) but codes with an unbounded destination, at threshold 0.95."""
    rng = np.random.default_rng(1000 + plen + seed)
    out = []
    for _ in range(200000):
        k = int(rng.integers(2, 81))
        p = rng.dirichlet(np.ones(k) * rng.uniform(0.05, 2.0))
        plane = rng.choice(k, plen, p=p).astype(np.uint8)
        if stored_size(plane, plen, 0.95) == 0 and stored_size(plane, 1 << 16, 0.95) > 1:
            out.append(plane)
            if len(out) == count:
                return out
    raise AssertionError(f"no capacity flips found at plen {plen}")


def exact_threshold_plane(plen: int, thr: float, seed: int = 0) -> np.ndarray:
    """A one-group plane whose coded size (destination = plen) is exactly plen * thr.  A hill climb from a
    Dirichlet plane: one byte at a time is set to the most frequent symbol (smaller) or a random one (larger)."""
    target = plen * thr
    assert target == int(target)
    target = int(target)
    rng = np.random.default_rng(7000 + plen + int(thr * 100) + seed)
    for _ in range(200):
        k = int(rng.integers(4, 160))
        p = rng.dirichlet(np.ones(k) * rng.uniform(0.2, 2.0))
        plane = rng.choice(k, plen, p=p).astype(np.uint8)
        alphabet = np.arange(k, dtype=np.uint8)
        for _ in range(400):
            r = _coded(plane, plen)
            if r == target:
                return plane
            if r == 0:
                break
            i = rng.integers(plen, size=max(1, abs(r - target) // 4))
            if r > target:
                plane[i] = np.bincount(plane, minlength=256).argmax()
            else:
                plane[i] = alphabet[rng.integers(alphabet.size, size=i.size)]
    raise AssertionError(f"no plane of {plen} bytes codes to exactly {target}")


def slack_plane() -> np.ndarray:
    """A 2^17-byte one-group plane whose coded size lies in the last 8 bytes below plen - 1.

    255 symbols near 514 occurrences each cost 8 bits; one heavy symbol (more than plen/128 + 4 occurrences, so
    the "probably not compressible" test lets it through) gets 7 bits, and two rare symbols get 9.  The rare
    count sets the saving to the bit, so the coded size can be placed anywhere near the plane length."""
    n = SLACK_PLEN
    rng = np.random.default_rng(17)
    heavy = n // 128 + 40
    for rare in range(380, 520):  # each extra rare occurrence adds a quarter byte; 400 lands 14 bytes short
        counts = np.zeros(256, np.int64)
        counts[0] = heavy
        counts[1] = counts[2] = rare
        rest = n - counts.sum()
        counts[3:] = rest // 253
        counts[3: 3 + rest % 253] += 1
        plane = rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), counts))
        blind = _coded(plane, 1 << 20)
        if n - 9 <= blind <= n - 2 and stored_size(plane, n, 1.0) == 0:
            return plane
    raise AssertionError("no plane in the slack window")


# ---------------------------------------------------------------- the cases
def _case(name, G, bits, chunk, thr, data, kind, **extra):
    d = {"name": name, "G": G, "bits": bits, "chunk": chunk, "thr": thr, "data": np.ascontiguousarray(data, np.uint8),
         "kind": kind}
    d.update(extra)
    return d


def header() -> bytes:
    h = bytearray(32)
    h[0:2] = b"ZN"
    return bytes(h)


def settings_inputs(big: bool = True):
    """-> list of case dicts {name, G, bits, chunk, thr, data, kind, ...}.  big=False leaves out the 2^19-2^21
    chunks."""
    cases = []
    seed = 0
    # chunks: every power of two from G to 4096, and three past the largest codable plane
    for G, bits in layouts():
        chunks = [1 << e for e in range(G.bit_length() - 1, 13)] + (list(BIG_CHUNKS) if big else [])
        for ci, chunk in enumerate(chunks):
            tails = _tails(G, chunk)
            for fi, fam in enumerate(FAMILIES):
                seed += 1
                rng = np.random.default_rng(seed)
                tail = tails[(ci + fi) % len(tails)]
                full = chunk if chunk >= (1 << 19) else max(4096, 8 * chunk)
                data = family_data(fam, rng, full + tail, G, chunk)
                cases.append(_case(f"chunk-G{G}b{bits}-c{chunk}-t{tail}-{fam}", G, bits, chunk, 0.95, data, "chunk",
                                   tail=tail, family=fam))
    # thresholds at two chunk sizes per G
    thr_chunks = {1: (32, 1 << 17), 2: (128, 1 << 18), 4: (256, 1 << 19)}
    for G, bits in ((1, 0), (2, 1), (4, 1)):
        for chunk in thr_chunks[G]:
            if chunk >= (1 << 19) and not big:
                continue
            for thr in THRESHOLDS:
                for fam in ("gauss", "two"):
                    seed += 1
                    rng = np.random.default_rng(seed)
                    n = chunk * (2 if chunk > 4096 else 64) + G
                    data = family_data(fam, rng, n, G, chunk)
                    cases.append(_case(f"thr-G{G}b{bits}-c{chunk}-{thr}-{fam}", G, bits, chunk, thr, data, "thr", family=fam))
    # 2- and 3-byte planes around the RLE rule 1 < plen * thr: constant elements, plen 2 in full chunks and 3 in
    # the ragged last chunk
    for G, bits in ((1, 0), (2, 1), (4, 1)):
        for thr in THRESHOLDS:
            rng = np.random.default_rng(500 + G)
            elem = rng.integers(0, 256, G, dtype=np.uint8)
            cases.append(_case(f"rle2-G{G}b{bits}-{thr}", G, bits, 2 * G, thr, np.tile(elem, 32), "rle", plen=2))
            # (zeros in the ragged chunk: its last len % 4 bytes are not rotated, so only a value the sign-bit
            # rotation leaves alone makes constant planes there)
            data = np.concatenate([np.tile(elem, 32), np.zeros(3 * G, np.uint8)])
            cases.append(_case(f"rle3-G{G}b{bits}-{thr}", G, bits, 4 * G, thr, data, "rle", plen=3))
    # coded size exactly plen * thr: strict comparison, raw
    for thr in (0.5, 0.75):
        for plen in EXACT_PLENS:
            planes = [exact_threshold_plane(plen, thr, s) for s in range(3)]
            cases.append(_case(f"exact-{plen}-{thr}", 1, 0, plen, thr, np.concatenate(planes), "exact", plen=plen))
    # capacity flips
    for plen in FLIP_PLENS:
        cases.append(_case(f"capflip-{plen}", 1, 0, plen, 0.95, np.concatenate(capacity_flip_planes(plen)), "capflip",
                           plen=plen))
    cases.append(_case("capslack-131072", 1, 0, SLACK_PLEN, 1.0, slack_plane(), "capslack", plen=SLACK_PLEN))
    return cases
