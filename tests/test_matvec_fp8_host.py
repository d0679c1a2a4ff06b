"""The fp8 matvec's numerics and corpus without a GPU: the numpy model of tests/fp8_streams.py against fp64 and against
exact integer sums, the scale grids of the checkpoint layouts, and every corpus case checked to be what it claims."""
import numpy as np
import pytest
import torch

import fp8_streams as F
import plane_inputs as P


def _x(nt, inn, xdt, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(nt, inn, generator=g).to(F.XDTYPES[xdt]).float().numpy()


def _block_quantized(fmt, out, inn, seed):
    """bf16 Gaussian weights (std 0.02) quantized per 128x128 block at amax / fp8 max -> (fp8 bytes, fp32 scales)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(out, inn, generator=g) * 0.02).to(torch.bfloat16).float()
    gr, gc = F.grid_shape(out, inn, 128, 128)
    top = float(torch.finfo(F.TORCH[fmt]).max)
    amax = torch.zeros(gr, gc)
    for i in range(gr):
        for j in range(gc):
            amax[i, j] = w[128 * i: 128 * (i + 1), 128 * j: 128 * (j + 1)].abs().max()
    scale = (amax / top).clamp_min(2.0 ** -30)
    full = scale.repeat_interleave(128, 0)[:out].repeat_interleave(128, 1)[:, :inn]
    q = (w / full).to(F.TORCH[fmt])
    return q.float().numpy(), scale.numpy().astype(np.float32)


@pytest.mark.parametrize("fmt", F.FORMATS)
@pytest.mark.parametrize("xdt", ("bf16", "fp16"))
def test_model_against_fp64(fmt, xdt):
    """|model - fp64| within the fp32 accumulation bound plus half an ulp of the output, on ragged 128x128 blocks."""
    for out, inn, chunk, nt in ((200, 400, 4096, 3), (64, 2064, 512, 8), (1, 4096, 1024, 1)):
        w, scale = _block_quantized(fmt, out, inn, out + inn)
        x = _x(nt, inn, xdt, nt)
        bias = _x(1, out, xdt, 7)[0]
        y = F.model(w, scale, 128, 128, x, chunk, xdt, bias=bias)
        wd = F.dequantized(w, scale, 128, 128)
        ref = x.astype(np.float64) @ wd.T + bias
        mag = np.abs(x.astype(np.float64)) @ np.abs(wd).T + np.abs(bias)
        rel = 2.0 ** -8 if xdt == "bf16" else 2.0 ** -11
        bound = (inn + 2) * 2.0 ** -24 * mag
        tol = bound + (np.abs(ref) + bound) * rel + (2.0 ** -25 if xdt == "fp16" else 0)
        assert np.all(np.abs(y - ref) <= tol), (fmt, xdt, out, inn, float(np.max(np.abs(y - ref) - tol)))


@pytest.mark.parametrize("fmt", F.FORMATS)
def test_model_against_exact_integer_sums(fmt):
    """Integer weights and x, power-of-two scales: every partial sum is exact, so the model is the exact product
    rounded once, whatever the order of the additions."""
    rng = np.random.default_rng(3)
    top = 16 if fmt == "e4m3" else 7
    for out, inn, chunk, (bn, bk) in ((130, 384, 512, (128, 128)), (5, 8192, 2048, (1, 8192)), (48, 160, 4096, (3, 16))):
        w = np.clip(np.round(rng.normal(0, top / 3, (out, inn))), -top, top).astype(np.float32)
        assert np.array_equal(torch.from_numpy(w).to(F.TORCH[fmt]).float().numpy(), w)
        scale = (2.0 ** rng.integers(-2, 3, F.grid_shape(out, inn, bn, bk))).astype(np.float32)
        x = rng.integers(-2, 3, (4, inn)).astype(np.float32)
        for xdt in ("bf16", "fp16"):
            y = F.model(w, scale, bn, bk, x, chunk, xdt)
            ref = x.astype(np.float64) @ F.dequantized(w, scale, bn, bk).T
            want = torch.from_numpy(ref).to(F.XDTYPES[xdt]).float().numpy()
            assert np.array_equal(y, want), (fmt, xdt, out, inn)


def test_one_hot_model_is_the_model_at_one_hot_x():
    w, scale = _block_quantized("e4m3", 150, 272, 9)
    cols = [0, 1, 127, 128, 271]
    x = np.zeros((len(cols), 272), dtype=np.float32)
    x[np.arange(len(cols)), cols] = 4.0
    for xdt in ("bf16", "fp16"):
        a = F.model(w, scale, 128, 128, x, 1024, xdt)
        b = F.one_hot_model(w, scale, 128, 128, cols, 2, xdt)
        assert np.array_equal(a, b)


def test_scale_grids_of_the_checkpoint_layouts():
    assert F.grid_shape(4096, 14336, 4096, 14336) == (1, 1)
    assert F.grid_shape(4096, 14336, 1, 14336) == (4096, 1)
    assert F.grid_shape(4096, 14336, 128, 128) == (32, 112)
    assert F.grid_shape(1000, 208, 128, 128) == (8, 2)          # ragged on both edges
    assert F.grid_shape(7, 48, 3, 16) == (3, 3)
    for out, inn in ((1000, 208), (7, 48)):
        for name, (bn, bk) in F.layouts(out, inn).items():
            assert bn >= 1 and bk >= 16 and bk % 16 == 0, name
            s = F.random_scales(out, inn, bn, bk, 1)
            assert s.shape == F.grid_shape(out, inn, bn, bk) and s.dtype == np.float32
            # block (o / bn, i / bk) is the scale of every element of that block
            wd = F.dequantized(np.ones((out, inn), np.float32), s, bn, bk)
            o, i = out - 1, inn - 1
            assert wd[o, i] == s[o // bn, i // bk] and wd[0, 0] == s[0, 0]


def test_fp8_conversion_is_exact_in_fp32():
    """Every finite byte of both formats is a float32 value exactly (the kernel's fp8 -> fp32 loses nothing)."""
    b = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    for fmt in F.FORMATS:
        v = b.view(F.TORCH[fmt]).double()
        fin = ~torch.from_numpy(F.not_finite(fmt, b.numpy()))
        assert torch.equal(torch.isfinite(v), fin), fmt
        assert torch.equal(v[fin].float().double(), v[fin]), fmt


# ---------------------------------------------------------------- the corpus
@pytest.mark.parametrize("chunk", F.CHUNKS)
def test_shape_cases_are_what_they_claim(chunk):
    cases = F.shape_cases(chunk)   # (Case asserts that every chunk is fused and every weight finite)
    assert {c.dtype for c in cases} == set(F.FORMATS)
    inns = {c.inn for c in cases}
    assert {16, 48, 144, 528} <= inns
    assert any(c.out == 1 for c in cases)
    assert any(c.pr["K"] == 1 and c.data.size == chunk for c in cases), "a one-chunk tensor"
    short = [c for c in cases if c.data.size % chunk]
    assert all(c.data.size % 512 == 0 for c in short), "a short last chunk stays fused"
    assert short or chunk == 512, "a short last chunk (at 512 bytes every fused chunk is whole)"
    quarter = chunk // 4
    assert any(c.inn < quarter for c in cases) or chunk == 512, "rows shorter than a quarter"
    if chunk < 32768:
        assert any(c.inn > chunk for c in cases), "rows spanning chunks"


def test_stream_cases_are_what_they_claim():
    cases = F.stream_cases()
    assert {c.dtype for c in cases} == set(F.FORMATS)
    for fmt in F.FORMATS:
        crafted = [c for c in cases if c.name == f"crafted_{fmt}"][0]
        logs = {crafted.pr["items"][0][k].lg for k in range(crafted.pr["K"])}
        assert logs == set(range(1, 12)), (fmt, logs)
        ring = [c for c in cases if c.name == f"ring_{fmt}"][0]
        assert max(max(it.s_len) for it in (ring.pr["items"][0][k] for k in range(ring.pr["K"]))) > P.SYNC_STREAM_CAP
        fixed = [c for c in cases if c.name.startswith("fixed") and c.dtype == fmt]
        assert sorted(c.pr["items"][0][0].fixed_len for c in fixed) == [2, 4, 6]
        for c in fixed:
            assert P.misaligned_sync_guesses(c.pr["items"][0][-1]) == 4, c.name


@pytest.mark.parametrize("fmt", F.FORMATS)
def test_special_case_positions(fmt):
    case, at = F.special_case(fmt)
    w = case.weights().double()
    for r, c in at["nan"]:
        assert torch.isnan(w[r, c])
    for r, c in at.get("inf", []):
        assert w[r, c] == float("inf")
    for r, c in at.get("-inf", []):
        assert w[r, c] == float("-inf")
    for r, c in at["-0"]:
        assert w[r, c] == 0 and torch.signbit(w[r, c])
    tiny = 2.0 ** (-6 if fmt == "e4m3" else -14)
    for r, c in at["subnormal"]:
        assert 0 < abs(float(w[r, c])) < tiny
    bad_rows = {r for k in ("nan", "inf", "-inf") for r, _ in at.get(k, [])}
    assert {r for r in range(case.out) if not torch.isfinite(w[r]).all()} == bad_rows
