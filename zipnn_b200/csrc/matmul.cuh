// matmul.cuh -- y = x W^T for up to 64 rows of x on tensor cores, with W a whole-tensor item of a decode plan that is
// never written dense.
//
// y[t][o] = sum_i x[t][i] * W[o][i] (+ bias[o]), t < n_tokens <= kMatmulMaxTokens, W row-major [out][in] of bf16 or
// fp16, every chunk of it in fused mode (the host checks, as for the matvec).  Two launches per call:
//
//   k_matmul         sync_process in replay mode, one CTA per coded bitstream, as k_matvec: only the epilogue differs.
//                    `MatmulEp::quarter` feeds the 16-byte vectors ZB_FUSED_VECTOR forms to mma.m16n8k16 as B fragments.
//   k_matmul_reduce  one thread per (token, output row) adds the row's partial sums in ascending element order, adds the
//                    bias, rounds once to the output type and stores.
//
// Fragments.  The quarter plane of a bitstream is a contiguous element range of W.  It is cut into row tiles of 8
// consecutive W rows (the first tile starts at the quarter's first row) and each tile into column steps of 32.  In a
// step, lane (g = lane >> 2, j = lane & 3) forms the vector of row g, columns 8j .. 8j + 7.  Its four registers are the
// B fragments (n = g) of two k16 mma steps s = 0, 1 with the k order
//     kappa = 2j + b      -> column 8j + 4s + b,        kappa = 2j + 8 + b  -> column 8j + 4s + 2 + b      (b = 0, 1)
// so register 2s is b0b1 and register 2s + 1 is b2b3 of step s, with no shuffle.  The A fragments under the same
// order are one 16-byte load of x per token row: columns 8j .. 8j + 7 of tokens g and g + 8 of each 16-row tile, whose
// words 2s and 2s + 1 are a0a1 / a4a5 (token g) and a2a3 / a6a7 (token g + 8).  D is [token][W row of the tile].
//
// k_matmul_fp8 is k_matmul for fp8 weights with an fp32 scale grid and bf16 / fp16 x (MatmulEp with FMT >= 0): a step is
// 8 rows x 64 columns, lane (g, j) forms the 16 fp8 weights of row g, columns 16j .. 16j + 15, and after the rotation
// below dequantizes them exactly as k_dequant_fp8 does (fp8_dequant8: one fp32 multiply by the block's scale, one
// rounding to x's type) into the B fragments of four k16 steps, register 2s / 2s + 1 = columns 16j + 4s + {0, 1} /
// {2, 3}; x is two 16-byte loads per token row.  The product is F.linear of dequant_fp8's weight, summed in fp32, and
// its partial sums go through k_matmul_reduce unchanged.
//
// Masking.  A vector outside the quarter's range (partial first and last rows, columns past `in`) is zero and reads no
// shared memory; x columns past `in` and tokens past n_tokens are zero fragments and are not loaded.  The zero B
// vectors of a row that straddles two quarters meet real x, so an infinite x there gives NaN where the dense product
// gives an infinity: x must be finite.
//
// Bank conflicts.  The 8 rows of a tile lie `in` bytes apart in the quarter plane (one byte per element): with `in` a
// multiple of 128 (every llama shape) the 8 lanes that read the same columns of 8 rows hit the same banks, 8 wavefronts
// for an 8-byte load instead of 2.  So the steps go in groups of 4: in its load i of a group, lane (g, j) forms the
// vector of step (i + g) & 3, which puts the 4 rows of each half warp in 4 different 32-byte column ranges, and two
// rounds of selects move the vectors back to step order.
//
// Work split and partial sums.  The warps take the column groups of a tile in turn (warp w: groups w, w + 8, ...) and
// keep 4 fp32 accumulators per lane per 16-token tile in registers.  At the end of a tile they add up in shared memory
// (S.sbuf: the staged bitstream is dead once the quarter plane is emitted), warp by warp in a fixed order, and the CTA
// writes one fp32 per (row of the tile, token) to part[(((chunk * 4 + bitstream) * rt + tile) * n_tokens + t) * 8 +
// row].  Every slot the reduce reads is written by exactly one CTA in every call; no atomics, no memset, and the order
// of every addition is fixed by the shapes, so two calls with the same inputs give the same bits at any grid size.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "matvec.cuh"

namespace zb {

constexpr int kMatmulMaxTokens = 64;
constexpr int kMatmulTileRows = 8;    // W rows per tile: n of the mma

// Row tiles a quarter of q elements may touch, wherever it starts (rows of `in` elements).
__host__ __device__ inline uint64_t matmul_quarter_tiles(uint64_t q, uint64_t in, uint64_t out) {
  return (matvec_block_rows(q, in, out) + kMatmulTileRows - 1) / kMatmulTileRows;
}

template <int DT>
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (DT == kMvBf16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
}

// MT: 16-token tiles a lane accumulates, n_tokens rounded up to 16, 32 or 64.  Tiles wholly past n_tokens are skipped.
// FMT < 0: W of DT (above).  FMT = kFp8E4m3 / kFp8E5m2: fp8 W with a scale grid and x of DT (k_matmul_fp8, below).
template <int DT, int MT, int FMT = -1>
struct MatmulEp {
  static_assert(DT == kMvBf16 || DT == kMvFp16, "x of bf16 or fp16");
  static constexpr bool on = true;
  static constexpr uint32_t EB = FMT < 0 ? 2 : 1;  // bytes of a W element
  static constexpr uint32_t VC = 16 / EB;          // columns of a lane's vector
  static constexpr uint32_t SC = 4 * VC;           // columns of a step
  static constexpr uint32_t GC = 4 * SC;           // columns of a group
  ProductCfg m;

  template <int G>
  __device__ __forceinline__ void quarter(const SyncShared& S, uint64_t c, int stream, uint32_t out_off, uint32_t count, bool rot) const {
    static_assert(G == (int)EB, "one byte plane per byte of a W element");
    constexpr int TT = 16 * MT;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t g = (uint32_t)lane >> 2, j = (uint32_t)lane & 3u;
    const uint64_t in = m.in;
    const uint64_t e0 = c * m.ce + out_off, e1 = e0 + count;
    const uint64_t r_first = e0 / in;
    const uint32_t tiles = (uint32_t)((e1 - 1) / in - r_first) / kMatmulTileRows + 1;
    const uint32_t groups = (uint32_t)((in + GC - 1) / GC);
    const uint32_t mts = min((uint32_t)MT, (m.nt + 15u) >> 4);  // token tiles with a token in them
    const uint8_t* const xb = reinterpret_cast<const uint8_t*>(m.x);
    float* const red = reinterpret_cast<float*>(const_cast<uint8_t*>(S.sbuf));  // [warp][row][TT]
    float* const slots = m.part + (c * 4 + (uint32_t)stream) * m.rt * m.nt * kMatmulTileRows;
    const uint32_t rg = g & 3u;
    for (uint32_t tile = 0; tile < tiles; tile++) {
      const uint64_t row = r_first + (uint64_t)tile * kMatmulTileRows + g;  // this lane's row
      const uint64_t rowe = row * in;                                        // ... as an element
      float acc[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; mt++) acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.f;
      for (uint32_t grp = (uint32_t)wid; grp < groups; grp += kSyncThreads / 32) {
        const uint64_t k0 = (uint64_t)grp * GC;
        uint32_t v[4][4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const uint64_t col = k0 + SC * (((uint32_t)i + g) & 3u) + VC * j;
          const uint64_t e = rowe + col;
          if (col < in && e >= e0 && e < e1) {
            const uint32_t vo = (uint32_t)(e - e0) * EB;
            uint32_t fv[4];  // (a plain name: the macro's own loop index is `i`)
            ZB_FUSED_VECTOR(G, S, out_off, vo, rot, fv);
#pragma unroll
            for (int q = 0; q < 4; q++) v[i][q] = fv[q];
          } else {
            v[i][0] = v[i][1] = v[i][2] = v[i][3] = 0u;
          }
        }
        // v[i] holds step (i + rg) & 3: rotate by rg so that v[t] holds step t
        uint32_t u[4][4];
#pragma unroll
        for (int t = 0; t < 4; t++)
#pragma unroll
          for (int q = 0; q < 4; q++) u[t][q] = (rg & 1u) ? v[(t + 3) & 3][q] : v[t][q];
#pragma unroll
        for (int t = 0; t < 4; t++)
#pragma unroll
          for (int q = 0; q < 4; q++) v[t][q] = (rg & 2u) ? u[(t + 2) & 3][q] : u[t][q];
#pragma unroll
        for (int t = 0; t < 4; t++) {
          const uint64_t kc = k0 + SC * (uint32_t)t;
          if (kc >= in) break;  // (uniform)
          const uint64_t col = kc + VC * j;
          const bool cv = col < in;
          if constexpr (FMT < 0) {
#pragma unroll
            for (int mt = 0; mt < MT; mt++) {
              if ((uint32_t)mt >= mts) break;  // (uniform)
              const uint32_t t0 = 16u * (uint32_t)mt + g, t1 = t0 + 8u;
              uint4 xa = make_uint4(0u, 0u, 0u, 0u), xc = xa;
              if (cv && t0 < m.nt) xa = __ldg(reinterpret_cast<const uint4*>(xb + ((uint64_t)t0 * m.xs + col) * 2u));
              if (cv && t1 < m.nt) xc = __ldg(reinterpret_cast<const uint4*>(xb + ((uint64_t)t1 * m.xs + col) * 2u));
              mma_16816<DT>(acc[mt], xa.x, xc.x, xa.y, xc.y, v[t][0], v[t][1]);
              mma_16816<DT>(acc[mt], xa.z, xc.z, xa.w, xc.w, v[t][2], v[t][3]);
            }
          } else {
            // the vector dequantized as k_dequant_fp8 writes it: a zero vector (outside the quarter) is +0 with no scale
            // read, so a row or column past the matrix reads nothing
            const uint64_t e = rowe + col;
            float sc = 0.f;
            if (cv && e >= e0 && e < e1)
              sc = __ldg(m.scale + matvec_fp8_div((uint32_t)row, m.srow) * m.scols + matvec_fp8_div((uint32_t)col, m.scol));
            // in two halves of 8 columns, the half loop not unrolled: only one half's B fragments and 16 bytes of x per
            // token row are live at once (unrolled, MT = 2 and 4 spill at 80 registers)
#pragma unroll 1
            for (int h = 0; h < 2; h++) {  // columns 16j + 8h .. 16j + 8h + 7: k steps 2h, 2h + 1
              const uint4 b = fp8_dequant8<FMT, DT>(h ? v[t][2] : v[t][0], h ? v[t][3] : v[t][1], sc);
#pragma unroll
              for (int mt = 0; mt < MT; mt++) {
                if ((uint32_t)mt >= mts) break;  // (uniform)
                const uint32_t t0 = 16u * (uint32_t)mt + g, t1 = t0 + 8u;
                uint4 xa = make_uint4(0u, 0u, 0u, 0u), xc = xa;
                if (cv && t0 < m.nt) xa = __ldg(reinterpret_cast<const uint4*>(xb + ((uint64_t)t0 * m.xs + col) * 2u) + h);
                if (cv && t1 < m.nt) xc = __ldg(reinterpret_cast<const uint4*>(xb + ((uint64_t)t1 * m.xs + col) * 2u) + h);
                mma_16816<DT>(acc[mt], xa.x, xc.x, xa.y, xc.y, b.x, b.y);
                mma_16816<DT>(acc[mt], xa.z, xc.z, xa.w, xc.w, b.z, b.w);
              }
            }
          }
        }
      }
      // D: acc[mt] = {[token 16mt + g][row 2j], [16mt + g][2j + 1], [16mt + g + 8][2j], [16mt + g + 8][2j + 1]}
#pragma unroll
      for (int mt = 0; mt < MT; mt++) {
        float* const r0 = red + ((uint32_t)wid * kMatmulTileRows + 2u * j) * TT + 16u * (uint32_t)mt + g;
        r0[0] = acc[mt][0];
        r0[TT] = acc[mt][1];
        r0[8] = acc[mt][2];
        r0[TT + 8] = acc[mt][3];
      }
      __syncthreads();
      float* const out = slots + (uint64_t)tile * m.nt * kMatmulTileRows;
      for (uint32_t idx = threadIdx.x; idx < m.nt * kMatmulTileRows; idx += kSyncThreads) {
        const uint32_t row = idx & (kMatmulTileRows - 1), t = idx / kMatmulTileRows;
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kSyncThreads / 32; w++) s += red[((uint32_t)w * kMatmulTileRows + row) * TT + t];
        out[idx] = s;
      }
      __syncthreads();  // the sums are read before the next tile writes them
    }
  }
};
static_assert(sizeof(((SyncShared*)0)->sbuf) >= (kSyncThreads / 32) * kMatmulTileRows * kMatmulMaxTokens * sizeof(float),
              "the warps' sums of a tile fit in the stream buffer");

template <int DT, int MT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_matmul(ProductCfg m) {
  product_streams<2>(m, MatmulEp<DT, MT>{m});
}

// fp8 weights: MatmulEp with 16 fp8 weights per vector; the partial sums are k_matmul_reduce<XDT>'s, whose geometry
// comes from the element counts (esize 1).
template <int FMT, int XDT, int MT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_matmul_fp8(ProductCfg m) {
  product_streams<1>(m, MatmulEp<XDT, MT, FMT>{m});
}

template <int DT>
__global__ void __launch_bounds__(256) k_matmul_reduce(ProductCfg m) {
  product_reduce<DT>(m, [&](uint64_t t, uint64_t o) {
    float s = 0.f;
    for (uint64_t e = o * m.in; e < (o + 1) * m.in;) {
      const uint64_t c = e / m.ce;
      const uint64_t q = (c == m.K - 1 ? m.total - c * m.ce : m.ce) / 4;
      const uint64_t st = (e - c * m.ce) / q;
      const uint64_t qs = c * m.ce + st * q;
      const uint64_t r = o - qs / m.in;  // the row within the quarter's rows
      s += m.part[((((c * 4 + st) * m.rt + r / kMatmulTileRows) * m.nt + t) * kMatmulTileRows) + r % kMatmulTileRows];
      e = qs + q;
    }
    return s;
  });
}

}  // namespace zb
