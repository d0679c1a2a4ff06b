// matvec.cuh -- y = x W^T for a few rows of x, with W a whole-tensor item of a decode plan that is never written dense.
//
// y[t][o] = sum_i x[t][i] * W[o][i] (+ bias[o]), t < n_tokens <= kMatvecMaxTokens, W row-major [out][in] of bf16, fp16
// or fp32, every chunk of it in fused mode (the host checks).  Two launches per call, whatever the shapes are:
//
//   k_matvec         sync_process in replay mode, one CTA per coded bitstream as in a plan run: tables, stream staging,
//                    segment index and the fused merge (ZB_FUSED_VECTOR) are the plan run's.  Where the run stores the 16
//                    bytes it formed, `MatvecEp::quarter` multiplies them with the activations.
//   k_matvec_reduce  one thread per (token, output row) adds the row's partial sums in ascending element order, adds the
//                    bias, rounds once to the output type and stores.
//
// k_matvec_fp8 is k_matvec for fp8 weights with an fp32 scale grid and bf16 / fp16 x: the same epilogue, MatvecEp, with
// the fp8 product of a lane's vector (below); its partial sums go through k_matvec_reduce unchanged.  k_dequant_fp8
// (end of file) writes such a weight dequantized to bf16 / fp16 through the same bitstream loop, with no reduce.
//
// Thread mapping.  The run's store loop gives thread t the vectors t, t + 256, ...: fine for stores, but it scatters a
// row of W over all threads, so every row would end in a CTA-wide reduction.  Here a warp owns a contiguous BLOCK of
// the quarter plane (an eighth of it, rounded up to whole 32-vector steps) and its lanes take consecutive vectors:
// the quarter plane in shared memory and x in L2 are read coalesced, a row's sum stays in per-lane fp32 accumulators
// across steps, and it ends in one butterfly of shuffles when the warp leaves the row.  With in_features a multiple of
// 32 vectors (every llama shape) a step lies in one row and the row test is uniform; a step that straddles rows (small
// or odd in_features) walks its rows one by one, each lane adding to the row its vector is in.
//
// Partial sums.  A block is identified by (chunk, bitstream, warp) and covers a fixed element range, so the rows it
// touches are known from the shapes alone: at most rs = (block elements + in - 2) / in + 1 of them.  The warp writes one
// fp32 per (row, token) to part[((block * rs) + row - block's first row) * n_tokens + t]: every slot the reduce reads
// is written by exactly one warp in every call, nothing is accumulated in memory, no atomics and no memset, and the
// order of every addition is fixed by the shapes: two calls with the same inputs give the same bits.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <type_traits>

#include "decode_sync.cuh"

namespace zb {

constexpr int kMatvecMaxTokens = 8;
enum : int { kMvBf16 = 0, kMvFp16 = 1, kMvFp32 = 2 };
__host__ __device__ constexpr int matvec_esize(int dt) { return dt == kMvFp32 ? 4 : 2; }

// The launch arguments of k_matvec and k_matmul and of their reduce kernels.
struct ProductCfg {
  const DecodeCfg* cfg;   // the item's piece, in plan memory
  SegEntry* seg;          // the piece's segment index
  uint32_t* error;        // the plan's error word
  const void* x;
  const void* bias;       // or nullptr
  void* y;
  float* part;            // the partial sums (scratch)
  uint64_t in, out;       // features
  uint64_t xs, ys;        // row strides of x and y, in elements
  uint64_t ce, total, K;  // elements of a full chunk and of the tensor; chunks
  uint32_t esize, nt, rs; // element bytes, tokens, slots (rows) per block of the matvec
  uint32_t step_rows, step_cols;  // one 32-vector step of the matvec as whole rows + columns
  uint32_t rt;            // row tiles per quarter in the matmul's slot layout
  // the fp8 matvec's scale grid S [ceil(out / bn)][scols]: the block of element (row, col) is
  // (matvec_fp8_div(row, srow), matvec_fp8_div(col, scol)), srow / scol the reciprocals of bn / bk (matvec_fp8_recip)
  const float* scale;
  uint64_t srow, scol;
  uint32_t scols;
  // the selected dequantize's per-slice grid (k_select_dequant_fp8, select.cuh): the tensor is `rows` slices of
  // slice_rows rows, each with a grid of its own of slice_grid scales; slice s of row r is matvec_fp8_div(r, sslice)
  uint64_t sslice;
  uint32_t slice_rows, slice_grid;
};

// The selected experts matvec's arguments (k_select_matvec_fp8, select.cuh): the item [E][out][in] as one matrix of
// E * out rows with the per-slice scale grid (sslice, slice_rows, slice_grid), nt = the pair slots per expert, and
// k_select_pairs' tables.  Slot t of expert e multiplies x row tab[e * nt + t] / k (one x row per token) or
// tab[e * nt + t] (one x row per pair), taken by a multiply-high by xdiv = matvec_fp8_recip(k or 1).  A type of its own
// rather than new ProductCfg fields, so that ProductCfg, and every kernel that takes it, stays as it was.
struct ExpertsCfg : ProductCfg {
  uint32_t* cnt;  // [E] pairs routed to expert e (at most nt)
  uint32_t* tab;  // [E][nt] their pair numbers, ascending
  uint32_t* pos;  // [pairs] pair p's slot in its expert's list
  uint64_t xdiv;
};

// Elements of a block of a chunk with n elements: a quarter's vectors split over 8 warps, in whole 32-vector steps.
__host__ __device__ inline uint64_t matvec_block_elems(uint64_t n, uint32_t esize) {
  const uint64_t epv = 16 / esize, nv = (n / 4) / epv;
  return ((nv + 255) / 256) * 32 * epv;
}
// Rows of `in` elements that `be` consecutive elements can touch, wherever they start.
__host__ __device__ inline uint64_t matvec_block_rows(uint64_t be, uint64_t in, uint64_t out) {
  const uint64_t r = (be + in - 2) / in + 1;
  return r < out ? r : out;
}
// The block that holds element e: its number and its element range [start, end).
struct MatvecBlock {
  uint64_t id, start, end;
};
__device__ __forceinline__ MatvecBlock matvec_block_of(const ProductCfg& m, uint64_t e) {
  const uint64_t c = e / m.ce;
  const uint64_t n = c == m.K - 1 ? m.total - c * m.ce : m.ce;
  const uint64_t q = n / 4, be = matvec_block_elems(n, m.esize);
  const uint64_t r = e - c * m.ce, s = r / q, w = (r - s * q) / be;
  MatvecBlock b;
  b.id = (c * 4 + s) * 8 + w;
  b.start = c * m.ce + s * q + w * be;
  b.end = min(b.start + be, c * m.ce + (s + 1) * q);
  return b;
}

template <int DT, int EPV>
__device__ __forceinline__ void matvec_floats(const uint32_t (&r)[4], float (&f)[EPV]) {
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if constexpr (DT == kMvBf16) {
      f[2 * i] = __uint_as_float(r[i] << 16);
      f[2 * i + 1] = __uint_as_float(r[i] & 0xFFFF0000u);
    } else if constexpr (DT == kMvFp16) {
      const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&r[i]));
      f[2 * i] = v.x;
      f[2 * i + 1] = v.y;
    } else {
      f[i] = __uint_as_float(r[i]);
    }
  }
}

// ---- fp8 weights with an fp32 scale grid (k_matvec_fp8) -------------------------------------------------------------
// y[t][o] = sum_i x[t][i] * (float(W[o][i]) * S[o / bn][i / bk]) (+ bias[o]), W of float8_e4m3fn or float8_e5m2 in one
// byte plane (G = 1), x, bias and y of bf16 or fp16.  bk % 16 == 0, so a lane's 16 weights (one vector) lie in one row
// and one scale block: the lane forms s = fma(w15, x15, ... fma(w0, x0, 0)) in fp32, in ascending column order, and
// p = s * S[block] with one multiply; everything else is the matvec's (per-lane row accumulators, the butterfly, one
// slot per (block, row, token), k_matvec_reduce).  A step is 32 lanes x 16 weights, and a lane reads 32 bytes of x per
// token and one scale per step (the grid is small and stays in L1 / L2).  fp8 -> fp32 is exact in both formats,
// subnormals included; an e4m3fn NaN or an e5m2 infinity or NaN acts as in the dense product of the dequantized matrix.
enum : int { kFp8E4m3 = 0, kFp8E5m2 = 1 };

// floor(n / d) for n, d < 2^31 as one 64-bit multiply-high by r = ceil(2^64 / (2 d)), no division: 2n * r / 2^64 =
// n / d + 2n * e / 2^64 with 0 <= e < 1, and 2n * e / 2^64 < 1 / (2d) because 2n * 2d < 2^64, so the floor is n / d's.
__host__ __device__ constexpr uint64_t matvec_fp8_recip(uint64_t d) { return ~0ull / (2 * d) + 1; }
__device__ __forceinline__ uint32_t matvec_fp8_div(uint32_t n, uint64_t r) { return (uint32_t)__umul64hi(2ull * n, r); }

// The 8 fp8 weights of two words as fp32 (exact: every e4m3fn and e5m2 value, NaN and infinities too, is an fp16 one).
template <int FMT>
__device__ __forceinline__ void fp8_floats(uint32_t a, uint32_t b, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const uint32_t word = i < 2 ? a : b;
    const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(word >> (16 * (i & 1))), FMT == kFp8E4m3 ? __NV_E4M3 : __NV_E5M2);
    const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&hr));
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}

// The matvec epilogue of sync_process: the warp-owns-a-block mapping and the row walk.  Only the product of a lane's
// 16 decoded bytes differs between weight types: FMT < 0, weights of DT, one FMA chain over the vector's EPV elements;
// FMT = kFp8E4m3 / kFp8E5m2, fp8 weights with a scale grid and x of DT (bf16 or fp16), the FMA chain over 16 weights
// and one multiply by the scale (above).
//
// NT: the accumulators a lane holds, n_tokens rounded up to a power of two.  Tokens past n_tokens repeat the last one
// and are not stored: 3 and 5 to 7 tokens pay for 4 and 8.  A uniform `t < n_tokens` exit from the token loop was
// measured instead: it keeps the loads of the tokens from being issued together, and 8 tokens took 1.3 to 1.5 times as long.
//
// EXPERTS (fp8 only; k_select_matvec_fp8): m is an ExpertsCfg, and the matrix is E experts of slice_rows rows.  A row's
// expert is matvec_fp8_div(row, sslice), its scale the expert's own grid (DequantEp's SLICED lookup), and token slot t
// of the row is the t-th pair routed to that expert: its x row comes from the pair table.  A lane reads the table again
// only when the expert of its row changes (a warp's rows almost always share one).  Slots past the expert's pair count
// repeat its last pair (row 0 of x for an expert with none) and are not stored: the flush writes slot t only for
// t < cnt[expert], so the rows of an unrouted expert in a chunk that straddles experts write nothing.
template <int DT, int NT, int FMT = -1, bool EXPERTS = false>
struct MatvecEp {
  static_assert(FMT < 0 || DT != kMvFp32, "fp8 weights: x of bf16 or fp16");
  static_assert(!EXPERTS || FMT >= 0, "the experts form is fp8's");
  static constexpr bool on = true;
  static constexpr int EPV = FMT < 0 ? 16 / matvec_esize(DT) : 16;
  std::conditional_t<EXPERTS, ExpertsCfg, ProductCfg> m;

  // The slots of `row` that are stored.
  __device__ __forceinline__ uint32_t stored(uint64_t row) const {
    if constexpr (EXPERTS) {
      return __ldg(m.cnt + matvec_fp8_div((uint32_t)row, m.sslice));
    } else {
      return m.nt;
    }
  }

  __device__ __forceinline__ void flush(float (&acc)[NT], float* slot, int lane, uint32_t ns) const {
#pragma unroll
    for (int t = 0; t < NT; t++) {
      float v = acc[t];
#pragma unroll
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == t && (uint32_t)t < ns) slot[t] = v;
      acc[t] = 0.f;
    }
  }

  // The quarter plane of bitstream `stream` of chunk c is in S.plane (count elements from plane byte out_off).
  template <int G>
  __device__ __forceinline__ void quarter(const SyncShared& S, uint64_t c, int stream, uint32_t out_off, uint32_t count, bool rot) const {
    static_assert(G == 16 / EPV, "one byte plane per byte of the element");
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t nv = count / EPV;
    const uint32_t vpw = ((nv + 255u) >> 8) << 5;
    const uint32_t v0 = (uint32_t)wid * vpw, v1 = min(nv, v0 + vpw);
    if (v0 >= v1) return;  // (warp-uniform) a short last chunk leaves the upper warps without a block
    const uint64_t in = m.in;
    const uint64_t e0 = c * m.ce + out_off + (uint64_t)v0 * EPV;
    uint64_t row0 = e0 / in, col0 = e0 - row0 * in;  // of the step's first element: the same in every lane
    float* const slots = m.part + ((c * 4 + (uint32_t)stream) * 8 + (uint32_t)wid) * m.rs * m.nt;  // the block's, from its first row
    const uint64_t first = row0;
    const uint8_t* const xb = reinterpret_cast<const uint8_t*>(m.x);
    float acc[NT];
#pragma unroll
    for (int t = 0; t < NT; t++) acc[t] = 0.f;
    [[maybe_unused]] uint32_t xo[NT];       // EXPERTS: the element offset of slot t's x row, for expert xe
    [[maybe_unused]] uint32_t xe = ~0u;
    uint64_t cur = row0;
    for (uint32_t v = v0; v < v1; v += 32) {
      const uint32_t nvalid = min(32u, v1 - v);
      const bool valid = (uint32_t)lane < nvalid;
      uint64_t lrow = row0, lcol = col0 + (uint32_t)lane * EPV;
      uint64_t last = row0;
      if (col0 + 32u * EPV > in) {  // (uniform) the step straddles rows
        const uint64_t q = lcol / in;
        lrow += q;
        lcol -= q * in;
        last += (col0 + nvalid * EPV - 1) / in;
      }
      float p[NT];
#pragma unroll
      for (int t = 0; t < NT; t++) p[t] = 0.f;
      // The lane's 16 decoded bytes times x.  Each product decodes in a `valid` block of its own: with one block shared
      // around both, ptxas assigned some k_matvec registers differently.
      if constexpr (FMT < 0) {
        if (valid) {
          uint32_t r[4];
          const uint32_t o = (v + (uint32_t)lane) * 16u;
          ZB_FUSED_VECTOR(G, S, out_off, o, rot, r);
          float w[EPV];
          matvec_floats<DT, EPV>(r, w);
#pragma unroll
          for (int t = 0; t < NT; t++) {
            const uint64_t tt = min((uint32_t)t, m.nt - 1u);
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xb + (tt * m.xs + lcol) * matvec_esize(DT)));
            const uint32_t xr[4] = {xv.x, xv.y, xv.z, xv.w};
            float xf[EPV];
            matvec_floats<DT, EPV>(xr, xf);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < EPV; i++) s = fmaf(w[i], xf[i], s);
            p[t] = s;
          }
        }
      } else if (valid) {
        uint32_t r[4];
        const uint32_t o = (v + (uint32_t)lane) * 16u;
        ZB_FUSED_VECTOR(G, S, out_off, o, rot, r);
        float sc;
        if constexpr (EXPERTS) {
          const uint32_t e = matvec_fp8_div((uint32_t)lrow, m.sslice), er = (uint32_t)lrow - e * m.slice_rows;
          sc = __ldg(m.scale + e * m.slice_grid + matvec_fp8_div(er, m.srow) * m.scols + matvec_fp8_div((uint32_t)lcol, m.scol));
          if (e != xe) {
            xe = e;
            const uint32_t n = __ldg(m.cnt + e);
#pragma unroll
            for (int t = 0; t < NT; t++) {
              const uint32_t p = n ? __ldg(m.tab + e * NT + min((uint32_t)t, n - 1u)) : 0u;
              xo[t] = matvec_fp8_div(p, m.xdiv) * (uint32_t)m.xs;
            }
          }
        } else {
          sc = __ldg(m.scale + matvec_fp8_div((uint32_t)lrow, m.srow) * m.scols + matvec_fp8_div((uint32_t)lcol, m.scol));
        }
        // in two halves of 8 columns, every token's sum carried from the first to the second (the order of each sum
        // is the same), the half loop not unrolled: only 16 bytes of x per token are in flight at once.  Unrolled, the
        // compiler issues all 32 bytes of every token together and NT = 8 spills at 80 registers.
#pragma unroll 1
        for (int h = 0; h < 2; h++) {
          float w[8];
          fp8_floats<FMT>(h ? r[2] : r[0], h ? r[3] : r[1], w);
#pragma unroll
          for (int t = 0; t < NT; t++) {
            uint64_t xrow;
            if constexpr (EXPERTS) {
              xrow = xo[t];
            } else {
              xrow = min((uint32_t)t, m.nt - 1u) * m.xs;
            }
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xb + (xrow + lcol) * 2) + h);
            const uint32_t xr[4] = {xv.x, xv.y, xv.z, xv.w};
            float xf[8];
            matvec_floats<DT, 8>(xr, xf);
#pragma unroll
            for (int i = 0; i < 8; i++) p[t] = fmaf(w[i], xf[i], p[t]);
          }
        }
#pragma unroll
        for (int t = 0; t < NT; t++) p[t] *= sc;
      }
      for (uint64_t rr = row0; rr <= last; rr++) {
        if (rr != cur) {
          flush(acc, slots + (cur - first) * m.nt, lane, stored(cur));
          cur = rr;
        }
        if (lrow == rr) {
#pragma unroll
          for (int t = 0; t < NT; t++) acc[t] += p[t];
        }
      }
      row0 += m.step_rows;
      col0 += m.step_cols;
      if (col0 >= in) {
        col0 -= in;
        row0++;
      }
    }
    flush(acc, slots + (cur - first) * m.nt, lane, stored(cur));
  }
};

// The bitstream loop of k_matvec and k_matmul: one CTA per coded bitstream of the item (every chunk is fused: its one
// coded item is the top byte plane), each decoded as by a plan run, with the epilogue's `quarter` in place of its stores.
template <int G, typename Ep>
__device__ __forceinline__ void product_streams(const ProductCfg& m, const Ep& ep) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const DecodeCfg& cfg = *m.cfg;
  const uint64_t works = 4ull * cfg.ctrl->huf_count;
  for (uint64_t work = blockIdx.x; work < works; work += gridDim.x) {
    __syncthreads();  // the previous bitstream's shared state is dead
    sync_process<G, false, kSyncReplay, false, Ep>(cfg, nullptr, S, cv.lut, cv.lut_s, work, m.seg + work * kSyncThreads, nullptr, &ep);
  }
}

// The reduce kernels' frame: one thread per (token t, output row o).  sum(t, o) adds the row's partial sums in
// ascending element order; the bias is added, the result rounded once to the output type and stored.
template <int DT, typename Sum>
__device__ __forceinline__ void product_reduce(const ProductCfg& m, Sum&& sum) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t e = *(volatile uint32_t*)&m.cfg->ctrl->error;  // a decode error of this call
    if (e) atomicOr(m.error, e);
  }
  const uint64_t idx = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (idx >= m.out * m.nt) return;
  const uint64_t t = idx / m.out, o = idx - t * m.out;
  float s = sum(t, o);
  if (DT == kMvBf16) {
    if (m.bias) s += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(m.bias)[o]);
    reinterpret_cast<__nv_bfloat16*>(m.y)[t * m.ys + o] = __float2bfloat16_rn(s);
  } else if (DT == kMvFp16) {
    if (m.bias) s += __half2float(reinterpret_cast<const __half*>(m.bias)[o]);
    reinterpret_cast<__half*>(m.y)[t * m.ys + o] = __float2half_rn(s);
  } else {
    if (m.bias) s += reinterpret_cast<const float*>(m.bias)[o];
    reinterpret_cast<float*>(m.y)[t * m.ys + o] = s;
  }
}

template <int DT, int NT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_matvec(ProductCfg m) {
  product_streams<matvec_esize(DT)>(m, MatvecEp<DT, NT>{m});
}

template <int DT>
__global__ void __launch_bounds__(256) k_matvec_reduce(ProductCfg m) {
  product_reduce<DT>(m, [&](uint64_t t, uint64_t o) {
    float s = 0.f;
    for (uint64_t e = o * m.in; e < (o + 1) * m.in;) {
      const MatvecBlock b = matvec_block_of(m, e);
      s += m.part[((b.id * m.rs) + o - b.start / m.in) * m.nt + t];
      e = b.end;
    }
    return s;
  });
}

// fp8 weights: the partial sums are k_matvec_reduce<XDT>'s, whose block geometry comes from m.esize (1).
template <int FMT, int XDT, int NT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_matvec_fp8(ProductCfg m) {
  product_streams<1>(m, MatvecEp<XDT, NT, FMT>{m});
}

// The 8 fp8 weights of two words a, b as ODT (bf16 or fp16), each converted exactly, multiplied by the scale sc in fp32
// and rounded once to nearest even: word i of the result holds weights 2i and 2i + 1.  The dequantize's store and the
// fp8 matmul's B fragments (matmul.cuh).
template <int FMT, int ODT>
__device__ __forceinline__ uint4 fp8_dequant8(uint32_t a, uint32_t b, float sc) {
  float w[8];
  fp8_floats<FMT>(a, b, w);
  uint32_t h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if constexpr (ODT == kMvBf16) {
      const __nv_bfloat162 v = __floats2bfloat162_rn(w[2 * i] * sc, w[2 * i + 1] * sc);
      h[i] = *reinterpret_cast<const uint32_t*>(&v);
    } else {
      const __half2 v = __floats2half2_rn(w[2 * i] * sc, w[2 * i + 1] * sc);
      h[i] = *reinterpret_cast<const uint32_t*>(&v);
    }
  }
  return make_uint4(h[0], h[1], h[2], h[3]);
}

// ---- the dequantized fp8 weight (k_dequant_fp8) ---------------------------------------------------------------------
// out[o][i] = ODT(float(W[o][i]) * S[o / bn][i / bk]), W and S as for k_matvec_fp8, out the contiguous bf16 / fp16
// tensor [out][in] at m.y.  Bit for bit torch's (W.to(float32) * S_expanded).to(ODT): fp8 -> fp32 is exact, then one
// fp32 multiply and one round to nearest even (fp16 overflow to +-inf); NaN stays NaN (its payload may differ).
// The run's store loop with a different store: thread t takes the vectors t, t + 256, ... of the quarter plane, and
// since out is contiguous a vector's element index is also its output index.  Only the scale lookup needs (row, col),
// by multiply-highs (every element index is below 2^31: the host admits total <= INT32_MAX).  A lane converts its 16
// bytes, multiplies each by the block's one scale (bk % 16 == 0, in % 16 == 0: the vector lies in one row and block)
// and stores 32 bytes.
// SLICED: the scale grid is one grid per slice [e] of a tensor [rows][slice_rows][in] (fp8 experts, whose slice rows
// need not be a multiple of bn): the slice comes first, s = row / slice_rows, then the block of row - s * slice_rows
// in the slice's grid at s * slice_grid.  The selected dequantize (select.cuh) only.
template <int FMT, int ODT, bool SLICED = false>
struct DequantEp {
  static_assert(ODT == kMvBf16 || ODT == kMvFp16, "bf16 or fp16 out");
  static constexpr bool on = true;
  ProductCfg m;

  template <int G>
  __device__ __forceinline__ void quarter(const SyncShared& S, uint64_t c, int stream, uint32_t out_off, uint32_t count, bool rot) const {
    static_assert(G == 1, "fp8: one byte plane");
    const uint64_t rin = matvec_fp8_recip(m.in);
    const uint32_t in = (uint32_t)m.in, e0 = (uint32_t)(c * m.ce) + out_off;
    for (uint32_t o = threadIdx.x * 16u; o < count; o += kSyncThreads * 16u) {
      uint32_t r[4];
      ZB_FUSED_VECTOR(G, S, out_off, o, rot, r);
      const uint32_t e = e0 + o, row = matvec_fp8_div(e, rin), col = e - row * in;
      float sc;
      if constexpr (SLICED) {
        const uint32_t s = matvec_fp8_div(row, m.sslice), r = row - s * m.slice_rows;
        sc = __ldg(m.scale + s * m.slice_grid + matvec_fp8_div(r, m.srow) * m.scols + matvec_fp8_div(col, m.scol));
      } else {
        sc = __ldg(m.scale + matvec_fp8_div(row, m.srow) * m.scols + matvec_fp8_div(col, m.scol));
      }
      const uint4 lo = fp8_dequant8<FMT, ODT>(r[0], r[1], sc), hi = fp8_dequant8<FMT, ODT>(r[2], r[3], sc);
      uint4* const dst = reinterpret_cast<uint4*>(m.y) + (e >> 3);
      dst[0] = lo;
      dst[1] = hi;
    }
  }
};

template <int FMT, int ODT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_dequant_fp8(ProductCfg m) {
  product_streams<1>(m, DequantEp<FMT, ODT>{m});
}

}  // namespace zb
