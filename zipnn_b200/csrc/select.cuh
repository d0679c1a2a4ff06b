// select.cuh -- a decode plan's run restricted to the slices [e] (along dim 0) that a list of ids selects.
//
// Every item of the plan is one whole-tensor piece of `rows` slices of orig / rows bytes each (the experts of a
// mixture-of-experts layer: gate_up_proj [E, 2I, H], down_proj [E, H, I]).  A selected run does the plan run's work
// for the chunks that meet a selected slice and nothing else, through the same device functions:
//
//   k_select_index     (one CTA) per item: marks the chunks each (id, chunk of its slice) touches in a shared-memory
//                      bitmap, raises kErrIndex for an id outside [0, rows), and compacts the item's three work lists
//                      in order: the hlist positions of coded items of marked chunks, the regroup tiles of marked
//                      rlist chunks, the marked olist chunks.  The counts go to the scratch, and for the overflow
//                      kernel a copy of the item's DecodeCfg whose olist and ctrl are the selection's;
//   k_select_sync      the replay decoder (sync_process, kSyncReplay) over the selected bitstreams;
//   k_select_regroup   regroup_tile over the selected tiles;
//   k_select_overflow  decode_overflow_part over the selected overflow chunks, on the plan's overflow plane slots;
//   (k_batch_errors    as after a plan run.)
// k_select_dequant_fp8 (below) is k_select_sync for fp8 experts with k_dequant_fp8's dequantizing stores.
// Grids come from bounds the host knows (ids, the most chunks a slice can touch, resident CTAs), never from the ids,
// so the launch sequence is fixed and a selected run can be captured in a CUDA graph and replayed with new ids.
// A chunk that straddles two slices is decoded whole; no byte of a chunk that meets no selected slice is written.
// The scratch holds nothing from one call to the next, so calls that share it are ordered on one stream; the run also
// uses the plan's own scratch (plane pools), under the plan run's rule.
#pragma once
#include "decode_sync.cuh"
#include "gather.cuh"
#include "matvec.cuh"

namespace zb {

struct SelectCfg {
  const void* ids;
  uint64_t n;         // ids
  int id8;            // 8-byte ids (else 4)
  uint64_t rows;      // slices per item
  uint32_t* error;    // the plan's error word
  uint32_t* count;    // [0] selected coded items, [1] selected regroup tiles (scratch)
  uint2* hsel;        // {piece, hlist position}                        [coded items of the plan]
  uint2* tsel;        // {piece, rlist position * tiles per chunk + tile} [regroup tiles of the plan]
  uint32_t* osel;     // piece t's selected olist chunks at chunk_start[t] [chunks of the plan]
  DecodeCfg* ocfg;    // [pieces] the piece's DecodeCfg with olist = its osel, ctrl = its octrl
  Ctrl* octrl;        // [pieces] overflow_count = its selected overflow chunks; error: raised by k_select_overflow
};

__device__ __forceinline__ int64_t select_id(const SelectCfg& s, uint64_t t) {
  return s.id8 ? reinterpret_cast<const int64_t*>(s.ids)[t] : (int64_t)reinterpret_cast<const int32_t*>(s.ids)[t];
}

// Block-wide exclusive prefix sum of v (all threads call); `total` = the sum.
__device__ __forceinline__ uint32_t select_scan(uint32_t v, uint32_t* warp_tot, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += u;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  uint32_t before = 0;
  total = 0;
  for (uint32_t w = 0; w < blockDim.x / 32; w++) {
    const uint32_t u = warp_tot[w];
    if (w < wid) before += u;
    total += u;
  }
  __syncthreads();  // warp_tot is free for the next scan
  return before + incl - v;
}

__global__ void __launch_bounds__(kGatherIndexThreads) k_select_index(BatchCfg B, SelectCfg s) {
  __shared__ uint32_t bits[kGatherMaxChunks / 32];
  __shared__ uint32_t warp_tot[kGatherIndexThreads / 32];
  const uint32_t tid = threadIdx.x;
  uint32_t hc = 0, tc = 0;  // (uniform) entries of hsel and tsel so far
  for (uint32_t t = 0; t < B.n; t++) {
    const DecodeCfg& cfg = B.cfgs[t];
    const uint64_t K = cfg.K, chunk = cfg.chunk, slice = cfg.orig / s.rows;
    const uint64_t span = min(K, (slice + chunk - 2) / chunk + 1);  // chunks one slice may touch at most
    const uint64_t wspan = (span + 30) / 32 + 1;                      // bitmap words those chunks may lie in
    const uint32_t nw = (uint32_t)((K + 31) / 32);
    for (uint32_t i = tid; i < nw; i += blockDim.x) bits[i] = 0;
    __syncthreads();
    // unit = (id, bitmap word of its slice's chunk range): one atomic marks up to 32 chunks
    for (uint64_t u = tid; u < s.n * wspan; u += blockDim.x) {
      const uint64_t i = u / wspan, j = u - i * wspan;
      const int64_t id = select_id(s, i);
      if (id < 0 || (uint64_t)id >= s.rows) {
        if (t == 0 && j == 0) atomicOr(s.error, kErrIndex);
        continue;
      }
      const uint64_t b = (uint64_t)id * slice;
      const uint64_t c0 = b / chunk, c1 = (b + slice - 1) / chunk;
      const uint64_t w = c0 / 32 + j;
      if (w > c1 / 32) continue;
      const uint32_t lo = (uint32_t)(max(c0, 32 * w) - 32 * w), hi = (uint32_t)(min(c1, 32 * w + 31) - 32 * w);
      atomicOr(&bits[w], (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo));
    }
    __syncthreads();
    auto marked = [&](uint64_t c) { return (bits[c >> 5] >> (c & 31)) & 1u; };
    // coded items (g * K + c) of marked chunks
    const uint32_t nh = cfg.ctrl->huf_count;
    for (uint32_t at = 0; at < nh; at += blockDim.x) {
      const uint32_t pos = at + tid;
      const uint32_t f = pos < nh ? marked(cfg.hlist[pos] % K) : 0u;
      uint32_t total;
      const uint32_t off = select_scan(f, warp_tot, total);
      if (f) s.hsel[hc + off] = make_uint2(t, pos);
      hc += total;
    }
    // regroup tiles of marked plain and general chunks
    const uint32_t tpc = (cfg.chunk + kMergeTile - 1) / kMergeTile;
    const uint32_t nr = cfg.ctrl->regroup_count;
    for (uint32_t at = 0; at < nr; at += blockDim.x) {
      const uint32_t j = at + tid;
      const uint32_t f = j < nr ? marked(cfg.rlist[j]) : 0u;
      uint32_t total;
      const uint32_t off = select_scan(f * tpc, warp_tot, total);
      for (uint32_t k = 0; k < f * tpc; k++) s.tsel[tc + off + k] = make_uint2(t, j * tpc + k);
      tc += total;
    }
    // marked overflow chunks, in olist order
    uint32_t* osel = s.osel + B.chunk_start[t];
    const uint32_t no = cfg.ctrl->overflow_count;
    uint32_t oc = 0;
    for (uint32_t at = 0; at < no; at += blockDim.x) {
      const uint32_t i = at + tid;
      const uint32_t c = i < no ? cfg.olist[i] : 0u;
      const uint32_t f = i < no ? marked(c) : 0u;
      uint32_t total;
      const uint32_t off = select_scan(f, warp_tot, total);
      if (f) osel[oc + off] = c;
      oc += total;
    }
    if (tid == 0) {
      Ctrl& oc_ctrl = s.octrl[t];
      oc_ctrl.error = 0;
      oc_ctrl.overflow_count = oc;
      DecodeCfg d = cfg;
      d.olist = osel;
      d.ctrl = &oc_ctrl;
      s.ocfg[t] = d;
    }
    __syncthreads();  // the bitmap is reused by the next item
  }
  if (tid == 0) {
    s.count[0] = hc;
    s.count[1] = tc;
  }
}

// The selected bitstreams: unit w = bitstream w & 3 of the coded item at hsel[w >> 2].  Whole-tensor pieces only (no
// box).  Bounded to k_huf_decode_sync_plan's budget: 80 registers, three CTAs per SM.
__global__ void __launch_bounds__(kSyncThreads, 3) k_select_sync(BatchCfg B, SegIndex X, SelectCfg s) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const uint64_t units = 4ull * *s.count;
  for (uint64_t w = blockIdx.x; w < units; w += gridDim.x) {
    const uint2 e = s.hsel[w >> 2];
    const DecodeCfg& cfg = B.cfgs[e.x];
    const uint64_t work = 4ull * e.y + (w & 3);
    __syncthreads();  // the previous unit's shared state is dead
    sync_process_any<false, kSyncReplay>(cfg, S, cv, work, X.seg + X.base[e.x] + work * kSyncThreads);
  }
}

// ---- the selected fp8 dequantize (k_select_dequant_fp8) -----------------------------------------------------------
// A selected run of a plan whose items are fp8 experts (every chunk fused, G = 1) with k_dequant_fp8's stores in place
// of the run's: the bitstreams k_select_index picked are decoded by the replay decoder, and DequantEp (matvec.cuh, the
// per-slice grid) writes each 16-byte vector dequantized to item t's d.m[t].y.  Fused items have no regroup tiles and
// no overflow chunks, so only hsel matters; a call is k_select_index, this kernel and k_batch_errors.  The items'
// ProductCfgs are a kernel parameter (no copy to the device per call): a graph replays with new ids and new scales.
constexpr int kSelectFp8MaxItems = 4;
struct SelectFp8Items {
  ProductCfg m[kSelectFp8MaxItems];  // per plan item, in item order
};

template <int FMT, int ODT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_select_dequant_fp8(SelectCfg s, const __grid_constant__ SelectFp8Items d) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const uint64_t units = 4ull * *s.count;
  for (uint64_t w = blockIdx.x; w < units; w += gridDim.x) {
    const uint2 e = s.hsel[w >> 2];
    const DequantEp<FMT, ODT, true> ep{d.m[e.x]};
    const uint64_t work = 4ull * e.y + (w & 3);
    __syncthreads();  // the previous unit's shared state is dead
    sync_process<1, false, kSyncReplay, false, DequantEp<FMT, ODT, true>>(*ep.m.cfg, nullptr, S, cv.lut, cv.lut_s, work,
                                                                         ep.m.seg + work * kSyncThreads, nullptr, &ep);
  }
}

// ---- the selected experts matvec (k_select_matvec_fp8) --------------------------------------------------------------
// y[p][o] = XDT(sum_i x_p[i] * (float(W[ids[p]][o][i]) * S[ids[p]][o / bn][i / bk])) for every pair p = t * k + j of
// ids [T][k], x_p = x[p / k] (one x row per token) or x[p] (one per pair), on one item [E][out][in] of fp8 experts
// (ExpertsCfg, matvec.cuh).  A call is five launches, whatever the ids: k_select_index on the one item, k_select_pairs,
// k_select_matvec_fp8, k_select_matvec_reduce, k_batch_errors.  The product kernel is k_select_dequant_fp8's loop over
// the selected bitstreams with MatvecEp's experts form: a warp's partial sums take the matvec's slots ([32 K blocks]
// [rs][nt] of the whole item), where slot t of a row is the t-th pair routed to the row's expert.  Only the slots of
// routed experts' rows in selected chunks are written, and the reduce reads only those, so the sums of a pair are
// matvec_fp8's for the expert's rows: the same products, the same order, the same rounding.

// (one CTA) The pair tables of the n = T * k ids over s.rows = E experts: cnt[e] pairs routed to e, tab[e][0..nt) their
// numbers in ascending p, pos[p] p's slot in its expert's list.  Each pair counts the equal ids before and after it
// (n is at most 4 * k), so nothing depends on thread order and there are no atomics but the error.  An id outside
// [0, E) marks nothing (k_select_index raises kErrIndex for it); an expert given more than nt pairs (a token that
// repeats an expert) raises kErrIndex, and its count stops at nt.  The counts are zeroed here: a call needs no memset.
__global__ void __launch_bounds__(kGatherIndexThreads) k_select_pairs(SelectCfg s, ExpertsCfg m) {
  for (uint64_t e = threadIdx.x; e < s.rows; e += blockDim.x) m.cnt[e] = 0;
  __syncthreads();
  for (uint64_t p = threadIdx.x; p < s.n; p += blockDim.x) {
    const int64_t id = select_id(s, p);
    if (id < 0 || (uint64_t)id >= s.rows) continue;
    uint32_t before = 0, after = 0;
    for (uint64_t q = 0; q < s.n; q++) {
      if (select_id(s, q) == id) {
        before += q < p;
        after += q > p;
      }
    }
    m.pos[p] = before;
    if (before < m.nt) {
      m.tab[(uint64_t)id * m.nt + before] = (uint32_t)p;
    } else {
      atomicOr(s.error, kErrIndex);
    }
    if (after == 0) m.cnt[id] = min(before + 1u, m.nt);
  }
}

// Pair slots per expert: 1, 2 or 4 (T rounded up to a power of two).  With 8, a lane's sums and x row offsets need more
// than the 80 registers of three CTAs per SM, and ptxas spills.
constexpr int kExpertsMaxTokens = 4;

template <int FMT, int XDT, int NT>
__global__ void __launch_bounds__(kSyncThreads, 3) k_select_matvec_fp8(SelectCfg s, ExpertsCfg m) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  static_assert(NT <= kExpertsMaxTokens, "no spills");
  using Ep = MatvecEp<XDT, NT, FMT, true>;
  const Ep ep{m};
  const uint64_t units = 4ull * *s.count;
  for (uint64_t w = blockIdx.x; w < units; w += gridDim.x) {
    const uint64_t work = 4ull * s.hsel[w >> 2].y + (w & 3);  // (one item: the piece is 0)
    __syncthreads();  // the previous unit's shared state is dead
    sync_process<1, false, kSyncReplay, false, Ep>(*m.cfg, nullptr, S, cv.lut, cv.lut_s, work, m.seg + work * kSyncThreads, nullptr, &ep);
  }
}

// One thread per (pair p, output o): R = ids[p] * out + o.  R's partial sums at slot pos[p], added in ascending element
// order from +0 as k_matvec_reduce adds them, rounded once to XDT and stored at y[p * ys + o].  A pair with an invalid
// id, or past its expert's slots, writes nothing.
template <int XDT>
__global__ void __launch_bounds__(256) k_select_matvec_reduce(SelectCfg s, ExpertsCfg m) {
  const uint64_t out = m.slice_rows;
  const uint64_t idx = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (idx >= s.n * out) return;
  const uint64_t p = idx / out, o = idx - p * out;
  const int64_t id = select_id(s, p);
  if (id < 0 || (uint64_t)id >= s.rows) return;
  const uint32_t slot = m.pos[p];
  if (slot >= m.nt) return;
  const uint64_t R = (uint64_t)id * out + o;
  float sum = 0.f;
  for (uint64_t e = R * m.in; e < (R + 1) * m.in;) {
    const MatvecBlock b = matvec_block_of(m, e);
    sum += m.part[((b.id * m.rs) + R - b.start / m.in) * m.nt + slot];
    e = b.end;
  }
  if constexpr (XDT == kMvBf16) {
    reinterpret_cast<__nv_bfloat16*>(m.y)[p * m.ys + o] = __float2bfloat16_rn(sum);
  } else {
    reinterpret_cast<__half*>(m.y)[p * m.ys + o] = __float2half_rn(sum);
  }
}

// The selected regroup tiles (k_regroup_batch's tile numbering within a piece).
__global__ void __launch_bounds__(kMergeThreads) k_select_regroup(BatchCfg B, SelectCfg s) {
  __shared__ PlaneSrc src[4];
  const uint32_t total = s.count[1];
  for (uint32_t w = blockIdx.x; w < total; w += gridDim.x) {
    const uint2 e = s.tsel[w];
    const DecodeCfg& cfg = B.cfgs[e.x];
    const uint32_t tpc = (cfg.chunk + kMergeTile - 1) / kMergeTile;
    regroup_tile_any<false>(cfg, cfg.rlist[e.y / tpc], e.y % tpc, src);
  }
}

// The selected overflow chunks.  grid = (overflow CTAs, pieces); CTA x of a piece owns the plan's plane slot
// max_slots + x, as in k_decode_overflow_batch.  Decode errors land in the selection's ctrl and go on to the plan's
// error word.
__global__ void __launch_bounds__(kMergeThreads) k_select_overflow(SelectCfg s) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ PlaneSrc src[4];
  const DecodeCfg& cfg = s.ocfg[blockIdx.y];
  const uint32_t ncta = min(cfg.ovf_slots, gridDim.x);
  if (blockIdx.x >= ncta || cfg.ctrl->overflow_count == 0) return;  // (uniform)
  decode_overflow_to<false>(cfg, cfg.out, *reinterpret_cast<DecodeSmem*>(smem_raw), src, blockIdx.x, ncta);
  if (threadIdx.x == 0) {
    const uint32_t e = atomicOr(&cfg.ctrl->error, 0u);
    if (e) atomicOr(s.error, e);
  }
}

}  // namespace zb
