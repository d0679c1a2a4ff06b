// gather.cuh -- rows of a decode plan's tensor, decoded from the chunks the ids touch and nothing else.
//
// out[t] = rows[ids[t]] for a whole-tensor item of a decode plan, with the ids on the device (an embedding lookup
// from compressed weights).  Everything the plan's create built for the item is reused: descriptors, item tables,
// chunk modes, parsed Huffman tables and the recorded segment index.  One call is a fixed sequence of launches that
// depends on n = number of ids and on the scratch's slot count only, never on the id values:
//
//   k_gather_index   (CTA 0) marks the chunks each (token, chunk of its row) needs in a shared-memory bitmap,
//                    raises kErrIndex for an id outside [0, rows), and compacts the bitmap into the ascending list
//                    of touched chunks (list[i]) and each chunk's list position (pos[c]);
//                    (the other CTAs) build the inverse of the piece's hlist: coded item -> hlist position, which
//                    addresses the tables and the segment index;
//   per pass p       chunks list[p * slots, (p + 1) * slots) take scratch slots 0 .. slots - 1:
//     k_gather_decode  decodes their coded bitstreams into the slots' planes: sync_process in replay mode for fused
//                      and general chunks, planar_decode_item (one lane per bitstream) for overflow chunks, whose
//                      items the plan never indexed;
//     k_gather_rows    merges the planes of those chunks (coded planes from the slots, raw and RLE planes straight
//                      from the stream, as regroup_tile), un-rotates, and writes the requested bytes to out.  Rows of
//                      bad ids are zeroed by pass 0.
// Passes past the last touched chunk return at once.  The scratch holds nothing from one call to the next (the bitmap
// lives in shared memory), so it follows the plan scratch's rule: calls that share it are ordered on one stream.
#pragma once
#include "decode_sync.cuh"

namespace zb {

constexpr int kGatherIndexThreads = 1024;
constexpr uint32_t kGatherMaxChunks = 16384;   // one whole-tensor piece of a plan (kSyncTablesMaxChunks)

struct GatherCfg {
  const DecodeCfg* cfg;   // the item's piece, in plan memory
  SegEntry* seg;          // the piece's segment index
  uint32_t* error;        // the plan's error word
  const void* ids;
  uint64_t n;             // ids
  int id8;                // 8-byte ids (else 4)
  int G;
  uint64_t K, orig, rows, row_bytes, span;  // span: chunks one row may touch at most
  uint32_t chunk, slots;
  uint8_t* out;
  uint32_t* count;        // touched chunks (scratch)
  uint32_t* list;         // [K]
  uint32_t* pos;          // [K]
  uint32_t* inv;          // [G * K]
  uint8_t* planes;        // [slots][G][pstride]
  uint64_t pstride;
};

__device__ __forceinline__ int64_t gather_id(const GatherCfg& g, uint64_t t) {
  return g.id8 ? reinterpret_cast<const int64_t*>(g.ids)[t] : (int64_t)reinterpret_cast<const int32_t*>(g.ids)[t];
}
__device__ __forceinline__ bool gather_bad(const GatherCfg& g, int64_t id) { return id < 0 || (uint64_t)id >= g.rows; }

__global__ void __launch_bounds__(kGatherIndexThreads) k_gather_index(GatherCfg g) {
  const uint32_t tid = threadIdx.x;
  if (blockIdx.x > 0) {
    const uint32_t nh = g.cfg->ctrl->huf_count;
    const uint32_t* hl = g.cfg->hlist;
    for (uint32_t i = (blockIdx.x - 1) * kGatherIndexThreads + tid; i < nh; i += (gridDim.x - 1) * kGatherIndexThreads) g.inv[hl[i]] = i;
    return;
  }
  __shared__ uint32_t bits[kGatherMaxChunks / 32];
  __shared__ uint32_t warp_tot[kGatherIndexThreads / 32];
  const uint32_t nw = (uint32_t)((g.K + 31) / 32);
  for (uint32_t i = tid; i < nw; i += kGatherIndexThreads) bits[i] = 0;
  __syncthreads();
  const uint64_t units = g.n * g.span;
  for (uint64_t u = tid; u < units; u += kGatherIndexThreads) {
    const uint64_t t = u / g.span, j = u - t * g.span;
    const int64_t id = gather_id(g, t);
    if (gather_bad(g, id)) {
      if (j == 0) atomicOr(g.error, kErrIndex);
      continue;
    }
    const uint64_t b = (uint64_t)id * g.row_bytes;
    const uint64_t c = b / g.chunk + j;
    if (c <= (b + g.row_bytes - 1) / g.chunk) atomicOr(&bits[c >> 5], 1u << (c & 31));
  }
  __syncthreads();
  // compaction: thread tid owns words [w0, w1); exclusive scan of their popcounts
  const uint32_t per = (nw + kGatherIndexThreads - 1) / kGatherIndexThreads;
  const uint32_t w0 = min(nw, tid * per), w1 = min(nw, w0 + per);
  uint32_t mine = 0;
  for (uint32_t w = w0; w < w1; w++) mine += __popc(bits[w]);
  const uint32_t lane = tid & 31, wid = tid >> 5;
  uint32_t incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += v;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  uint32_t before = 0, total = 0;
  for (uint32_t w = 0; w < kGatherIndexThreads / 32; w++) {
    const uint32_t v = warp_tot[w];
    if (w < wid) before += v;
    total += v;
  }
  uint32_t at = before + incl - mine;
  for (uint32_t w = w0; w < w1; w++) {
    uint32_t m = bits[w];
    while (m) {
      const uint32_t c = 32u * w + (uint32_t)(__ffs(m) - 1);
      m &= m - 1;
      g.list[at] = c;
      g.pos[c] = at;
      at++;
    }
  }
  if (tid == 0) *g.count = total;
}

// The coded planes of the chunks of pass `pass`.  Work unit = (list entry, group, bitstream).
template <int G>
__device__ __forceinline__ void gather_sync_unit(const DecodeCfg& cfg, SyncShared& S, const SyncCarve& cv, uint64_t work, SegEntry* seg,
                                                 uint8_t* gplanes) {
  sync_process<G, false, kSyncReplay, true>(cfg, nullptr, S, cv.lut, cv.lut_s, work, seg, gplanes);
}
// An overflow chunk (warp 0): one lane per bitstream, as decode_overflow_part, into the chunk's slot planes.  A call of
// its own, so that its registers do not weigh on the replay decoder.
__device__ __noinline__ void gather_overflow(const GatherCfg& g, const DecodeCfg& cfg, DecodeSmem& D, uint32_t c, uint8_t* gp) {
  const int lane = threadIdx.x, sl = lane >> 2, stream = lane & 3;
  ItemDesc d;
  d.kind = kRaw;
  d.src_off = 0;
  d.src_len = d.dec_len = 0;
  bool active = false;
  if (sl < g.G) {
    d = cfg.items[(uint64_t)sl * g.K + c];
    active = d.kind == kHuf;
  }
  planar_decode_item(D, cfg, d, active, sl, stream, gp + (uint64_t)(sl < g.G ? sl : 0) * g.pstride);
}
__global__ void __launch_bounds__(kSyncThreads, 1) k_gather_decode(GatherCfg g, uint32_t pass) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const uint32_t m = *g.count;
  const uint64_t first = (uint64_t)pass * g.slots;
  if (first >= m) return;
  const DecodeCfg& cfg = *g.cfg;
  const uint32_t per = 4u * (uint32_t)g.G;
  const uint64_t units = min((uint64_t)g.slots, m - first) * per;
  for (uint64_t w = blockIdx.x; w < units; w += gridDim.x) {
    const uint64_t e = w / per;
    const uint32_t r = (uint32_t)(w - e * per);
    const uint32_t c = g.list[first + e];
    const uint32_t mode = cfg.mode[c];
    uint8_t* gp = g.planes + e * (uint64_t)g.G * g.pstride;
    if (mode == kModeOverflow) {
      if (r != 0) continue;  // (uniform) one CTA per overflow chunk: its warp 0 decodes every coded bitstream
      __syncthreads();       // the shared memory's previous use is over
      if (threadIdx.x < 32) gather_overflow(g, cfg, *reinterpret_cast<DecodeSmem*>(smem_raw), c, gp);
      continue;
    }
    if (mode != kModeFused && mode != kModeGeneral) continue;  // (uniform) no coded plane
    const uint64_t item = (uint64_t)(r >> 2) * g.K + c;
    if (cfg.items[item].kind != kHuf) continue;  // (uniform)
    const uint64_t work = 4ull * g.inv[item] + (r & 3);
    __syncthreads();  // the previous unit's shared state is dead
    if (g.G == 1) gather_sync_unit<1>(cfg, S, cv, work, g.seg + work * kSyncThreads, gp);
    else if (g.G == 2) gather_sync_unit<2>(cfg, S, cv, work, g.seg + work * kSyncThreads, gp);
    else gather_sync_unit<4>(cfg, S, cv, work, g.seg + work * kSyncThreads, gp);
  }
}

// Byte idx of plane gsel, with a static index into src (a dynamic one puts src in local memory).
template <int G>
__device__ __forceinline__ uint8_t gather_byte(const PlaneSrc (&src)[G], uint32_t gsel, uint32_t idx) {
  uint8_t b = 0;
#pragma unroll
  for (int q = 0; q < G; q++)
    if (gsel == (uint32_t)q) b = plane_byte(src[q], idx);
  return b;
}
// Plane source of group q of chunk c: raw bytes in the stream, one RLE byte, or the decoded plane in the slot.
template <int G>
__device__ __forceinline__ void gather_srcs(const GatherCfg& g, const DecodeCfg& cfg, uint64_t c, const uint8_t* gp, PlaneSrc (&src)[G]) {
#pragma unroll
  for (int q = 0; q < G; q++) {
    const ItemDesc d = cfg.items[(uint64_t)q * g.K + c];
    src[q].len = d.dec_len;
    src[q].fill = 0;
    if (d.kind == kRaw) {
      src[q].ptr = cfg.body + d.src_off;
    } else if (d.kind == kRle) {
      src[q].ptr = nullptr;
      src[q].fill = cfg.body[d.src_off];
    } else {
      src[q].ptr = gp + (uint64_t)q * g.pstride;
    }
  }
}

// Unit = 16 bytes of the decoded tensor (16-byte aligned) that meet row t's bytes [id * R, id * R + R).  Units per row:
// (R + 15) / 16 + 1, whatever the row's alignment, so the grid does not depend on the ids.
template <int G>
__global__ void __launch_bounds__(256, 1) k_gather_rows(GatherCfg g, uint32_t pass) {
  const uint32_t m = *g.count;
  const uint64_t first = (uint64_t)pass * g.slots;
  const DecodeCfg& cfg = *g.cfg;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t e = *(volatile uint32_t*)&cfg.ctrl->error;  // a decode error of this call's passes so far
    if (e) atomicOr(g.error, e);
  }
  if (pass > 0 && first >= m) return;
  const uint64_t R = g.row_bytes;
  const uint64_t per = (R + 15) / 16 + 1;
  const uint64_t total = g.n * per;
  const bool rot = cfg.bits_mode == 1 && G > 1;
  for (uint64_t u = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; u < total; u += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t t = u / per, k = u - t * per;
    const int64_t id = gather_id(g, t);
    const bool bad = gather_bad(g, id);
    const uint64_t s = bad ? 0 : (uint64_t)id * R;
    const uint64_t a = (s & ~15ull) + 16 * k;
    const uint64_t lo = max(a, s), hi = min(a + 16, s + R);
    if (lo >= hi) continue;
    uint8_t* dst = g.out + t * R - s;  // the output byte of decoded byte p is dst[p]
    if (bad) {
      if (pass == 0)
        for (uint64_t p = lo; p < hi; p++) dst[p] = 0;
      continue;
    }
    if (g.chunk < 4) {  // chunks shorter than a word: no rotated word (a chunk rotates chunk_len / 4 words)
      for (uint64_t p = lo; p < hi; p++) {
        const uint64_t c = p / g.chunk;
        const uint32_t e = g.pos[c] - (uint32_t)first;
        if (e >= g.slots) continue;
        PlaneSrc src[G];
        gather_srcs<G>(g, cfg, c, g.planes + e * (uint64_t)G * g.pstride, src);
        const uint32_t q = (uint32_t)(p - c * g.chunk);
        dst[p] = gather_byte<G>(src, q % G, q / G);
      }
      continue;
    }
    // a word never straddles chunks (chunk >= 4, a power of two): at most one chunk per word, usually per unit
    uint64_t c_have = ~0ull;
    uint32_t e = 0, clen = 0;
    PlaneSrc src[G];
    for (uint64_t wa = a; wa < a + 16; wa += 4) {
      if (wa + 4 <= lo || wa >= hi) continue;
      const uint64_t c = wa / g.chunk;
      if (c != c_have) {
        c_have = c;
        e = g.pos[c] - (uint32_t)first;
        if (e < g.slots) gather_srcs<G>(g, cfg, c, g.planes + e * (uint64_t)G * g.pstride, src);
        clen = c == g.K - 1 ? (uint32_t)(g.orig - c * g.chunk) : g.chunk;
      }
      if (e >= g.slots) continue;  // another pass writes this chunk's bytes
      const uint32_t q = (uint32_t)(wa - c * g.chunk);  // (a multiple of 4: byte i of the word is in plane i % G)
      uint32_t w = 0;
#pragma unroll
      for (int i = 0; i < 4; i++)
        if (q + i < clen) w |= (uint32_t)plane_byte(src[i % G], (q + i) / G) << (8 * i);
      if (rot && (q >> 2) < (clen >> 2)) w = unrot_word<G>(w);
      if (wa >= lo && wa + 4 <= hi && ((uintptr_t)(dst + wa) & 3) == 0) {
        *reinterpret_cast<uint32_t*>(dst + wa) = w;
      } else {
        for (uint64_t p = max(wa, lo); p < min(wa + 4, hi); p++) dst[p] = (uint8_t)(w >> (8 * (p - wa)));
      }
    }
  }
}

}  // namespace zb
