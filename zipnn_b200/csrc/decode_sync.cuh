// decode_sync.cuh -- intra-stream parallel Huffman decode for small and medium tensors.
//
// k_huf_decode_fused gives every huff0 bitstream ONE thread (huf_decompress.c:203-260 is a serial
// loop: symbol i+1 starts where symbol i ends), so a decode takes the same time whether the tensor has 4
// chunks or 20 000.  Huffman codes self-synchronise: a decoder started at a wrong bit position
// falls into step with the true parse after a few symbols.  This kernel uses that (Klein & Wiseman;
// Weissenberger & Schmidt for GPUs), with the reference's stream format untouched:
//
//   one CTA = one bitstream of one coded item; the stream's bits are cut into one segment per
//   thread;
//   1. every thread decodes from its segment start (a guess, except thread 0) to the segment's
//      lower bound and publishes where it stopped -- a code boundary just beyond the bound -- and
//      how many symbols it saw;
//   2. every thread takes its predecessor's stop as its start; whoever's start changed decodes
//      again; repeat until nothing changes.  Thread 0 is right from the beginning and each round
//      makes at least one more thread right, so this ends; in practice after 2 rounds, because a
//      stop is right as soon as the parse synchronised anywhere inside the segment;
//   3. a block-wide prefix sum of the symbol counts gives each thread its output offset; the
//      total must be the stream's symbol count and the last stop the stream's first bit
//      (huf_decompress.c:348-349);
//   4. every thread decodes its segment once more, now writing into the quarter plane in shared
//      memory;
//   5. the CTA merges the quarter plane with the matching bytes of the other planes (+ sign-bit
//      un-rotate) and writes elements with coalesced 128-bit stores -- or, for chunks that need
//      the general regroup (several coded groups, ragged tail), copies the quarter plane to the
//      chunk's workspace plane.
// About 2.6 decode passes instead of 1, but over 256 threads per bitstream instead of 1: a 1 MiB
// tensor is 16 CTAs of short passes instead of 16 threads that each walk a whole bitstream.  The bitstream is copied into shared
// memory once and every pass reads it there; one full 2^11-entry table per CTA (built by 256 threads, from the
// weights k_parse_tables extracted once per item), so no two-level lookup.
#pragma once
#include "decode.cuh"

namespace zb {

constexpr int kSyncThreads = 256;
constexpr uint32_t kSyncMinSegBits = 192;  // shorter segments only add overshoot work

constexpr uint32_t kSyncStreamCap = 28u * 1024u;   // bitstream bytes kept in shared memory (bf16 ~10.6 KB, fp16 ~22, fp8 ~26)
constexpr uint32_t kSyncPad = 32u;                // readable bytes below the stream's first aligned block

struct SyncShared {
  // The whole bitstream, copied once by the CTA (aligned 16-byte blocks, so the stream keeps its offset mod 16):
  // every pass of every thread reads it from here -- no per-thread ring, no cp.async, no refill latency on a
  // re-seek.  A stream longer than the buffer (possible in the format, not seen in float tensors) falls back
  // to the per-thread rings of the one-thread-per-bitstream kernels, which alias this buffer.
  __align__(64) uint8_t sbuf[kSyncPad + kSyncStreamCap + 32];
  uint32_t stop[kSyncThreads];                     // bit offset where segment m's decode stopped
  uint32_t warp_tot[kSyncThreads / 32];
  uint32_t cls_start[kHufLogMax + 2];              // index-space start of weight class w (11-bit space)
  uint32_t cls_warp[kSyncThreads / 32][16];        // symbols of weight class w in warp q (w <= kHufLogMax = 12)
  PlaneSrc src[4];
  __align__(16) uint8_t plane[kHufBlockMax / 4 + 16];  // the decoded quarter plane
};
static_assert(sizeof(((SyncShared*)0)->sbuf) >= kSyncThreads * kRingBytes, "the fallback rings alias the stream buffer");
static_assert(sizeof(((SyncShared*)0)->plane) >= 2u * 32u * kSyncThreads, "the checkpoints of the scan passes alias the plane");
// Parsed table description of one coded item (k_parse_tables -> k_huf_decode_sync), in the workspace.
struct ItemTable {
  uint8_t weights[256];
  int32_t hsize, lg, nsym, pad;
};

// Symbols of the quarter plane [i0, i0 + 4*NW) as words (4 symbols each).
template <int NW>
__device__ __forceinline__ void smem_plane_words(const uint8_t* plane, uint32_t i0, uint32_t (&out)[NW]) {
#pragma unroll
  for (int i = 0; i < NW; i++) out[i] = *reinterpret_cast<const uint32_t*>(plane + i0 + 4 * i);
}

// The CTA's full table (symbol | (-length << 8), replicated into 11 bits) lies on a 4 KiB boundary of the shared
// address space, so that the address of an entry is ONE operation: (x & 0xFFE) | table address.  The dynamic
// buffer is only 1 KiB aligned, hence the slack: [pad to 4 KiB][table 4 KiB][SyncShared].
constexpr size_t kSyncSmemBytes = sizeof(SyncShared) + 4096 + 3072;
struct SyncCarve {
  uint16_t* lut;
  uint32_t lut_s;
  SyncShared* S;
};
__device__ __forceinline__ SyncCarve sync_carve(unsigned char* raw) {
  const uint32_t base_s = (uint32_t)__cvta_generic_to_shared(raw);
  const uint32_t off = (4096u - (base_s & 4095u)) & 4095u;
  SyncCarve c;
  c.lut = reinterpret_cast<uint16_t*>(raw + off);
  c.lut_s = base_s + off;
  c.S = reinterpret_cast<SyncShared*>(raw + off + 4096);
  return c;
}

// Window over a bitstream that lies in shared memory (byte offsets from the buffer start).  Same 64-bit
// container and word-granular refill as BitWindow, without the ring.  The shift is kept one lower than
// BitWindow's (s1 = 52 - bits consumed from the top of `cont`), so that (uint32_t)(cont >> s1) carries the
// next 11 stream bits in [11:1]: masked with 0xFFE that IS the byte offset of the 16-bit table entry.  s1 is
// >= 10 at every peek (<= 31 bits are consumed after a refill, <= 42 before the second symbol of a pair).
struct SmemWindow {
  uint64_t cont;
  int32_t s1;
  uint32_t next;      // the word below the container
  uint32_t ra;        // shared address of the word the next refill reads
  uint32_t base_s;    // shared address of the buffer
  uint32_t lut_s;     // shared address of g_sync_lut (4 KiB aligned)
};
__device__ __forceinline__ void swin_seek(SmemWindow& b, uint32_t mark) {  // next unread bit = mark - 1
  const uint32_t top_byte = (mark - 1) >> 3;
  const uint32_t q = (top_byte & ~3u) - 4u;
  b.s1 = 52 - (int32_t)(8u * (q + 8u) - mark);
  b.cont = ((uint64_t)lds_u32(b.base_s + q + 4u) << 32) | lds_u32(b.base_s + q);
  b.next = lds_u32(b.base_s + q - 4u);
  b.ra = b.base_s + q - 8u;
}
__device__ __forceinline__ void swin_refill(SmemWindow& b) {
  // if (s1 <= 20) { cont = cont << 32 | next; s1 += 32; next = *ra; ra -= 4; }   (32 or more bits consumed)
  uint32_t lo = (uint32_t)b.cont, hi = (uint32_t)(b.cont >> 32);
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.le.s32 p, %0, 20;\n\t"
      "@p mov.b32 %2, %1;\n\t"
      "@p mov.b32 %1, %3;\n\t"
      "@p add.s32 %0, %0, 32;\n\t"
      "@p ld.shared.u32 %3, [%4];\n\t"
      "@p add.u32 %4, %4, -4;\n\t}"
      : "+r"(b.s1), "+r"(lo), "+r"(hi), "+r"(b.next), "+r"(b.ra));
  b.cont = ((uint64_t)hi << 32) | lo;
}
// One symbol: the table entry (symbol in byte 0, minus the code length above it, sign-extended).
__device__ __forceinline__ int32_t swin_entry(SmemWindow& b) {
  const uint32_t x = (uint32_t)(b.cont >> b.s1);
  const int32_t e = lds_s16((x & 0xFFEu) | b.lut_s);
  b.s1 += e >> 8;
  return e;
}
// Two symbols after one refill.  (The fused kernel peeks the first one BEFORE the refill, window_pair in decode.cuh;
// here the shift is one lower, s1 = -1 is possible in front of a refill, and the peek has to follow it.)
__device__ __forceinline__ void swin_pair(SmemWindow& b, int32_t& e0, int32_t& e1) {
  swin_refill(b);
  e0 = swin_entry(b);
  e1 = swin_entry(b);
}
// Decode from bit offset `from` down to the first code boundary at or below `bound`.  -> symbols seen.
// Two symbols per test: a pair may run one symbol past the boundary (into readable bytes: the stream buffer
// has kSyncPad bytes below the stream), which the exit undoes.  Every eighth code boundary is RECORDED (its
// distance to `bound`, checkpoint j after 8 (j + 1) symbols, cp[j * kSyncThreads + tid]): a later pass that starts
// somewhere else only has to decode until it stands on one of them (swin_rescan).
constexpr int kSyncCheckpoints = 32;   // per thread; segments with more than 256 symbols record only their first 256
__device__ __forceinline__ uint32_t swin_scan(SmemWindow& b, uint32_t from, uint32_t bound, uint32_t& stop, uint16_t* cp, int tid, int& ncp) {
  int32_t rem = (int32_t)(from - bound);
  uint32_t n = 0;
  ncp = 0;
  if (rem > 0) {
    swin_seek(b, from);
    int32_t rem1;
    do {
      int32_t e0, e1;
      swin_pair(b, e0, e1);
      rem1 = rem + (e0 >> 8);
      rem = rem1 + (e1 >> 8);
      n += 2;
      if ((n & 7u) == 0 && rem > 0 && n <= 8u * kSyncCheckpoints) cp[((n >> 3) - 1u) * kSyncThreads + (uint32_t)tid] = (uint16_t)rem;
    } while (rem > 0);
    if (rem1 <= 0) {  // the first symbol of the last pair already reached the boundary
      rem = rem1;
      n--;
    }
    const uint32_t full = (rem > 0 ? n : n - 1u) >> 3;   // (n - 1: a checkpoint is only written while rem > 0)
    ncp = (int)(full < (uint32_t)kSyncCheckpoints ? full : (uint32_t)kSyncCheckpoints);
  }
  stop = (uint32_t)((int32_t)bound + rem);
  return n;
}
// The same segment again from another start (`from` <= the start of the recorded pass): decoding is deterministic,
// so from the first recorded boundary it stands on, this pass would repeat the recorded one -- its stop is the
// recorded stop and its symbol count = symbols up to that boundary + what the recorded pass (n_rec symbols) had
// left after it.  Huffman codes synchronise within a few symbols, so this costs ~15 symbols instead of a segment.
// Returns the symbol count; if the boundary is reached without a match the checkpoints are dropped and
// `stop` is this pass's own.
__device__ __forceinline__ uint32_t swin_rescan(SmemWindow& b, uint32_t from, uint32_t bound, uint32_t& stop, const uint16_t* cp, int tid, int& ncp,
                                                uint32_t n_rec) {
  int32_t rem = (int32_t)(from - bound);
  uint32_t n = 0;
  if (rem > 0) {
    swin_seek(b, from);
    int j = 0;
    int32_t c = ncp ? (int32_t)cp[tid] : -1;
    for (;;) {
      swin_refill(b);
      rem += swin_entry(b) >> 8;
      n++;
      if (rem <= 0) break;
      while (c > rem) {
        j++;
        c = j < ncp ? (int32_t)cp[(uint32_t)j * kSyncThreads + (uint32_t)tid] : -1;
      }
      if (c == rem) return n + n_rec - 8u * (uint32_t)(j + 1);
    }
  }
  ncp = 0;
  stop = (uint32_t)((int32_t)bound + rem);
  return n;
}
// Symbols [off, off + n) of the quarter plane: single bytes up to the first word boundary, then four symbols
// per 32-bit store, single bytes at the end (the neighbouring threads own the other bytes of those words).
__device__ __forceinline__ void swin_emit(SmemWindow& b, uint32_t from, uint32_t n, uint8_t* plane, uint32_t off) {
  if (n == 0) return;
  swin_seek(b, from);
  uint32_t pos = off;
  const uint32_t end = off + n;
  while (pos < end && (pos & 3u)) {
    swin_refill(b);
    plane[pos++] = (uint8_t)swin_entry(b);
  }
  for (; pos + 4 <= end; pos += 4) {
    int32_t e0, e1, e2, e3;
    swin_pair(b, e0, e1);
    swin_pair(b, e2, e3);
    *reinterpret_cast<uint32_t*>(plane + pos) = __byte_perm(__byte_perm(e0, e1, 0x0040), __byte_perm(e2, e3, 0x0040), 0x5410);
  }
  while (pos < end) {
    swin_refill(b);
    plane[pos++] = (uint8_t)swin_entry(b);
  }
}
// Whole words where the thread owns all four bytes, single bytes at its two ends (ring fallback only).
struct PlaneWriter {
  uint8_t* plane;
  uint32_t off, pos, acc;
  __device__ __forceinline__ PlaneWriter(uint8_t* p, uint32_t o) : plane(p), off(o), pos(o), acc(0) {}
  __device__ __forceinline__ void put(uint32_t sym) {
    acc |= sym << ((pos & 3u) * 8u);
    pos++;
    if ((pos & 3u) == 0) {
      if (pos - 4 >= off) {
        *reinterpret_cast<uint32_t*>(plane + pos - 4) = acc;
      } else {
        for (uint32_t q = off; q < pos; q++) plane[q] = (uint8_t)(acc >> ((q & 3u) * 8u));
      }
      acc = 0;
    }
  }
  __device__ __forceinline__ void finish() {
    if (pos & 3u) {
      const uint32_t w0 = pos & ~3u;
      for (uint32_t q = (w0 > off ? w0 : off); q < pos; q++) plane[q] = (uint8_t)(acc >> ((q & 3u) * 8u));
    }
  }
};

// ---- fallback: the stream stays in global memory, each thread feeds a private ring (decode.cuh) ----
template <class LUT>
__device__ __forceinline__ uint32_t sync_decode(BitWindow& b, const LUT& lut, int32_t& rem) {
  const uint32_t x = (uint32_t)(b.cont >> b.s);
  const int32_t e = lut.get(x);
  b.s += e >> 8;
  rem += e >> 8;
  return (uint32_t)e;
}
__device__ __forceinline__ uint32_t sync_scan(BitWindow& b, const LutFull& lut, uint32_t from, uint32_t bound, uint32_t& stop) {
  int32_t rem = (int32_t)(from - bound);
  uint32_t n = 0;
  if (rem > 0) {
    window_seek(b, from);
    for (;;) {
      ring_top_up(b, 1);
      cp_async_commit();
      bool done = false;
#pragma unroll
      for (int k = 0; k < 4 && !done; k++) {
        window_refill(b);
        sync_decode(b, lut, rem);
        n++;
        if (rem <= 0) {
          done = true;
          break;
        }
        sync_decode(b, lut, rem);
        n++;
        if (rem <= 0) done = true;
      }
      cp_async_wait<1>();
      if (done) break;
    }
    cp_async_wait<0>();
  }
  stop = (uint32_t)((int32_t)bound + rem);
  return n;
}
__device__ __forceinline__ void sync_emit(BitWindow& b, const LutFull& lut, uint32_t from, uint32_t n, uint8_t* plane, uint32_t off) {
  if (n == 0) return;
  window_seek(b, from);
  int32_t dummy = 0;
  PlaneWriter w(plane, off);
  const uint32_t end = off + n;
  while (w.pos < end) {
    ring_top_up(b, 1);
    cp_async_commit();
#pragma unroll
    for (int k = 0; k < 8; k++) {
      if (w.pos < end) {
        if ((k & 1) == 0) window_refill(b);
        w.put(sync_decode(b, lut, dummy) & 0xFFu);
      }
    }
    cp_async_wait<1>();
  }
  cp_async_wait<0>();
  w.finish();
}

// ====================================================================================
// Table descriptions of all coded items, one warp per item (lane 0 runs the <= 255 serial tANS
// steps of entropy_common.c:41-215 once per ITEM; the four bitstream CTAs of the item read the result).
// ====================================================================================
constexpr int kParseWarps = 4;
constexpr uint32_t kParseHdrMax = 272;   // a table description is at most 1 + 255 bytes (huf_compress.c:140-167); + slack for the 4-byte peeks
struct ParseSmem {
  FseDec D;
  __align__(16) uint8_t hdr[kParseHdrMax];
  uint8_t weights[256];
};
// All 32 lanes call: the warp copies the item's first bytes into shared memory (the serial parser reads them a
// byte at a time), lane 0 parses, the warp writes the result out.
__device__ __forceinline__ void parse_item(const DecodeCfg& cfg, uint32_t hi, ParseSmem& P) {
  const int lane = threadIdx.x & 31;
  const uint64_t item = cfg.hlist[hi];
  const ItemDesc d = cfg.items[item];
  ItemTable& T = cfg.tables[hi];
  const uint32_t take = d.src_len < kParseHdrMax ? d.src_len : kParseHdrMax;
  for (uint32_t i = lane; i < take; i += 32) P.hdr[i] = cfg.body[d.src_off + i];
  __syncwarp();
  int nsym = 0, lg = 0, hsize = -1;
  if (lane == 0) {
    hsize = huf_read_weights(P.weights, &nsym, &lg, P.hdr, take, P.D);
    if (hsize >= 0 && lg > kDecLutLog) {
      atomicOr(&cfg.ctrl->error, kErrUnsupported);
      hsize = -1;
    } else if (hsize < 0) {
      atomicOr(&cfg.ctrl->error, kErrCorrupt);
    }
    T.hsize = hsize;
    T.lg = lg;
    T.nsym = nsym;
  }
  __syncwarp();
  reinterpret_cast<uint2*>(T.weights)[lane] = reinterpret_cast<const uint2*>(P.weights)[lane];
}
__global__ void __launch_bounds__(kParseWarps * 32) k_parse_tables(DecodeCfg cfg) {
  __shared__ ParseSmem P[kParseWarps];
  const uint32_t nh = cfg.ctrl->huf_count;
  const uint32_t w = blockIdx.x * kParseWarps + (threadIdx.x >> 5);
  if (w < nh) parse_item(cfg, w, P[threadIdx.x >> 5]);
}

// items: hlist[0 .. ctrl->huf_count) = coded items (g * K + c) of chunks in fused or general mode.
// One bitstream: work = 4 * (index into hlist) + stream.  The caller has synchronised the CTA since
// the previous call (the shared state is reused).
__device__ __forceinline__ bool off_in_slack(uint32_t lut_s, const SyncShared& S) {  // the table must end where S begins
  return lut_s + 4096u != (uint32_t)__cvta_generic_to_shared(&S);
}
template <int G>
__device__ __forceinline__ void sync_process(const DecodeCfg& cfg, uint8_t* __restrict__ out, SyncShared& S, uint16_t* lut_tab, uint32_t lut_s,
                                             uint64_t work) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint64_t K = cfg.K;
  {
    const uint64_t item = cfg.hlist[work >> 2];
    const int stream = (int)(work & 3);
    const int g = (int)(item / K);
    const uint64_t c = item - (uint64_t)g * K;
    const ItemDesc d = cfg.items[item];
    const uint32_t mode = cfg.mode[c];

    // ---- table description: parsed once per item by k_parse_tables ----
    const ItemTable& T = cfg.tables[work >> 2];
    const int hsize = T.hsize, lg = T.lg, nsym = T.nsym;
    if (hsize < 0) return;  // (uniform; the parse kernel raised the error)
    if (tid < (kSyncThreads / 32) * 16) (&S.cls_warp[0][0])[tid] = 0;
    __syncthreads();
    // ---- full table, one thread per symbol (huf_decompress.c:151-183: weights ascending, symbols
    //      ascending within a weight, 2^(w-1) consecutive entries each).  A symbol's rank inside its weight
    //      class = equal weights among the lower lanes of its warp (one match + popc) + the class counts of
    //      the warps below ----
    const int w_mine = tid < nsym ? (int)T.weights[tid] : 0;
    const uint32_t same = __match_any_sync(0xffffffffu, w_mine);
    uint32_t rank = (uint32_t)__popc(same & ((1u << lane) - 1u));
    if (w_mine && rank == 0) S.cls_warp[wid][w_mine] = (uint32_t)__popc(same);
    __syncthreads();
    if (tid == 0) {
      uint32_t at = 0;
      for (int w = 1; w <= lg; w++) {
        uint32_t cnt = 0;
#pragma unroll
        for (int q = 0; q < kSyncThreads / 32; q++) cnt += S.cls_warp[q][w];
        S.cls_start[w] = at;
        at += (cnt << (w - 1)) << (kDecLutLog - lg);
      }
    }
    for (int q = 0; q < wid; q++) rank += S.cls_warp[q][w_mine];
    __syncthreads();
    if (w_mine) {
      const int len = lg + 1 - w_mine;
      const uint32_t span = 1u << (kDecLutLog - len);
      const uint32_t u = S.cls_start[w_mine] + rank * span;
      const uint16_t e = (uint16_t)(tid | (((256 - len) & 0xFF) << 8));  // symbol | -length
      if (span >= 2) {
        const uint32_t ee = (uint32_t)e | ((uint32_t)e << 16);
        uint32_t* p = reinterpret_cast<uint32_t*>(lut_tab + u);  // u is a multiple of span, so even
        for (uint32_t q = 0; q < (span >> 1); q++) p[q] = ee;
      } else {
        lut_tab[u] = e;
      }
    }
    // ---- this CTA's bitstream (jump table, huf_decompress.c:283-290) ----
    const uint8_t* p = cfg.body + d.src_off + hsize;
    const uint32_t rest = d.src_len - (uint32_t)hsize;
    bool ok = rest >= 10;
    uint32_t l0 = 0, l1 = 0, l2 = 0, l3 = 0;
    if (ok) {
      l0 = p[0] | (p[1] << 8);
      l1 = p[2] | (p[3] << 8);
      l2 = p[4] | (p[5] << 8);
      ok = l0 + l1 + l2 + 6 <= rest;
      l3 = rest - (l0 + l1 + l2 + 6);
      ok = ok && l0 && l1 && l2 && l3;
    }
    const uint32_t seg = (d.dec_len + 3) >> 2;
    ok = ok && 3 * seg <= d.dec_len;
    uint32_t s_off = 6, s_len = l0;
    if (stream == 1) { s_off += l0; s_len = l1; }
    if (stream == 2) { s_off += l0 + l1; s_len = l2; }
    if (stream == 3) { s_off += l0 + l1 + l2; s_len = l3; }
    const uint32_t out_off = (uint32_t)stream * seg;
    const uint32_t count = ok ? ((stream == 3) ? d.dec_len - 3 * seg : seg) : 0;
    uint8_t lastb = 0;
    if (ok) {
      lastb = p[s_off + s_len - 1];
      ok = lastb != 0;
    }
    if (!ok) {
      if (tid == 0) atomicOr(&cfg.ctrl->error, kErrCorrupt);
      return;  // (uniform: every thread computed the same)
    }
    const LutFull lut{lut_tab, kDecLutLog};   // (the ring fallback goes through the generic table type)
    const uint8_t* sp = p + s_off;                       // the bitstream: s_len bytes
    const bool in_smem = s_len <= kSyncStreamCap;        // (uniform)
    uint32_t mark, first;
    SmemWindow sw;
    BitWindow b;
    if (in_smem) {
      // aligned 16-byte blocks from kSyncPad bytes below the block that holds the first byte; blocks that would
      // start in front of the body are skipped (never needed: a stream starts >= 16 bytes into the body)
      const uintptr_t blk0 = ((uintptr_t)sp & ~(uintptr_t)15) - kSyncPad;
      const uint32_t head = (uint32_t)((uintptr_t)sp - blk0);               // offset of the stream inside sbuf
      const uint32_t nblk = (head + s_len + 15u) >> 4;
      for (uint32_t i = tid; i < nblk; i += kSyncThreads) {
        const uint8_t* g = reinterpret_cast<const uint8_t*>(blk0) + 16u * i;
        if (g >= cfg.body - 15) cp_async16(S.sbuf + 16u * i, g);
      }
      cp_async_commit();
      cp_async_wait<0>();
      sw.base_s = (uint32_t)__cvta_generic_to_shared(S.sbuf);
      sw.lut_s = lut_s;
      if ((lut_s & 4095u) || off_in_slack(lut_s, S)) {  // cannot happen (sync_carve), but never decode wrongly
        if (tid == 0) atomicOr(&cfg.ctrl->error, kErrUnsupported);
        return;
      }
      first = 8u * head;
      mark = 8u * (head + s_len - 1) + (uint32_t)hb32(lastb);
    } else {
      const uint32_t so = window_frame(b, sp, cfg.body, S.sbuf + (size_t)tid * kRingBytes);
      mark = 8u * (so + s_len - 1) + (uint32_t)hb32(lastb);
      first = b.start_bit;
    }
    __syncthreads();  // table and stream complete
    // ---- segments ----
    const uint32_t bits = mark - first;
    uint32_t segbits = (bits + kSyncThreads - 1) / kSyncThreads;
    if (segbits < kSyncMinSegBits) segbits = kSyncMinSegBits;
    const uint32_t top = (uint64_t)tid * segbits < bits ? mark - (uint32_t)tid * segbits : first;          // guess (exact for tid 0)
    const uint32_t bound = (uint64_t)(tid + 1) * segbits < bits ? mark - (uint32_t)(tid + 1) * segbits : first;
    uint32_t from = top, stop = top, n = 0, n_rec = 0;
    int ncp = 0;                                                    // recorded boundaries of this thread's first pass
    uint16_t* cp = reinterpret_cast<uint16_t*>(S.plane);            // [kSyncCheckpoints][kSyncThreads]; the plane is written after the rounds
    bool need = true;
    for (int round = 0; round <= kSyncThreads; round++) {
      if (need) {
        if (!in_smem) {
          n = sync_scan(b, lut, from, bound, stop);
        } else if (ncp == 0) {
          n = n_rec = swin_scan(sw, from, bound, stop, cp, tid, ncp);
        } else {
          n = swin_rescan(sw, from, bound, stop, cp, tid, ncp, n_rec);
        }
      }
      S.stop[tid] = stop;
      __syncthreads();
      const uint32_t nf = tid ? S.stop[tid - 1] : mark;
      need = nf != from;
      from = nf;
      if (!__syncthreads_or(need)) break;
    }
    // ---- output offsets; the stream must hold exactly `count` symbols and be consumed exactly ----
    uint32_t incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) S.warp_tot[wid] = incl;
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kSyncThreads / 32; w++) {
      const uint32_t v = S.warp_tot[w];
      if (w < wid) before += v;
      total += v;
    }
    const uint32_t off = before + incl - n;
    if (total != count || S.stop[kSyncThreads - 1] != first) {
      if (tid == 0) atomicOr(&cfg.ctrl->error, kErrCorrupt);
      return;  // (uniform)
    }
    if (in_smem) swin_emit(sw, from, n, S.plane, off);
    else sync_emit(b, lut, from, n, S.plane, off);
    __syncthreads();
    // ---- quarter plane -> elements, or -> the chunk's workspace plane ----
    if (mode == kModeFused) {
      // fused chunks: the coded plane is the top byte plane, dec_len % 128 == 0, every other plane raw or RLE
      if (tid < G - 1) {
        const ItemDesc t = cfg.items[(uint64_t)tid * K + c];
        PlaneSrc s;
        s.len = t.dec_len;
        s.fill = 0;
        if (t.kind == kRle) {
          s.ptr = nullptr;
          s.fill = 0x01010101u * (uint32_t)cfg.body[t.src_off];
        } else {
          s.ptr = cfg.body + t.src_off;
        }
        S.src[tid] = s;
      }
      __syncthreads();
      uint8_t* out_q = out + c * (uint64_t)cfg.chunk + (uint64_t)out_off * G;
      const bool rot = (cfg.bits_mode == 1) && (G > 1);
      const uint32_t obytes = count * (uint32_t)G;
      for (uint32_t o = (uint32_t)tid * 16u; o < obytes; o += kSyncThreads * 16u) {
        uint32_t r[4];
        if (G == 1) {
          smem_plane_words<4>(S.plane, o, r);
        } else if (G == 2) {
          uint32_t a[2], e2[2];
          load_plane_words<2>(S.src[0], out_off + (o >> 1), a);
          smem_plane_words<2>(S.plane, o >> 1, e2);
          r[0] = __byte_perm(a[0], e2[0], 0x5140);
          r[1] = __byte_perm(a[0], e2[0], 0x7362);
          r[2] = __byte_perm(a[1], e2[1], 0x5140);
          r[3] = __byte_perm(a[1], e2[1], 0x7362);
        } else {
          uint32_t p0[1], p1[1], p2[1], p3[1];
          load_plane_words<1>(S.src[0], out_off + (o >> 2), p0);
          load_plane_words<1>(S.src[1 % 3], out_off + (o >> 2), p1);
          load_plane_words<1>(S.src[2 % 3], out_off + (o >> 2), p2);
          smem_plane_words<1>(S.plane, o >> 2, p3);
          const uint32_t t0 = __byte_perm(p0[0], p1[0], 0x5140), t1 = __byte_perm(p2[0], p3[0], 0x5140);
          const uint32_t t2 = __byte_perm(p0[0], p1[0], 0x7362), t3 = __byte_perm(p2[0], p3[0], 0x7362);
          r[0] = __byte_perm(t0, t1, 0x5410);
          r[1] = __byte_perm(t0, t1, 0x7632);
          r[2] = __byte_perm(t2, t3, 0x5410);
          r[3] = __byte_perm(t2, t3, 0x7632);
        }
        if (rot) {
#pragma unroll
          for (int i = 0; i < 4; i++) r[i] = unrot_word<G>(r[i]);
        }
        *reinterpret_cast<uint4*>(out_q + o) = make_uint4(r[0], r[1], r[2], r[3]);
      }
    } else {
      uint8_t* dst = cfg.planes + ((uint64_t)cfg.slot[c] * G + g) * cfg.pstride + out_off;
      if (((uintptr_t)dst & 3) == 0) {
        const uint32_t nw = count >> 2;
        for (uint32_t i = tid; i < nw; i += kSyncThreads) reinterpret_cast<uint32_t*>(dst)[i] = reinterpret_cast<const uint32_t*>(S.plane)[i];
        for (uint32_t i = (nw << 2) + tid; i < count; i += kSyncThreads) dst[i] = S.plane[i];
      } else {
        for (uint32_t i = tid; i < count; i += kSyncThreads) dst[i] = S.plane[i];
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kSyncThreads) k_huf_decode_sync(DecodeCfg cfg, uint8_t* __restrict__ out) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const uint32_t nh = cfg.ctrl->huf_count;
  for (uint64_t work = blockIdx.x; work < 4ull * nh; work += gridDim.x) {
    __syncthreads();  // the previous item's shared state is dead
    sync_process<G>(cfg, out, S, cv.lut, cv.lut_s, work);
  }
}

// Bitstreams of every tensor of a batch in one grid (flat index -> tensor by binary search).
__global__ void __launch_bounds__(kSyncThreads) k_huf_decode_sync_batch(BatchCfg B) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const SyncCarve cv = sync_carve(smem_raw);
  SyncShared& S = *cv.S;
  const uint64_t total = B.item_start[B.n];
  for (uint64_t w = blockIdx.x; w < total; w += gridDim.x) {
    const uint32_t t = batch_find(B.item_start, B.n, w);
    const DecodeCfg& cfg = B.cfgs[t];
    const uint64_t work = w - B.item_start[t];
    if (work >= 4ull * cfg.ctrl->huf_count) continue;  // (uniform) the bound counts every item, only the coded ones are queued
    __syncthreads();
    if (cfg.G == 1) sync_process<1>(cfg, cfg.out, S, cv.lut, cv.lut_s, work);
    else if (cfg.G == 2) sync_process<2>(cfg, cfg.out, S, cv.lut, cv.lut_s, work);
    else sync_process<4>(cfg, cfg.out, S, cv.lut, cv.lut_s, work);
  }
}

// one warp per coded item of every tensor of a batch (flat index over item_start / 4)
__global__ void __launch_bounds__(kParseWarps * 32) k_parse_tables_batch(BatchCfg B) {
  __shared__ ParseSmem P[kParseWarps];
  const uint64_t total = B.item_start[B.n] >> 2;
  const uint64_t w = (uint64_t)blockIdx.x * kParseWarps + (threadIdx.x >> 5);
  if (w >= total) return;
  const uint32_t t = batch_find(B.item_start, B.n, 4 * w);
  const DecodeCfg& cfg = B.cfgs[t];
  const uint64_t hi = w - (B.item_start[t] >> 2);
  if (hi < cfg.ctrl->huf_count) parse_item(cfg, (uint32_t)hi, P[threadIdx.x >> 5]);
}

}  // namespace zb
