// decode.cuh -- decompress side:  stream metadata -> item table, Huffman bit-unpack fused
// with byte-group regroup (+ sign-bit un-rotate).
//
// Replaces reference csrc/zipnn_core.c:881-1142 (py_combine_dtype), :768-861
// (decompression_chunk_worker), huf_decompress.c:118-354 (table + 4-stream decode),
// data_manipulation_dtype16.c:167-216 and data_manipulation_dtype32.c:391-456 (combine).
//
// Kernels
//   k_decode_meta        one thread per chunk: item table, per-chunk mode, RLE fill blocks
//   k_huf_decode_fused   chunks with exactly one Huffman-coded group (the normal case:
//                        the exponent plane) -> decoded, merged with the raw/RLE planes,
//                        un-rotated and written as elements, in one pass
//   k_huf_decode_planar  chunks with several Huffman-coded groups, or a ragged last chunk:
//                        decode each coded plane into a workspace plane ...
//   k_regroup            ... and regroup planes (raw / RLE / workspace) into elements; also
//                        handles chunks with no coded group at all
#pragma once
#include <cuda.h>
#include "common.cuh"

// L2 fetch granularity of the 16-byte cp.async copies that feed the bitstream rings and the side-plane slots.
// Every lane walks its own stream, 16 bytes at a time, so the DRAM sees hundreds of thousands of interleaved
// sequential streams; with plain sector fills each miss opens a DRAM row for 32 bytes.
#ifndef ZB_CPASYNC_L2
#define ZB_CPASYNC_L2 ".L2::128B"
#endif

#ifndef ZB_SIDE_SLOTS
#define ZB_SIDE_SLOTS 4  // 16-byte cp.async slots per lane and side plane of the fused kernel.  2 would do (block k+3 is
                         // requested two iterations before it is read) and saves 1 KiB per plane, but a cp.async into a slot
                         // that an LDS read an instant earlier is slow
#endif

namespace zb {

struct ItemTable;

enum : uint32_t { kModePlain = 0, kModeFused = 1, kModeGeneral = 2, kModeSkip = 3, kModeOverflow = 4 };
constexpr uint32_t kOverflowCtas = 32;  // persistent CTAs (each with private plane scratch) for general chunks beyond the slot pool
constexpr uint32_t kFillBytes = 64;  // replicated RLE byte block per item (read with stride 0)

struct DecodeCfg {
  const uint8_t* body;
  uint8_t* out;         // decoded tensor (used by the batch kernels; the single-tensor kernels take it as an argument)
  uint64_t body_len;
  int G;
  uint64_t K;
  uint32_t chunk;
  uint64_t orig;
  int bits_mode;
  Ctrl* ctrl;
  ItemDesc* items;      // [G*K]
  uint8_t* mode;        // [K]
  uint32_t* slot;       // [K] workspace plane slot of a general-mode chunk (G planes per slot)
  uint32_t* rlist;      // [K] chunks that k_regroup has to write (plain and general mode), ctrl->regroup_count of them
  uint8_t* fill;        // [G*K*kFillBytes]
  uint8_t* planes;      // [slots][G][pstride]
  uint64_t pstride;
  uint32_t max_slots;   // plane slots of the pool (general chunks 0 .. max_slots-1 by arrival)
  uint32_t ovf_slots;   // plane slots behind the pool, one per CTA of k_decode_overflow (0: none, an overflow is an error)
  uint32_t* olist;      // [K] chunks for k_decode_overflow, ctrl->overflow_count of them
  uint32_t* hlist;      // [G*K] coded items (g*K + c) for k_huf_decode_sync, ctrl->huf_count of them; nullptr: not used
  struct ItemTable* tables;  // [G*K] parsed table descriptions, parallel to hlist (k_parse_tables)
  uint32_t tma_flags;   // kTmaOut | kTmaSide: which tensor maps of the fused kernel's TmaMaps argument are valid
  uint32_t fused_claim; // k_huf_decode_fused: warps claim their groups from ctrl->fused_next instead of striding
  uint64_t k_full;      // chunks of full length (K, or K - 1 with a ragged last chunk)
  uint64_t side_pred[3];  // payload offset (inside body) of byte plane g's first item IF every group in front of it is all raw
  uint32_t side_r0[3];    // (body + side_pred[g]) & 15: the tensor maps start at the 16-byte boundary below
  // Window over the decoded bytes (zipnn_b200_decompress_slices; batch kernels only): row r of the box is
  // [box_base + r * box_pitch, + box_len), written packed to `out` at r * box_len.  box_len == 0: no window.
  uint64_t box_base, box_rows, box_pitch, box_len;
  uint64_t box_step_rows, box_step_cols;  // kBoxStep bytes as whole rows + columns: a thread's cursor advance per store step
  uint32_t box_fast;                      // base, pitch and len are multiples of 16: every vector is in one row or outside
  uint64_t c0;                            // first chunk the batch kernels visit (chunk_start counts from here)
};

// ---- the window's store path --------------------------------------------------------------------
// Both output write sites (regroup_tile, the fused merge of sync_process) step a thread through the decoded
// bytes kBoxStep at a time, so the row and column of its vector are computed once and then advanced.
constexpr uint32_t kBoxStep = 4096;

// Does the box meet decoded bytes [a, a + n)?  The first row whose end lies beyond a is the only candidate.
__device__ __forceinline__ bool box_meets(const DecodeCfg& cfg, uint64_t a, uint64_t n) {
  const uint64_t e0 = cfg.box_base + cfg.box_len;
  const uint64_t r = a < e0 ? 0 : (a - e0) / cfg.box_pitch + 1;
  return r < cfg.box_rows && cfg.box_base + r * cfg.box_pitch < a + n;
}
struct BoxCursor {
  int64_t row;   // row of the vector's first byte (negative in front of the box)
  uint64_t col;  // its offset from that row's start, in [0, box_pitch)
};
__device__ __forceinline__ BoxCursor box_cursor(const DecodeCfg& cfg, uint64_t v) {
  BoxCursor k;
  if (v >= cfg.box_base) {
    const uint64_t q = (v - cfg.box_base) / cfg.box_pitch;
    k.row = (int64_t)q;
    k.col = v - cfg.box_base - q * cfg.box_pitch;
  } else {
    const uint64_t d = cfg.box_base - v, q = (d + cfg.box_pitch - 1) / cfg.box_pitch;
    k.row = -(int64_t)q;
    k.col = q * cfg.box_pitch - d;
  }
  return k;
}
__device__ __forceinline__ void box_advance(const DecodeCfg& cfg, BoxCursor& k) {
  k.row += (int64_t)cfg.box_step_rows;
  k.col += cfg.box_step_cols;
  if (k.col >= cfg.box_pitch) {
    k.col -= cfg.box_pitch;
    k.row++;
  }
}
// The 16 decoded bytes at the cursor (16-byte aligned in the decoded stream) -> those of them inside the box.
// No store covers a byte outside the box: other CTAs own the rest of the output.
__device__ __forceinline__ void box_store16(const DecodeCfg& cfg, uint8_t* __restrict__ out, const BoxCursor& k, const uint32_t (&r)[4]) {
  if (cfg.box_fast) {
    if (k.row >= 0 && (uint64_t)k.row < cfg.box_rows && k.col < cfg.box_len)
      *reinterpret_cast<uint4*>(out + (uint64_t)k.row * cfg.box_len + k.col) = make_uint4(r[0], r[1], r[2], r[3]);
    return;
  }
  int64_t row = k.row;
  uint64_t col = k.col;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    if (row >= 0 && (uint64_t)row < cfg.box_rows && col < cfg.box_len) out[(uint64_t)row * cfg.box_len + col] = (uint8_t)(r[i >> 2] >> (8 * (i & 3)));
    if (++col == cfg.box_pitch) {
      col = 0;
      row++;
    }
  }
}
// One decoded byte at v (the ragged tail of a stream's last chunk).
__device__ __forceinline__ void box_put(const DecodeCfg& cfg, uint8_t* __restrict__ out, uint64_t v, uint8_t b) {
  if (v < cfg.box_base) return;
  const uint64_t q = (v - cfg.box_base) / cfg.box_pitch, col = v - cfg.box_base - q * cfg.box_pitch;
  if (q < cfg.box_rows && col < cfg.box_len) out[q * cfg.box_len + col] = b;
}


// A chunk needs plane scratch (several coded groups, a ragged tail, or a table the fused kernel could not hold).
// The first max_slots of them get a slot in the pool and are decoded by k_huf_decode_planar + k_regroup with
// the whole GPU; the rest are queued for k_decode_overflow, which works through them with a few persistent
// CTAs that own their scratch -- slower, but every chunk is written in stream order whatever the stream looks
// like (an fp32 checkpoint upcast from bf16 has two coded groups in EVERY chunk).
__device__ __forceinline__ uint32_t assign_general(const DecodeCfg& cfg, uint64_t c) {
  const uint32_t s = atomicAdd(&cfg.ctrl->work_counter, 1u);
  if (s < cfg.max_slots) {
    cfg.slot[c] = s;
    cfg.rlist[atomicAdd(&cfg.ctrl->regroup_count, 1u)] = (uint32_t)c;
    return kModeGeneral;
  }
  if (cfg.ovf_slots) {
    cfg.olist[atomicAdd(&cfg.ctrl->overflow_count, 1u)] = (uint32_t)c;
    return kModeOverflow;
  }
  atomicOr(&cfg.ctrl->error, kErrWorkspace);
  return kModeSkip;
}

// ====================================================================================
// Kernel 1: parse + validate the per-(group,chunk) metadata.
// Stream body layout (csrc/zipnn_core.c:105-244):
//   types u8[G][K] | cum u64le[G][K] (inclusive, per group) | group-major payload
// ====================================================================================
// Chunks c = first, first + stride, ... of one tensor.  W: the tensor may carry a box; chunks outside it are
// skipped before any of their table entries is read.
template <bool W = false>
__device__ __forceinline__ void decode_meta_body(const DecodeCfg& cfg, uint64_t first, uint64_t stride, bool leader) {
  const int G = cfg.G;
  const uint64_t K = cfg.K;
  const uint64_t nitems = (uint64_t)G * K;
  const uint8_t* types = cfg.body;
  const uint8_t* cum = cfg.body + nitems;
  const uint64_t payload0 = 9 * nitems;
  const uint64_t payload_len = cfg.body_len - payload0;
  // Group bases: every addition is checked against what is left of the payload, so a crafted size
  // table cannot wrap a u64 and point an item in front of the body.  With an impossible total
  // nothing of the stream is trusted: every chunk is skipped.
  uint64_t base[4] = {0, 0, 0, 0};
  bool totals_ok = true;
  {
    uint64_t room = payload_len;
    for (int g = 0; g < G; g++) {
      const uint64_t tot = ld_u64_bytes(cum + 8 * ((uint64_t)g * K + (K - 1)));
      if (tot > room) {
        totals_ok = false;
        break;
      }
      room -= tot;
      if (g + 1 < G) base[g + 1] = base[g] + tot;
    }
  }
  if (leader) {
    for (int g = 0; g < 4; g++) cfg.ctrl->base[g] = payload0 + base[g];
    if (!totals_ok) atomicOr(&cfg.ctrl->error, kErrCorrupt);
  }
  for (uint64_t c = first; c < K; c += stride) {
    const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(cfg.orig - c * (uint64_t)cfg.chunk) : cfg.chunk;
    if (W && cfg.box_len && !box_meets(cfg, c * (uint64_t)cfg.chunk, chunk_len)) {
      cfg.mode[c] = (uint8_t)kModeSkip;
      continue;
    }
    int nhuf = 0, last_huf = -1;
    bool bad_chunk = !totals_ok;
    for (int g = 0; g < G; g++) {
      const uint64_t i = (uint64_t)g * K + c;
      const uint64_t hi = ld_u64_bytes(cum + 8 * i);
      const uint64_t lo = c ? ld_u64_bytes(cum + 8 * (i - 1)) : 0;
      const uint32_t dlen = plane_len(chunk_len, G, g);
      const uint8_t type = types[i];
      ItemDesc d;
      d.src_off = payload0 + base[g] + lo;
      d.dec_len = dlen;
      d.pad = 0;
      // hi <= this group's total <= payload_len - base[g] (checked above when totals_ok): no sum can wrap
      bool bad = !totals_ok || (hi < lo) || (hi > payload_len - base[g]) || (type > 1) || (hi - lo > 0xFFFFFFFFull);
      const uint32_t slen = (uint32_t)(hi - lo);
      d.src_len = slen;
      if (type == 0) {
        d.kind = kRaw;
        bad = bad || (slen != dlen);
      } else {
        // HUF_decompress (huf_decompress.c:1056-1081): csize > dst -> error; == -> copy; 1 -> RLE
        if (dlen == 0) {
          d.kind = kRaw;
          d.src_len = 0;
        } else if (slen > dlen || slen == 0) {
          bad = true;
          d.kind = kRaw;
        } else if (slen == dlen) {
          d.kind = kRaw;
        } else if (slen == 1) {
          d.kind = kRle;
        } else {
          d.kind = kHuf;
          bad = bad || (dlen > (uint32_t)kHufBlockMax);
        }
      }
      if (bad) {
        atomicOr(&cfg.ctrl->error, kErrCorrupt);
        d.kind = kRaw;
        d.src_len = 0;
        d.dec_len = 0;
        bad_chunk = true;
      }
      if (d.kind == kHuf) {
        nhuf++;
        last_huf = g;
      }
      if (d.kind == kRle) {
        const uint32_t v = 0x01010101u * (uint32_t)cfg.body[d.src_off];
        uint4* f = reinterpret_cast<uint4*>(cfg.fill + i * kFillBytes);
#pragma unroll
        for (int q = 0; q < (int)(kFillBytes / 16); q++) f[q] = make_uint4(v, v, v, v);
      }
      cfg.items[i] = d;
    }
    // The fused kernel wants the one coded plane to be the top byte plane (the exponent side: what
    // float tensors produce), and whole, equally long planes whose quarter streams are a whole
    // number of 128-byte output rows: chunk_len a multiple of 512.  Anything else goes the general way.
    uint32_t m = kModePlain;
    if (bad_chunk) {
      m = kModeSkip;  // rejected: nothing may be read through its (untrusted) offsets
    } else if (nhuf == 1 && last_huf == G - 1 && (chunk_len % 512u) == 0) {
      m = kModeFused;
    } else if (nhuf >= 1) {
      m = assign_general(cfg, c);
    }
    cfg.mode[c] = (uint8_t)m;
    if (m == kModePlain) cfg.rlist[atomicAdd(&cfg.ctrl->regroup_count, 1u)] = (uint32_t)c;
    if (cfg.hlist && (m == kModeFused || m == kModeGeneral)) {  // small tensors: one CTA per bitstream (decode_sync.cuh)
      for (int g = 0; g < G; g++) {
        const uint64_t i = (uint64_t)g * K + c;
        if (cfg.items[i].kind == kHuf) cfg.hlist[atomicAdd(&cfg.ctrl->huf_count, 1u)] = (uint32_t)i;
      }
    }
  }
}

__global__ void k_decode_meta(DecodeCfg cfg) {
  decode_meta_body(cfg, blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, (uint64_t)gridDim.x * blockDim.x, blockIdx.x == 0 && threadIdx.x == 0);
}

// ---- batches of tensors (the load path: one launch per kernel for all tensors of a checkpoint shard) ----
// cfgs[t] describes tensor t (its own workspace slice, body and output); work_start[t] is the exclusive
// prefix sum of a per-tensor work bound, work_start[n] the total.  A flat work index finds its tensor by
// binary search, so tensors of any size mix share the grid evenly.
struct BatchCfg {
  const DecodeCfg* cfgs;
  const uint64_t* chunk_start;   // [n + 1] prefix of K
  const uint64_t* item_start;    // [n + 1] prefix of 4 * G * K (bitstreams)
  const uint64_t* tile_start;    // [n + 1] prefix of K * tiles_per_chunk (regroup tiles)
  uint32_t n;
  uint32_t* error_out;           // OR of every tensor's error word (first word of the batch workspace)
};
__global__ void k_decode_meta_batch(BatchCfg B) {
  const uint64_t total = B.chunk_start[B.n];
  for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t t = batch_find(B.chunk_start, B.n, w);
    const uint64_t local = w - B.chunk_start[t];
    decode_meta_body<true>(B.cfgs[t], B.cfgs[t].c0 + local, ~0ull >> 1, local == 0);  // exactly one chunk
  }
}
__global__ void k_batch_errors(BatchCfg B) {
  uint32_t e = 0;
  for (uint32_t t = threadIdx.x; t < B.n; t += blockDim.x) e |= B.cfgs[t].ctrl->error;
  if (e) atomicOr(B.error_out, e);
}

// ====================================================================================
// Shared pieces of the two Huffman kernels.
//
// One thread per bitstream (a huff0 block is 4 independent backward bitstreams,
// huf_decompress.c:283-298); one warp = 8 blocks.  Each block's single-symbol decode
// table (2^tableLog x {symbol, length}) lives in shared memory.
//
// Stream bytes reach the thread through a private 128-byte ring in shared memory that is
// filled with cp.async (16-byte, L2-only) two iterations ahead of use.  Registers never
// wait on a global load: a per-lane "prefetch into a register" does not work on a GPU,
// because lanes refill at different symbols while the scoreboard is per warp, so every
// refill ends up waiting for some other lane's load.
// The refill itself is branch-free: every second symbol all lanes execute the same
// select/shift/LDS sequence, whether or not their window needed a word.
// ====================================================================================
constexpr int kDecItemsPerWarp = 8;
constexpr int kDecLutLog = 11;  // the reference encoder never exceeds 11 (HUF_TABLELOG_DEFAULT)
constexpr int kDecLutEntries = 1 << kDecLutLog;
constexpr uint32_t kRingBytes = 64;

struct DecodeSmem {
  uint16_t lut[kDecItemsPerWarp][kDecLutEntries];  // also scratch for the table parse
  __align__(64) uint8_t ring[32][kRingBytes];      // per lane; weights[8][256] alias it during the parse
};
static_assert(sizeof(FseDec) <= sizeof(uint16_t) * kDecLutEntries, "FseDec must fit in one LUT slot");
static_assert(32 * kRingBytes >= kDecItemsPerWarp * 256, "weights alias the ring");

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global" ZB_CPASYNC_L2 " [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16_s(uint32_t saddr, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global" ZB_CPASYNC_L2 " [%0], [%1], 16;\n" ::"r"(saddr), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// Bit window: a 64-bit container `cont` holding bytes [q, q+8) of the stream (q 4-aligned in the
// ring's offset space) and a count `c` of bits already consumed from its top, as in
// bitstream.h:272-443, but refilled one aligned 32-bit word at a time: when 32 or more bits are
// gone, cont = cont << 32 | next, where `next` (the word below q) was read from the ring at the
// PREVIOUS refill.  A symbol costs peek = cont >> (53 - c) and c += length; the refill check runs
// every 2 symbols (31 + 2 x 11 <= 64 - 11).  The shared-memory read is off the dependent chain
// (its result is needed one refill later) and happens once per 32 stream bits instead of three
// times per 4 symbols.
struct BitWindow {
  uint64_t cont;         // bytes [q, q+8) of the stream, little endian
  int32_t s;             // 53 - (bits consumed from the top of `cont`): (uint32_t)(cont >> s) has the next 11 bits in [10:0]
  uint32_t qm;           // q - 8: byte offset (from gbase) of the word the NEXT refill reads; moves down by 4.  The ring
                         // address of that word is ring_s | (qm & 60): one LOP3, so no second pointer has to be kept
  uint32_t next;         // the word at q - 4
  uint32_t ring_s;       // shared-space address of the ring (64-byte aligned)
  uint32_t fetch48;      // 48 + byte offset (from gbase) of the lowest 16-byte block already requested: biased so that
                         // "the next block's ring slot is free" is the single compare fetch48 > qm (ring_top_up)
  uint32_t start_bit;    // bit offset (from gbase) of the first stream bit (exact-consumption check)
  const uint8_t* gsrc;   // (the 64-byte aligned global address the offsets are relative to) - 64: block source = gsrc + fetch48
  uint32_t floor64;      // 64 + the offset below which no block may be requested (start of the stream buffer)
  const uint8_t* ring;
};

__device__ __forceinline__ uint32_t ring_word(const uint8_t* ring, uint32_t off) {
  return *reinterpret_cast<const uint32_t*>(ring + (off & (kRingBytes - 4)));
}

// Request every 16-byte block that fits in the ring below what is still needed (<= `maxn`).
__device__ __forceinline__ void ring_top_up(BitWindow& b, int maxn) {
#pragma unroll 2
  for (int i = 0; i < maxn; i++) {
    // The next block is [f, f + 16) with f = fetch - 16 = fetch48 - 64.  It replaces ring bytes [f + 64, f + 80): free
    // once they lie at or above qm + 4 (the container and `next` hold everything from there up; later reads are at
    // qm and below), i.e. f + 60 >= qm, i.e. fetch48 > qm (both are multiples of 4).
    if (b.fetch48 >= b.floor64 && b.fetch48 > b.qm) {
      uint64_t src;  // gsrc + fetch48 as ONE instruction (IMAD.WIDE.U32) instead of an add with carry
      asm("mad.wide.u32 %0, %1, 1, %2;" : "=l"(src) : "r"(b.fetch48), "l"((uint64_t)(uintptr_t)b.gsrc));
      cp_async16_s(b.ring_s | (b.fetch48 & (kRingBytes - 16)), reinterpret_cast<const void*>((uintptr_t)src));  // (f & 48) == (fetch48 & 48)
      b.fetch48 -= 16;
    }
  }
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) {
  uint32_t v;
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void window_refill(BitWindow& b) {
  // if (s <= 21) { cont = cont << 32 | next; s += 32; next = ring[qm & 60]; qm -= 4; }  -- 32 or more bits consumed.
  // Written out as predicated PTX: the C++ form loads into a temporary and moves it (one more instruction per
  // refill), and the kernel's time follows the number of instructions issued per symbol (DESIGN.md 3.1).
  uint32_t lo = (uint32_t)b.cont, hi = (uint32_t)(b.cont >> 32);
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 a;\n\t"
      "setp.le.s32 p, %0, 21;\n\t"
      "lop3.b32 a, %4, %6, %5, 0xEA;\n\t"  // (qm & (ring - 4)) | ring_s
      "@p mov.b32 %2, %1;\n\t"
      "@p mov.b32 %1, %3;\n\t"
      "@p add.s32 %0, %0, 32;\n\t"
      "@p ld.shared.u32 %3, [a];\n\t"
      "@p add.u32 %4, %4, -4;\n\t}"
      : "+r"(b.s), "+r"(lo), "+r"(hi), "+r"(b.next), "+r"(b.qm)
      : "r"(b.ring_s), "n"(kRingBytes - 4));
  b.cont = ((uint64_t)hi << 32) | lo;
}

// Frame of reference of a stream at `s`: offsets are taken from a 64-byte aligned address one ring
// below the stream start, so every offset the decoder forms is non-negative.  `lo` is the first
// readable byte of the buffer.  Returns the stream's byte offset in that frame.
__device__ __forceinline__ uint32_t window_frame(BitWindow& b, const uint8_t* s, const uint8_t* lo, uint8_t* ring) {
  b.ring = ring;
  b.ring_s = (uint32_t)__cvta_generic_to_shared(ring);
  const uint8_t* gbase = reinterpret_cast<const uint8_t*>(((uintptr_t)s & ~(uintptr_t)(kRingBytes - 1)) - kRingBytes);
  b.gsrc = gbase - 64;
  b.floor64 = 64u + ((gbase < lo) ? (uint32_t)(((uintptr_t)lo - (uintptr_t)gbase + 15) & ~(uintptr_t)15) : 0u);
  const uint32_t s_off = (uint32_t)((uintptr_t)s - (uintptr_t)gbase);
  b.start_bit = 8u * s_off;
  return s_off;
}
// Position the window so that the next unread bit is the one below bit offset `mark` (> start_bit).
__device__ __forceinline__ void window_seek(BitWindow& b, uint32_t mark) {
  const uint32_t top_byte = (mark - 1) >> 3;
  const uint32_t q = (top_byte & ~3u) - 4u;
  b.qm = q - 8u;
  b.s = 53 - (int32_t)(8u * (q + 8u) - mark);  // 1..32 bits lie above the first unread bit
  b.fetch48 = (top_byte & ~15u) + 16 + 48;
  ring_top_up(b, (int)(kRingBytes / 16));
  cp_async_commit();
  cp_async_wait<0>();
  b.cont = ((uint64_t)ring_word(b.ring, q + 4u) << 32) | ring_word(b.ring, q);
  b.next = ring_word(b.ring, q - 4u);
}
// Bit offset of the lowest consumed bit (== start_bit when the stream has been consumed exactly).
__device__ __forceinline__ uint32_t window_tell(const BitWindow& b) { return 8u * (b.qm + 16u) - (uint32_t)(53 - b.s); }

// s points at the stream (len bytes); `lo` is the first readable byte of the buffer.
__device__ __forceinline__ bool window_init(BitWindow& b, const uint8_t* s, uint32_t len, const uint8_t* lo, uint8_t* ring) {
  const uint8_t lastb = s[len - 1];
  if (lastb == 0) return false;
  const uint32_t s_off = window_frame(b, s, lo, ring);
  const uint32_t mark = 8u * (s_off + len - 1) + (uint32_t)hb32(lastb);  // bit offset of the end mark
  if (mark == b.start_bit) return false;
  window_seek(b, mark);
  return true;
}

__device__ __forceinline__ bool window_exact(const BitWindow& b) {
  return window_tell(b) == b.start_bit;  // every bit down to the stream start consumed, none below
}

// ---- decode tables ------------------------------------------------------------------
// Full table: 2^lg entries {symbol, length} (what huf_decompress.c:151-183 builds).
struct LutFull {
  const uint16_t* lut;
  int lg;
  __device__ __forceinline__ int32_t get(uint32_t x) const {
    return (int32_t)reinterpret_cast<const int16_t*>(lut)[(x & 0x7FFu) >> (11 - lg)];
  }
};
// Two-level table in an 11-bit index space (shorter table logs are replicated into it):
// codes of <= 8 bits resolve in a 256-entry primary indexed by the top 8 bits; longer codes
// sit at the bottom of the canonical order (index < x_long) and resolve in a tail table
// indexed by all 11 bits (read only by the lanes that need it); the tail serves every index below
// x_cut = the power of two at or above x_long, so that the test is one instruction (LutCol::get).
// 1 KiB per block instead of 4 KiB: three times as many bitstreams resident per SM.
__device__ __forceinline__ int32_t lds_s16(uint32_t saddr) {
  int32_t v;  // sign-extended: byte 1 of an entry is minus the code length
  asm("ld.shared.s16 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
struct LutTwo {
  uint32_t prim_s;  // shared-space byte address of the 256-entry primary
  uint32_t tail_s;  // ... of the x_cut-entry tail (32-bit shared addresses: a generic pointer makes
                    // the compiler rebuild the shared window base for every lookup)
  uint32_t hi_mask;  // 0x7FF & ~(x_cut - 1): the tail serves every index below x_cut (see LutCol::get)
  __device__ __forceinline__ int32_t get(uint32_t x) const {
    // (idx & hi_mask) == 0 ? tail_s + 2 * idx : ((x >> 2) & 0x1FE) | prim_s -- one load, address selected, the test
    // one LOP3 with a predicate result (see LutCol for why this is PTX); every primary is 512-byte aligned
    int32_t v;
    asm("{\n\t.reg .pred p;\n\t.reg .b32 i, a, t;\n\t"
        "and.b32 t, %1, %4;\n\t"
        "setp.eq.u32 p, t, 0;\n\t"
        "and.b32 i, %1, 0x7FF;\n\t"
        "shr.u32 a, %1, 2;\n\t"
        "lop3.b32 a, a, 0x1FE, %2, 0xEA;\n\t"
        "@p mad.lo.u32 a, i, 2, %3;\n\t"
        "ld.shared.s16 %0, [a];\n\t}"
        : "=r"(v)
        : "r"(x), "r"(prim_s), "r"(tail_s), "r"(hi_mask));
    return v;
  }
};

// Private-column table for planes with short codes (the exponent plane of bf16 / fp32: 98 % of the
// symbols have codes of <= 5 bits).  The shared 256-entry primary above is read at random words by
// 32 lanes: ~3.5 bank conflicts per lookup, and the LSU pipe becomes the limit of the whole kernel.
// Here every lane owns a column of a [32][32] u16 array indexed by the top 5 window bits (two lanes
// share a 4-byte bank word, which is not a conflict), 2 KiB per warp.  The array is 2 KiB ALIGNED in
// the shared address space, so that (x & 0x7C0) | column address is the entry's address in ONE LOP3:
// row stride 64 bytes = bit 6, the 5 index bits are x[10:6].  Codes longer than 5 bits resolve in
// the shared tail (index < x_long), which few lanes touch.
template <int PB>
struct LutCol {
  static_assert(PB == 5, "the one-instruction address needs 2^(11-PB) = 64 bytes = one row of 32 u16");
  uint32_t col_s;   // shared-space address of this lane's entry 0 (2 KiB aligned array + 2 * lane)
  uint32_t tail_s;
  uint32_t hi_mask; // index bits that are all zero exactly for the indices the tail serves: 0x7FF & ~(x_cut - 1)
  __device__ __forceinline__ int32_t get(uint32_t x) const {
    // ONE load per symbol: the address is SELECTED between the lane's column and the chunk's tail,
    //   (idx & hi_mask) == 0 ? tail_s + 2 * idx : (x & 0x7C0) | col_s.
    // The tail serves every index below x_cut = the power of two at or above the canonical bound x_long of the
    // codes longer than 5 bits (fill_lut_col copies the few short codes below x_cut into it as well), so that the
    // test is ONE operation on the peeked word (`LOP3` with a predicate result) instead of mask + compare: the
    // test sits on the symbol-to-symbol dependent chain (peek -> test -> select -> load -> advance), which is what
    // the kernel's time follows.  Written as PTX because the compiler turns the C++ form into five instructions.
    int32_t v;
    asm("{\n\t.reg .pred p;\n\t.reg .b32 i, a, t;\n\t"
        "and.b32 t, %1, %4;\n\t"
        "setp.eq.u32 p, t, 0;\n\t"
        "and.b32 i, %1, 0x7FF;\n\t"
        "lop3.b32 a, %1, 0x7C0, %2, 0xEA;\n\t"
        "@p mad.lo.u32 a, i, 2, %3;\n\t"
        "ld.shared.s16 %0, [a];\n\t}"
        : "=r"(v)
        : "r"(x), "r"(col_s), "r"(tail_s), "r"(hi_mask));
    return v;
  }
};

// What a table entry of the fused kernel stores for symbol n.  When the top plane is the exponent plane of a
// rotated type the symbol is stored rotated right by one bit: the un-rotation of an element,
// hi' = sign | exp >> 1, lo' = exp << 7 | mant7, then needs no shift at all -- with E = ror8(exp) it is two
// bit selects per four elements, hi' = (E & 0x7F) | (sm & 0x80), lo' = (E & 0x80) | (sm & 0x7F).
__device__ __forceinline__ uint32_t lut_symbol(uint32_t n, bool pre_rot) { return pre_rot ? ((n >> 1) | ((n & 1u) << 7)) : n; }

// Tail size for a PB-bit primary (or -1): x_cut, the power of two (>= 64) at or above the index bound x_long of the
// codes longer than PB bits.  Typical exponent planes: x_long = 64 or 128.  Run by ONE lane per chunk; it leaves what
// the chunk's four lanes need to fill their columns in `cls` (shared memory, 16 entries): cls[w] = index-space start
// of weight class w (1 <= w <= lg), cls[0] = the first symbol with a non-zero weight -- float exponent planes use a
// contiguous band of ~35 of their ~130 symbol values, so the fill starts there instead of walking 95 zeros (the
// per-group setup was 5.5 % of the kernel's samples).
__device__ __forceinline__ int lut_tail_size(const uint8_t* weights, int nsym, int lg, int pb, uint16_t* cls) {
  if (lg > kDecLutLog) return -1;
  int n0 = 0;
  while (n0 + 4 <= nsym && *reinterpret_cast<const uint32_t*>(weights + n0) == 0) n0 += 4;  // (weights: 256-byte aligned)
  uint32_t cnt[kHufLogMax + 2];
#pragma unroll
  for (int i = 0; i < kHufLogMax + 2; i++) cnt[i] = 0;
  for (int n = n0; n < nsym; n++) cnt[weights[n]]++;
  uint32_t at = 0, x_long = 0;
  cls[0] = (uint16_t)n0;
  for (int w = 1; w <= lg; w++) {
    cls[w] = (uint16_t)at;
    at += (cnt[w] << (w - 1)) << (kDecLutLog - lg);
    if (lg + 1 - w > pb) x_long = at;
  }
  uint32_t x_cut = 64;
  while (x_cut < x_long) x_cut <<= 1;
  return (int)x_cut;
}

// Fill one lane's column (all 4 lanes of a chunk run it) and, when `with_tail`, the chunk's tail.
template <int PB>
__device__ __forceinline__ void fill_lut_col(uint16_t* col /* entry k at col[32 * k] */, uint16_t* tail, bool with_tail,
                                             const uint8_t* weights, int nsym, int lg, bool pre_rot, uint32_t x_cut, const uint16_t* cls) {
  uint32_t start[kHufLogMax + 2];
#pragma unroll
  for (int w = 0; w < kHufLogMax + 2; w++) start[w] = (w >= 1 && w <= lg) ? cls[w] : 0u;
  for (int n = cls[0]; n < nsym; n++) {
    const int w = weights[n];
    if (w == 0) continue;
    const int len = lg + 1 - w;
    const uint32_t span = 1u << (kDecLutLog - len);
    const uint32_t e = lut_symbol((uint32_t)n, pre_rot) | (((256u - (uint32_t)len) & 0xFFu) << 8);  // symbol | -length
    const uint32_t u = start[w];
    start[w] = u + span;
    if (len > PB) {
      if (with_tail)
        for (uint32_t q = 0; q < span; q++) tail[u + q] = (uint16_t)e;
    } else {
      const uint32_t p0 = u >> (kDecLutLog - PB), pn = span >> (kDecLutLog - PB);
      for (uint32_t q = 0; q < pn; q++) col[32 * (p0 + q)] = (uint16_t)e;
      if (with_tail && u < x_cut) {  // the tail serves every index below x_cut (LutCol::get)
        const uint32_t end = u + span < x_cut ? u + span : x_cut;
        for (uint32_t q = u; q < end; q++) tail[q] = (uint16_t)e;
      }
    }
  }
}

// Table entries are 16 bits: symbol in byte 0, MINUS the code length in byte 1 (two's complement), read
// with a sign-extending load.  With s = 53 - consumed the dependent chain per symbol is
//   SHF.R.U64 (cont >> s)  ->  LOP3 (table address)  ->  LDS.S16  ->  LEA.HI.SX32 (s += e >> 8)
// three ALU operations and the load; the straightforward (cont << c) >> 32, index, address, c += len
// takes four.
template <class LUT>
__device__ __forceinline__ uint32_t window_decode(BitWindow& b, const LUT& lut) {
  const uint32_t x = (uint32_t)(b.cont >> b.s);  // next 11 stream bits in [10:0], later bits below... above them: older bits
  const int32_t e = lut.get(x);
  b.s += e >> 8;  // s -= length
  return (uint32_t)e;  // symbol in byte 0
}

// Two symbols around one refill.  The first peek is taken BEFORE the refill: s >= 0 there (<= 31 bits are consumed
// after a refill and <= 22 by the pair since), and a refill only re-bases `cont` and `s` -- the peeked bits are the
// same -- so the compare / select / add of the refill leave the symbol-to-symbol dependent chain (advance -> peek ->
// index -> compare -> select -> load -> advance), which is what the kernel's time follows (DESIGN.md 3.1), and run in
// the shadow of the first table load instead.
template <class LUT>
__device__ __forceinline__ void window_pair(BitWindow& b, const LUT& lut, uint32_t& e0, uint32_t& e1) {
  const uint32_t x0 = (uint32_t)(b.cont >> b.s);
  window_refill(b);
  const int32_t a = lut.get(x0);
  b.s += a >> 8;
  e0 = (uint32_t)a;
  e1 = window_decode(b, lut);
}

// 16 symbols -> 4 words (symbol j in byte j).  Ring maintenance for the NEXT iterations is
// issued first so the copies overlap the decode.
template <class LUT>
__device__ __forceinline__ void decode16(BitWindow& b, const LUT& lut, uint32_t (&o)[4]) {
  // The ring is 64 bytes and one block is requested per 8 symbols (one "half").  With span = requested bytes not
  // yet read (qm + 4 - fetch, a multiple of 4) a block is requested when span <= 48; a half moves qm by <= 12 bytes
  // (88 bits + a leftover of < 32 = three refills), so after every request span >= 56 (no request: >= 52), and the
  // block just requested, the lowest 16 bytes of the span, is first read when span < 20: more than 36 bytes = more
  // than THREE halves later.  It therefore only has to have landed at the end of the half after next:
  // cp.async.wait_group 2 -- a lead of ~3000 cycles, which covers a block that comes from DRAM (with wait_group 1
  // 7 % of the kernel's samples sat behind this wait).  Side-plane slots (cp.async path) ride the same groups: the
  // block requested at the top of iteration k is read at the end of iteration k + 1, four halves later.
#pragma unroll
  for (int h = 0; h < 2; h++) {
    ring_top_up(b, 1);
    cp_async_commit();
#pragma unroll
    for (int q = 2 * h; q < 2 * h + 2; q++) {
      uint32_t e0, e1, e2, e3;
      window_pair(b, lut, e0, e1);
      window_pair(b, lut, e2, e3);
      o[q] = __byte_perm(__byte_perm(e0, e1, 0x0040), __byte_perm(e2, e3, 0x0040), 0x5410);
    }
    cp_async_wait<2>();  // everything but the two newest groups has landed
  }
}

template <class LUT>
__device__ __forceinline__ uint32_t decode1(BitWindow& b, const LUT& lut) {
  ring_top_up(b, 1);
  cp_async_commit();
  window_refill(b);
  const uint32_t s = window_decode(b, lut) & 0xFFu;
  cp_async_wait<0>();
  return s;
}

// Serial single-symbol table fill, one lane per item (huf_decompress.c:151-183): weights
// ascending, symbols ascending within a weight, 2^(w-1) consecutive entries each.
__device__ __forceinline__ void fill_lut(uint16_t* lut, const uint8_t* weights, int nsym, int lg) {
  uint32_t cnt[kHufLogMax + 2];
#pragma unroll
  for (int i = 0; i < kHufLogMax + 2; i++) cnt[i] = 0;
  for (int n = 0; n < nsym; n++) cnt[weights[n]]++;
  uint32_t start[kHufLogMax + 2];
  uint32_t at = 0;
  start[0] = 0;
  for (int w = 1; w <= lg; w++) {
    start[w] = at;
    at += cnt[w] << (w - 1);
  }
  for (int n = 0; n < nsym; n++) {
    const int w = weights[n];
    if (w == 0) continue;
    const uint32_t len = 1u << (w - 1);
    const uint16_t e = (uint16_t)(n | (((256 - (lg + 1 - w)) & 0xFF) << 8));  // symbol | -length
    uint32_t u = start[w];
    start[w] = u + len;
    if (len >= 4 && (u & 1) == 0) {
      const uint32_t ee = (uint32_t)e | ((uint32_t)e << 16);
      uint32_t* p = reinterpret_cast<uint32_t*>(lut + u);
      for (uint32_t q = 0; q < (len >> 1); q++) p[q] = ee;
    } else {
      for (uint32_t q = 0; q < len; q++) lut[u + q] = e;
    }
  }
}

// Two-level table, step 1: the tail size in the 11-bit index space = x_cut, the power of two (>= 8) at or above the
// index bound x_long of the codes longer than 8 bits (fp16 / fp8 planes: x_long ~ 80 .. 160), or -1 when the table log
// exceeds 11 (the caller demotes the chunk).
__device__ __forceinline__ int lut2_tail_size(const uint8_t* weights, int nsym, int lg) {
  if (lg > kDecLutLog) return -1;
  uint32_t cnt[kHufLogMax + 2];
#pragma unroll
  for (int i = 0; i < kHufLogMax + 2; i++) cnt[i] = 0;
  for (int n = 0; n < nsym; n++) cnt[weights[n]]++;
  uint32_t at = 0, x_long = 0;
  for (int w = 1; w <= lg; w++) {
    at += (cnt[w] << (w - 1)) << (kDecLutLog - lg);
    if (lg + 1 - w > 8) x_long = at;
  }
  uint32_t x_cut = 8;
  while (x_cut < x_long) x_cut <<= 1;
  return (int)x_cut;
}

// Step 2: fill the 256-entry primary and the x_cut-entry tail (the codes longer than 8 bits and whatever of the shorter
// ones lies below x_cut).
__device__ __forceinline__ void fill_lut2(uint16_t* prim, uint16_t* tail, const uint8_t* weights, int nsym, int lg, bool pre_rot, uint32_t x_cut) {
  uint32_t cnt[kHufLogMax + 2];
#pragma unroll
  for (int i = 0; i < kHufLogMax + 2; i++) cnt[i] = 0;
  for (int n = 0; n < nsym; n++) cnt[weights[n]]++;
  const int up = kDecLutLog - lg;  // replicate into the 11-bit index space
  uint32_t start[kHufLogMax + 2];
  uint32_t at = 0;
  start[0] = 0;
  for (int w = 1; w <= lg; w++) {
    start[w] = at;
    at += (cnt[w] << (w - 1)) << up;
  }
  for (int n = 0; n < nsym; n++) {
    const int w = weights[n];
    if (w == 0) continue;
    const int len = lg + 1 - w;
    const uint32_t span = 1u << (kDecLutLog - len);
    const uint16_t e = (uint16_t)(lut_symbol((uint32_t)n, pre_rot) | (uint32_t)(((256 - len) & 0xFF) << 8));  // symbol | -length
    const uint32_t u = start[w];
    start[w] = u + span;
    if (len > 8) {
      for (uint32_t q = 0; q < span; q++) tail[u + q] = e;
    } else {
      const uint32_t p0 = u >> 3, pn = span >> 3;
      for (uint32_t q = 0; q < pn; q++) prim[p0 + q] = e;
      if (u < x_cut) {
        const uint32_t end = u + span < x_cut ? u + span : x_cut;
        for (uint32_t q = u; q < end; q++) tail[q] = e;
      }
    }
  }
}

struct StreamSetup {
  int lg;
  uint32_t s_off, s_len;   // stream position inside the item (after the table description)
  uint32_t out_off, count; // first symbol index and symbol count of this stream
  const uint8_t* p;        // item payload after the table description
};

// Table description -> LUT (lane 0 of each item), then the jump table.  All 32 lanes call it;
// returns false for lanes that have nothing to decode.
__device__ __forceinline__ bool setup_item(DecodeSmem& S, const uint8_t* body, const ItemDesc& d, bool active, int slot,
                                           int stream, Ctrl* ctrl, StreamSetup& st) {
  const int lane = threadIdx.x;
  int lg = 0, hsize = -1;
  uint8_t* weights = &S.ring[0][0] + slot * 256;
  if (active && stream == 0) {
    int nsym = 0;
    FseDec& D = *reinterpret_cast<FseDec*>(&S.lut[slot][0]);
    hsize = huf_read_weights(weights, &nsym, &lg, body + d.src_off, d.src_len, D);
    if (hsize >= 0 && lg > kDecLutLog) {
      atomicOr(&ctrl->error, kErrUnsupported);
      hsize = -1;
    } else if (hsize < 0) {
      atomicOr(&ctrl->error, kErrCorrupt);
    }
    if (hsize >= 0) fill_lut(S.lut[slot], weights, nsym, lg);
  }
  __syncwarp();
  lg = __shfl_sync(0xffffffffu, lg, lane & ~3);
  hsize = __shfl_sync(0xffffffffu, hsize, lane & ~3);
  __syncwarp();  // the ring (aliased by weights) is free from here on
  if (!active || hsize < 0) return false;
  const uint8_t* p = body + d.src_off + hsize;
  const uint32_t rest = d.src_len - (uint32_t)hsize;
  if (rest < 10) {
    atomicOr(&ctrl->error, kErrCorrupt);
    return false;
  }
  const uint32_t l0 = p[0] | (p[1] << 8), l1 = p[2] | (p[3] << 8), l2 = p[4] | (p[5] << 8);
  if (l0 + l1 + l2 + 6 > rest) {
    atomicOr(&ctrl->error, kErrCorrupt);
    return false;
  }
  const uint32_t l3 = rest - (l0 + l1 + l2 + 6);
  const uint32_t seg = (d.dec_len + 3) >> 2;
  if (3 * seg > d.dec_len || l0 == 0 || l1 == 0 || l2 == 0 || l3 == 0) {
    atomicOr(&ctrl->error, kErrCorrupt);
    return false;
  }
  uint32_t s_off = 6, s_len = l0;
  if (stream == 1) { s_off += l0; s_len = l1; }
  if (stream == 2) { s_off += l0 + l1; s_len = l2; }
  if (stream == 3) { s_off += l0 + l1 + l2; s_len = l3; }
  st.lg = lg;
  st.p = p;
  st.s_off = s_off;
  st.s_len = s_len;
  st.out_off = (uint32_t)stream * seg;
  st.count = (stream == 3) ? d.dec_len - 3 * seg : seg;
  return true;
}

// ====================================================================================
// Kernel 2a: general mode -- decode coded planes into workspace planes.
// ====================================================================================
// One lane = one bitstream of item `d` (all 32 lanes call; 4 lanes per item slot): decode it into the
// item's workspace plane.
__device__ __forceinline__ void planar_decode_item(DecodeSmem& S, const DecodeCfg& cfg, const ItemDesc& d, bool active, int slot, int stream,
                                                   uint8_t* plane) {
  const int lane = threadIdx.x & 31;
  StreamSetup st;
  if (!setup_item(S, cfg.body, d, active, slot, stream, cfg.ctrl, st)) return;
  uint8_t* dst = plane + st.out_off;
  BitWindow b;
  const LutFull lut{S.lut[slot], st.lg};
  bool ok = window_init(b, st.p + st.s_off, st.s_len, cfg.body, S.ring[lane]);
  if (ok) {
    uint32_t done = 0;
    if ((((uintptr_t)dst) & 15) == 0) {
      const uint32_t n16 = st.count >> 4;
      uint4* d4 = reinterpret_cast<uint4*>(dst);
      for (uint32_t it = 0; it < n16; it++) {
        uint32_t o[4];
        decode16(b, lut, o);
        d4[it] = make_uint4(o[0], o[1], o[2], o[3]);
      }
      done = n16 << 4;
    }
    for (; done < st.count; done++) dst[done] = (uint8_t)decode1(b, lut);
    ok = window_exact(b);
  }
  if (!ok) atomicOr(&cfg.ctrl->error, kErrCorrupt);
}

__global__ void __launch_bounds__(32) k_huf_decode_planar(DecodeCfg cfg) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  DecodeSmem& S = *reinterpret_cast<DecodeSmem*>(smem_raw);
  const int lane = threadIdx.x, slot = lane >> 2, stream = lane & 3;
  const uint64_t nitems = (uint64_t)cfg.G * cfg.K;
  const uint64_t item = (uint64_t)blockIdx.x * kDecItemsPerWarp + slot;
  ItemDesc d;
  d.kind = kRaw;
  d.src_off = 0;
  d.src_len = d.dec_len = 0;
  bool active = false;
  uint64_t c = 0;
  int g = 0;
  if (item < nitems) {
    g = (int)(item / cfg.K);
    c = item - (uint64_t)g * cfg.K;
    if (cfg.mode[c] == kModeGeneral) {
      d = cfg.items[item];
      active = (d.kind == kHuf);
    }
  }
  if (__ballot_sync(0xffffffffu, active) == 0) return;
  planar_decode_item(S, cfg, d, active, slot, stream, active ? cfg.planes + ((uint64_t)cfg.slot[c] * cfg.G + g) * cfg.pstride : nullptr);
}

// ====================================================================================
// Kernel 2b: fused mode.  The lane that decodes 16 symbols of the coded plane also takes
// the 16 matching bytes of each other plane (raw bytes in the stream at any alignment, or
// a replicated RLE block read with stride 0), interleaves, un-rotates and emits 16*G bytes
// of elements.
//
// Warps work alone: a CTA of W warps is W independent decoders, each with its own shared-memory
// region (fused_smem_carve) and its own pair of mbarriers; nothing after the setup synchronises
// the CTA.  A warp takes chunk groups by a static stride or claims them one at a time.  Packing the
// warps into one CTA per SM pays Hopper's per-CTA shared-memory reserve once instead of once per
// warp, which is what makes room for the 16th and 17th bf16 warp.  With W = 1 the same code is
// one CTA per group, or a persistent grid of one-warp CTAs (the host's ZIPNN_B200_GRID_MODE).
//
// Bulk tensor copies (TMA) carry everything that is regular:
//   * side planes: for full chunks whose other planes are all stored raw (what float
//     tensors produce) the 32 quarter-plane segments of a warp lie at a fixed stride in
//     the stream -- byte plane g of chunk c at side_pred[g] + c * plane_len, stream j a
//     quarter plane further.  A 2-D tensor map over the payload (inner = bytes of one
//     segment, outer = segment index) delivers the next 16*T bytes of all 32 lanes as one
//     [32][16*T] box, at ANY byte alignment, into a swizzled tile that the lanes read with
//     conflict-free LDS.128 -- no per-lane cp.async (32 LSU wavefronts per instruction,
//     26 % of all shared-memory wavefronts of the round-1 kernel), no funnel shifts.
//   * output: the [32][128] stage is written with one 2-D bulk store per row (the 32 rows
//     are a quarter chunk apart), SWIZZLE_128B = the XOR pattern the stage already used.
// Anything irregular (RLE side planes, the ragged last chunk, groups with idle lanes, a
// driver without the tensor-map entry point) takes the cp.async / LDS+STG path below, in
// the same kernel.
// ====================================================================================
struct alignas(64) TmaMaps {
  CUtensorMap out;      // bytes {chunk / 4, 4 * k_full}, box {128, 32}, SWIZZLE_128B
  CUtensorMap side[3];  // per side plane: bytes {plane_len / 4 (+16), 4 * k_full}, box {16 * T, 32}
};
enum : uint32_t { kTmaOut = 1u, kTmaSide = 2u };

__device__ __forceinline__ void mbar_init(uint32_t bar_s, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_s), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar_s, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_s), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar_s, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(bar_s), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_s, const CUtensorMap* map, uint32_t x, uint32_t y, uint32_t bar_s) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst_s),
               "l"((uint64_t)(uintptr_t)map), "r"(x), "r"(y), "r"(bar_s)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src_s, uint32_t x, uint32_t y) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"((uint64_t)(uintptr_t)map), "r"(src_s), "r"(x), "r"(y)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared memory of one warp (dynamic; offsets from the 1 KiB aligned base, A = its shared address).  The number of
// resident warps is what the kernel's speed follows (DESIGN.md 3.1), and
// shared memory is what limits it, so nothing here is slack:
//   PB = 5 (bf16 / fp32 exponent planes):
//     cols  [32][32] u16   2 KiB   private 5-bit columns; must start on a 2 KiB boundary of the shared
//                                  address space (LutCol): at A's next 2 KiB boundary, 0 or 1 KiB in
//     ring lanes 0..15     1 KiB   the other KiB of the first three
//   PB = 0 (fp16 / fp8): prim [8][256] u16, 4 KiB
//   tail  [tail_cap] u16   2 (4) KiB  tail tables of the 8 chunks packed back to back (8 x 128 entries fit exactly)
//   ring  [..][64]                 per-lane stream rings (PB = 5: lanes 16..31, 1 KiB; PB = 0: all 32, 2 KiB);
//                                  weights[8][256] alias the two halves during the parse
//   stage [32][128]        4 KiB   one 128-byte output row per lane (1 KiB aligned, 16-byte units XOR-
//                                  swizzled by the row); the tANS scratch of the parse aliases it
//   side                           cp.async path: (G-1) x 2 KiB of slots (4 x 16 bytes per lane and plane);
//                                  bulk-tensor path (16-bit types): 2 stages x [32 lanes][48 bytes] = 3 KiB.
//                                  The two uses alias.
// bf16: 2 + 1 + 2 + 1 + 4 + 3 = 13 KiB;  fp32: 3 + 2 + 1 + 4 + 6 = 16 KiB;  fp16: 17 KiB;  fp8: 14 KiB.
// A CTA holds W such regions back to back (fused_warp_stride, a whole number of KiB, so every region starts 0 or 1 KiB
// past a 2 KiB boundary, which the carve absorbs) and behind them one pair of mbarriers per warp (16 B each).
template <int G>
struct FusedGeom {
  static constexpr int kIters = 8 / G;                 // iterations (16 symbols) per 128-byte output row
  static constexpr int NS = (G > 1) ? G - 1 : 1;
  static constexpr uint32_t kSlotBytes = 512u * ZB_SIDE_SLOTS;   // one side plane's cp.async slots (32 lanes)
  // Bulk-tensor side tiles (16-bit types): one tile serves two iterations: [32 lanes][32 bytes + 16], because a box
  // must start on a 16-byte boundary of global memory and the raw plane sits at any byte offset inside the stream.
  static constexpr int kTileIters = 2;
  static constexpr uint32_t kTileRow = 16u * kTileIters + 16u, kTileBytes = 32u * kTileRow;
  static constexpr uint32_t kTileRegion = (G == 2) ? 2u * kTileBytes : 0u;
  static constexpr uint32_t kSlotRegion = (G == 1) ? 0u : (uint32_t)(G - 1) * kSlotBytes;
  static constexpr uint32_t kSideAll = kSlotRegion > kTileRegion ? kSlotRegion : kTileRegion;
};
__host__ __device__ constexpr uint32_t fused_tail_bytes(int pb) { return pb == 0 ? 4096u : 2048u; }
__host__ __device__ constexpr uint32_t fused_tail_cap(int pb) { return fused_tail_bytes(pb) / 2u; }  // entries: 8 chunks x 128 fit exactly
template <int G>
__host__ __device__ constexpr uint32_t fused_warp_stride(int pb) {  // one warp's region, without its mbarriers
  return (pb == 0 ? 4096u + 32 * kRingBytes : 3072u + 16 * kRingBytes) + FusedGeom<G>::kSideAll + fused_tail_bytes(pb) + 32 * 128;
}
constexpr uint32_t kFusedBarBytes = 16;  // the two mbarriers of a warp
template <int G>
__host__ __device__ constexpr size_t fused_smem_bytes(int pb, int warps = 1) {
  return (size_t)warps * (fused_warp_stride<G>(pb) + kFusedBarBytes);
}
// Warps per CTA the kernel is compiled for (__launch_bounds__, and so its register budget): as many regions as the
// 227 KiB a Hopper CTA may opt into hold (bf16 17, fp8 16, fp32 14, fp16 13), but at most ZB_FUSED_MAX_WARPS.  The
// register file is split between the SM's four schedulers, so ptxas budgets for W rounded up to a multiple of 4:
// 17 warps leave 96 registers per thread (bf16 spills), 16 leave 128 (no spills), and the 17th warp would be a fifth
// one on a scheduler whose other four already keep it busy.  DESIGN.md 3.1 has the measurements.
#ifndef ZB_FUSED_MAX_WARPS
#define ZB_FUSED_MAX_WARPS 16
#endif
constexpr uint32_t kFusedCtaSmemMax = 232448;
template <int G, int PB>
__host__ __device__ constexpr int fused_smem_warps() {
  return (int)(kFusedCtaSmemMax / (fused_warp_stride<G>(PB) + kFusedBarBytes));
}
template <int G, int PB>
__host__ __device__ constexpr int fused_max_warps() {
  return fused_smem_warps<G, PB>() < ZB_FUSED_MAX_WARPS ? fused_smem_warps<G, PB>() : ZB_FUSED_MAX_WARPS;
}
static_assert(fused_warp_stride<1>(0) % 1024 == 0 && fused_warp_stride<2>(0) % 1024 == 0 && fused_warp_stride<2>(5) % 1024 == 0 &&
                  fused_warp_stride<4>(0) % 1024 == 0 && fused_warp_stride<4>(5) % 1024 == 0,
              "every warp region must start on a 1 KiB boundary (fused_smem_carve)");
static_assert(fused_smem_warps<2, 5>() == 17 && fused_smem_warps<4, 5>() == 14 && fused_smem_warps<2, 0>() == 13 && fused_smem_warps<1, 0>() == 16,
              "the warps per CTA that DESIGN.md 3.1 lists");
struct FusedSmem {
  unsigned char* raw;
  uint32_t base_s;     // shared address of raw
  uint32_t table_off;  // cols (PB = 5) or prim (PB = 0)
  uint32_t ring_lo_off, ring_hi_off;  // rings of lanes 0..15 / 16..31 (PB = 5: the first half fills the KiB next to the columns)
  uint32_t tail_off, stage_off, side_off;
  __device__ __forceinline__ uint16_t* tail() const { return reinterpret_cast<uint16_t*>(raw + tail_off); }
  __device__ __forceinline__ uint8_t* ring(int lane) const { return raw + (lane < 16 ? ring_lo_off : ring_hi_off) + kRingBytes * (uint32_t)(lane & 15); }
  // parse scratch: 256 weight bytes per chunk slot, four slots in each half of the rings
  __device__ __forceinline__ uint8_t* weights(int slot) const { return raw + (slot < 4 ? ring_lo_off : ring_hi_off) + 256u * (uint32_t)(slot & 3); }
  __device__ __forceinline__ uint8_t (*stage() const)[128] { return reinterpret_cast<uint8_t (*)[128]>(raw + stage_off); }
};
template <int G, int PB>
__device__ __forceinline__ FusedSmem fused_smem_carve(unsigned char* raw) {
  FusedSmem S;
  S.raw = raw;
  S.base_s = (uint32_t)__cvta_generic_to_shared(raw);
  // Opaque from here on: ptxas otherwise treats every address derived from it as "window base + constant"
  // and REBUILDS the base (S2R SR_CgaCtaId, MOV, LEA) at each use -- three extra instructions per symbol
  // in front of the predicated tail lookup.
  asm volatile("" : "+r"(S.base_s));
  uint32_t at;
  if (PB == 0) {
    S.table_off = 0;
    at = 4096;
  } else {
    S.table_off = (2048u - (S.base_s & 2047u)) & 2047u;  // 0 or 1024 for a 1 KiB aligned base
    S.ring_lo_off = S.table_off ? 0u : 2048u;
    at = 3072;
  }
  S.tail_off = at;
  at += fused_tail_bytes(PB);
  if (PB == 0) {
    S.ring_lo_off = at;
    at += 16 * kRingBytes;
  }
  S.ring_hi_off = at;
  at += 16 * kRingBytes;
  S.stage_off = at;  // 1 KiB multiple in both layouts
  at += 32 * 128;
  S.side_off = at;
  return S;
}
// Shared address of side-tile stage st / of plane g's cp.async slots (both inside the side region).
template <int G>
__device__ __forceinline__ uint32_t side_tile_s(const FusedSmem& S, uint32_t st) { return S.base_s + S.side_off + st * FusedGeom<G>::kTileBytes; }
template <int G>
__device__ __forceinline__ uint32_t side_slots_s(const FusedSmem& S, int g) { return S.base_s + S.side_off + (uint32_t)g * FusedGeom<G>::kSlotBytes; }
static_assert(sizeof(FseDecSmall) <= 512, "small tANS scratch must fit in 4 stage rows");

struct SidePlane {
  const uint4* blk;  // aligned block holding the plane byte that pairs with the lane's next symbol
  uint32_t shift;    // byte offset (0..15) of that byte inside the block
  uint32_t step;     // 1 for stream bytes, 0 for an RLE fill block
  uint4 a, b;        // blocks k, k+1
  uint32_t slots_s;  // shared address of this lane's two 16-byte slots; block j waits in slot (j & 1) ^ swz
  uint32_t swz;      // -- the XOR spreads the 8 lanes of a quarter warp over all banks
};

// The blocks in flight (k+2, k+3) are NOT held in registers.  A register load has a first use, and ptxas
// schedules the load right in front of it whatever the source order says (even for ld.volatile): with
// a register rotation a = b, b = c, c = d the first use of `d` is that move, at the end of the very
// iteration that requested it -- 12 % of all stall samples sat on that one instruction, and an L2
// prefetch only shortened the wait.  cp.async has no destination register: block k+3 is requested
// at the top of iteration k, joins the commit groups of the stream ring, and an LDS picks it up at
// the end of iteration k+1, after which its slot is free for block k+5: two slots per lane and plane.
__device__ __forceinline__ uint4 lds_u128(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
  return v;
}
constexpr uint32_t kSideSlots = ZB_SIDE_SLOTS;  // 16-byte slots per lane and side plane (2 or 4)
__device__ __forceinline__ uint32_t side_slot(const SidePlane& sp, uint32_t j) { return sp.slots_s + (((j & (kSideSlots - 1u)) ^ sp.swz) << 4); }

__device__ __forceinline__ uint4 ldg128(const uint4* p) { return __ldg(p); }
// 16 bytes starting `shift` bytes into the 32-byte pair (a, b).
__device__ __forceinline__ void take16(const uint4& a, const uint4& b, uint32_t shift, uint32_t (&out)[4]) {
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  const uint32_t bs = (shift & 3) * 8;
  uint32_t t[7];
#pragma unroll
  for (int i = 0; i < 7; i++) t[i] = __funnelshift_r(w[i], w[i + 1], bs);
  const bool s4 = shift & 4, s8 = shift & 8;
  uint32_t u[5];
#pragma unroll
  for (int i = 0; i < 5; i++) u[i] = s8 ? t[i + 2] : t[i];
#pragma unroll
  for (int i = 0; i < 4; i++) out[i] = s4 ? u[i + 1] : u[i];
}

// The same with the word part of the shift (W = shift / 4) known at compile time: four funnel shifts, no selects.
template <int W>
__device__ __forceinline__ void take16_w(const uint4& a, const uint4& b, uint32_t bit_shift, uint32_t (&out)[4]) {
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 4; i++) out[i] = __funnelshift_r(w[i + W], w[i + W + 1], bit_shift);
}

// Un-rotate at plane level: the two top byte planes hold [sign|mant7] (lo) and [exponent] (hi) of every element;
// the element's real top bytes are hi' = sign | exp >> 1, lo' = exp << 7 | mant7.
// The fused kernel's tables hold the exponent bytes already rotated right by one (lut_symbol), E = ror8(exp), so
// hi' = (E & 0x7F) | (sm & 0x80), lo' = (E & 0x80) | (sm & 0x7F): two bit selects per four elements, written as
// LOP3 because the compiler splits each into two operations.
__device__ __forceinline__ uint32_t bitselect(uint32_t a, uint32_t b, uint32_t m) {  // (a & m) | (b & ~m)
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
  return d;
}
// m = 0x80808080 for a rotated type, 0 otherwise (then hi = e, lo = sm: nothing happens, without a branch)
__device__ __forceinline__ void unrotate_planes_pre(uint32_t& lo, uint32_t& hi, uint32_t m) {
  const uint32_t sm = lo, e = hi;
  hi = bitselect(sm, e, m);
  lo = bitselect(e, sm, m);
}

// Output rows.  A lane produces 16*G bytes per iteration, 64 KiB away from its neighbours'
// data, so direct stores cost one LSU wavefront per lane.  Instead each lane fills a 128-byte
// row in shared memory (16-byte units XOR-swizzled by the row so that the 128-bit stores of 8
// lanes cover 32 banks -- which is exactly the tensor-map SWIZZLE_128B pattern), and once per row
// the 32 rows leave with one bulk tensor store (or, on the fallback path, 8 stores of four whole
// 128-byte lines each).
__device__ __forceinline__ uint4* stage_unit(uint8_t (*stage)[128], int row, int unit) {
  return reinterpret_cast<uint4*>(&stage[row][((unit ^ row) & 7) * 16]);
}

// Planes of 16 elements (pl[g][q] = bytes 4q..4q+3 of plane g) -> un-rotated, interleaved, into
// units [unit0, unit0 + G) of the lane's stage row.
template <int G>
__device__ __forceinline__ void emit_elements(uint32_t (&pl)[G][4], uint32_t rot_mask, uint8_t (*stage)[128], int lane, int unit0) {
  if (G == 1) {
    *stage_unit(stage, lane, unit0) = make_uint4(pl[0][0], pl[0][1], pl[0][2], pl[0][3]);
    return;
  }
#pragma unroll
  for (int q = 0; q < 4; q++) unrotate_planes_pre(pl[(G - 2) % G][q], pl[G - 1][q], rot_mask);  // the tables hold ror8(symbol)
  uint32_t w[4 * G];
  if (G == 2) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      w[2 * q] = __byte_perm(pl[0][q], pl[1 % G][q], 0x5140);
      w[2 * q + 1] = __byte_perm(pl[0][q], pl[1 % G][q], 0x7362);
    }
  } else {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const uint32_t t0 = __byte_perm(pl[0][q], pl[1 % G][q], 0x5140), t1 = __byte_perm(pl[2 % G][q], pl[3 % G][q], 0x5140);
      const uint32_t t2 = __byte_perm(pl[0][q], pl[1 % G][q], 0x7362), t3 = __byte_perm(pl[2 % G][q], pl[3 % G][q], 0x7362);
      w[4 * q] = __byte_perm(t0, t1, 0x5410);
      w[4 * q + 1] = __byte_perm(t0, t1, 0x7632);
      w[4 * q + 2] = __byte_perm(t2, t3, 0x5410);
      w[4 * q + 3] = __byte_perm(t2, t3, 0x7632);
    }
  }
#pragma unroll
  for (int q = 0; q < G; q++) *stage_unit(stage, lane, unit0 + q) = make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
}

// One iteration of the cp.async path: 16 symbols of the coded (top) plane + the matching bytes of
// the G-1 other planes -> 16*G bytes of elements into units [unit0, unit0+G) of the lane's stage row.
// guard = clamp the look-ahead block loads to the end of the stream buffer (only the last
// iterations of a stream can reach past it).  wait_store: the previous row's bulk store still
// reads the stage -- lane 0 waits for it after the decode, right before the first write.
template <int G, class LUT>
__device__ __forceinline__ void fused_iteration(BitWindow& b, const LUT& lut, SidePlane (&side)[(G > 1) ? G - 1 : 1],
                                                const uint4* hi_block, bool guard, bool rot, uint8_t (*stage)[128], int lane, int unit0, uint32_t it,
                                                bool wait_store) {
  if (G > 1) {
#pragma unroll
    for (int g = 0; g < G - 1; g++) {  // block k+3 of every side plane, used two iterations later
      const uint4* nb = side[g].blk + 3 * side[g].step;
      if (guard && side[g].step && nb > hi_block) nb = hi_block;  // (an RLE fill block lives in the workspace)
      cp_async16_s(side_slot(side[g], it + 3u), nb);  // joins the next commit group of decode16
    }
  }
  uint32_t pl[G][4];
  decode16(b, lut, pl[G - 1]);
  if (wait_store) {
    if (lane == 0) tma_store_wait_read();
    __syncwarp();
  }
  if (G > 1) {
#pragma unroll
    for (int g = 0; g < G - 1; g++) take16(side[g].a, side[g].b, side[g].shift, pl[g]);
  }
  emit_elements<G>(pl, rot ? 0x80808080u : 0u, stage, lane, unit0);
  if (G > 1) {
#pragma unroll
    for (int g = 0; g < G - 1; g++) {
      side[g].a = side[g].b;
      side[g].b = lds_u128(side_slot(side[g], it + 2u));  // requested in the previous iteration, landed since
      side[g].blk += side[g].step;
    }
  }
}

template <int G, int PB>
__global__ void __launch_bounds__(32 * fused_max_warps<G, PB>(), 1) k_huf_decode_fused(DecodeCfg cfg, uint8_t* __restrict__ out, const __grid_constant__ TmaMaps maps) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  using Geo = FusedGeom<G>;
  using LUT = typename std::conditional<PB == 0, LutTwo, LutCol<(PB ? PB : 5)>>::type;
  constexpr int kIters = Geo::kIters;
  constexpr int NS = Geo::NS;
  constexpr uint32_t kStride = fused_warp_stride<G>(PB);
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const FusedSmem S = fused_smem_carve<G, PB>(smem_raw + warp * kStride);
  const int lane = threadIdx.x & 31, slot = lane >> 2, stream = lane & 3;
  const uint64_t K = cfg.K;
  const uint64_t ngroups = (K + kDecItemsPerWarp - 1) / kDecItemsPerWarp;
  if (PB != 0 && S.table_off > 1024u) {  // the dynamic buffer is not 1 KiB aligned: cannot happen, but never decode wrongly
    if (lane == 0 && blockIdx.x == 0) atomicOr(&cfg.ctrl->error, kErrUnsupported);
    return;
  }
  // two mbarriers, one per side-tile stage, in the array behind the W regions (from the opaque base: see the carve)
  const uint32_t bar_s = S.base_s + (nwarps - warp) * kStride + kFusedBarBytes * warp;
  if (lane == 0) {
    mbar_init(bar_s, 1);
    mbar_init(bar_s + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  uint32_t tiles_done = 0;      // side tiles this warp has consumed: tile n sits in stage n & 1, its barrier phase is (n >> 1) & 1
  bool store_pending = false;   // a bulk store of this warp may still be reading the stage
  uint8_t (*const stage)[128] = S.stage();
  const uint32_t stage_s = S.base_s + S.stage_off;
  const bool rot = (cfg.bits_mode == 1) && (G > 1);
  const uint32_t rot_mask = rot ? 0x80808080u : 0u;
  const uint4* hi_block = reinterpret_cast<const uint4*>(((uintptr_t)(cfg.body + cfg.body_len) - 1) & ~(uintptr_t)15);

  // Static: warp w of CTA b takes groups b W + w, + grid W, ...  Claimed (cfg.fused_claim): each warp takes the next
  // unclaimed group when it is done with one, so no SM runs out of groups while another still has a round to go.
  const bool claim = cfg.fused_claim != 0;
  auto next_group = [&](uint64_t after) -> uint64_t {
    if (!claim) return after + (uint64_t)gridDim.x * nwarps;
    uint32_t g = 0;
    if (lane == 0) g = atomicAdd(&cfg.ctrl->fused_next, 1u);
    return __shfl_sync(0xffffffffu, g, 0);
  };
  for (uint64_t grp = claim ? next_group(0) : (uint64_t)blockIdx.x * nwarps + warp; grp < ngroups; grp = next_group(grp)) {
    const uint64_t c = grp * kDecItemsPerWarp + slot;
    const bool active = (c < K) && cfg.mode[c] == kModeFused;
    if (__ballot_sync(0xffffffffu, active) == 0) continue;
    if (store_pending) {  // the parse scratch aliases the stage
      if (lane == 0) tma_store_wait_read();
      store_pending = false;
    }
    __syncwarp();

    ItemDesc d;  // the coded plane: always group G-1 in fused mode
    d.kind = kRaw;
    d.src_off = 0;
    d.src_len = d.dec_len = 0;
    if (active) d = cfg.items[(uint64_t)(G - 1) * K + c];

    // ---- table description -> two-level table (lane 0 of each chunk) ----
    int lg = 0, hsize = -1, x_long = 0;
    uint32_t tail_at = 0;
    {
      uint8_t* weights = S.weights(slot);
      const bool builder = active && stream == 0;
      int nsym = 0;
      // The table description (<= 128 bytes: 1 + 127 of tANS-coded weights, or 1 + 64 of 4-bit weights,
      // huf_compress.c:140-167) goes to shared memory first, 16-byte blocks by the chunk's four lanes: the parser is
      // serial and reads it a byte at a time -- from global memory that was a DRAM / L2 round trip per pair of
      // weights (2 % of the kernel's samples sat on it).  The tail pool is free until the fill.
      constexpr uint32_t kHdrSlot = 176;  // 15 bytes of misalignment + 128 + the parser's 4-byte peeks, in 16-byte blocks
      uint8_t* hdr = reinterpret_cast<uint8_t*>(S.tail()) + kHdrSlot * (uint32_t)slot;
      const uint8_t* tsrc = cfg.body + d.src_off;
      const uint32_t mis = (uint32_t)((uintptr_t)tsrc & 15u);
      if (active) {
        const uint8_t* body_end = cfg.body + cfg.body_len;
#pragma unroll
        for (int q = 0; q < 3; q++) {
          const int blk = stream + 4 * q;
          const uint8_t* g = tsrc - mis + 16 * blk;
          if (blk < (int)(kHdrSlot / 16) && g < body_end) *reinterpret_cast<uint4*>(hdr + 16 * blk) = ldg128(reinterpret_cast<const uint4*>(g));
        }
      }
      __syncwarp();
      if (builder) {
        FseDecSmall& D = *reinterpret_cast<FseDecSmall*>(&stage[4 * slot][0]);
        const uint32_t avail = kHdrSlot - mis;
        hsize = huf_read_weights(weights, &nsym, &lg, hdr + mis, d.src_len < avail ? d.src_len : avail, D);
        if (hsize >= 0) {
          // (the tANS scratch D is dead once the weights are out: its first 32 bytes carry the class starts to the fill)
          x_long = PB == 0 ? lut2_tail_size(weights, nsym, lg) : lut_tail_size(weights, nsym, lg, PB, reinterpret_cast<uint16_t*>(&stage[4 * slot][0]));
          if (x_long < 0) hsize = -1;
        }
      }
      // the 8 tails share one pool: exclusive prefix over the chunks of the warp
      {
        const uint32_t mine = (builder && hsize >= 0) ? (uint32_t)x_long : 0u;
        uint32_t run = mine;
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, run, o);
          if (lane >= o) run += v;
        }
        tail_at = run - mine;
        if (builder && hsize >= 0 && run > fused_tail_cap(PB)) hsize = -1;  // does not fit: general path
      }
      if (builder) {
        if (hsize >= 0) {
          if (PB == 0) fill_lut2(reinterpret_cast<uint16_t*>(S.raw + S.table_off) + 256 * slot, S.tail() + tail_at, weights, nsym, lg, rot, (uint32_t)x_long);
        } else {
          // Not an error yet: a table that needs the big scratch, a long tail or log 12, or a
          // corrupt one.  Hand the chunk to the general kernels, which decide.
          cfg.mode[c] = (uint8_t)assign_general(cfg, c);
        }
      }
      __syncwarp();
      lg = __shfl_sync(0xffffffffu, lg, lane & ~3);
      hsize = __shfl_sync(0xffffffffu, hsize, lane & ~3);
      x_long = __shfl_sync(0xffffffffu, x_long, lane & ~3);
      tail_at = __shfl_sync(0xffffffffu, tail_at, lane & ~3);
      if (PB != 0) {  // private columns: the 4 lanes of a chunk fill their own copy in parallel
        nsym = __shfl_sync(0xffffffffu, nsym, lane & ~3);
        if (active && hsize >= 0)
          fill_lut_col<(PB ? PB : 5)>(reinterpret_cast<uint16_t*>(S.raw + S.table_off) + lane, S.tail() + tail_at, stream == 0, weights, nsym, lg, rot, (uint32_t)x_long,
                                      reinterpret_cast<const uint16_t*>(&stage[4 * slot][0]));
      }
      __syncwarp();  // the ring and the stage (aliased by the parse scratch) are free from here on
    }
    // From here on no lane leaves early: the output flush is a warp-wide exchange.
    bool live = active && hsize >= 0;

    // ---- jump table (huf_decompress.c:283-290) ----
    const uint8_t* p = cfg.body + d.src_off + (live ? hsize : 0);
    const uint32_t rest = live ? d.src_len - (uint32_t)hsize : 0;
    uint32_t l0 = 0, l1 = 0, l2 = 0, l3 = 0;
    if (live) {
      bool ok = rest >= 10;
      if (ok) {
        l0 = p[0] | (p[1] << 8);
        l1 = p[2] | (p[3] << 8);
        l2 = p[4] | (p[5] << 8);
        ok = l0 + l1 + l2 + 6 <= rest;
        l3 = rest - (l0 + l1 + l2 + 6);
        ok = ok && l0 && l1 && l2 && l3;
      }
      if (!ok) {
        atomicOr(&cfg.ctrl->error, kErrCorrupt);
        live = false;
      }
    }
    const uint32_t seg = d.dec_len >> 2;  // fused chunks: dec_len % 128 == 0
    uint32_t s_off = 6, s_len = l0;
    if (stream == 1) { s_off += l0; s_len = l1; }
    if (stream == 2) { s_off += l0 + l1; s_len = l2; }
    if (stream == 3) { s_off += l0 + l1 + l2; s_len = l3; }
    const uint32_t out_off = (uint32_t)stream * seg;

    LUT lut;
    if constexpr (PB == 0) {
      lut.prim_s = S.base_s + S.table_off + 512u * (uint32_t)slot;
    } else {
      lut.col_s = S.base_s + S.table_off + 2u * (uint32_t)lane;
    }
    lut.tail_s = S.base_s + S.tail_off + 2u * tail_at;
    lut.hi_mask = 0x7FFu & ~((uint32_t)x_long - 1u);   // x_long holds x_cut here (lut_tail_size / lut2_tail_size)

    // ---- which way do the other planes and the output travel?  (warp-uniform) ----
    // Bulk tensor copies need all 32 lanes live on full chunks and every other plane stored raw at its
    // predicted place (cfg.side_pred: all groups in front of it raw, which the host cannot know).
    bool regular = live && c < cfg.k_full;
    if (G > 1 && regular) {
#pragma unroll
      for (int g = 0; g < G - 1; g++) {
        const ItemDesc t = cfg.items[(uint64_t)g * K + c];
        regular = regular && t.kind == kRaw && t.src_off == cfg.side_pred[g] + c * (uint64_t)(cfg.chunk / (uint32_t)G);
      }
    }
    regular = __all_sync(0xffffffffu, regular);
    const bool out_tma = regular && (cfg.tma_flags & kTmaOut);
    const bool side_tma = (G == 2) && regular && (cfg.tma_flags & kTmaSide);

    BitWindow b;
    if (live && !window_init(b, p + s_off, s_len, cfg.body, S.ring(lane))) {
      atomicOr(&cfg.ctrl->error, kErrCorrupt);
      live = false;
    }
    // (a lane that drops out here only happens on a corrupt stream; `regular` groups keep going with the
    //  lane decoding garbage from its zeroed window -- the error bit is already set, the output is discarded)
    if (regular && !live) {
      b.cont = 0; b.s = 53; b.qm = 0; b.next = 0; b.fetch48 = 0; b.floor64 = 0xffffffffu; b.start_bit = 0;
      b.ring = S.ring(lane);
      b.ring_s = (uint32_t)__cvta_generic_to_shared(b.ring);
      b.gsrc = cfg.body;
    }

    const uint32_t rows_full = (seg >> 4) / kIters;
    if constexpr (G == 2) {
      if (side_tma) {
        // ================= side plane through bulk-tensor tiles (16-bit types, regular groups) =================
        // The 32 quarter planes of this warp's 8 chunks are rows 32 * grp .. +31 of maps.side[0] (row pitch = one
        // quarter plane).  Tile t = bytes [32 t, 32 t + 48) of every row, counted from the 16-byte boundary below
        // the plane's first byte: the 32 bytes iterations 2t and 2t+1 pair with their symbols start side_r0 (0..15)
        // bytes into it.  One thread asks for tile t+1 while the warp works on tile t; the bytes land in shared
        // memory without a single LSU instruction (the cp.async path pays 32 L1 wavefronts per instruction because
        // every lane's 16 bytes lie in a different line: a fifth of the kernel's LSU time).
        const uint32_t y0 = (uint32_t)(grp * 32u);
        constexpr int kTI = Geo::kTileIters;              // iterations served by one tile
        constexpr int kTilesPerRow = kIters / kTI;
        const uint32_t ntiles = rows_full * (uint32_t)kTilesPerRow;
        const uint32_t r0 = cfg.side_r0[0];
        auto issue_tile = [&](uint32_t t) {
          const uint32_t st = (tiles_done + t) & 1u;
          mbar_expect_tx(bar_s + 8u * st, Geo::kTileBytes);
          tma_load_2d(side_tile_s<G>(S, st), &maps.side[0], 16u * (uint32_t)kTI * t, y0, bar_s + 8u * st);
        };
        if (lane == 0 && ntiles) issue_tile(0);
        // The 8 stage rows this lane writes out each round are rows 4r + lane/8 = stream lane/8 of chunk slot r, 16-byte
        // unit lane%8: with full chunks (this path) they lie at flush_ptr + r * chunk, so ONE pointer that moves on by
        // 128 per row serves all eight stores -- as immediate offsets for the reference's default chunk size.
        uint8_t* flush_ptr = out + (grp * (uint64_t)kDecItemsPerWarp) * (uint64_t)cfg.chunk + (uint64_t)((uint32_t)(lane >> 3) * seg) * G +
                             (uint32_t)(lane & 7) * 16u;
        const uint32_t chunk_b = cfg.chunk;
        const bool chunk_256k = chunk_b == 262144u;
        // side_r0 is the same for every warp of the launch: the word part of the alignment shift is a 4-way switch
        // around the row loop (four funnel shifts per iteration instead of seven shifts + nine selects)
        const uint32_t bit_shift = (r0 & 3u) * 8u;
        auto run_rows = [&](auto wtag) {
          constexpr int W = decltype(wtag)::value;
          for (uint32_t row = 0; row < rows_full; row++) {
#pragma unroll
            for (int tr = 0; tr < kTilesPerRow; tr++) {
              const uint32_t t = row * (uint32_t)kTilesPerRow + (uint32_t)tr;
              const uint32_t n = tiles_done + t;
              __syncwarp();  // every lane has read tile t-1: its stage may be overwritten by tile t+1
              if (lane == 0 && t + 1 < ntiles) issue_tile(t + 1);
              mbar_wait(bar_s + 8u * (n & 1u), (n >> 1) & 1u);
              const uint32_t my_row = side_tile_s<G>(S, n & 1u) + (uint32_t)lane * Geo::kTileRow;
              uint4 blk[kTI + 1];
#pragma unroll
              for (int q = 0; q <= kTI; q++) blk[q] = lds_u128(my_row + 16u * (uint32_t)q);
#pragma unroll
              for (int ki = 0; ki < kTI; ki++) {
                uint32_t pl[G][4];
                decode16(b, lut, pl[G - 1]);
                take16_w<W>(blk[ki], blk[ki + 1], bit_shift, pl[0]);
                emit_elements<G>(pl, rot_mask, stage, lane, (tr * kTI + ki) * G);
              }
            }
            // (a bulk tensor store of the 32 rows instead of these 8 x (LDS.128 + STG.128) is ZIPNN_B200_TMA=1: the fence
            //  and the wait for the store's reads cost what the LSU work saves)
            __syncwarp();
            if (chunk_256k) {
#pragma unroll
              for (int r = 0; r < 8; r++) *reinterpret_cast<uint4*>(flush_ptr + (size_t)r * 262144u) = *stage_unit(stage, r * 4 + (lane >> 3), lane & 7);
            } else {
#pragma unroll
              for (int r = 0; r < 8; r++) *reinterpret_cast<uint4*>(flush_ptr + (size_t)r * chunk_b) = *stage_unit(stage, r * 4 + (lane >> 3), lane & 7);
            }
            flush_ptr += 128;
            __syncwarp();
          }
        };
        switch (r0 >> 2) {
          case 0: run_rows(std::integral_constant<int, 0>{}); break;
          case 1: run_rows(std::integral_constant<int, 1>{}); break;
          case 2: run_rows(std::integral_constant<int, 2>{}); break;
          default: run_rows(std::integral_constant<int, 3>{}); break;
        }
        tiles_done += ntiles;
        if (live && !window_exact(b)) atomicOr(&cfg.ctrl->error, kErrCorrupt);
        continue;
      }
    }
    // ================= cp.async / LDS + STG path =================
    // ---- the other planes: groups 0 .. G-2 ----
    SidePlane side[NS];
    if (G > 1 && live) {
#pragma unroll
      for (int g = 0; g < G - 1; g++) {
        const uint64_t i = (uint64_t)g * K + c;
        const ItemDesc t = cfg.items[i];
        const uint8_t* q;
        if (t.kind == kRle) {
          q = cfg.fill + i * kFillBytes;
          side[g].step = 0;
        } else {
          q = cfg.body + t.src_off + out_off;
          side[g].step = 1;
        }
        side[g].shift = (uint32_t)((uintptr_t)q & 15);
        side[g].blk = reinterpret_cast<const uint4*>((uintptr_t)q & ~(uintptr_t)15);
        side[g].a = ldg128(side[g].blk);
        const uint4* nb = side[g].blk + side[g].step;
        side[g].b = ldg128((side[g].step && nb > hi_block) ? hi_block : nb);
        nb += side[g].step;
        // block 2 waits in slot 0 (committed and waited for by the first decode16 group)
        side[g].swz = kSideSlots == 2 ? (((uint32_t)lane >> 2) & 1u) : (((uint32_t)lane >> 1) & 3u);
        side[g].slots_s = side_slots_s<G>(S, g) + 16u * kSideSlots * (uint32_t)lane;
        cp_async16_s(side_slot(side[g], 2u), (side[g].step && nb > hi_block) ? hi_block : nb);
      }
      cp_async_commit();
      cp_async_wait<0>();
    }

    // ---- rows: 128 bytes of output = 128/G elements = kIters iterations of 16 symbols ----
    const uint32_t my_rows = live ? rows_full : 0;
    uint32_t max_rows = my_rows;
#pragma unroll
    for (int o = 16; o; o >>= 1) max_rows = max(max_rows, __shfl_xor_sync(0xffffffffu, max_rows, o));
    if (out_tma) {
      const uint32_t y0 = (uint32_t)(grp * 32u);
      for (uint32_t row = 0; row < max_rows; row++) {
        const bool guard = row + 2 >= my_rows;
#pragma unroll
        for (int k = 0; k < kIters; k++)
          fused_iteration<G, LUT>(b, lut, side, hi_block, guard, rot, stage, lane, k * G, row * (uint32_t)kIters + (uint32_t)k, k == 0 && store_pending);
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) tma_store_2d(&maps.out, stage_s, row * 128u, y0);
        store_pending = true;
      }
    } else {
      // the 8 stage rows this lane writes out each round: row r*4 + lane/8, 16-byte unit lane%8
      const uint64_t my_out = (uint64_t)(uintptr_t)(out + c * (uint64_t)cfg.chunk + (uint64_t)out_off * G);
      uint64_t row_out[8];
      uint32_t row_cnt[8];
#pragma unroll
      for (int r = 0; r < 8; r++) {
        const int src = r * 4 + (lane >> 3);
        row_out[r] = __shfl_sync(0xffffffffu, my_out, src) + (uint64_t)(lane & 7) * 16;
        row_cnt[r] = __shfl_sync(0xffffffffu, my_rows, src);
      }
      if (store_pending) {
        if (lane == 0) tma_store_wait_read();
        store_pending = false;
        __syncwarp();
      }
      for (uint32_t row = 0; row < max_rows; row++) {
        if (row < my_rows) {
          const bool guard = row + 2 >= my_rows;  // look-ahead of 3 blocks: clamp in the last two rows
#pragma unroll
          for (int k = 0; k < kIters; k++)
            fused_iteration<G, LUT>(b, lut, side, hi_block, guard, rot, stage, lane, k * G, row * (uint32_t)kIters + (uint32_t)k, false);
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 8; r++) {
          const int src = r * 4 + (lane >> 3);
          if (row < row_cnt[r]) {
            const uint4 v = *stage_unit(stage, src, lane & 7);
            *reinterpret_cast<uint4*>((uintptr_t)(row_out[r] + (uint64_t)row * 128)) = v;
          }
        }
        __syncwarp();
      }
    }
    if (live && !window_exact(b)) atomicOr(&cfg.ctrl->error, kErrCorrupt);
  }
  if (store_pending && lane == 0) tma_store_wait_all();  // the stage must outlive the last bulk store's reads
}

// ====================================================================================
// Kernel 3: regroup byte planes into the element stream (+ un-rotate the sign bit), for
// chunks the fused kernel did not take.  Sources per (group, chunk): raw bytes inside the
// stream (unaligned), one RLE byte, or a decoded plane in the workspace.
// ====================================================================================
struct PlaneSrc {
  const uint8_t* ptr;  // first plane byte (any alignment); nullptr => constant fill
  uint32_t fill;       // the RLE byte replicated into 4 lanes
  uint32_t len;        // plane bytes
};

template <int NW>
__device__ __forceinline__ void load_plane_words(const PlaneSrc& s, uint32_t j, uint32_t (&out)[NW]) {
  if (s.ptr == nullptr) {
#pragma unroll
    for (int i = 0; i < NW; i++) out[i] = s.fill;
    return;
  }
  const uintptr_t a = (uintptr_t)(s.ptr + j);
  const uint32_t* base = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  uint32_t w[NW + 1];
#pragma unroll
  for (int i = 0; i < NW; i++) w[i] = __ldg(base + i);
  w[NW] = sh ? __ldg(base + NW) : 0u;  // only touched when the run really spills into it
#pragma unroll
  for (int i = 0; i < NW; i++) out[i] = __funnelshift_r(w[i], w[i + 1], sh);
}

__device__ __forceinline__ uint8_t plane_byte(const PlaneSrc& s, uint32_t j) {
  return s.ptr ? s.ptr[j] : (uint8_t)s.fill;
}

constexpr int kMergeThreads = 256;
constexpr uint32_t kMergeTile = kMergeThreads * 16 * 4;  // bytes of output per block step (16 KiB)

static_assert(kMergeThreads * 16 == kBoxStep, "regroup_tile advances the box cursor by kBoxStep");

// One 16 KiB output tile of chunk c, by the kMergeThreads threads of a CTA.  `pslot` = the chunk's plane slot.
// W: `out` is the box of cfg (box_store16) instead of the whole tensor.
template <int G, bool W = false>
__device__ __forceinline__ void regroup_tile(const DecodeCfg& cfg, uint8_t* __restrict__ out, uint64_t c, uint32_t tile, uint32_t pslot,
                                             PlaneSrc (&src)[G]) {
  const uint64_t K = cfg.K;
  const uint32_t chunk = cfg.chunk;
  const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(cfg.orig - c * (uint64_t)chunk) : chunk;
  const uint32_t o_begin = tile * kMergeTile;
  if (o_begin >= chunk_len) return;  // (uniform across the CTA)
  if (W && !box_meets(cfg, c * (uint64_t)chunk + o_begin, min(kMergeTile, chunk_len - o_begin))) return;  // (uniform)
  __syncthreads();
  if (threadIdx.x < G) {
    const int g = threadIdx.x;
    const ItemDesc d = cfg.items[(uint64_t)g * K + c];
    PlaneSrc s;
    s.len = d.dec_len;
    s.fill = 0;
    if (d.kind == kRaw) {
      s.ptr = cfg.body + d.src_off;
    } else if (d.kind == kRle) {
      s.ptr = nullptr;
      s.fill = 0x01010101u * (uint32_t)cfg.body[d.src_off];
    } else {
      s.ptr = cfg.planes + ((uint64_t)pslot * G + g) * cfg.pstride;
    }
    src[g] = s;
  }
  __syncthreads();
  uint8_t* out_c = out + c * (uint64_t)chunk;
  const uint32_t o_end = min(chunk_len, o_begin + kMergeTile);
  const uint32_t rot_words = (cfg.bits_mode == 1 && G > 1) ? (chunk_len >> 2) : 0;  // words that get un-rotated
  BoxCursor bc;
  if (W) bc = box_cursor(cfg, c * (uint64_t)chunk + o_begin + threadIdx.x * 16);
  for (uint32_t o = o_begin + threadIdx.x * 16; o < o_end; o += kMergeThreads * 16) {
    if (o + 16 <= o_end) {
      uint32_t r[4];
      if (G == 1) {
        load_plane_words<4>(src[0], o, r);
      } else if (G == 2) {
        uint32_t a[2], b2[2];
        load_plane_words<2>(src[0], o >> 1, a);
        load_plane_words<2>(src[1 % G], o >> 1, b2);
        r[0] = __byte_perm(a[0], b2[0], 0x5140);
        r[1] = __byte_perm(a[0], b2[0], 0x7362);
        r[2] = __byte_perm(a[1], b2[1], 0x5140);
        r[3] = __byte_perm(a[1], b2[1], 0x7362);
      } else {
        uint32_t p0[1], p1[1], p2[1], p3[1];
        load_plane_words<1>(src[0], o >> 2, p0);
        load_plane_words<1>(src[1 % G], o >> 2, p1);
        load_plane_words<1>(src[2 % G], o >> 2, p2);
        load_plane_words<1>(src[3 % G], o >> 2, p3);
        const uint32_t t0 = __byte_perm(p0[0], p1[0], 0x5140), t1 = __byte_perm(p2[0], p3[0], 0x5140);
        const uint32_t t2 = __byte_perm(p0[0], p1[0], 0x7362), t3 = __byte_perm(p2[0], p3[0], 0x7362);
        r[0] = __byte_perm(t0, t1, 0x5410);
        r[1] = __byte_perm(t0, t1, 0x7632);
        r[2] = __byte_perm(t2, t3, 0x5410);
        r[3] = __byte_perm(t2, t3, 0x7632);
      }
      const uint32_t w0 = o >> 2;
#pragma unroll
      for (int i = 0; i < 4; i++)
        if (w0 + i < rot_words) r[i] = unrot_word<G>(r[i]);
      if (W) {
        box_store16(cfg, out, bc, r);
        box_advance(cfg, bc);
      } else {
        *reinterpret_cast<uint4*>(out_c + o) = make_uint4(r[0], r[1], r[2], r[3]);
      }
    } else {
      // ragged tail of the last chunk: byte by byte, whole words still get un-rotated
      for (uint32_t q = o; q < min(o + 16, o_end); q += 4) {
        uint32_t w = 0;
        const uint32_t nb = min(4u, o_end - q);
        for (uint32_t i = 0; i < nb; i++) {
          const uint32_t pos = q + i;
          w |= (uint32_t)plane_byte(src[pos % G], pos / G) << (8 * i);
        }
        if ((q >> 2) < rot_words) w = unrot_word<G>(w);
        for (uint32_t i = 0; i < nb; i++) {
          if (W) box_put(cfg, out, c * (uint64_t)chunk + q + i, (uint8_t)(w >> (8 * i)));
          else out_c[q + i] = (uint8_t)(w >> (8 * i));
        }
      }
    }
  }
}

template <bool W>
__device__ __forceinline__ void regroup_tile_any(const DecodeCfg& cfg, uint64_t c, uint32_t tile, PlaneSrc (&src)[4]) {
  if (cfg.G == 1) regroup_tile<1, W>(cfg, cfg.out, c, tile, cfg.slot[c], reinterpret_cast<PlaneSrc (&)[1]>(src));
  else if (cfg.G == 2) regroup_tile<2, W>(cfg, cfg.out, c, tile, cfg.slot[c], reinterpret_cast<PlaneSrc (&)[2]>(src));
  else regroup_tile<4, W>(cfg, cfg.out, c, tile, cfg.slot[c], src);
}
// a call of its own: the window's registers must not spill into the unwindowed loop of k_regroup_batch
__device__ __noinline__ void regroup_tile_boxed(const DecodeCfg& cfg, uint64_t c, uint32_t tile, PlaneSrc (&src)[4]) {
  regroup_tile_any<true>(cfg, c, tile, src);
}
__global__ void __launch_bounds__(kMergeThreads) k_regroup_batch(BatchCfg B) {
  __shared__ PlaneSrc src[4];
  const uint64_t total = B.tile_start[B.n];
  for (uint64_t w = blockIdx.x; w < total; w += gridDim.x) {
    const uint32_t t = batch_find(B.tile_start, B.n, w);
    const DecodeCfg& cfg = B.cfgs[t];
    const uint32_t tiles_per_chunk = (cfg.chunk + kMergeTile - 1) / kMergeTile;
    const uint64_t local = w - B.tile_start[t];
    if (local >= (uint64_t)cfg.ctrl->regroup_count * tiles_per_chunk) continue;  // (uniform)
    const uint64_t c = cfg.rlist[local / tiles_per_chunk];
    const uint32_t tile = (uint32_t)(local % tiles_per_chunk);
    if (cfg.box_len) regroup_tile_boxed(cfg, c, tile, src);
    else regroup_tile_any<false>(cfg, c, tile, src);
  }
}

template <int G>
__global__ void __launch_bounds__(kMergeThreads) k_regroup(DecodeCfg cfg, uint8_t* __restrict__ out) {
  __shared__ PlaneSrc src[G];
  const uint32_t tiles_per_chunk = (cfg.chunk + kMergeTile - 1) / kMergeTile;
  const uint64_t ntiles = (uint64_t)cfg.ctrl->regroup_count * tiles_per_chunk;  // usually none: the fused kernel wrote everything
  for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const uint64_t c = cfg.rlist[t / tiles_per_chunk];
    regroup_tile<G>(cfg, out, c, (uint32_t)(t % tiles_per_chunk), cfg.slot[c], src);
  }
}

// ====================================================================================
// Kernel 4: general chunks beyond the slot pool.  kOverflowCtas persistent CTAs, each owning the
// plane slot max_slots + blockIdx.x: warp 0 decodes the chunk's coded planes (one lane per
// bitstream, G x 4 <= 16 of them), then the whole CTA regroups the chunk and takes the next
// one.  Costs nothing when the queue is empty (the normal case).
// ====================================================================================
template <int G, bool W = false>
__device__ __forceinline__ void decode_overflow_body(const DecodeCfg& cfg, uint8_t* __restrict__ out, DecodeSmem& S, PlaneSrc (&src)[G]) {
  const uint32_t n = cfg.ctrl->overflow_count;
  const uint32_t pslot = cfg.max_slots + blockIdx.x;
  const uint32_t tiles_per_chunk = (cfg.chunk + kMergeTile - 1) / kMergeTile;
  for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
    const uint64_t c = cfg.olist[i];
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x, slot = lane >> 2, stream = lane & 3;
      ItemDesc d;
      d.kind = kRaw;
      d.src_off = 0;
      d.src_len = d.dec_len = 0;
      bool active = false;
      if (slot < G) {
        d = cfg.items[(uint64_t)slot * cfg.K + c];
        active = (d.kind == kHuf);
      }
      planar_decode_item(S, cfg, d, active, slot, stream, cfg.planes + ((uint64_t)pslot * G + (slot < G ? slot : 0)) * cfg.pstride);
    }
    __threadfence_block();
    __syncthreads();  // the planes are complete
    for (uint32_t tile = 0; tile < tiles_per_chunk; tile++) regroup_tile<G, W>(cfg, out, c, tile, pslot, src);
    __syncthreads();  // ... and read, before the next chunk overwrites them
  }
}

// The same for CTA `cta` of `ncta` (at most ovf_slots): it owns plane slot max_slots + cta and takes queued chunks cta,
// cta + ncta, ...  (k_plan_replay_persistent, whose grid is not the overflow grid.  A copy rather than a parameter of
// decode_overflow_body: the parameter changes the code the existing launches compile to.)
template <int G, bool W>
__device__ __forceinline__ void decode_overflow_part(const DecodeCfg& cfg, uint8_t* __restrict__ out, DecodeSmem& S, PlaneSrc (&src)[G], uint32_t cta,
                                                     uint32_t ncta) {
  const uint32_t n = cfg.ctrl->overflow_count;
  const uint32_t pslot = cfg.max_slots + cta;
  const uint32_t tiles_per_chunk = (cfg.chunk + kMergeTile - 1) / kMergeTile;
  for (uint32_t i = cta; i < n; i += ncta) {
    const uint64_t c = cfg.olist[i];
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x, slot = lane >> 2, stream = lane & 3;
      ItemDesc d;
      d.kind = kRaw;
      d.src_off = 0;
      d.src_len = d.dec_len = 0;
      bool active = false;
      if (slot < G) {
        d = cfg.items[(uint64_t)slot * cfg.K + c];
        active = (d.kind == kHuf);
      }
      planar_decode_item(S, cfg, d, active, slot, stream, cfg.planes + ((uint64_t)pslot * G + (slot < G ? slot : 0)) * cfg.pstride);
    }
    __threadfence_block();
    __syncthreads();  // the planes are complete
    for (uint32_t tile = 0; tile < tiles_per_chunk; tile++) regroup_tile<G, W>(cfg, out, c, tile, pslot, src);
    __syncthreads();  // ... and read, before the next chunk overwrites them
  }
}

template <int G>
__global__ void __launch_bounds__(kMergeThreads) k_decode_overflow(DecodeCfg cfg, uint8_t* __restrict__ out) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ PlaneSrc src[G];
  decode_overflow_body<G>(cfg, out, *reinterpret_cast<DecodeSmem*>(smem_raw), src);
}
template <bool W>
__device__ __forceinline__ void decode_overflow_any(const DecodeCfg& cfg, DecodeSmem& S, PlaneSrc (&src)[4]) {
  if (cfg.G == 1) decode_overflow_body<1, W>(cfg, cfg.out, S, reinterpret_cast<PlaneSrc (&)[1]>(src));
  else if (cfg.G == 2) decode_overflow_body<2, W>(cfg, cfg.out, S, reinterpret_cast<PlaneSrc (&)[2]>(src));
  else decode_overflow_body<4, W>(cfg, cfg.out, S, src);
}
// grid = (kOverflowCtas, tensors)
__global__ void __launch_bounds__(kMergeThreads) k_decode_overflow_batch(BatchCfg B) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ PlaneSrc src[4];
  const DecodeCfg& cfg = B.cfgs[blockIdx.y];
  if (blockIdx.x >= cfg.ovf_slots || cfg.ctrl->overflow_count == 0) return;
  DecodeSmem& S = *reinterpret_cast<DecodeSmem*>(smem_raw);
  if (cfg.box_len) decode_overflow_any<true>(cfg, S, src);
  else decode_overflow_any<false>(cfg, S, src);
}

}  // namespace zb
