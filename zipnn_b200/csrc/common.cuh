// common.cuh -- shared device helpers for the zipnn_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "huf_serial.cuh"

namespace zb {

// ---- workspace control block (first 256 bytes of every workspace) ----------------
struct Ctrl {
  uint32_t error;        // OR of ZIPNN_B200_E_* bits raised by kernels
  uint32_t overflow_count; // decode: chunks queued for k_decode_overflow (DecodeCfg::olist)
  uint64_t base[4];      // payload offset of group g inside `body`
  uint64_t total_len;    // compress: total stream length
  uint64_t group_total[4];
  uint32_t work_counter; // persistent-kernel work queue
  uint32_t regroup_count; // decode: chunks that go through k_regroup (listed in DecodeCfg::rlist)
  uint32_t huf_count;     // decode: coded items queued for k_huf_decode_sync (DecodeCfg::hlist)
  uint32_t fused_next;    // decode: next chunk group a warp of the packed k_huf_decode_fused launch claims
};
static_assert(sizeof(Ctrl) <= 256, "ctrl block");
constexpr size_t kCtrlBytes = 256;

// One (group, chunk) payload item of the stream.
struct ItemDesc {
  uint64_t src_off;   // offset of the payload inside `body`
  uint32_t src_len;   // payload bytes
  uint32_t dec_len;   // decoded plane bytes
  uint32_t kind;      // kRaw / kRle / kHuf
  uint32_t pad;
};
enum : uint32_t { kRaw = 0, kRle = 1, kHuf = 2 };

// error bits kept in Ctrl::error
// (kErrIndex: a gather met an id outside [0, rows); raised in a decode plan's error word only)
enum : uint32_t { kErrCorrupt = 1u, kErrUnsupported = 2u, kErrWorkspace = 4u, kErrIndex = 8u };

// ---- sign-bit rotation (reference data_manipulation_dtype16.c:10-20,145-155;
//      data_manipulation_dtype32.c:39-49,275-285) ----------------------------------
// 16-bit types: one 32-bit word holds two elements; [s e8 m7] <-> [e8 s m7].
__host__ __device__ __forceinline__ uint32_t rot16(uint32_t u) {
  return ((u >> 8) & 0x00800080u) | ((u << 1) & 0xFF00FF00u) | (u & 0x007F007Fu);
}
__host__ __device__ __forceinline__ uint32_t unrot16(uint32_t u) {
  return ((u << 8) & 0x80008000u) | ((u >> 1) & 0x7F807F80u) | (u & 0x007F007Fu);
}
__host__ __device__ __forceinline__ uint32_t rot32(uint32_t u) {
  return ((u >> 8) & 0x00800000u) | ((u << 1) & 0xFF000000u) | (u & 0x007FFFFFu);
}
__host__ __device__ __forceinline__ uint32_t unrot32(uint32_t u) {
  return ((u << 8) & 0x80000000u) | ((u >> 1) & 0x7F800000u) | (u & 0x007FFFFFu);
}
template <int G>
__host__ __device__ __forceinline__ uint32_t rot_word(uint32_t u) {
  return G == 2 ? rot16(u) : (G == 4 ? rot32(u) : u);
}
template <int G>
__host__ __device__ __forceinline__ uint32_t unrot_word(uint32_t u) {
  return G == 2 ? unrot16(u) : (G == 4 ? unrot32(u) : u);
}

__host__ __device__ __forceinline__ uint32_t plane_len(uint32_t chunk_len, int G, int g) {
  return chunk_len / (uint32_t)G + ((uint32_t)g < chunk_len % (uint32_t)G ? 1u : 0u);
}

// ---- batches of tensors: start[t] is the exclusive prefix sum of tensor t's work, start[n] the total;
//      the tensor that owns flat work index w (w < start[n]; tensors without work are never returned)
__device__ __forceinline__ uint32_t batch_find(const uint64_t* start, uint32_t n, uint64_t w) {
  uint32_t lo = 0, hi = n;  // start[lo] <= w < start[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (start[mid] <= w) lo = mid; else hi = mid;
  }
  return lo;
}

// ---- unaligned little-endian loads from global memory -----------------------------
__device__ __forceinline__ uint64_t ld_u64_bytes(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i);
  return v;
}
__device__ __forceinline__ void st_u64_bytes(uint8_t* p, uint64_t v) {
#pragma unroll
  for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (8 * i));
}

// Aligned 32-bit word that may straddle the ends of [lo, hi): bytes outside read as 0.
__device__ __forceinline__ uint32_t ld_word_guarded(const uint32_t* p, const uint8_t* lo, const uint8_t* hi) {
  const uint8_t* b = reinterpret_cast<const uint8_t*>(p);
  if (b >= lo && b + 4 <= hi) return __ldg(p);
  uint32_t v = 0;
#pragma unroll
  for (int i = 0; i < 4; i++)
    if (b + i >= lo && b + i < hi) v |= (uint32_t)b[i] << (8 * i);
  return v;
}

// 4 consecutive bytes starting at an arbitrary byte address, built from aligned words.
// `base` is the address rounded down to 4, `sh` = 8*(addr&3); w0,w1 the words at base, base+4.
__device__ __forceinline__ uint32_t align_bytes(uint32_t w0, uint32_t w1, uint32_t sh) {
  return __funnelshift_r(w0, w1, sh);  // sh in {0,8,16,24}
}

}  // namespace zb
