// encode.cuh -- compress side.
//
//   pass A  k_encode_stats : per chunk, per byte-group: four per-stream 256-bin histograms,
//                            then (one warp per group) the reference's block decisions --
//                            RLE / "not compressible" early-outs, length-limited Huffman
//                            code lengths, table description, exact compressed size,
//                            threshold -> type byte + payload size + saved code lengths.
//   scan    k_encode_scan  : per group inclusive prefix sums of payload sizes -> the
//                            stream's cumulative table, group bases, item offsets, total
//                            length, python header.
//   pass B  k_encode_write : per (chunk, group): raw planes copied, Huffman blocks
//                            bit-packed (per-thread runs, block-wide exclusive scan of bit
//                            lengths, OR into a shared bit buffer, word-coalesced flush)
//                            straight to their final position in the stream.
//
// Replaces reference csrc/zipnn_core.c:294-390 (compression_worker), :105-244
// (prepare_python_return_buffer), hist.c, huf_compress.c:215-724, and the split halves of
// data_manipulation_dtype16.c:64-138 / data_manipulation_dtype32.c:78-133.
#pragma once
#include "common.cuh"
#include "stage1.cuh"

#include <type_traits>

namespace zb {

// Saved per item by pass A for pass B.
struct EncSave {
  uint8_t nb[256];      // code length per symbol (0 = absent)
  uint8_t hdr[128];     // table description (RLE: hdr[0] = the byte)
  uint32_t hsize;       // table description bytes
  uint32_t sbytes[4];   // byte size of each of the 4 bitstreams
  uint32_t lg;          // table log
  uint32_t pad[2];
};
static_assert(sizeof(EncSave) == 416, "EncSave layout");

constexpr int kEncThreads = 256;

// ---- batches of tensors ------------------------------------------------------------------------------------
// A batch kernel runs the single-tensor kernel's per-chunk or per-item code for every tensor of one byte-group
// class in one launch.  A flat work index finds its tensor by binary search over an exclusive prefix sum of that
// kernel's per-tensor work (batch_find), so tensors of any size share one grid.  The hist body and the write kernels
// take the batch as a template parameter; its NoBatch form is the single-tensor kernel, whose code is unchanged, with
// the tensor's arguments taken from the kernel parameters.
struct EncTensor {
  const uint8_t* in;
  uint8_t* out;
  const uint8_t* hdr;        // this tensor's python header inside the batch's packed header area
  uint64_t n, K;
  uint32_t chunk, hdr_len;
  int G, bits_mode;
  double thr;
  Ctrl* ctrl;                // Ctrl and scan partials: the batch's zeroed region
  unsigned long long* partials;
  uint8_t* types;            // the tensor's slice of the workspace (enc_ws_layout)
  uint32_t* sizes;
  uint64_t* item_off;
  EncSave* saves;
  uint16_t* hist;
};

struct EncBatch {
  const EncTensor* t;        // the class's tensors
  const uint64_t* start;     // [n + 1] exclusive prefix of this kernel's work per tensor
  uint32_t n;
};
struct NoBatch {};
template <class Batch>
constexpr bool kIsBatch = !std::is_same<Batch, NoBatch>::value;
__device__ __forceinline__ uint64_t batch_work(NoBatch, uint64_t single) { return single; }
__device__ __forceinline__ uint64_t batch_work(const EncBatch& B, uint64_t) { return B.start[B.n]; }

// A byte of the (rotated) chunk at byte position pos; words [0, rot_words) are rotated.
template <int G>
__device__ __forceinline__ uint32_t rot_byte_at(const uint8_t* __restrict__ in_c, uint32_t chunk_len, uint32_t rot_words,
                                                uint32_t pos) {
  const uint32_t wi = pos >> 2;
  if (wi >= rot_words) return in_c[pos];
  (void)chunk_len;
  const uint32_t w = rot_word<G>(__ldg(reinterpret_cast<const uint32_t*>(in_c) + wi));
  return (w >> (8 * (pos & 3))) & 0xFFu;
}

// =====================================================================================
// pass A1: histograms.  Pure streaming: every input byte is read once (128-bit loads, four in
// flight per thread), rotated, and counted with one shared-memory atomic.
//
// Counter layout rep[g][bin][col], col = lane % R, 32-bit counters: a warp's 32 atomics go to
// 32 / (32/R) distinct columns, so two lanes can only collide when they hold the same byte
// value -- and the address is one shift + one LOP3 from the loaded word (3 instructions per
// byte including the atomic; the first version spent 11).  Per stream quarter the columns are
// folded into hist[item][stream][256] (u16) in global memory for pass A2.
// =====================================================================================
// Columns per bin.  32 = one per lane: no two lanes of a warp ever meet in a bank (1 wavefront per
// atomic instead of 2), at 32 KiB of counters per plane; fp32 has four planes and keeps 16.
template <int G>
struct HistCfg {
  static constexpr int R = (G == 4) ? 16 : 32;
  static constexpr int kShift = (G == 4) ? 6 : 7;      // log2(R * 4): byte offset of a bin
};

template <int G>
struct HistSmem {
  uint32_t rep[G][256][HistCfg<G>::R];
};

// The whole kernel, inlined into k_encode_hist (B = NoBatch) and k_encode_hist_batch, which differ only in their
// launch bounds.
template <int G, class Batch>
__device__ __forceinline__ void encode_hist(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk, uint64_t K, int bits_mode,
                                            uint16_t* __restrict__ hist, Batch B) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  HistSmem<G>& S = *reinterpret_cast<HistSmem<G>*>(smem_raw);
  constexpr int R = HistCfg<G>::R;
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t col_bytes = (uint32_t)(lane % R) * 4;
  unsigned char* const col_p = reinterpret_cast<unsigned char*>(&S.rep[0][0][0]) + col_bytes;  // rep[0][0][lane % R]
  for (int i = tid; i < G * 256 * R; i += kEncThreads) (&S.rep[0][0][0])[i] = 0;
  __syncthreads();
  for (uint64_t w = blockIdx.x; w < batch_work(B, K); w += gridDim.x) {
    uint64_t c = w;
    if constexpr (kIsBatch<Batch>) {  // work = chunks
      const uint32_t i = batch_find(B.start, B.n, w);
      const EncTensor& T = B.t[i];
      in = T.in; n = T.n; chunk = T.chunk; K = T.K; bits_mode = T.bits_mode; hist = T.hist;
      c = w - B.start[i];
    }
    const uint8_t* in_c = in + c * (uint64_t)chunk;
    const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(n - c * (uint64_t)chunk) : chunk;
    const uint32_t rot_words = (bits_mode == 1 && G > 1) ? (chunk_len >> 2) : 0;
    const bool fast = (chunk_len % 64u) == 0;
    for (int q = 0; q < 4; q++) {
      // Two stream quarters share one fold: quarter q counts in the low (q even) or high (q odd) half
      // of the 32-bit counters.  A column receives at most 8 threads x 128 bytes = 1024 per quarter,
      // and a bin at most 32768 in total, so neither half overflows.
      const uint32_t inc = (q & 1) ? 0x10000u : 1u;
      if (fast) {
        const uint32_t qbytes = chunk_len >> 2;  // bytes of input per stream quarter
        const uint4* src = reinterpret_cast<const uint4*>(in_c + (uint64_t)q * qbytes);
        const uint32_t nvec = qbytes >> 4;
        // double-buffered: the next four vectors are in flight while the current four are counted
        uint4 v[4], nv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const uint32_t u = k * kEncThreads + tid;
          nv[k] = (u < nvec) ? __ldg(src + u) : make_uint4(0, 0, 0, 0);
        }
        for (uint32_t u0 = 0; u0 < nvec; u0 += 4 * kEncThreads) {
#pragma unroll
          for (int k = 0; k < 4; k++) v[k] = nv[k];
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const uint32_t u = u0 + (4 + k) * kEncThreads + tid;
            if (u < nvec) nv[k] = __ldg(src + u);
          }
#pragma unroll
          for (int k = 0; k < 4; k++) {
            if (u0 + k * kEncThreads + tid < nvec) {
              uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
              for (int i = 0; i < 4; i++) {
                if (rot_words) w[i] = rot_word<G>(w[i]);
#pragma unroll
                for (int b = 0; b < 4; b++) {
                  // byte b of the word -> address of its counter in THREE instructions: extract (PRMT with zeros),
                  // bin * (R * 4) + this lane's column (one multiply-add on the FMA pipe), shared-memory reduction
                  // with the plane as an immediate offset.  (Shift, mask | column, add the array base, ATOMS took four,
                  // and the kernel is bound by instruction issue)
                  const uint32_t byte = __byte_perm(w[i], 0u, 0x4440u | (uint32_t)b);
                  atomicAdd(reinterpret_cast<uint32_t*>(col_p + ((4 * i + b) % G) * (256 * R * 4) + byte * (uint32_t)(R * 4)), inc);
                }
              }
            }
          }
        }
      } else {
        for (int g = 0; g < G; g++) {
          const uint32_t pl = plane_len(chunk_len, G, g);
          const uint32_t seg = (pl + 3) >> 2;
          const uint32_t j0 = min(pl, (uint32_t)q * seg), j1 = (q == 3) ? pl : min(pl, j0 + seg);
          for (uint32_t j = j0 + tid; j < j1; j += kEncThreads)
            atomicAdd(&S.rep[g][rot_byte_at<G>(in_c, chunk_len, rot_words, j * G + g)][lane % R], inc);
        }
      }
      if ((q & 1) == 0) continue;
      __syncthreads();
      // fold the columns of each bin (and clear them); thread t owns bin t of every group
      for (int g = 0; g < G; g++) {
        uint32_t sum = 0;
#pragma unroll
        for (int r = 0; r < R; r++) {
          const int rr = (r + tid) % R;
          sum += S.rep[g][tid][rr];
          S.rep[g][tid][rr] = 0;
        }
        uint16_t* h = hist + (((uint64_t)g * K + c) * 4 + (q - 1)) * 256 + tid;
        h[0] = (uint16_t)(sum & 0xFFFFu);
        h[256] = (uint16_t)(sum >> 16);
      }
      __syncthreads();
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kEncThreads) k_encode_hist(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk,
                                                             uint64_t K, int bits_mode, uint16_t* __restrict__ hist) {
  encode_hist<G>(in, n, chunk, K, bits_mode, hist, NoBatch{});
}

// work = chunks.  Held to the CTAs per SM of the single-tensor kernel (two for one group, three -- the shared-memory
// limit -- for two and four): left alone the two-group form takes 111 registers instead of 80, only two CTAs fit,
// and a 16 GiB bf16 tensor codes 2-3 % slower.
template <int G>
__global__ void __launch_bounds__(kEncThreads, G == 1 ? 2 : 3) k_encode_hist_batch(EncBatch B) {
  encode_hist<G>(nullptr, 0, 0, 0, 0, nullptr, B);
}

// =====================================================================================
// pass A2: one warp per (group, chunk) item: everything the reference does per block after
// the histogram (huf_compress.c:671-724 + csrc/zipnn_core.c:371-385).
// =====================================================================================
constexpr uint64_t kScanItems = 2048;  // chunks of one group per k_encode_scan CTA

struct __align__(16) TableWarp {
  uint32_t total[256];
  uint8_t nb[256];
  uint8_t nzsym[256];
  TreeScratch tree;
};
constexpr int kTableWarps = 4;

// hist = this item's four per-stream histograms, u16[4][256] in global memory (read twice: totals, exact sizes)
// cap = the chunk size: the destination capacity the reference gives HUF_compress (zipnn_core.c:365-368)
__device__ void warp_block_decision(TableWarp& S, const uint16_t* __restrict__ hist, uint32_t plen, uint32_t cap, double thr,
                                    uint8_t* type_out, uint32_t* size_out, EncSave* save) {
  const int lane = threadIdx.x & 31;
  uint32_t* total = S.total;
  uint32_t largest = 0;
  int max_sym = -1;
  for (int s = lane; s < 256; s += 32) {
    const uint32_t t = (uint32_t)__ldg(hist + s) + __ldg(hist + 256 + s) + __ldg(hist + 512 + s) + __ldg(hist + 768 + s);
    total[s] = t;
    largest = max(largest, t);
    if (t) max_sym = s;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    largest = max(largest, __shfl_xor_sync(0xffffffffu, largest, o));
    max_sym = max(max_sym, __shfl_xor_sync(0xffffffffu, max_sym, o));
  }
  __syncwarp();
  uint32_t stored = 0;  // huf_block_decision: 0 = raw, 1 = RLE, else the coded block's size
  const int early = huf_early_out(largest, plen);
  if (early == 1) {
    stored = huf_block_decision(true, nullptr, 0, plen, cap, thr);  // RLE block of 1 byte (huf_compress.c:673)
    if (stored && lane == 0) {
      save->hdr[0] = (uint8_t)max_sym;
      save->hsize = 0;
    }
  }
  if (early == 2) {
    // ---- order the present symbols: count descending, symbol ascending ----
    TreeScratch& T = S.tree;
    uint8_t* nz = S.nzsym;
    int k = 0;
    for (int base = 0; base < 256; base += 32) {
      const int s = base + lane;
      const bool p = total[s] != 0;
      const uint32_t m = __ballot_sync(0xffffffffu, p);
      if (p) nz[k + __popc(m & ((1u << lane) - 1u))] = (uint8_t)s;
      k += __popc(m);
    }
    __syncwarp();
    for (int i = lane; i < k; i += 32) {
      const uint32_t c = total[nz[i]];
      int rank = 0;
      for (int j = 0; j < k; j++) {
        const uint32_t cj = total[nz[j]];
        rank += (cj > c) || (cj == c && j < i);
      }
      T.cnt[rank] = c;
      T.sym[rank] = nz[i];
    }
    __syncwarp();
    int lg = 0, hsize = -1;
    if (lane == 0) {
      const int want = fse_pick_log(kHufLogDefault, plen, (uint32_t)max_sym, 1);
      lg = huf_lengths_from_sorted(T, k - 1, want, S.nb);
      hsize = huf_write_table(T, S.nb, max_sym, lg);
    }
    lg = __shfl_sync(0xffffffffu, lg, 0);
    hsize = __shfl_sync(0xffffffffu, hsize, 0);
    __syncwarp();
    if (hsize > 0 && (uint32_t)hsize + 12 < plen) {
      uint32_t bits[4] = {0, 0, 0, 0};
      for (int s = lane; s <= max_sym; s += 32) {
        const uint32_t l = S.nb[s];
#pragma unroll
        for (int q = 0; q < 4; q++) bits[q] += (uint32_t)__ldg(hist + 256 * q + s) * l;
      }
#pragma unroll
      for (int q = 0; q < 4; q++)
#pragma unroll
        for (int o = 16; o; o >>= 1) bits[q] += __shfl_xor_sync(0xffffffffu, bits[q], o);
      // The capacity binds for one byte group, where it equals the plane length: a block that fits in
      // plen - 1 bytes can still be refused for the 8-byte slack of a bitstream.
      stored = huf_block_decision(false, bits, hsize, plen, cap, thr);
      if (stored) {
        for (int s = lane; s < 256; s += 32) save->nb[s] = S.nb[s];
        for (int i = lane; i < hsize; i += 32) save->hdr[i] = T.hdr[i];
        if (lane == 0) {
          save->hsize = (uint32_t)hsize;
          save->lg = (uint32_t)lg;
#pragma unroll
          for (int q = 0; q < 4; q++) save->sbytes[q] = (bits[q] >> 3) + 1;  // bitstream.h:254-260
        }
      }
    }
  }
  if (lane == 0) {
    *type_out = stored ? 1 : 0;
    *size_out = stored ? stored : plen;
  }
}

// One warp: item (g, c) of one tensor, item = g * K + c.
template <int G>
__device__ __forceinline__ void encode_table_item(TableWarp& S, const uint16_t* __restrict__ hist, uint64_t n, uint32_t chunk, uint64_t K,
                                                  double thr, uint8_t* types, uint32_t* sizes, EncSave* saves,
                                                  unsigned long long* partials, const int lane, uint64_t item) {
  {
    const int g = (int)(item / K);
    const uint64_t c = item - (uint64_t)g * K;
    const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(n - c * (uint64_t)chunk) : chunk;
    warp_block_decision(S, hist + item * 1024, plane_len(chunk_len, G, g), chunk, thr, types + item, sizes + item, saves + item);
    __syncwarp();
    // payload bytes of this group per block of kScanItems chunks: lets the scan run on many CTAs
    if (lane == 0) atomicAdd(partials + (uint64_t)g * ((K + kScanItems - 1) / kScanItems) + c / kScanItems, (unsigned long long)sizes[item]);
  }
}

template <int G>
__global__ void __launch_bounds__(kTableWarps * 32) k_encode_table(const uint16_t* __restrict__ hist, uint64_t n, uint32_t chunk,
                                                                   uint64_t K, double thr, uint8_t* types, uint32_t* sizes,
                                                                   EncSave* saves, unsigned long long* partials) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  TableWarp& S = reinterpret_cast<TableWarp*>(smem_raw)[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const uint64_t nitems = (uint64_t)G * K;
  for (uint64_t item = (uint64_t)blockIdx.x * kTableWarps + (threadIdx.x >> 5); item < nitems;
       item += (uint64_t)gridDim.x * kTableWarps)
    encode_table_item<G>(S, hist, n, chunk, K, thr, types, sizes, saves, partials, lane, item);
}

// =====================================================================================
// scan: sizes -> cumulative table (written into the stream), bases, item offsets, header.
// =====================================================================================
constexpr int kScanThreads = 256;
// (kScanItems = kScanThreads * 8 chunks of one group per CTA, declared above k_encode_table)

// One CTA per (group, block of kScanItems chunks).  The table kernel left the payload bytes of every
// such block in partials[g][blk]; a CTA adds up what lies in front of it (all blocks of the groups
// before, the earlier blocks of its own group), scans its own 2048 sizes (8 per thread) and writes its
// slice of the cumulative table, the item offsets and the type bytes.  CTA 0 also writes the header.
// CTA `bid` of one tensor's scan (bid < G * nblk).
__device__ __forceinline__ void encode_scan_block(const uint32_t* __restrict__ sizes, const uint8_t* __restrict__ types, int G, uint64_t K,
                                                  const uint8_t* __restrict__ hdr_dev, uint32_t hdr_len, uint8_t* out, uint64_t* item_off,
                                                  Ctrl* ctrl, const unsigned long long* __restrict__ partials, uint32_t bid) {
  __shared__ uint64_t warp_tot[kScanThreads / 32];
  __shared__ uint64_t red[kScanThreads / 32][3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint64_t nitems = (uint64_t)G * K;
  const uint64_t nblk = (K + kScanItems - 1) / kScanItems;
  const int g = (int)(bid / nblk);
  const uint64_t blk = bid - (uint64_t)g * nblk;
  // ---- what lies in front of this CTA: whole earlier groups, earlier blocks of this group, everything
  uint64_t s_groups = 0, s_blocks = 0, s_all = 0;
  for (uint64_t i = tid; i < (uint64_t)G * nblk; i += kScanThreads) {
    const uint64_t v = partials[i];
    const uint64_t gi = i / nblk;
    s_all += v;
    if (gi < (uint64_t)g) s_groups += v;
    if (gi == (uint64_t)g && i - gi * nblk < blk) s_blocks += v;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s_groups += __shfl_xor_sync(0xffffffffu, s_groups, o);
    s_blocks += __shfl_xor_sync(0xffffffffu, s_blocks, o);
    s_all += __shfl_xor_sync(0xffffffffu, s_all, o);
  }
  if (lane == 0) { red[warp][0] = s_groups; red[warp][1] = s_blocks; red[warp][2] = s_all; }
  __syncthreads();
  s_groups = s_blocks = s_all = 0;
  for (int w = 0; w < kScanThreads / 32; w++) { s_groups += red[w][0]; s_blocks += red[w][1]; s_all += red[w][2]; }
  const uint64_t payload0 = (uint64_t)hdr_len + 9 * nitems;
  const uint64_t base = payload0 + s_groups;  // first payload byte of group g
  // ---- this CTA's chunks: 8 consecutive ones per thread
  const uint64_t c_first = blk * kScanItems + (uint64_t)tid * 8;
  uint32_t v[8];
  uint64_t run = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    v[j] = (c_first + j < K) ? sizes[(uint64_t)g * K + c_first + j] : 0u;
    run += v[j];
  }
  uint64_t x = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[warp] = x;
  __syncthreads();
  uint64_t pre = s_blocks + x - run;
  for (int w = 0; w < warp; w++) pre += warp_tot[w];
  uint8_t* cum_out = out + hdr_len + nitems;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint64_t c = c_first + j;
    if (c < K) {
      const uint64_t i = (uint64_t)g * K + c;
      item_off[i] = base + pre;
      pre += v[j];
      st_u64_bytes(cum_out + 8 * i, pre);  // inclusive, counted from the start of the group
      out[hdr_len + i] = types[i];
    }
  }
  if (blk == 0 && tid == 0) {
    ctrl->base[g] = base;
    uint64_t tot = 0;
    for (uint64_t j = 0; j < nblk; j++) tot += partials[(uint64_t)g * nblk + j];
    ctrl->group_total[g] = tot;
  }
  if (bid == 0) {
    // python header with the total length patched in (csrc/zipnn_core.c:121)
    const uint64_t total = payload0 + s_all;
    for (uint32_t i = tid; i < hdr_len; i += kScanThreads) {
      uint8_t b = hdr_dev[i];
      if (i >= 24 && i < 32) b = (uint8_t)(total >> (8 * (i - 24)));
      out[i] = b;
    }
    if (tid == 0) ctrl->total_len = total;
  }
}

// The python header rides in the kernel's parameters (CUDA 12.1 and later take up to 32 KiB of them): no host-to-device
// copy in front of the encode kernels.
constexpr size_t kHdrMax = 4096;
struct EncHeader {
  uint8_t b[kHdrMax];
};

__global__ void __launch_bounds__(kScanThreads) k_encode_scan(const uint32_t* __restrict__ sizes, const uint8_t* __restrict__ types,
                                                              int G, uint64_t K, const __grid_constant__ EncHeader hdr,
                                                              uint32_t hdr_len, uint8_t* out, uint64_t* item_off, Ctrl* ctrl,
                                                              const unsigned long long* __restrict__ partials) {
  encode_scan_block(sizes, types, G, K, hdr.b, hdr_len, out, item_off, ctrl, partials, blockIdx.x);
}

// =====================================================================================
// pass B
// =====================================================================================
constexpr uint32_t kEncTile = kEncThreads * 16;             // plane bytes per tile (4096)
constexpr uint32_t kBitBufWords = (kEncTile * 11) / 32 + 8;  // worst-case tile bits + carry

struct WriteSmem {
  __align__(16) uint8_t tile[kEncTile + 16];
  uint32_t bitbuf[kBitBufWords];
  uint32_t code[256];  // val | nb << 16
  uint32_t warp_sum[kEncThreads / 32];
  EncSave save;
};

// Fill S.tile[0..cnt) with bytes [p0, p0+cnt) of plane g of the (rotated) chunk.
template <int G>
__device__ __forceinline__ void stage_tile(uint8_t* tile, const uint8_t* __restrict__ in_c, uint32_t chunk_len,
                                           uint32_t rot_words, int g, uint32_t p0, uint32_t cnt) {
  const int tid = threadIdx.x;
  const bool fast = ((p0 * G) % 16u) == 0 && (cnt % 16u) == 0 && ((p0 + cnt) * (uint32_t)G <= (chunk_len & ~3u));
  if (fast) {
    for (uint32_t u = tid; u < (cnt >> 4); u += kEncThreads) {
      const uint4* src = reinterpret_cast<const uint4*>(in_c + (uint64_t)(p0 + 16 * u) * G);
      uint32_t w[4 * G];
#pragma unroll
      for (int i = 0; i < G; i++) {
        const uint4 v = __ldg(src + i);
        w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
      }
      if (rot_words) {
#pragma unroll
        for (int i = 0; i < 4 * G; i++) w[i] = rot_word<G>(w[i]);
      }
      uint4 pv[G];
      split16<G>(w, pv);
      uint4 mine = pv[0];
#pragma unroll
      for (int k = 1; k < G; k++)
        if (g == k) mine = pv[k];
      *reinterpret_cast<uint4*>(tile + 16 * u) = mine;
    }
  } else {
    for (uint32_t j = tid; j < cnt; j += kEncThreads)
      tile[j] = (uint8_t)rot_byte_at<G>(in_c, chunk_len, rot_words, (p0 + j) * G + g);
  }
}

// Copy tile[0..cnt) to the (arbitrarily aligned) global address dst.
__device__ __forceinline__ void tile_to_global(const uint8_t* tile, uint8_t* dst, uint32_t cnt) {
  const int tid = threadIdx.x;
  const uint32_t head = min(cnt, (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15));
  if ((uint32_t)tid < head) dst[tid] = tile[tid];
  const uint32_t nvec = (cnt - head) >> 4;
  const uint32_t* t32 = reinterpret_cast<const uint32_t*>(tile);
  for (uint32_t v = tid; v < nvec; v += kEncThreads) {
    const uint32_t o = head + 16 * v;
    const uint32_t sh = (o & 3) * 8;
    const uint32_t* p = t32 + (o >> 2);
    const uint32_t a0 = p[0], a1 = p[1], a2 = p[2], a3 = p[3], a4 = p[4];  // tile has 16 B of slack
    *reinterpret_cast<uint4*>(dst + o) = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh),
                                                    __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
  }
  const uint32_t done = head + 16 * nvec;
  if ((uint32_t)tid < cnt - done) dst[done + tid] = tile[done + tid];
}

// Canonical code values from lengths, one warp (huf_compress.c:390-407).
template <bool kValHigh>
__device__ __forceinline__ void warp_build_codes(const uint8_t* nb, int lg, uint32_t* code) {
  const int lane = threadIdx.x & 31;
  uint32_t per_len[kHufLogMax + 1];
#pragma unroll
  for (int l = 0; l <= kHufLogMax; l++) per_len[l] = 0;
  for (int base = 0; base < 256; base += 32) {
    const int mine = nb[base + lane];
#pragma unroll
    for (int l = 1; l <= kHufLogMax; l++) per_len[l] += __popc(__ballot_sync(0xffffffffu, mine == l));
  }
  uint32_t start[kHufLogMax + 1];
  {
    uint32_t v = 0;
#pragma unroll
    for (int l = kHufLogMax; l >= 1; l--) {
      if (l <= lg) {
        start[l] = v;
        v = (v + per_len[l]) >> 1;
      } else {
        start[l] = 0;
      }
    }
  }
  for (int base = 0; base < 256; base += 32) {
    const int mine = nb[base + lane];
    uint32_t val = 0;
#pragma unroll
    for (int l = 1; l <= kHufLogMax; l++) {
      const uint32_t m = __ballot_sync(0xffffffffu, mine == l);
      if (mine == l) val = start[l] + __popc(m & ((1u << lane) - 1u));
      start[l] += __popc(m);
    }
    code[base + lane] = kValHigh ? ((val << 8) | (uint32_t)mine) : (val | ((uint32_t)mine << 16));
  }
}

template <int G, class Batch = NoBatch>
__global__ void __launch_bounds__(kEncThreads) k_encode_write(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk, uint64_t K,
                                                              int bits_mode, const uint8_t* __restrict__ types,
                                                              const uint32_t* __restrict__ sizes, const EncSave* __restrict__ saves,
                                                              const uint64_t* __restrict__ item_off, uint8_t* out,
                                                              int only_ragged, Batch B = {}) {
  __shared__ WriteSmem S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint64_t nitems = (uint64_t)G * K;
  // only_ragged: just the G items of the last chunk (launched with G blocks)
  const uint64_t first = only_ragged ? (uint64_t)blockIdx.x * K + (K - 1) : blockIdx.x;
  const uint64_t step = only_ragged ? nitems : gridDim.x;
  for (uint64_t w = first; w < batch_work(B, nitems); w += step) {
    uint64_t item = w;
    if constexpr (kIsBatch<Batch>) {
      // work = every item of a tensor whose chunk is under 64*G, the G items of its last chunk when that one
      // is not a multiple of 64*G (only_ragged is 0: the prefix already holds just those)
      const uint32_t i = batch_find(B.start, B.n, w);
      const EncTensor& T = B.t[i];
      in = T.in; n = T.n; chunk = T.chunk; K = T.K; bits_mode = T.bits_mode;
      types = T.types; sizes = T.sizes; saves = T.saves; item_off = T.item_off; out = T.out;
      const uint64_t j = w - B.start[i];
      item = (chunk % (64u * G) != 0) ? j : j * K + (K - 1);
    }
    const int g = (int)(item / K);
    const uint64_t c = item - (uint64_t)g * K;
    const uint8_t* in_c = in + c * (uint64_t)chunk;
    const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(n - c * (uint64_t)chunk) : chunk;
    if (only_ragged && chunk_len % (64u * G) == 0) continue;  // k_encode_write_warp takes those
    const uint32_t rot_words = (bits_mode == 1 && G > 1) ? (chunk_len >> 2) : 0;
    const uint32_t plen = plane_len(chunk_len, G, g);
    uint8_t* dest = out + item_off[item];
    const uint8_t type = types[item];
    const uint32_t size = sizes[item];
    if (plen == 0) continue;
    __syncthreads();
    if (type == 0) {
      for (uint32_t p0 = 0; p0 < plen; p0 += kEncTile) {
        const uint32_t cnt = min(kEncTile, plen - p0);
        stage_tile<G>(S.tile, in_c, chunk_len, rot_words, g, p0, cnt);
        __syncthreads();
        tile_to_global(S.tile, dest + p0, cnt);
        __syncthreads();
      }
      continue;
    }
    if (size == 1) {
      if (tid == 0) dest[0] = saves[item].hdr[0];
      continue;
    }
    // ---- Huffman block: table description, jump table, 4 bitstreams ----
    {
      const uint32_t* sv = reinterpret_cast<const uint32_t*>(saves + item);
      uint32_t* dv = reinterpret_cast<uint32_t*>(&S.save);
      for (int i = tid; i < (int)(sizeof(EncSave) / 4); i += kEncThreads) dv[i] = sv[i];
    }
    __syncthreads();
    const uint32_t hsize = S.save.hsize;
    if (warp == 0) warp_build_codes<false>(S.save.nb, (int)S.save.lg, S.code);
    if (warp == 1) {
      for (uint32_t i = lane; i < hsize; i += 32) dest[i] = S.save.hdr[i];
      if (lane < 3) {
        dest[hsize + 2 * lane] = (uint8_t)S.save.sbytes[lane];
        dest[hsize + 2 * lane + 1] = (uint8_t)(S.save.sbytes[lane] >> 8);
      }
    }
    __syncthreads();
    const uint32_t seg = (plen + 3) >> 2;
    uint32_t stream_at = hsize + 6;
    for (int i = 0; i < 4; i++) {
      const uint32_t s_begin = (uint32_t)i * seg;
      const uint32_t s_end = (i == 3) ? plen : s_begin + seg;
      uint8_t* gaddr = dest + stream_at;
      const uint32_t sbytes = S.save.sbytes[i];
      stream_at += sbytes;
      const uint32_t a = (uint32_t)((uintptr_t)gaddr & 3);
      uint32_t* gword = reinterpret_cast<uint32_t*>(gaddr - a);
      uint32_t B = 8 * a;       // bits placed so far, counted from the aligned word base
      uint32_t flushed = 0;     // whole words already written to global
      for (uint32_t w = tid; w < kBitBufWords; w += kEncThreads) S.bitbuf[w] = 0;
      __syncthreads();
      for (uint32_t p1 = s_end; p1 > s_begin;) {
        const uint32_t p0 = (p1 - s_begin > kEncTile) ? p1 - kEncTile : s_begin;
        const uint32_t cnt = p1 - p0;
        stage_tile<G>(S.tile, in_c, chunk_len, rot_words, g, p0, cnt);
        __syncthreads();
        // ---- this thread's 16 symbols, in emission order (last plane byte first) ----
        const uint32_t e0 = 16u * tid;
        const int nvalid = (int)min(16u, cnt > e0 ? cnt - e0 : 0u);
        uint64_t v[4] = {0, 0, 0, 0};
        uint32_t l[4] = {0, 0, 0, 0};
        if (nvalid == 16 && (cnt & 15u) == 0) {
          const uint4 q = *reinterpret_cast<const uint4*>(S.tile + (cnt - 16 - e0));
          const uint32_t wv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int k = 0; k < 16; k++) {
            const uint32_t sym = (wv[(15 - k) >> 2] >> (8 * ((15 - k) & 3))) & 0xFFu;
            const uint32_t cd = S.code[sym];
            v[k >> 2] |= (uint64_t)(cd & 0xFFFFu) << l[k >> 2];
            l[k >> 2] += cd >> 16;
          }
        } else {
          for (int k = 0; k < nvalid; k++) {
            const uint32_t cd = S.code[S.tile[cnt - 1 - (e0 + k)]];
            v[k >> 2] |= (uint64_t)(cd & 0xFFFFu) << l[k >> 2];
            l[k >> 2] += cd >> 16;
          }
        }
        const uint32_t mine = l[0] + l[1] + l[2] + l[3];
        // ---- block-wide exclusive scan of bit lengths ----
        uint32_t x = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
          if (lane >= o) x += y;
        }
        if (lane == 31) S.warp_sum[warp] = x;
        __syncthreads();
        uint32_t pre = 0, tile_bits = 0;
#pragma unroll
        for (int w = 0; w < kEncThreads / 32; w++) {
          const uint32_t t = S.warp_sum[w];
          if (w < warp) pre += t;
          tile_bits += t;
        }
        uint32_t off = (B - 32 * flushed) + pre + x - mine;
#pragma unroll
        for (int r = 0; r < 4; r++) {
          if (l[r]) {
            const uint32_t sh = off & 31, wi = off >> 5;
            const uint32_t lo32 = (uint32_t)v[r], hi32 = (uint32_t)(v[r] >> 32);
            const uint32_t w0 = lo32 << sh;
            const uint32_t w1 = __funnelshift_l(lo32, hi32, sh);
            const uint32_t w2 = sh ? (hi32 >> (32 - sh)) : 0u;
            if (w0) atomicOr(&S.bitbuf[wi], w0);
            if (w1) atomicOr(&S.bitbuf[wi + 1], w1);
            if (w2) atomicOr(&S.bitbuf[wi + 2], w2);
            off += l[r];
          }
        }
        __syncthreads();
        B += tile_bits;
        // ---- flush the words that are complete ----
        const uint32_t complete = (B >> 5) - flushed;
        for (uint32_t w = tid; w < complete; w += kEncThreads) {
          const uint32_t val = S.bitbuf[w];
          if (flushed + w == 0 && a != 0) {
            for (uint32_t bb = a; bb < 4; bb++) gaddr[bb - a] = (uint8_t)(val >> (8 * bb));
          } else {
            gword[flushed + w] = val;
          }
        }
        const uint32_t carry = S.bitbuf[complete];
        __syncthreads();
        for (uint32_t w = tid; w <= complete + 1 && w < kBitBufWords; w += kEncThreads) S.bitbuf[w] = 0;
        __syncthreads();
        if (tid == 0) S.bitbuf[0] = carry;
        flushed += complete;
        p1 = p0;
        __syncthreads();
      }
      // ---- end mark + the last (partial) bytes ----
      if (tid == 0) S.bitbuf[(B - 32 * flushed) >> 5] |= 1u << (B & 31);
      __syncthreads();
      {
        const uint32_t first_byte = max(4 * flushed, a);   // relative to the aligned base
        const uint32_t end_byte = a + sbytes;              // exclusive
        for (uint32_t bb = first_byte + tid; bb < end_byte; bb += kEncThreads) {
          const uint32_t rel = bb - 4 * flushed;
          gaddr[bb - a] = (uint8_t)(S.bitbuf[rel >> 2] >> (8 * (rel & 3)));
        }
      }
      __syncthreads();
    }
  }
}

// =====================================================================================
// pass B, regular chunks (chunk_len % (64*G) == 0): one CTA of 4 warps per chunk, warp s owns
// the s-th quarter of every byte plane -- exactly one huff0 bitstream of each coded plane
// (huf_compress.c:552-603) and a contiguous quarter of each raw plane.  The chunk is read
// once (128-bit loads, the next tile prefetched), split in registers, and every plane is
// finished by the same warp: no block-wide synchronisation after the per-chunk setup.
//   coded plane: 16 symbols per lane -> 4 runs of <= 44 bits, warp suffix scan of the bit
//                lengths (the last symbol is emitted first, huf_compress.c:474-499), OR into a
//                warp-private bit buffer whose words are aligned with the destination's
//                32-bit words, coalesced flush of the completed words;
//   raw plane  : 512 bytes staged in shared memory, written with aligned 128-bit stores
//                (funnel-shifted to the destination's alignment), byte stores at the edges.
// =====================================================================================
constexpr int kWbWarps = 4;
constexpr uint32_t kWbTile = 512;                          // plane bytes per warp step (16 per lane)
constexpr uint32_t kWbBitWords = (kWbTile * 11) / 32 + 4;  // worst-case tile bits + carry

// (lo, hi) = 4 bytes each of the two top byte planes of 4 elements; the element-level rotation
// [sign][exp8][mant] -> [exp8][sign][mant] (data_manipulation_dtype16.c:10-20, dtype32.c:39-49) becomes
// hi' = exp8 = hi << 1 | lo >> 7, lo' = sign | low 7 bits, per byte.
__device__ __forceinline__ void rotate_planes(uint32_t& lo, uint32_t& hi) {
  const uint32_t l = lo, h = hi;
  hi = ((h << 1) & 0xFEFEFEFEu) | ((l >> 7) & 0x01010101u);
  lo = (h & 0x80808080u) | (l & 0x7F7F7F7Fu);
}

struct WbItem {
  uint8_t* dest;
  uint32_t size;
  uint32_t hsize;
  uint32_t sbytes[4];
  uint32_t lg;
  uint32_t type;  // 0 raw, 1 coded (size 1 = RLE)
};

template <int G>
struct WbSmem {
  uint32_t code[G][256];                       // val << 8 | nb
  WbItem item[G];
  __align__(16) uint8_t nb[G][256];
  uint32_t bitbuf[kWbWarps][G][kWbBitWords];
  __align__(16) uint8_t stage[kWbWarps][kWbTile + 32];
};

// Per-stream bit writer state kept in registers by every lane of the warp (uniform values).
struct WbStream {
  uint8_t* gaddr;    // first byte of the bitstream in the output
  uint32_t a;        // gaddr & 3
  uint32_t B;        // bits placed so far, counted from the aligned word below gaddr
  uint32_t flushed;  // whole words already written
};

__device__ __forceinline__ void wb_flush(uint32_t* bitbuf, WbStream& st, int lane) {
  uint32_t* gword = reinterpret_cast<uint32_t*>(st.gaddr - st.a);
  const uint32_t complete = (st.B >> 5) - st.flushed;
  // a stream that starts in the middle of a word: bytes [a, 4) of its first word go out one by one
  const bool split_first = (st.flushed == 0 && st.a != 0);
  if (split_first && lane == 0 && complete > 0) {
    const uint32_t val = bitbuf[0];
    for (uint32_t bb = st.a; bb < 4; bb++) st.gaddr[bb - st.a] = (uint8_t)(val >> (8 * bb));
  }
  for (uint32_t w = lane; w < complete; w += 32) {
    const uint32_t val = bitbuf[w];
    bitbuf[w] = 0;  // cleared as it leaves; only lane 0 touches word 0 and word `complete` below
    if (!(split_first && w == 0)) gword[st.flushed + w] = val;
  }
  if (lane == 0 && complete > 0) {  // the partial word becomes word 0 of the next tile (after lane 0 cleared word 0 above)
    bitbuf[0] = bitbuf[complete];
    bitbuf[complete] = 0;
  }
  st.flushed += complete;
  __syncwarp();
}

template <int G, class Batch = NoBatch>
__global__ void __launch_bounds__(kWbWarps * 32) k_encode_write_warp(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk,
                                                                     uint64_t K, int bits_mode, const uint8_t* __restrict__ types,
                                                                     const uint32_t* __restrict__ sizes,
                                                                     const EncSave* __restrict__ saves,
                                                                     const uint64_t* __restrict__ item_off, uint8_t* out,
                                                                     Batch B = {}) {
  __shared__ WbSmem<G> S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint64_t w = blockIdx.x; w < batch_work(B, K); w += gridDim.x) {
    uint64_t c = w;
    if constexpr (kIsBatch<Batch>) {  // work = K chunks of every tensor whose chunk is a multiple of 64*G
      const uint32_t i = batch_find(B.start, B.n, w);
      const EncTensor& T = B.t[i];
      in = T.in; n = T.n; chunk = T.chunk; K = T.K; bits_mode = T.bits_mode;
      types = T.types; sizes = T.sizes; saves = T.saves; item_off = T.item_off; out = T.out;
      c = w - B.start[i];
    }
    const uint32_t chunk_len = (c == K - 1) ? (uint32_t)(n - c * (uint64_t)chunk) : chunk;
    if (chunk_len % (64u * G) != 0) continue;  // ragged tail: k_encode_write
    const uint8_t* in_c = in + c * (uint64_t)chunk;
    const uint32_t plen = chunk_len / G;
    const uint32_t seg = plen >> 2;
    const bool rot = (bits_mode == 1 && G > 1);
    __syncthreads();
    // ---- per-chunk setup: warp g prepares group g ----
    if (warp < G) {
      const int g = warp;
      const uint64_t item = (uint64_t)g * K + c;
      WbItem it;
      it.dest = out + item_off[item];
      it.type = types[item];
      it.size = sizes[item];
      it.hsize = 0;
      it.lg = 0;
      it.sbytes[0] = it.sbytes[1] = it.sbytes[2] = it.sbytes[3] = 0;
      if (it.type == 1 && it.size == 1) {
        if (lane == 0) it.dest[0] = saves[item].hdr[0];
      } else if (it.type == 1) {
        const EncSave* sv = saves + item;
        it.hsize = sv->hsize;
        it.lg = sv->lg;
#pragma unroll
        for (int q = 0; q < 4; q++) it.sbytes[q] = sv->sbytes[q];
        reinterpret_cast<uint2*>(S.nb[g])[lane] = reinterpret_cast<const uint2*>(sv->nb)[lane];
        __syncwarp();
        warp_build_codes<true>(S.nb[g], (int)it.lg, S.code[g]);
        for (uint32_t i = lane; i < it.hsize; i += 32) it.dest[i] = sv->hdr[i];
        if (lane < 3) {
          it.dest[it.hsize + 2 * lane] = (uint8_t)it.sbytes[lane];
          it.dest[it.hsize + 2 * lane + 1] = (uint8_t)(it.sbytes[lane] >> 8);
        }
      }
      if (lane == 0) S.item[g] = it;
    }
    __syncthreads();

    // ---- warp `warp` = stream index ----
    const int s = warp;
    WbStream st[G];
    uint32_t raw_shift[G];  // destination misalignment of the raw plane quarter (bytes, mod 16)
#pragma unroll
    for (int g = 0; g < G; g++) {
      const WbItem& it = S.item[g];
      st[g].gaddr = it.dest;
      st[g].a = st[g].B = st[g].flushed = 0;
      raw_shift[g] = 0;
      if (it.type == 1 && it.size > 1) {
        uint32_t at = it.hsize + 6;
        for (int q = 0; q < s; q++) at += it.sbytes[q];
        st[g].gaddr = it.dest + at;
        st[g].a = (uint32_t)((uintptr_t)st[g].gaddr & 3);
        st[g].B = 8 * st[g].a;
        for (uint32_t w = lane; w < kWbBitWords; w += 32) S.bitbuf[warp][g][w] = 0;
      } else if (it.type == 0) {
        st[g].gaddr = it.dest + (uint64_t)s * seg;
        raw_shift[g] = (uint32_t)((uintptr_t)st[g].gaddr & 15);
      }
    }
    __syncwarp();

    const uint8_t* src_s = in_c + (uint64_t)s * seg * G;
    const uint32_t ntiles = (seg + kWbTile - 1) / kWbTile;
    uint4 cur[G], nxt[G];
    {
      const uint32_t t0 = (ntiles - 1) * kWbTile;
      if (t0 + 16 * lane < seg) {
        const uint4* p = reinterpret_cast<const uint4*>(src_s + (uint64_t)(t0 + 16 * lane) * G);
#pragma unroll
        for (int i = 0; i < G; i++) nxt[i] = __ldg(p + i);
      }
    }
    // Tiles run from the end of the stream to its start (huff0 emits the last symbol first); only the
    // first one processed can be partial, so the others are compiled with `have` known to be true.
    auto do_tile = [&](auto full_tag, const uint32_t ti) {
      constexpr bool kFull = decltype(full_tag)::value;
      const uint32_t t0 = ti * kWbTile;
      const uint32_t cnt = kFull ? kWbTile : min(kWbTile, seg - t0);  // multiple of 16
      const bool have = kFull ? true : (16u * lane < cnt);
#pragma unroll
      for (int i = 0; i < G; i++) cur[i] = nxt[i];
      if (ti > 0) {  // prefetch the next (lower) tile, always full
        const uint4* p = reinterpret_cast<const uint4*>(src_s + (uint64_t)(t0 - kWbTile + 16 * lane) * G);
#pragma unroll
        for (int i = 0; i < G; i++) nxt[i] = __ldg(p + i);
      }
      uint4 pv[G];
      if (have) {
        uint32_t w[4 * G];
#pragma unroll
        for (int i = 0; i < G; i++) {
          w[4 * i] = cur[i].x; w[4 * i + 1] = cur[i].y; w[4 * i + 2] = cur[i].z; w[4 * i + 3] = cur[i].w;
        }
        split16<G>(w, pv);
        if (rot) {  // sign-bit rotation at plane level: 4 operations per 4 elements instead of 5 per word
          rotate_planes(pv[(G - 2) % G].x, pv[G - 1].x);
          rotate_planes(pv[(G - 2) % G].y, pv[G - 1].y);
          rotate_planes(pv[(G - 2) % G].z, pv[G - 1].z);
          rotate_planes(pv[(G - 2) % G].w, pv[G - 1].w);
        }
      }
#pragma unroll
      for (int g = 0; g < G; g++) {
        const uint32_t type = S.item[g].type, size = S.item[g].size;
        if (type == 0) {
          // ---- raw plane: 16 bytes per lane -> dest + t0 .. ----
          uint8_t* stg = S.stage[warp];
          if (have) *reinterpret_cast<uint4*>(stg + 16 * lane) = pv[g];
          __syncwarp();
          uint8_t* D = st[g].gaddr + t0;
          const uint32_t m = raw_shift[g];
          if (m == 0) {
            if (have) *reinterpret_cast<uint4*>(D + 16 * lane) = pv[g];
          } else {
            const uint32_t head = 16 - m;  // bytes before the first aligned destination block
            const uint32_t nblk = (cnt - head) >> 4;
            {  // every lane computes (the stage has 32 spare bytes behind the tile); only the store is conditional
              const uint4 a4 = *reinterpret_cast<const uint4*>(stg + 16 * lane);
              const uint4 b4 = *reinterpret_cast<const uint4*>(stg + 16 * lane + 16);
              const uint32_t wv[8] = {a4.x, a4.y, a4.z, a4.w, b4.x, b4.y, b4.z, b4.w};
              // 16 bytes starting `head` bytes into (a4, b4): the word part of the shift is uniform over
              // the warp, so it is a 4-way switch (4 funnel shifts) rather than 7 shifts + 9 selects
              const uint32_t bs = (head & 3) * 8;
              uint32_t o[4];
              switch (head >> 2) {
                case 0:
#pragma unroll
                  for (int i = 0; i < 4; i++) o[i] = __funnelshift_r(wv[i], wv[i + 1], bs);
                  break;
                case 1:
#pragma unroll
                  for (int i = 0; i < 4; i++) o[i] = __funnelshift_r(wv[i + 1], wv[i + 2], bs);
                  break;
                case 2:
#pragma unroll
                  for (int i = 0; i < 4; i++) o[i] = __funnelshift_r(wv[i + 2], wv[i + 3], bs);
                  break;
                default:
#pragma unroll
                  for (int i = 0; i < 4; i++) o[i] = __funnelshift_r(wv[i + 3], wv[i + 4], bs);
                  break;
              }
              if ((uint32_t)lane < nblk) *reinterpret_cast<uint4*>(D + head + 16 * lane) = make_uint4(o[0], o[1], o[2], o[3]);
            }
            if (kFull) {  // the 16 bytes around the 31 aligned blocks: head bytes in front, 16 - head behind
              if (lane < 16) {
                const uint32_t idx = (uint32_t)lane < head ? (uint32_t)lane : (kWbTile - 16u + (uint32_t)lane);
                D[idx] = stg[idx];
              }
            } else {
              if ((uint32_t)lane < head) D[lane] = stg[lane];
              const uint32_t done = head + 16 * nblk;
              if ((uint32_t)lane < cnt - done) D[done + lane] = stg[done + lane];
            }
          }
          __syncwarp();
        } else if (size > 1) {
          // ---- coded plane: this lane's 16 symbols, last byte first ----
          // Run r = symbols 4r..4r+3 = bytes 3,2,1,0 of word 3-r.  Table entries are val << 8 | nb;
          // the byte is turned into the table's byte offset with one shift + one mask, two codes are
          // joined in 32 bits (<= 22), two pairs in 64 (<= 44).
          const unsigned char* code = reinterpret_cast<const unsigned char*>(S.code[g]);
          uint64_t v[4] = {0, 0, 0, 0};
          uint32_t l[4] = {0, 0, 0, 0};
          if (have) {
            const uint32_t wv[4] = {pv[g].x, pv[g].y, pv[g].z, pv[g].w};
#pragma unroll
            for (int r = 0; r < 4; r++) {
              const uint32_t w = wv[3 - r];
              const uint32_t e3 = *reinterpret_cast<const uint32_t*>(code + ((w >> 22) & 0x3FCu));
              const uint32_t e2 = *reinterpret_cast<const uint32_t*>(code + ((w >> 14) & 0x3FCu));
              const uint32_t e1 = *reinterpret_cast<const uint32_t*>(code + ((w >> 6) & 0x3FCu));
              const uint32_t e0 = *reinterpret_cast<const uint32_t*>(code + ((w << 2) & 0x3FCu));
              const uint32_t n3 = e3 & 0xFFu, n2 = e2 & 0xFFu, n1 = e1 & 0xFFu, n0 = e0 & 0xFFu;
              const uint32_t hi = (e3 >> 8) | ((e2 >> 8) << n3);  // emitted first
              const uint32_t lo = (e1 >> 8) | ((e0 >> 8) << n1);
              const uint32_t lh = n3 + n2;
              v[r] = (uint64_t)hi | ((uint64_t)lo << lh);
              l[r] = lh + n1 + n0;
            }
          }
          const uint32_t mine = l[0] + l[1] + l[2] + l[3];
          uint32_t x = mine;  // suffix sum over lanes: lane 31 is emitted first
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_down_sync(0xffffffffu, x, o);
            if (lane + o < 32) x += y;
          }
          const uint32_t tile_bits = __shfl_sync(0xffffffffu, x, 0);
          uint32_t* bitbuf = S.bitbuf[warp][g];
          uint32_t off = (st[g].B - 32 * st[g].flushed) + (x - mine);
          // Branch-free: a run of <= 44 bits touches words wi, wi+1 (always written, OR of 0 is harmless,
          // an idle lane of the last partial tile ORs zeros at a valid offset) and, when it starts past
          // bit 20, wi+2 (predicated reduction, no branch around it).
          const uint32_t bitbuf_s = (uint32_t)__cvta_generic_to_shared(bitbuf);
#pragma unroll
          for (int r = 0; r < 4; r++) {
            const uint32_t sh = off & 31, sa = bitbuf_s + ((off >> 5) << 2);
            const uint32_t lo32 = (uint32_t)v[r], hi32 = (uint32_t)(v[r] >> 32);
            const uint32_t w0 = lo32 << sh;
            const uint32_t w1 = __funnelshift_l(lo32, hi32, sh);
            const uint32_t w2 = (hi32 >> 1) >> (31 - sh);
            asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(sa), "r"(w0) : "memory");
            asm volatile("red.shared.or.b32 [%0+4], %1;" ::"r"(sa), "r"(w1) : "memory");
            asm volatile("{ .reg .pred p; setp.ne.u32 p, %1, 0; @p red.shared.or.b32 [%0+8], %1; }" ::"r"(sa), "r"(w2) : "memory");
            off += l[r];
          }
          __syncwarp();
          st[g].B += tile_bits;
          wb_flush(bitbuf, st[g], lane);
        }
      }
        };
    do_tile(std::false_type{}, ntiles - 1);
    for (uint32_t ti = ntiles - 1; ti-- > 0;) do_tile(std::true_type{}, ti);
    // ---- end marks and the last partial bytes of every bitstream ----
#pragma unroll
    for (int g = 0; g < G; g++) {
      if (S.item[g].type == 1 && S.item[g].size > 1) {
        uint32_t* bitbuf = S.bitbuf[warp][g];
        if (lane == 0) bitbuf[(st[g].B - 32 * st[g].flushed) >> 5] |= 1u << (st[g].B & 31);
        __syncwarp();
        const uint32_t first_byte = max(4 * st[g].flushed, st[g].a);
        const uint32_t end_byte = st[g].a + S.item[g].sbytes[s];
        for (uint32_t bb = first_byte + lane; bb < end_byte; bb += 32) {
          const uint32_t rel = bb - 4 * st[g].flushed;
          st[g].gaddr[bb - st[g].a] = (uint8_t)(bitbuf[rel >> 2] >> (8 * (rel & 3)));
        }
        __syncwarp();
      }
    }
  }
}

// =====================================================================================
// batches: the table and scan kernels' bodies for many tensors of one byte-group class, one launch
// per kernel (the hist body and the write kernels take a batch through their `Batch` parameter).
// =====================================================================================
// work = G * K items, one warp each
template <int G>
__global__ void __launch_bounds__(kTableWarps * 32) k_encode_table_batch(EncBatch B) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  TableWarp& S = reinterpret_cast<TableWarp*>(smem_raw)[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const uint64_t total = B.start[B.n];
  for (uint64_t w = (uint64_t)blockIdx.x * kTableWarps + (threadIdx.x >> 5); w < total; w += (uint64_t)gridDim.x * kTableWarps) {
    const uint32_t i = batch_find(B.start, B.n, w);
    const EncTensor& T = B.t[i];
    encode_table_item<G>(S, T.hist, T.n, T.chunk, T.K, T.thr, T.types, T.sizes, T.saves, T.partials, lane, w - B.start[i]);
  }
}

// work = G * nblk scan CTAs; an empty tensor has one, which writes its header-only stream
__global__ void __launch_bounds__(kScanThreads) k_encode_scan_batch(EncBatch B) {
  const uint32_t i = batch_find(B.start, B.n, blockIdx.x);
  const EncTensor& T = B.t[i];
  if (T.K == 0) {  // reference: zero chunks -> the header alone, total length = header length
    for (uint32_t j = threadIdx.x; j < T.hdr_len; j += kScanThreads)
      T.out[j] = (j >= 24 && j < 32) ? (uint8_t)((uint64_t)T.hdr_len >> (8 * (j - 24))) : T.hdr[j];
    if (threadIdx.x == 0) T.ctrl->total_len = T.hdr_len;
    return;
  }
  encode_scan_block(T.sizes, T.types, T.G, T.K, T.hdr, T.hdr_len, T.out, T.item_off, T.ctrl, T.partials,
                    (uint32_t)(blockIdx.x - B.start[i]));
}

}  // namespace zb
