// zipnn_b200.cu -- C ABI (include/zipnn_b200.h) over the sm_90a kernels.
//
// Build:  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo \
//              -Xcompiler -fPIC -shared -o libzipnn_b200.so zipnn_b200.cu
#include "../../include/zipnn_b200.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <numeric>
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "decode_sync.cuh"
#include "encode.cuh"
#include "stage1.cuh"

using namespace zb;

namespace {

std::atomic<int> g_last_cuda_error{0};
std::atomic<unsigned long long> g_launches{0};

inline bool cuda_ok(cudaError_t e) {
  if (e != cudaSuccess) {
    g_last_cuda_error.store((int)e);
    return false;
  }
  return true;
}
#define ZB_CUDA(x)                          \
  do {                                      \
    if (!cuda_ok((x))) return ZIPNN_B200_E_CUDA; \
  } while (0)
#define ZB_LAUNCHED()                                       \
  do {                                                      \
    g_launches.fetch_add(1, std::memory_order_relaxed);     \
    if (!cuda_ok(cudaGetLastError())) return ZIPNN_B200_E_CUDA; \
  } while (0)

// ---- optional per-kernel timing (CUDA events on the launching stream) ----------------
// Off by default.  bench.py turns it on to attribute the step time to kernels; the events
// sit between launches on the same stream, so they do not change the schedule.
enum KernelId { kKDecodeMeta = 0, kKHufDecode, kKHufDecodePlanar, kKRegroup, kKEncodeStats, kKEncodeTable, kKEncodeScan, kKEncodeWrite, kKEncodeWriteRagged, kKSplit,
                kKRegroupPlanar, kKDecodeOverflow, kKHufDecodeSync, kKParseTables, kKCount };
const char* const kKernelNames[kKCount] = {"k_decode_meta", "k_huf_decode_fused", "k_huf_decode_planar", "k_regroup", "k_encode_hist", "k_encode_table",
                                           "k_encode_scan", "k_encode_write_warp", "k_encode_write_ragged", "k_split_planar", "k_regroup_planar", "k_decode_overflow", "k_huf_decode_sync", "k_parse_tables"};
struct TimedSpan {
  int id;
  cudaEvent_t a, b;
};
std::atomic<int> g_timing{0};
std::mutex g_timing_mu;
std::vector<TimedSpan> g_spans;
std::vector<cudaEvent_t> g_event_pool;

cudaEvent_t take_event() {
  cudaEvent_t e = nullptr;
  if (!g_event_pool.empty()) {
    e = g_event_pool.back();
    g_event_pool.pop_back();
  } else {
    cudaEventCreate(&e);
  }
  return e;
}
struct ScopedTimer {
  int id;
  cudaStream_t st;
  cudaEvent_t a = nullptr;
  ScopedTimer(int id_, cudaStream_t st_) : id(id_), st(st_) {
    if (g_timing.load(std::memory_order_relaxed)) {
      std::lock_guard<std::mutex> lk(g_timing_mu);
      a = take_event();
      cudaEventRecord(a, st);
    }
  }
  ~ScopedTimer() {
    if (a) {
      std::lock_guard<std::mutex> lk(g_timing_mu);
      cudaEvent_t b = take_event();
      cudaEventRecord(b, st);
      g_spans.push_back({id, a, b});
    }
  }
};

int sm_count_cached() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      return 132;
  }
  return cached;
}

// ---- tensor maps (TMA descriptors) ------------------------------------------------------
// cuTensorMapEncodeTiled lives in the driver; taken through the runtime so that the library
// links against nothing but cudart.  A driver without it only costs the fused decode kernel
// its bulk-copy path.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    (void)cudaGetLastError();
    return (EncodeTiledFn)p;
  }();
  return fn;
}
// bytes viewed as {inner, rows} with a row pitch of `pitch` bytes; box {box_inner, 32}
bool byte_map_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch, uint32_t box_inner, CUtensorMapSwizzle sw,
                 CUtensorMapL2promotion l2) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc || ((uintptr_t)base & 15) || (pitch & 15) || inner == 0 || rows == 0 || inner > 0xffffffffull || rows > 0xffffffffull) return false;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {pitch};
  cuuint32_t box[2] = {box_inner, 32};
  cuuint32_t es[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, l2,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Knobs {
  int tma = 2, grid_mode = 1, warps_per_sm = 0;  // tma: 1 = bulk-tensor stores of the output rows, 2 = bulk-tensor tiles for the side plane.
  long long sync_max = -1;  // chunks up to which k_huf_decode_sync replaces the one-thread-per-bitstream kernels (-1: default)
  long long slice_piece = -1;  // covering chunks above which a slice item is split into pieces (-1: kSyncTablesMaxChunks; tests lower it)
  size_t smem_pad = 0;
};
Knobs knobs() {
  Knobs k;
  if (const char* e = getenv("ZIPNN_B200_SLICE_PIECE_CHUNKS")) k.slice_piece = atoll(e);
  if (const char* e = getenv("ZIPNN_B200_TMA")) k.tma = atoi(e);
  if (const char* e = getenv("ZIPNN_B200_GRID_MODE")) k.grid_mode = atoi(e);
  if (const char* e = getenv("ZIPNN_B200_WARPS_PER_SM")) k.warps_per_sm = atoi(e);
  if (const char* e = getenv("ZIPNN_B200_SMEM_PAD")) k.smem_pad = (size_t)atoi(e);
  if (const char* e = getenv("ZIPNN_B200_SYNC_MAX")) k.sync_max = atoll(e);
  return k;
}

template <typename Kernel>
int resident_blocks(Kernel k, size_t smem) {
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, 32, smem) != cudaSuccess || nb < 1) nb = 1;
  return nb;
}

inline bool valid_layout(int num_buf, int bytes_mode, size_t chunk) {
  if (!(num_buf == 1 || num_buf == 2 || num_buf == 4)) return false;
  // reference: mode 10 for one or two groups (dtype16.c:44,81), 220 for four (dtype32.c:241)
  if (num_buf == 4 ? bytes_mode != 220 : bytes_mode != 10) return false;
  if (chunk == 0 || (chunk & (chunk - 1)) != 0 || chunk > (1ull << 31)) return false;
  if (chunk % (size_t)num_buf) return false;
  return true;
}

inline size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline uint64_t num_chunks(size_t n, size_t chunk) { return (n + chunk - 1) / chunk; }

// ---- decompress workspace layout ----
//   [Ctrl 256][ItemDesc G*K][mode u8 K][slot u32 K][rlist u32 K][olist u32 K][hlist u32 G*K][fill 64*G*K][planes slots*G*pstride]
// `planes` is only used by chunks the fused kernel cannot take (several coded groups, or the
// ragged last chunk).  The default size provides a pool of kDefaultSlots of them, decoded by
// whole-GPU kernels, plus kOverflowCtas more that belong to the persistent CTAs of
// k_decode_overflow, which take every further such chunk: any stream decodes with the default
// workspace.  The "full" size gives every chunk a pool slot (faster for streams that are all
// general chunks, e.g. fp32 tensors upcast from bf16).
constexpr uint64_t kDefaultSlots = 64;
constexpr uint64_t kSyncTablesMaxChunks = 16384;  // largest tensor the sync decoder can be asked to take (ZIPNN_B200_SYNC_MAX is clamped to it)
constexpr uint64_t kSyncDefaultMaxChunks = 3072;  // crossover with the one-thread-per-bitstream kernels for one- and two-plane types
                                                  // (H100 SXM at 400 W: they win up to 3072 chunks and lose from 3584 on)
struct DecWs {
  size_t items_off, mode_off, slot_off, rlist_off, olist_off, hlist_off, tables_off, fill_off, planes_off, pstride, fixed;
};
// table_chunks: chunks whose coded items may be queued for the per-bitstream-CTA decoder (default: all of a
// tensor it takes, none of a larger one; a slice piece: its covering chunk range)
inline DecWs dec_ws_layout(size_t orig, int G, size_t chunk, uint64_t table_chunks = UINT64_MAX) {
  DecWs L;
  const uint64_t K = num_chunks(orig, chunk);
  if (table_chunks == UINT64_MAX) table_chunks = K <= kSyncTablesMaxChunks ? K : 0;
  L.items_off = kCtrlBytes;
  L.mode_off = round_up(L.items_off + sizeof(ItemDesc) * (size_t)G * K, 256);
  L.slot_off = round_up(L.mode_off + K, 256);
  L.rlist_off = round_up(L.slot_off + 4 * K, 256);
  L.olist_off = round_up(L.rlist_off + 4 * K, 256);
  L.hlist_off = round_up(L.olist_off + 4 * K, 256);
  // parsed table descriptions for the per-bitstream-CTA decoder: only tensors it takes (K <= kSyncTablesMaxChunks)
  L.tables_off = round_up(L.hlist_off + 4 * (size_t)G * K, 256);
  L.fill_off = round_up(L.tables_off + sizeof(ItemTable) * (size_t)G * table_chunks, 256);
  L.planes_off = round_up(L.fill_off + (size_t)kFillBytes * G * K, 256);
  L.pstride = round_up(chunk / (size_t)G, 16) + 16;
  L.fixed = L.planes_off + 256;
  return L;
}

template <typename F>
int dispatch_G(int G, F&& f) {
  switch (G) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    default: return f(std::integral_constant<int, 4>());
  }
}

int read_ctrl_error(void* d_ws, cudaStream_t st) {
  uint32_t err = 0;
  ZB_CUDA(cudaMemcpyAsync(&err, d_ws, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  ZB_CUDA(cudaStreamSynchronize(st));
  if (err & kErrCorrupt) return ZIPNN_B200_E_CORRUPT;
  if (err & kErrUnsupported) return ZIPNN_B200_E_UNSUPPORTED;
  if (err & kErrWorkspace) return ZIPNN_B200_E_CAPACITY;
  return ZIPNN_B200_OK;
}

}  // namespace

extern "C" {

int zipnn_b200_version(void) { return 0x000200; }

const char* zipnn_b200_strerror(int s) {
  switch (s) {
    case ZIPNN_B200_OK: return "ok";
    case ZIPNN_B200_E_ARG: return "invalid argument";
    case ZIPNN_B200_E_CAPACITY: return "output or workspace too small";
    case ZIPNN_B200_E_CORRUPT: return "corrupt ZipNN stream";
    case ZIPNN_B200_E_CUDA: return "CUDA runtime error";
    case ZIPNN_B200_E_UNSUPPORTED: return "unsupported stream feature (Huffman table log 12)";
    default: return "unknown status";
  }
}

int zipnn_b200_last_cuda_error(void) { return g_last_cuda_error.load(); }
int zipnn_b200_sm_count(void) { return sm_count_cached(); }
unsigned long long zipnn_b200_launch_count(void) { return g_launches.load(); }

void zipnn_b200_timing_enable(int on) {
  std::lock_guard<std::mutex> lk(g_timing_mu);
  g_timing.store(on ? 1 : 0);
  for (auto& sp : g_spans) {
    g_event_pool.push_back(sp.a);
    g_event_pool.push_back(sp.b);
  }
  g_spans.clear();
}

int zipnn_b200_timing_kernel_count(void) { return kKCount; }
const char* zipnn_b200_timing_kernel_name(int id) { return (id >= 0 && id < kKCount) ? kKernelNames[id] : ""; }

int zipnn_b200_timing_collect(double* ms_total, unsigned long long* launches, int n) {
  if (!ms_total || !launches || n < kKCount) return ZIPNN_B200_E_ARG;
  ZB_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_timing_mu);
  for (int i = 0; i < n; i++) {
    ms_total[i] = 0;
    launches[i] = 0;
  }
  for (auto& sp : g_spans) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, sp.a, sp.b) == cudaSuccess) {
      ms_total[sp.id] += ms;
      launches[sp.id] += 1;
    }
    g_event_pool.push_back(sp.a);
    g_event_pool.push_back(sp.b);
  }
  g_spans.clear();
  return ZIPNN_B200_OK;
}

int zipnn_b200_compress_bound(size_t n, int num_buf, size_t chunk, size_t hdr_len, size_t* out) {
  if (!out || chunk == 0 || !(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  *out = hdr_len + 9 * (size_t)num_buf * num_chunks(n, chunk) + n;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decompress_workspace_size(size_t orig, int num_buf, size_t chunk, size_t* out) {
  if (!out || chunk == 0 || !(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  const DecWs L = dec_ws_layout(orig, num_buf, chunk);
  const uint64_t K = num_chunks(orig, chunk);
  const uint64_t slots = K <= kDefaultSlots ? K : kDefaultSlots + kOverflowCtas;
  *out = L.fixed + (size_t)slots * num_buf * L.pstride;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decompress_workspace_size_full(size_t orig, int num_buf, size_t chunk, size_t* out) {
  if (!out || chunk == 0 || !(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  const DecWs L = dec_ws_layout(orig, num_buf, chunk);
  *out = L.fixed + (size_t)num_chunks(orig, chunk) * num_buf * L.pstride;
  return ZIPNN_B200_OK;
}

// Fill a DecodeCfg for one tensor whose workspace slice is [ws, ws + ws_bytes).
static int fill_decode_cfg(DecodeCfg& cfg, const void* d_body, size_t body_len, int G, int bits_mode, size_t chunk, size_t orig, void* d_out,
                           uint8_t* ws, size_t ws_bytes, bool use_sync, uint64_t table_chunks = UINT64_MAX) {
  const uint64_t K = num_chunks(orig, chunk);
  if (body_len < 9ull * G * K) return ZIPNN_B200_E_CORRUPT;
  const DecWs L = dec_ws_layout(orig, G, chunk, table_chunks);
  if (ws_bytes < L.fixed) return ZIPNN_B200_E_CAPACITY;
  memset(&cfg, 0, sizeof(cfg));
  cfg.body = (const uint8_t*)d_body;
  cfg.out = (uint8_t*)d_out;
  cfg.body_len = body_len;
  cfg.G = G;
  cfg.K = K;
  cfg.chunk = (uint32_t)chunk;
  cfg.orig = orig;
  cfg.bits_mode = bits_mode;
  cfg.ctrl = (Ctrl*)ws;
  cfg.items = (ItemDesc*)(ws + L.items_off);
  cfg.mode = ws + L.mode_off;
  cfg.slot = (uint32_t*)(ws + L.slot_off);
  cfg.rlist = (uint32_t*)(ws + L.rlist_off);
  cfg.fill = ws + L.fill_off;
  cfg.planes = ws + L.planes_off;
  cfg.pstride = L.pstride;
  cfg.olist = (uint32_t*)(ws + L.olist_off);
  const uint64_t have = (ws_bytes - L.fixed) / ((size_t)G * L.pstride);
  if (have >= K) {
    cfg.max_slots = (uint32_t)K;
    cfg.ovf_slots = 0;
  } else if (have > kOverflowCtas) {
    cfg.max_slots = (uint32_t)(have - kOverflowCtas);
    cfg.ovf_slots = kOverflowCtas;
  } else {
    cfg.max_slots = (uint32_t)have;  // a caller-sized scratch below the documented minimum: overflow is an error
    cfg.ovf_slots = 0;
  }
  cfg.hlist = use_sync ? (uint32_t*)(ws + L.hlist_off) : nullptr;
  cfg.tables = (ItemTable*)(ws + L.tables_off);
  return ZIPNN_B200_OK;
}
static uint64_t sync_max_chunks(int G) {
  const Knobs kn = knobs();
  // four-plane types: the CTA's merge phase writes twice as much per decoded symbol, the crossover is lower
  // (fp32 on the same H100: between 1536 and 2048 chunks)
  const uint64_t dflt = G == 4 ? kSyncDefaultMaxChunks / 2 : kSyncDefaultMaxChunks;
  return std::min<uint64_t>(kn.sync_max >= 0 ? (uint64_t)kn.sync_max : dflt, kSyncTablesMaxChunks);
}

int zipnn_b200_decompress(const void* d_body, size_t body_len, int num_buf, int bits_mode, int bytes_mode,
                          size_t chunk, size_t orig, void* d_out, void* d_ws, size_t ws_bytes, void* cuda_stream,
                          int check) {
  if (!valid_layout(num_buf, bytes_mode, chunk)) return ZIPNN_B200_E_ARG;
  if (orig == 0) return ZIPNN_B200_OK;
  if (!d_body || !d_out || !d_ws) return ZIPNN_B200_E_ARG;
  if (((uintptr_t)d_out & 15) || ((uintptr_t)d_ws & 255)) return ZIPNN_B200_E_ARG;
  const int G = num_buf;
  const uint64_t K = num_chunks(orig, chunk);
  cudaStream_t st = (cudaStream_t)cuda_stream;
  // Small and medium tensors: one CTA per bitstream (decode_sync.cuh) instead of one thread per bitstream.
  // The one-thread kernels take about the same time for anything up to ~20 000 chunks (a bitstream is serial);
  // the per-bitstream CTAs cost time in proportion to K, so they win below the crossover.
  const bool use_sync = K <= sync_max_chunks(G);
  DecodeCfg cfg;
  {
    const int rc = fill_decode_cfg(cfg, d_body, body_len, G, bits_mode, chunk, orig, d_out, (uint8_t*)d_ws, ws_bytes, use_sync);
    if (rc) return rc;
  }
  const Knobs kn = knobs();
  const uint64_t nitems = (uint64_t)G * K;

  ZB_CUDA(cudaMemsetAsync(cfg.ctrl, 0, kCtrlBytes, st));
  {
    const int threads = 128;
    const int blocks = (int)std::min<uint64_t>((K + threads - 1) / threads, 4096);
    ScopedTimer tm(kKDecodeMeta, st);
    k_decode_meta<<<blocks, threads, 0, st>>>(cfg);
    ZB_LAUNCHED();
  }
  if (use_sync) {
    static bool attr_done[5] = {false, false, false, false, false};
    int rc = dispatch_G(G, [&](auto g) -> int {
      constexpr int GG = decltype(g)::value;
      if (!attr_done[GG]) {
        ZB_CUDA(cudaFuncSetAttribute(k_huf_decode_sync<GG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyncSmemBytes));
        attr_done[GG] = true;
      }
      static const int nb = [] {
        int v = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_huf_decode_sync<GG>, kSyncThreads, kSyncSmemBytes) != cudaSuccess || v < 1) v = 1;
        return v;
      }();
      const unsigned grid = (unsigned)std::min<uint64_t>(4 * nitems, (uint64_t)nb * sm_count_cached());
      {
        ScopedTimer tp(kKParseTables, st);
        k_parse_tables<<<(unsigned)((nitems + kParseWarps - 1) / kParseWarps), kParseWarps * 32, 0, st>>>(cfg);
        ZB_LAUNCHED();
      }
      ScopedTimer tm(kKHufDecodeSync, st);
      k_huf_decode_sync<GG><<<grid, kSyncThreads, kSyncSmemBytes, st>>>(cfg, (uint8_t*)d_out);
      ZB_LAUNCHED();
      return ZIPNN_B200_OK;
    });
    if (rc) return rc;
  } else {
    {
      const uint64_t groups = (K + kDecItemsPerWarp - 1) / kDecItemsPerWarp;
      if (groups > 0x7fffffffull) return ZIPNN_B200_E_ARG;
      // Short-code planes (the exponent plane of the rotated types, ~2.6 bits per symbol) use
      // conflict-free private 5-bit table columns and a ~1000-entry tail pool (8 chunks x ~64 entries
      // for the codes longer than 5 bits, so 2x slack).  fp16 / fp8 planes (6-7 bits per symbol, 90-150
      // entries of > 8 bits per chunk) keep the shared 8-bit primaries.  A chunk whose tail does not
      // fit the pool takes the general path.
      const bool short_codes = (G >= 2 && bits_mode == 1);
      // ---- tensor maps for the bulk-copy path (decode.cuh, "Kernel 2b") ----
      TmaMaps maps;
      memset(&maps, 0, sizeof(maps));
      cfg.tma_flags = 0;
      cfg.k_full = orig / chunk;
      const uint64_t last_len = orig - cfg.k_full * chunk;
      uint64_t at = 9ull * G * K;
      for (int g = 0; g < 3; g++) {
        cfg.side_pred[g] = at;
        cfg.side_r0[g] = (uint32_t)(((uintptr_t)d_body + at) & 15);
        if (g < G) at += cfg.k_full * (chunk / G) + plane_len((uint32_t)last_len, G, g);
      }
      if (cfg.k_full >= (uint64_t)kDecItemsPerWarp && chunk >= 2048 && (chunk / 4) * 4 == chunk) {
        if (byte_map_2d(&maps.out, d_out, chunk / 4, 4 * cfg.k_full, chunk / 4, 128, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE)) {
          cfg.tma_flags |= kTmaOut;
        if (G == 2) {
          // the raw byte plane of group 0 as rows of one quarter plane each, 16 bytes longer than the pitch: a box
          // starts at the 16-byte boundary below the byte it needs (the payload is not aligned inside the stream)
          const uint64_t seg = chunk / G / 4;
          const uint8_t* base = (const uint8_t*)d_body + cfg.side_pred[0] - cfg.side_r0[0];
          if (seg >= 64 && body_len >= cfg.side_pred[0] + 4 * cfg.k_full * seg &&
              byte_map_2d(&maps.side[0], base, seg + 16, 4 * cfg.k_full, seg, FusedGeom<2>::kTileRow, CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
            cfg.tma_flags |= kTmaSide;
        }
        }
      }
      // tuning knobs for experiments (tools/decode_probe.py); unset in normal use
      cfg.tma_flags &= (uint32_t)kn.tma;
      if (getenv("ZIPNN_B200_DEBUG")) fprintf(stderr, "[zipnn_b200] fused decode: K=%llu k_full=%llu tma_flags=%u side_r0=%u encoder=%p\n", (unsigned long long)K,
                                              (unsigned long long)cfg.k_full, cfg.tma_flags, cfg.side_r0[0], (void*)tensor_map_encoder());
      ScopedTimer tm(kKHufDecode, st);
      int rc = dispatch_G(G, [&](auto g) -> int {
        constexpr int GG = decltype(g)::value;
        const int sms = sm_count_cached();
        auto grid_for = [&](int nb) -> unsigned {
          if (kn.grid_mode == 1) return (unsigned)groups;                            // one CTA per chunk group
          if (kn.warps_per_sm > 0) nb = std::min(nb, kn.warps_per_sm);
          return (unsigned)std::min<uint64_t>(groups, (uint64_t)nb * sms);          // persistent
        };
        if (short_codes) {
          const size_t smem = fused_smem_bytes<GG>(5) + kn.smem_pad;
          const int nb = resident_blocks(k_huf_decode_fused<GG, 5>, smem);
          k_huf_decode_fused<GG, 5><<<grid_for(nb), 32, smem, st>>>(cfg, (uint8_t*)d_out, maps);
        } else {
          const size_t smem = fused_smem_bytes<GG>(0) + kn.smem_pad;
          const int nb = resident_blocks(k_huf_decode_fused<GG, 0>, smem);
          k_huf_decode_fused<GG, 0><<<grid_for(nb), 32, smem, st>>>(cfg, (uint8_t*)d_out, maps);
        }
        ZB_LAUNCHED();
        return ZIPNN_B200_OK;
      });
      if (rc) return rc;
    }
    {
      const uint64_t warps = (nitems + kDecItemsPerWarp - 1) / kDecItemsPerWarp;
      if (warps > 0x7fffffffull) return ZIPNN_B200_E_ARG;
      ScopedTimer tm(kKHufDecodePlanar, st);
      k_huf_decode_planar<<<(unsigned)warps, 32, sizeof(DecodeSmem), st>>>(cfg);
      ZB_LAUNCHED();
    }
  }
  {
    const uint32_t tiles_per_chunk = (uint32_t)((chunk + kMergeTile - 1) / kMergeTile);
    const uint64_t ntiles = K * tiles_per_chunk;
    const int blocks = (int)std::min<uint64_t>(ntiles, (uint64_t)sm_count_cached() * 16);
    ScopedTimer tm(kKRegroup, st);
    int rc = dispatch_G(G, [&](auto g) -> int {
      k_regroup<decltype(g)::value><<<blocks, kMergeThreads, 0, st>>>(cfg, (uint8_t*)d_out);
      ZB_LAUNCHED();
      return ZIPNN_B200_OK;
    });
    if (rc) return rc;
  }
  if (cfg.ovf_slots) {
    ScopedTimer tm(kKDecodeOverflow, st);
    int rc = dispatch_G(G, [&](auto g) -> int {
      k_decode_overflow<decltype(g)::value><<<cfg.ovf_slots, kMergeThreads, sizeof(DecodeSmem), st>>>(cfg, (uint8_t*)d_out);
      ZB_LAUNCHED();
      return ZIPNN_B200_OK;
    });
    if (rc) return rc;
  }
  if (check) return read_ctrl_error(d_ws, st);
  return ZIPNN_B200_OK;
}

// ---- batches: every small/medium tensor of a checkpoint shard in ONE launch per kernel ------------------
// Workspace: [256 B: error word][DecodeCfg n][chunk_start n+1][item_start n+1][tile_start n+1][per-tensor slices]
static size_t batch_header_bytes(int n) {
  return round_up(256 + sizeof(DecodeCfg) * (size_t)n + 3 * sizeof(uint64_t) * ((size_t)n + 1), 256);
}
static size_t batch_slice_bytes(const zipnn_b200_batch_item& it) {
  size_t w = 0;
  if (it.orig == 0) return 0;
  zipnn_b200_decompress_workspace_size(it.orig, it.num_buf, it.chunk, &w);
  return round_up(w, 256);
}

int zipnn_b200_decompress_batch_workspace_size(const zipnn_b200_batch_item* items, int n, size_t* out) {
  if (!out || n < 0 || (n && !items)) return ZIPNN_B200_E_ARG;
  size_t total = batch_header_bytes(n);
  for (int i = 0; i < n; i++) {
    if (!valid_layout(items[i].num_buf, items[i].bytes_mode, items[i].chunk)) return ZIPNN_B200_E_ARG;
    total += batch_slice_bytes(items[i]);
  }
  *out = total;
  return ZIPNN_B200_OK;
}

static int run_batch_kernels(const std::vector<DecodeCfg>& cfgs, const std::vector<uint64_t>& starts, int n, uint8_t* ws, uint64_t max_ovf,
                             cudaStream_t st, BatchCfg& B);

int zipnn_b200_decompress_batch(const zipnn_b200_batch_item* items, int n, void* d_ws, size_t ws_bytes, void* cuda_stream, int check) {
  if (n < 0 || (n && !items) || !d_ws || ((uintptr_t)d_ws & 255)) return ZIPNN_B200_E_ARG;
  if (n == 0) return ZIPNN_B200_OK;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  uint8_t* ws = (uint8_t*)d_ws;
  const size_t hdr = batch_header_bytes(n);
  if (ws_bytes < hdr) return ZIPNN_B200_E_CAPACITY;
  std::vector<DecodeCfg> cfgs((size_t)n);
  std::vector<uint64_t> starts(3 * ((size_t)n + 1), 0);
  uint64_t* chunk_start = starts.data();
  uint64_t* item_start = chunk_start + (n + 1);
  uint64_t* tile_start = item_start + (n + 1);
  size_t at = hdr;
  std::vector<int> big;  // tensors that go through the single-tensor path on the same stream
  uint64_t max_ovf = 0;
  ZB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
  for (int i = 0; i < n; i++) {
    const zipnn_b200_batch_item& it = items[i];
    if (!valid_layout(it.num_buf, it.bytes_mode, it.chunk)) return ZIPNN_B200_E_ARG;
    const size_t slice = batch_slice_bytes(it);
    if (at + slice > ws_bytes) return ZIPNN_B200_E_CAPACITY;
    chunk_start[i + 1] = chunk_start[i];
    item_start[i + 1] = item_start[i];
    tile_start[i + 1] = tile_start[i];
    memset(&cfgs[i], 0, sizeof(DecodeCfg));
    cfgs[i].ctrl = (Ctrl*)ws;  // (never raised: an empty tensor has no kernel work)
    if (it.orig == 0) continue;
    if (!it.d_body || !it.d_out || ((uintptr_t)it.d_out & 15)) return ZIPNN_B200_E_ARG;
    const uint64_t K = num_chunks(it.orig, it.chunk);
    const bool small = K <= sync_max_chunks(it.num_buf);
    const int rc = fill_decode_cfg(cfgs[i], it.d_body, it.body_len, it.num_buf, it.bits_mode, it.chunk, it.orig, it.d_out, ws + at, slice, small);
    if (rc) return rc;
    ZB_CUDA(cudaMemsetAsync(ws + at, 0, kCtrlBytes, st));
    if (small) {
      chunk_start[i + 1] += K;
      item_start[i + 1] += 4ull * it.num_buf * K;
      tile_start[i + 1] += K * ((it.chunk + kMergeTile - 1) / kMergeTile);
      max_ovf = std::max<uint64_t>(max_ovf, cfgs[i].ovf_slots);
    } else {
      big.push_back(i);
    }
    at += slice;
  }
  BatchCfg B;
  {
    const int rc = run_batch_kernels(cfgs, starts, n, ws, max_ovf, st, B);
    if (rc) return rc;
  }
  for (int i : big) {
    const zipnn_b200_batch_item& it = items[i];
    const int rc = zipnn_b200_decompress(it.d_body, it.body_len, it.num_buf, it.bits_mode, it.bytes_mode, it.chunk, it.orig, it.d_out,
                                         (void*)cfgs[i].ctrl, batch_slice_bytes(it), st, 0);
    if (rc) return rc;
  }
  k_batch_errors<<<1, 256, 0, st>>>(B);
  ZB_LAUNCHED();
  if (check) return read_ctrl_error(d_ws, st);
  return ZIPNN_B200_OK;
}

// ---- slices: a box of each stream's decoded bytes, by the batch kernels -------------------------------------
namespace {
struct SlicePiece {
  int item;
  uint64_t base, rows, pitch, len, out_off, c0, c1;  // the piece's box, where its output starts, its covering chunks
};
uint64_t slice_piece_limit() {
  const Knobs kn = knobs();
  return kn.slice_piece >= 0 ? std::max<uint64_t>(2, (uint64_t)kn.slice_piece) : kSyncTablesMaxChunks;
}
// Checks item i and appends its pieces: the box, split so that no piece covers more than `limit` chunks -- by rows,
// or by bytes at chunk boundaries (moved by less than 16 bytes) when the box is one run -- with every piece's output
// on a 16-byte boundary.
int slice_pieces(const zipnn_b200_slice_item& it, int i, uint64_t limit, std::vector<SlicePiece>& out) {
  if (!valid_layout(it.num_buf, it.bytes_mode, it.chunk)) return ZIPNN_B200_E_ARG;
  if (it.rows == 0 || it.len == 0) return ZIPNN_B200_OK;
  if (it.base > it.orig || it.len > it.orig - it.base) return ZIPNN_B200_E_ARG;
  if (it.rows > 1 && (it.len > it.pitch || it.rows - 1 > (it.orig - it.base - it.len) / it.pitch)) return ZIPNN_B200_E_ARG;
  if (!it.d_body || !it.d_out || ((uintptr_t)it.d_out & 15)) return ZIPNN_B200_E_ARG;
  const uint64_t chunk = it.chunk;
  auto push = [&](uint64_t base, uint64_t rows, uint64_t pitch, uint64_t len, uint64_t off) {
    if (rows == 1) pitch = round_up(len, 16);  // (one row: the pitch only has to keep the store path's invariants)
    out.push_back({i, base, rows, pitch, len, off, base / chunk, (base + (rows - 1) * pitch + len + chunk - 1) / chunk});
  };
  auto run = [&](uint64_t b, uint64_t e, uint64_t off) {  // bytes [b, e) to output offset off (16-byte aligned)
    const uint64_t unit = std::max<uint64_t>(chunk, 16);
    // units per piece; at least one, also when limit * chunk < 16 (chunks under 8 bytes with a small limit), where
    // such a piece covers more than `limit` chunks (its tables are sized by its own chunk range)
    const uint64_t per = limit * chunk / unit;
    const uint64_t step = per > 1 ? per - 1 : 1;
    const uint64_t delta = b & 15;  // split points p = b (mod 16) keep off + (p - b) aligned
    while (b < e) {
      const uint64_t p = std::min<uint64_t>(e, (b / unit + step) * unit + delta);
      push(b, 1, 0, p - b, off);
      off += p - b;
      b = p;
    }
  };
  if (it.rows == 1 || it.pitch == it.len) {
    run(it.base, it.base + it.rows * it.len, 0);
    return ZIPNN_B200_OK;
  }
  const uint64_t m = 16 / std::gcd<uint64_t>(it.len, 16);  // rows per piece come in multiples of m: piece outputs start at r * len
  const uint64_t span = (limit - 1) * chunk;                // what a piece may span and still cover at most `limit` chunks
  uint64_t R = span >= it.len ? (span - it.len) / it.pitch + 1 : 0;
  R = R / m * m;
  if (R == 0 && m == 1) {  // rows longer than a piece: each row on its own
    for (uint64_t r = 0; r < it.rows; r++) run(it.base + r * it.pitch, it.base + r * it.pitch + it.len, r * it.len);
    return ZIPNN_B200_OK;
  }
  R = std::max(R, m);  // (pieces past the limit only when 16 rows of an odd row length span more than it; their tables are sized to fit)
  for (uint64_t r0 = 0; r0 < it.rows; r0 += R) push(it.base + r0 * it.pitch, std::min(R, it.rows - r0), it.pitch, it.len, r0 * it.len);
  return ZIPNN_B200_OK;
}
int plan_slices(const zipnn_b200_slice_item* items, int n, std::vector<SlicePiece>& pieces) {
  if (n < 0 || (n && !items)) return ZIPNN_B200_E_ARG;
  const uint64_t limit = slice_piece_limit();
  for (int i = 0; i < n; i++) {
    const int rc = slice_pieces(items[i], i, limit, pieces);
    if (rc) return rc;
  }
  if (pieces.size() > 0x7fffffffull) return ZIPNN_B200_E_ARG;
  return ZIPNN_B200_OK;
}
size_t slice_piece_bytes(const zipnn_b200_slice_item& it, const SlicePiece& p) {
  const uint64_t kc = p.c1 - p.c0;
  const DecWs L = dec_ws_layout(it.orig, it.num_buf, it.chunk, kc);
  const uint64_t slots = kc <= kDefaultSlots ? kc : kDefaultSlots + kOverflowCtas;
  return round_up(L.fixed + (size_t)slots * it.num_buf * L.pstride, 256);
}
}  // namespace

int zipnn_b200_decompress_slices_workspace_size(const zipnn_b200_slice_item* items, int n, size_t* out) {
  if (!out) return ZIPNN_B200_E_ARG;
  std::vector<SlicePiece> pieces;
  const int rc = plan_slices(items, n, pieces);
  if (rc) return rc;
  size_t total = batch_header_bytes((int)pieces.size());
  for (const SlicePiece& p : pieces) total += slice_piece_bytes(items[p.item], p);
  *out = total;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decompress_slices(const zipnn_b200_slice_item* items, int n, void* d_ws, size_t ws_bytes, void* cuda_stream, int check) {
  if (!d_ws || ((uintptr_t)d_ws & 255)) return ZIPNN_B200_E_ARG;
  std::vector<SlicePiece> pieces;
  {
    const int rc = plan_slices(items, n, pieces);
    if (rc) return rc;
  }
  const int np = (int)pieces.size();
  if (np == 0) return ZIPNN_B200_OK;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  uint8_t* ws = (uint8_t*)d_ws;
  size_t at = batch_header_bytes(np);
  if (ws_bytes < at) return ZIPNN_B200_E_CAPACITY;
  std::vector<DecodeCfg> cfgs((size_t)np);
  std::vector<uint64_t> starts(3 * ((size_t)np + 1), 0);
  uint64_t* chunk_start = starts.data();
  uint64_t* item_start = chunk_start + (np + 1);
  uint64_t* tile_start = item_start + (np + 1);
  uint64_t max_ovf = 1;  // the overflow kernel always runs (its CTAs return at once when no piece has overflow slots): a fixed launch count
  ZB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
  for (int j = 0; j < np; j++) {
    const SlicePiece& p = pieces[j];
    const zipnn_b200_slice_item& it = items[p.item];
    const size_t slice = slice_piece_bytes(it, p);
    if (at + slice > ws_bytes) return ZIPNN_B200_E_CAPACITY;
    const uint64_t kc = p.c1 - p.c0;
    DecodeCfg& cfg = cfgs[j];
    const int rc = fill_decode_cfg(cfg, it.d_body, it.body_len, it.num_buf, it.bits_mode, it.chunk, it.orig, (uint8_t*)it.d_out + p.out_off,
                                   ws + at, slice, true, kc);
    if (rc) return rc;
    cfg.box_base = p.base;
    cfg.box_rows = p.rows;
    cfg.box_pitch = p.pitch;
    cfg.box_len = p.len;
    cfg.box_step_rows = kBoxStep / p.pitch;
    cfg.box_step_cols = kBoxStep % p.pitch;
    cfg.box_fast = ((p.base | p.pitch | p.len) & 15) == 0;
    cfg.c0 = p.c0;
    ZB_CUDA(cudaMemsetAsync(ws + at, 0, kCtrlBytes, st));
    chunk_start[j + 1] = chunk_start[j] + kc;
    item_start[j + 1] = item_start[j] + 4ull * it.num_buf * kc;
    tile_start[j + 1] = tile_start[j] + kc * ((it.chunk + kMergeTile - 1) / kMergeTile);
    max_ovf = std::max<uint64_t>(max_ovf, cfg.ovf_slots);
    at += slice;
  }
  BatchCfg B;
  {
    const int rc = run_batch_kernels(cfgs, starts, np, ws, max_ovf, st, B);
    if (rc) return rc;
  }
  k_batch_errors<<<1, 256, 0, st>>>(B);
  ZB_LAUNCHED();
  if (check) return read_ctrl_error(d_ws, st);
  return ZIPNN_B200_OK;
}

// Descriptors to the device, then one launch of each kernel of the per-bitstream-CTA family for all of them.
static int run_batch_kernels(const std::vector<DecodeCfg>& cfgs, const std::vector<uint64_t>& starts, int n, uint8_t* ws, uint64_t max_ovf,
                             cudaStream_t st, BatchCfg& B) {
  const uint64_t* chunk_start = starts.data();
  const uint64_t* item_start = chunk_start + (n + 1);
  const uint64_t* tile_start = item_start + (n + 1);
  // descriptors to the device (pageable source: the copy is staged before the call returns)
  uint8_t* d_cfgs = ws + 256;
  uint8_t* d_starts = d_cfgs + sizeof(DecodeCfg) * (size_t)n;
  ZB_CUDA(cudaMemcpyAsync(d_cfgs, cfgs.data(), sizeof(DecodeCfg) * (size_t)n, cudaMemcpyHostToDevice, st));
  ZB_CUDA(cudaMemcpyAsync(d_starts, starts.data(), sizeof(uint64_t) * starts.size(), cudaMemcpyHostToDevice, st));
  B.cfgs = (const DecodeCfg*)d_cfgs;
  B.chunk_start = (const uint64_t*)d_starts;
  B.item_start = B.chunk_start + (n + 1);
  B.tile_start = B.item_start + (n + 1);
  B.n = (uint32_t)n;
  B.error_out = (uint32_t*)ws;
  const int sms = sm_count_cached();
  if (chunk_start[n]) {
    {
      const int threads = 128;
      const unsigned blocks = (unsigned)std::min<uint64_t>((chunk_start[n] + threads - 1) / threads, 4096);
      ScopedTimer tm(kKDecodeMeta, st);
      k_decode_meta_batch<<<blocks, threads, 0, st>>>(B);
      ZB_LAUNCHED();
    }
    {
      static bool attr_done = false;
      if (!attr_done) {
        ZB_CUDA(cudaFuncSetAttribute(k_huf_decode_sync_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyncSmemBytes));
        attr_done = true;
      }
      static const int nb = [] {
        int v = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_huf_decode_sync_batch, kSyncThreads, kSyncSmemBytes) != cudaSuccess || v < 1) v = 1;
        return v;
      }();
      const unsigned grid = (unsigned)std::min<uint64_t>(item_start[n], (uint64_t)nb * sms);
      {
        ScopedTimer tp(kKParseTables, st);
        k_parse_tables_batch<<<(unsigned)(((item_start[n] >> 2) + kParseWarps - 1) / kParseWarps), kParseWarps * 32, 0, st>>>(B);
        ZB_LAUNCHED();
      }
      ScopedTimer tm(kKHufDecodeSync, st);
      k_huf_decode_sync_batch<<<grid, kSyncThreads, kSyncSmemBytes, st>>>(B);
      ZB_LAUNCHED();
    }
    {
      const unsigned grid = (unsigned)std::min<uint64_t>(tile_start[n], (uint64_t)sms * 16);
      ScopedTimer tm(kKRegroup, st);
      k_regroup_batch<<<grid, kMergeThreads, 0, st>>>(B);
      ZB_LAUNCHED();
    }
    if (max_ovf) {
      ScopedTimer tm(kKDecodeOverflow, st);
      k_decode_overflow_batch<<<dim3((unsigned)max_ovf, (unsigned)n), kMergeThreads, sizeof(DecodeSmem), st>>>(B);
      ZB_LAUNCHED();
    }
  }
  return ZIPNN_B200_OK;
}

int zipnn_b200_split(const void* d_in, size_t n, int num_buf, int bits_mode, void* d_planes, size_t stride,
                     void* cuda_stream) {
  if (!(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  if (n == 0) return ZIPNN_B200_OK;
  if (!d_in || !d_planes || ((uintptr_t)d_in & 15) || ((uintptr_t)d_planes & 15) || (stride & 15)) return ZIPNN_B200_E_ARG;
  if (stride < (n + num_buf - 1) / num_buf) return ZIPNN_B200_E_CAPACITY;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const uint64_t units = n / (16ull * num_buf);
  const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((units + kStage1Threads - 1) / kStage1Threads,
                                                                    (uint64_t)sm_count_cached() * 32));
  ScopedTimer tm(kKSplit, st);
  return dispatch_G(num_buf, [&](auto g) -> int {
    k_split_planar<decltype(g)::value><<<blocks, kStage1Threads, 0, st>>>((const uint8_t*)d_in, n, bits_mode,
                                                                          (uint8_t*)d_planes, stride);
    ZB_LAUNCHED();
    return ZIPNN_B200_OK;
  });
}

int zipnn_b200_regroup(const void* d_planes, size_t stride, size_t n, int num_buf, int bits_mode, void* d_out,
                       void* cuda_stream) {
  if (!(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  if (n == 0) return ZIPNN_B200_OK;
  if (!d_out || !d_planes || ((uintptr_t)d_out & 15) || ((uintptr_t)d_planes & 15) || (stride & 15)) return ZIPNN_B200_E_ARG;
  if (stride < (n + num_buf - 1) / num_buf) return ZIPNN_B200_E_CAPACITY;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const uint64_t units = n / (16ull * num_buf);
  const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((units + kStage1Threads - 1) / kStage1Threads,
                                                                    (uint64_t)sm_count_cached() * 32));
  ScopedTimer tm(kKRegroupPlanar, st);
  return dispatch_G(num_buf, [&](auto g) -> int {
    k_regroup_planar<decltype(g)::value><<<blocks, kStage1Threads, 0, st>>>((const uint8_t*)d_planes, stride, n,
                                                                            bits_mode, (uint8_t*)d_out);
    ZB_LAUNCHED();
    return ZIPNN_B200_OK;
  });
}

}  // extern "C"

#include "api_compress.inc"
#include "api_host.inc"
