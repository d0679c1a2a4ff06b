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
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "decode_sync.cuh"
#include "encode.cuh"
#include "gather.cuh"
#include "matmul.cuh"
#include "matvec.cuh"
#include "select.cuh"
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

// ---- launch plans: what the runtime says about a kernel, asked once per device ----------------------------------
// Occupancy queries and cudaFuncSetAttribute cost host time on every call while the GPU waits for the launch, and
// their answers only change with the device (an attribute set on one device does not hold on another).  So each is
// asked once per (what, kernel, block size, shared memory, current device) and kept for the life of the process.
struct PlanKey {
  int what;  // kPlan* below
  const void* fn;
  int threads;
  size_t smem;
  int dev;
  bool operator==(const PlanKey& o) const { return what == o.what && fn == o.fn && threads == o.threads && smem == o.smem && dev == o.dev; }
};
struct PlanKeyHash {
  size_t operator()(const PlanKey& k) const {
    size_t h = std::hash<const void*>()(k.fn);
    for (size_t v : {(size_t)k.what, (size_t)k.threads, k.smem, (size_t)k.dev}) h = h * 1000003u ^ std::hash<size_t>()(v);
    return h;
  }
};
enum { kPlanSmCount = 0, kPlanBlocksPerSm, kPlanSmemAttr, kPlanFusedWarps };
std::mutex g_launch_mu;
std::unordered_map<PlanKey, int, PlanKeyHash> g_launch_plans;

// compute() > 0 is kept; anything else is returned and asked again next time (a failing runtime call is not cached).
template <typename F>
int launch_plan(int what, const void* fn, int threads, size_t smem, F&& compute) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = -1;
  const PlanKey key{what, fn, threads, smem, dev};
  {
    std::lock_guard<std::mutex> lk(g_launch_mu);
    auto it = g_launch_plans.find(key);
    if (it != g_launch_plans.end()) return it->second;
  }
  const int v = compute(dev);
  if (v > 0) {
    std::lock_guard<std::mutex> lk(g_launch_mu);
    g_launch_plans.emplace(key, v);
  }
  return v;
}

int sm_count_cached() {
  const int n = launch_plan(kPlanSmCount, nullptr, 0, 0, [](int dev) {
    int v = 0;
    return dev >= 0 && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess ? v : 0;
  });
  return n > 0 ? n : 132;
}

// CTAs of `threads` threads and `smem` bytes of dynamic shared memory resident on one SM of the current device (at
// least 1).  A kernel that needs more than 48 KiB must have had smem_attr() first.
template <typename Kernel>
int resident_blocks(Kernel k, size_t smem, int threads = 32) {
  const int nb = launch_plan(kPlanBlocksPerSm, (const void*)k, threads, smem, [&](int) {
    int v = 0;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k, threads, smem) == cudaSuccess ? v : 0;
  });
  return nb > 0 ? nb : 1;
}

// Raise the dynamic shared-memory limit of kernel k on the current device to `smem` (every caller passes the most
// the kernel ever launches with).  false: the runtime refused.
template <typename Kernel>
bool smem_attr(Kernel k, size_t smem) {
  return launch_plan(kPlanSmemAttr, (const void*)k, 0, smem, [&](int) {
    return cuda_ok(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) ? 1 : 0;
  }) > 0;
}

// A grid of at most `want` CTAs of kernel k that are all resident at once on the current device.  0: the runtime
// refused the shared-memory limit (smem_attr).
template <typename Kernel>
unsigned resident_grid(Kernel k, size_t smem, int threads, uint64_t want) {
  if (!smem_attr(k, smem)) return 0;
  return (unsigned)std::min<uint64_t>(want, (uint64_t)resident_blocks(k, smem, threads) * sm_count_cached());
}

// ---- small pinned host blocks for the results a call reads back -------------------------------------------------
// A device-to-host copy into pageable memory is staged by the driver and holds the host for longer; into pinned
// memory it is one DMA, and the caller waits once, on the stream.  Blocks are taken per call and given back, so
// calls on several threads never share one.
constexpr size_t kPinnedBlock = 4096;
std::mutex g_pinned_mu;
std::vector<void*> g_pinned_free;

struct PinnedBlock {
  void* p = nullptr;
  PinnedBlock() {
    {
      std::lock_guard<std::mutex> lk(g_pinned_mu);
      if (!g_pinned_free.empty()) {
        p = g_pinned_free.back();
        g_pinned_free.pop_back();
        return;
      }
    }
    if (!cuda_ok(cudaHostAlloc(&p, kPinnedBlock, cudaHostAllocPortable))) p = nullptr;
  }
  ~PinnedBlock() {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pinned_mu);
    g_pinned_free.push_back(p);
  }
  PinnedBlock(const PinnedBlock&) = delete;
  PinnedBlock& operator=(const PinnedBlock&) = delete;
};

// Events a call waits on (no timing), taken per call and given back.  An event can only be recorded on a stream of
// the device it was made on, so they are kept per device.
std::mutex g_wait_mu;
std::unordered_map<int, std::vector<cudaEvent_t>> g_wait_free;

struct WaitEvent {
  cudaEvent_t e = nullptr;
  int dev = -1;
  WaitEvent() {
    if (!cuda_ok(cudaGetDevice(&dev))) return;
    {
      std::lock_guard<std::mutex> lk(g_wait_mu);
      std::vector<cudaEvent_t>& v = g_wait_free[dev];
      if (!v.empty()) {
        e = v.back();
        v.pop_back();
        return;
      }
    }
    if (!cuda_ok(cudaEventCreateWithFlags(&e, cudaEventDisableTiming))) e = nullptr;
  }
  ~WaitEvent() {
    if (!e) return;
    std::lock_guard<std::mutex> lk(g_wait_mu);
    g_wait_free[dev].push_back(e);
  }
  WaitEvent(const WaitEvent&) = delete;
  WaitEvent& operator=(const WaitEvent&) = delete;
};

// `n` <= kPinnedBlock bytes of device memory at d_src to host memory at h_dst, after the work enqueued on st before.
int read_back(void* h_dst, const void* d_src, size_t n, cudaStream_t st) {
  PinnedBlock b;
  if (!b.p) return ZIPNN_B200_E_CUDA;
  ZB_CUDA(cudaMemcpyAsync(b.p, d_src, n, cudaMemcpyDeviceToHost, st));
  ZB_CUDA(cudaStreamSynchronize(st));
  memcpy(h_dst, b.p, n);
  return ZIPNN_B200_OK;
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
  int tma = 2;  // 1 = bulk-tensor stores of the output rows, 2 = bulk-tensor tiles for the side plane
  // The fused decode's launch (launch_fused): 1 = one one-warp CTA per chunk group, 2 = one CTA of several warps per SM
  // that claim their groups, 0 = a persistent grid of one-warp CTAs, -1 = the variant's default (fused_default_warps).
  // warps_per_sm > 0 caps the resident warps: in mode 2 it sets the warps per CTA (up to what fits), in mode 0 the CTAs
  // per SM.  smem_pad only pads the one-warp modes.
  int grid_mode = -1, warps_per_sm = 0;
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

// Most warps one CTA of k_huf_decode_fused<G, PB> can hold and still be resident: fused_max_warps by the shared-memory
// arithmetic, confirmed by the occupancy calculator (which knows the per-CTA reserve and the allocation granularity).
template <int G, int PB>
int fused_cta_warps() {
  return launch_plan(kPlanFusedWarps, (const void*)k_huf_decode_fused<G, PB>, 0, 0, [](int) {
    constexpr int wmax = fused_max_warps<G, PB>();
    int best = 1;
    if (smem_attr(k_huf_decode_fused<G, PB>, fused_smem_bytes<G>(PB, wmax))) {
      for (int v = wmax; v > 1; v--) {
        int nb = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_huf_decode_fused<G, PB>, 32 * v, fused_smem_bytes<G>(PB, v)) == cudaSuccess && nb >= 1) {
          best = v;
          break;
        }
      }
    }
    (void)cudaGetLastError();
    return best;
  });
}

// Warps per CTA of the default launch of each variant, 0 for one one-warp CTA per chunk group.  From about 9 warps per SM
// on an SM's decode rate hardly grows with more warps, and more warps make more concurrent bitstreams; the fewest that
// keep the rate were fastest for the rotated types (16 GiB tensors, H100 80GB HBM3 at 400 W, tools/decode_packing.py:
// bf16 13 warps 13.2 ms against 13.9 for one-warp CTAs at 16 per SM, fp32 10 warps 15.5 ms against 19.7 at 13 per SM);
// fp16 and fp8 showed no clear winner and keep the one-warp launch (DESIGN.md 3.1).
template <int G, int PB>
constexpr int fused_default_warps() {
  return PB == 5 ? (G == 2 ? 13 : 10) : 0;
}

// Mode 2: one CTA of W warps per SM whose warps claim chunk groups one at a time (DecodeCfg::fused_claim), so the
// groups spread over the SMs as evenly as their speed allows whatever W is.  W: ZIPNN_B200_WARPS_PER_SM if set, else the
// variant's default, and below one round of the machine no more warps per SM than it takes to give every SM its share.
template <int G, int PB>
void launch_fused(DecodeCfg cfg, uint8_t* out, const TmaMaps& maps, uint64_t groups, const Knobs& kn, cudaStream_t st) {
  const uint64_t sms = (uint64_t)sm_count_cached();
  constexpr int kDefault = fused_default_warps<G, PB>();
  const int mode = kn.grid_mode >= 0 ? kn.grid_mode : (kDefault > 0 ? 2 : 1);
  int W = 1;
  unsigned grid;
  size_t smem;
  cfg.fused_claim = 0;
  if (mode == 2) {
    const int wmax = fused_cta_warps<G, PB>();
    if (kn.warps_per_sm > 0) {
      W = std::min(wmax, kn.warps_per_sm);
    } else {
      W = std::min(wmax, kDefault > 0 ? kDefault : wmax);
      W = (int)std::min<uint64_t>((uint64_t)W, (groups + sms - 1) / sms);
    }
    grid = (unsigned)std::min<uint64_t>((groups + W - 1) / W, sms);
    smem = fused_smem_bytes<G>(PB, W);
    cfg.fused_claim = 1;
  } else {
    smem = fused_smem_bytes<G>(PB) + kn.smem_pad;
    grid = (unsigned)groups;
    if (mode == 0) {
      int nb = resident_blocks(k_huf_decode_fused<G, PB>, smem);
      if (kn.warps_per_sm > 0) nb = std::min(nb, kn.warps_per_sm);
      grid = (unsigned)std::min<uint64_t>(groups, (uint64_t)nb * sms);
    }
  }
  if (getenv("ZIPNN_B200_DEBUG"))
    fprintf(stderr, "[zipnn_b200] fused launch: G=%d PB=%d mode=%d warps_per_cta=%d grid=%u resident_warps_per_sm=%d\n", G, PB, mode, W, grid,
            W * resident_blocks(k_huf_decode_fused<G, PB>, smem, 32 * W));
  k_huf_decode_fused<G, PB><<<grid, 32 * W, smem, st>>>(cfg, out, maps);
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
// Plane-pool slots of the default workspace of K chunks: one per chunk up to kDefaultSlots, else the pool and the
// overflow CTAs' slots.
inline uint64_t pool_slots(uint64_t K) { return K <= kDefaultSlots ? K : kDefaultSlots + kOverflowCtas; }
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
  const int rc = read_back(&err, d_ws, sizeof(uint32_t), st);
  if (rc) return rc;
  if (err & kErrCorrupt) return ZIPNN_B200_E_CORRUPT;
  if (err & kErrUnsupported) return ZIPNN_B200_E_UNSUPPORTED;
  if (err & kErrWorkspace) return ZIPNN_B200_E_CAPACITY;
  if (err & kErrIndex) return ZIPNN_B200_E_INDEX;
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
    case ZIPNN_B200_E_INDEX: return "gather id out of range";
    default: return "unknown status";
  }
}

int zipnn_b200_last_cuda_error(void) { return g_last_cuda_error.load(); }
int zipnn_b200_sm_count(void) { return sm_count_cached(); }

int zipnn_b200_peek(const void* d_src, size_t n, void* h_dst, void* cuda_stream) {
  if (n > kPinnedBlock || (n && (!d_src || !h_dst))) return ZIPNN_B200_E_ARG;
  return n ? read_back(h_dst, d_src, n, (cudaStream_t)cuda_stream) : ZIPNN_B200_OK;
}
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
  *out = L.fixed + (size_t)pool_slots(num_chunks(orig, chunk)) * num_buf * L.pstride;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decompress_workspace_size_full(size_t orig, int num_buf, size_t chunk, size_t* out) {
  if (!out || chunk == 0 || !(num_buf == 1 || num_buf == 2 || num_buf == 4)) return ZIPNN_B200_E_ARG;
  const DecWs L = dec_ws_layout(orig, num_buf, chunk);
  *out = L.fixed + (size_t)num_chunks(orig, chunk) * num_buf * L.pstride;
  return ZIPNN_B200_OK;
}

// Fill a DecodeCfg for one tensor whose workspace slice is [ws, ws + ws_bytes).  With `planes` the slice holds only
// what precedes the plane pool (L.planes_off bytes: a decode plan's metadata) and the pool is [planes, + planes_bytes).
static int fill_decode_cfg(DecodeCfg& cfg, const void* d_body, size_t body_len, int G, int bits_mode, size_t chunk, size_t orig, void* d_out,
                           uint8_t* ws, size_t ws_bytes, bool use_sync, uint64_t table_chunks = UINT64_MAX, uint8_t* planes = nullptr,
                           size_t planes_bytes = 0) {
  const uint64_t K = num_chunks(orig, chunk);
  if (body_len < 9ull * G * K) return ZIPNN_B200_E_CORRUPT;
  const DecWs L = dec_ws_layout(orig, G, chunk, table_chunks);
  if (ws_bytes < (planes ? L.planes_off : L.fixed)) return ZIPNN_B200_E_CAPACITY;
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
  cfg.planes = planes ? planes : ws + L.planes_off;
  cfg.pstride = L.pstride;
  cfg.olist = (uint32_t*)(ws + L.olist_off);
  const uint64_t have = (planes ? planes_bytes : ws_bytes - L.fixed) / ((size_t)G * L.pstride);
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
    int rc = dispatch_G(G, [&](auto g) -> int {
      constexpr int GG = decltype(g)::value;
      const unsigned grid = resident_grid(k_huf_decode_sync<GG>, kSyncSmemBytes, kSyncThreads, 4 * nitems);
      if (!grid) return ZIPNN_B200_E_CUDA;
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
        if constexpr (GG > 1) {  // (short codes only occur with two or four groups: no <1, 5> instance)
          if (short_codes) {
            launch_fused<GG, 5>(cfg, (uint8_t*)d_out, maps, groups, kn, st);
            ZB_LAUNCHED();
            return ZIPNN_B200_OK;
          }
        }
        launch_fused<GG, 0>(cfg, (uint8_t*)d_out, maps, groups, kn, st);
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

// ---- the per-bitstream-CTA family over a batch, in two halves ----
// The prepare half depends on the streams only: descriptors to the device, item tables, modes and work lists
// (k_decode_meta_batch), parsed Huffman table descriptions (k_parse_tables_batch).  The decode half writes the
// output: it only reads the counts, lists and tables the prepare half left, and writes the output, the plane pool
// and the error bits, so a decode plan enqueues it again for every run.
struct BatchGrid {
  uint64_t chunks, items, tiles, max_ovf;  // chunk_start[n], item_start[n], tile_start[n]; overflow CTAs per tensor
};

// The descriptors of a batch of n pieces, as batch_prepare copies them behind the error word: a DecodeCfg per piece,
// then chunk_start, item_start and tile_start (n + 1 each: prefix sums of the chunks, coded-bitstream items and merge
// tiles the batch kernels take from each piece).
struct BatchDescs {
  int n;
  std::vector<DecodeCfg> cfgs;
  std::vector<uint64_t> starts;
  uint64_t max_ovf;  // overflow CTAs per piece: the largest ovf_slots of a piece with chunks, at least the start value
  BatchDescs(int n_, uint64_t max_ovf_) : n(n_), starts(3 * ((size_t)n_ + 1), 0), max_ovf(max_ovf_) { cfgs.reserve((size_t)n_); }
  uint64_t start(int array, int j) const { return starts[(size_t)array * (n + 1) + j]; }
  // The next piece: cfg, of which the batch kernels decode kc chunks (0: none, the piece is only a descriptor).
  void add(const DecodeCfg& cfg, uint64_t kc) {
    const size_t j = cfgs.size();
    cfgs.push_back(cfg);
    const uint64_t counts[3] = {kc, 4ull * cfg.G * kc, kc * ((cfg.chunk + kMergeTile - 1) / kMergeTile)};
    for (int a = 0; a < 3; a++) starts[(size_t)a * (n + 1) + j + 1] = starts[(size_t)a * (n + 1) + j] + counts[a];
    if (kc) max_ovf = std::max<uint64_t>(max_ovf, cfg.ovf_slots);
  }
};

static int batch_prepare(const BatchDescs& D, uint8_t* ws, cudaStream_t st, BatchCfg& B, BatchGrid& grid) {
  const int n = D.n;
  grid.chunks = D.start(0, n);
  grid.items = D.start(1, n);
  grid.tiles = D.start(2, n);
  grid.max_ovf = D.max_ovf;
  // descriptors to the device (pageable source: the copy is staged before the call returns)
  uint8_t* d_cfgs = ws + 256;
  uint8_t* d_starts = d_cfgs + sizeof(DecodeCfg) * (size_t)n;
  ZB_CUDA(cudaMemcpyAsync(d_cfgs, D.cfgs.data(), sizeof(DecodeCfg) * (size_t)n, cudaMemcpyHostToDevice, st));
  ZB_CUDA(cudaMemcpyAsync(d_starts, D.starts.data(), sizeof(uint64_t) * D.starts.size(), cudaMemcpyHostToDevice, st));
  B.cfgs = (const DecodeCfg*)d_cfgs;
  B.chunk_start = (const uint64_t*)d_starts;
  B.item_start = B.chunk_start + (n + 1);
  B.tile_start = B.item_start + (n + 1);
  B.n = (uint32_t)n;
  B.error_out = (uint32_t*)ws;
  if (grid.chunks) {
    {
      const int threads = 128;
      const unsigned blocks = (unsigned)std::min<uint64_t>((grid.chunks + threads - 1) / threads, 4096);
      ScopedTimer tm(kKDecodeMeta, st);
      k_decode_meta_batch<<<blocks, threads, 0, st>>>(B);
      ZB_LAUNCHED();
    }
    {
      ScopedTimer tp(kKParseTables, st);
      k_parse_tables_batch<<<(unsigned)(((grid.items >> 2) + kParseWarps - 1) / kParseWarps), kParseWarps * 32, 0, st>>>(B);
      ZB_LAUNCHED();
    }
  }
  return ZIPNN_B200_OK;
}

// The sync decoder of a decode plan: record (create) or replay (run) of the segment starts.
extern "C++" template <int M>
int launch_sync_plan(const BatchCfg& B, const SegIndex& X, uint64_t items, cudaStream_t st) {
  const unsigned blocks = resident_grid(k_huf_decode_sync_plan<M>, kSyncSmemBytes, kSyncThreads, items);
  if (!blocks) return ZIPNN_B200_E_CUDA;
  ScopedTimer tm(kKHufDecodeSync, st);
  k_huf_decode_sync_plan<M><<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(B, X);
  ZB_LAUNCHED();
  return ZIPNN_B200_OK;
}

// No host work besides the launches once a first call has set the kernel attribute (a decode plan's create does).
// mode: kSyncDecode (the batch and slice calls), or kSyncRecord / kSyncReplay with a plan's segment index X.
static int batch_decode(const BatchCfg& B, const BatchGrid& grid, cudaStream_t st, int mode = kSyncDecode, const SegIndex* X = nullptr) {
  if (!grid.chunks) return ZIPNN_B200_OK;
  const int sms = sm_count_cached();
  if (mode != kSyncDecode) {
    const int rc = mode == kSyncRecord ? launch_sync_plan<kSyncRecord>(B, *X, grid.items, st) : launch_sync_plan<kSyncReplay>(B, *X, grid.items, st);
    if (rc) return rc;
  } else {
    const unsigned blocks = resident_grid(k_huf_decode_sync_batch, kSyncSmemBytes, kSyncThreads, grid.items);
    if (!blocks) return ZIPNN_B200_E_CUDA;
    ScopedTimer tm(kKHufDecodeSync, st);
    k_huf_decode_sync_batch<<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(B);
    ZB_LAUNCHED();
  }
  {
    const unsigned blocks = (unsigned)std::min<uint64_t>(grid.tiles, (uint64_t)sms * 16);
    ScopedTimer tm(kKRegroup, st);
    k_regroup_batch<<<blocks, kMergeThreads, 0, st>>>(B);
    ZB_LAUNCHED();
  }
  if (grid.max_ovf) {
    ScopedTimer tm(kKDecodeOverflow, st);
    k_decode_overflow_batch<<<dim3((unsigned)grid.max_ovf, B.n), kMergeThreads, sizeof(DecodeSmem), st>>>(B);
    ZB_LAUNCHED();
  }
  return ZIPNN_B200_OK;
}

// OR of every tensor's error word into the batch's (its workspace's first word).
static int batch_errors(const BatchCfg& B, cudaStream_t st) {
  k_batch_errors<<<1, 256, 0, st>>>(B);
  ZB_LAUNCHED();
  return ZIPNN_B200_OK;
}

static int run_batch_kernels(const BatchDescs& D, uint8_t* ws, cudaStream_t st, BatchCfg& B) {
  BatchGrid grid;
  const int rc = batch_prepare(D, ws, st, B, grid);
  return rc ? rc : batch_decode(B, grid, st);
}

int zipnn_b200_decompress_batch(const zipnn_b200_batch_item* items, int n, void* d_ws, size_t ws_bytes, void* cuda_stream, int check) {
  if (n < 0 || (n && !items) || !d_ws || ((uintptr_t)d_ws & 255)) return ZIPNN_B200_E_ARG;
  if (n == 0) return ZIPNN_B200_OK;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  uint8_t* ws = (uint8_t*)d_ws;
  const size_t hdr = batch_header_bytes(n);
  if (ws_bytes < hdr) return ZIPNN_B200_E_CAPACITY;
  BatchDescs D(n, 0);
  size_t at = hdr;
  std::vector<int> big;  // tensors that go through the single-tensor path on the same stream
  ZB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
  for (int i = 0; i < n; i++) {
    const zipnn_b200_batch_item& it = items[i];
    if (!valid_layout(it.num_buf, it.bytes_mode, it.chunk)) return ZIPNN_B200_E_ARG;
    const size_t slice = batch_slice_bytes(it);
    if (at + slice > ws_bytes) return ZIPNN_B200_E_CAPACITY;
    DecodeCfg cfg;
    memset(&cfg, 0, sizeof(DecodeCfg));
    cfg.ctrl = (Ctrl*)ws;  // (never raised: an empty tensor has no kernel work)
    if (it.orig == 0) {
      D.add(cfg, 0);
      continue;
    }
    if (!it.d_body || !it.d_out || ((uintptr_t)it.d_out & 15)) return ZIPNN_B200_E_ARG;
    const uint64_t K = num_chunks(it.orig, it.chunk);
    const bool small = K <= sync_max_chunks(it.num_buf);
    const int rc = fill_decode_cfg(cfg, it.d_body, it.body_len, it.num_buf, it.bits_mode, it.chunk, it.orig, it.d_out, ws + at, slice, small);
    if (rc) return rc;
    ZB_CUDA(cudaMemsetAsync(ws + at, 0, kCtrlBytes, st));
    D.add(cfg, small ? K : 0);
    if (!small) big.push_back(i);
    at += slice;
  }
  BatchCfg B;
  {
    const int rc = run_batch_kernels(D, ws, st, B);
    if (rc) return rc;
  }
  for (int i : big) {
    const zipnn_b200_batch_item& it = items[i];
    const int rc = zipnn_b200_decompress(it.d_body, it.body_len, it.num_buf, it.bits_mode, it.bytes_mode, it.chunk, it.orig, it.d_out,
                                         (void*)D.cfgs[i].ctrl, batch_slice_bytes(it), st, 0);
    if (rc) return rc;
  }
  {
    const int rc = batch_errors(B, st);
    if (rc) return rc;
  }
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
    // units per piece; at least one, also when limit * chunk < 32 (chunks under 16 bytes with a small limit), where
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
  return round_up(L.fixed + (size_t)pool_slots(kc) * it.num_buf * L.pstride, 256);
}
// The piece's box as the window of cfg: the decoders write only its bytes, packed, and start at chunk p.c0.
void set_box(DecodeCfg& cfg, const SlicePiece& p) {
  cfg.box_base = p.base;
  cfg.box_rows = p.rows;
  cfg.box_pitch = p.pitch;
  cfg.box_len = p.len;
  cfg.box_step_rows = kBoxStep / p.pitch;
  cfg.box_step_cols = kBoxStep % p.pitch;
  cfg.box_fast = ((p.base | p.pitch | p.len) & 15) == 0;
  cfg.c0 = p.c0;
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
  BatchDescs D(np, 1);  // the overflow kernel always runs (its CTAs return at once when no piece has overflow slots): a fixed launch count
  ZB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
  for (int j = 0; j < np; j++) {
    const SlicePiece& p = pieces[j];
    const zipnn_b200_slice_item& it = items[p.item];
    const size_t slice = slice_piece_bytes(it, p);
    if (at + slice > ws_bytes) return ZIPNN_B200_E_CAPACITY;
    const uint64_t kc = p.c1 - p.c0;
    DecodeCfg cfg;
    const int rc = fill_decode_cfg(cfg, it.d_body, it.body_len, it.num_buf, it.bits_mode, it.chunk, it.orig, (uint8_t*)it.d_out + p.out_off,
                                   ws + at, slice, true, kc);
    if (rc) return rc;
    set_box(cfg, p);
    ZB_CUDA(cudaMemsetAsync(ws + at, 0, kCtrlBytes, st));
    D.add(cfg, kc);
    at += slice;
  }
  BatchCfg B;
  {
    const int rc = run_batch_kernels(D, ws, st, B);
    if (rc) return rc;
  }
  {
    const int rc = batch_errors(B, st);
    if (rc) return rc;
  }
  if (check) return read_ctrl_error(d_ws, st);
  return ZIPNN_B200_OK;
}

// ---- decode plans: the prepare half once, the decode half per run ------------------------------------------
// Plan memory: [256 B: error word][DecodeCfg np][chunk_start, item_start, tile_start][segment index base, np + 1]
// [per piece: the workspace slice up to its plane pool][segment index].  Scratch: per piece, the plane pool of a
// slice piece.
namespace {
constexpr uint64_t kPlanMagic = 0x7a6e6e706c616e32ull;  // "znnplan2"
constexpr uint64_t kSegPerItem = 4ull * kSyncThreads;   // index entries per coded item (4 bitstreams x 256 threads)
struct PlanState {
  uint64_t magic;  // kPlanMagic once create succeeded
  BatchCfg B;
  BatchGrid grid;
  SegIndex X;
  uint64_t coded;  // coded items the segment index has room for
  int32_t mode;    // kSyncReplay, or kSyncDecode for a plan without an index
  uint32_t gen;    // create's number: which host record (g_plan_items) describes this plan's items
};
// What a gather needs to know of each item on the host, without reading the device: recorded by create under the
// plan memory's address (a later create at the same address replaces the record; `gen` tells a stale plan apart).
struct GatherItem {
  int piece;          // the item's one piece, -1 when it has none or several (empty, or split) or is a box
  int G;
  uint32_t chunk;
  uint64_t K, orig;
  uint64_t seg_base;  // the piece's first segment index entry
  const uint8_t* d_mode;  // the piece's chunk modes (device, [K])
  int fused;          // every chunk is in fused mode (a matvec needs that): -1 until a matvec call has read d_mode
};
struct PlanItems {
  uint32_t gen;
  std::vector<GatherItem> items;
};
std::mutex g_plan_mu;
std::unordered_map<uintptr_t, PlanItems> g_plan_items;  // by plan memory address
uint32_t g_plan_gen = 0;
static_assert(sizeof(PlanState) <= sizeof(zipnn_b200_decode_plan), "the plan state must fit the ABI's opaque struct");
size_t plan_piece_meta_bytes(const zipnn_b200_slice_item& it, const SlicePiece& p) {
  return round_up(dec_ws_layout(it.orig, it.num_buf, it.chunk, p.c1 - p.c0).planes_off, 256);
}
size_t plan_piece_scratch_bytes(const zipnn_b200_slice_item& it, const SlicePiece& p) {
  const uint64_t kc = p.c1 - p.c0;
  const DecWs L = dec_ws_layout(it.orig, it.num_buf, it.chunk, kc);
  return round_up((size_t)pool_slots(kc) * it.num_buf * L.pstride, 256);
}
bool plan_state(const zipnn_b200_decode_plan* plan, PlanState& s) {
  if (!plan) return false;
  memcpy(&s, plan->opaque, sizeof(s));
  return s.magic == kPlanMagic;
}
constexpr int64_t kAllItems = INT64_MIN;  // (no int item is)
// f(items) on the host records of plan s, under g_plan_mu: every read and write of g_plan_items happens here.  E_ARG
// for a plan whose memory a later create has taken, and unless `item` is kAllItems, for an item the plan does not have.
extern "C++" template <typename F>
int with_plan_items(const PlanState& s, int64_t item, F&& f) {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  const auto it = g_plan_items.find((uintptr_t)s.B.error_out);
  if (it == g_plan_items.end() || it->second.gen != s.gen) return ZIPNN_B200_E_ARG;
  std::vector<GatherItem>& items = it->second.items;
  if (item != kAllItems && (item < 0 || (uint64_t)item >= items.size())) return ZIPNN_B200_E_ARG;
  f(items);
  return ZIPNN_B200_OK;
}
struct PlanLayout {
  std::vector<SlicePiece> pieces;
  std::vector<uint64_t> seg_base;  // [np + 1] index entries in front of each piece
  size_t base_off, metas_off, index_off, plan_bytes, scratch_bytes;
  bool replay;
};
// Pieces, the coded items each of them may queue and the memory split.  The coded items of a piece are the type-1
// entries of its stream's type rows over the piece's covering chunks: every item k_decode_meta_batch can put on the
// piece's hlist is one of them.  Reading the type rows synchronises `st`.  ZIPNN_B200_PLAN_REPLAY=0 builds plans
// without an index, whose runs take the rounds of the decode mode (tools/plan_bench.py compares the two).
int plan_layout(const zipnn_b200_slice_item* items, int n, cudaStream_t st, PlanLayout& P) {
  const int rc = plan_slices(items, n, P.pieces);
  if (rc) return rc;
  const char* e = getenv("ZIPNN_B200_PLAN_REPLAY");
  P.replay = !(e && atoi(e) == 0);
  const size_t np = P.pieces.size();
  std::vector<std::vector<uint8_t>> types((size_t)n);
  if (P.replay) {
    for (const SlicePiece& p : P.pieces) {
      const zipnn_b200_slice_item& it = items[p.item];
      const uint64_t K = num_chunks(it.orig, it.chunk), rows = (uint64_t)it.num_buf * K;
      if (!types[p.item].empty() || it.body_len < 9 * rows) continue;  // (a short body fails at create)
      types[p.item].resize(rows);
      ZB_CUDA(cudaMemcpyAsync(types[p.item].data(), it.d_body, rows, cudaMemcpyDeviceToHost, st));
    }
    ZB_CUDA(cudaStreamSynchronize(st));
  }
  P.seg_base.assign(np + 1, 0);
  for (size_t j = 0; j < np; j++) {
    const SlicePiece& p = P.pieces[j];
    const zipnn_b200_slice_item& it = items[p.item];
    const std::vector<uint8_t>& ty = types[p.item];
    uint64_t coded = 0;
    if (!ty.empty()) {
      const uint64_t K = num_chunks(it.orig, it.chunk);
      for (int g = 0; g < it.num_buf; g++)
        for (uint64_t c = p.c0; c < p.c1; c++) coded += ty[(uint64_t)g * K + c] == 1;
    }
    P.seg_base[j + 1] = P.seg_base[j] + coded * kSegPerItem;
  }
  P.base_off = batch_header_bytes((int)np);
  P.metas_off = P.base_off + round_up(sizeof(uint64_t) * (np + 1), 256);
  size_t at = P.metas_off, scratch = 0;
  for (const SlicePiece& p : P.pieces) {
    at += plan_piece_meta_bytes(items[p.item], p);
    scratch += plan_piece_scratch_bytes(items[p.item], p);
  }
  P.index_off = at;
  P.plan_bytes = at + sizeof(SegEntry) * (size_t)P.seg_base[np];
  P.scratch_bytes = scratch;
  return ZIPNN_B200_OK;
}
}  // namespace

int zipnn_b200_decode_plan_size(const zipnn_b200_slice_item* items, int n, void* cuda_stream, size_t* plan_bytes, size_t* scratch_bytes) {
  if (!plan_bytes || !scratch_bytes) return ZIPNN_B200_E_ARG;
  PlanLayout P;
  const int rc = plan_layout(items, n, (cudaStream_t)cuda_stream, P);
  if (rc) return rc;
  *plan_bytes = P.plan_bytes;
  *scratch_bytes = P.scratch_bytes;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_create(const zipnn_b200_slice_item* items, int n, void* d_plan, size_t plan_bytes, void* d_scratch,
                                  size_t scratch_bytes, zipnn_b200_decode_plan* plan, void* cuda_stream) {
  if (!plan) return ZIPNN_B200_E_ARG;
  memset(plan, 0, sizeof(*plan));
  if (!d_plan || ((uintptr_t)d_plan & 255) || ((uintptr_t)d_scratch & 255) || (scratch_bytes && !d_scratch)) return ZIPNN_B200_E_ARG;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  PlanLayout P;
  {
    const int rc = plan_layout(items, n, st, P);
    if (rc) return rc;
  }
  if (plan_bytes < P.plan_bytes || scratch_bytes < P.scratch_bytes) return ZIPNN_B200_E_CAPACITY;
  const int np = (int)P.pieces.size();
  uint8_t* meta = (uint8_t*)d_plan;
  uint8_t* scratch = (uint8_t*)d_scratch;
  size_t at = P.metas_off, sat = 0;
  BatchDescs D(np, 1);  // (as in the slice call: a fixed launch count)
  for (int j = 0; j < np; j++) {
    const SlicePiece& p = P.pieces[j];
    const zipnn_b200_slice_item& it = items[p.item];
    const size_t mb = plan_piece_meta_bytes(it, p), sb = plan_piece_scratch_bytes(it, p);
    const uint64_t kc = p.c1 - p.c0;
    DecodeCfg cfg;
    const int rc = fill_decode_cfg(cfg, it.d_body, it.body_len, it.num_buf, it.bits_mode, it.chunk, it.orig, (uint8_t*)it.d_out + p.out_off,
                                   meta + at, mb, true, kc, scratch + sat, sb);
    if (rc) return rc;
    // a piece that is a whole tensor decodes without the window, as in the batch call
    const bool whole = p.base == 0 && p.rows == 1 && p.len == it.orig;
    if (!whole) set_box(cfg, p);
    D.add(cfg, kc);
    at += mb;
    sat += sb;
  }
  // error word, every piece's control block, and the index (entries of items that turn out raw or RLE stay empty)
  ZB_CUDA(cudaMemsetAsync(meta, 0, P.plan_bytes, st));
  ZB_CUDA(cudaMemcpyAsync(meta + P.base_off, P.seg_base.data(), sizeof(uint64_t) * P.seg_base.size(), cudaMemcpyHostToDevice, st));
  PlanState s;
  memset(&s, 0, sizeof(s));
  s.X.seg = (SegEntry*)(meta + P.index_off);
  s.X.base = (const uint64_t*)(meta + P.base_off);
  s.coded = P.seg_base[np] / kSegPerItem;
  s.mode = P.replay ? kSyncReplay : kSyncDecode;
  {
    int rc = batch_prepare(D, meta, st, s.B, s.grid);
    if (!rc) rc = batch_decode(s.B, s.grid, st, P.replay ? kSyncRecord : kSyncDecode, &s.X);
    if (!rc) rc = batch_errors(s.B, st);
    if (!rc) rc = read_ctrl_error(meta, st);
    if (rc) return rc;
  }
  {
    PlanItems rec;
    rec.items.resize((size_t)n);
    for (int i = 0; i < n; i++) {
      const zipnn_b200_slice_item& it = items[i];
      rec.items[i] = GatherItem{-1, it.num_buf, (uint32_t)it.chunk, num_chunks(it.orig, it.chunk), it.orig, 0, nullptr, -1};
    }
    for (int j = 0; j < np; j++) {
      const SlicePiece& p = P.pieces[j];
      const zipnn_b200_slice_item& it = items[p.item];
      GatherItem& g = rec.items[p.item];
      const bool whole = p.base == 0 && p.rows == 1 && p.len == it.orig;
      g.piece = whole && g.piece == -1 ? j : -2;   // (-2: a box or a split item; the pieces of an item are consecutive)
      g.seg_base = P.seg_base[j];
      g.d_mode = D.cfgs[j].mode;
    }
    for (GatherItem& g : rec.items)
      if (g.piece < 0) g.piece = -1;
    std::lock_guard<std::mutex> lk(g_plan_mu);
    s.gen = rec.gen = ++g_plan_gen;
    g_plan_items[(uintptr_t)d_plan] = std::move(rec);
  }
  s.magic = kPlanMagic;
  memcpy(plan->opaque, &s, sizeof(s));
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_index(const zipnn_b200_decode_plan* plan, size_t* index_bytes, size_t* coded_items) {
  PlanState s;
  if (!plan_state(plan, s) || !index_bytes || !coded_items) return ZIPNN_B200_E_ARG;
  *coded_items = s.mode == kSyncReplay ? s.coded : 0;
  *index_bytes = *coded_items * kSegPerItem * sizeof(SegEntry);
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_run(const zipnn_b200_decode_plan* plan, void* cuda_stream) {
  PlanState s;
  if (!plan_state(plan, s)) return ZIPNN_B200_E_ARG;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const int rc = batch_decode(s.B, s.grid, st, s.mode, &s.X);
  return rc ? rc : batch_errors(s.B, st);
}

int zipnn_b200_decode_plan_run_shifted(const zipnn_b200_decode_plan* plan, int64_t out_shift, int max_ctas, void* cuda_stream) {
  PlanState s;
  if (!plan_state(plan, s) || (out_shift & 15)) return ZIPNN_B200_E_ARG;
  if (s.mode != kSyncReplay) return ZIPNN_B200_E_UNSUPPORTED;
  // more CTAs than units (or than the overflow CTAs a tensor may use) would only claim nothing
  const uint64_t useful = std::max<uint64_t>(std::max<uint64_t>(1, s.grid.items + s.grid.tiles), s.grid.max_ovf);
  const unsigned ctas = resident_grid(k_plan_replay_persistent, kPlanReplaySmemBytes, kSyncThreads,
                                      max_ctas <= 0 ? useful : std::min<uint64_t>((uint64_t)max_ctas, useful));
  if (!ctas) return ZIPNN_B200_E_CUDA;
  k_plan_replay_persistent<<<ctas, kSyncThreads, kPlanReplaySmemBytes, (cudaStream_t)cuda_stream>>>(s.B, s.X, out_shift);
  ZB_LAUNCHED();
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_status(const zipnn_b200_decode_plan* plan, void* cuda_stream) {
  PlanState s;
  if (!plan_state(plan, s)) return ZIPNN_B200_E_ARG;
  return read_ctrl_error(s.B.error_out, (cudaStream_t)cuda_stream);
}

// ---- gathers: rows of one whole-tensor item, decoded from the chunks the ids touch (gather.cuh) ----------------
// Scratch: [256 B: touched-chunk count][list u32 K][pos u32 K][inv u32 G*K][slots x G planes of pstride bytes].
namespace {
struct GatherLayout {
  size_t list_off, pos_off, inv_off, planes_off;
  uint64_t pstride;
};
GatherLayout gather_layout(const GatherItem& gi) {
  GatherLayout L;
  L.list_off = 256;
  L.pos_off = round_up(L.list_off + 4 * gi.K, 256);
  L.inv_off = round_up(L.pos_off + 4 * gi.K, 256);
  L.planes_off = round_up(L.inv_off + 4 * (size_t)gi.G * gi.K, 256);
  L.pstride = dec_ws_layout(gi.orig, gi.G, gi.chunk, 0).pstride;
  return L;
}
// Chunks a row of `row_bytes` may touch, wherever it starts: floor((chunk - 1 + row_bytes - 1) / chunk) + 1, at most K.
uint64_t gather_span(uint64_t row_bytes, uint64_t chunk, uint64_t K) { return std::min<uint64_t>(K, (row_bytes + chunk - 2) / chunk + 1); }
// The host-side checks shared by both calls.
int gather_item(const zipnn_b200_decode_plan* plan, int item, size_t row_bytes, PlanState& s, GatherItem& gi) {
  if (!plan_state(plan, s)) return ZIPNN_B200_E_ARG;
  {
    const int rc = with_plan_items(s, item, [&](std::vector<GatherItem>& v) { gi = v[(size_t)item]; });
    if (rc) return rc;
  }
  if (gi.piece < 0 || s.mode != kSyncReplay) return ZIPNN_B200_E_UNSUPPORTED;
  if (row_bytes == 0 || gi.orig % row_bytes) return ZIPNN_B200_E_ARG;
  return ZIPNN_B200_OK;
}
}  // namespace

int zipnn_b200_decode_plan_gather_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t row_bytes, size_t slots, size_t* out) {
  if (!out || slots == 0) return ZIPNN_B200_E_ARG;
  PlanState s;
  GatherItem gi;
  const int rc = gather_item(plan, item, row_bytes, s, gi);
  if (rc) return rc;
  const GatherLayout L = gather_layout(gi);
  *out = L.planes_off + std::min<uint64_t>(slots, gi.K) * gi.G * L.pstride;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_gather(const zipnn_b200_decode_plan* plan, int item, size_t row_bytes, const void* d_ids, size_t n_ids, int id_bytes,
                                  void* d_out, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (id_bytes != 4 && id_bytes != 8) return ZIPNN_B200_E_ARG;
  PlanState s;
  GatherItem gi;
  {
    const int rc = gather_item(plan, item, row_bytes, s, gi);
    if (rc) return rc;
  }
  if (n_ids == 0) return ZIPNN_B200_OK;
  if (!d_ids || !d_out || !d_scratch || ((uintptr_t)d_ids % (uintptr_t)id_bytes) || ((uintptr_t)d_scratch & 255)) return ZIPNN_B200_E_ARG;
  if (n_ids > (1ull << 40)) return ZIPNN_B200_E_ARG;
  const GatherLayout L = gather_layout(gi);
  const uint64_t slot_bytes = (uint64_t)gi.G * L.pstride;
  const uint64_t slots = std::min<uint64_t>(scratch_bytes < L.planes_off ? 0 : (scratch_bytes - L.planes_off) / slot_bytes, gi.K);
  if (slots == 0) return ZIPNN_B200_E_ARG;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  uint8_t* ws = (uint8_t*)d_scratch;
  GatherCfg g;
  g.cfg = s.B.cfgs + gi.piece;
  g.seg = s.X.seg + gi.seg_base;
  g.error = s.B.error_out;
  g.ids = d_ids;
  g.n = n_ids;
  g.id8 = id_bytes == 8;
  g.G = gi.G;
  g.K = gi.K;
  g.orig = gi.orig;
  g.rows = gi.orig / row_bytes;
  g.row_bytes = row_bytes;
  g.span = gather_span(row_bytes, gi.chunk, gi.K);
  g.chunk = gi.chunk;
  g.slots = (uint32_t)slots;
  g.out = (uint8_t*)d_out;
  g.count = (uint32_t*)ws;
  g.list = (uint32_t*)(ws + L.list_off);
  g.pos = (uint32_t*)(ws + L.pos_off);
  g.inv = (uint32_t*)(ws + L.inv_off);
  g.planes = ws + L.planes_off;
  g.pstride = L.pstride;
  // passes: the distinct chunks are at most min(n * span, K), `slots` per pass (a bound of n alone, not of the ids)
  const uint64_t most = n_ids > gi.K / g.span ? gi.K : std::min<uint64_t>(gi.K, n_ids * g.span);
  const uint64_t passes = (most + slots - 1) / slots;
  const unsigned dec_blocks = resident_grid(k_gather_decode, kPlanReplaySmemBytes, kSyncThreads, slots * 4 * gi.G);
  if (!dec_blocks) return ZIPNN_B200_E_CUDA;
  const unsigned inv_blocks = (unsigned)std::max<uint64_t>(1, ((uint64_t)gi.G * gi.K + kGatherIndexThreads - 1) / kGatherIndexThreads);
  k_gather_index<<<1 + inv_blocks, kGatherIndexThreads, 0, st>>>(g);
  ZB_LAUNCHED();
  const uint64_t units = n_ids * ((row_bytes + 15) / 16 + 1);
  const unsigned row_blocks = (unsigned)std::min<uint64_t>((units + 255) / 256, (uint64_t)sm_count_cached() * 16);
  for (uint64_t p = 0; p < passes; p++) {
    k_gather_decode<<<dec_blocks, kSyncThreads, kPlanReplaySmemBytes, st>>>(g, (uint32_t)p);
    ZB_LAUNCHED();
    dispatch_G(gi.G, [&](auto gg) -> int {
      k_gather_rows<decltype(gg)::value><<<row_blocks, 256, 0, st>>>(g, (uint32_t)p);
      return 0;
    });
    ZB_LAUNCHED();
  }
  return ZIPNN_B200_OK;
}

// ---- selected runs: the plan run for the chunks of the slices [e] that ids select (select.cuh) -----------------
// Scratch: [256 B: counts][DecodeCfg np][Ctrl np][hsel uint2 per coded item][tsel uint2 per tile][osel u32 per chunk].
namespace {
struct SelectLayout {
  size_t ocfg_off, octrl_off, hsel_off, tsel_off, osel_off, bytes;
};
SelectLayout select_layout(const PlanState& s) {
  SelectLayout L;
  const size_t np = s.B.n;
  L.ocfg_off = 256;
  L.octrl_off = round_up(L.ocfg_off + sizeof(DecodeCfg) * np, 256);
  L.hsel_off = round_up(L.octrl_off + sizeof(Ctrl) * np, 256);
  L.tsel_off = round_up(L.hsel_off + sizeof(uint2) * (s.grid.items / 4), 256);
  L.osel_off = round_up(L.tsel_off + sizeof(uint2) * s.grid.tiles, 256);
  L.bytes = round_up(L.osel_off + sizeof(uint32_t) * s.grid.chunks, 256);
  return L;
}
// The host-side checks shared by both calls: every item is one whole-tensor piece (so piece j is item j) of a plan with
// a segment index, and its bytes split into `rows` equal slices.  -> the items' records.
int select_items(const zipnn_b200_decode_plan* plan, size_t rows, PlanState& s, std::vector<GatherItem>& items) {
  if (!plan_state(plan, s)) return ZIPNN_B200_E_ARG;
  {
    const int rc = with_plan_items(s, kAllItems, [&](std::vector<GatherItem>& v) { items = v; });
    if (rc) return rc;
  }
  if (s.mode != kSyncReplay || items.empty() || items.size() > 65535) return ZIPNN_B200_E_UNSUPPORTED;  // (grid.y of the overflow)
  for (const GatherItem& gi : items)
    if (gi.piece < 0) return ZIPNN_B200_E_UNSUPPORTED;
  for (const GatherItem& gi : items)
    if (rows == 0 || gi.orig % rows) return ZIPNN_B200_E_ARG;
  return ZIPNN_B200_OK;
}
// The host checks of the ids and the scratch that both selected calls make once the items passed: E_ARG or OK.
int select_args_ok(const SelectLayout& L, const void* d_ids, size_t n_ids, int id_bytes, const void* d_scratch, size_t scratch_bytes) {
  if (!d_ids || !d_scratch || ((uintptr_t)d_ids % (uintptr_t)id_bytes) || ((uintptr_t)d_scratch & 255)) return ZIPNN_B200_E_ARG;
  if (n_ids > (1ull << 40)) return ZIPNN_B200_E_ARG;
  return scratch_bytes < L.bytes ? ZIPNN_B200_E_ARG : ZIPNN_B200_OK;
}
SelectCfg select_cfg(const PlanState& s, const SelectLayout& L, uint8_t* ws, size_t rows, const void* d_ids, size_t n_ids, int id_bytes) {
  SelectCfg sel;
  sel.ids = d_ids;
  sel.n = n_ids;
  sel.id8 = id_bytes == 8;
  sel.rows = rows;
  sel.error = s.B.error_out;
  sel.count = (uint32_t*)ws;
  sel.ocfg = (DecodeCfg*)(ws + L.ocfg_off);
  sel.octrl = (Ctrl*)(ws + L.octrl_off);
  sel.hsel = (uint2*)(ws + L.hsel_off);
  sel.tsel = (uint2*)(ws + L.tsel_off);
  sel.osel = (uint32_t*)(ws + L.osel_off);
  return sel;
}
// Grids from bounds of n alone: an item's touched chunks are at most min(n * span, K).  -> the bitstreams and regroup
// tiles of every item's touched chunks, and the most touched chunks of one item.
void select_bounds(const std::vector<GatherItem>& items, size_t rows, size_t n_ids, uint64_t& bitstreams, uint64_t& tiles, uint64_t& most) {
  for (const GatherItem& gi : items) {
    const uint64_t span = gather_span(gi.orig / rows, gi.chunk, gi.K);
    const uint64_t m = n_ids > gi.K / span ? gi.K : std::min<uint64_t>(gi.K, n_ids * span);
    bitstreams += 4ull * gi.G * m;
    tiles += m * ((gi.chunk + kMergeTile - 1) / kMergeTile);
    most = std::max(most, m);
  }
}
}  // namespace

int zipnn_b200_decode_plan_select_scratch_size(const zipnn_b200_decode_plan* plan, size_t rows, size_t* out) {
  if (!out) return ZIPNN_B200_E_ARG;
  PlanState s;
  std::vector<GatherItem> items;
  const int rc = select_items(plan, rows, s, items);
  if (rc) return rc;
  *out = select_layout(s).bytes;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_run_select(const zipnn_b200_decode_plan* plan, size_t rows, const void* d_ids, size_t n_ids, int id_bytes,
                                      void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (id_bytes != 4 && id_bytes != 8) return ZIPNN_B200_E_ARG;
  PlanState s;
  std::vector<GatherItem> items;
  {
    const int rc = select_items(plan, rows, s, items);
    if (rc) return rc;
  }
  if (n_ids == 0) return ZIPNN_B200_OK;
  const SelectLayout L = select_layout(s);
  {
    const int rc = select_args_ok(L, d_ids, n_ids, id_bytes, d_scratch, scratch_bytes);
    if (rc) return rc;
  }
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const SelectCfg sel = select_cfg(s, L, (uint8_t*)d_scratch, rows, d_ids, n_ids, id_bytes);
  uint64_t bitstreams = 0, tiles = 0, most = 0;
  select_bounds(items, rows, n_ids, bitstreams, tiles, most);
  const unsigned sync_blocks = resident_grid(k_select_sync, kSyncSmemBytes, kSyncThreads, bitstreams);
  if (!sync_blocks) return ZIPNN_B200_E_CUDA;
  k_select_index<<<1, kGatherIndexThreads, 0, st>>>(s.B, sel);
  ZB_LAUNCHED();
  {
    ScopedTimer tm(kKHufDecodeSync, st);
    k_select_sync<<<sync_blocks, kSyncThreads, kSyncSmemBytes, st>>>(s.B, s.X, sel);
    ZB_LAUNCHED();
  }
  {
    ScopedTimer tm(kKRegroup, st);
    k_select_regroup<<<(unsigned)std::min<uint64_t>(tiles, (uint64_t)sm_count_cached() * 16), kMergeThreads, 0, st>>>(s.B, sel);
    ZB_LAUNCHED();
  }
  {
    ScopedTimer tm(kKDecodeOverflow, st);
    k_select_overflow<<<dim3((unsigned)std::min<uint64_t>(s.grid.max_ovf, most), s.B.n), kMergeThreads, sizeof(DecodeSmem), st>>>(sel);
    ZB_LAUNCHED();
  }
  return batch_errors(s.B, st);
}

// ---- matvec and matmul: x W^T from the coded bitstreams of one whole-tensor item, no dense W ------------------------
// Scratch: fp32 partial sums, for the matvec (matvec.cuh) [32 K blocks][rs rows][n_tokens], for the matmul on tensor
// cores (matmul.cuh) [4 K quarters][rt row tiles][n_tokens][8 rows].  The fp8 matvec's are the matvec's, the fp8
// matmul's the matmul's.
namespace {
enum ProductKind { kMatvec, kMatmul, kMatvecFp8, kMatmulFp8 };
bool fp8_kind(ProductKind kind) { return kind == kMatvecFp8 || kind == kMatmulFp8; }
bool matmul_kind(ProductKind kind) { return kind == kMatmul || kind == kMatmulFp8; }
size_t max_tokens(ProductKind kind) { return matmul_kind(kind) ? (size_t)kMatmulMaxTokens : (size_t)kMatvecMaxTokens; }

// The host-side checks shared by all four calls, and the fields of m that the item and the shapes settle.  The first
// call for an item reads its chunk modes (one synchronising copy of K bytes); the answer is kept with the plan's record.
// The matmul takes 16-bit weights only: fp32 would need TF32 or a split scheme, so it is left to the decode.  For the
// fp8 matvec and matmul, `dtype` is x's (bf16 or fp16) and the weights are one byte: their scale lookup takes element
// indices in 32 bits, which every fp8 piece has (at most 16383 chunks of 128 KiB).
int product_item(ProductKind kind, const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, cudaStream_t st, ProductCfg& m) {
  PlanState s;
  GatherItem gi;
  if (!plan_state(plan, s)) return ZIPNN_B200_E_ARG;
  {
    const int rc = with_plan_items(s, item, [&](std::vector<GatherItem>& v) { gi = v[(size_t)item]; });
    if (rc) return rc;
  }
  if (dtype != kMvBf16 && dtype != kMvFp16 && (dtype != kMvFp32 || fp8_kind(kind))) return ZIPNN_B200_E_ARG;
  const uint32_t esize = fp8_kind(kind) ? 1u : (uint32_t)matvec_esize(dtype);
  const uint64_t total = gi.orig / esize;
  if (in_features == 0 || gi.orig % esize || total % in_features) return ZIPNN_B200_E_ARG;
  if (gi.piece < 0 || s.mode != kSyncReplay || gi.G != (int)esize || (in_features * esize) % 16) return ZIPNN_B200_E_UNSUPPORTED;
  if (gi.fused < 0) {
    std::vector<uint8_t> mode((size_t)gi.K);
    ZB_CUDA(cudaMemcpyAsync(mode.data(), gi.d_mode, (size_t)gi.K, cudaMemcpyDeviceToHost, st));
    ZB_CUDA(cudaStreamSynchronize(st));
    int fused = 1;
    for (const uint8_t c : mode) fused &= c == kModeFused;
    const int rc = with_plan_items(s, item, [&](std::vector<GatherItem>& v) {
      v[(size_t)item].fused = fused;
      gi = v[(size_t)item];
    });
    if (rc) return rc;
  }
  if (!gi.fused) return ZIPNN_B200_E_UNSUPPORTED;
  if (kind == kMatmul && dtype == kMvFp32) return ZIPNN_B200_E_UNSUPPORTED;
  if (fp8_kind(kind) && total > (uint64_t)INT32_MAX) return ZIPNN_B200_E_UNSUPPORTED;
  memset(&m, 0, sizeof(m));
  m.cfg = s.B.cfgs + gi.piece;
  m.seg = s.X.seg + gi.seg_base;
  m.error = s.B.error_out;
  m.in = in_features;
  m.out = total / in_features;
  m.ce = gi.chunk / esize;
  m.total = total;
  m.K = gi.K;
  m.esize = esize;
  const uint64_t first = std::min<uint64_t>(m.ce, total);  // elements of the first chunk
  m.rs = (uint32_t)matvec_block_rows(matvec_block_elems(first, esize), m.in, m.out);
  m.rt = (uint32_t)matmul_quarter_tiles(first / 4, m.in, m.out);
  const uint64_t step = 32ull * (16 / esize);
  m.step_rows = (uint32_t)(step / m.in);
  m.step_cols = (uint32_t)(step % m.in);
  return ZIPNN_B200_OK;
}
size_t product_scratch_bytes(ProductKind kind, const ProductCfg& m, size_t n_tokens) {
  if (matmul_kind(kind)) return (size_t)4 * m.K * m.rt * n_tokens * kMatmulTileRows * sizeof(float);
  return (size_t)32 * m.K * m.rs * n_tokens * sizeof(float);
}

// The bitstream kernel of a product, by how many tokens its lanes hold (matvec: 1, 2, 4 or 8; matmul: 1, 2 or 4 tiles of
// 16), and its reduce.  DT is the type of x and y; `fmt` the fp8 products' weight format (ignored by the others).
using ProductKernel = void (*)(ProductCfg);
struct ProductKernels {
  ProductKernel streams, reduce;
};
extern "C++" template <int DT, int NT>
ProductKernel matvec_kernel(ProductKind kind, int fmt) {
  if constexpr (DT != kMvFp32) {  // (product_item refuses fp32 x for fp8 weights)
    if (kind == kMatvecFp8) return fmt == kFp8E4m3 ? &k_matvec_fp8<kFp8E4m3, DT, NT> : &k_matvec_fp8<kFp8E5m2, DT, NT>;
  }
  return &k_matvec<DT, NT>;
}
extern "C++" template <int DT>
ProductKernels product_kernels(ProductKind kind, int fmt, uint32_t nt) {
  if constexpr (DT != kMvFp32) {  // (product_item refuses an fp32 matmul, and fp32 x for fp8 weights)
    if (kind == kMatmul) return {nt <= 16 ? &k_matmul<DT, 1> : nt <= 32 ? &k_matmul<DT, 2> : &k_matmul<DT, 4>, &k_matmul_reduce<DT>};
    if (kind == kMatmulFp8) {
      if (fmt == kFp8E4m3)
        return {nt <= 16 ? &k_matmul_fp8<kFp8E4m3, DT, 1> : nt <= 32 ? &k_matmul_fp8<kFp8E4m3, DT, 2> : &k_matmul_fp8<kFp8E4m3, DT, 4>,
                &k_matmul_reduce<DT>};
      return {nt <= 16 ? &k_matmul_fp8<kFp8E5m2, DT, 1> : nt <= 32 ? &k_matmul_fp8<kFp8E5m2, DT, 2> : &k_matmul_fp8<kFp8E5m2, DT, 4>,
              &k_matmul_reduce<DT>};
    }
  }
  return {nt <= 1   ? matvec_kernel<DT, 1>(kind, fmt)
          : nt <= 2 ? matvec_kernel<DT, 2>(kind, fmt)
          : nt <= 4 ? matvec_kernel<DT, 4>(kind, fmt)
                    : matvec_kernel<DT, 8>(kind, fmt),
          &k_matvec_reduce<DT>};
}
int product_launch(const ProductKernels& f, const ProductCfg& m, cudaStream_t st) {
  const unsigned blocks = resident_grid(f.streams, kSyncSmemBytes, kSyncThreads, 4 * m.K);
  if (!blocks) return ZIPNN_B200_E_CUDA;
  f.streams<<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(m);
  ZB_LAUNCHED();
  f.reduce<<<(unsigned)((m.out * m.nt + 255) / 256), 256, 0, st>>>(m);
  ZB_LAUNCHED();
  return ZIPNN_B200_OK;
}

int product_scratch_size(ProductKind kind, const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, size_t n_tokens,
                         size_t* out) {
  if (!out || n_tokens > max_tokens(kind)) return ZIPNN_B200_E_ARG;
  ProductCfg m;
  const int rc = product_item(kind, plan, item, dtype, in_features, nullptr, m);
  if (rc) return rc;
  *out = product_scratch_bytes(kind, m, n_tokens);
  return ZIPNN_B200_OK;
}

// The weight format and scale grid of the fp8 matvec, matmul and dequantize (fp8_args_ok has checked all but the pointer).
struct Fp8Scale {
  int format;
  const float* d_scale;
  size_t block_rows, block_cols;
};
bool fp8_args_ok(const Fp8Scale& f8) {
  return (f8.format == kFp8E4m3 || f8.format == kFp8E5m2) && f8.block_rows && f8.block_cols >= 16 && f8.block_cols % 16 == 0;
}
// ProductCfg's scale-grid fields.  slices > 1 (the selected dequantize): the weight is `slices` matrices of m.out / slices
// rows, each with a grid of its own, back to back; the per-slice fields are set for any count (1: the whole matrix).
void fp8_grid(const Fp8Scale& f8, ProductCfg& m, uint64_t slices = 1) {
  const uint64_t out = m.out / slices;
  // a block at least as tall or wide as the matrix is the whole of it: clamped, bn and bk stay below 2^31
  const uint64_t bn = std::min<uint64_t>(f8.block_rows, out), bk = std::min<uint64_t>(f8.block_cols, m.in);
  m.scale = f8.d_scale;
  m.srow = matvec_fp8_recip(bn);
  m.scol = matvec_fp8_recip(bk);
  m.scols = (uint32_t)((m.in + bk - 1) / bk);
  m.sslice = matvec_fp8_recip(out);
  m.slice_rows = (uint32_t)out;
  m.slice_grid = (uint32_t)((out + bn - 1) / bn * m.scols);
}

int product(ProductKind kind, const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, const void* d_x, size_t x_stride,
            size_t n_tokens, const void* d_bias, void* d_y, size_t y_stride, void* d_scratch, size_t scratch_bytes, cudaStream_t st,
            const Fp8Scale* f8 = nullptr) {
  if (n_tokens > max_tokens(kind)) return ZIPNN_B200_E_ARG;
  ProductCfg m;
  {
    const int rc = product_item(kind, plan, item, dtype, in_features, st, m);
    if (rc) return rc;
  }
  if (n_tokens == 0) return ZIPNN_B200_OK;
  const uint32_t xes = (uint32_t)matvec_esize(dtype);  // bytes of an element of x, y and the bias
  if (!d_x || !d_y || !d_scratch || ((uintptr_t)d_x & 15) || ((uintptr_t)d_scratch & 255) || ((uintptr_t)d_y % xes) ||
      ((uintptr_t)d_bias % xes))
    return ZIPNN_B200_E_ARG;
  if (f8 && (!f8->d_scale || ((uintptr_t)f8->d_scale & 3))) return ZIPNN_B200_E_ARG;
  if (n_tokens > 1 && ((x_stride * xes) % 16 || x_stride < m.in || y_stride < m.out)) return ZIPNN_B200_E_ARG;
  if (scratch_bytes < product_scratch_bytes(kind, m, n_tokens)) return ZIPNN_B200_E_ARG;
  m.x = d_x;
  m.bias = d_bias;
  m.y = d_y;
  m.part = (float*)d_scratch;
  m.xs = x_stride;
  m.ys = y_stride;
  m.nt = (uint32_t)n_tokens;
  if (f8) fp8_grid(*f8, m);
  const int fmt = f8 ? f8->format : kFp8E4m3;
  if (dtype == kMvBf16) return product_launch(product_kernels<kMvBf16>(kind, fmt, m.nt), m, st);
  if (dtype == kMvFp16) return product_launch(product_kernels<kMvFp16>(kind, fmt, m.nt), m, st);
  return product_launch(product_kernels<kMvFp32>(kind, fmt, m.nt), m, st);
}

// The fp8 dequantize: the fp8 matvec's item checks and scale grid, k_dequant_fp8, then the decode error folded into the
// plan's error word as after a run (k_batch_errors).  No scratch, no host read after the first call for an item.
int dequant_fp8(const zipnn_b200_decode_plan* plan, int item, const Fp8Scale& f8, int out_dtype, size_t in_features, void* d_out,
                cudaStream_t st) {
  ProductCfg m;
  {
    const int rc = product_item(kMatvecFp8, plan, item, out_dtype, in_features, st, m);
    if (rc) return rc;
  }
  if (!d_out || ((uintptr_t)d_out & 15) || !f8.d_scale || ((uintptr_t)f8.d_scale & 3)) return ZIPNN_B200_E_ARG;
  PlanState s;
  plan_state(plan, s);  // (product_item has checked it)
  m.y = d_out;
  fp8_grid(f8, m);
  const bool e4 = f8.format == kFp8E4m3;
  const ProductKernel k = out_dtype == kMvBf16 ? (e4 ? &k_dequant_fp8<kFp8E4m3, kMvBf16> : &k_dequant_fp8<kFp8E5m2, kMvBf16>)
                                               : (e4 ? &k_dequant_fp8<kFp8E4m3, kMvFp16> : &k_dequant_fp8<kFp8E5m2, kMvFp16>);
  const unsigned blocks = resident_grid(k, kSyncSmemBytes, kSyncThreads, 4 * m.K);
  if (!blocks) return ZIPNN_B200_E_CUDA;
  k<<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(m);
  ZB_LAUNCHED();
  return batch_errors(s.B, st);
}
}  // namespace

static_assert(kMatvecMaxTokens == ZIPNN_B200_MATVEC_MAX_TOKENS && kMvBf16 == ZIPNN_B200_MATVEC_BF16 && kMvFp16 == ZIPNN_B200_MATVEC_FP16 &&
                  kMvFp32 == ZIPNN_B200_MATVEC_FP32 && kMatmulMaxTokens == ZIPNN_B200_MATMUL_MAX_TOKENS &&
                  kFp8E4m3 == ZIPNN_B200_FP8_E4M3 && kFp8E5m2 == ZIPNN_B200_FP8_E5M2 &&
                  kExpertsMaxTokens == ZIPNN_B200_EXPERTS_MATVEC_MAX_TOKENS,
              "the header's constants are the kernels'");

int zipnn_b200_decode_plan_matvec_scratch_size(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, size_t n_tokens,
                                               size_t* out) {
  return product_scratch_size(kMatvec, plan, item, dtype, in_features, n_tokens, out);
}

int zipnn_b200_decode_plan_matvec(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, const void* d_x, size_t x_stride,
                                  size_t n_tokens, const void* d_bias, void* d_y, size_t y_stride, void* d_scratch, size_t scratch_bytes,
                                  void* cuda_stream) {
  return product(kMatvec, plan, item, dtype, in_features, d_x, x_stride, n_tokens, d_bias, d_y, y_stride, d_scratch, scratch_bytes,
                 (cudaStream_t)cuda_stream);
}

int zipnn_b200_decode_plan_matmul_scratch_size(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, size_t n_tokens,
                                               size_t* out) {
  return product_scratch_size(kMatmul, plan, item, dtype, in_features, n_tokens, out);
}

int zipnn_b200_decode_plan_matmul(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features, const void* d_x, size_t x_stride,
                                  size_t n_tokens, const void* d_bias, void* d_y, size_t y_stride, void* d_scratch, size_t scratch_bytes,
                                  void* cuda_stream) {
  return product(kMatmul, plan, item, dtype, in_features, d_x, x_stride, n_tokens, d_bias, d_y, y_stride, d_scratch, scratch_bytes,
                 (cudaStream_t)cuda_stream);
}

int zipnn_b200_decode_plan_matvec_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t in_features, size_t n_tokens,
                                                   size_t* out) {
  return product_scratch_size(kMatvecFp8, plan, item, kMvBf16, in_features, n_tokens, out);
}

int zipnn_b200_decode_plan_matvec_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int x_dtype, size_t in_features,
                                      const void* d_x, size_t x_stride, size_t n_tokens, const float* d_scale, size_t block_rows,
                                      size_t block_cols, const void* d_bias, void* d_y, size_t y_stride, void* d_scratch,
                                      size_t scratch_bytes, void* cuda_stream) {
  const Fp8Scale f8{fp8_format, d_scale, block_rows, block_cols};
  if (!fp8_args_ok(f8)) return ZIPNN_B200_E_ARG;
  return product(kMatvecFp8, plan, item, x_dtype, in_features, d_x, x_stride, n_tokens, d_bias, d_y, y_stride, d_scratch, scratch_bytes,
                 (cudaStream_t)cuda_stream, &f8);
}

int zipnn_b200_decode_plan_matmul_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t in_features, size_t n_tokens,
                                                   size_t* out) {
  return product_scratch_size(kMatmulFp8, plan, item, kMvBf16, in_features, n_tokens, out);
}

int zipnn_b200_decode_plan_matmul_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int x_dtype, size_t in_features,
                                      const void* d_x, size_t x_stride, size_t n_tokens, const float* d_scale, size_t block_rows,
                                      size_t block_cols, const void* d_bias, void* d_y, size_t y_stride, void* d_scratch,
                                      size_t scratch_bytes, void* cuda_stream) {
  const Fp8Scale f8{fp8_format, d_scale, block_rows, block_cols};
  if (!fp8_args_ok(f8)) return ZIPNN_B200_E_ARG;
  return product(kMatmulFp8, plan, item, x_dtype, in_features, d_x, x_stride, n_tokens, d_bias, d_y, y_stride, d_scratch, scratch_bytes,
                 (cudaStream_t)cuda_stream, &f8);
}

int zipnn_b200_decode_plan_dequant_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int out_dtype, size_t in_features,
                                       const float* d_scale, size_t block_rows, size_t block_cols, void* d_out, void* cuda_stream) {
  const Fp8Scale f8{fp8_format, d_scale, block_rows, block_cols};
  if (!fp8_args_ok(f8)) return ZIPNN_B200_E_ARG;
  return dequant_fp8(plan, item, f8, out_dtype, in_features, d_out, (cudaStream_t)cuda_stream);
}

int zipnn_b200_decode_plan_dequant_fp8_select(const zipnn_b200_decode_plan* plan, size_t rows, const void* d_ids, size_t n_ids, int id_bytes,
                                              int fp8_format, int out_dtype, int n_items, const zipnn_b200_fp8_select_item* items,
                                              void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (id_bytes != 4 && id_bytes != 8) return ZIPNN_B200_E_ARG;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  PlanState s;
  std::vector<GatherItem> gis;
  {
    const int rc = select_items(plan, rows, s, gis);
    if (rc) return rc;
  }
  if (!items || n_items <= 0 || (size_t)n_items != gis.size()) return ZIPNN_B200_E_ARG;
  if (n_items > kSelectFp8MaxItems) return ZIPNN_B200_E_UNSUPPORTED;
  SelectFp8Items d;
  memset(&d, 0, sizeof(d));
  for (int i = 0; i < n_items; i++) {
    const zipnn_b200_fp8_select_item& it = items[i];
    const Fp8Scale f8{fp8_format, it.d_scale, it.block_rows, it.block_cols};
    if (!fp8_args_ok(f8)) return ZIPNN_B200_E_ARG;
    ProductCfg& m = d.m[i];
    const int rc = product_item(kMatvecFp8, plan, i, out_dtype, it.in_features, st, m);
    if (rc) return rc;
    if (m.out % rows) return ZIPNN_B200_E_ARG;  // a slice is whole rows
    if (!it.d_out || ((uintptr_t)it.d_out & 15) || !it.d_scale || ((uintptr_t)it.d_scale & 3)) return ZIPNN_B200_E_ARG;
    m.y = it.d_out;
    fp8_grid(f8, m, rows);
  }
  if (n_ids == 0) return ZIPNN_B200_OK;
  const SelectLayout L = select_layout(s);
  {
    const int rc = select_args_ok(L, d_ids, n_ids, id_bytes, d_scratch, scratch_bytes);
    if (rc) return rc;
  }
  const SelectCfg sel = select_cfg(s, L, (uint8_t*)d_scratch, rows, d_ids, n_ids, id_bytes);
  uint64_t bitstreams = 0, tiles = 0, most = 0;
  select_bounds(gis, rows, n_ids, bitstreams, tiles, most);
  const bool e4 = fp8_format == kFp8E4m3;
  void (*const k)(SelectCfg, const SelectFp8Items) =
      out_dtype == kMvBf16 ? (e4 ? &k_select_dequant_fp8<kFp8E4m3, kMvBf16> : &k_select_dequant_fp8<kFp8E5m2, kMvBf16>)
                           : (e4 ? &k_select_dequant_fp8<kFp8E4m3, kMvFp16> : &k_select_dequant_fp8<kFp8E5m2, kMvFp16>);
  const unsigned blocks = resident_grid(k, kSyncSmemBytes, kSyncThreads, bitstreams);
  if (!blocks) return ZIPNN_B200_E_CUDA;
  k_select_index<<<1, kGatherIndexThreads, 0, st>>>(s.B, sel);
  ZB_LAUNCHED();
  k<<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(sel, d);
  ZB_LAUNCHED();
  return batch_errors(s.B, st);
}

// ---- the selected experts matvec (select.cuh): x times the routed experts of one item, from its coded bitstreams ----
// Scratch: [the select scratch][cnt u32 E][tab u32 E * nt][pos u32 n_ids][the matvec's partial sums with nt tokens],
// nt = T = n_ids / top_k rounded up to a power of two.
namespace {
struct ExpertsLayout {
  size_t cnt_off, tab_off, pos_off, part_off, bytes;
};
uint32_t experts_slots(size_t tokens) { return tokens <= 1 ? 1u : tokens <= 2 ? 2u : 4u; }
ExpertsLayout experts_layout(const PlanState& s, const ProductCfg& m, size_t rows, size_t n_ids, uint32_t nt) {
  ExpertsLayout L;
  L.cnt_off = select_layout(s).bytes;
  L.tab_off = round_up(L.cnt_off + sizeof(uint32_t) * rows, 256);
  L.pos_off = round_up(L.tab_off + sizeof(uint32_t) * rows * nt, 256);
  L.part_off = round_up(L.pos_off + sizeof(uint32_t) * n_ids, 256);
  L.bytes = L.part_off + product_scratch_bytes(kMatvecFp8, m, nt);
  return L;
}
// The checks both calls make: the plan and item (select_items, product_item), whole rows per slice, and the pairs.
// -> the item's records, m with its fields of the item and the shapes, and T.
int experts_item(const zipnn_b200_decode_plan* plan, int item, size_t rows, int x_dtype, size_t in_features, size_t n_ids,
                 size_t top_k, cudaStream_t st, PlanState& s, std::vector<GatherItem>& gis, ExpertsCfg& m, size_t& tokens) {
  {
    const int rc = select_items(plan, rows, s, gis);
    if (rc) return rc;
  }
  if (item < 0 || (size_t)item >= gis.size()) return ZIPNN_B200_E_ARG;
  memset(&m, 0, sizeof(m));
  {
    const int rc = product_item(kMatvecFp8, plan, item, x_dtype, in_features, st, m);
    if (rc) return rc;
  }
  if (m.out % rows) return ZIPNN_B200_E_ARG;  // a slice is whole rows
  if (top_k == 0 || n_ids % top_k) return ZIPNN_B200_E_ARG;
  tokens = n_ids / top_k;
  if (tokens > (size_t)kExpertsMaxTokens) return ZIPNN_B200_E_ARG;
  return ZIPNN_B200_OK;
}
}  // namespace

int zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t rows, size_t in_features,
                                                           size_t n_ids, size_t top_k, size_t* out) {
  if (!out) return ZIPNN_B200_E_ARG;
  PlanState s;
  std::vector<GatherItem> gis;
  ExpertsCfg m;
  size_t tokens = 0;
  const int rc = experts_item(plan, item, rows, kMvBf16, in_features, n_ids, top_k, nullptr, s, gis, m, tokens);
  if (rc) return rc;
  *out = experts_layout(s, m, rows, n_ids, experts_slots(tokens)).bytes;
  return ZIPNN_B200_OK;
}

int zipnn_b200_decode_plan_experts_matvec_fp8(const zipnn_b200_decode_plan* plan, int item, size_t rows, const void* d_ids, size_t n_ids,
                                              int id_bytes, size_t top_k, int fp8_format, int x_dtype, size_t in_features, const void* d_x,
                                              size_t x_stride, int x_per_pair, const float* d_scale, size_t block_rows, size_t block_cols,
                                              void* d_y, size_t y_stride, void* d_scratch, size_t scratch_bytes, void* cuda_stream) {
  if (id_bytes != 4 && id_bytes != 8) return ZIPNN_B200_E_ARG;
  const Fp8Scale f8{fp8_format, d_scale, block_rows, block_cols};
  if (!fp8_args_ok(f8)) return ZIPNN_B200_E_ARG;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  PlanState s;
  std::vector<GatherItem> gis;
  ExpertsCfg m;
  size_t tokens = 0;
  {
    const int rc = experts_item(plan, item, rows, x_dtype, in_features, n_ids, top_k, st, s, gis, m, tokens);
    if (rc) return rc;
  }
  if (n_ids == 0) return ZIPNN_B200_OK;
  const uint32_t nt = experts_slots(tokens);
  const ExpertsLayout L = experts_layout(s, m, rows, n_ids, nt);
  {
    const int rc = select_args_ok(select_layout(s), d_ids, n_ids, id_bytes, d_scratch, scratch_bytes);
    if (rc) return rc;
  }
  const uint64_t out = m.out / rows, xrows = x_per_pair ? n_ids : tokens;
  const uint32_t xes = (uint32_t)matvec_esize(x_dtype);
  if (!d_x || !d_y || ((uintptr_t)d_x & 15) || ((uintptr_t)d_y % xes) || !d_scale || ((uintptr_t)d_scale & 3)) return ZIPNN_B200_E_ARG;
  if (xrows > 1 && ((x_stride * xes) % 16 || x_stride < m.in)) return ZIPNN_B200_E_ARG;
  if (n_ids > 1 && y_stride < out) return ZIPNN_B200_E_ARG;
  if (xrows * std::max<uint64_t>(x_stride, m.in) > UINT32_MAX) return ZIPNN_B200_E_ARG;  // the x row offsets are 32-bit
  if (scratch_bytes < L.bytes) return ZIPNN_B200_E_ARG;
  uint8_t* const ws = (uint8_t*)d_scratch;
  m.x = d_x;
  m.y = d_y;
  m.part = (float*)(ws + L.part_off);
  m.xs = x_stride;
  m.ys = y_stride;
  m.nt = nt;
  fp8_grid(f8, m, rows);
  m.cnt = (uint32_t*)(ws + L.cnt_off);
  m.tab = (uint32_t*)(ws + L.tab_off);
  m.pos = (uint32_t*)(ws + L.pos_off);
  m.xdiv = matvec_fp8_recip(x_per_pair ? 1 : top_k);
  // k_select_index on a one-item view of the plan's batch: its hsel holds the item's selected bitstreams (piece 0)
  BatchCfg one = s.B;
  one.cfgs += item;
  one.chunk_start += item;
  one.n = 1;
  const SelectCfg sel = select_cfg(s, select_layout(s), ws, rows, d_ids, n_ids, id_bytes);
  uint64_t bitstreams = 0, tiles = 0, most = 0;
  select_bounds(std::vector<GatherItem>{gis[(size_t)item]}, rows, n_ids, bitstreams, tiles, most);
  const bool e4 = fp8_format == kFp8E4m3;
  void (*k)(SelectCfg, ExpertsCfg) = nullptr;
  void (*reduce)(SelectCfg, ExpertsCfg) = nullptr;
  auto pick = [&](auto xdt) {
    constexpr int XDT = decltype(xdt)::value;
    reduce = &k_select_matvec_reduce<XDT>;
    if (e4) {
      k = nt == 1 ? &k_select_matvec_fp8<kFp8E4m3, XDT, 1> : nt == 2 ? &k_select_matvec_fp8<kFp8E4m3, XDT, 2> : &k_select_matvec_fp8<kFp8E4m3, XDT, 4>;
    } else {
      k = nt == 1 ? &k_select_matvec_fp8<kFp8E5m2, XDT, 1> : nt == 2 ? &k_select_matvec_fp8<kFp8E5m2, XDT, 2> : &k_select_matvec_fp8<kFp8E5m2, XDT, 4>;
    }
  };
  if (x_dtype == kMvBf16) {
    pick(std::integral_constant<int, kMvBf16>());
  } else {
    pick(std::integral_constant<int, kMvFp16>());
  }
  const unsigned blocks = resident_grid(k, kSyncSmemBytes, kSyncThreads, bitstreams);
  if (!blocks) return ZIPNN_B200_E_CUDA;
  k_select_index<<<1, kGatherIndexThreads, 0, st>>>(one, sel);
  ZB_LAUNCHED();
  k_select_pairs<<<1, kGatherIndexThreads, 0, st>>>(sel, m);
  ZB_LAUNCHED();
  k<<<blocks, kSyncThreads, kSyncSmemBytes, st>>>(sel, m);
  ZB_LAUNCHED();
  reduce<<<(unsigned)((n_ids * out + 255) / 256), 256, 0, st>>>(sel, m);
  ZB_LAUNCHED();
  return batch_errors(s.B, st);
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
