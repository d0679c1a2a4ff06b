// tma_probe.cu -- validates the TMA descriptor shapes the decode kernel relies on (run on an H100).
//   nvcc -O2 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tma_probe tma_probe.cu && ./tma_probe
// 1. a byte tensor {seg + 16, rows} with row stride seg (rows overlap by 16 bytes): does cuTensorMapEncodeTiled accept it?
// 2. 2-D box loads at an arbitrary byte x coordinate (the unaligned raw plane inside a stream), SWIZZLE_32B / 64B / NONE
// 3. 2-D box store {128, 32} with SWIZZLE_128B from a [32][128] stage
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <cstdlib>
#include <vector>

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeFn get_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
  return (EncodeFn)fn;
}

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int INNER>
__global__ void k_load(const __grid_constant__ CUtensorMap map, uint32_t x0, uint32_t y0, uint8_t* dst) {
  __shared__ __align__(1024) uint8_t tile[32 * INNER];
  __shared__ __align__(8) uint64_t bar;
  const int lane = threadIdx.x;
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  if (lane == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&bar)), "r"(32u * INNER) : "memory");
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(s32(tile)),
                 "l"((uint64_t)&map), "r"(x0), "r"(y0), "r"(s32(&bar))
                 : "memory");
  }
  asm volatile(
      "{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(s32(&bar)), "r"(0u)
      : "memory");
  for (int i = lane; i < 32 * INNER; i += 32) dst[i] = tile[i];
}

__global__ void k_store(const __grid_constant__ CUtensorMap map, uint32_t x0, uint32_t y0) {
  __shared__ __align__(1024) uint8_t stage[32][128];
  const int lane = threadIdx.x;
  // row = lane, 16-byte unit u at physical unit (u ^ lane) & 7; byte value encodes (row, logical byte)
  for (int u = 0; u < 8; u++)
    for (int b = 0; b < 16; b++) stage[lane][((u ^ lane) & 7) * 16 + b] = (uint8_t)(lane * 7 + u * 16 + b);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  if (lane == 0) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"((uint64_t)&map), "r"(s32(stage)), "r"(x0), "r"(y0)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  __syncwarp();
}

static int check_load(EncodeFn enc, uint8_t* d_buf, const std::vector<uint8_t>& h, size_t base_off, uint64_t seg, uint64_t rows, int inner,
                      CUtensorMapSwizzle sw, const char* name, bool overlap) {
  // tensor starts at the 16-byte aligned address at or below d_buf + base_off
  const uint64_t r0 = ((uintptr_t)(d_buf + base_off)) & 15;
  void* ga = d_buf + base_off - r0;
  CUtensorMap m;
  cuuint64_t dims[2] = {overlap ? seg + 16 : seg, rows};
  cuuint64_t strides[1] = {seg};
  cuuint32_t box[2] = {(cuuint32_t)inner, 32};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, ga, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  printf("%-28s encode(overlap=%d) -> %d\n", name, (int)overlap, (int)r);
  if (r != CUDA_SUCCESS) return 1;
  uint8_t* d_dst;
  cudaMalloc(&d_dst, 32 * inner);
  int bad_total = 0;
  const uint32_t xs[3] = {(uint32_t)r0, (uint32_t)(r0 + (seg / 2 / 16) * 16), (uint32_t)(r0 + seg - inner + (overlap ? 16 : 0))};  // first, middle, LAST tile of a segment
  for (int t = 0; t < 3; t++) {
    const uint32_t y0 = 32;
    cudaMemset(d_dst, 0xEE, 32 * inner);
    if (inner == 16) k_load<16><<<1, 32>>>(m, xs[t], y0, d_dst);
    if (inner == 32) k_load<32><<<1, 32>>>(m, xs[t], y0, d_dst);
    if (inner == 64) k_load<64><<<1, 32>>>(m, xs[t], y0, d_dst);
    if (inner == 48) k_load<48><<<1, 32>>>(m, xs[t], y0, d_dst);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("  kernel error %s\n", cudaGetErrorString(e)); return 1; }
    std::vector<uint8_t> got(32 * inner);
    cudaMemcpy(got.data(), d_dst, got.size(), cudaMemcpyDeviceToHost);
    int bad = 0;
    const int chunks = inner / 16;
    for (int row = 0; row < 32; row++)
      for (int i = 0; i < inner; i++) {
        const size_t src = base_off - r0 + (size_t)(y0 + row) * seg + xs[t] + i;
        int phys_chunk = i / 16;
        if (sw == CU_TENSOR_MAP_SWIZZLE_32B) phys_chunk ^= ((row * inner) >> 7) & 1;
        if (sw == CU_TENSOR_MAP_SWIZZLE_64B) phys_chunk ^= ((row * inner) >> 7) & 3;
        if (sw == CU_TENSOR_MAP_SWIZZLE_128B) phys_chunk ^= ((row * inner) >> 7) & 7;
        (void)chunks;
        const uint8_t g = got[row * inner + phys_chunk * 16 + (i & 15)];
        if (g != h[src]) bad++;
      }
    printf("  x0=%u: %d mismatching bytes of %d\n", xs[t], bad, 32 * inner);
    bad_total += bad;
  }
  cudaFree(d_dst);
  return bad_total;
}

int main(int argc, char** argv) {
  // one test per process: a faulting kernel poisons the context
  const int test = argc > 1 ? atoi(argv[1]) : 0;
  EncodeFn enc = get_encode();
  if (!enc) { printf("no cuTensorMapEncodeTiled entry point\n"); return 2; }
  const uint64_t seg = 32768, rows = 256;
  const size_t total = seg * rows + 4096;
  std::vector<uint8_t> h(total);
  for (size_t i = 0; i < total; i++) h[i] = (uint8_t)((i * 2654435761u) >> 13);
  uint8_t* d;
  cudaMalloc(&d, total);
  cudaMemcpy(d, h.data(), total, cudaMemcpyHostToDevice);
  int fails = 0;
  switch (test) {
    case 0: fails = check_load(enc, d, h, 0, seg, rows, 16, CU_TENSOR_MAP_SWIZZLE_NONE, "T0 aligned, 16B, no swizzle", false); break;
    case 1: fails = check_load(enc, d, h, 1029, seg, rows, 16, CU_TENSOR_MAP_SWIZZLE_NONE, "T1 unaligned x, 16B, no swizzle", false); break;
    case 2: fails = check_load(enc, d, h, 77, seg, rows, 32, CU_TENSOR_MAP_SWIZZLE_32B, "T2 unaligned x, 32B, swizzle32", false); break;
    case 3: fails = check_load(enc, d, h, 77, seg, rows, 64, CU_TENSOR_MAP_SWIZZLE_64B, "T3 unaligned x, 64B, swizzle64", false); break;
    case 4: fails = check_load(enc, d, h, 1024, seg, rows, 16, CU_TENSOR_MAP_SWIZZLE_NONE, "T4 overlap rows, 16B, aligned x", true); break;
    case 5: fails = check_load(enc, d, h, 64, seg, rows, 32, CU_TENSOR_MAP_SWIZZLE_32B, "T5 overlap rows, 32B swizzle32, aligned x", true); break;
    case 6: fails = check_load(enc, d, h, 64, seg, rows, 64, CU_TENSOR_MAP_SWIZZLE_64B, "T6 overlap rows, 64B swizzle64, aligned x", true); break;
    case 9: fails = check_load(enc, d, h, 64, seg, rows, 48, CU_TENSOR_MAP_SWIZZLE_NONE, "T9 overlap rows, 48B rows, last tile spills 16 B into the next row", true); break;
    case 7: fails = check_load(enc, d, h, 0, seg, rows, 32, CU_TENSOR_MAP_SWIZZLE_NONE, "T7 aligned, 32B, no swizzle", false); break;
    case 8: {
      const uint64_t rowb = 65536, nrows = 64;
      uint8_t* o;
      cudaMalloc(&o, rowb * nrows);
      cudaMemset(o, 0, rowb * nrows);
      CUtensorMap m;
      cuuint64_t dims[2] = {rowb, nrows};
      cuuint64_t strides[1] = {rowb};
      cuuint32_t box[2] = {128, 32}, es[2] = {1, 1};
      CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, o, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      printf("T8 store map encode -> %d\n", (int)r);
      if (r == CUDA_SUCCESS) {
        k_store<<<1, 32>>>(m, 128 * 5, 32);
        cudaError_t e = cudaDeviceSynchronize();
        printf("store kernel: %s\n", cudaGetErrorString(e));
        std::vector<uint8_t> ho(rowb * nrows);
        cudaMemcpy(ho.data(), o, ho.size(), cudaMemcpyDeviceToHost);
        int bad = 0;
        for (int row = 0; row < 32; row++)
          for (int b = 0; b < 128; b++)
            if (ho[(size_t)(32 + row) * rowb + 128 * 5 + b] != (uint8_t)(row * 7 + b)) bad++;
        printf("store: %d mismatching bytes of 4096\n", bad);
        fails = bad;
      } else fails = 1;
    } break;
  }
  printf("test %d: %s\n", test, fails ? "FAILED" : "ok");
  return 0;
}
