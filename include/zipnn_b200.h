/*
 * zipnn_b200.h -- C ABI of the H100-native ZipNN encode/decode path.
 *
 * This is the drop-in boundary for the reference's native extension `zipnn_core`
 * (reference csrc/zipnn_core_module.c:9-23).  Entry points map one to one:
 *
 *   zipnn_core.zipnn_core(header, data, numBuf, bits_mode, bytes_mode, is_redata,
 *                         origChunkSize, compThreshold, checkThAfterPercent, threads)
 *       csrc/zipnn_core.c:401-417  (format "y*y*iiiinfii")
 *     -> zipnn_b200_compress / zipnn_b200_compress_host
 *
 *   zipnn_core.combine_dtype(data_after_header, numBuf, bits_mode, bytes_mode,
 *                            origChunkSize, origSize, threads)
 *       csrc/zipnn_core.c:881-892  (format "y*iiinni")
 *     -> zipnn_b200_decompress / zipnn_b200_decompress_host
 *
 *   split_bytearray_dtype{8,16,32} / combine_buffers_dtype{16,32}
 *       csrc/data_manipulation_dtype16.c:33-138,167-216, dtype32.c:78-133,219-268,391-456
 *     -> zipnn_b200_split / zipnn_b200_regroup   (stage 1 alone)
 *
 * Differences from the reference by design (SURVEY.md section 8b):
 *   - the caller owns every buffer; nothing is allocated and handed back, nothing leaks;
 *   - the input is never written to (the reference rotates sign bits in place);
 *   - `threads`, `is_redata`, `checkThAfterPercent` have no GPU meaning and are absent;
 *   - all work is enqueued on the caller's CUDA stream; the device variants only
 *     synchronise to return `*out_len` (pass out_len == NULL to stay asynchronous and
 *     read the length from the stream header bytes [24:32] yourself).
 *
 * The compressed stream is byte-for-byte the reference's stream.
 * Plain C types only: device/host pointers, sizes, `void*` for cudaStream_t.
 */
#ifndef ZIPNN_B200_H
#define ZIPNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (0 = ok).  Mirrors the reference's error sites: ------------- */
#define ZIPNN_B200_OK 0
#define ZIPNN_B200_E_ARG 1        /* bad num_buf / modes / chunk / NULL pointer                 */
#define ZIPNN_B200_E_CAPACITY 2   /* out_cap or workspace too small                              */
#define ZIPNN_B200_E_CORRUPT 3    /* stream rejected: bad type byte (zipnn_core.c:986-997), bad
                                     sizes, invalid weight table (entropy_common.c:189-210),
                                     bitstream not consumed exactly (huf_decompress.c:348-349)   */
#define ZIPNN_B200_E_CUDA 4       /* a CUDA runtime call failed; see zipnn_b200_last_cuda_error  */
#define ZIPNN_B200_E_UNSUPPORTED 5 /* valid stream using a table log of 12 (never produced by
                                     the reference encoder, which asks for 11)                   */

int zipnn_b200_version(void);                 /* 0x000200 = 0.2.0 */
const char* zipnn_b200_strerror(int status);
int zipnn_b200_last_cuda_error(void);         /* cudaError_t of the last failing runtime call */
int zipnn_b200_sm_count(void);                /* multiprocessor count of the current device   */

/* ---- sizing ------------------------------------------------------------------ */
/* Upper bound of the whole stream (python header included). */
int zipnn_b200_compress_bound(size_t n, int num_buf, size_t chunk, size_t hdr_len, size_t* out);
int zipnn_b200_compress_workspace_size(size_t n, int num_buf, size_t chunk, size_t* out);
/* Decompress workspace.  The normal size decodes ANY stream in one call: chunks that need plane scratch
 * (several Huffman-coded byte groups, a ragged tail) get one of 64 pool slots, decoded by whole-GPU
 * kernels, and every further such chunk is taken in stream order by a few persistent CTAs that own 32
 * more slots.  The `_full` size gives every chunk a pool slot: faster for streams in which EVERY chunk is
 * of that kind (e.g. an fp32 tensor upcast from bf16), never required. */
int zipnn_b200_decompress_workspace_size(size_t orig, int num_buf, size_t chunk, size_t* out);
int zipnn_b200_decompress_workspace_size_full(size_t orig, int num_buf, size_t chunk, size_t* out);

/* ---- device-resident buffers ------------------------------------------------- */
/*
 * d_in   : n bytes, the tensor viewed as bytes, 16-byte aligned, device memory (read only)
 * h_hdr  : hdr_len >= 32 bytes of python-level header (+ packed shape), HOST memory; bytes
 *          [24:32] are overwritten in the output with the total stream length
 *          (reference csrc/zipnn_core.c:121)
 * num_buf: 1 (fp8), 2 (bf16/fp16), 4 (fp32);  bits_mode: 1 = rotate the sign bit below the
 *          exponent;  bytes_mode: 10 (1 or 2 groups) or 220 (4 groups)
 * chunk  : bytes per chunk, power of two (reference default 256 KiB; 128 KiB for fp8)
 * threshold: keep a Huffman block only if size < plane_bytes * (double)threshold (:371-373)
 * d_out  : out_cap bytes of device memory;  *out_len (host, may be NULL) receives the length
 */
int zipnn_b200_compress(const void* d_in, size_t n, const void* h_hdr, size_t hdr_len, int num_buf,
                        int bits_mode, int bytes_mode, size_t chunk, float threshold, void* d_out,
                        size_t out_cap, size_t* out_len, void* d_ws, size_t ws_bytes, void* cuda_stream);

/*
 * d_body : the stream AFTER the python header (what the reference passes to combine_dtype)
 * d_out  : orig bytes, 16-byte aligned
 * Returns ZIPNN_B200_E_CORRUPT (after synchronising the stream) if the stream is invalid;
 * pass check == 0 to skip the synchronising error read-back (errors then surface on the next
 * checked call through the same workspace).
 */
int zipnn_b200_decompress(const void* d_body, size_t body_len, int num_buf, int bits_mode, int bytes_mode,
                          size_t chunk, size_t orig, void* d_out, void* d_ws, size_t ws_bytes,
                          void* cuda_stream, int check);

/* ---- many tensors at once (the checkpoint load path) --------------------------------
 * The reference decodes a safetensors file one tensor per call (zipnn/zipnn.py:1601-1607, called
 * from vLLM's weight iterator); a GPU wants the whole shard in one go.  Every item is what one
 * zipnn_b200_decompress call would take; all of them are decoded by ONE launch of each kernel
 * (tensors of up to ~3000 chunks; larger ones run one by one on the same stream).
 * Status of the whole batch: OR of the tensors' error words. */
typedef struct zipnn_b200_batch_item {
  const void* d_body;   /* stream after the python header, device memory */
  size_t body_len;
  int num_buf, bits_mode, bytes_mode;
  size_t chunk, orig;
  void* d_out;          /* orig bytes, 16-byte aligned */
} zipnn_b200_batch_item;
int zipnn_b200_decompress_batch_workspace_size(const zipnn_b200_batch_item* items, int n, size_t* out);
int zipnn_b200_decompress_batch(const zipnn_b200_batch_item* items, int n, void* d_ws, size_t ws_bytes,
                                void* cuda_stream, int check);

/* ---- stage 1 alone ------------------------------------------------------------ */
/* d_planes: num_buf planes of `stride` bytes each; plane g receives byte g of every element
 * of the (optionally rotated) input.  Lengths as in the reference: n/num_buf, the first
 * n%num_buf planes one byte longer.  The rotation covers floor(n/4) 32-bit words. */
int zipnn_b200_split(const void* d_in, size_t n, int num_buf, int bits_mode, void* d_planes, size_t stride,
                     void* cuda_stream);
int zipnn_b200_regroup(const void* d_planes, size_t stride, size_t n, int num_buf, int bits_mode, void* d_out,
                       void* cuda_stream);

/* ---- host buffers (the call the reference's Python layer makes) ----------------- */
/* Same contracts with HOST pointers: the library stages through pinned memory, copies
 * H2D, runs the kernels and copies the result D2H, all inside the call.  `h_out` must hold
 * zipnn_b200_compress_bound(...) bytes (compress) or `orig` bytes (decompress). */
int zipnn_b200_compress_host(const void* h_in, size_t n, const void* h_hdr, size_t hdr_len, int num_buf,
                             int bits_mode, int bytes_mode, size_t chunk, float threshold, void* h_out,
                             size_t out_cap, size_t* out_len);
int zipnn_b200_decompress_host(const void* h_body, size_t body_len, int num_buf, int bits_mode, int bytes_mode,
                               size_t chunk, size_t orig, void* h_out);

/* Number of kernel launches this library has enqueued since load (bench.py's gpu_launches). */
unsigned long long zipnn_b200_launch_count(void);

/* ---- optional per-kernel timing (the reference has only commented-out gettimeofday prints,
 * csrc/zipnn_core.c:409-410,562-566) ---------------------------------------------------------
 * When enabled, every kernel launch is bracketed by CUDA events on its own stream.
 * zipnn_b200_timing_collect synchronises the device, adds the elapsed milliseconds and launch
 * counts per kernel id into the caller's arrays (length >= zipnn_b200_timing_kernel_count())
 * and clears the log. */
void zipnn_b200_timing_enable(int on);
int zipnn_b200_timing_kernel_count(void);
const char* zipnn_b200_timing_kernel_name(int id);
int zipnn_b200_timing_collect(double* ms_total, unsigned long long* launches, int n);

#ifdef __cplusplus
}
#endif
#endif /* ZIPNN_B200_H */
