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
 *     read the length from the stream header bytes [24:32] yourself).  zipnn_b200_compress
 *     waits for the length alone: it returns while the last kernels that write the stream
 *     may still run, so the stream is ready for what is enqueued on the same CUDA stream
 *     after the call (another stream must wait for that one first).
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
#define ZIPNN_B200_E_CORRUPT 3    /* stream rejected (DESIGN §6): body shorter than its tables, a
                                     group total past the payload, a decreasing or out-of-group
                                     size row, bad type byte (zipnn_core.c:986-997), a stored item
                                     not exactly its plane's length, a coded item on an empty plane
                                     or longer than its plane, invalid weight table
                                     (entropy_common.c:189-210), a bitstream not consumed exactly
                                     as HUF_decompress4X1 requires (huf_decompress.c:348-349)    */
#define ZIPNN_B200_E_CUDA 4       /* a CUDA runtime call failed; see zipnn_b200_last_cuda_error  */
#define ZIPNN_B200_E_UNSUPPORTED 5 /* valid stream using a table log of 12 (never produced by
                                     the reference encoder, which asks for 11)                   */
#define ZIPNN_B200_E_INDEX 6      /* a decode plan gather met an id outside [0, rows)            */

int zipnn_b200_version(void);                 /* 0x000200 = 0.2.0 */
const char* zipnn_b200_strerror(int status);
int zipnn_b200_last_cuda_error(void);         /* cudaError_t of the last failing runtime call */
int zipnn_b200_sm_count(void);                /* multiprocessor count of the current device   */
/* Copy n <= 4096 bytes of device memory to host memory once the work enqueued on cuda_stream before the call
 * is done (synchronises the stream, through a pinned block): the look at a stream's header that sizes a decode. */
int zipnn_b200_peek(const void* d_src, size_t n, void* h_dst, void* cuda_stream);

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

/* ---- many tensors at once (the checkpoint save path) --------------------------------
 * The reference compresses a safetensors file one zipnn_core call per tensor
 * (scripts/zipnn_compress_safetensors.py:77-97).  Every item is what one zipnn_b200_compress call
 * would take, and its stream is byte for byte what that call writes, whatever the other items are.
 * All items are coded by ONE launch of each encode kernel per byte-group class (num_buf) present,
 * plus one memset and one host-to-device copy, all on cuda_stream; the launch count does not depend
 * on the number of items.  Every item is checked before anything is enqueued (the rules of
 * zipnn_b200_compress: E_ARG, E_CAPACITY); a bad item means nothing is written.
 * out_lens: NULL -> the call stays asynchronous, each stream's bytes [24:32] carry its length;
 *           else a host array of n lengths, filled after ONE synchronisation of the stream. */
typedef struct zipnn_b200_compress_item {
  const void* d_in; size_t n;          /* device, 16-byte aligned (as zipnn_b200_compress)          */
  const void* h_hdr; size_t hdr_len;   /* host, 32..4096 bytes; [24:32] patched in the output        */
  int num_buf, bits_mode, bytes_mode;
  size_t chunk; float threshold;
  void* d_out; size_t out_cap;         /* out_cap >= zipnn_b200_compress_bound(n, num_buf, chunk, hdr_len) */
} zipnn_b200_compress_item;
int zipnn_b200_compress_batch_workspace_size(const zipnn_b200_compress_item* items, int n, size_t* out);
int zipnn_b200_compress_batch(const zipnn_b200_compress_item* items, int n, size_t* out_lens,
                              void* d_ws, size_t ws_bytes, void* cuda_stream);

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
 * Status of the whole batch: OR of the tensors' error words.  An item whose body is shorter than its own
 * type and size tables is refused (E_CORRUPT) before anything is enqueued: no item is decoded then. */
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

/* ---- slices: a box of each stream's decoded bytes (sharded loads) --------------------------
 * Row r of the box is decoded bytes [base + r*pitch, base + r*pitch + len), r in [0, rows); d_out
 * receives the rows*len bytes packed row after row.  A slice of a row-major tensor along dim 0 is
 * one row; along a later dim, one row per index of the dims in front of it.
 * Only the chunks the box touches are read and validated: a chunk outside it is never dereferenced
 * (the totals of the size table are still checked), so a corrupt byte there goes unnoticed.  Every
 * item is decoded by the per-bitstream-CTA kernels, all items by ONE launch of each, whatever their
 * size; a box that covers more than 16384 chunks is split into several pieces internally.
 * E_ARG: a box past `orig`, len > pitch with rows > 1, or a misaligned d_out.  Empty boxes (rows or
 * len 0) are valid and do nothing.  Status: OR of the items' error words, as in the batch call. */
typedef struct zipnn_b200_slice_item {
  const void* d_body; size_t body_len;   /* a whole stream after the python header, or a sub-stream of
                                            consecutive chunks with rebased size rows                  */
  int num_buf, bits_mode, bytes_mode;
  size_t chunk, orig;                    /* orig = decoded bytes of THIS (sub)stream                    */
  size_t base, rows, pitch, len;         /* the box, in the decoded bytes of this (sub)stream           */
  void* d_out;                           /* rows*len bytes, 16-byte aligned                              */
} zipnn_b200_slice_item;
int zipnn_b200_decompress_slices_workspace_size(const zipnn_b200_slice_item* items, int n, size_t* out);
int zipnn_b200_decompress_slices(const zipnn_b200_slice_item* items, int n, void* d_ws, size_t ws_bytes,
                                 void* cuda_stream, int check);

/* ---- decode plans: decode the same streams again and again (weights kept compressed in HBM) ----------
 * A plan splits a slice decode into what depends only on the streams -- validation, item tables, work lists,
 * parsed Huffman tables and the start of every segment of the per-bitstream-CTA decoder, done once by _create --
 * and a run that only enqueues kernels: at most four launches whatever n is (one when every item is empty), no
 * host-to-device copy, no memset, no synchronisation, so a run can be captured in a CUDA graph.  A run decodes
 * each segment once from its recorded start instead of searching for the starts.  Every run writes the same
 * bytes to the same d_out addresses.
 * Items are slice items (a whole tensor: base 0, rows 1, len orig); they follow the rules of
 * zipnn_b200_decompress_slices, large boxes are split into pieces the same way, and a piece that is a whole
 * tensor decodes without the window.
 * Memory, owned by the caller, split by lifetime:
 *   plan memory  (plan_bytes, 256-byte aligned): descriptors, item tables, work lists, parsed tables, RLE fill
 *                blocks, the error word and the segment index (8 KiB per Huffman-coded item); must stay
 *                allocated and untouched while the plan is used;
 *   scratch      (scratch_bytes, 256-byte aligned): plane pools, written and read within one run only.  Plans
 *                whose runs are ordered on one stream may share one scratch buffer.
 * The streams (d_body) must stay allocated at the same address and unchanged, and d_out allocated, for the life
 * of the plan.
 * _size synchronises cuda_stream: it reads each item's type rows to count its coded items.
 * _create checks every item, decodes once into every d_out (recording the segment starts), synchronises
 * cuda_stream and returns that decode's status (E_CORRUPT, E_UNSUPPORTED, ...); a plan whose create failed makes
 * _run, _status and _index return E_ARG.
 * _status synchronises cuda_stream and returns the error word of the plan's runs so far.
 * _index gives the bytes of the plan's segment index and the coded items it covers. */
typedef struct zipnn_b200_decode_plan { uint64_t opaque[16]; } zipnn_b200_decode_plan;   /* host, filled by _create */
int zipnn_b200_decode_plan_size(const zipnn_b200_slice_item* items, int n, void* cuda_stream,
                                size_t* plan_bytes, size_t* scratch_bytes);
int zipnn_b200_decode_plan_create(const zipnn_b200_slice_item* items, int n, void* d_plan, size_t plan_bytes,
                                  void* d_scratch, size_t scratch_bytes, zipnn_b200_decode_plan* plan, void* cuda_stream);
int zipnn_b200_decode_plan_run(const zipnn_b200_decode_plan* plan, void* cuda_stream);
int zipnn_b200_decode_plan_status(const zipnn_b200_decode_plan* plan, void* cuda_stream);
int zipnn_b200_decode_plan_index(const zipnn_b200_decode_plan* plan, size_t* index_bytes, size_t* coded_items);
/* _run_shifted: the decode of _run as ONE kernel launch (no copy, memset or synchronisation: capturable in a CUDA
 * graph) of at most max_ctas CTAs, with every item's output at d_out + out_shift instead of d_out.  Each target
 * must be allocated and as large as the item's output; out_shift must be a multiple of 16 (else E_ARG).
 * max_ctas <= 0: as many CTAs as fit on the device at once; larger values are capped to that.  With few CTAs the
 * decode leaves the other SMs to concurrent work (a decode of the next layer's weights next to this layer's GEMMs).
 * Plans without a segment index (ZIPNN_B200_PLAN_REPLAY=0 at create) return E_UNSUPPORTED.  Errors reach the
 * word _status reads.  Lifetime and scratch rules are _run's: runs of one plan, and runs of plans that share a
 * scratch buffer, must be ordered on one stream, whichever of _run and _run_shifted enqueues them. */
int zipnn_b200_decode_plan_run_shifted(const zipnn_b200_decode_plan* plan, int64_t out_shift, int max_ctas,
                                       void* cuda_stream);
/* _gather: rows of item `item` (a whole tensor) looked up by ids on the device, decoding only the chunks they touch.
 * The item's decoded bytes are rows of row_bytes bytes; for t in [0, n_ids): d_out[t*row_bytes, +row_bytes) =
 * row d_ids[t] (int32 or int64 ids: id_bytes 4 or 8, aligned to their size).  No alignment is asked of d_out.
 * Launches only (no copy, memset or synchronisation: capturable in a CUDA graph, replayable with new ids in d_ids):
 * 1 + 2 * passes launches, passes = ceil(min(n_ids * span, K) / slots), where span = floor((row_bytes + chunk - 2) /
 * chunk) + 1 (at most K) is the most chunks a row can touch, K the item's chunks, and slots what scratch_bytes holds.
 * So the count depends on n_ids and the buffers, never on the id values.  n_ids == 0 launches nothing.
 * An id outside [0, rows) (negative included) reads nothing and its row of d_out is zeroed; it sets ZIPNN_B200_E_INDEX
 * in the plan's error word, which _status returns (after E_CORRUPT, E_UNSUPPORTED and E_CAPACITY) from then on: the
 * word is sticky for the plan's life, like every error of its runs.
 * d_scratch (256-byte aligned, scratch_bytes from _gather_scratch_size for some slot count >= 1; more slots mean
 * fewer passes) holds nothing between calls: like the plan scratch, calls that share it must be ordered on one
 * stream, and it may be the scratch of plan runs ordered on that stream.  The plan's own scratch is not used, so a
 * gather may run next to a _run_shifted of the same plan on another stream.
 * Host-side rejections launch and write nothing: E_ARG for id_bytes other than 4 or 8, row_bytes 0 or not dividing
 * the item's bytes, a NULL d_ids, d_out or d_scratch (n_ids > 0), misaligned ids or scratch, a scratch smaller than
 * one slot, an item index out of range, or a plan whose create failed; E_UNSUPPORTED for an item that is a box, is
 * empty or was split into several pieces (16384 chunks or more), and for a plan without a segment index.
 * _gather_scratch_size: the scratch bytes of `slots` slots (capped to K; slots >= 1), same checks. */
int zipnn_b200_decode_plan_gather_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t row_bytes,
                                               size_t slots, size_t* out);
int zipnn_b200_decode_plan_gather(const zipnn_b200_decode_plan* plan, int item, size_t row_bytes, const void* d_ids,
                                  size_t n_ids, int id_bytes, void* d_out, void* d_scratch, size_t scratch_bytes,
                                  void* cuda_stream);

/* _run_select: the plan run for the slices that ids select, and nothing else (the routed experts of a mixture-of-
 * experts layer).  Every item is seen as `rows` slices along dim 0 of item bytes / rows bytes each; for every id e in
 * d_ids (n_ids of them, int32 or int64: id_bytes 4 or 8, aligned to their size, duplicates allowed) the bytes of slice
 * e of every item are written to the item's d_out, as _run writes them.  Exactly the chunks that meet a selected slice
 * are decoded, whole (a chunk that straddles two slices included), and no other byte of any d_out is written: the
 * other slices keep whatever they held.
 * Launches only (no copy, memset or synchronisation: capturable in a CUDA graph, replayable with new ids in d_ids): 5
 * launches whatever the id values are -- an index kernel that compacts the plan's work lists to the selected chunks,
 * the replay decoder, the regroup and the overflow decoder over those lists, and the plan run's error pass.  The
 * grids depend on n_ids, never on the id values.  n_ids == 0 launches nothing.
 * An id outside [0, rows) (negative included) selects nothing and sets ZIPNN_B200_E_INDEX in the plan's error word,
 * which _status returns (sticky, as for _gather).
 * d_scratch (256-byte aligned, at least _select_scratch_size bytes) holds nothing between calls: calls that share it
 * must be ordered on one stream, as for _gather.  It must not overlap the plan's own scratch, which a selected run
 * uses as _run does (runs of one plan, and of plans sharing that scratch, ordered on one stream).
 * Host-side rejections launch and write nothing: E_ARG for id_bytes other than 4 or 8, rows 0 or not dividing some
 * item's bytes, a NULL d_ids or d_scratch (n_ids > 0), misaligned ids or scratch, a scratch below
 * _select_scratch_size, or a plan whose create failed; E_UNSUPPORTED for a plan without items, a plan without a
 * segment index, or an item that is not one whole-tensor piece (a box, an empty item, or one split into pieces:
 * 16384 chunks or more).
 * _select_scratch_size: the scratch bytes, same checks; they depend on the plan alone. */
int zipnn_b200_decode_plan_select_scratch_size(const zipnn_b200_decode_plan* plan, size_t rows, size_t* out);
int zipnn_b200_decode_plan_run_select(const zipnn_b200_decode_plan* plan, size_t rows, const void* d_ids, size_t n_ids,
                                      int id_bytes, void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* _matvec: y = x W^T (+ bias) for a few rows of x, straight from the coded bitstreams of item `item`: the dense W is
 * never written or read back.  W is the item's decoded tensor, row-major [out_features][in_features] of `dtype`
 * (out_features = the item's elements / in_features); x is n_tokens rows of in_features elements, x_stride elements
 * apart; y is n_tokens rows of out_features elements, y_stride apart; x, y and the optional d_bias (out_features
 * elements, or NULL) have the weight's dtype.  Products and sums are fp32; each y is rounded once.
 * Launches: 2 whatever n_tokens and the shapes are -- the plan run's per-bitstream replay decoder, whose fused merge
 * multiplies each 16 bytes it forms with x instead of storing them and writes one fp32 partial sum per (block of the
 * tensor, row it touches, token) to d_scratch, and a reduction that adds each row's partial sums in ascending element
 * order.  No atomics on floats, no copy, memset or synchronisation: capturable in a CUDA graph, replayable with new x,
 * and two calls with the same inputs give the same bits.  n_tokens == 0 launches nothing.
 * Eligible items (else E_UNSUPPORTED, and the caller decodes the item as before): a whole tensor in one piece (not a
 * box, not empty, at most 16383 chunks) of a plan with a segment index; num_buf equal to the dtype's size;
 * in_features * element size a multiple of 16; every chunk in the fused decode mode (one coded plane, the top byte
 * plane; chunk length a multiple of 512) -- what float weights produce.  The first _matvec or _matvec_scratch_size call
 * for an item reads its chunk modes from the device and synchronises cuda_stream (the null stream for _scratch_size);
 * later calls do not.
 * Host-side rejections launch and write nothing: E_ARG for n_tokens above ZIPNN_B200_MATVEC_MAX_TOKENS, a dtype other
 * than the three below, in_features 0 or not dividing the item's elements, an item index out of range, a plan whose
 * create failed, and with n_tokens > 0: a NULL d_x, d_y or d_scratch, d_x not 16-byte aligned, x_stride * element size
 * not a multiple of 16 or a stride shorter than its row (n_tokens > 1), d_y or d_bias not aligned to the element,
 * d_scratch not 256-byte aligned, scratch_bytes below _matvec_scratch_size.
 * d_scratch holds nothing between calls: calls that share it must be ordered on one stream, and it may be the plan
 * scratch of runs ordered on that stream.  The plan's own scratch and outputs are not touched, so a matvec may run next
 * to a _run_shifted of the same plan on another stream.  Decode errors reach the word _status reads. */
#define ZIPNN_B200_MATVEC_MAX_TOKENS 8
#define ZIPNN_B200_MATVEC_BF16 0
#define ZIPNN_B200_MATVEC_FP16 1
#define ZIPNN_B200_MATVEC_FP32 2
int zipnn_b200_decode_plan_matvec_scratch_size(const zipnn_b200_decode_plan* plan, int item, int dtype,
                                               size_t in_features, size_t n_tokens, size_t* out);
int zipnn_b200_decode_plan_matvec(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features,
                                  const void* d_x, size_t x_stride, size_t n_tokens, const void* d_bias, void* d_y,
                                  size_t y_stride, void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* _matmul: what _matvec computes, for up to ZIPNN_B200_MATMUL_MAX_TOKENS rows of x, on tensor cores (mma.m16n8k16
 * with fp32 accumulation): the dense W is never written or read back.  Arguments, eligible items, the first call's
 * read of the chunk modes, the scratch and stream rules and the error reporting are those of _matvec.  bf16 and fp16
 * only: ZIPNN_B200_MATVEC_FP32 answers E_UNSUPPORTED, and the caller decodes the item as before.
 * Launches: 2 whatever n_tokens and the shapes are -- the plan run's per-bitstream replay decoder, whose fused merge
 * hands each 16 bytes it forms to the tensor cores as a fragment of 8 rows x 32 columns of W, and writes one fp32
 * partial sum per (bitstream, tile of 8 rows it touches, token, row) to d_scratch, and a reduction that adds each row's
 * partial sums in ascending element order, adds the bias and rounds once.  No atomics on floats, no copy, memset or
 * synchronisation: capturable in a CUDA graph, replayable with new x, and two calls with the same inputs give the same
 * bits.  The tensor cores' fp32 sums are not rounded to nearest at every addition, so a result may differ from
 * _matvec's in the last bits.  n_tokens == 0 launches nothing.  x must be finite: an infinity in x can give NaN in a
 * row that straddles two bitstreams where the dense product gives an infinity.
 * Host-side rejections launch and write nothing: E_ARG as for _matvec, with ZIPNN_B200_MATMUL_MAX_TOKENS as the row
 * limit and scratch_bytes below _matmul_scratch_size; E_UNSUPPORTED for fp32 and for every item _matvec refuses. */
#define ZIPNN_B200_MATMUL_MAX_TOKENS 64
int zipnn_b200_decode_plan_matmul_scratch_size(const zipnn_b200_decode_plan* plan, int item, int dtype,
                                               size_t in_features, size_t n_tokens, size_t* out);
int zipnn_b200_decode_plan_matmul(const zipnn_b200_decode_plan* plan, int item, int dtype, size_t in_features,
                                  const void* d_x, size_t x_stride, size_t n_tokens, const void* d_bias, void* d_y,
                                  size_t y_stride, void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* _matvec_fp8: y = x (S . W)^T (+ bias) for fp8 weights with an fp32 scale grid, straight from the coded bitstreams of
 * item `item` as _matvec does it: W is the item's decoded tensor, row-major [out_features][in_features] of
 * float8_e4m3fn (fp8_format ZIPNN_B200_FP8_E4M3) or float8_e5m2 (ZIPNN_B200_FP8_E5M2); d_scale is the contiguous fp32
 * grid [ceil(out_features / block_rows)][ceil(in_features / block_cols)], and the weight the product uses is
 * float(W[o][i]) * S[o / block_rows][i / block_cols] (the stored scale multiplies, as `weight_scale_inv` in fp8
 * checkpoints).  (out_features, in_features) is one scale for the tensor, (1, in_features) one per row, (128, 128)
 * DeepSeek's blocks, ragged at the edges.  x, y and the optional d_bias have x_dtype, ZIPNN_B200_MATVEC_BF16 or _FP16.
 * Each lane of the kernel adds the products of 16 consecutive weights of a row with x in ascending column order (fp32
 * FMAs), multiplies the sum by the block's scale once, and from there the sums, their order, the rounding, the launches
 * (2; none for n_tokens == 0), graph capture, determinism and the first call's read of the chunk modes are _matvec's.
 * An e4m3fn NaN or an e5m2 infinity or NaN in W gives what the dense product of the dequantized matrix gives: NaN or
 * an infinity in that row of y.
 * Eligible items (else E_UNSUPPORTED): those _matvec takes, with num_buf 1 (fp8 streams).
 * Host-side rejections launch and write nothing: E_ARG as for _matvec (x_dtype in place of dtype, the alignments of x,
 * y and d_bias those of x_dtype), and for an fp8_format other than the two below, an x_dtype other than BF16 or FP16,
 * block_rows 0, block_cols below 16 or not a multiple of 16, and with n_tokens > 0 a NULL or not 4-byte aligned
 * d_scale.  _matvec_fp8_scratch_size: the scratch bytes (_matvec's formula), the same item checks. */
#define ZIPNN_B200_FP8_E4M3 0
#define ZIPNN_B200_FP8_E5M2 1
int zipnn_b200_decode_plan_matvec_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t in_features,
                                                   size_t n_tokens, size_t* out);
int zipnn_b200_decode_plan_matvec_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int x_dtype,
                                      size_t in_features, const void* d_x, size_t x_stride, size_t n_tokens,
                                      const float* d_scale, size_t block_rows, size_t block_cols,
                                      const void* d_bias, void* d_y, size_t y_stride,
                                      void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* _matmul_fp8: y = x D^T (+ bias) for up to ZIPNN_B200_MATMUL_MAX_TOKENS rows of x, on tensor cores, with D the weight
 * _dequant_fp8 writes for the same arguments: D[o][i] = x_dtype(float(W[o][i]) * S[o / block_rows][i / block_cols]),
 * neither written nor read dense.  Arguments, eligible items, the host-side rejections (E_ARG as _matvec_fp8, with
 * ZIPNN_B200_MATMUL_MAX_TOKENS as the row limit and scratch_bytes below _matmul_fp8_scratch_size; E_UNSUPPORTED for
 * every item _matvec_fp8 refuses) and the first call's read of the chunk modes are _matvec_fp8's.  Each 16 fp8 weights
 * the replay decoder forms are dequantized to x_dtype exactly as _dequant_fp8 rounds them, and go to mma.m16n8k16 in
 * x_dtype with fp32 accumulation as B fragments of 8 rows x 64 columns; from there the partial sums, their order, the
 * rounding, the launches (2; none for n_tokens == 0), graph capture, determinism and the finite-x rule are _matmul's.
 * So a result is F.linear of _dequant_fp8's weight up to the order of the fp32 sums.  An e4m3fn NaN or an e5m2
 * infinity or NaN in W, or an fp16 overflow in D, gives NaN or an infinity in that row of y as that F.linear does.
 * _matmul_fp8_scratch_size: the scratch bytes (_matmul's formula), the same item checks. */
int zipnn_b200_decode_plan_matmul_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t in_features,
                                                   size_t n_tokens, size_t* out);
int zipnn_b200_decode_plan_matmul_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int x_dtype,
                                      size_t in_features, const void* d_x, size_t x_stride, size_t n_tokens,
                                      const float* d_scale, size_t block_rows, size_t block_cols,
                                      const void* d_bias, void* d_y, size_t y_stride,
                                      void* d_scratch, size_t scratch_bytes, void* cuda_stream);

/* _dequant_fp8: the dequantized weight of an item _matvec_fp8 takes, written straight from its coded bitstreams:
 * d_out[o][i] = out_dtype(float(W[o][i]) * S[o / block_rows][i / block_cols]), W, d_scale and the blocks as for
 * _matvec_fp8, d_out a contiguous [out_features][in_features] tensor of out_dtype, ZIPNN_B200_MATVEC_BF16 or _FP16.
 * The values are bit for bit torch's (W.to(float32) * S_expanded).to(out_dtype): fp8 -> fp32 is exact, then one fp32
 * multiply and one round to nearest even; fp16 overflow gives +-inf, NaN stays NaN (its payload may differ).  Exactly
 * out_features * in_features elements are written.  Two launches (the decode with the dequantizing store, then the
 * fold of a decode error into the plan's error word, which _status reports), no scratch, no host read but the first
 * call's read of the chunk modes (as _matvec): capturable in a CUDA graph.
 * Eligible items (else E_UNSUPPORTED): those _matvec_fp8 takes.
 * Host-side rejections launch and write nothing: E_ARG as _matvec_fp8 refuses fp8_format, the blocks, d_scale, the
 * plan, the item and in_features, and for an out_dtype other than BF16 or FP16 and a NULL or not 16-byte aligned d_out. */
int zipnn_b200_decode_plan_dequant_fp8(const zipnn_b200_decode_plan* plan, int item, int fp8_format, int out_dtype,
                                       size_t in_features, const float* d_scale, size_t block_rows, size_t block_cols,
                                       void* d_out, void* cuda_stream);

/* _dequant_fp8_select: _dequant_fp8 restricted to the slices that ids select, the selected run of _run_select with
 * _dequant_fp8's stores (the routed experts of an fp8 mixture-of-experts layer: gate_up_proj [E, 2I, H] and down_proj
 * [E, H, I] with a scale grid per expert).  Every item is `rows` slices along dim 0 (E experts); item i is seen as
 * rows * out_i rows of items[i].in_features elements, slice e its rows [e * out_i, (e + 1) * out_i), and
 * items[i].d_out is a contiguous [rows * out_i][in_features] tensor of out_dtype (ZIPNN_B200_MATVEC_BF16 or _FP16),
 * 16-byte aligned.  items[i].d_scale is the contiguous fp32 [rows][ceil(out_i / bn)][ceil(in / bk)] of the per-slice
 * grids, (bn, bk) = (block_rows, block_cols) clamped to (out_i, in_features) as for _dequant_fp8: (out_i, in) is one
 * scale per slice.  For every chunk of an item that meets a selected slice, every element of the chunk is written,
 * d_out[r][c] = out_dtype(float(W[r][c]) * S[r / out_i][(r % out_i) / bn][c / bk]): bit for bit torch's dequantize of
 * each slice, as _dequant_fp8 writes it.  A chunk that straddles two slices writes its neighbour's elements too (with
 * their own scales), and no other element of any d_out is written.
 * Three launches whatever the id values are (the index kernel of _run_select, the replay decoder with the dequantizing
 * stores, the plan run's error pass), no copy and no host read but the first call's read of each item's chunk modes:
 * capturable in a CUDA graph, replayable with new ids and new scales.  Ids, the scratch (_select_scratch_size bytes,
 * not the plan's own scratch), E_INDEX and n_ids == 0 as for _run_select.
 * Eligible plans (else E_UNSUPPORTED): those _run_select takes, with at most 4 items, each of which _dequant_fp8 takes
 * (fused fp8 chunks, in_features a multiple of 16); all items in one fp8_format.
 * Host-side rejections launch and write nothing: E_ARG as _run_select refuses rows, ids and scratch, as _dequant_fp8
 * refuses fp8_format, out_dtype, in_features, the blocks, d_scale and d_out, for NULL items, n_items other than the
 * plan's item count, and an item whose slices are not whole rows. */
typedef struct zipnn_b200_fp8_select_item {
  size_t in_features;
  const float* d_scale;
  size_t block_rows, block_cols;
  void* d_out;
} zipnn_b200_fp8_select_item;
int zipnn_b200_decode_plan_dequant_fp8_select(const zipnn_b200_decode_plan* plan, size_t rows, const void* d_ids,
                                              size_t n_ids, int id_bytes, int fp8_format, int out_dtype, int n_items,
                                              const zipnn_b200_fp8_select_item* items, void* d_scratch,
                                              size_t scratch_bytes, void* cuda_stream);

/* _experts_matvec_fp8: the routed experts of one item of an fp8 mixture-of-experts plan times x, from the coded
 * bitstreams of the chunks they meet; no weight is written.  The plan is one _dequant_fp8_select takes (every item
 * `rows` = E slices along dim 0); item `item` is seen as E experts [out][in_features], out = its rows / E, with the
 * per-expert scale grid d_scale [E][ceil(out / bn)][ceil(in / bk)] and blocks as for _dequant_fp8_select.  d_ids holds
 * n_ids = T * top_k expert ids (id_bytes 4 or 8), pair p = t * top_k + j; T <= ZIPNN_B200_EXPERTS_MATVEC_MAX_TOKENS (4:
 * a lane holds one fp32 sum per pair slot, and 8 slots do not fit the decoder's 80 registers without spills).  For every
 * pair p with an id in [0, E):
 *   d_y[p * y_stride + o] = x_dtype(sum_i x_p[i] * (float(W[ids[p]][o][i]) * S[ids[p]][o / bn][i / bk]))
 * with x_p row p / top_k of d_x (x_per_pair == 0: one row per token) or row p (x_per_pair != 0: one row per pair), rows
 * x_stride elements apart, of x_dtype (ZIPNN_B200_MATVEC_BF16 or _FP16).  Bit for bit _matvec_fp8 of the item seen as
 * [E * out][in] with x = x_p, rows ids[p] * out + o: the same products, sums in the same order, one rounding.  Pairs
 * with an invalid id write nothing.
 * Five launches whatever the id values are (the index kernel of _run_select on this item, the pair tables, the product,
 * the reduce, the plan run's error pass; none for n_ids == 0), no copy and no host read but the first call's read of
 * the item's chunk modes: capturable in a CUDA graph, replayable with new ids, x and scales.  An id outside [0, E), or
 * an expert routed more than T rounded up to a power of two times (a token that repeats an expert), raises E_INDEX.
 * _experts_matvec_fp8_scratch_size: the scratch bytes for (rows, in_features, n_ids, top_k): the select scratch, the
 * pair tables and _matvec_fp8's partial sums.  The scratch holds nothing between calls.
 * Host-side rejections launch and write nothing: E_ARG as _dequant_fp8_select refuses the plan, rows, ids, scratch,
 * fp8_format, the blocks and d_scale, as _matvec_fp8 refuses x_dtype, in_features, d_x, d_y and their strides, for
 * an item out of range, top_k == 0, n_ids not a multiple of top_k, T over the limit, an item whose slices are not whole
 * rows, x rows spanning more than 2^32 elements and a scratch under the stated size. */
#define ZIPNN_B200_EXPERTS_MATVEC_MAX_TOKENS 4
int zipnn_b200_decode_plan_experts_matvec_fp8_scratch_size(const zipnn_b200_decode_plan* plan, int item, size_t rows,
                                                           size_t in_features, size_t n_ids, size_t top_k, size_t* out);
int zipnn_b200_decode_plan_experts_matvec_fp8(const zipnn_b200_decode_plan* plan, int item, size_t rows, const void* d_ids,
                                              size_t n_ids, int id_bytes, size_t top_k, int fp8_format, int x_dtype,
                                              size_t in_features, const void* d_x, size_t x_stride, int x_per_pair,
                                              const float* d_scale, size_t block_rows, size_t block_cols, void* d_y,
                                              size_t y_stride, void* d_scratch, size_t scratch_bytes, void* cuda_stream);

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
 * zipnn_b200_compress_bound(...) bytes (compress) or `orig` bytes (decompress).
 * Every return, errors included, means the call no longer reads `h_in` / `h_body` or writes
 * `h_out`: the buffers may be freed or reused at once.
 * Compress: large inputs are compressed slab by slab and may be accepted with a smaller
 * `out_cap` than the bound (E_CAPACITY when the stream does not fit).  Nothing is written at or
 * past `out_cap`, but bytes in [*out_len, out_cap) may be overwritten: groups behind the first
 * are copied out early to where they would sit if every group in front of them stayed raw. */
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
