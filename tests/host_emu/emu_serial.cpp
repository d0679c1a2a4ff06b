// Host-compiled unit-test shim for zipnn_b200/csrc/huf_serial.cuh.
// TEST ONLY: lets `pytest -m "not gpu"` fuzz the single-thread device routines
// (tree build, table header encode/decode) against the oracle without a GPU.
// It is not part of the product library and is never loaded by zipnn_b200.
#include <cstdint>

// Count every branch of the table build a crafted histogram reaches (huf_serial.cuh, enum HufTrace).
static thread_local uint32_t g_trace[64];
#define ZB_HUF_TRACE(id) (++g_trace[(id)])

#include "../../zipnn_b200/csrc/huf_serial.cuh"
#include <cstring>

static_assert(zb::kTrCount <= 64, "trace counters");

extern "C" {

// counts[256] -> nb[256], val[256], header bytes.  Returns header length or -1.
int emu_table_from_counts(const uint32_t* count, uint32_t n, uint8_t* nb, uint16_t* val, uint8_t* hdr, int* lg_out) {
  static thread_local zb::TreeScratch T;
  int max_sym = 255;
  while (max_sym > 0 && count[max_sym] == 0) max_sym--;
  int last = zb::huf_sort_serial(T, count, max_sym);
  int want = zb::fse_pick_log(zb::kHufLogDefault, n, (uint32_t)max_sym, 1);
  int lg = zb::huf_lengths_from_sorted(T, last, want, nb);
  zb::huf_assign_values(nb, max_sym, lg, val);
  *lg_out = lg;
  int h = zb::huf_write_table(T, nb, max_sym, lg);
  if (h > 0) memcpy(hdr, T.hdr, (size_t)h);
  return h;
}

// The branches reached since the last call (trace[kTrCount]), then zeroed.  Returns kTrCount.
int emu_trace_take(uint32_t* trace) {
  for (int i = 0; i < zb::kTrCount; i++) {
    trace[i] = g_trace[i];
    g_trace[i] = 0;
  }
  return zb::kTrCount;
}

// zb::huf_early_out: 0 = raw, 1 = one symbol, 2 = build the table.
int emu_early_out(uint32_t largest, uint32_t plen) { return zb::huf_early_out(largest, plen); }

// zb::huf_block_decision: 0 = raw, 1 = RLE, else the coded block's size.
uint32_t emu_block_decision(int rle, const uint32_t* bits, int hsize, uint32_t plen, uint64_t cap, double thr) {
  return zb::huf_block_decision(rle != 0, bits, hsize, plen, cap, thr);
}

int emu_read_weights(const uint8_t* src, uint32_t size, uint8_t* weights, int* nsym, int* lg) {
  static thread_local zb::FseDec D;
  return zb::huf_read_weights(weights, nsym, lg, src, size, D);
}
}
