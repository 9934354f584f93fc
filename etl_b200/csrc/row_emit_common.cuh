// row_emit_common.cuh — the pieces the row-payload emitters (rowbinary_emit.cu, bigquery_emit.cu) share: the Json
// canonicalisation staging and the warp-per-row scan of cell lengths.  Each emitter includes it once; the kernels have
// internal linkage, so every translation unit gets its own copy.
//
// Json staging: an emitter numbers its Json "items" (RowBinary: (row, Json column); BigQuery: (record, Json column,
// image)) and passes a locator, a default-copyable functor with
//   __device__ bool operator()(uint64_t item, uint64_t* cell) const
// that gives the cell behind an item (false: no cell).  k_json_len sizes each item at 4 + input bytes per document (the
// Json cell, or each Json element of an array cell); the emitter scans those lengths into item offsets, and
// k_json_canon writes every document as [u32 canonical length][text] (etl_fmt::json_canon) at its item's offset.  The
// canonical text is never longer than the input, so the records of an item are walked with the input lengths.
#pragma once
#include <stdint.h>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "rowbinary_format.cuh"

namespace {

struct JsonStage {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  uint64_t n_items;
  const uint64_t* off;          // n_items + 1: offset of each item's records in canon
  uint8_t* canon; uint32_t* work;
  unsigned long long* flags;    // bad_flag is OR-ed in when a document does not parse again
  unsigned long long bad_flag;
};

__device__ __forceinline__ uint32_t stage_rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
// a String / Json cell's text: a span of the staged stream, or of the heap (COPY values that needed unescaping)
__device__ __forceinline__ const uint8_t* cell_text(const uint8_t* stream, const uint8_t* heap, uint64_t val) {
  return val & ETL_COPY_VAL_IN_HEAP ? heap + (val & ~ETL_COPY_VAL_IN_HEAP) : stream + val;
}
__device__ __forceinline__ const etl_array_elem* array_elems(const uint8_t* heap, uint64_t val) {
  return reinterpret_cast<const etl_array_elem*>(heap + val + sizeof(etl_array_hdr));
}

template <class Locate>
__global__ void __launch_bounds__(256) k_json_len(JsonStage J, Locate L, uint32_t* lens) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= J.n_items) return;
  uint64_t cell = 0, n = 0;
  if (L(i, &cell)) {
    const uint32_t tag = J.cell_tag[cell], aux = J.cell_aux[cell];
    if (tag == ETL_CELL_JSON) n = 4ull + aux;
    else if (tag == ETL_CELL_ARRAY) {
      const etl_array_elem* E = array_elems(J.heap, J.cell_val[cell]);
      for (uint32_t k = 0; k < aux; k++) if (E[k].tag == ETL_CELL_JSON) n += 4ull + E[k].aux;
    }
  }
  lens[i] = (uint32_t)n;
}
// thread per item: canonicalise its documents in order; a document's node scratch sits at 4 words per byte of its
// record, which json_canon_work_words (<= 4n + 16) fits
template <class Locate>
__global__ void __launch_bounds__(128) k_json_canon(JsonStage J, Locate L) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= J.n_items) return;
  uint64_t cell = 0;
  if (!L(i, &cell)) return;
  const uint32_t tag = J.cell_tag[cell], aux = J.cell_aux[cell];
  uint64_t at = J.off[i];
  auto one = [&](const uint8_t* s, uint32_t n) {
    uint32_t r = etl_fmt::json_canon(s, n, J.canon + at + 4, J.work + 4 * at);
    if (r == etl_fmt::kJsonCanonBad) { atomicOr(J.flags, J.bad_flag); r = 0; }   // json_valid let it through
    etl_rb::le_write(r, 4, J.canon + at);
    at += 4ull + n;
  };
  if (tag == ETL_CELL_JSON) one(cell_text(J.stream, J.heap, J.cell_val[cell]), aux);
  else if (tag == ETL_CELL_ARRAY) {
    const etl_array_elem* E = array_elems(J.heap, J.cell_val[cell]);
    for (uint32_t k = 0; k < aux; k++) if (E[k].tag == ETL_CELL_JSON) one(J.heap + E[k].val, E[k].aux);
  }
}

// warp per row: the row's w cell lengths (cell_len[row * w ..]) → offsets inside the row, and the row's length; a row
// of 4 GiB or more ORs too_long into *flags
__global__ void __launch_bounds__(256) k_row_scan(uint32_t* cell_len, uint32_t w, uint64_t n_rows, uint32_t* row_len,
                                                  unsigned long long* flags, unsigned long long too_long) {
  const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (row >= n_rows) return;                          // whole warps
  uint32_t* L = cell_len + row * w;
  unsigned long long run = 0;
  for (uint32_t base = 0; base < w; base += 32) {
    const uint32_t c = base + lane;
    const unsigned long long v = c < w ? L[c] : 0u;
    unsigned long long x = v;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= (uint32_t)d) x += y;
    }
    if (c < w) L[c] = (uint32_t)(run + x - v);
    run += __shfl_sync(0xffffffffu, x, 31);
  }
  if (lane == 0) {
    if (run > 0xffffffffull) atomicOr(flags, too_long);
    row_len[row] = (uint32_t)run;
  }
}

}  // namespace
