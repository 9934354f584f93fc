// row_emit_common.cuh — the pieces the row-payload emitters (rowbinary_emit.cu, bigquery_emit.cu, ducklake_emit.cu)
// share: the cell readers, the warp-reduced issue report, the Json canonicalisation staging (stage_json), the
// warp-per-row scan of cell lengths, and the result buffers of a row payload (RowPayload).  Each emitter includes it
// once; the kernels have internal linkage, so every translation unit gets its own copy.
//
// Json staging: an emitter numbers its Json "items" (RowBinary: (row, Json column); BigQuery: (record, Json column,
// image)) and passes a locator, a default-copyable functor with
//   __device__ bool operator()(uint64_t item, uint64_t* cell) const
// that gives the cell behind an item (false: no cell).  k_json_len sizes each item at 4 + input bytes per document (the
// Json cell, or each Json element of an array cell); stage_json scans those lengths into item offsets, and
// k_json_canon writes every document as [u32 canonical length][text] (etl_fmt::json_canon) at its item's offset.  The
// canonical text is never longer than the input, so the records of an item are walked with the input lengths.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "rowbinary_format.cuh"
#include "emit_scan.cuh"

namespace {

struct JsonStage {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  uint64_t n_items;
  const uint64_t* off;          // n_items + 1: offset of each item's records in canon
  uint8_t* canon; uint32_t* work;
  unsigned long long* flags;    // bad_flag is OR-ed in when a document does not parse again
  unsigned long long bad_flag;
};

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
// a String / Json cell's text: a span of the staged stream, or of the heap (COPY values that needed unescaping)
__device__ __forceinline__ const uint8_t* cell_text(const uint8_t* stream, const uint8_t* heap, uint64_t val) {
  return val & ETL_COPY_VAL_IN_HEAP ? heap + (val & ~ETL_COPY_VAL_IN_HEAP) : stream + val;
}
__device__ __forceinline__ const etl_array_elem* array_elems(const uint8_t* heap, uint64_t val) {
  return reinterpret_cast<const etl_array_elem*>(heap + val + sizeof(etl_array_hdr));
}
// the smallest key of the warp (~0: none) into *slot by one atomicMin
__device__ __forceinline__ void report_min(unsigned long long key, unsigned long long* slot) {
  if (!__any_sync(0xffffffffu, key != ~0ull)) return;
  for (int d = 16; d > 0; d >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, d));
  if ((threadIdx.x & 31) == 0) atomicMin(slot, key);
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

// the Json items of J (n_items, flags, the planes): input lengths → item offsets J.off → (sync) canonical text J.canon,
// with its node scratch J.work.  ETL_OK, ETL_ERR_ALLOC or ETL_ERR_CUDA
template <class Locate>
int stage_json(Scratch& scratch, JsonStage& J, Locate L, cudaStream_t st) {
  const uint64_t n = J.n_items;
  const uint32_t nb = scan_blocks(n);
  uint32_t* lens = (uint32_t*)scratch(n * 4);
  uint64_t* off = (uint64_t*)scratch((n + 1) * 8);
  unsigned long long* blk = (unsigned long long*)scratch((nb + 1) * 8ull);
  if (!lens || !off || !blk) return ETL_ERR_ALLOC;
  J.off = off;
  k_json_len<Locate><<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(J, L, lens);
  scan_lengths(lens, n, blk, blk + nb, off, st);
  unsigned long long total = 0;
  if (cudaMemcpyAsync(&total, blk + nb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
    return ETL_ERR_CUDA;
  J.canon = (uint8_t*)scratch(total);
  J.work = (uint32_t*)scratch(16 * total);
  if (!J.canon || !J.work) return ETL_ERR_ALLOC;
  if (total) k_json_canon<Locate><<<(uint32_t)((n + 127) / 128), 128, 0, st>>>(J, L);
  return ETL_OK;
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

// the result of a row-payload emit (etl_rowbinary_batch, etl_bigquery_batch): the rows' offsets and records, the bytes
struct RowPayload {
  uint64_t n_rows = 0, bytes = 0;
  uint8_t* meta = nullptr;    // device: n_rows + 1 row offsets | n_rows row records
  uint8_t* data = nullptr;    // device: the payload
  uint8_t* host = nullptr;    // pinned: meta | data (to_host)
  RowPayload() = default;
  RowPayload(const RowPayload&) = delete;
  RowPayload& operator=(const RowPayload&) = delete;
  ~RowPayload() {
    if (meta) cudaFree(meta);
    if (data) cudaFree(data);
    if (host) cudaFreeHost(host);
  }
  uint64_t meta_bytes() const { return (2 * n_rows + 1) * 8; }
  // pinned meta | data, copied on st
  int copy_to_host(cudaStream_t st) {
    if (cudaHostAlloc((void**)&host, meta_bytes() + bytes + 64, cudaHostAllocDefault) != cudaSuccess) { host = nullptr; return ETL_ERR_ALLOC; }
    if (cudaMemcpyAsync(host, meta, meta_bytes(), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(host + meta_bytes(), data, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return ETL_ERR_CUDA;
    return ETL_OK;
  }
  static uint64_t rows_of(const RowPayload* b) { return b ? b->n_rows : 0; }
  static uint64_t bytes_of(const RowPayload* b) { return b ? b->bytes : 0; }
  static const uint8_t* data_of(const RowPayload* b, int host) {
    if (!b) return nullptr;
    if (!host) return b->data;
    return b->host ? b->host + b->meta_bytes() : nullptr;
  }
  static const uint64_t* offsets_of(const RowPayload* b, int host) {
    if (!b) return nullptr;
    const uint8_t* base = host ? b->host : b->meta;
    return base ? reinterpret_cast<const uint64_t*>(base) : nullptr;
  }
  static const uint64_t* records_of(const RowPayload* b, int host) {
    const uint64_t* off = offsets_of(b, host);
    return off ? off + b->n_rows + 1 : nullptr;
  }
};
