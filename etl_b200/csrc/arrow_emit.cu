// arrow_emit.cu — columnar emitter (SURVEY §8f N2): the rows of ONE replicated-schema version of a decoded batch as
// Arrow-layout column buffers, built on the device from the cell plane.
//
// Replaces the per-row walk of the destinations' encoders — build_array_for_field / build_primitive_array /
// build_boolean_array / build_string_array / build_binary_array / build_uuid_array and the cell_to_* converters of
// crates/etl-destinations/src/iceberg/encoding.rs:61-330 (the DuckLake and BigQuery encoders walk the same
// Vec<TableRow>) — for the column types whose Arrow value is a function of the decoded cell alone:
//   Bool → Boolean (bit-packed) · I16/I32 → Int32 · I64/U32 → Int64 (:200-221) · F32 · F64 · Date → Date32 days (:257-262)
//   Time → Time64 µs (:270-275) · Timestamp / TimestampTz → Timestamp µs (:284-301) · Uuid → FixedSizeBinary(16) (:313-318)
//   String → Utf8 (int32 offsets) · Bytes → LargeBinary (int64 offsets) (:245-250).
// A cell of another variant in such a column becomes null, exactly as the converters return None.  Numeric, Json and
// Array columns go through cell_to_string / build_list_array in the reference: without ETL_ARROW_ALL_COLUMNS they are
// reported as ETL_ARROW_UNSUPPORTED and stay on the shim's row path (the output is what it was before the bit existed).
// Pure gather / scan / copy kernels over planes that are already in HBM: HBM-bound, no parsing.
//
// With ETL_ARROW_ALL_COLUMNS in row_kinds every column type of the reference's Iceberg schema (iceberg/schema.rs:9-63)
// is built here, with the formatters of arrow_format.cuh:
//   * Numeric → Utf8: k_col_fixed computes each row's Display length from the numeric header, the length scan turns
//     lengths into offsets, k_gather_text writes the text in place.  No scratch.
//   * Json → Utf8: the input lengths are scanned into scratch offsets; k_json_canon canonicalises each document once
//     (thread per document, any size) into that scratch, which the input length bounds, and records the canonical
//     length; a second scan gives the offsets and k_gather_text copies.  One parse per document instead of a count pass
//     plus a write pass.  A document json_valid should have rejected raises a flag → ETL_ERR_INTERNAL.
//   * Array → List<child> (build_list_array, encoding.rs:386-776): per-row element counts (k_col_fixed) scanned into
//     int32 list offsets; k_list_elems, element-parallel, finds each element's row by binary search over them and writes
//     the child's element planes, over which the child is one more column: fixed_value and one ballot per warp for
//     validity / Boolean words (k_col_fixed), or lengths → offsets → gather for Utf8 / LargeBinary children, Numeric
//     and Json elements through the formatters.  An element's String / Json / Numeric / Bytes / Uuid payload is a heap
//     offset (array_parse.cuh), a top-level String / Json cell a span of the staged stream.
// Each stage that sizes a buffer syncs once: after the row lengths, after the Json / List child lengths, and after the
// Json children's canonical lengths (only when a List has Json elements).
// A COPY batch (rec_kind == NULL) is one implicit schema: k_copy_sel maps every row of the valid prefix to its cells
// (no selection sync), then every column stage runs unchanged; String / Json text with ETL_COPY_VAL_IN_HEAP is read from
// the heap.  ETL_ARROW_CDC_COLUMNS appends cdc_operation / sequence_number, sized from n_rows alone and written by k_cdc.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "arrow_internal.h"
#include "batch_internal.h"
#include "emit_scan.cuh"

namespace {

// which image of record r is a row of this batch?  kRow and the cell offset of the image inside the record; kSkipped
// for a record whose kind row_kinds selects but which has no full image to emit (write_events, iceberg/core.rs:311-322
// and :336-357, returns InvalidState there); kNotRow otherwise
struct ArrowRows {
__device__ __forceinline__ int operator()(const SelParams& S, uint64_t r, uint64_t* cell0) const {
  if (r >= S.n_records || S.rec_schema[r] != S.schema) return kNotRow;
  const uint32_t k = S.rec_kind[r], f = S.rec_flags[r];
  if (!(f & ETL_RF_EVENT)) return kNotRow;
  const uint64_t c0 = S.rec_cell_base[r];
  if (k == 'I' && (S.row_kinds & 1u)) { *cell0 = c0; return kRow; }
  if (k == 'U' && (S.row_kinds & 2u)) {
    if (f & ETL_RF_NEW_PARTIAL) return kSkipped;                          // UpdatedTableRow::Full only: a partial row has holes
    *cell0 = S.rec_cell_base[r + 1] - S.n_cols;                           // the new image is the record's last n_cols cells
    return kRow;
  }
  if (k == 'D' && (S.row_kinds & 4u)) {
    if (!(f & ETL_RF_OLD_FULL)) return kSkipped;
    *cell0 = c0;
    return kRow;
  }
  return kNotRow;
}
};

struct ColParams {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  const uint64_t* row_cell0; uint64_t n_rows; uint32_t col; uint32_t arrow_type;
  uint32_t* validity;     // one word per 32 rows
  void* values;           // fixed width
  uint32_t* lens;         // var width: byte length per row (→ scanned into offsets)
  uint32_t text;          // Utf8 by cell_to_string: Numeric and Json cells are formatted too (ETL_ARROW_ALL_COLUMNS)
};
// the cell of item `row`: a row's cell of column `col`, or (row_cell0 == NULL) the row-th entry of a list child's
// element planes, where `stream` is the heap (an array element's String / Json text lives in the heap)
__device__ __forceinline__ uint64_t cell_of(const ColParams& C, uint64_t row) { return C.row_cell0 ? C.row_cell0[row] + C.col : row; }
// the text of a String / Json cell: a span of `stream`, or (COPY rows whose field needed unescaping, bit 63 of val) of
// the heap.  A stream offset is below 1 TiB, so the bit is checked unconditionally
__device__ __forceinline__ const uint8_t* text_of(const ColParams& C, uint64_t val) {
  return val & ETL_COPY_VAL_IN_HEAP ? C.heap + (val & ~ETL_COPY_VAL_IN_HEAP) : C.stream + val;
}
// iceberg/encoding.rs:200-318: value of a cell for the column's Arrow type, or "null"
__device__ __forceinline__ bool fixed_value(uint32_t at, uint32_t tag, uint64_t val, uint32_t aux, int64_t* out) {
  switch (at) {
    case ETL_ARROW_BOOLEAN: if (tag != ETL_CELL_BOOL) return false; *out = (int64_t)(val & 1u); return true;
    case ETL_ARROW_INT32: if (tag != ETL_CELL_I16 && tag != ETL_CELL_I32) return false; *out = (int64_t)val; return true;
    case ETL_ARROW_INT64: if (tag != ETL_CELL_I64 && tag != ETL_CELL_U32) return false; *out = tag == ETL_CELL_U32 ? (int64_t)(uint32_t)val : (int64_t)val; return true;
    case ETL_ARROW_FLOAT32: if (tag != ETL_CELL_F32) return false; *out = (int64_t)(uint32_t)val; return true;
    case ETL_ARROW_FLOAT64: if (tag != ETL_CELL_F64) return false; *out = (int64_t)val; return true;
    case ETL_ARROW_DATE32: if (tag != ETL_CELL_DATE) return false; *out = (int64_t)val; return true;
    case ETL_ARROW_TIME64_US: if (tag != ETL_CELL_TIME) return false; *out = (int64_t)val * 1000000ll + (int64_t)(aux / 1000u); return true;
    case ETL_ARROW_TIMESTAMP_US: if (tag != ETL_CELL_TIMESTAMP) return false; *out = (int64_t)val * 1000000ll + (int64_t)(aux / 1000u); return true;
    case ETL_ARROW_TIMESTAMPTZ_US: if (tag != ETL_CELL_TIMESTAMPTZ) return false; *out = (int64_t)val * 1000000ll + (int64_t)(aux / 1000u); return true;
    default: return false;
  }
}
// one thread per row of one column: value / length + the validity word of its warp
__global__ void __launch_bounds__(256) k_col_fixed(ColParams C) {
  const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  int64_t v = 0;
  uint32_t len = 0;
  if (row < C.n_rows) {
    const uint64_t cell = cell_of(C, row);
    const uint32_t tag = C.cell_tag[cell];
    const uint64_t val = C.cell_val[cell];
    const uint32_t aux = C.cell_aux[cell];
    switch (C.arrow_type) {
      case ETL_ARROW_UTF8:
        valid = tag == ETL_CELL_STRING || (C.text && (tag == ETL_CELL_NUMERIC || tag == ETL_CELL_JSON));
        // Numeric: the Display length from the header; Json: the input length (the canonical text is never longer)
        len = !valid ? 0u : (tag == ETL_CELL_NUMERIC ? etl_fmt::numeric_len(C.heap + val, aux) : aux);
        break;
      case ETL_ARROW_LARGE_BINARY: valid = tag == ETL_CELL_BYTES; len = valid ? aux : 0u; break;
      case ETL_ARROW_UUID: valid = tag == ETL_CELL_UUID; break;
      case ETL_ARROW_LIST: valid = tag == ETL_CELL_ARRAY; len = valid ? aux : 0u; break;    // element count
      default: valid = fixed_value(C.arrow_type, tag, val, aux, &v); break;
    }
    switch (C.arrow_type) {
      case ETL_ARROW_INT32: case ETL_ARROW_DATE32: case ETL_ARROW_FLOAT32: static_cast<int32_t*>(C.values)[row] = valid ? (int32_t)v : 0; break;
      case ETL_ARROW_INT64: case ETL_ARROW_FLOAT64: case ETL_ARROW_TIME64_US: case ETL_ARROW_TIMESTAMP_US: case ETL_ARROW_TIMESTAMPTZ_US:
        static_cast<int64_t*>(C.values)[row] = valid ? v : 0; break;
      case ETL_ARROW_UUID: {
        uint64_t a = 0, b = 0;
        if (valid) { const uint64_t* s = reinterpret_cast<const uint64_t*>(C.heap + val); a = s[0]; b = s[1]; }   // heap reservations are 8-byte aligned
        static_cast<uint64_t*>(C.values)[2 * row] = a; static_cast<uint64_t*>(C.values)[2 * row + 1] = b;
        break;
      }
      case ETL_ARROW_UTF8: case ETL_ARROW_LARGE_BINARY: case ETL_ARROW_LIST: C.lens[row] = len; break;
      default: break;
    }
  }
  const unsigned vb = __ballot_sync(0xffffffffu, valid);
  const unsigned bb = __ballot_sync(0xffffffffu, valid && v != 0);
  if ((threadIdx.x & 31) == 0 && (row >> 5) < ((C.n_rows + 31) >> 5)) {
    C.validity[row >> 5] = vb;
    if (C.arrow_type == ETL_ARROW_BOOLEAN) static_cast<uint32_t*>(C.values)[row >> 5] = bb;   // Boolean values are bit-packed too
  }
}
// warp per row: copy the row's bytes to their place in the column's data buffer (16 B per lane where aligned)
template <typename OffT>
__global__ void __launch_bounds__(256) k_gather(ColParams C, const OffT* offs, uint8_t* data) {
  const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (row >= C.n_rows) return;
  const uint64_t cell = cell_of(C, row);
  const uint32_t tag = C.cell_tag[cell];
  const bool str = C.arrow_type == ETL_ARROW_UTF8;
  if (tag != (str ? (uint32_t)ETL_CELL_STRING : (uint32_t)ETL_CELL_BYTES)) return;
  const uint8_t* src = str ? text_of(C, C.cell_val[cell]) : C.heap + C.cell_val[cell];
  const uint32_t n = C.cell_aux[cell];
  uint8_t* dst = data + (uint64_t)offs[row];
  for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}

// ---------------------------------------------------------------- ETL_ARROW_ALL_COLUMNS
// Json: one thread per document canonicalises it once (arrow_format.cuh) into `canon` at the document's input offset
// (the scan of the input lengths) and replaces its length by the canonical one; the lengths are then scanned again
// into the column's offsets and k_gather_text copies the text.  The node scratch of a document sits at
// 4 * in_off + 16 * item words: json_canon_work_words(n) <= 4n + 16.  One work buffer serves every Json item set of an
// emit in turn (the canonicalisations run one after the other on the stream).
constexpr uint64_t kJsonWorkPerByte = 4, kJsonWorkPerItem = 16;
__global__ void __launch_bounds__(128) k_json_canon(ColParams C, const uint64_t* in_off, uint8_t* canon, uint32_t* work, unsigned* bad) {
  const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= C.n_rows) return;
  const uint64_t cell = cell_of(C, row);
  if (C.cell_tag[cell] != ETL_CELL_JSON) return;
  const uint64_t at = in_off[row];
  const uint32_t n = C.cell_aux[cell];
  const uint32_t r = etl_fmt::json_canon(text_of(C, C.cell_val[cell]), n, canon + at, work + kJsonWorkPerByte * at + kJsonWorkPerItem * row);
  if (r == etl_fmt::kJsonCanonBad) { atomicOr(bad, 1u); C.lens[row] = 0; return; }   // json_valid let through what it must reject
  C.lens[row] = r;
}
// warp per item of a cell_to_string Utf8 column: String text and canonical Json text are copied, Numeric is written by
// one lane (its Display is a few dozen bytes)
__global__ void __launch_bounds__(256) k_gather_text(ColParams C, const int32_t* offs, uint8_t* data, const uint64_t* in_off, const uint8_t* canon) {
  const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (row >= C.n_rows) return;
  const uint64_t cell = cell_of(C, row);
  const uint32_t tag = C.cell_tag[cell];
  uint8_t* dst = data + (uint32_t)offs[row];
  const uint8_t* src;
  uint32_t n;
  if (tag == ETL_CELL_NUMERIC) {
    if (lane == 0) etl_fmt::numeric_write(C.heap + C.cell_val[cell], C.cell_aux[cell], dst);
    return;
  }
  if (tag == ETL_CELL_STRING) { src = text_of(C, C.cell_val[cell]); n = C.cell_aux[cell]; }
  else if (tag == ETL_CELL_JSON && canon) { src = canon + in_off[row]; n = (uint32_t)(offs[row + 1] - offs[row]); }
  else return;
  for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}
// element-parallel: the element planes of a List column's child.  Each element finds its row by binary search over the
// list offsets, then reads its etl_array_elem from the row's array in the heap
__global__ void __launch_bounds__(256) k_list_elems(ColParams C, const int32_t* loffs, uint64_t n_elems, uint8_t* el_tag, uint64_t* el_val, uint32_t* el_aux) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elems) return;
  uint64_t lo = 0, hi = C.n_rows - 1;                 // last row whose first element is <= e
  while (lo < hi) {
    const uint64_t mid = (lo + hi + 1) >> 1;
    if ((uint64_t)(uint32_t)loffs[mid] <= e) lo = mid; else hi = mid - 1;
  }
  const uint64_t cell = C.row_cell0[lo] + C.col;
  const uint8_t* el = C.heap + C.cell_val[cell] + sizeof(etl_array_hdr) + sizeof(etl_array_elem) * (e - (uint32_t)loffs[lo]);
  const etl_array_elem x = *reinterpret_cast<const etl_array_elem*>(el);
  el_tag[e] = x.tag; el_val[e] = x.val; el_aux[e] = x.aux;
}

// ---------------------------------------------------------------- ETL_ARROW_CDC_COLUMNS
// thread per row: cdc_operation and sequence_number (write_table_rows / write_events, iceberg/core.rs:239-366), two
// never-null Utf8 columns whose texts have fixed lengths, so their offsets are 6 * row and 33 * row.  COPY rows
// (rec_kind == NULL) are INSERT with the key of (0, 0).
struct CdcParams {
  const uint64_t* row_rec; const uint8_t* rec_kind; const uint64_t* rec_commit_lsn; const uint64_t* rec_tx_ordinal;
  uint64_t n_rows;
  uint32_t* op_validity; int32_t* op_offs; uint8_t* op_data;
  uint32_t* seq_validity; int32_t* seq_offs; uint8_t* seq_data;
};
__global__ void __launch_bounds__(256) k_cdc(CdcParams Q) {
  const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= Q.n_rows) return;
  uint32_t kind = 'I';
  uint64_t lsn = 0, ord = 0;
  if (Q.rec_kind) {
    const uint64_t r = Q.row_rec[row];
    kind = Q.rec_kind[r]; lsn = Q.rec_commit_lsn[r]; ord = Q.rec_tx_ordinal[r];
  }
  etl_fmt::cdc_op_write(kind, Q.op_data + etl_fmt::kCdcOpLen * row);
  etl_fmt::seq_key_write(lsn, ord, Q.seq_data + etl_fmt::kSeqKeyLen * row);
  Q.op_offs[row] = (int32_t)(etl_fmt::kCdcOpLen * row);
  Q.seq_offs[row] = (int32_t)(etl_fmt::kSeqKeyLen * row);
  if (row + 1 == Q.n_rows) { Q.op_offs[Q.n_rows] = (int32_t)(etl_fmt::kCdcOpLen * Q.n_rows); Q.seq_offs[Q.n_rows] = (int32_t)(etl_fmt::kSeqKeyLen * Q.n_rows); }
  if ((row & 31) == 0) {                               // validity: every row of the word that exists
    const uint64_t left = Q.n_rows - row;
    const uint32_t w = left >= 32 ? 0xffffffffu : (1u << left) - 1u;
    Q.op_validity[row >> 5] = w; Q.seq_validity[row >> 5] = w;
  }
}

uint32_t arrow_type_of(uint32_t k, bool all) {
  switch (k) {
    case ETL_K_BOOL: return ETL_ARROW_BOOLEAN;
    case ETL_K_I16: case ETL_K_I32: return ETL_ARROW_INT32;
    case ETL_K_I64: case ETL_K_U32: return ETL_ARROW_INT64;
    case ETL_K_F32: return ETL_ARROW_FLOAT32;
    case ETL_K_F64: return ETL_ARROW_FLOAT64;
    case ETL_K_STRING: return ETL_ARROW_UTF8;
    case ETL_K_BYTES: return ETL_ARROW_LARGE_BINARY;
    case ETL_K_DATE: return ETL_ARROW_DATE32;
    case ETL_K_TIME: return ETL_ARROW_TIME64_US;
    case ETL_K_TIMESTAMP: return ETL_ARROW_TIMESTAMP_US;
    case ETL_K_TIMESTAMPTZ: return ETL_ARROW_TIMESTAMPTZ_US;
    case ETL_K_UUID: return ETL_ARROW_UUID;
    case ETL_K_NUMERIC: case ETL_K_JSON: return all ? ETL_ARROW_UTF8 : ETL_ARROW_UNSUPPORTED;   // cell_to_string
    default: return all && (k & ETL_K_ARRAY) ? ETL_ARROW_LIST : ETL_ARROW_UNSUPPORTED;
  }
}
// child type of a List column (build_list_array, encoding.rs:386-776): String / Numeric / Json elements → Utf8
uint32_t list_child_type(uint32_t k) {
  const uint32_t ek = k & ~(uint32_t)ETL_K_ARRAY;
  return ek == ETL_K_NUMERIC || ek == ETL_K_JSON ? (uint32_t)ETL_ARROW_UTF8 : arrow_type_of(ek, false);
}
using etl_arrow::Col;
using etl_arrow::is_var;
using etl_arrow::value_width;

}  // namespace

extern "C" {

int etl_dec_arrow_emit(const etl_dec_batch* batch, uint32_t schema_index, uint32_t row_kinds, int to_host, etl_arrow_batch** out) {
  if (!batch || !out) return ETL_ERR_INVALID_ARG;
  const bool all = (row_kinds & ETL_ARROW_ALL_COLUMNS) != 0;
  const bool cdc = (row_kinds & ETL_ARROW_CDC_COLUMNS) != 0;
  // a COPY batch (no record kinds) has one implicit schema: the columns it was decoded with
  EmitBatch E;
  if (open_emit_batch(batch, schema_index, &E) != ETL_OK) return ETL_ERR_INVALID_ARG;
  const etl_dec_planes& P = E.P;
  const etl_dec_schema_info& sc = E.sc;
  const uint8_t* dev_stream = E.stream;
  cudaStream_t st = cudaStreamPerThread;
  etl_arrow_batch* A = new etl_arrow_batch();
  // scratch of the ETL_ARROW_ALL_COLUMNS stages, freed on every exit
  std::vector<void*> pool;
  auto free_pool = [&]() { for (void* p : pool) cudaFree(p); pool.clear(); };
  auto fail = [&](int rc) { free_pool(); if (A->dev) cudaFree(A->dev); if (A->host) cudaFreeHost(A->host); delete A; return rc; };
#define CKA(call) do { if ((call) != cudaSuccess) { cudaGetLastError(); return fail(ETL_ERR_CUDA); } } while (0)
  // rows of the valid prefix only
  const uint64_t n_valid = E.n_valid;
  const uint32_t nb = (uint32_t)((n_valid + kSelThreads - 1) / kSelThreads);
  uint32_t* d_blk = nullptr; uint64_t* d_cell0 = nullptr; uint64_t* d_rec = nullptr; unsigned long long* d_n = nullptr;
  CKA(cudaMalloc(&d_blk, (nb + 1) * 4ull)); CKA(cudaMalloc(&d_cell0, (n_valid + 1) * 8)); CKA(cudaMalloc(&d_rec, (n_valid + 1) * 8)); CKA(cudaMalloc(&d_n, 16));
  auto free_tmp = [&]() { cudaFree(d_blk); cudaFree(d_cell0); cudaFree(d_rec); cudaFree(d_n); };
  SelParams Sp{P.rec_kind, P.rec_flags, P.rec_schema, P.rec_cell_base, n_valid, (int32_t)schema_index, row_kinds, sc.n_cols, d_blk, d_cell0, d_rec, d_n};
  // COPY: every row of the valid prefix when inserts are selected
  unsigned long long sel[2] = {0, UINT64_MAX};          // rows, first skipped record
  if (!E.copy && nb) cudaMemsetAsync(d_n + 1, 0xff, 8, st);
  if (select_rows<ArrowRows>(Sp, E.copy, (row_kinds & 1u) ? n_valid : 0, st, sel) != ETL_OK) { free_tmp(); return fail(ETL_ERR_CUDA); }
  const uint64_t n_rows = sel[0];
  A->first_skipped = sel[1];
  A->n_rows = n_rows;
  // pass 1: validity + fixed values + lengths (into a scratch), per column; var-width sizes need a sync before the data buffers exist
  const uint64_t vbytes = ((n_rows + 31) / 32 * 4 + 63) & ~63ull;
  uint64_t cur = ((n_rows * 8) + 63) & ~63ull;        // row_rec first
  A->row_rec_off = 0;
  A->cols.resize(sc.n_cols);
  uint32_t n_var = 0;
  for (uint32_t c = 0; c < sc.n_cols; c++) {
    Col& col = A->cols[c];
    col.kind = sc.col_kind[c];
    col.arrow_type = arrow_type_of(col.kind, all);
    col.text = all && (col.kind == ETL_K_NUMERIC || col.kind == ETL_K_JSON);
    if (col.arrow_type == ETL_ARROW_UNSUPPORTED) continue;
    col.validity_off = cur; cur += vbytes;
    if (col.arrow_type == ETL_ARROW_BOOLEAN) { col.values_off = cur; col.values_bytes = vbytes; cur += vbytes; }
    else if (value_width(col.arrow_type)) { col.values_off = cur; col.values_bytes = (n_rows * value_width(col.arrow_type) + 63) & ~63ull; cur += col.values_bytes; }
    else { col.offsets_off = cur; col.offsets_bytes = ((n_rows + 1) * (col.arrow_type == ETL_ARROW_LARGE_BINARY ? 8 : 4) + 63) & ~63ull; cur += col.offsets_bytes; n_var++; }
  }
  const uint64_t fixed_bytes = cur;
  uint32_t* d_lens = nullptr; unsigned long long* d_lblk = nullptr; unsigned long long* d_tot = nullptr;
  const uint32_t lb = scan_blocks(n_rows);
  if (n_var) { if (cudaMalloc(&d_lens, (size_t)n_var * (n_rows + 1) * 4) != cudaSuccess || cudaMalloc(&d_lblk, (size_t)n_var * (lb + 1) * 8) != cudaSuccess || cudaMalloc(&d_tot, n_var * 8 + 8) != cudaSuccess) { free_tmp(); return fail(ETL_ERR_ALLOC); } }
  uint8_t* d_fixed = nullptr;
  if (cudaMalloc(&d_fixed, fixed_bytes + 64) != cudaSuccess) { free_tmp(); cudaFree(d_lens); cudaFree(d_lblk); cudaFree(d_tot); return fail(ETL_ERR_ALLOC); }
  auto free_stage = [&]() { free_tmp(); cudaFree(d_lens); cudaFree(d_lblk); cudaFree(d_tot); cudaFree(d_fixed); };
  cudaMemsetAsync(d_fixed, 0, fixed_bytes + 64, st);
  if (n_rows) cudaMemcpyAsync(d_fixed, d_rec, n_rows * 8, cudaMemcpyDeviceToDevice, st);
  std::vector<unsigned long long> totals(n_var + 1, 0);
  std::vector<uint64_t*> json_in(sc.n_cols, nullptr);   // Json columns: input offsets of the documents (scan of pass 1)
  auto dalloc = [&](uint64_t bytes) -> void* { void* p = nullptr; if (cudaMalloc(&p, bytes + 64) != cudaSuccess) return nullptr; pool.push_back(p); return p; };
  uint32_t vi = 0;
  for (uint32_t c = 0; c < sc.n_cols && n_rows; c++) {
    Col& col = A->cols[c];
    if (col.arrow_type == ETL_ARROW_UNSUPPORTED) continue;
    ColParams Cp{P.cell_tag, P.cell_val, P.cell_aux, P.heap, dev_stream, d_cell0, n_rows, c, col.arrow_type,
                 (uint32_t*)(d_fixed + col.validity_off), col.values_bytes ? (void*)(d_fixed + col.values_off) : nullptr, nullptr, col.text};
    const bool var = is_var(col.arrow_type);
    if (var) Cp.lens = d_lens + (size_t)vi * (n_rows + 1);
    k_col_fixed<<<(uint32_t)((n_rows + 255) / 256), 256, 0, st>>>(Cp);
    if (var) {
      unsigned long long* blk = d_lblk + (size_t)vi * (lb + 1);
      if (col.text && col.kind == ETL_K_JSON) {
        if (!(json_in[c] = (uint64_t*)dalloc((n_rows + 1) * 8))) { free_stage(); return fail(ETL_ERR_ALLOC); }
        scan_lengths(Cp.lens, n_rows, blk, d_tot + vi, json_in[c], st);
      } else if (col.arrow_type == ETL_ARROW_LARGE_BINARY) scan_lengths(Cp.lens, n_rows, blk, d_tot + vi, (int64_t*)(d_fixed + col.offsets_off), st);
      else scan_lengths(Cp.lens, n_rows, blk, d_tot + vi, (int32_t*)(d_fixed + col.offsets_off), st);
      vi++;
    }
  }
  if (n_var && n_rows) cudaMemcpyAsync(totals.data(), d_tot, n_var * 8, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) { free_stage(); return fail(ETL_ERR_CUDA); }
  // ETL_ARROW_ALL_COLUMNS: Json documents canonicalised, List children built; each step that sizes a buffer syncs once
  unsigned* d_bad = nullptr;
  std::vector<uint8_t*> kid_fixed;                      // per child: validity | values or offsets, laid out from 0
  std::vector<const uint8_t*> canon_of(sc.n_cols, nullptr);
  struct KidSrc { uint8_t* tag; uint64_t* val; uint32_t* aux; uint32_t* lens; uint64_t* in_off; uint8_t* canon; };
  std::vector<KidSrc> kid_src;
  if (all && n_rows) {
    if (!(d_bad = (unsigned*)dalloc(8))) { free_stage(); return fail(ETL_ERR_ALLOC); }
    cudaMemsetAsync(d_bad, 0, 4, st);
    // Json canonicalisation of n items whose input offsets are in_off (total input bytes t_in); new lengths → offs
    uint32_t* work = nullptr;
    uint64_t work_words = 0;
    auto canon_items = [&](const ColParams& Cp, const uint64_t* in_off, uint64_t t_in, uint8_t** canon_out, int32_t* offs, unsigned long long* tot) -> bool {
      uint8_t* canon = (uint8_t*)dalloc(t_in);
      const uint64_t words = kJsonWorkPerByte * t_in + kJsonWorkPerItem * Cp.n_rows;
      if (words > work_words) {                          // grows rarely: the first Json column, then a larger one
        if (work) { cudaFree(work); pool.erase(std::find(pool.begin(), pool.end(), (void*)work)); }
        work = (uint32_t*)dalloc(words * 4);
        work_words = work ? words : 0;
      }
      if (!canon || !work) return false;
      k_json_canon<<<(uint32_t)((Cp.n_rows + 127) / 128), 128, 0, st>>>(Cp, in_off, canon, work, d_bad);
      *canon_out = canon;
      unsigned long long* blk = (unsigned long long*)dalloc((scan_blocks(Cp.n_rows) + 1) * 8ull);
      if (!blk) return false;
      scan_lengths(Cp.lens, Cp.n_rows, blk, tot, offs, st);
      return true;
    };
    unsigned long long* d_tot2 = (unsigned long long*)dalloc(8ull * (2 * sc.n_cols + 2));
    if (!d_tot2) { free_stage(); return fail(ETL_ERR_ALLOC); }
    cudaMemsetAsync(d_tot2, 0, 8ull * (2 * sc.n_cols + 2), st);
    std::vector<unsigned long long> tot2(2 * sc.n_cols + 2, 0);
    vi = 0;
    for (uint32_t c = 0; c < sc.n_cols; c++) {
      Col& col = A->cols[c];
      if (!is_var(col.arrow_type)) continue;
      const uint64_t total = totals[vi];
      uint32_t* lens = d_lens + (size_t)vi * (n_rows + 1);
      vi++;
      ColParams Cp{P.cell_tag, P.cell_val, P.cell_aux, P.heap, dev_stream, d_cell0, n_rows, c, col.arrow_type, nullptr, nullptr, lens, 1};
      if (col.text && col.kind == ETL_K_JSON) {
        uint8_t* canon = nullptr;
        if (!canon_items(Cp, json_in[c], total, &canon, (int32_t*)(d_fixed + col.offsets_off), d_tot2 + c)) { free_stage(); return fail(ETL_ERR_ALLOC); }
        canon_of[c] = canon;
      }
      if (col.arrow_type != ETL_ARROW_LIST) continue;
      if (total > 0x7FFFFFFFull) { A->error = "List column exceeds 2^31 - 1 elements: split the batch"; free_stage(); return fail(ETL_ERR_INVALID_ARG); }
      Col kid;
      kid.kind = col.kind & ~(uint32_t)ETL_K_ARRAY;
      kid.arrow_type = list_child_type(col.kind);
      kid.text = kid.arrow_type == ETL_ARROW_UTF8;
      kid.n_items = total;
      const uint64_t ne = total, kv = ((ne + 31) / 32 * 4 + 63) & ~63ull;
      uint64_t kcur = kv;
      if (kid.arrow_type == ETL_ARROW_BOOLEAN) { kid.values_off = kcur; kid.values_bytes = kv; kcur += kv; }
      else if (value_width(kid.arrow_type)) { kid.values_off = kcur; kid.values_bytes = (ne * value_width(kid.arrow_type) + 63) & ~63ull; kcur += kid.values_bytes; }
      else if (kid.arrow_type != ETL_ARROW_UNSUPPORTED) { kid.offsets_off = kcur; kid.offsets_bytes = ((ne + 1) * (kid.arrow_type == ETL_ARROW_LARGE_BINARY ? 8 : 4) + 63) & ~63ull; kcur += kid.offsets_bytes; }
      kid.data_off = kcur;                                 // relative to the child's base until the final layout
      uint8_t* kf = (uint8_t*)dalloc(kcur);
      KidSrc ks{(uint8_t*)dalloc(ne), (uint64_t*)dalloc(ne * 8), (uint32_t*)dalloc(ne * 4), (uint32_t*)dalloc((ne + 1) * 4), nullptr, nullptr};
      if (!kf || !ks.tag || !ks.val || !ks.aux || !ks.lens) { free_stage(); return fail(ETL_ERR_ALLOC); }
      cudaMemsetAsync(kf, 0, kcur + 64, st);
      col.child = (int32_t)A->kids.size();
      if (ne) {
        Cp.lens = nullptr;
        k_list_elems<<<(uint32_t)((ne + 255) / 256), 256, 0, st>>>(Cp, (const int32_t*)(d_fixed + col.offsets_off), ne, ks.tag, ks.val, ks.aux);
        ColParams Kp{ks.tag, ks.val, ks.aux, P.heap, P.heap, nullptr, ne, 0, kid.arrow_type, (uint32_t*)kf,
                     kid.values_bytes ? (void*)(kf + kid.values_off) : nullptr, ks.lens, kid.text ? 1u : 0u};
        k_col_fixed<<<(uint32_t)((ne + 255) / 256), 256, 0, st>>>(Kp);
        if (is_var(kid.arrow_type)) {
          const bool json = kid.kind == ETL_K_JSON;
          if (json && !(ks.in_off = (uint64_t*)dalloc((ne + 1) * 8))) { free_stage(); return fail(ETL_ERR_ALLOC); }
          unsigned long long* blk = (unsigned long long*)dalloc((scan_blocks(ne) + 1) * 8ull);
          if (!blk) { free_stage(); return fail(ETL_ERR_ALLOC); }
          unsigned long long* tot = d_tot2 + sc.n_cols + A->kids.size();
          if (json) scan_lengths(ks.lens, ne, blk, tot, ks.in_off, st);
          else if (kid.arrow_type == ETL_ARROW_UTF8) scan_lengths(ks.lens, ne, blk, tot, (int32_t*)(kf + kid.offsets_off), st);
          else scan_lengths(ks.lens, ne, blk, tot, (uint64_t*)(kf + kid.offsets_off), st);
        }
      }
      A->kids.push_back(kid);
      kid_fixed.push_back(kf);
      kid_src.push_back(ks);
    }
    if (cudaMemcpyAsync(tot2.data(), d_tot2, 8ull * tot2.size(), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) { free_stage(); return fail(ETL_ERR_CUDA); }
    // Json children: their input sizes are known now
    bool again = false;
    for (size_t k = 0; k < A->kids.size(); k++) {
      Col& kid = A->kids[k];
      if (kid.kind != ETL_K_JSON || !kid.n_items) continue;
      KidSrc& ks = kid_src[k];
      ColParams Kp{ks.tag, ks.val, ks.aux, P.heap, P.heap, nullptr, kid.n_items, 0, kid.arrow_type, nullptr, nullptr, ks.lens, 1};
      if (!canon_items(Kp, ks.in_off, tot2[sc.n_cols + k], &ks.canon, (int32_t*)(kid_fixed[k] + kid.offsets_off), d_tot2 + sc.n_cols + k)) { free_stage(); return fail(ETL_ERR_ALLOC); }
      again = true;
    }
    if (again && (cudaMemcpyAsync(tot2.data(), d_tot2, 8ull * tot2.size(), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)) { free_stage(); return fail(ETL_ERR_CUDA); }
    vi = 0;
    for (uint32_t c = 0; c < sc.n_cols; c++) {
      if (!is_var(A->cols[c].arrow_type)) continue;
      if (A->cols[c].text && A->cols[c].kind == ETL_K_JSON) totals[vi] = tot2[c];     // canonical bytes, not input bytes
      vi++;
    }
    for (size_t k = 0; k < A->kids.size(); k++) A->kids[k].data_bytes = is_var(A->kids[k].arrow_type) ? tot2[sc.n_cols + k] : 0;
  }
  // pass 2: data buffers
  vi = 0;
  for (uint32_t c = 0; c < sc.n_cols; c++) {
    Col& col = A->cols[c];
    if (!is_var(col.arrow_type)) continue;
    if (col.arrow_type == ETL_ARROW_LIST) { vi++; continue; }
    col.data_off = cur; col.data_bytes = n_rows ? totals[vi] : 0; cur += (col.data_bytes + 63) & ~63ull;
    if (col.arrow_type == ETL_ARROW_UTF8 && col.data_bytes > 0x7FFFFFFFull) { A->error = "Utf8 column exceeds 2 GiB: split the batch"; }
    vi++;
  }
  std::vector<uint64_t> kid_base(A->kids.size());
  for (size_t k = 0; k < A->kids.size(); k++) {             // child: validity | values or offsets | data
    Col& kid = A->kids[k];
    kid_base[k] = cur;
    const uint64_t fixed_part = kid.data_off;
    kid.validity_off = cur;
    if (kid.values_bytes) kid.values_off += cur;
    if (kid.offsets_bytes) kid.offsets_off += cur;
    kid.data_off = cur + fixed_part;
    cur += fixed_part + ((kid.data_bytes + 63) & ~63ull);
    if (kid.arrow_type == ETL_ARROW_UTF8 && kid.data_bytes > 0x7FFFFFFFull) { A->error = "Utf8 list child exceeds 2 GiB: split the batch"; }
  }
  // ETL_ARROW_CDC_COLUMNS: cdc_operation and sequence_number after the table's columns, validity | offsets | data each;
  // their sizes follow from n_rows alone
  if (cdc) {
    for (uint32_t len : {etl_fmt::kCdcOpLen, etl_fmt::kSeqKeyLen}) {
      Col col;
      col.arrow_type = ETL_ARROW_UTF8;
      col.validity_off = cur; cur += vbytes;
      col.offsets_off = cur; col.offsets_bytes = ((n_rows + 1) * 4 + 63) & ~63ull; cur += col.offsets_bytes;
      col.data_off = cur; col.data_bytes = n_rows * len; cur += (col.data_bytes + 63) & ~63ull;
      if (col.data_bytes > 0x7FFFFFFFull) A->error = "Utf8 column exceeds 2 GiB: split the batch";
      A->cols.push_back(col);
    }
  }
  A->bytes = cur + 64;
  bool ok = A->error.empty() && cudaMalloc(&A->dev, A->bytes) == cudaSuccess;
  if (ok) ok = cudaMemcpyAsync(A->dev, d_fixed, fixed_bytes, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  for (size_t k = 0; ok && k < A->kids.size(); k++)
    ok = cudaMemcpyAsync(A->dev + kid_base[k], kid_fixed[k], A->kids[k].data_off - kid_base[k], cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  for (uint32_t c = 0; ok && c < sc.n_cols && n_rows; c++) {
    Col& col = A->cols[c];
    if (col.arrow_type != ETL_ARROW_UTF8 && col.arrow_type != ETL_ARROW_LARGE_BINARY) continue;
    ColParams Cp{P.cell_tag, P.cell_val, P.cell_aux, P.heap, dev_stream, d_cell0, n_rows, c, col.arrow_type, nullptr, nullptr, nullptr, col.text};
    const uint32_t grid = (uint32_t)((n_rows * 32 + 255) / 256);
    if (col.text) k_gather_text<<<grid, 256, 0, st>>>(Cp, (const int32_t*)(A->dev + col.offsets_off), A->dev + col.data_off, json_in[c], canon_of[c]);
    else if (col.arrow_type == ETL_ARROW_UTF8) k_gather<int32_t><<<grid, 256, 0, st>>>(Cp, (const int32_t*)(A->dev + col.offsets_off), A->dev + col.data_off);
    else k_gather<int64_t><<<grid, 256, 0, st>>>(Cp, (const int64_t*)(A->dev + col.offsets_off), A->dev + col.data_off);
  }
  for (size_t k = 0; ok && k < A->kids.size(); k++) {
    const Col& kid = A->kids[k];
    const KidSrc& ks = kid_src[k];
    if (!kid.n_items || (kid.arrow_type != ETL_ARROW_UTF8 && kid.arrow_type != ETL_ARROW_LARGE_BINARY)) continue;
    ColParams Kp{ks.tag, ks.val, ks.aux, P.heap, P.heap, nullptr, kid.n_items, 0, kid.arrow_type, nullptr, nullptr, nullptr, kid.text ? 1u : 0u};
    const uint32_t grid = (uint32_t)((kid.n_items * 32 + 255) / 256);
    if (kid.arrow_type == ETL_ARROW_UTF8) k_gather_text<<<grid, 256, 0, st>>>(Kp, (const int32_t*)(A->dev + kid.offsets_off), A->dev + kid.data_off, ks.in_off, ks.canon);
    else k_gather<int64_t><<<grid, 256, 0, st>>>(Kp, (const int64_t*)(A->dev + kid.offsets_off), A->dev + kid.data_off);
  }
  if (ok && cdc) {
    const Col& op = A->cols[sc.n_cols];
    const Col& seq = A->cols[sc.n_cols + 1];
    for (const Col* c : {&op, &seq})                   // validity padding; offsets[0] of 0 rows
      if (ok) ok = cudaMemsetAsync(A->dev + c->validity_off, 0, c->data_off - c->validity_off, st) == cudaSuccess;
    CdcParams Q{d_rec, P.rec_kind, P.rec_commit_lsn, P.rec_tx_ordinal, n_rows,
                (uint32_t*)(A->dev + op.validity_off), (int32_t*)(A->dev + op.offsets_off), A->dev + op.data_off,
                (uint32_t*)(A->dev + seq.validity_off), (int32_t*)(A->dev + seq.offsets_off), A->dev + seq.data_off};
    if (ok && n_rows) k_cdc<<<(uint32_t)((n_rows + 255) / 256), 256, 0, st>>>(Q);
  }
  if (ok && to_host) {
    ok = cudaHostAlloc((void**)&A->host, A->bytes, cudaHostAllocDefault) == cudaSuccess;
    if (ok) ok = cudaMemcpyAsync(A->host, A->dev, A->bytes, cudaMemcpyDeviceToHost, st) == cudaSuccess;
  }
  unsigned bad = 0;
  if (ok && d_bad) ok = cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st) == cudaSuccess;
  if (ok) ok = cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess;
  free_stage();
  if (!ok) return fail(A->error.empty() ? ETL_ERR_CUDA : ETL_ERR_INVALID_ARG);
  if (bad) { A->error = "a Json value the decode accepted did not parse again"; return fail(ETL_ERR_INTERNAL); }
  free_pool();
  *out = A;
  return ETL_OK;
#undef CKA
}
uint64_t etl_dec_arrow_rows(const etl_arrow_batch* a) { return a ? a->n_rows : 0; }
uint32_t etl_dec_arrow_cols(const etl_arrow_batch* a) { return a ? (uint32_t)a->cols.size() : 0; }
uint64_t etl_dec_arrow_first_skipped(const etl_arrow_batch* a) { return a ? a->first_skipped : UINT64_MAX; }
const uint64_t* etl_dec_arrow_row_records(const etl_arrow_batch* a, int host) {
  if (!a) return nullptr;
  const uint8_t* base = host ? a->host : a->dev;
  return base ? reinterpret_cast<const uint64_t*>(base + a->row_rec_off) : nullptr;
}
int etl_dec_arrow_column(const etl_arrow_batch* a, uint32_t c, int host, etl_arrow_column* out) {
  if (!a || !out || c >= a->cols.size()) return ETL_ERR_INVALID_ARG;
  const uint8_t* base = host ? a->host : a->dev;
  if (!base) return ETL_ERR_INVALID_ARG;
  const Col& col = a->cols[c];
  memset(out, 0, sizeof *out);
  out->arrow_type = col.arrow_type;
  if (col.arrow_type == ETL_ARROW_UNSUPPORTED) return ETL_OK;
  out->validity = base + col.validity_off;
  if (col.values_bytes) out->values = base + col.values_off;
  if (col.arrow_type == ETL_ARROW_LIST) out->offsets = base + col.offsets_off;     // the elements: etl_dec_arrow_list_child
  else if (col.offsets_bytes) { out->offsets = base + col.offsets_off; out->data = base + col.data_off; out->data_bytes = col.data_bytes; }
  return ETL_OK;
}
int etl_dec_arrow_list_child(const etl_arrow_batch* a, uint32_t c, int host, etl_arrow_column* out, uint64_t* n_elems) {
  if (!a || !out || c >= a->cols.size() || a->cols[c].arrow_type != ETL_ARROW_LIST) return ETL_ERR_INVALID_ARG;
  const uint8_t* base = host ? a->host : a->dev;
  if (!base) return ETL_ERR_INVALID_ARG;
  memset(out, 0, sizeof *out);
  if (n_elems) *n_elems = 0;
  const Col& col = a->cols[c];
  if (col.child < 0) { out->arrow_type = list_child_type(col.kind); return ETL_OK; }   // no rows: no elements
  const Col& kid = a->kids[(size_t)col.child];
  out->arrow_type = kid.arrow_type;
  out->validity = base + kid.validity_off;
  if (kid.values_bytes) out->values = base + kid.values_off;
  if (kid.offsets_bytes) { out->offsets = base + kid.offsets_off; out->data = base + kid.data_off; out->data_bytes = kid.data_bytes; }
  if (n_elems) *n_elems = kid.n_items;
  return ETL_OK;
}
void etl_dec_arrow_free(etl_arrow_batch* a) {
  if (!a) return;
  if (a->dev) cudaFree(a->dev);
  if (a->host) cudaFreeHost(a->host);
  delete a;
}

}  // extern "C"
