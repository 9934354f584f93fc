// rowbinary_emit.cu — ClickHouse RowBinary emitter: the rows of ONE replicated-schema version of a decoded batch as the
// exact byte stream the ClickHouse destination sends in its INSERT bodies, plus the row offsets that split it.
//
// Replaces the per-row host walk of crates/etl-destinations/src/clickhouse: write_events_inner / flush_pending_rows /
// write_table_rows_inner (core.rs:489-521, :694-863) building Vec<ClickHouseValue> per row with
// cell_to_clickhouse_value (encoding.rs:50-78), expand_key_row / default_cell for key-only deletes (core.rs:920-997),
// and encode_to_row_binary (encoding.rs:249-273) called row by row from insert_rows (client.rs:336-379).
//
// Rows: Insert → new image; Update → new image when Full (a partial one is reported, not emitted); Delete → the Full old
// image, or the key image expanded to full width; COPY batches (rec_kind == NULL): every row of the valid prefix.  The
// columns are the schema's, then cdc_operation (String) and cdc_lsn (UInt64).  Values follow the cell's variant.
//
// Passes (one CUDA stream, three syncs: selection, Json sizes when a Json column exists, output size):
//   1. select_rows<ClickHouseRows> (emit_scan.cuh): rows in record order, first partial update.  COPY: k_copy_sel, no
//      sync.
//   2. Json (stage_json, row_emit_common.cuh): every Json cell and Json array element is canonicalised
//      once (etl_fmt::json_canon) into scratch laid out per item (row, Json column) from a scan of the input lengths:
//      [u32 canonical length][text] per document, each record 4 + input bytes long (the canonical text is never longer
//      than the input).
//   3. k_rb_size: thread per (row, column) over W = n_cols + 2 in row-major order: the cell's byte length with its
//      marker; the first Date32 violation and the first NULL under a cleared flag by warp-reduced atomicMin.
//   4. k_row_scan (warp per row, row_emit_common.cuh): lengths → u32 in-row cell offsets + the row's length; the row
//      lengths are scanned into u64 row offsets (scan_lengths, emit_scan.cuh); the total sizes the output.
//   5. k_rb_write: thread per (row, column), so consecutive lanes store adjacent bytes of a row; String / Json / hex
//      payloads above kLongCell bytes are copied by the whole warp.  k_rb_date_elem finds the element of an array
//      Date32 violation.
// Scratch: 4 B per (row, column) + 4 B per row + the selection's 16 B per record; with Json columns 4 B per (row, Json
// column) + 8 B per item + 17 B per input Json byte.  Scratch is stream-ordered (cudaMallocAsync), the output is not.
#include <cuda_runtime.h>

#include <vector>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "rowbinary_format.cuh"
#include "batch_internal.h"
#include "emit_scan.cuh"
#include "row_emit_common.cuh"

namespace {

// write_events_inner (core.rs:694-802): which image of record r is a row
struct ClickHouseRows {
  __device__ __forceinline__ int operator()(const SelParams& S, uint64_t r, uint64_t* cell0) const {
    if (r >= S.n_records || S.rec_schema[r] != S.schema) return kNotRow;
    const uint32_t k = S.rec_kind[r], f = S.rec_flags[r];
    if (!(f & ETL_RF_EVENT)) return kNotRow;
    const uint64_t c0 = S.rec_cell_base[r];
    if (k == 'I') { *cell0 = c0; return kRow; }
    if (k == 'U') {
      if (f & ETL_RF_NEW_PARTIAL) return kSkipped;                   // InvalidState (core.rs:721-735)
      *cell0 = S.rec_cell_base[r + 1] - S.n_cols;
      return kRow;
    }
    if (k == 'D' && (f & (ETL_RF_OLD_FULL | ETL_RF_OLD_KEY))) { *cell0 = c0; return kRow; }   // old image first
    return kNotRow;
  }
};

// how a column of a key image is filled (expand_key_row, core.rs:944-962)
enum : uint8_t { kFromCell = 0, kKeyNull = 1, kKeyDefault = 2 };
struct RbCol {
  uint8_t kind;       // ETL_K_* (0 for the CDC columns)
  uint8_t nullable;   // Nullable(...) in ClickHouse: a marker byte precedes the value
  uint8_t key_mode;   // in a key image: kFromCell (primary-key column, key cell key_slot), kKeyNull or kKeyDefault
  uint8_t _pad;
  uint16_t key_slot;
  int16_t json;       // index among the columns whose cells can hold Json text (Json, Json[]); -1 otherwise
};
constexpr uint32_t kLongCell = 64;   // payload bytes above which a String / Json / hex value is copied by the warp
constexpr unsigned kFull = 0xffffffffu;
enum { kIssueDate = 0, kIssueNull = 1, kIssueFlags = 2, kIssueElem = 3, kIssueSlots = 4 };
enum { kFlagBadJson = 1, kFlagRowTooLong = 2 };

struct RbParams {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  const uint8_t* rec_kind; const uint8_t* rec_flags; const uint64_t* rec_commit_lsn;   // rec_kind NULL: COPY rows
  const uint64_t* row_cell0; const uint64_t* row_rec; uint64_t n_rows;
  const RbCol* cols; const uint32_t* json_col;   // W entries; n_json column indices
  uint32_t n_cols, w, n_ident, n_json;
  const uint64_t* json_off; uint8_t* canon;   // per Json item: offset of its records in canon
  uint32_t* cell_len;        // n_rows * w: lengths, then offsets inside the row
  uint32_t* row_len;
  const uint64_t* row_off;   // n_rows + 1
  uint8_t* out;
  unsigned long long* issues;   // kIssue*: (row << 32 | column) of the first Date32 / NULL issue, flags, element
};

// the cell behind column c of row `row`: kFromCell and its index, or a key image's kKeyNull / kKeyDefault
__device__ __forceinline__ uint32_t cell_at(const RbParams& P, uint64_t row, uint32_t c, uint64_t* cell) {
  const uint64_t c0 = P.row_cell0[row];
  if (P.rec_kind) {
    const uint64_t r = P.row_rec[row];
    if (P.rec_kind[r] == 'D' && !(P.rec_flags[r] & ETL_RF_OLD_FULL)) {   // OldTableRow::Key
      const RbCol& col = P.cols[c];
      if (col.key_mode != kFromCell) return col.key_mode;
      if (col.key_slot >= P.n_ident) return kKeyNull;                   // key_iter.next().unwrap_or(Cell::Null)
      *cell = c0 + col.key_slot;
      return kFromCell;
    }
  }
  *cell = c0 + c;
  return kFromCell;
}

// default_cell (core.rs:970-997) on the wire: all zero bytes, as many as the decode class's value takes; String-like
// classes and arrays are an empty string / array, one varint byte
__device__ __forceinline__ uint32_t default_width(uint32_t k) {
  switch (k) {
    case ETL_K_BOOL: return 1;
    case ETL_K_I16: return 2;
    case ETL_K_I32: case ETL_K_U32: case ETL_K_F32: case ETL_K_DATE: return 4;
    case ETL_K_I64: case ETL_K_F64: case ETL_K_TIMESTAMP: case ETL_K_TIMESTAMPTZ: return 8;
    case ETL_K_UUID: return 16;
    default: return 1;
  }
}

// rb_encode_value (encoding.rs:201-246) of a non-NULL scalar: its length.  String / Json / Bytes: the payload length is
// `n` (text, canonical Json, input bytes before hex)
__device__ __forceinline__ uint64_t scalar_len(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, uint32_t n) {
  switch (tag) {
    case ETL_CELL_BOOL: return 1;
    case ETL_CELL_I16: return 2;
    case ETL_CELL_I32: case ETL_CELL_U32: case ETL_CELL_F32: case ETL_CELL_DATE: return 4;
    case ETL_CELL_I64: case ETL_CELL_F64: case ETL_CELL_TIMESTAMP: case ETL_CELL_TIMESTAMPTZ: return 8;
    case ETL_CELL_UUID: return 16;
    case ETL_CELL_STRING: case ETL_CELL_JSON: return etl_rb::varint_len(n) + n;
    case ETL_CELL_BYTES: return etl_rb::varint_len(2ull * n) + 2ull * n;
    case ETL_CELL_NUMERIC: { const uint32_t k = etl_fmt::numeric_len(heap + val, aux); return etl_rb::varint_len(k) + k; }
    case ETL_CELL_TIME: return 1 + etl_rb::time_len(aux);
    default: return 0;
  }
}
// ... and its bytes; `src` is the payload of a String / Json / Bytes value (n bytes; Bytes are written as hex)
__device__ __forceinline__ uint64_t scalar_write(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, const uint8_t* src, uint32_t n, uint8_t* o) {
  switch (tag) {
    case ETL_CELL_BOOL: *o = (uint8_t)(val & 1u); return 1;
    case ETL_CELL_I16: etl_rb::le_write(val, 2, o); return 2;
    case ETL_CELL_I32: case ETL_CELL_U32: case ETL_CELL_F32: case ETL_CELL_DATE: etl_rb::le_write(val, 4, o); return 4;
    case ETL_CELL_I64: case ETL_CELL_F64: etl_rb::le_write(val, 8, o); return 8;
    case ETL_CELL_TIMESTAMP: case ETL_CELL_TIMESTAMPTZ:   // timestamp_micros(): the Arrow TIMESTAMP_US arithmetic
      etl_rb::le_write((uint64_t)((int64_t)val * 1000000ll + (int64_t)(aux / 1000u)), 8, o); return 8;
    case ETL_CELL_UUID: etl_rb::uuid_write(heap + val, o); return 16;
    case ETL_CELL_STRING: case ETL_CELL_JSON: {
      const uint32_t v = etl_rb::varint_write(n, o);
      for (uint32_t k = 0; k < n; k++) o[v + k] = src[k];
      return v + n;
    }
    case ETL_CELL_BYTES: {
      const uint32_t v = etl_rb::varint_write(2ull * n, o);
      etl_rb::hex_write(src, n, o + v);
      return v + 2ull * n;
    }
    case ETL_CELL_NUMERIC: {
      const uint32_t k = etl_fmt::numeric_len(heap + val, aux);
      const uint32_t v = etl_rb::varint_write(k, o);
      etl_fmt::numeric_write(heap + val, aux, o + v);
      return v + k;
    }
    case ETL_CELL_TIME: { o[0] = (uint8_t)etl_rb::time_len(aux); return 1 + etl_rb::time_write(val, aux, o + 1); }
    default: return 0;
  }
}

// an array value: varint(n), then every element as Nullable (encoding.rs:238-244).  `canon` walks the item's Json
// records (Json elements).  Sizing when o == NULL; *bad_date = first element out of the Date32 range
__device__ uint64_t array_value(const RbParams& P, uint64_t val, uint32_t aux, const uint8_t* canon, uint8_t* o, uint32_t* bad_date) {
  const etl_array_elem* E = array_elems(P.heap, val);
  uint64_t len = o ? etl_rb::varint_write(aux, o) : etl_rb::varint_len(aux);
  for (uint32_t k = 0; k < aux; k++) {
    const etl_array_elem e = E[k];
    if (e.tag == ETL_CELL_NULL) { if (o) o[len] = 1; len += 1; continue; }
    const uint8_t* src = P.heap + e.val;
    uint32_t n = e.aux;
    if (e.tag == ETL_CELL_JSON) { n = rd32(canon); src = canon + 4; canon += 4 + e.aux; }
    if (e.tag == ETL_CELL_DATE && !etl_rb::date32_ok((int64_t)e.val) && *bad_date == UINT32_MAX) *bad_date = k;
    if (o) { o[len] = 0; len += 1 + scalar_write(e.tag, e.val, e.aux, P.heap, src, n, o + len + 1); }
    else len += 1 + scalar_len(e.tag, e.val, e.aux, P.heap, n);
  }
  return len;
}

// ---------------------------------------------------------------- Json
// item i = (row, Json column j), staged by row_emit_common.cuh
struct RbJsonCells {
  RbParams P;
  __device__ __forceinline__ bool operator()(uint64_t i, uint64_t* cell) const {
    const uint64_t row = i / P.n_json;
    return cell_at(P, row, P.json_col[i - row * P.n_json], cell) == kFromCell;
  }
};

// ---------------------------------------------------------------- size, offsets, write
// the payload of a String / Json / Bytes scalar cell
__device__ __forceinline__ const uint8_t* payload(const RbParams& P, uint64_t row, const RbCol& col, uint32_t tag, uint64_t val, uint32_t* n) {
  if (tag == ETL_CELL_JSON) { const uint8_t* r = P.canon + P.json_off[row * P.n_json + col.json]; *n = rd32(r); return r + 4; }
  if (tag == ETL_CELL_STRING) return cell_text(P.stream, P.heap, val);
  return P.heap + val;
}

__global__ void __launch_bounds__(256) k_rb_size(RbParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long date_key = ~0ull, null_key = ~0ull;
  if (i < P.n_rows * P.w) {
    const uint64_t row = i / P.w;
    const uint32_t c = (uint32_t)(i - row * P.w);
    const RbCol col = P.cols[c];
    const uint32_t m = col.nullable;
    uint64_t len = m;
    uint64_t cell = 0;
    const uint32_t how = c < P.n_cols ? cell_at(P, row, c, &cell) : kFromCell;
    if (c >= P.n_cols) len += c == P.n_cols ? 1u + etl_fmt::kCdcOpLen : 8u;    // cdc_operation, cdc_lsn
    else if (how == kKeyDefault) len += default_width(col.kind);
    else {
      const uint32_t tag = how == kKeyNull ? (uint32_t)ETL_CELL_NULL : P.cell_tag[cell];
      if (tag == ETL_CELL_NULL) { if (!m) null_key = row << 32 | c; }
      else {
        const uint64_t val = P.cell_val[cell];
        uint32_t aux = P.cell_aux[cell];
        if (tag == ETL_CELL_ARRAY) {
          uint32_t bad = UINT32_MAX;
          len += array_value(P, val, aux, col.json >= 0 ? P.canon + P.json_off[row * P.n_json + col.json] : nullptr, nullptr, &bad);
          if (bad != UINT32_MAX) date_key = row << 32 | c;
        } else {
          if (tag == ETL_CELL_JSON) payload(P, row, col, tag, val, &aux);
          if (tag == ETL_CELL_DATE && !etl_rb::date32_ok((int64_t)val)) date_key = row << 32 | c;
          len += scalar_len(tag, val, P.cell_aux[cell], P.heap, aux);
        }
      }
    }
    P.cell_len[i] = len > 0xffffffffull ? 0xffffffffu : (uint32_t)len;
  }
  report_min(date_key, P.issues + kIssueDate);
  report_min(null_key, P.issues + kIssueNull);
}

__global__ void __launch_bounds__(256) k_rb_write(RbParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const uint8_t* lsrc = nullptr;
  uint8_t* ldst = nullptr;
  uint32_t ln = 0, lhex = 0;
  if (i < P.n_rows * P.w) {
    const uint64_t row = i / P.w;
    const uint32_t c = (uint32_t)(i - row * P.w);
    const RbCol col = P.cols[c];
    uint8_t* o = P.out + P.row_off[row] + P.cell_len[i];
    uint64_t cell = 0;
    const uint32_t how = c < P.n_cols ? cell_at(P, row, c, &cell) : kFromCell;
    if (c >= P.n_cols) {
      if (col.nullable) *o++ = 0;
      const uint64_t r = P.rec_kind ? P.row_rec[row] : 0;
      if (c == P.n_cols) { *o = (uint8_t)etl_fmt::kCdcOpLen; etl_fmt::cdc_op_write(P.rec_kind ? P.rec_kind[r] : 'I', o + 1); }
      else etl_rb::le_write(P.rec_kind ? P.rec_commit_lsn[r] : 0ull, 8, o);   // COPY rows: LSN 0
    } else if (how == kKeyDefault) {
      for (uint32_t k = 0, n = col.nullable + default_width(col.kind); k < n; k++) o[k] = 0;
    } else {
      const uint32_t tag = how == kKeyNull ? (uint32_t)ETL_CELL_NULL : P.cell_tag[cell];
      if (tag == ETL_CELL_NULL) { if (col.nullable) *o = 1; }         // no bytes under a cleared flag (reported)
      else {
        if (col.nullable) *o++ = 0;
        const uint64_t val = P.cell_val[cell];
        const uint32_t aux = P.cell_aux[cell];
        if (tag == ETL_CELL_ARRAY) {
          uint32_t bad = UINT32_MAX;
          array_value(P, val, aux, col.json >= 0 ? P.canon + P.json_off[row * P.n_json + col.json] : nullptr, o, &bad);
        } else if (tag == ETL_CELL_STRING || tag == ETL_CELL_JSON || tag == ETL_CELL_BYTES) {
          uint32_t n = aux;
          const uint8_t* src = payload(P, row, col, tag, val, &n);
          const bool hex = tag == ETL_CELL_BYTES;
          if ((hex ? 2ull * n : n) > kLongCell) {          // the warp copies it below
            ldst = o + etl_rb::varint_write(hex ? 2ull * n : n, o);
            lsrc = src; ln = n; lhex = hex;
          } else scalar_write(tag, val, aux, P.heap, src, n, o);
        } else scalar_write(tag, val, aux, P.heap, nullptr, 0, o);
      }
    }
  }
  unsigned todo = __ballot_sync(kFull, ldst != nullptr);
  while (todo) {
    const int src_lane = __ffs(todo) - 1;
    todo &= todo - 1;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(kFull, reinterpret_cast<unsigned long long>(lsrc), src_lane));
    uint8_t* d = reinterpret_cast<uint8_t*>(__shfl_sync(kFull, reinterpret_cast<unsigned long long>(ldst), src_lane));
    const uint32_t n = __shfl_sync(kFull, ln, src_lane);
    if (__shfl_sync(kFull, lhex, src_lane)) { for (uint32_t k = lane; k < n; k += 32) etl_rb::hex_byte(s[k], d + 2 * k); }
    else for (uint32_t k = lane; k < n; k += 32) d[k] = s[k];
  }
}

// the element of the first Date32 violation when its cell is an array (UINT32_MAX stays for a scalar)
__global__ void k_rb_date_elem(RbParams P) {
  const unsigned long long key = P.issues[kIssueDate];
  if (key == ~0ull) return;
  const uint64_t row = key >> 32;
  const uint32_t c = (uint32_t)(key & 0xffffffffu);
  uint64_t cell = 0;
  if (cell_at(P, row, c, &cell) != kFromCell || P.cell_tag[cell] != ETL_CELL_ARRAY) return;
  const etl_array_elem* E = array_elems(P.heap, P.cell_val[cell]);
  for (uint32_t k = 0; k < P.cell_aux[cell]; k++)
    if (E[k].tag == ETL_CELL_DATE && !etl_rb::date32_ok((int64_t)E[k].val)) { P.issues[kIssueElem] = k; return; }
}

}  // namespace

struct etl_rowbinary_batch : RowPayload {
  etl_rowbinary_issues issues{};
};

extern "C" {

int etl_dec_rowbinary_emit(const etl_dec_batch* batch, uint32_t schema_index, const uint8_t* nullable_flags, uint32_t n_flags,
                           int to_host, etl_rowbinary_batch** out) {
  if (!batch || !out || (n_flags && !nullable_flags)) return ETL_ERR_INVALID_ARG;
  EmitBatch E;
  if (open_emit_batch(batch, schema_index, &E) != ETL_OK) return ETL_ERR_INVALID_ARG;
  const etl_dec_planes& P = E.P;
  const etl_dec_schema_info& sc = E.sc;
  const uint8_t* pk = nullptr;
  if (!E.copy && !etl_schema_pk_columns(batch, schema_index, &pk)) return ETL_ERR_INVALID_ARG;
  if (n_flags != sc.n_cols + 2) return ETL_ERR_INVALID_ARG;
  const uint32_t W = sc.n_cols + 2;
  // column descriptors: the flags, expand_key_row's rule per column, the Json item index
  std::vector<RbCol> cols(W);
  std::vector<uint32_t> json_col;
  uint32_t key_slot = 0;
  for (uint32_t c = 0; c < W; c++) {
    RbCol& d = cols[c];
    d.kind = c < sc.n_cols ? sc.col_kind[c] : 0;
    d.nullable = nullable_flags[c] ? 1 : 0;
    d.json = -1;
    if (c >= sc.n_cols) continue;
    if (pk && pk[c]) { d.key_mode = kFromCell; d.key_slot = (uint16_t)key_slot++; }
    else d.key_mode = (sc.col_flags && (sc.col_flags[c] & 1u) && !(d.kind & ETL_K_ARRAY)) ? kKeyNull : kKeyDefault;
    if ((d.kind & ~(uint32_t)ETL_K_ARRAY) == ETL_K_JSON) { d.json = (int16_t)json_col.size(); json_col.push_back(c); }
  }

  cudaStream_t st = cudaStreamPerThread;
  etl_rowbinary_batch* B = new etl_rowbinary_batch();
  Scratch scratch(st);
  auto fail = [&](int rc) {
    scratch.release();
    cudaStreamSynchronize(st);
    cudaGetLastError();
    delete B;
    return rc;
  };
  const uint64_t n_valid = E.n_valid;
  const uint32_t nb = (uint32_t)((n_valid + kSelThreads - 1) / kSelThreads);
  uint32_t* d_blk = (uint32_t*)scratch((nb + 1) * 4ull);
  uint64_t* d_cell0 = (uint64_t*)scratch((n_valid + 1) * 8);
  uint64_t* d_rec = (uint64_t*)scratch((n_valid + 1) * 8);
  unsigned long long* d_n = (unsigned long long*)scratch(8 * (2 + kIssueSlots));   // rows, first partial | issues
  RbCol* d_cols = (RbCol*)scratch(sizeof(RbCol) * W + 4ull * json_col.size());
  if (!d_blk || !d_cell0 || !d_rec || !d_n || !d_cols) return fail(ETL_ERR_ALLOC);
  unsigned long long* d_issues = d_n + 2;
  uint32_t* d_json_col = reinterpret_cast<uint32_t*>(d_cols + W);
  if (cudaMemsetAsync(d_n, 0xff, 8 * (2 + kIssueSlots), st) != cudaSuccess || cudaMemsetAsync(d_issues + kIssueFlags, 0, 8, st) != cudaSuccess ||
      cudaMemcpyAsync(d_cols, cols.data(), sizeof(RbCol) * W, cudaMemcpyHostToDevice, st) != cudaSuccess ||
      (!json_col.empty() && cudaMemcpyAsync(d_json_col, json_col.data(), 4 * json_col.size(), cudaMemcpyHostToDevice, st) != cudaSuccess))
    return fail(ETL_ERR_CUDA);
  unsigned long long sel[2] = {0, UINT64_MAX};          // rows, first partial update
  const SelParams Sp{P.rec_kind, P.rec_flags, P.rec_schema, P.rec_cell_base, n_valid, (int32_t)schema_index, 0u, sc.n_cols, d_blk, d_cell0, d_rec, d_n};
  if (select_rows<ClickHouseRows>(Sp, E.copy, n_valid, st, sel) != ETL_OK) return fail(ETL_ERR_CUDA);
  const uint64_t n_rows = sel[0];
  B->n_rows = n_rows;
  B->issues.first_partial_update = sel[1];
  if (cudaMalloc(&B->meta, B->meta_bytes()) != cudaSuccess) { B->meta = nullptr; return fail(ETL_ERR_ALLOC); }
  if (cudaMemsetAsync(B->meta, 0, 8, st) != cudaSuccess ||
      (n_rows && cudaMemcpyAsync(B->meta + (n_rows + 1) * 8, d_rec, n_rows * 8, cudaMemcpyDeviceToDevice, st) != cudaSuccess))
    return fail(ETL_ERR_CUDA);

  RbParams R{P.cell_tag, P.cell_val, P.cell_aux, P.heap, E.stream, P.rec_kind, P.rec_flags, P.rec_commit_lsn,
             d_cell0, d_rec, n_rows, d_cols, d_json_col, sc.n_cols, W, sc.n_identity, (uint32_t)json_col.size(),
             nullptr, nullptr, nullptr, nullptr, (const uint64_t*)B->meta, nullptr, d_issues};
  unsigned long long tot[2] = {0, 0};                   // output bytes, issue flags
  if (n_rows) {
    // Json: input lengths → item offsets → (sync) canonical text
    const uint64_t n_items = n_rows * R.n_json;
    if (n_items) {
      JsonStage J{P.cell_tag, P.cell_val, P.cell_aux, P.heap, E.stream, n_items, nullptr, nullptr, nullptr,
                  d_issues + kIssueFlags, (unsigned long long)kFlagBadJson};
      if (int rc = stage_json(scratch, J, RbJsonCells{R}, st)) return fail(rc);
      R.json_off = J.off;
      R.canon = J.canon;
    }
    // sizes → in-row offsets → row offsets (sync)
    const uint64_t n_cells = n_rows * W;
    const uint32_t rb = scan_blocks(n_rows);
    R.cell_len = (uint32_t*)scratch(n_cells * 4);
    R.row_len = (uint32_t*)scratch(n_rows * 4);
    unsigned long long* rblk = (unsigned long long*)scratch((rb + 1) * 8ull);
    if (!R.cell_len || !R.row_len || !rblk) return fail(ETL_ERR_ALLOC);
    k_rb_size<<<(uint32_t)((n_cells + 255) / 256), 256, 0, st>>>(R);
    k_row_scan<<<(uint32_t)((n_rows * 32 + 255) / 256), 256, 0, st>>>(R.cell_len, W, n_rows, R.row_len, d_issues + kIssueFlags,
                                                                       (unsigned long long)kFlagRowTooLong);
    scan_lengths(R.row_len, n_rows, rblk, rblk + rb, (uint64_t*)B->meta, st);
    if (cudaMemcpyAsync(&tot[0], rblk + rb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(&tot[1], d_issues + kIssueFlags, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    if (tot[1] & kFlagBadJson) return fail(ETL_ERR_INTERNAL);       // a Json value the decode accepted did not parse again
    if (tot[1] & kFlagRowTooLong) return fail(ETL_ERR_INVALID_ARG); // one row of 4 GiB or more
  }
  B->bytes = tot[0];
  if (cudaMalloc(&B->data, B->bytes + 64) != cudaSuccess) { B->data = nullptr; return fail(ETL_ERR_ALLOC); }
  if (n_rows) {
    R.out = B->data;
    k_rb_write<<<(uint32_t)((n_rows * W + 255) / 256), 256, 0, st>>>(R);
    k_rb_date_elem<<<1, 1, 0, st>>>(R);
  }
  if (to_host) {
    if (int rc = B->copy_to_host(st)) return fail(rc);
  }
  unsigned long long iss[kIssueSlots];
  if (cudaMemcpyAsync(iss, d_issues, sizeof iss, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  scratch.release();
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ETL_ERR_CUDA);
  auto issue = [](unsigned long long key, uint32_t elem) {
    etl_rb_issue x{UINT64_MAX, UINT32_MAX, UINT32_MAX};
    if (key != ~0ull) { x.row = key >> 32; x.column = (uint32_t)(key & 0xffffffffu); x.element = elem; }
    return x;
  };
  B->issues.date_range = issue(iss[kIssueDate], (uint32_t)iss[kIssueElem]);
  B->issues.null_value = issue(iss[kIssueNull], UINT32_MAX);
  *out = B;
  return ETL_OK;
}
uint64_t etl_dec_rowbinary_rows(const etl_rowbinary_batch* b) { return RowPayload::rows_of(b); }
uint64_t etl_dec_rowbinary_bytes(const etl_rowbinary_batch* b) { return RowPayload::bytes_of(b); }
const uint8_t* etl_dec_rowbinary_data(const etl_rowbinary_batch* b, int host) { return RowPayload::data_of(b, host); }
const uint64_t* etl_dec_rowbinary_row_offsets(const etl_rowbinary_batch* b, int host) { return RowPayload::offsets_of(b, host); }
const uint64_t* etl_dec_rowbinary_row_records(const etl_rowbinary_batch* b, int host) { return RowPayload::records_of(b, host); }
int etl_dec_rowbinary_issues(const etl_rowbinary_batch* b, etl_rowbinary_issues* out) {
  if (!b || !out) return ETL_ERR_INVALID_ARG;
  *out = b->issues;
  return ETL_OK;
}
void etl_dec_rowbinary_free(etl_rowbinary_batch* b) { delete b; }

}  // extern "C"
