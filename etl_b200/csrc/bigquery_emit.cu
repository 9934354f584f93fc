// bigquery_emit.cu — BigQuery Storage Write emitter: the rows of ONE replicated-schema version of a decoded batch as the
// serialized protobuf messages that go into ProtoRows.serialized_rows, plus the row offsets that split them.
//
// Replaces the per-row host walk of crates/etl-destinations/src/bigquery: write_events (core.rs:792-970) pushing the
// _CHANGE_TYPE / _CHANGE_SEQUENCE_NUMBER cells, bigquery_update_rows / bigquery_primary_key_changed (:1255-1403)
// splitting a primary-key change into DELETE + UPSERT, bigquery_delete_row (:1406-1524), write_table_rows (:530-546),
// BigQueryTableRow::try_from_tagged_cells (encoding.rs:49-83) with validate_cell_for_bigquery (validation.rs), and the
// prost serialisation cell_encode_prost / array_cell_encode_prost (encoding.rs:151-342).
//
// Rows: Insert → UPSERT of the new image; Update → UPSERT of the new image, preceded by a DELETE of the old key when a
// primary-key cell changed; Delete → DELETE of the old key.  A DELETE row holds only the primary-key columns.  Field
// c + 1 is column c, n_cols + 1 is _CHANGE_TYPE, n_cols + 2 is _CHANGE_SEQUENCE_NUMBER
// "{commit_lsn:016x}/{tx_ordinal:016x}/{ordinal:016x}".  COPY batches (rec_kind == NULL): every row of the valid prefix
// as an UPSERT without the sequence field.
//
// Passes (one CUDA stream, four syncs: selection, Json sizes when a Json column exists, row count (not for COPY),
// output size):
//   1. select_rows<BigQueryRecords> (emit_scan.cuh): the version's records that give rows, in record order, and the
//      first record write_events rejects.  COPY: k_copy_sel, no sync.
//   2. Json (stage_json, row_emit_common.cuh): items are (record, Json column, image): the new image's
//      Json cells and the old image's primary-key Json cells, canonicalised once.  The key comparison and the rows read
//      the canonical text.
//   3. k_bq_expand (warp per record): 1 or 2 rows; an Update compares its old and new primary-key cells with Cell's
//      PartialEq, long payloads compared by the warp.  The counts are scanned (scan_lengths, emit_scan.cuh) and k_bq_rows writes each row's descriptor and record.
//   4. k_bq_size: thread per (row, field) over W = n_cols + 2: the field's bytes; the first value issue by warp-reduced
//      atomicMin of (row << 32 | column).  k_row_scan (row_emit_common.cuh) turns them into in-row offsets and row
//      lengths, scanned into u64 row offsets.
//   5. k_bq_write: thread per (row, field); String / Json / Bytes payloads above kLongCell bytes are copied by the warp.
//      k_bq_issue finds the kind and element of the reported issue.
// Scratch: 4 B per (row, field) + 12 B per row + 28 B per record of the batch (selection 16 B, row counts 4 B, first
// row 8 B); with Json columns 12 B per (record, Json column, image) + 17 B per input Json byte.  Scratch is
// stream-ordered (cudaMallocAsync), the output is not.
// ptxas (-Xptxas -v, sm_90a): k_bq_expand 37 registers, k_bq_size 32 (16 B stack, 44 B spill stores / 24 B loads around
// the out-of-line array_field call), k_bq_write 40, k_bq_rows 16, k_bq_issue 28, k_json_canon 56 (80 B stack, 16 B
// spills, as in the RowBinary emitter), k_json_len 22, k_row_scan 24; no other spills.
#include <cuda_runtime.h>

#include <vector>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "rowbinary_format.cuh"
#include "bigquery_format.cuh"
#include "batch_internal.h"
#include "emit_scan.cuh"
#include "row_emit_common.cuh"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr uint32_t kLongCell = 64;   // payload bytes above which a String / Json / Bytes value is copied by the warp
constexpr uint32_t kSeqLen = 50, kOpLen = 6;
enum { kIssueKey = 0, kIssueFlags = 1, kIssueKind = 2, kIssueElem = 3, kIssueSlots = 4 };
enum { kFlagBadJson = 1, kFlagRowTooLong = 2 };

// write_events (core.rs:815-903): which records give rows.  S.row_kinds = 1 when the version's identity columns are its
// primary-key columns (identity_matches_primary_key); a key image is rejected otherwise
struct BigQueryRecords {
  __device__ __forceinline__ int operator()(const SelParams& S, uint64_t r, uint64_t* cell0) const {
    if (r >= S.n_records || S.rec_schema[r] != S.schema) return kNotRow;
    const uint32_t k = S.rec_kind[r], f = S.rec_flags[r];
    if (!(f & ETL_RF_EVENT)) return kNotRow;
    *cell0 = S.rec_cell_base[r];
    const bool key_image = (f & ETL_RF_OLD_KEY) && !(f & ETL_RF_OLD_FULL);
    if (k == 'I') return kRow;
    if (k == 'U') {
      if (f & ETL_RF_NEW_PARTIAL) return kSkipped;                   // core.rs:837-850
      return key_image && !S.row_kinds ? kSkipped : kRow;            // core.rs:1347-1359
    }
    if (k == 'D') {
      if (!(f & (ETL_RF_OLD_FULL | ETL_RF_OLD_KEY))) return kSkipped;  // core.rs:868-879
      return key_image && !S.row_kinds ? kSkipped : kRow;            // core.rs:1439-1451
    }
    return kNotRow;
  }
};

struct BqCol {
  uint8_t kind;       // ETL_K_*
  uint8_t pk;         // the stored TableSchema column has a primary_key_ordinal_position
  uint16_t key_slot;  // primary-key columns: index among them (the key image's cell)
  int16_t json;       // index among the columns whose cells can hold Json text (Json, Json[]); -1 otherwise
  uint16_t _pad;
};

struct BqParams {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  const uint8_t* rec_kind; const uint8_t* rec_flags; const uint64_t* rec_commit_lsn; const uint64_t* rec_tx_ordinal;
  const uint64_t* rec_cell_base;                         // rec_kind NULL: COPY rows
  const uint64_t* sel_cell0; const uint64_t* sel_rec; uint64_t n_sel;
  const BqCol* cols; const uint32_t* json_col; const uint32_t* pk_col;
  uint32_t n_cols, w, n_json, n_pk;
  const uint64_t* json_off; const uint8_t* canon;        // item (s, j, img) = (s * n_json + j) * 2 + img
  uint32_t* sel_cnt; const uint64_t* sel_row0;           // rows per selected record, its first row
  uint64_t* row_desc; uint64_t* row_rec; uint64_t n_rows;   // row: s << 2 | ordinal << 1 | delete
  uint32_t* cell_len; uint32_t* row_len; const uint64_t* row_off;
  uint8_t* out;
  unsigned long long* issues;   // kIssue*: (row << 32 | column) of the first value issue, flags, its kind, its element
};

// the cell of column c in image img (0 new, 1 old) of selected record s; false: no such cell (a Delete has no new
// image, an Insert no old one, an old image only gives the primary-key columns)
__device__ __forceinline__ bool image_cell(const BqParams& P, uint64_t s, uint32_t img, uint32_t c, uint64_t* cell) {
  const uint64_t c0 = P.sel_cell0[s];
  if (!P.rec_kind) { *cell = c0 + c; return img == 0; }
  const uint64_t r = P.sel_rec[s];
  const uint32_t k = P.rec_kind[r], f = P.rec_flags[r];
  if (img == 0) {
    if (k == 'D') return false;
    *cell = k == 'U' ? P.rec_cell_base[r + 1] - P.n_cols + c : c0 + c;
    return true;
  }
  if (k == 'I' || !P.cols[c].pk) return false;
  if (f & ETL_RF_OLD_FULL) { *cell = c0 + c; return true; }
  if (f & ETL_RF_OLD_KEY) { *cell = c0 + P.cols[c].key_slot; return true; }   // identity == primary key (selection)
  return false;
}
__device__ __forceinline__ const uint8_t* canon_of(const BqParams& P, uint64_t s, uint32_t json, uint32_t img) {
  return P.canon + P.json_off[((uint64_t)s * P.n_json + json) * 2 + img];
}

struct BqJsonCells {
  BqParams P;
  __device__ __forceinline__ bool operator()(uint64_t i, uint64_t* cell) const {
    const uint64_t s = i / (2ull * P.n_json);
    const uint32_t rem = (uint32_t)(i - s * 2ull * P.n_json);
    return image_cell(P, s, rem & 1u, P.json_col[rem >> 1], cell);
  }
};

// ---------------------------------------------------------------- key comparison (Cell's derived PartialEq)
__device__ __forceinline__ bool bytes_eq_warp(const uint8_t* a, const uint8_t* b, uint32_t n) {
  bool ok = true;
  for (uint32_t k = threadIdx.x & 31; k < n; k += 32) if (a[k] != b[k]) { ok = false; break; }
  return __all_sync(kFull, ok);
}
// one non-NULL value of variant tag on both sides; pa / pb: the payload of a String / Bytes / Uuid / Numeric value
// (Numeric: its heap entry) or the canonical text of a Json value (xa / xb its length)
__device__ bool value_eq_warp(uint32_t tag, uint64_t va, uint32_t xa, const uint8_t* pa, uint64_t vb, uint32_t xb, const uint8_t* pb) {
  switch (tag) {
    case ETL_CELL_BOOL: case ETL_CELL_I16: case ETL_CELL_I32: case ETL_CELL_U32: case ETL_CELL_I64: case ETL_CELL_DATE:
      return va == vb;
    case ETL_CELL_F32: return __uint_as_float((uint32_t)va) == __uint_as_float((uint32_t)vb);
    case ETL_CELL_F64: return __longlong_as_double((long long)va) == __longlong_as_double((long long)vb);
    case ETL_CELL_TIME: case ETL_CELL_TIMESTAMP: case ETL_CELL_TIMESTAMPTZ: return va == vb && xa == xb;
    case ETL_CELL_UUID: return bytes_eq_warp(pa, pb, 16);
    case ETL_CELL_STRING: case ETL_CELL_BYTES: case ETL_CELL_JSON: return xa == xb && bytes_eq_warp(pa, pb, xa);
    case ETL_CELL_NUMERIC: {   // kind, sign, weight, scale, digits (pushed_groups is decode bookkeeping)
      if (xa != xb) return false;
      const etl_numeric_hdr a = *reinterpret_cast<const etl_numeric_hdr*>(pa), b = *reinterpret_cast<const etl_numeric_hdr*>(pb);
      if (a.kind != b.kind) return false;
      if (a.kind != 0) return true;
      return a.sign == b.sign && a.weight == b.weight && a.scale == b.scale &&
             bytes_eq_warp(pa + sizeof(etl_numeric_hdr), pb + sizeof(etl_numeric_hdr), 2 * xa);
    }
    default: return true;
  }
}
__device__ __forceinline__ const uint8_t* scalar_payload(const BqParams& P, uint32_t tag, uint64_t val) {
  return tag == ETL_CELL_STRING || tag == ETL_CELL_JSON ? cell_text(P.stream, P.heap, val) : P.heap + val;
}
// cells a (old image) and b (new image) of column c; ja / jb: the canonical records of their Json items
__device__ bool cells_eq_warp(const BqParams& P, uint64_t a, uint64_t b, const uint8_t* ja, const uint8_t* jb) {
  const uint32_t ta = P.cell_tag[a], tb = P.cell_tag[b];
  if (ta != tb) return false;
  if (ta == ETL_CELL_NULL) return true;
  const uint64_t va = P.cell_val[a], vb = P.cell_val[b];
  const uint32_t xa = P.cell_aux[a], xb = P.cell_aux[b];
  if (ta == ETL_CELL_JSON) return value_eq_warp(ta, 0, rd32(ja), ja + 4, 0, rd32(jb), jb + 4);
  if (ta != ETL_CELL_ARRAY) return value_eq_warp(ta, va, xa, scalar_payload(P, ta, va), vb, xb, scalar_payload(P, tb, vb));
  if (xa != xb) return false;
  const etl_array_elem* A = array_elems(P.heap, va);
  const etl_array_elem* B = array_elems(P.heap, vb);
  for (uint32_t k = 0; k < xa; k++) {
    const etl_array_elem ea = A[k], eb = B[k];
    if (ea.tag != eb.tag) return false;
    if (ea.tag == ETL_CELL_NULL) continue;
    bool eq;
    if (ea.tag == ETL_CELL_JSON) {
      eq = value_eq_warp(ea.tag, 0, rd32(ja), ja + 4, 0, rd32(jb), jb + 4);
      ja += 4 + ea.aux;
      jb += 4 + eb.aux;
    } else eq = value_eq_warp(ea.tag, ea.val, ea.aux, P.heap + ea.val, eb.val, eb.aux, P.heap + eb.val);
    if (!eq) return false;
  }
  return true;
}

// warp per selected record: 2 rows for an Update whose primary key changed (bigquery_primary_key_changed), else 1
__global__ void __launch_bounds__(256) k_bq_expand(BqParams P) {
  const uint64_t s = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s >= P.n_sel) return;                             // whole warps
  const uint64_t r = P.sel_rec[s];
  bool changed = false;
  if (P.rec_kind[r] == 'U' && (P.rec_flags[r] & (ETL_RF_OLD_FULL | ETL_RF_OLD_KEY))) {
    for (uint32_t q = 0; q < P.n_pk && !changed; q++) {
      const uint32_t c = P.pk_col[q];
      uint64_t a = 0, b = 0;
      image_cell(P, s, 1, c, &a);
      image_cell(P, s, 0, c, &b);
      const int16_t j = P.cols[c].json;
      changed = !cells_eq_warp(P, a, b, j >= 0 ? canon_of(P, s, j, 1) : nullptr, j >= 0 ? canon_of(P, s, j, 0) : nullptr);
    }
  }
  if ((threadIdx.x & 31) == 0) P.sel_cnt[s] = changed ? 2u : 1u;
}
// thread per selected record: its rows' descriptors and records (COPY: sel_row0 NULL, row s is record s)
__global__ void __launch_bounds__(256) k_bq_rows(BqParams P) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= P.n_sel) return;
  const uint64_t r = P.sel_rec[s];
  if (!P.sel_row0) { P.row_desc[s] = s << 2; P.row_rec[s] = r; return; }
  const uint64_t at = P.sel_row0[s];
  if (P.sel_cnt[s] == 2u) {                              // DELETE of the old key (ordinal 0), UPSERT (ordinal 1)
    P.row_desc[at] = s << 2 | 1u; P.row_rec[at] = r;
    P.row_desc[at + 1] = s << 2 | 2u; P.row_rec[at + 1] = r;
  } else {
    P.row_desc[at] = s << 2 | (P.rec_kind[r] == 'D' ? 1u : 0u);
    P.row_rec[at] = r;
  }
}

// ---------------------------------------------------------------- size, write
__device__ __forceinline__ bool packed_kind(uint32_t tag) {
  return tag == ETL_CELL_BOOL || tag == ETL_CELL_I16 || tag == ETL_CELL_I32 || tag == ETL_CELL_U32 || tag == ETL_CELL_I64 ||
         tag == ETL_CELL_F32 || tag == ETL_CELL_F64;
}
// a packed element / scalar numeric value without its key: its bytes (varints of the sign-extended value, IEEE bits)
__device__ __forceinline__ uint32_t num_len(uint32_t tag, uint64_t val) {
  if (tag == ETL_CELL_BOOL) return 1;
  if (tag == ETL_CELL_F32) return 4;
  if (tag == ETL_CELL_F64) return 8;
  return etl_rb::varint_len(tag == ETL_CELL_U32 ? (val & 0xffffffffull) : val);
}
__device__ __forceinline__ uint32_t num_write(uint32_t tag, uint64_t val, uint8_t* o) {
  if (tag == ETL_CELL_BOOL) { *o = (uint8_t)(val & 1u); return 1; }
  if (tag == ETL_CELL_F32) { etl_rb::le_write(val, 4, o); return 4; }
  if (tag == ETL_CELL_F64) { etl_rb::le_write(val, 8, o); return 8; }
  return etl_rb::varint_write(tag == ETL_CELL_U32 ? (val & 0xffffffffull) : val, o);
}
// the UTF-8 text of a text-kind value (String, Numeric, Json, Date, Time, Timestamp, TimestampTz, Uuid) or the bytes
// of a Bytes value: its length.  `n` is the length of String / Json (canonical) / Bytes payloads
__device__ __forceinline__ uint32_t text_len(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, uint32_t n) {
  switch (tag) {
    case ETL_CELL_NUMERIC: return etl_fmt::numeric_len(heap + val, aux);
    case ETL_CELL_DATE: return etl_bq::date_len((int64_t)val);
    case ETL_CELL_TIME: return etl_rb::time_len(aux);
    case ETL_CELL_TIMESTAMP: return etl_bq::timestamp_len((int64_t)val, aux, false);
    case ETL_CELL_TIMESTAMPTZ: return etl_bq::timestamp_len((int64_t)val, aux, true);
    case ETL_CELL_UUID: return etl_bq::kUuidLen;
    default: return n;
  }
}
__device__ __forceinline__ void text_write(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, const uint8_t* src, uint32_t n, uint8_t* o) {
  switch (tag) {
    case ETL_CELL_NUMERIC: etl_fmt::numeric_write(heap + val, aux, o); return;
    case ETL_CELL_DATE: etl_bq::date_write((int64_t)val, o); return;
    case ETL_CELL_TIME: etl_rb::time_write(val, aux, o); return;
    case ETL_CELL_TIMESTAMP: etl_bq::timestamp_write((int64_t)val, aux, false, o); return;
    case ETL_CELL_TIMESTAMPTZ: etl_bq::timestamp_write((int64_t)val, aux, true, o); return;
    case ETL_CELL_UUID: etl_bq::uuid_text_write(heap + val, o); return;
    default: for (uint32_t k = 0; k < n; k++) o[k] = src[k];
  }
}

// an array cell: packed (one key, the payload length, the elements) or one field per element; an empty array writes
// nothing, a NULL element writes nothing (the cell is reported).  Sizing when o == NULL; *issue = the cell has a NULL
// element or an element that fails a check
__device__ uint64_t array_field(const BqParams& P, uint32_t field, uint64_t val, uint32_t aux, const uint8_t* canon, uint8_t* o, bool* issue) {
  if (aux == 0) return 0;
  const etl_array_elem* E = array_elems(P.heap, val);
  const uint32_t ek = reinterpret_cast<const etl_array_hdr*>(P.heap + val)->elem_kind;
  const bool packed = ek == ETL_K_BOOL || ek == ETL_K_I16 || ek == ETL_K_I32 || ek == ETL_K_U32 || ek == ETL_K_I64 ||
                      ek == ETL_K_F32 || ek == ETL_K_F64;
  if (packed) {
    uint64_t pay = 0;
    for (uint32_t k = 0; k < aux; k++) {
      if (E[k].tag == ETL_CELL_NULL) { *issue = true; continue; }
      pay += num_len(E[k].tag, E[k].val);
    }
    if (!o) return etl_bq::key_len(field) + etl_rb::varint_len(pay) + pay;
    uint64_t at = etl_bq::key_write(field, etl_bq::kWtLen, o);
    at += etl_rb::varint_write(pay, o + at);
    for (uint32_t k = 0; k < aux; k++) if (E[k].tag != ETL_CELL_NULL) at += num_write(E[k].tag, E[k].val, o + at);
    return at;
  }
  uint64_t at = 0;
  const uint32_t kl = etl_bq::key_len(field);
  for (uint32_t k = 0; k < aux; k++) {
    const etl_array_elem e = E[k];
    if (e.tag == ETL_CELL_NULL) { *issue = true; continue; }
    const uint8_t* src = P.heap + e.val;
    uint32_t n = e.aux;
    if (e.tag == ETL_CELL_JSON) {
      n = rd32(canon); src = canon + 4; canon += 4 + e.aux;
      if (etl_bq::json_int_bad(src, n)) *issue = true;
    }
    if (e.tag == ETL_CELL_NUMERIC && etl_bq::numeric_scale_bad(P.heap + e.val, e.aux)) *issue = true;
    const uint32_t t = text_len(e.tag, e.val, e.aux, P.heap, n);
    if (o) {
      at += etl_bq::key_write(field, etl_bq::kWtLen, o + at);
      at += etl_rb::varint_write(t, o + at);
      text_write(e.tag, e.val, e.aux, P.heap, src, n, o + at);
    } else at += kl + etl_rb::varint_len(t);
    at += t;
  }
  return at;
}

// (row, field) → the cell behind a user column; false for a NULL-free absence (a DELETE row's non-key column)
__device__ __forceinline__ bool field_cell(const BqParams& P, uint64_t row, uint32_t c, uint64_t* s, uint32_t* img, uint64_t* cell) {
  const uint64_t d = P.row_desc[row];
  *s = d >> 2;
  *img = (uint32_t)(d & 1u);
  return image_cell(P, *s, *img, c, cell);
}

__global__ void __launch_bounds__(256) k_bq_size(BqParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long key = ~0ull;
  if (i < P.n_rows * P.w) {
    const uint64_t row = i / P.w;
    const uint32_t c = (uint32_t)(i - row * P.w);
    uint64_t len = 0;
    if (c == P.n_cols) len = etl_bq::key_len(c + 1) + 1 + kOpLen;
    else if (c > P.n_cols) len = P.rec_kind ? etl_bq::key_len(c + 1) + 1 + kSeqLen : 0;
    else {
      uint64_t s, cell;
      uint32_t img;
      if (field_cell(P, row, c, &s, &img, &cell)) {
        const uint32_t tag = P.cell_tag[cell];
        const uint64_t val = P.cell_val[cell];
        const uint32_t aux = P.cell_aux[cell];
        const int16_t j = P.cols[c].json;
        bool issue = false;
        if (tag == ETL_CELL_NULL) {
        } else if (tag == ETL_CELL_ARRAY) {
          len = array_field(P, c + 1, val, aux, j >= 0 ? canon_of(P, s, j, img) : nullptr, nullptr, &issue);
        } else if (packed_kind(tag)) {
          len = etl_bq::key_len(c + 1) + num_len(tag, val);
        } else {
          uint32_t n = aux;
          if (tag == ETL_CELL_JSON) {
            const uint8_t* t = canon_of(P, s, j, img);
            n = rd32(t);
            issue = etl_bq::json_int_bad(t + 4, n);
          }
          if (tag == ETL_CELL_NUMERIC) issue = etl_bq::numeric_scale_bad(P.heap + val, aux);
          const uint32_t t = text_len(tag, val, aux, P.heap, n);
          len = etl_bq::key_len(c + 1) + etl_rb::varint_len(t) + (uint64_t)t;
        }
        if (issue) key = row << 32 | c;
      }
    }
    P.cell_len[i] = len > 0xffffffffull ? 0xffffffffu : (uint32_t)len;
  }
  report_min(key, P.issues + kIssueKey);
}

__global__ void __launch_bounds__(256) k_bq_write(BqParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const uint8_t* lsrc = nullptr;
  uint8_t* ldst = nullptr;
  uint32_t ln = 0;
  if (i < P.n_rows * P.w) {
    const uint64_t row = i / P.w;
    const uint32_t c = (uint32_t)(i - row * P.w);
    uint8_t* o = P.out + P.row_off[row] + P.cell_len[i];
    const uint64_t d = P.row_desc[row];
    if (c == P.n_cols) {                                  // _CHANGE_TYPE
      o += etl_bq::key_write(c + 1, etl_bq::kWtLen, o);
      *o++ = (uint8_t)kOpLen;
      const char* op = d & 1u ? "DELETE" : "UPSERT";
      for (uint32_t k = 0; k < kOpLen; k++) o[k] = (uint8_t)op[k];
    } else if (c > P.n_cols) {                            // _CHANGE_SEQUENCE_NUMBER (none for COPY rows)
      if (P.rec_kind) {
        const uint64_t r = P.row_rec[row];
        o += etl_bq::key_write(c + 1, etl_bq::kWtLen, o);
        *o++ = (uint8_t)kSeqLen;
        etl_fmt::seq_key_write(P.rec_commit_lsn[r], P.rec_tx_ordinal[r], o);
        o[etl_fmt::kSeqKeyLen] = '/';
        etl_fmt::hex16_write((d >> 1) & 1u, o + etl_fmt::kSeqKeyLen + 1);
      }
    } else {
      uint64_t s, cell;
      uint32_t img;
      if (field_cell(P, row, c, &s, &img, &cell)) {
        const uint32_t tag = P.cell_tag[cell];
        const uint64_t val = P.cell_val[cell];
        const uint32_t aux = P.cell_aux[cell];
        const int16_t j = P.cols[c].json;
        bool issue = false;
        if (tag == ETL_CELL_NULL) {
        } else if (tag == ETL_CELL_ARRAY) {
          array_field(P, c + 1, val, aux, j >= 0 ? canon_of(P, s, j, img) : nullptr, o, &issue);
        } else if (packed_kind(tag)) {
          const uint32_t wt = tag == ETL_CELL_F32 ? etl_bq::kWtI32 : (tag == ETL_CELL_F64 ? etl_bq::kWtI64 : etl_bq::kWtVarint);
          o += etl_bq::key_write(c + 1, wt, o);
          num_write(tag, val, o);
        } else {
          uint32_t n = aux;
          const uint8_t* src = nullptr;
          if (tag == ETL_CELL_JSON) { const uint8_t* t = canon_of(P, s, j, img); n = rd32(t); src = t + 4; }
          else if (tag == ETL_CELL_STRING) src = cell_text(P.stream, P.heap, val);
          else if (tag == ETL_CELL_BYTES) src = P.heap + val;
          const uint32_t t = text_len(tag, val, aux, P.heap, n);
          o += etl_bq::key_write(c + 1, etl_bq::kWtLen, o);
          o += etl_rb::varint_write(t, o);
          if (src && n > kLongCell) { ldst = o; lsrc = src; ln = n; }   // the warp copies it below
          else text_write(tag, val, aux, P.heap, src, n, o);
        }
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
    for (uint32_t k = lane; k < n; k += 32) d[k] = s[k];
  }
}

// the kind and element of the reported value issue: a NULL element first (the conversion), then the first element (or
// the scalar) that fails a check
__global__ void k_bq_issue(BqParams P) {
  const unsigned long long key = P.issues[kIssueKey];
  if (key == ~0ull) return;
  const uint64_t row = key >> 32;
  const uint32_t c = (uint32_t)(key & 0xffffffffu);
  uint64_t s, cell;
  uint32_t img;
  if (!field_cell(P, row, c, &s, &img, &cell)) return;
  const uint32_t tag = P.cell_tag[cell], aux = P.cell_aux[cell];
  const int16_t j = P.cols[c].json;
  if (tag == ETL_CELL_NUMERIC) { P.issues[kIssueKind] = ETL_BQ_ISSUE_NUMERIC_SCALE; return; }
  if (tag == ETL_CELL_JSON) { P.issues[kIssueKind] = ETL_BQ_ISSUE_JSON_INTEGER; return; }
  if (tag != ETL_CELL_ARRAY) return;
  const etl_array_elem* E = array_elems(P.heap, P.cell_val[cell]);
  for (uint32_t k = 0; k < aux; k++)
    if (E[k].tag == ETL_CELL_NULL) { P.issues[kIssueKind] = ETL_BQ_ISSUE_ARRAY_NULL; P.issues[kIssueElem] = k; return; }
  const uint8_t* canon = j >= 0 ? canon_of(P, s, j, img) : nullptr;
  for (uint32_t k = 0; k < aux; k++) {
    if (E[k].tag == ETL_CELL_NUMERIC && etl_bq::numeric_scale_bad(P.heap + E[k].val, E[k].aux)) {
      P.issues[kIssueKind] = ETL_BQ_ISSUE_NUMERIC_SCALE; P.issues[kIssueElem] = k; return;
    }
    if (E[k].tag == ETL_CELL_JSON) {
      const bool bad = etl_bq::json_int_bad(canon + 4, rd32(canon));
      canon += 4 + E[k].aux;
      if (bad) { P.issues[kIssueKind] = ETL_BQ_ISSUE_JSON_INTEGER; P.issues[kIssueElem] = k; return; }
    }
  }
}

}  // namespace

struct etl_bigquery_batch : RowPayload {
  etl_bigquery_issues issues{};
};

extern "C" {

int etl_dec_bigquery_emit(const etl_dec_batch* batch, uint32_t schema_index, int to_host, etl_bigquery_batch** out) {
  if (!batch || !out) return ETL_ERR_INVALID_ARG;
  EmitBatch E;
  if (open_emit_batch(batch, schema_index, &E) != ETL_OK) return ETL_ERR_INVALID_ARG;
  const etl_dec_planes& P = E.P;
  const etl_dec_schema_info& sc = E.sc;
  const bool copy = E.copy;
  const uint8_t* pk = nullptr;
  if (!copy && !etl_schema_pk_columns(batch, schema_index, &pk)) return ETL_ERR_INVALID_ARG;
  const uint32_t W = sc.n_cols + 2;
  // column descriptors: primary-key membership and key slot, the Json item index; identity_matches_primary_key
  std::vector<BqCol> cols(sc.n_cols);
  std::vector<uint32_t> json_col, pk_col;
  bool identity_is_pk = true;
  for (uint32_t c = 0; c < sc.n_cols; c++) {
    BqCol& d = cols[c];
    d.kind = sc.col_kind[c];
    d.json = -1;
    d.pk = pk && pk[c] ? 1 : 0;
    if (d.pk) { d.key_slot = (uint16_t)pk_col.size(); pk_col.push_back(c); }
    if (!copy && ((sc.col_flags[c] & 2u) != 0) != (d.pk != 0)) identity_is_pk = false;
    if ((d.kind & ~(uint32_t)ETL_K_ARRAY) == ETL_K_JSON) { d.json = (int16_t)json_col.size(); json_col.push_back(c); }
  }

  cudaStream_t st = cudaStreamPerThread;
  etl_bigquery_batch* B = new etl_bigquery_batch();
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
  unsigned long long* d_n = (unsigned long long*)scratch(8 * (2 + kIssueSlots));   // records, first invalid | issues
  const size_t cols_bytes = (sizeof(BqCol) * cols.size() + 7) & ~(size_t)7;
  uint8_t* d_cols = (uint8_t*)scratch(cols_bytes + 4ull * (json_col.size() + pk_col.size()));
  if (!d_blk || !d_cell0 || !d_rec || !d_n || !d_cols) return fail(ETL_ERR_ALLOC);
  unsigned long long* d_issues = d_n + 2;
  uint32_t* d_json_col = reinterpret_cast<uint32_t*>(d_cols + cols_bytes);
  uint32_t* d_pk_col = d_json_col + json_col.size();
  if (cudaMemsetAsync(d_n, 0xff, 8 * (2 + kIssueSlots), st) != cudaSuccess ||
      cudaMemsetAsync(d_issues + kIssueFlags, 0, 16, st) != cudaSuccess ||   // flags, kind
      (!cols.empty() && cudaMemcpyAsync(d_cols, cols.data(), sizeof(BqCol) * cols.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
      (!json_col.empty() && cudaMemcpyAsync(d_json_col, json_col.data(), 4 * json_col.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
      (!pk_col.empty() && cudaMemcpyAsync(d_pk_col, pk_col.data(), 4 * pk_col.size(), cudaMemcpyHostToDevice, st) != cudaSuccess))
    return fail(ETL_ERR_CUDA);
  unsigned long long sel[2] = {0, UINT64_MAX};          // selected records, first invalid record
  const SelParams Sp{P.rec_kind, P.rec_flags, P.rec_schema, P.rec_cell_base, n_valid, (int32_t)schema_index, identity_is_pk ? 1u : 0u,
                     sc.n_cols, d_blk, d_cell0, d_rec, d_n};
  if (select_rows<BigQueryRecords>(Sp, copy, n_valid, st, sel) != ETL_OK) return fail(ETL_ERR_CUDA);
  const uint64_t n_sel = sel[0];
  B->issues.first_invalid_record = sel[1];

  BqParams R{P.cell_tag, P.cell_val, P.cell_aux, P.heap, E.stream, P.rec_kind, P.rec_flags, P.rec_commit_lsn, P.rec_tx_ordinal,
             P.rec_cell_base, d_cell0, d_rec, n_sel, reinterpret_cast<const BqCol*>(d_cols), d_json_col, d_pk_col,
             sc.n_cols, W, (uint32_t)json_col.size(), (uint32_t)pk_col.size(), nullptr, nullptr, nullptr, nullptr,
             nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, d_issues};
  // Json: input lengths → item offsets → (sync) canonical text
  const uint64_t n_items = n_sel * 2 * R.n_json;
  if (n_items) {
    JsonStage J{P.cell_tag, P.cell_val, P.cell_aux, P.heap, E.stream, n_items, nullptr, nullptr, nullptr,
                d_issues + kIssueFlags, (unsigned long long)kFlagBadJson};
    if (int rc = stage_json(scratch, J, BqJsonCells{R}, st)) return fail(rc);
    R.json_off = J.off;
    R.canon = J.canon;
  }
  // rows: 1 or 2 per record, scanned (sync); COPY: one per record
  uint64_t n_rows = n_sel;
  if (n_sel && !copy) {
    const uint32_t sb = scan_blocks(n_sel);
    R.sel_cnt = (uint32_t*)scratch(n_sel * 4);
    uint64_t* row0 = (uint64_t*)scratch((n_sel + 1) * 8);
    unsigned long long* sblk = (unsigned long long*)scratch((sb + 1) * 8ull);
    if (!R.sel_cnt || !row0 || !sblk) return fail(ETL_ERR_ALLOC);
    k_bq_expand<<<(uint32_t)((n_sel * 32 + 255) / 256), 256, 0, st>>>(R);
    scan_lengths(R.sel_cnt, n_sel, sblk, sblk + sb, row0, st);
    unsigned long long nr = 0;
    if (cudaMemcpyAsync(&nr, sblk + sb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    n_rows = nr;
    R.sel_row0 = row0;
  }
  B->n_rows = n_rows;
  R.n_rows = n_rows;
  if (cudaMalloc(&B->meta, B->meta_bytes()) != cudaSuccess) { B->meta = nullptr; return fail(ETL_ERR_ALLOC); }
  if (cudaMemsetAsync(B->meta, 0, 8, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  R.row_off = reinterpret_cast<const uint64_t*>(B->meta);
  R.row_rec = reinterpret_cast<uint64_t*>(B->meta) + n_rows + 1;
  unsigned long long tot[2] = {0, 0};                   // output bytes, issue flags
  if (n_rows) {
    R.row_desc = (uint64_t*)scratch(n_rows * 8);
    const uint64_t n_cells = n_rows * W;
    const uint32_t rb = scan_blocks(n_rows);
    R.cell_len = (uint32_t*)scratch(n_cells * 4);
    R.row_len = (uint32_t*)scratch(n_rows * 4);
    unsigned long long* rblk = (unsigned long long*)scratch((rb + 1) * 8ull);
    if (!R.row_desc || !R.cell_len || !R.row_len || !rblk) return fail(ETL_ERR_ALLOC);
    k_bq_rows<<<(uint32_t)((n_sel + 255) / 256), 256, 0, st>>>(R);
    // sizes → in-row offsets → row offsets (sync)
    k_bq_size<<<(uint32_t)((n_cells + 255) / 256), 256, 0, st>>>(R);
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
    k_bq_write<<<(uint32_t)((n_rows * W + 255) / 256), 256, 0, st>>>(R);
    k_bq_issue<<<1, 1, 0, st>>>(R);
  }
  if (to_host) {
    if (int rc = B->copy_to_host(st)) return fail(rc);
  }
  unsigned long long iss[kIssueSlots];
  if (cudaMemcpyAsync(iss, d_issues, sizeof iss, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  scratch.release();
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ETL_ERR_CUDA);
  etl_bq_issue v{UINT64_MAX, UINT32_MAX, UINT32_MAX, 0, 0};
  if (iss[kIssueKey] != ~0ull) {
    v.row = iss[kIssueKey] >> 32;
    v.column = (uint32_t)(iss[kIssueKey] & 0xffffffffu);
    v.element = (uint32_t)iss[kIssueElem];
    v.kind = (uint32_t)iss[kIssueKind];
  }
  B->issues.value = v;
  *out = B;
  return ETL_OK;
}
uint64_t etl_dec_bigquery_rows(const etl_bigquery_batch* b) { return RowPayload::rows_of(b); }
uint64_t etl_dec_bigquery_bytes(const etl_bigquery_batch* b) { return RowPayload::bytes_of(b); }
const uint8_t* etl_dec_bigquery_data(const etl_bigquery_batch* b, int host) { return RowPayload::data_of(b, host); }
const uint64_t* etl_dec_bigquery_row_offsets(const etl_bigquery_batch* b, int host) { return RowPayload::offsets_of(b, host); }
const uint64_t* etl_dec_bigquery_row_records(const etl_bigquery_batch* b, int host) { return RowPayload::records_of(b, host); }
int etl_dec_bigquery_issues(const etl_bigquery_batch* b, etl_bigquery_issues* out) {
  if (!b || !out) return ETL_ERR_INVALID_ARG;
  *out = b->issues;
  return ETL_OK;
}
void etl_dec_bigquery_free(etl_bigquery_batch* b) { delete b; }

}  // extern "C"
