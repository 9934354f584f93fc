// ducklake_emit.cu — DuckLake emitter: the row mutations of ONE replicated-schema version of a decoded batch, with the
// SQL-literal texts the DuckLake destination builds for them, and the fingerprints of its retry-safe batch identity.
//
// Replaces the host work of crates/etl-destinations/src/ducklake: write_events_inner accumulating TableMutations
// (core.rs:715-836, key_row_from_updated_partial_row :266-359, validate_ducklake_replica_identity :237-258), the
// SQL literals of cell_to_sql_literal_ref / table_row_to_sql_literal_ref (encoding.rs:28-272) behind
// delete_predicate_from_row (batches.rs:1099-1186), update_assignments_from_partial_row (:1189-1269),
// delete_predicate_from_copy_row (:1338-1371) and prepare_rows (encoding.rs:13-26), and the FNV-1a batch identity
// (build_mutation_batch_identity :1272-1316, build_copy_batch_identity :1319-1336, hash_table_row_ref :1418-1456) over
// the CDC_MUTATION_BATCH_SIZE chunks of prepare_mutation_table_batches (:594-622) after
// retain_mutations_after_sequence_key (:806-820).
//
// Passes of etl_dec_ducklake_emit (one CUDA stream, three syncs: mutation count, Json sizes when a Json column exists,
// text sizes):
//   1. k_dl_trunc + scan (emit_scan.cuh): the truncate-free segment of each record.  COPY: none.
//   2. k_dl_decide (warp per record): the mutation kind, the reject reason, empty partial rows, MF_ARRAY, and the
//      segment flags behind mixed_versions; the mutations are scanned into place (scan_lengths) and k_dl_scatter writes
//      their records, kinds, segments and LSNs.
//   3. Json (stage_json, row_emit_common.cuh): items (mutation, Json column, image), canonicalised once.
//   4. k_dl_size: thread per (text, mutation, column + 1) over the three texts: the piece's bytes (separator, name,
//      literal); a String / Json value above kLongCell bytes has its quotes counted by the warp.  k_row_scan
//      (row_emit_common.cuh) turns them into in-text offsets and text lengths, scanned into u64 text offsets.
//   5. k_dl_write: thread per (text, mutation, column + 1); String / Json / Bytes values above kLongCell bytes are
//      quoted or hex-encoded by the whole warp.
// etl_dec_ducklake_sub_batches (one sync, the chunk count): k_dl_first_kept, k_dl_chunk_mark + scan, k_dl_chunk_fill,
// k_dl_fingerprint (thread per chunk of up to 16 mutations, one serial FNV chain reading the texts with 8-byte loads).
// Scratch: 4 B per (text, mutation, column + 1) + 4 B per mutation + 29 B per record of the batch (truncate flags 4 B,
// segment offsets 8 B, mutation flag, kind and segment flags 9 B, mutation offsets 8 B), plus the scan blocks; with
// Json columns 12 B per (mutation, Json column, image) + 17 B per input Json byte.  Scratch is stream-ordered (cudaMallocAsync), the output
// is not.  Output: 41 B per mutation + 24 B of text offsets per mutation + the texts, and 4 B per (mutation, column + 1)
// when a partial update is among the mutations (the assignment pieces the fingerprint walks).
// ptxas (-Xptxas -v, sm_90a): k_dl_decide 28 registers, k_dl_size 40, k_dl_write 48, k_dl_fingerprint 32, k_dl_scatter 22,
// k_dl_chunk_mark 21, k_dl_chunk_fill 19, k_dl_trunc 14, k_dl_first_kept 10, k_dl_mixed 8, k_json_canon 56 (16 B spills, as
// in the other emitters), k_json_len 22, k_row_scan 24; no other spills and no stack frames.
#include <cuda_runtime.h>

#include <cstring>
#include <vector>

#include "etl_decode.h"
#include "arrow_format.cuh"
#include "rowbinary_format.cuh"
#include "bigquery_format.cuh"
#include "ducklake_format.cuh"
#include "batch_internal.h"
#include "emit_scan.cuh"
#include "row_emit_common.cuh"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr uint32_t kLongCell = 64;   // payload bytes above which a String / Json / Bytes value is handled by the warp
constexpr uint32_t kChunk = 16;      // CDC_MUTATION_BATCH_SIZE (batches.rs)
enum { kIssueReject = 0, kIssueEmpty = 1, kIssueFlags = 2, kIssueSlots = 3 };
enum { kFlagBadJson = 1, kFlagTextTooLong = 2, kFlagMixed = 4, kFlagPartial = 8 };
enum { kDeferNone = 0, kDeferString = 1, kDeferJson = 2, kDeferBytes = 3 };

struct DlCol {
  uint8_t kind;       // ETL_K_*
  uint8_t _pad;
  int16_t pred;       // index among the predicate columns (identity; COPY: primary key), -1 otherwise
  int16_t json;       // index among the columns whose cells can hold Json text (Json, Json[]); -1 otherwise
  uint16_t _pad2;
  uint32_t name_off, name_len;   // the quoted name in `names`
};

struct DlParams {
  const uint8_t* cell_tag; const uint64_t* cell_val; const uint32_t* cell_aux; const uint8_t* heap; const uint8_t* stream;
  const uint8_t* rec_kind; const uint8_t* rec_flags; const int32_t* rec_schema; const uint32_t* rec_rel;
  const uint64_t* rec_cell_base; const uint64_t* rec_start_lsn; const uint64_t* rec_commit_lsn; const uint64_t* rec_tx_ordinal;
  uint64_t n_valid;
  int32_t schema; uint32_t table_id, n_cols, n_pred;
  bool copy;
  const DlCol* cols; const uint8_t* names; const uint32_t* json_col; uint32_t n_json;
  const uint64_t* seg_off;      // per record: Truncate events before it (NULL: COPY, one segment)
  uint32_t* seg_flags;          // per segment: 1 this version's DML, 2 the table's DML under another version
  uint32_t* rec_mut; uint8_t* rec_mkind; const uint64_t* mut_pos;
  unsigned long long* issues;
  // per mutation
  uint64_t* mut_rec; uint64_t* mut_start; uint64_t* mut_commit; uint64_t* mut_tx; uint64_t* mut_seg; uint8_t* mut_kind;
  uint64_t n_mut;
  const uint64_t* json_off; const uint8_t* canon;   // item (m, j, img) = (m * n_json + j) * 2 + img; img 0 new, 1 old
  uint32_t w;                                       // pieces per text: n_cols + 1
  uint32_t* cell_len;                               // [text][mutation][piece]
  const uint64_t* text_off[3]; uint8_t* out[3];
};

// ---------------------------------------------------------------- images
__device__ __forceinline__ bool has_old(const DlParams& P, uint64_t r) {
  return !P.copy && (P.rec_flags[r] & (ETL_RF_OLD_FULL | ETL_RF_OLD_KEY));
}
__device__ __forceinline__ uint64_t new_cell(const DlParams& P, uint64_t r, uint32_t c) {
  if (P.copy) return r * P.n_cols + c;
  return P.rec_kind[r] == 'U' && has_old(P, r) ? P.rec_cell_base[r + 1] - P.n_cols + c : P.rec_cell_base[r] + c;
}
// the old image's cell of column c: Full → the column's cell, Key → the key cell of a predicate column
__device__ __forceinline__ bool old_cell(const DlParams& P, uint64_t r, uint32_t c, uint64_t* cell) {
  if (!has_old(P, r)) return false;
  const uint64_t c0 = P.rec_cell_base[r];
  if (P.rec_flags[r] & ETL_RF_OLD_FULL) { *cell = c0 + c; return true; }
  if (P.cols[c].pred < 0) return false;
  *cell = c0 + (uint32_t)P.cols[c].pred;
  return true;
}
__device__ __forceinline__ bool has_row(uint32_t kind) { return kind == ETL_DL_INSERT || kind == ETL_DL_UPDATE || kind == ETL_DL_REPLACE; }
__device__ __forceinline__ const uint8_t* canon_of(const DlParams& P, uint64_t m, uint32_t c, uint32_t img) {
  const int16_t j = P.cols[c].json;
  return j < 0 ? nullptr : P.canon + P.json_off[((uint64_t)m * P.n_json + (uint32_t)j) * 2 + img];
}

struct DlJsonCells {
  DlParams P;
  __device__ __forceinline__ bool operator()(uint64_t i, uint64_t* cell) const {
    const uint64_t m = i / (2ull * P.n_json);
    const uint32_t rem = (uint32_t)(i - m * 2ull * P.n_json);
    const uint32_t c = P.json_col[rem >> 1];
    const uint64_t r = P.mut_rec[m];
    if (rem & 1u) return old_cell(P, r, c, cell);
    if ((P.mut_kind[m] & 0x7fu) == ETL_DL_DELETE) return false;
    *cell = new_cell(P, r, c);
    return true;
  }
};

// ---------------------------------------------------------------- mutations
__global__ void __launch_bounds__(256) k_dl_trunc(DlParams P, uint32_t* tr) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < P.n_valid) tr[r] = P.rec_kind[r] == ETL_REC_TRUNCATE && (P.rec_flags[r] & ETL_RF_EVENT) ? 1u : 0u;
}

// warp per record: write_events_inner's verdict (core.rs:737-830)
__global__ void __launch_bounds__(256) k_dl_decide(DlParams P) {
  const uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (r >= P.n_valid) return;                             // whole warps
  uint32_t kind = 0, reject = 0, seg_bits = 0;
  bool empty = false;
  if (P.copy) kind = ETL_DL_INSERT;
  else {
    const uint32_t k = P.rec_kind[r], f = P.rec_flags[r];
    const bool dml = (f & ETL_RF_EVENT) && (k == ETL_REC_INSERT || k == ETL_REC_UPDATE || k == ETL_REC_DELETE);
    if (dml && P.rec_schema[r] != P.schema && P.rec_rel[r] == P.table_id) seg_bits = 2;
    if (dml && P.rec_schema[r] == P.schema) {
      seg_bits = 1;
      const bool old = has_old(P, r);
      if (k == ETL_REC_INSERT) kind = ETL_DL_INSERT;
      else if (P.n_pred == 0) reject = k == ETL_REC_UPDATE ? ETL_DL_REJECT_UPDATE_NO_IDENTITY : ETL_DL_REJECT_DELETE_NO_IDENTITY;
      else if (k == ETL_REC_DELETE) { if (old) kind = ETL_DL_DELETE; else reject = ETL_DL_REJECT_DELETE_NO_OLD_ROW; }
      else if (!(f & ETL_RF_NEW_PARTIAL)) kind = old ? ETL_DL_UPDATE : ETL_DL_REPLACE;
      else {
        bool present = false, key_missing = false;
        for (uint32_t base = 0; base < P.n_cols; base += 32) {
          const uint32_t c = base + lane;
          const bool miss = c < P.n_cols && P.cell_tag[new_cell(P, r, c)] == ETL_CELL_MISSING;
          present = present || __any_sync(kFull, c < P.n_cols && !miss);
          key_missing = key_missing || __any_sync(kFull, miss && P.cols[c].pred >= 0);
        }
        if (!old && key_missing) reject = ETL_DL_REJECT_PARTIAL_KEY_MISSING;
        else { kind = ETL_DL_UPDATE_PARTIAL; empty = !present; }
      }
    }
  }
  bool array = false;
  if (has_row(kind))
    for (uint32_t base = 0; base < P.n_cols; base += 32) {
      const uint32_t c = base + lane;
      array = array || __any_sync(kFull, c < P.n_cols && P.cell_tag[new_cell(P, r, c)] == ETL_CELL_ARRAY);
    }
  if (lane) return;
  P.rec_mut[r] = kind ? 1u : 0u;
  P.rec_mkind[r] = (uint8_t)(kind | (array ? (uint32_t)ETL_DL_MF_ARRAY : 0u));
  if (reject) atomicMin(P.issues + kIssueReject, (unsigned long long)(r << 3 | reject));
  if (empty) atomicMin(P.issues + kIssueEmpty, (unsigned long long)r);
  if (kind == ETL_DL_UPDATE_PARTIAL) atomicOr(P.issues + kIssueFlags, (unsigned long long)kFlagPartial);
  if (seg_bits) atomicOr(P.seg_flags + P.seg_off[r], seg_bits);
}
__global__ void __launch_bounds__(256) k_dl_scatter(DlParams P) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P.n_valid || !P.rec_mut[r]) return;
  const uint64_t m = P.mut_pos[r];
  P.mut_rec[m] = r;
  P.mut_kind[m] = P.rec_mkind[r];
  P.mut_seg[m] = P.seg_off ? P.seg_off[r] : 0;
  P.mut_start[m] = P.copy ? 0 : P.rec_start_lsn[r];
  P.mut_commit[m] = P.copy ? 0 : P.rec_commit_lsn[r];
  P.mut_tx[m] = P.copy ? 0 : P.rec_tx_ordinal[r];
}
__global__ void __launch_bounds__(256) k_dl_mixed(const uint32_t* seg_flags, uint64_t n, unsigned long long* flags) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n && seg_flags[s] == 3u) atomicOr(flags, (unsigned long long)kFlagMixed);
}

// ---------------------------------------------------------------- literals
// one non-NULL, non-array value; src / n: the text of a String, the canonical text of a Json, the payload of a Bytes
__device__ uint64_t value_len(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, const uint8_t* src, uint32_t n) {
  bool bs;
  switch (tag) {
    case ETL_CELL_BOOL: return val ? 4u : 5u;
    case ETL_CELL_I16: case ETL_CELL_I32: case ETL_CELL_I64: return etl_dl::int_len((int64_t)val);
    case ETL_CELL_U32: return etl_dl::dec_len(val & 0xffffffffull);
    case ETL_CELL_F32: return etl_dl::float_lit_len(etl_dl::f32_bits_as_f64((uint32_t)val), false);
    case ETL_CELL_F64: return etl_dl::float_lit_len(val, true);
    case ETL_CELL_NUMERIC: return 2u + etl_fmt::numeric_len(heap + val, aux);
    case ETL_CELL_DATE: return etl_dl::date_lit_len((int64_t)val);
    case ETL_CELL_TIME: return etl_dl::kTimeLitLen;
    case ETL_CELL_TIMESTAMP: return etl_dl::ts_lit_len((int64_t)val, false);
    case ETL_CELL_TIMESTAMPTZ: return etl_dl::ts_lit_len((int64_t)val, true);
    case ETL_CELL_UUID: return etl_dl::kUuidLitLen;
    case ETL_CELL_STRING: return etl_dl::quote_len(src, n, &bs);
    case ETL_CELL_JSON: return 14u + etl_dl::quote_len(src, n, &bs);
    case ETL_CELL_BYTES: return etl_dl::bytes_lit_len(n);
    default: return 4u;                                   // NULL
  }
}
__device__ uint32_t value_write(uint32_t tag, uint64_t val, uint32_t aux, const uint8_t* heap, const uint8_t* src, uint32_t n, uint8_t* o) {
  uint32_t at = 0;
  switch (tag) {
    case ETL_CELL_BOOL: return etl_dl::cstr_write(val ? "TRUE" : "FALSE", o);
    case ETL_CELL_I16: case ETL_CELL_I32: case ETL_CELL_I64: return etl_dl::int_write((int64_t)val, o);
    case ETL_CELL_U32: { const uint32_t d = etl_dl::dec_len(val & 0xffffffffull); etl_dl::dec_write(val & 0xffffffffull, d, o); return d; }
    case ETL_CELL_F32: return etl_dl::float_lit_write(etl_dl::f32_bits_as_f64((uint32_t)val), false, o);
    case ETL_CELL_F64: return etl_dl::float_lit_write(val, true, o);
    case ETL_CELL_NUMERIC:
      o[0] = '\'';
      at = 1u + etl_fmt::numeric_write(heap + val, aux, o + 1);
      o[at] = '\'';
      return at + 1u;
    case ETL_CELL_DATE: return etl_dl::date_lit_write((int64_t)val, o);
    case ETL_CELL_TIME: return etl_dl::time_lit_write(val, aux, o);
    case ETL_CELL_TIMESTAMP: return etl_dl::ts_lit_write((int64_t)val, aux, false, o);
    case ETL_CELL_TIMESTAMPTZ: return etl_dl::ts_lit_write((int64_t)val, aux, true, o);
    case ETL_CELL_UUID: return etl_dl::uuid_lit_write(heap + val, o);
    case ETL_CELL_STRING: return etl_dl::quote_write(src, n, o);
    case ETL_CELL_JSON:
      at = etl_dl::cstr_write("CAST(", o);
      at += etl_dl::quote_write(src, n, o + at);
      return at + etl_dl::cstr_write(" AS JSON)", o + at);
    case ETL_CELL_BYTES: return etl_dl::bytes_lit_write(src, n, o);
    default: return etl_dl::cstr_write("NULL", o);
  }
}
// "[" elements joined by ", " "]", NULL for a NULL element; canon: the cell's Json item record.  Sizing when o == NULL
__device__ uint64_t array_lit(const DlParams& P, uint64_t val, uint32_t aux, const uint8_t* canon, uint8_t* o) {
  const etl_array_elem* E = array_elems(P.heap, val);
  uint64_t at = 1;
  if (o) o[0] = '[';
  for (uint32_t k = 0; k < aux; k++) {
    const etl_array_elem e = E[k];
    if (k) { if (o) { o[at] = ','; o[at + 1] = ' '; } at += 2; }
    const uint8_t* src = P.heap + e.val;
    uint32_t n = e.aux;
    if (e.tag == ETL_CELL_JSON) { n = rd32(canon); src = canon + 4; canon += 4 + e.aux; }
    at += o ? value_write(e.tag, e.val, e.aux, P.heap, src, n, o + at) : value_len(e.tag, e.val, e.aux, P.heap, src, n);
  }
  if (o) o[at] = ']';
  return at + 1;
}

struct Defer { const uint8_t* src; uint8_t* dst; uint32_t n; uint32_t mode; };

// the literal of a cell; sizing when o == NULL.  A String / Json / Bytes value above kLongCell bytes is left to the
// warp (*d, returns 0): it is always the last part of its piece
__device__ uint64_t cell_lit(const DlParams& P, uint64_t cell, const uint8_t* canon, uint8_t* o, Defer* d) {
  const uint32_t tag = P.cell_tag[cell], aux = P.cell_aux[cell];
  const uint64_t val = P.cell_val[cell];
  if (tag == ETL_CELL_ARRAY) return array_lit(P, val, aux, canon, o);
  const uint8_t* src = nullptr;
  uint32_t n = aux;
  if (tag == ETL_CELL_JSON) { n = rd32(canon); src = canon + 4; }
  else if (tag == ETL_CELL_STRING) src = cell_text(P.stream, P.heap, val);
  else if (tag == ETL_CELL_BYTES) src = P.heap + val;
  if (src && n > kLongCell) {
    *d = Defer{src, o, n, tag == ETL_CELL_STRING ? (uint32_t)kDeferString : (tag == ETL_CELL_JSON ? (uint32_t)kDeferJson : (uint32_t)kDeferBytes)};
    return 0;
  }
  return o ? value_write(tag, val, aux, P.heap, src, n, o) : value_len(tag, val, aux, P.heap, src, n);
}

// piece c of text t of mutation m (pieces 0 .. n_cols - 1 are columns, piece n_cols the row's closing parenthesis);
// sizing when o == NULL
__device__ uint64_t piece(const DlParams& P, uint32_t t, uint64_t m, uint32_t c, uint8_t* o, Defer* d) {
  const uint64_t r = P.mut_rec[m];
  const uint32_t kind = P.mut_kind[m] & 0x7fu;
  uint64_t at = 0;
  auto put = [&](const char* s) { at += o ? etl_dl::cstr_write(s, o + at) : etl_dl::cstr_len(s); };
  auto name = [&]() {
    const DlCol& col = P.cols[c];
    if (o) for (uint32_t k = 0; k < col.name_len; k++) o[at + k] = P.names[col.name_off + k];
    at += col.name_len;
  };
  auto lit = [&](uint64_t cell, const uint8_t* canon) { at += cell_lit(P, cell, canon, o ? o + at : nullptr, d); };
  if (t == 0) {                                           // row: "(" v ", " v … ")"
    if (!has_row(kind)) return 0;
    if (c == P.n_cols) { put(P.n_cols ? ")" : "()"); return at; }
    put(c ? ", " : "(");
    lit(new_cell(P, r, c), canon_of(P, m, c, 0));
    return at;
  }
  if (c == P.n_cols) return 0;
  if (t == 1) {                                           // predicate: name = v | name IS NULL, joined by " AND "
    const int16_t slot = P.cols[c].pred;
    if (slot < 0 || (!P.copy && kind == ETL_DL_INSERT)) return 0;
    uint64_t cell = 0;
    uint32_t img = 1;
    if (!old_cell(P, r, c, &cell)) { cell = new_cell(P, r, c); img = 0; }   // REPLACE, partial without an old image, COPY
    if (slot) put(" AND ");
    name();
    if (P.cell_tag[cell] == ETL_CELL_NULL) { put(" IS NULL"); return at; }
    put(" = ");
    lit(cell, canon_of(P, m, c, img));
    return at;
  }
  if (kind != ETL_DL_UPDATE_PARTIAL) return 0;            // assignments: the present columns, name = v, joined by ", "
  const uint64_t cell = new_cell(P, r, c);
  if (P.cell_tag[cell] == ETL_CELL_MISSING) return 0;
  bool first = true;
  for (uint32_t k = 0; k < c && first; k++) first = P.cell_tag[new_cell(P, r, k)] == ETL_CELL_MISSING;
  if (!first) put(", ");
  name();
  put(" = ");
  lit(cell, canon_of(P, m, c, 0));
  return at;
}

__device__ __forceinline__ void item_of(const DlParams& P, uint64_t i, uint32_t* t, uint64_t* m, uint32_t* c) {
  const uint64_t per = P.n_mut * P.w;
  *t = (uint32_t)(i / per);
  const uint64_t rem = i - *t * per;
  *m = rem / P.w;
  *c = (uint32_t)(rem - *m * P.w);
}

__global__ void __launch_bounds__(256) k_dl_size(DlParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  Defer d{nullptr, nullptr, 0, kDeferNone};
  uint64_t len = 0;
  if (i < 3 * P.n_mut * P.w) {
    uint32_t t, c;
    uint64_t m;
    item_of(P, i, &t, &m, &c);
    len = piece(P, t, m, c, nullptr, &d);
  }
  // long values: quote_literal's length needs the quotes and backslashes counted
  unsigned todo = __ballot_sync(kFull, d.mode != kDeferNone);
  while (todo) {
    const int src_lane = __ffs(todo) - 1;
    todo &= todo - 1;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(kFull, reinterpret_cast<unsigned long long>(d.src), src_lane));
    const uint32_t n = __shfl_sync(kFull, d.n, src_lane), mode = __shfl_sync(kFull, d.mode, src_lane);
    uint64_t add;
    if (mode == kDeferBytes) add = etl_dl::bytes_lit_len(n);
    else {
      uint32_t extra = 0;
      bool bs = false;
      for (uint32_t k = lane; k < n; k += 32) { extra += etl_dl::quote_esc(s[k]) ? 1u : 0u; bs = bs || s[k] == '\\'; }
      extra = __reduce_add_sync(kFull, extra);
      bs = __any_sync(kFull, bs);
      add = (uint64_t)n + extra + 2u + (bs ? 1u : 0u) + (mode == kDeferJson ? 14u : 0u);
    }
    if ((int)lane == src_lane) len += add;
  }
  if (i < 3 * P.n_mut * P.w) P.cell_len[i] = len > 0xffffffffull ? 0xffffffffu : (uint32_t)len;
}

__global__ void __launch_bounds__(256) k_dl_write(DlParams P) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  Defer d{nullptr, nullptr, 0, kDeferNone};
  if (i < 3 * P.n_mut * P.w) {
    uint32_t t, c;
    uint64_t m;
    item_of(P, i, &t, &m, &c);
    piece(P, t, m, c, P.out[t] + P.text_off[t][m] + P.cell_len[i], &d);
  }
  unsigned todo = __ballot_sync(kFull, d.mode != kDeferNone);
  while (todo) {
    const int src_lane = __ffs(todo) - 1;
    todo &= todo - 1;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(kFull, reinterpret_cast<unsigned long long>(d.src), src_lane));
    uint8_t* o = reinterpret_cast<uint8_t*>(__shfl_sync(kFull, reinterpret_cast<unsigned long long>(d.dst), src_lane));
    const uint32_t n = __shfl_sync(kFull, d.n, src_lane), mode = __shfl_sync(kFull, d.mode, src_lane);
    if (mode == kDeferBytes) {
      if (lane == 0) etl_dl::cstr_write("from_hex('", o);
      for (uint32_t k = lane; k < n; k += 32) etl_rb::hex_byte_upper(s[k], o + 10 + 2 * k);
      if (lane == 0) etl_dl::cstr_write("')", o + 10 + 2ull * n);
      continue;
    }
    bool bs = false;
    for (uint32_t k = lane; k < n && !bs; k += 32) bs = s[k] == '\\';
    bs = __any_sync(kFull, bs);
    uint64_t at = 0;
    if (mode == kDeferJson) at = 5;                       // "CAST("
    if (lane == 0) {
      if (mode == kDeferJson) etl_dl::cstr_write("CAST(", o);
      if (bs) o[at] = 'E';
      o[at + (bs ? 1 : 0)] = '\'';
    }
    at += bs ? 2 : 1;
    for (uint32_t base = 0; base < n; base += 32) {       // the body with ' and \ doubled: a warp prefix sum of escapes
      const uint32_t k = base + lane;
      const uint8_t b = k < n ? s[k] : 0;
      const bool e = k < n && etl_dl::quote_esc(b);
      const unsigned mask = __ballot_sync(kFull, e);
      if (k < n) {
        const uint64_t pos = at + lane + __popc(mask & ((1u << lane) - 1u));
        o[pos] = b;
        if (e) o[pos + 1] = b;
      }
      at += min(32u, n - base) + __popc(mask);
    }
    if (lane == 0) {
      o[at] = '\'';
      if (mode == kDeferJson) etl_dl::cstr_write(" AS JSON)", o + at + 1);
    }
  }
}

// ---------------------------------------------------------------- sub-batches and fingerprints
struct SubParams {
  const uint64_t* mut_start; const uint64_t* mut_commit; const uint64_t* mut_tx; const uint64_t* mut_seg; const uint8_t* mut_kind;
  uint64_t n_mut;
  const uint8_t* text[3]; const uint64_t* text_off[3];
  const uint32_t* asg_piece; uint32_t w, n_cols;
  const uint32_t* name_len;
  const uint8_t* table_name; uint32_t table_len;
  uint64_t key_commit, key_tx;
  unsigned long long* first;     // first kept mutation
  uint32_t* start;               // 1 at the first mutation of each chunk
  const uint64_t* chunk_of;      // scan of start
  etl_dl_sub_batch* out;
  uint64_t n_chunks;
};

__device__ __forceinline__ uint64_t seg_lower(const SubParams& S, uint64_t seg) {
  uint64_t lo = 0, hi = S.n_mut;
  while (lo < hi) { const uint64_t mid = (lo + hi) / 2; if (S.mut_seg[mid] < seg) lo = mid + 1; else hi = mid; }
  return lo;
}
__device__ __forceinline__ uint64_t seg_upper(const SubParams& S, uint64_t seg) {
  uint64_t lo = 0, hi = S.n_mut;
  while (lo < hi) { const uint64_t mid = (lo + hi) / 2; if (S.mut_seg[mid] <= seg) lo = mid + 1; else hi = mid; }
  return lo;
}
// retain_mutations_after_sequence_key: (commit_lsn, tx_ordinal) greater than the key; keys rise, so a suffix
__global__ void __launch_bounds__(256) k_dl_first_kept(SubParams S) {
  const uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= S.n_mut) return;
  const uint64_t a = S.mut_commit[m], b = S.mut_tx[m];
  if (a > S.key_commit || (a == S.key_commit && b > S.key_tx)) atomicMin(S.first, (unsigned long long)m);
}
__global__ void __launch_bounds__(256) k_dl_chunk_mark(SubParams S) {
  const uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= S.n_mut) return;
  const uint64_t first = *S.first;
  uint32_t st = 0;
  if (m >= first) {
    const uint64_t s0 = max((uint64_t)first, seg_lower(S, S.mut_seg[m]));
    st = (m - s0) % kChunk == 0 ? 1u : 0u;
  }
  S.start[m] = st;
}
__global__ void __launch_bounds__(256) k_dl_chunk_fill(SubParams S) {
  const uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= S.n_mut || !S.start[m]) return;
  const uint64_t end = min(m + kChunk, seg_upper(S, S.mut_seg[m]));
  etl_dl_sub_batch b;
  b.first_mutation = m; b.n_mutations = (uint32_t)(end - m); b._pad = 0; b.fingerprint = 0;
  S.out[S.chunk_of[m]] = b;
}
__device__ __forceinline__ uint64_t fnv_text(const SubParams& S, uint64_t h, uint32_t t, uint64_t m) {
  const uint64_t a = S.text_off[t][m];
  return etl_dl::fnv_str(h, S.text[t] + a, S.text_off[t][m + 1] - a);
}
// build_mutation_batch_identity over one chunk: one serial FNV-1a chain
__global__ void __launch_bounds__(128) k_dl_fingerprint(SubParams S) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= S.n_chunks) return;
  const etl_dl_sub_batch b = S.out[j];
  uint64_t h = etl_dl::fnv_cstr(etl_dl::kFnvBasis, "mutation");
  h = etl_dl::fnv_str(h, S.table_name, S.table_len);
  for (uint64_t m = b.first_mutation; m < b.first_mutation + b.n_mutations; m++) {
    h = etl_dl::fnv_u64(h, S.mut_start[m]);
    h = etl_dl::fnv_u64(h, S.mut_commit[m]);
    switch (S.mut_kind[m] & 0x7fu) {
      case ETL_DL_INSERT: h = fnv_text(S, etl_dl::fnv_cstr(h, "insert"), 0, m); break;
      case ETL_DL_DELETE: h = fnv_text(S, etl_dl::fnv_cstr(h, "delete"), 1, m); break;
      case ETL_DL_UPDATE: h = fnv_text(S, fnv_text(S, etl_dl::fnv_cstr(h, "update"), 1, m), 0, m); break;
      case ETL_DL_REPLACE: h = fnv_text(S, fnv_text(S, etl_dl::fnv_cstr(h, "replace"), 1, m), 0, m); break;
      default: {                                          // UPDATE_PARTIAL: predicate, n_cols, (index, literal) per present column
        h = fnv_text(S, etl_dl::fnv_cstr(h, "update"), 1, m);
        h = etl_dl::fnv_u64(h, S.n_cols);
        const uint8_t* txt = S.text[2] + S.text_off[2][m];
        const uint32_t* pc = S.asg_piece + m * S.w;
        bool first = true;
        for (uint32_t c = 0; c < S.n_cols; c++) {
          const uint32_t a = pc[c], e = pc[c + 1];
          if (a == e) continue;
          const uint32_t lit = a + (first ? 0u : 2u) + S.name_len[c] + 3u;
          first = false;
          h = etl_dl::fnv_str(etl_dl::fnv_u64(h, c), txt + lit, e - lit);
        }
      }
    }
  }
  S.out[j].fingerprint = h;
}

// host FNV-1a 64 (the COPY fingerprint)
uint64_t host_fnv(uint64_t h, const uint8_t* p, uint64_t n) {
  for (uint64_t k = 0; k < n; k++) h = (h ^ p[k]) * etl_dl::kFnvPrime;
  return h;
}
uint64_t host_fnv_str(uint64_t h, const uint8_t* p, uint64_t n) {
  const uint8_t ff = 0xff;
  return host_fnv(host_fnv(h, p, n), &ff, 1);
}

}  // namespace

struct etl_ducklake_batch {
  bool copy = false;
  uint32_t n_cols = 0;
  uint64_t n_mut = 0, bytes[3] = {0, 0, 0};
  uint8_t* meta = nullptr;      // device: records | start | commit | tx | segment (u64 each) | 3 x (n_mut + 1) text offsets | kinds
  uint8_t* text[3] = {nullptr, nullptr, nullptr};   // device texts
  uint32_t* asg_piece = nullptr;                    // device: in-text piece offsets of the assignments (partial updates)
  uint32_t* name_len = nullptr;                     // device: the quoted names' lengths
  uint8_t* host = nullptr;      // pinned: records | 3 x text offsets | kinds | texts (to_host)
  etl_dl_sub_batch* sub = nullptr;       // device
  etl_dl_sub_batch* sub_host = nullptr;  // pinned
  uint64_t n_sub = 0, sub_cap = 0;
  etl_ducklake_issues issues{};
  const uint64_t* dev_u64(int k) const { return reinterpret_cast<const uint64_t*>(meta) + (uint64_t)k * n_mut; }
  const uint64_t* dev_text_off(int t) const { return reinterpret_cast<const uint64_t*>(meta) + 5 * n_mut + (uint64_t)t * (n_mut + 1); }
  const uint8_t* dev_kinds() const { return meta + 8 * (5 * n_mut + 3 * (n_mut + 1)); }
  uint64_t host_meta_bytes() const { return 8 * (n_mut + 3 * (n_mut + 1)) + ((n_mut + 7) & ~7ull); }
};

extern "C" {

int etl_dec_ducklake_emit(const etl_dec_batch* batch, uint32_t schema_index, const char* const* quoted_names, uint32_t n_names,
                          int to_host, etl_ducklake_batch** out) {
  if (!batch || !out) return ETL_ERR_INVALID_ARG;
  EmitBatch E;
  if (open_emit_batch(batch, schema_index, &E) != ETL_OK) return ETL_ERR_INVALID_ARG;
  const etl_dec_planes& P = E.P;
  const etl_dec_schema_info& sc = E.sc;
  const bool copy = E.copy;
  const uint8_t* pk = nullptr;
  if (copy && !etl_copy_batch_pk_columns(batch, &pk)) return ETL_ERR_INVALID_ARG;
  if (n_names != sc.n_cols || (sc.n_cols && !quoted_names)) return ETL_ERR_INVALID_ARG;
  // column descriptors: predicate slot (identity; COPY: primary key), Json item index, quoted names
  std::vector<DlCol> cols(sc.n_cols);
  std::vector<uint32_t> json_col, name_len(sc.n_cols);
  std::vector<uint8_t> names;
  uint32_t n_pred = 0;
  for (uint32_t c = 0; c < sc.n_cols; c++) {
    if (!quoted_names[c]) return ETL_ERR_INVALID_ARG;
    DlCol& d = cols[c];
    d.kind = sc.col_kind[c];
    d.json = -1;
    const bool pred = copy ? pk[c] != 0 : (sc.col_flags[c] & 2u) != 0;
    d.pred = pred ? (int16_t)n_pred++ : (int16_t)-1;
    if ((d.kind & ~(uint32_t)ETL_K_ARRAY) == ETL_K_JSON) { d.json = (int16_t)json_col.size(); json_col.push_back(c); }
    const size_t ln = strlen(quoted_names[c]);
    d.name_off = (uint32_t)names.size();
    d.name_len = name_len[c] = (uint32_t)ln;
    names.insert(names.end(), quoted_names[c], quoted_names[c] + ln);
  }

  cudaStream_t st = cudaStreamPerThread;
  etl_ducklake_batch* B = new etl_ducklake_batch();
  B->copy = copy;
  B->n_cols = sc.n_cols;
  Scratch scratch(st);
  auto fail = [&](int rc) {
    scratch.release();
    cudaStreamSynchronize(st);
    cudaGetLastError();
    etl_dec_ducklake_free(B);
    return rc;
  };
  const uint64_t n_valid = E.n_valid;
  const uint32_t W = sc.n_cols + 1;
  const size_t cols_bytes = (sizeof(DlCol) * cols.size() + 7) & ~(size_t)7;
  uint8_t* d_cols = (uint8_t*)scratch(cols_bytes + 4ull * json_col.size() + names.size());
  unsigned long long* d_issues = (unsigned long long*)scratch(8 * kIssueSlots);
  if (cudaMalloc(&B->name_len, 4ull * sc.n_cols + 4) != cudaSuccess) { B->name_len = nullptr; return fail(ETL_ERR_ALLOC); }
  if (!d_cols || !d_issues) return fail(ETL_ERR_ALLOC);
  uint32_t* d_json_col = reinterpret_cast<uint32_t*>(d_cols + cols_bytes);
  uint8_t* d_names = d_cols + cols_bytes + 4ull * json_col.size();
  if (cudaMemsetAsync(d_issues, 0xff, 16, st) != cudaSuccess || cudaMemsetAsync(d_issues + kIssueFlags, 0, 8, st) != cudaSuccess ||
      (!cols.empty() && cudaMemcpyAsync(d_cols, cols.data(), sizeof(DlCol) * cols.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
      (!json_col.empty() && cudaMemcpyAsync(d_json_col, json_col.data(), 4 * json_col.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
      (!names.empty() && cudaMemcpyAsync(d_names, names.data(), names.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
      (sc.n_cols && cudaMemcpyAsync(B->name_len, name_len.data(), 4ull * sc.n_cols, cudaMemcpyHostToDevice, st) != cudaSuccess))
    return fail(ETL_ERR_CUDA);

  DlParams R{};
  R.cell_tag = P.cell_tag; R.cell_val = P.cell_val; R.cell_aux = P.cell_aux; R.heap = P.heap; R.stream = E.stream;
  R.rec_kind = P.rec_kind; R.rec_flags = P.rec_flags; R.rec_schema = P.rec_schema; R.rec_rel = P.rec_rel;
  R.rec_cell_base = P.rec_cell_base; R.rec_start_lsn = P.rec_start_lsn; R.rec_commit_lsn = P.rec_commit_lsn;
  R.rec_tx_ordinal = P.rec_tx_ordinal;
  R.n_valid = n_valid; R.schema = (int32_t)schema_index; R.table_id = sc.table_id; R.n_cols = sc.n_cols; R.n_pred = n_pred;
  R.copy = copy;
  R.cols = reinterpret_cast<const DlCol*>(d_cols); R.names = d_names; R.json_col = d_json_col; R.n_json = (uint32_t)json_col.size();
  R.issues = d_issues; R.w = W;

  // 1-2. segments, mutations (sync)
  const uint32_t rb = scan_blocks(n_valid);
  const uint32_t tb = (uint32_t)((n_valid + 255) / 256);
  uint64_t n_mut = 0;
  unsigned long long iss[kIssueSlots] = {~0ull, ~0ull, 0};
  if (n_valid) {
    uint32_t* lens = (uint32_t*)scratch(n_valid * 4);
    unsigned long long* blk = (unsigned long long*)scratch((rb + 1) * 8ull);
    R.seg_flags = (uint32_t*)scratch((n_valid + 1) * 4);
    R.rec_mkind = (uint8_t*)scratch(n_valid);
    uint64_t* mpos = (uint64_t*)scratch((n_valid + 1) * 8);
    if (!lens || !blk || !R.seg_flags || !R.rec_mkind || !mpos) return fail(ETL_ERR_ALLOC);
    if (cudaMemsetAsync(R.seg_flags, 0, (n_valid + 1) * 4, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    if (!copy) {
      uint64_t* seg = (uint64_t*)scratch((n_valid + 1) * 8);
      if (!seg) return fail(ETL_ERR_ALLOC);
      k_dl_trunc<<<tb, 256, 0, st>>>(R, lens);
      scan_lengths(lens, n_valid, blk, blk + rb, seg, st);
      R.seg_off = seg;
    } else {
      uint64_t* seg = (uint64_t*)scratch((n_valid + 1) * 8);
      if (!seg || cudaMemsetAsync(seg, 0, (n_valid + 1) * 8, st) != cudaSuccess) return fail(ETL_ERR_ALLOC);
      R.seg_off = seg;
    }
    R.rec_mut = (uint32_t*)scratch(n_valid * 4);
    if (!R.rec_mut) return fail(ETL_ERR_ALLOC);
    k_dl_decide<<<(uint32_t)((n_valid * 32 + 255) / 256), 256, 0, st>>>(R);
    scan_lengths(R.rec_mut, n_valid, blk, blk + rb, mpos, st);
    R.mut_pos = mpos;
    k_dl_mixed<<<(uint32_t)((n_valid + 1 + 255) / 256), 256, 0, st>>>(R.seg_flags, n_valid + 1, d_issues + kIssueFlags);
    unsigned long long nm = 0;
    if (cudaMemcpyAsync(&nm, blk + rb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(iss, d_issues, sizeof iss, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    n_mut = nm;
  }
  B->n_mut = n_mut;
  R.n_mut = n_mut;
  B->issues.first_rejected_record = iss[kIssueReject] == ~0ull ? UINT64_MAX : iss[kIssueReject] >> 3;
  B->issues.rejected_reason = iss[kIssueReject] == ~0ull ? 0u : (uint32_t)(iss[kIssueReject] & 7u);
  B->issues.mixed_versions = (iss[kIssueFlags] & kFlagMixed) ? 1u : 0u;
  B->issues.first_empty_partial_record = iss[kIssueEmpty] == ~0ull ? UINT64_MAX : iss[kIssueEmpty];
  const bool any_partial = (iss[kIssueFlags] & kFlagPartial) != 0;

  const uint64_t meta_bytes = 8 * (5 * n_mut + 3 * (n_mut + 1)) + n_mut + 8;
  if (cudaMalloc(&B->meta, meta_bytes) != cudaSuccess) { B->meta = nullptr; return fail(ETL_ERR_ALLOC); }
  uint64_t* mu = reinterpret_cast<uint64_t*>(B->meta);
  R.mut_rec = mu; R.mut_start = mu + n_mut; R.mut_commit = mu + 2 * n_mut; R.mut_tx = mu + 3 * n_mut; R.mut_seg = mu + 4 * n_mut;
  R.mut_kind = B->meta + 8 * (5 * n_mut + 3 * (n_mut + 1));
  for (int t = 0; t < 3; t++) {
    R.text_off[t] = B->dev_text_off(t);
    if (cudaMemsetAsync((void*)R.text_off[t], 0, 8, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  }
  if (n_mut) k_dl_scatter<<<tb, 256, 0, st>>>(R);

  // 3. Json: input lengths → item offsets → (sync) canonical text
  const uint64_t n_items = n_mut * 2 * R.n_json;
  if (n_items) {
    JsonStage J{P.cell_tag, P.cell_val, P.cell_aux, P.heap, E.stream, n_items, nullptr, nullptr, nullptr,
                d_issues + kIssueFlags, (unsigned long long)kFlagBadJson};
    if (int rc = stage_json(scratch, J, DlJsonCells{R}, st)) return fail(rc);
    R.json_off = J.off;
    R.canon = J.canon;
  }

  // 4. sizes → in-text offsets → text offsets (sync)
  unsigned long long tot[4] = {0, 0, 0, 0};             // bytes of each text, flags
  if (n_mut) {
    const uint64_t n_pieces = 3 * n_mut * W;
    const uint32_t mb = scan_blocks(n_mut);
    R.cell_len = (uint32_t*)scratch(n_pieces * 4);
    uint32_t* tlen = (uint32_t*)scratch(n_mut * 4);
    unsigned long long* mblk = (unsigned long long*)scratch(3 * (mb + 1) * 8ull);
    if (!R.cell_len || !tlen || !mblk) return fail(ETL_ERR_ALLOC);
    k_dl_size<<<(uint32_t)((n_pieces + 255) / 256), 256, 0, st>>>(R);
    for (int t = 0; t < 3; t++) {
      unsigned long long* tb_ = mblk + t * (mb + 1);
      k_row_scan<<<(uint32_t)((n_mut * 32 + 255) / 256), 256, 0, st>>>(R.cell_len + t * n_mut * W, W, n_mut, tlen, d_issues + kIssueFlags,
                                                                        (unsigned long long)kFlagTextTooLong);
      scan_lengths(tlen, n_mut, tb_, tb_ + mb, const_cast<uint64_t*>(R.text_off[t]), st);
      if (cudaMemcpyAsync(&tot[t], tb_ + mb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    }
    if (cudaMemcpyAsync(&tot[3], d_issues + kIssueFlags, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    if (tot[3] & kFlagBadJson) return fail(ETL_ERR_INTERNAL);        // a Json value the decode accepted did not parse again
    if (tot[3] & kFlagTextTooLong) return fail(ETL_ERR_INVALID_ARG); // one text of 4 GiB or more
  }
  // 5. texts
  for (int t = 0; t < 3; t++) {
    B->bytes[t] = tot[t];
    if (cudaMalloc(&B->text[t], B->bytes[t] + 64) != cudaSuccess) { B->text[t] = nullptr; return fail(ETL_ERR_ALLOC); }
    R.out[t] = B->text[t];
  }
  if (n_mut) k_dl_write<<<(uint32_t)((3 * n_mut * W + 255) / 256), 256, 0, st>>>(R);
  if (n_mut && any_partial) {                           // keep the assignment pieces for the fingerprint
    if (cudaMalloc(&B->asg_piece, 4ull * n_mut * W) != cudaSuccess) { B->asg_piece = nullptr; return fail(ETL_ERR_ALLOC); }
    if (cudaMemcpyAsync(B->asg_piece, R.cell_len + 2 * n_mut * W, 4ull * n_mut * W, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  }
  if (to_host) {
    const uint64_t hm = B->host_meta_bytes();
    if (cudaHostAlloc((void**)&B->host, hm + B->bytes[0] + B->bytes[1] + B->bytes[2] + 64, cudaHostAllocDefault) != cudaSuccess) {
      B->host = nullptr;
      return fail(ETL_ERR_ALLOC);
    }
    uint8_t* h = B->host;
    if (cudaMemcpyAsync(h, B->meta, 8 * n_mut, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(h + 8 * n_mut, B->dev_text_off(0), 24 * (n_mut + 1), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (n_mut && cudaMemcpyAsync(h + 8 * (n_mut + 3 * (n_mut + 1)), B->dev_kinds(), n_mut, cudaMemcpyDeviceToHost, st) != cudaSuccess))
      return fail(ETL_ERR_CUDA);
    uint64_t at = hm;
    for (int t = 0; t < 3; t++) {
      if (B->bytes[t] && cudaMemcpyAsync(h + at, B->text[t], B->bytes[t], cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
      at += B->bytes[t];
    }
  }
  scratch.release();
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ETL_ERR_CUDA);
  *out = B;
  return ETL_OK;
}

uint64_t etl_dec_ducklake_mutations(const etl_ducklake_batch* b) { return b ? b->n_mut : 0; }
const uint8_t* etl_dec_ducklake_kinds(const etl_ducklake_batch* b, int host) {
  if (!b) return nullptr;
  if (!host) return b->dev_kinds();
  return b->host ? b->host + 8 * (b->n_mut + 3 * (b->n_mut + 1)) : nullptr;
}
const uint64_t* etl_dec_ducklake_records(const etl_ducklake_batch* b, int host) {
  if (!b) return nullptr;
  if (!host) return reinterpret_cast<const uint64_t*>(b->meta);
  return b->host ? reinterpret_cast<const uint64_t*>(b->host) : nullptr;
}
int etl_dec_ducklake_text(const etl_ducklake_batch* b, uint32_t which, int host, const uint8_t** data, const uint64_t** offsets, uint64_t* bytes) {
  if (!b || which > ETL_DL_TEXT_ASSIGNMENTS || !data || !offsets || !bytes) return ETL_ERR_INVALID_ARG;
  if (host && !b->host) return ETL_ERR_INVALID_ARG;
  *bytes = b->bytes[which];
  if (!host) { *data = b->text[which]; *offsets = b->dev_text_off((int)which); return ETL_OK; }
  uint64_t at = b->host_meta_bytes();
  for (uint32_t t = 0; t < which; t++) at += b->bytes[t];
  *data = b->host + at;
  *offsets = reinterpret_cast<const uint64_t*>(b->host) + b->n_mut + (uint64_t)which * (b->n_mut + 1);
  return ETL_OK;
}
int etl_dec_ducklake_issues(const etl_ducklake_batch* b, etl_ducklake_issues* out) {
  if (!b || !out) return ETL_ERR_INVALID_ARG;
  *out = b->issues;
  return ETL_OK;
}

int etl_dec_ducklake_sub_batches(etl_ducklake_batch* b, const uint8_t* table_name, uint32_t name_len, const uint64_t* last_key,
                                 int host, const etl_dl_sub_batch** out, uint64_t* n) {
  if (!b || !out || !n || b->copy || (name_len && !table_name)) return ETL_ERR_INVALID_ARG;
  cudaStream_t st = cudaStreamPerThread;
  const uint64_t nm = b->n_mut;
  Scratch scratch(st);
  auto done = [&](int rc) {
    scratch.release();
    if (cudaStreamSynchronize(st) != cudaSuccess && rc == ETL_OK) rc = ETL_ERR_CUDA;
    if (cudaGetLastError() != cudaSuccess && rc == ETL_OK) rc = ETL_ERR_CUDA;
    return rc;
  };
  SubParams S{};
  S.mut_start = b->dev_u64(1); S.mut_commit = b->dev_u64(2); S.mut_tx = b->dev_u64(3); S.mut_seg = b->dev_u64(4);
  S.mut_kind = b->dev_kinds(); S.n_mut = nm;
  for (int t = 0; t < 3; t++) { S.text[t] = b->text[t]; S.text_off[t] = b->dev_text_off(t); }
  S.asg_piece = b->asg_piece; S.w = b->n_cols + 1; S.n_cols = b->n_cols; S.name_len = b->name_len;
  S.table_len = name_len;
  S.key_commit = last_key ? last_key[0] : 0; S.key_tx = last_key ? last_key[1] : 0;
  uint64_t n_chunks = 0;
  if (nm) {
    const uint32_t tb = (uint32_t)((nm + 255) / 256), mb = scan_blocks(nm);
    uint8_t* tname = (uint8_t*)scratch(name_len);
    S.first = (unsigned long long*)scratch(8);
    S.start = (uint32_t*)scratch(nm * 4);
    uint64_t* chunk_of = (uint64_t*)scratch((nm + 1) * 8);
    unsigned long long* blk = (unsigned long long*)scratch((mb + 1) * 8ull);
    if (!tname || !S.first || !S.start || !chunk_of || !blk) return done(ETL_ERR_ALLOC);
    S.table_name = tname;
    S.chunk_of = chunk_of;
    if ((name_len && cudaMemcpyAsync(tname, table_name, name_len, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemsetAsync(S.first, last_key ? 0xff : 0, 8, st) != cudaSuccess) return done(ETL_ERR_CUDA);
    if (last_key) k_dl_first_kept<<<tb, 256, 0, st>>>(S);
    k_dl_chunk_mark<<<tb, 256, 0, st>>>(S);
    scan_lengths(S.start, nm, blk, blk + mb, chunk_of, st);
    unsigned long long nc = 0;
    if (cudaMemcpyAsync(&nc, blk + mb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) return done(ETL_ERR_CUDA);
    n_chunks = nc;
    if (n_chunks > b->sub_cap) {
      if (b->sub) cudaFree(b->sub);
      if (b->sub_host) cudaFreeHost(b->sub_host);
      b->sub = nullptr; b->sub_host = nullptr; b->sub_cap = 0;
      if (cudaMalloc(&b->sub, n_chunks * sizeof(etl_dl_sub_batch)) != cudaSuccess) { b->sub = nullptr; return done(ETL_ERR_ALLOC); }
      b->sub_cap = n_chunks;
    }
    S.out = b->sub;
    S.n_chunks = n_chunks;
    if (n_chunks) {
      k_dl_chunk_fill<<<tb, 256, 0, st>>>(S);
      k_dl_fingerprint<<<(uint32_t)((n_chunks + 127) / 128), 128, 0, st>>>(S);
    }
  }
  b->n_sub = n_chunks;
  if (host && n_chunks) {
    if (!b->sub_host && cudaHostAlloc((void**)&b->sub_host, b->sub_cap * sizeof(etl_dl_sub_batch), cudaHostAllocDefault) != cudaSuccess) {
      b->sub_host = nullptr;
      return done(ETL_ERR_ALLOC);
    }
    if (cudaMemcpyAsync(b->sub_host, b->sub, n_chunks * sizeof(etl_dl_sub_batch), cudaMemcpyDeviceToHost, st) != cudaSuccess) return done(ETL_ERR_CUDA);
  }
  const int rc = done(ETL_OK);
  if (rc != ETL_OK) return rc;
  *out = host ? b->sub_host : b->sub;
  *n = n_chunks;
  return ETL_OK;
}

int etl_dec_ducklake_copy_fingerprint(const etl_ducklake_batch* b, const uint8_t* table_name, uint32_t name_len, uint64_t* out) {
  if (!b || !out || !b->copy || !b->host || (name_len && !table_name)) return ETL_ERR_INVALID_ARG;
  const uint8_t copy_word[4] = {'c', 'o', 'p', 'y'};
  uint64_t h = host_fnv_str(etl_dl::kFnvBasis, copy_word, 4);
  h = host_fnv_str(h, table_name, name_len);
  const uint8_t *row, *pred;
  const uint64_t *row_off, *pred_off;
  uint64_t nb;
  etl_dec_ducklake_text(b, ETL_DL_TEXT_ROW, 1, &row, &row_off, &nb);
  etl_dec_ducklake_text(b, ETL_DL_TEXT_PREDICATE, 1, &pred, &pred_off, &nb);
  for (uint64_t m = 0; m < b->n_mut; m++) {
    h = host_fnv_str(h, pred + pred_off[m], pred_off[m + 1] - pred_off[m]);
    h = host_fnv_str(h, row + row_off[m], row_off[m + 1] - row_off[m]);
  }
  *out = h;
  return ETL_OK;
}

void etl_dec_ducklake_free(etl_ducklake_batch* b) {
  if (!b) return;
  if (b->meta) cudaFree(b->meta);
  for (int t = 0; t < 3; t++) if (b->text[t]) cudaFree(b->text[t]);
  if (b->asg_piece) cudaFree(b->asg_piece);
  if (b->name_len) cudaFree(b->name_len);
  if (b->host) cudaFreeHost(b->host);
  if (b->sub) cudaFree(b->sub);
  if (b->sub_host) cudaFreeHost(b->sub_host);
  delete b;
}

}  // extern "C"
