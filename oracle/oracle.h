/*
 * oracle.h — CPU oracle for the pgoutput decode path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this. The product (etl_b200/, libetl_decode.so) never links or calls it.
 *
 * Parity status: the reference (Rust) needs a Rust toolchain and its un-vendored crates to build,
 * so this is a restatement ("port"). It is pinned against every known-answer test the
 * reference holds for the path (tests/test_oracle_reference_vectors.py quotes them with
 * file:line). Behaviour that lives in third-party crates absent from the reference tree and is not
 * covered by an in-tree reference test is marked "parity unpinned" where it is implemented
 * (chrono leniency, uuid alternate spellings, serde_json depth limit, pgoutput Begin/Commit/
 * Relation/Insert/Truncate layouts which follow the PostgreSQL protocol documentation).
 */
#ifndef ETL_ORACLE_H
#define ETL_ORACLE_H

#include "../include/etl_decode.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_ctx orc_ctx;

typedef struct orc_schema {
  uint32_t table_id;
  uint32_t n_cols;
  uint32_t n_identity;
  uint32_t _pad;
  uint64_t snapshot_id;
  uint64_t effective_off;
  uint8_t* col_kind;
  uint8_t* col_flags;
  int32_t* col_index;
} orc_schema;

typedef struct orc_batch {
  uint64_t n_records, n_cells, heap_bytes;
  uint64_t* rec_off;
  uint8_t* rec_kind;
  uint8_t* rec_flags;
  uint32_t* rec_rel;
  int32_t* rec_schema;
  uint64_t* rec_start_lsn;
  uint64_t* rec_commit_lsn;
  uint64_t* rec_tx_ordinal;
  uint64_t* rec_cell_base; /* n_records + 1 */
  uint32_t* rec_tuple_bytes; /* DML: Σ text lengths of the frame's tuples (ETL_ROW_SIZE_BYTES sample), else 0 */
  uint32_t* rec_heap_hint;   /* DML: Σ heap bytes of the String / Bytes / Numeric cells (size hints), else 0 */
  uint8_t* cell_tag;
  uint64_t* cell_val;
  uint32_t* cell_aux;
  uint8_t* heap;
  etl_first_error first_error;
  etl_stream_state carry_out;
  uint64_t insert_bytes, update_bytes, delete_bytes, n_events;
  uint32_t n_schemas;
  uint32_t _pad;
  orc_schema* schemas;
  /* capacities (internal) */
  uint64_t cap_records, cap_cells, cap_heap, cap_schemas;
} orc_batch;

orc_ctx* orc_create(void);
void orc_destroy(orc_ctx*);
int orc_put_table_schema(orc_ctx*, uint32_t table_id, uint64_t snapshot_id,
                         const etl_column_schema* cols, uint32_t n_cols);
void orc_reset_relations(orc_ctx*);
/* decode a framed stream; `out` is zero-initialised by the callee and must be released with
 * orc_batch_free. Returns 0; data errors are in out->first_error. */
int orc_decode(orc_ctx*, const uint8_t* buf, uint64_t len, const etl_stream_state* carry_in,
               orc_batch* out);
void orc_batch_free(orc_batch*);

/* text.rs:28 parse_cell_from_postgres_text for one value. heap receives numeric/bytes/uuid/array
 * payloads (offsets in val are relative to heap). Returns etl_error_code (0 = ok). */
uint32_t orc_parse_cell(uint32_t type_oid, const uint8_t* text, uint32_t len, uint8_t* tag,
                        uint64_t* val, uint32_t* aux, uint8_t* heap, uint32_t heap_cap,
                        uint32_t* heap_len);
/* type oid → ETL_K_* exactly as text.rs:28-173 + utils.rs:7-16 dispatch */
uint32_t orc_kind_for_oid(uint32_t type_oid);

/* COPY-text row (table_row.rs:25-165; SURVEY §8f N1 groundwork).  Cells of kind string/json carry offsets
 * into `text_out` (the unescaped field values); numeric/bytea/uuid/array offsets into `heap_out`.
 * Returns 0 or an error code: an ETL_E_* cell error, or one of the two row-level errors below. */
#define ORC_E_COPY_NOT_TERMINATED 101u   /* "Row data not properly terminated" (ConversionError) */
#define ORC_E_COPY_COLUMN_COUNT 102u     /* "Column count mismatch between schema and row" (ConversionError) */
uint32_t orc_parse_copy_row(const uint32_t* type_oids, uint32_t n_cols, const uint8_t* row, uint64_t len,
                            uint8_t* tags, uint64_t* vals, uint32_t* auxs, uint32_t* n_values,
                            uint8_t* text_out, uint64_t text_cap, uint64_t* text_len,
                            uint8_t* heap_out, uint64_t heap_cap, uint64_t* heap_len, uint32_t* err_col);
uint32_t orc_error_kind(uint32_t code);

/* canonical 256-bit digest of records [0, n_valid) of a decoded batch (oracle_digest.c): var-width payloads are
 * dereferenced, so two decodes of the same stream compare equal whatever their heap placement */
void orc_planes_digest(const etl_dec_planes* p, uint64_t n_valid, uint64_t out[4]);
void orc_batch_digest(const orc_batch* b, uint64_t out[4]);
/* COPY rows: digest of device planes / of the oracle's own row-by-row parse (strings by content) */
void orc_copy_planes_digest(const uint8_t* tags, const uint64_t* vals, const uint32_t* auxs, uint64_t n_valid_rows, uint32_t n_cols,
                            const uint8_t* stream, const uint8_t* heap, uint64_t out[4]);
void orc_copy_rows_digest(const uint32_t* type_oids, uint32_t n_cols, const uint8_t* buf, const uint64_t* row_off, uint64_t n_rows,
                          uint64_t out[4], uint64_t* err_row, uint32_t* err_col, uint32_t* err_code);

#ifdef __cplusplus
}
#endif
#endif
