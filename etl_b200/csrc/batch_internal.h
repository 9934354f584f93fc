// batch_internal.h — library-internal accessors of etl_dec_batch shared between decode_api.cu, the destination
// emitters and shim_materialise.cpp (not part of include/etl_decode.h: the public view of a COPY batch has no schema
// entries).
#pragma once
#include <stdint.h>

#include "etl_decode.h"

// A COPY batch (etl_dec_copy_decode): the table id and the ETL_K_* class of each column as they were when the batch was
// decoded (a later etl_dec_put_table_schema does not change them).  False for a streaming batch.
bool etl_copy_batch_columns(const etl_dec_batch*, uint32_t* table_id, const uint8_t** col_kind, uint32_t* n_cols);
// A COPY batch: per column, 1 when the stored TableSchema column has a primary_key_ordinal_position, as it was when the
// batch was decoded.  False for a streaming batch.
bool etl_copy_batch_pk_columns(const etl_dec_batch*, const uint8_t** pk);
// Replicated-schema version `index` of a streaming batch: per replicated column, 1 when the stored TableSchema's column
// (col_index) has a primary_key_ordinal_position, as it was when the Relation installed the version.  False when there
// is no such version.
bool etl_schema_pk_columns(const etl_dec_batch*, uint32_t index, const uint8_t** pk);
// The records of the batch's valid prefix: all of them, or those before the first error.
uint64_t etl_batch_valid_records(const etl_dec_batch*);

// What an emitter reads of a batch: its planes and device stream, the columns of the version it emits (a COPY batch,
// copy: the columns it was decoded with, schema_index 0 only) and the valid prefix's record count.
struct EmitBatch {
  etl_dec_planes P;
  const uint8_t* stream;
  bool copy;
  etl_dec_schema_info sc;
  uint64_t n_valid;
};
inline int open_emit_batch(const etl_dec_batch* batch, uint32_t schema_index, EmitBatch* E) {
  E->stream = etl_dec_batch_device_stream(batch);
  E->sc = etl_dec_schema_info{};
  if (etl_dec_batch_planes(batch, 0, &E->P) != ETL_OK) return ETL_ERR_INVALID_ARG;
  E->copy = E->P.rec_kind == nullptr;
  if (E->copy) {
    if (schema_index != 0 || !etl_copy_batch_columns(batch, &E->sc.table_id, &E->sc.col_kind, &E->sc.n_cols)) return ETL_ERR_INVALID_ARG;
  } else if (etl_dec_batch_schema(batch, schema_index, &E->sc) != ETL_OK) {
    return ETL_ERR_INVALID_ARG;
  }
  E->n_valid = etl_batch_valid_records(batch);
  return ETL_OK;
}
