// batch_internal.h — library-internal accessors of etl_dec_batch shared between decode_api.cu and arrow_emit.cu
// / rowbinary_emit.cu (not part of include/etl_decode.h: the public view of a COPY batch has no schema entries).
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
