// arrow_internal.h — the layout of an etl_arrow_batch, shared by the translation units that build one: the emitter
// (arrow_emit.cu) and the Iceberg partition step (iceberg_partition.cu), which builds a permuted copy.  Readers go
// through the public accessors (etl_dec_arrow_column, etl_dec_arrow_list_child, …) instead.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "etl_decode.h"

namespace etl_arrow {

struct Col {
  uint32_t arrow_type = 0;
  uint64_t validity_off = 0, values_off = 0, offsets_off = 0, data_off = 0, data_bytes = 0, values_bytes = 0, offsets_bytes = 0;
  uint32_t kind = 0;            // ETL_K_* of the column (children: of the element)
  bool text = false;            // Utf8 by cell_to_string (Numeric / Json formatted)
  int32_t child = -1;           // List: index into etl_arrow_batch::kids
  uint64_t n_items = 0;         // children: element count
};
inline uint32_t value_width(uint32_t at) {
  switch (at) {
    case ETL_ARROW_INT32: case ETL_ARROW_DATE32: case ETL_ARROW_FLOAT32: return 4;
    case ETL_ARROW_INT64: case ETL_ARROW_FLOAT64: case ETL_ARROW_TIME64_US: case ETL_ARROW_TIMESTAMP_US: case ETL_ARROW_TIMESTAMPTZ_US: return 8;
    case ETL_ARROW_UUID: return 16;
    default: return 0;
  }
}
inline bool is_var(uint32_t at) { return at == ETL_ARROW_UTF8 || at == ETL_ARROW_LARGE_BINARY || at == ETL_ARROW_LIST; }

}  // namespace etl_arrow

struct etl_arrow_batch {
  uint64_t n_rows = 0;
  std::vector<etl_arrow::Col> cols;
  std::vector<etl_arrow::Col> kids;      // List children (ETL_ARROW_ALL_COLUMNS)
  uint8_t* dev = nullptr;     // one device allocation: row_rec | per column validity, values / offsets | data | children
  uint8_t* host = nullptr;    // pinned host image (to_host)
  uint64_t bytes = 0, row_rec_off = 0;
  uint64_t first_skipped = UINT64_MAX;   // etl_dec_arrow_first_skipped
  std::string error;
};
