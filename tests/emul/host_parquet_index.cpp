// host_parquet_index.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the page index pieces of the Parquet writer (etl_b200/csrc/parquet_format.cuh — the very source nvcc compiles
// for sm_90a) for the host, so that the CPU suite can check the ColumnIndex bound truncation and the PageLocation of
// ETL_PQ_PAGE_INDEX against the Python restatement (tests/parquet_index_ref.py, tests/test_parquet_index_cpu.py).
// Nothing outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "parquet_format.cuh"

// the truncated ColumnIndex minimum / maximum of v[0, len) into out (room for len bytes); returns its length
extern "C" uint64_t emu_index_min(const uint8_t* v, uint64_t len, int utf8, uint8_t* out) {
  return etl_pq::index_min(v, len, utf8 != 0, out);
}
extern "C" uint64_t emu_index_max(const uint8_t* v, uint64_t len, int utf8, uint8_t* out) {
  return etl_pq::index_max(v, len, utf8 != 0, out);
}
extern "C" uint32_t emu_page_location(uint64_t offset, uint32_t size, uint64_t first_row, uint8_t* out) {
  return etl_pq::page_location(out, offset, size, first_row);
}
