// host_rowbinary.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE formatters of the ClickHouse RowBinary emitter (etl_b200/csrc/rowbinary_format.cuh — the very
// source nvcc compiles for sm_90a) for the host, so that the CPU suite can fuzz them against the Python restatement
// (tests/clickhouse_ref.py, tests/test_rowbinary_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "rowbinary_format.cuh"

// LEB128 of v into out (10 bytes of room); returns the length, -1 when varint_len disagrees with varint_write
extern "C" int64_t emu_varint(uint64_t v, uint8_t* out) {
  const uint32_t n = etl_rb::varint_write(v, out);
  return n == etl_rb::varint_len(v) ? (int64_t)n : -1;
}
// NaiveTime's Display of (seconds since midnight, nanoseconds) into out (18 bytes of room); -1 when time_len disagrees
extern "C" int64_t emu_time(uint64_t secs, uint32_t nanos, uint8_t* out) {
  const uint32_t n = etl_rb::time_write(secs, nanos, out);
  return n == etl_rb::time_len(nanos) ? (int64_t)n : -1;
}
extern "C" void emu_hex(const uint8_t* src, uint32_t n, uint8_t* out) { etl_rb::hex_write(src, n, out); }
extern "C" int emu_date32_ok(int64_t days) { return etl_rb::date32_ok(days) ? 1 : 0; }
extern "C" void emu_uuid(const uint8_t* be, uint8_t* out) { etl_rb::uuid_write(be, out); }
