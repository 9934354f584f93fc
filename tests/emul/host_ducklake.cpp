// host_ducklake.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE formatters of the DuckLake emitter (etl_b200/csrc/ducklake_format.cuh — the very source nvcc
// compiles for sm_90a) for the host, so that the CPU suite can fuzz them against the Python restatement
// (tests/ducklake_ref.py, tests/test_ducklake_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "ducklake_format.cuh"

// float_literal of an F64 (is_double 1) or of the F64 an F32 widens to (is_double 0, bits = the f32's bits) into out
// (400 bytes of room); -1 when the length function disagrees with the writer
extern "C" int64_t emu_float_lit(uint64_t bits, int is_double, uint8_t* out) {
  const uint64_t b = is_double ? bits : etl_dl::f32_bits_as_f64((uint32_t)bits);
  const uint32_t n = etl_dl::float_lit_write(b, is_double != 0, out);
  return n == etl_dl::float_lit_len(b, is_double != 0) ? (int64_t)n : -1;
}
extern "C" int64_t emu_quote(const uint8_t* s, uint32_t n, uint8_t* out) {
  bool bs = false;
  const uint32_t w = etl_dl::quote_write(s, n, out);
  return w == etl_dl::quote_len(s, n, &bs) ? (int64_t)w : -1;
}
extern "C" int64_t emu_bytes_lit(const uint8_t* s, uint32_t n, uint8_t* out) {
  const uint32_t w = etl_dl::bytes_lit_write(s, n, out);
  return w == etl_dl::bytes_lit_len(n) ? (int64_t)w : -1;
}
extern "C" int64_t emu_time_lit(uint64_t secs, uint32_t nanos, uint8_t* out) {
  const uint32_t w = etl_dl::time_lit_write(secs, nanos, out);
  return w == etl_dl::kTimeLitLen ? (int64_t)w : -1;
}
extern "C" int64_t emu_date_lit(int64_t days, uint8_t* out) {
  const uint32_t w = etl_dl::date_lit_write(days, out);
  return w == etl_dl::date_lit_len(days) ? (int64_t)w : -1;
}
extern "C" int64_t emu_ts_lit(int64_t secs, uint32_t nanos, int tz, uint8_t* out) {
  const uint32_t w = etl_dl::ts_lit_write(secs, nanos, tz != 0, out);
  return w == etl_dl::ts_lit_len(secs, tz != 0) ? (int64_t)w : -1;
}
extern "C" int64_t emu_int_lit(int64_t v, uint8_t* out) {
  const uint32_t w = etl_dl::int_write(v, out);
  return w == etl_dl::int_len(v) ? (int64_t)w : -1;
}
extern "C" uint64_t emu_fnv_str(const uint8_t* s, uint64_t n) { return etl_dl::fnv_str(etl_dl::kFnvBasis, s, n); }
extern "C" uint64_t emu_fnv_bytes(const uint8_t* s, uint64_t n) { return etl_dl::fnv_bytes(etl_dl::kFnvBasis, s, n); }
