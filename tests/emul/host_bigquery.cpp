// host_bigquery.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE formatters of the BigQuery emitter (etl_b200/csrc/bigquery_format.cuh — the very source nvcc
// compiles for sm_90a) for the host, so that the CPU suite can fuzz them against the Python restatement
// (tests/bigquery_ref.py, tests/test_bigquery_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "bigquery_format.cuh"

// %Y-%m-%d of a day count into out (32 bytes of room); -1 when date_len disagrees with date_write
extern "C" int64_t emu_date(int64_t days, uint8_t* out) {
  const uint32_t n = etl_bq::date_write(days, out);
  return n == etl_bq::date_len(days) ? (int64_t)n : -1;
}
// %Y-%m-%d %H:%M:%S%.f[+00:00] into out (64 bytes of room); -1 when timestamp_len disagrees
extern "C" int64_t emu_timestamp(int64_t secs, uint32_t nanos, int tz, uint8_t* out) {
  const uint32_t n = etl_bq::timestamp_write(secs, nanos, tz != 0, out);
  return n == etl_bq::timestamp_len(secs, nanos, tz != 0) ? (int64_t)n : -1;
}
extern "C" void emu_uuid_text(const uint8_t* be, uint8_t* out) { etl_bq::uuid_text_write(be, out); }
// the field key followed by the varint prost writes for an int32 / int64 (sign-extended) or uint32 value
extern "C" int64_t emu_int_field(uint32_t field, uint64_t val, uint8_t* out) {
  const uint32_t k = etl_bq::key_write(field, etl_bq::kWtVarint, out);
  if (k != etl_bq::key_len(field)) return -1;
  return k + etl_rb::varint_write(val, out + k);
}
extern "C" int emu_numeric_scale_bad(const uint8_t* num, uint32_t nd) { return etl_bq::numeric_scale_bad(num, nd) ? 1 : 0; }
extern "C" int emu_json_int_bad(const uint8_t* s, uint32_t n) { return etl_bq::json_int_bad(s, n) ? 1 : 0; }
