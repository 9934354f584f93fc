// host_iceberg_partition.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the Iceberg partition transforms (etl_b200/csrc/iceberg_partition.cuh — the very source nvcc compiles for
// sm_90a) for the host, so that the CPU suite can check murmur3, bucket, truncate and the calendar fields against the
// Python restatement (tests/iceberg_partition_ref.py, tests/test_iceberg_partition_cpu.py).  Nothing outside tests/
// loads it.
#include <stdint.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "iceberg_partition.cuh"

extern "C" uint32_t emu_murmur3(const uint8_t* p, uint64_t len, uint32_t seed) { return etl_ice::murmur3_32(p, len, seed); }
extern "C" uint32_t emu_murmur3_i64(int64_t v) { return etl_ice::murmur3_i64(v); }
extern "C" int64_t emu_bucket(uint32_t hash, uint32_t n) { return etl_ice::bucket_of(hash, n); }
extern "C" int64_t emu_truncate_i32(int32_t v, uint32_t w) { return etl_ice::truncate_i32(v, w); }
extern "C" int64_t emu_truncate_i64(int64_t v, uint32_t w) { return etl_ice::truncate_i64(v, w); }
extern "C" uint32_t emu_utf8_prefix(const uint8_t* p, uint32_t len, uint32_t w) { return etl_ice::utf8_prefix(p, len, w); }
extern "C" int64_t emu_years(int64_t days) { return etl_ice::years_of_days(days); }
extern "C" int64_t emu_months(int64_t days) { return etl_ice::months_of_days(days); }
extern "C" int64_t emu_days(int64_t micros) { return etl_ice::days_of_micros(micros); }
extern "C" int64_t emu_hours(int64_t micros) { return etl_ice::hours_of_micros(micros); }
