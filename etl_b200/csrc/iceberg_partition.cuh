// iceberg_partition.cuh — the Iceberg partition transforms (spec "Partition Transforms", Appendix B for the hash) as
// host + device functions: murmur3_x86_32, bucket, truncate (integers and UTF-8 code points), and the calendar fields
// year / month / day / hour.  iceberg_partition.cu runs them per (row, field) on the device; tests/emul compiles this
// same file for the host.
#pragma once
#include <stdint.h>

namespace etl_ice {

__host__ __device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__host__ __device__ __forceinline__ uint32_t fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}
__host__ __device__ __forceinline__ uint32_t mm3_k(uint32_t k) { k *= 0xcc9e2d51u; k = rotl32(k, 15); return k * 0x1b873593u; }
__host__ __device__ __forceinline__ uint32_t mm3_mix(uint32_t h, uint32_t k) { h ^= mm3_k(k); h = rotl32(h, 13); return h * 5u + 0xe6546b64u; }
// MurmurHash3_x86_32 (Austin Appleby), little-endian blocks, byte reads (no alignment assumed)
__host__ __device__ inline uint32_t murmur3_32(const uint8_t* p, uint64_t len, uint32_t seed) {
  uint32_t h = seed;
  const uint64_t nb = len >> 2;
  for (uint64_t i = 0; i < nb; i++) {
    const uint8_t* b = p + 4 * i;
    h = mm3_mix(h, (uint32_t)b[0] | (uint32_t)b[1] << 8 | (uint32_t)b[2] << 16 | (uint32_t)b[3] << 24);
  }
  const uint8_t* t = p + 4 * nb;
  uint32_t k = 0;
  switch (len & 3) {
    case 3: k ^= (uint32_t)t[2] << 16; [[fallthrough]];
    case 2: k ^= (uint32_t)t[1] << 8; [[fallthrough]];
    case 1: k ^= t[0]; h ^= mm3_k(k);
  }
  h ^= (uint32_t)len;
  return fmix32(h);
}
// the hash of an integer-valued source: the value widened to a little-endian int64 (Appendix B)
__host__ __device__ __forceinline__ uint32_t murmur3_i64(int64_t v) {
  const uint64_t u = (uint64_t)v;
  uint32_t h = mm3_mix(0u, (uint32_t)u);
  h = mm3_mix(h, (uint32_t)(u >> 32));
  return fmix32(h ^ 8u);
}
// bucket[N] of a hash: (hash & INT32_MAX) % N
__host__ __device__ __forceinline__ int64_t bucket_of(uint32_t hash, uint32_t n) { return (int64_t)((hash & 0x7FFFFFFFu) % n); }

// truncate[W] of an integer, v - (((v % W) + W) % W), wrapping in the source's width like Java / Rust two's complement
__host__ __device__ __forceinline__ int64_t truncate_i32(int32_t v, uint32_t w) {
  const int64_t r = (((int64_t)v % (int64_t)w) + (int64_t)w) % (int64_t)w;
  return (int64_t)(int32_t)((uint32_t)v - (uint32_t)r);
}
__host__ __device__ __forceinline__ int64_t truncate_i64(int64_t v, uint32_t w) {
  const int64_t r = ((v % (int64_t)w) + (int64_t)w) % (int64_t)w;
  return (int64_t)((uint64_t)v - (uint64_t)r);
}
// truncate[W] of UTF-8 text: the byte length of its first W code points (a code point starts at every byte that is not
// a continuation byte 10xxxxxx); the whole text when it has fewer
__host__ __device__ inline uint32_t utf8_prefix(const uint8_t* p, uint32_t len, uint32_t w) {
  uint32_t starts = 0;
  for (uint32_t i = 0; i < len; i++) {
    if ((p[i] & 0xC0u) != 0x80u && starts++ == w) return i;
  }
  return len;
}

// floor division and the proleptic Gregorian civil date of a day count (days since 1970-01-01)
__host__ __device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) { const int64_t q = a / b; return q - ((a % b != 0) & ((a < 0) != (b < 0))); }
__host__ __device__ inline void civil_from_days(int64_t z, int64_t* y, uint32_t* m) {
  z += 719468;
  const int64_t era = floor_div(z, 146097);
  const uint32_t doe = (uint32_t)(z - era * 146097);
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp = (5 * doy + 2) / 153;
  *m = mp < 10 ? mp + 3 : mp - 9;
  *y = (int64_t)yoe + era * 400 + (*m <= 2);
}
constexpr int64_t kMicrosPerDay = 86400000000ll, kMicrosPerHour = 3600000000ll;
// year / month of a day count: year(d) - 1970 and (year(d) - 1970) * 12 + month(d) - 1 (so 1969-12-31 is -1 and -1)
__host__ __device__ __forceinline__ int64_t years_of_days(int64_t d) { int64_t y; uint32_t m; civil_from_days(d, &y, &m); return y - 1970; }
__host__ __device__ __forceinline__ int64_t months_of_days(int64_t d) { int64_t y; uint32_t m; civil_from_days(d, &y, &m); return (y - 1970) * 12 + (int64_t)m - 1; }
__host__ __device__ __forceinline__ int64_t days_of_micros(int64_t us) { return floor_div(us, kMicrosPerDay); }
__host__ __device__ __forceinline__ int64_t hours_of_micros(int64_t us) { return floor_div(us, kMicrosPerHour); }

}  // namespace etl_ice
