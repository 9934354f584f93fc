// rowbinary_format.cuh — the value formatters of the ClickHouse RowBinary emitter (rowbinary_emit.cu) that
// arrow_format.cuh does not already have.  Plain device functions: tests/emul/host_rowbinary.cpp compiles this same file
// for the host so that the CPU suite can fuzz it against a Python restatement (tests/clickhouse_ref.py).
//   * LEB128 lengths (rb_varint, crates/etl-destinations/src/clickhouse/encoding.rs:176-187);
//   * chrono NaiveTime's Display (the String a Time cell becomes, encoding.rs:61);
//   * lowercase hex (bytes_to_hex, encoding.rs:162-172);
//   * the Date32 range check (date_to_date32_days, encoding.rs:131-148);
//   * the UUID wire order (rb_encode_value, encoding.rs:230-237).
// The DuckLake emitter's variants sit next to the functions they vary: the fixed 6-digit time fraction and uppercase hex.
#pragma once
#include <stdint.h>

namespace etl_rb {

// LEB128: 7 bits per byte, low bits first, the high bit set on every byte but the last
__device__ __forceinline__ uint32_t varint_len(uint64_t v) {
  uint32_t n = 1;
  while (v >= 0x80u) { v >>= 7; n++; }
  return n;
}
__device__ __forceinline__ uint32_t varint_write(uint64_t v, uint8_t* out) {
  uint32_t n = 0;
  while (v >= 0x80u) { out[n++] = (uint8_t)(v | 0x80u); v >>= 7; }
  out[n++] = (uint8_t)v;
  return n;
}

// NaiveTime's Display: "HH:MM:SS", then ".mmm" / ".uuuuuu" / ".nnnnnnnnn" when the nanoseconds are divisible by 10^6 /
// by 10^3 / neither, nothing when they are 0.  A nanosecond value >= 10^9 is chrono's leap-second representation
// (the decoder stores :60 that way): second 59 + 1 = 60, the fraction is what is left above 10^9.
constexpr uint32_t kNanos = 1000000000u;
__device__ __forceinline__ uint32_t time_frac_digits(uint32_t nanos) {
  if (nanos >= kNanos) nanos -= kNanos;
  return nanos == 0u ? 0u : (nanos % 1000000u == 0u ? 3u : (nanos % 1000u == 0u ? 6u : 9u));
}
__device__ __forceinline__ uint32_t time_len(uint32_t nanos) {
  const uint32_t d = time_frac_digits(nanos);
  return 8u + (d ? d + 1u : 0u);
}
__device__ __forceinline__ void put2(uint32_t v, uint8_t* out) { out[0] = (uint8_t)('0' + v / 10u); out[1] = (uint8_t)('0' + v % 10u); }
__device__ __forceinline__ uint32_t time_write(uint64_t secs, uint32_t nanos, uint8_t* out) {
  uint32_t sec = (uint32_t)(secs % 60u);
  if (nanos >= kNanos) { sec += 1u; nanos -= kNanos; }
  put2((uint32_t)(secs / 3600u), out);
  out[2] = ':';
  put2((uint32_t)(secs / 60u % 60u), out + 3);
  out[5] = ':';
  put2(sec, out + 6);
  const uint32_t d = time_frac_digits(nanos);
  if (!d) return 8u;
  out[8] = '.';
  uint32_t f = d == 3u ? nanos / 1000000u : (d == 6u ? nanos / 1000u : nanos);
  for (uint32_t k = d; k > 0; k--) { out[8 + k] = (uint8_t)('0' + f % 10u); f /= 10u; }
  return 9u + d;
}
// chrono's "%H:%M:%S%.6f" (the DuckLake TIME / TIMESTAMP literals): always 6 fraction digits, truncated; a leap second
// is second 60 as above.  15 bytes
constexpr uint32_t kTime6Len = 15;
__device__ __forceinline__ uint32_t time6_write(uint64_t secs, uint32_t nanos, uint8_t* out) {
  uint32_t sec = (uint32_t)(secs % 60u);
  if (nanos >= kNanos) { sec += 1u; nanos -= kNanos; }
  put2((uint32_t)(secs / 3600u), out);
  out[2] = ':';
  put2((uint32_t)(secs / 60u % 60u), out + 3);
  out[5] = ':';
  put2(sec, out + 6);
  out[8] = '.';
  uint32_t f = nanos / 1000u;
  for (uint32_t k = 6; k > 0; k--) { out[8 + k] = (uint8_t)('0' + f % 10u); f /= 10u; }
  return kTime6Len;
}

// lowercase hex, two characters per byte
__device__ __forceinline__ void hex_byte(uint8_t b, uint8_t* out) {
  const uint32_t hi = b >> 4, lo = b & 15u;
  out[0] = (uint8_t)(hi < 10u ? '0' + hi : 'a' - 10u + hi);
  out[1] = (uint8_t)(lo < 10u ? '0' + lo : 'a' - 10u + lo);
}
__device__ __forceinline__ void hex_write(const uint8_t* src, uint32_t n, uint8_t* out) {
  for (uint32_t i = 0; i < n; i++) hex_byte(src[i], out + 2 * i);
}
// uppercase hex (DuckLake's from_hex literal, encode_hex in crates/etl-destinations/src/ducklake/encoding.rs)
__device__ __forceinline__ void hex_byte_upper(uint8_t b, uint8_t* out) {
  const uint32_t hi = b >> 4, lo = b & 15u;
  out[0] = (uint8_t)(hi < 10u ? '0' + hi : 'A' - 10u + hi);
  out[1] = (uint8_t)(lo < 10u ? '0' + lo : 'A' - 10u + lo);
}

// Date32 holds 1900-01-01 ..= 2299-12-31: days -25567 ..= 120529 from 1970-01-01
constexpr int64_t kDate32Min = -25567, kDate32Max = 120529;
__device__ __forceinline__ bool date32_ok(int64_t days) { return days >= kDate32Min && days <= kDate32Max; }

// a UUID's 16 big-endian bytes read as a u128: the high u64 little-endian, then the low u64 little-endian
__device__ __forceinline__ void uuid_write(const uint8_t* be, uint8_t* out) {
  for (int k = 0; k < 8; k++) { out[k] = be[7 - k]; out[8 + k] = be[15 - k]; }
}

// little-endian store of the low `n` bytes of v (the output is byte-addressed: a cell starts anywhere)
__device__ __forceinline__ void le_write(uint64_t v, uint32_t n, uint8_t* out) {
  for (uint32_t k = 0; k < n; k++) { out[k] = (uint8_t)v; v >>= 8; }
}

}  // namespace etl_rb
