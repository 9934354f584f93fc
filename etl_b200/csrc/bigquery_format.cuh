// bigquery_format.cuh — the wire rules and value formatters of the BigQuery Storage Write emitter (bigquery_emit.cu)
// that arrow_format.cuh and rowbinary_format.cuh do not already have.  Plain device functions: tests/emul/
// host_bigquery.cpp compiles this same file for the host so that the CPU suite can fuzz it against a Python restatement
// (tests/bigquery_ref.py).
//   * protobuf field keys and the int32 / int64 / uint32 varints prost writes (crates/etl-destinations/src/bigquery/
//     encoding.rs:151-342; the varint itself is etl_rb::varint_*);
//   * chrono's `%Y-%m-%d` of a NaiveDate and `%Y-%m-%d %H:%M:%S%.f` of a NaiveDateTime (DATE_FORMAT / TIMESTAMP_FORMAT,
//     etl-postgres/src/types/time.rs), TIMESTAMPTZ_FORMAT_HH_MM with `+00:00`;
//   * a Uuid's Display (lowercase, hyphenated);
//   * the two value checks of validate_cell_for_bigquery (validation.rs:11-170): a Numeric's Display with more than 38
//     fractional digits, a Json integer literal outside i64 / u64.
#pragma once
#include <stdint.h>

#include "etl_decode.h"
#include "rowbinary_format.cuh"

namespace etl_bq {

enum : uint32_t { kWtVarint = 0, kWtI64 = 1, kWtLen = 2, kWtI32 = 5 };
// varint(field << 3 | wire_type)
__device__ __forceinline__ uint32_t key_len(uint32_t field) { return etl_rb::varint_len((uint64_t)field << 3); }
__device__ __forceinline__ uint32_t key_write(uint32_t field, uint32_t wt, uint8_t* out) {
  return etl_rb::varint_write((uint64_t)field << 3 | wt, out);
}

// ------------------------------------------------------------------------------------------------ dates
// days since 1970-01-01 → proleptic Gregorian (year, month, day), any int64 day count the decoder produces
__device__ __forceinline__ void civil_from_days(int64_t days, int64_t* y, uint32_t* m, uint32_t* d) {
  const int64_t z = days + 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const uint64_t doe = (uint64_t)(z - era * 146097);
  const uint64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const uint64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint64_t mp = (5 * doy + 2) / 153;
  *d = (uint32_t)(doy - (153 * mp + 2) / 5 + 1);
  *m = (uint32_t)(mp < 10 ? mp + 3 : mp - 9);
  *y = (int64_t)yoe + era * 400 + (*m <= 2 ? 1 : 0);
}
// chrono's %Y: years 0..=9999 as 4 digits, any other year with its sign and at least 4 digits
__device__ __forceinline__ uint32_t year_len(int64_t y) {
  if (y >= 0 && y <= 9999) return 4u;
  uint64_t a = y < 0 ? (uint64_t)(-y) : (uint64_t)y;
  uint32_t n = 0;
  while (a) { n++; a /= 10u; }
  return 1u + (n < 4u ? 4u : n);
}
__device__ __forceinline__ uint32_t year_write(int64_t y, uint8_t* out) {
  const uint32_t n = year_len(y);
  uint32_t o = 0;
  if (n != 4u || y < 0) out[o++] = (uint8_t)(y < 0 ? '-' : '+');
  uint64_t a = y < 0 ? (uint64_t)(-y) : (uint64_t)y;
  for (uint32_t k = n; k > o; k--) { out[k - 1] = (uint8_t)('0' + a % 10u); a /= 10u; }
  return n;
}
__device__ __forceinline__ uint32_t date_len(int64_t days) {
  int64_t y; uint32_t m, d;
  civil_from_days(days, &y, &m, &d);
  return year_len(y) + 6u;
}
__device__ __forceinline__ uint32_t date_write(int64_t days, uint8_t* out) {
  int64_t y; uint32_t m, d;
  civil_from_days(days, &y, &m, &d);
  uint32_t o = year_write(y, out);
  out[o] = '-';
  etl_rb::put2(m, out + o + 1);
  out[o + 3] = '-';
  etl_rb::put2(d, out + o + 4);
  return o + 6u;
}

// ------------------------------------------------------------------------------------------------ timestamps
// (seconds since the epoch, nanoseconds) → "date time[.f]", and "+00:00" for a TimestampTz
__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) { return a / b - ((a % b != 0) && ((a < 0) != (b < 0))); }
__device__ __forceinline__ uint32_t timestamp_len(int64_t secs, uint32_t nanos, bool tz) {
  return date_len(floor_div(secs, 86400)) + 1u + etl_rb::time_len(nanos) + (tz ? 6u : 0u);
}
__device__ __forceinline__ uint32_t timestamp_write(int64_t secs, uint32_t nanos, bool tz, uint8_t* out) {
  const int64_t days = floor_div(secs, 86400);
  uint32_t o = date_write(days, out);
  out[o++] = ' ';
  o += etl_rb::time_write((uint64_t)(secs - days * 86400), nanos, out + o);
  if (tz) {
    const char* z = "+00:00";
    for (uint32_t k = 0; k < 6u; k++) out[o + k] = (uint8_t)z[k];
    o += 6u;
  }
  return o;
}

// ------------------------------------------------------------------------------------------------ uuid
constexpr uint32_t kUuidLen = 36;
__device__ __forceinline__ void uuid_text_write(const uint8_t* be, uint8_t* out) {
  uint32_t o = 0;
  for (uint32_t k = 0; k < 16u; k++) {
    if (k == 4u || k == 6u || k == 8u || k == 10u) out[o++] = '-';
    etl_rb::hex_byte(be[k], out + o);
    o += 2u;
  }
}

// ------------------------------------------------------------------------------------------------ checks
// validate_numeric_for_bigquery: a Value whose Display has more than 38 fractional digits (zero prints as "0")
constexpr uint32_t kMaxScale = 38;
__device__ __forceinline__ bool numeric_scale_bad(const uint8_t* num, uint32_t nd) {
  const etl_numeric_hdr h = *reinterpret_cast<const etl_numeric_hdr*>(num);
  return h.kind == 0 && nd != 0 && h.scale > kMaxScale;
}
// validate_json_number_for_bigquery over every number token of a Json text (outside strings): an integer literal (no
// '.', 'e', 'E') outside i64 when it starts with '-', outside u64 otherwise
__device__ __forceinline__ bool json_int_token_bad(const uint8_t* t, uint32_t n) {
  for (uint32_t k = 0; k < n; k++) if (t[k] == '.' || t[k] == 'e' || t[k] == 'E') return false;
  const bool neg = n && t[0] == '-';
  uint32_t k = neg ? 1u : 0u;
  while (k + 1u < n && t[k] == '0') k++;            // leading zeros do not count toward the magnitude
  const char* lim = neg ? "9223372036854775808" : "18446744073709551615";
  const uint32_t ln = neg ? 19u : 20u, dn = n - k;
  if (dn != ln) return dn > ln;
  for (uint32_t q = 0; q < ln; q++) if (t[k + q] != (uint8_t)lim[q]) return t[k + q] > (uint8_t)lim[q];
  return false;
}
__device__ __forceinline__ bool json_int_bad(const uint8_t* s, uint32_t n) {
  uint32_t i = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c == '"') {                                   // skip the string
      for (i++; i < n && s[i] != '"'; i++) if (s[i] == '\\') i++;
      i++;
    } else if (c == '-' || (c >= '0' && c <= '9')) {
      const uint32_t j = i;
      while (i < n && (s[i] == '-' || s[i] == '+' || s[i] == '.' || s[i] == 'e' || s[i] == 'E' || (s[i] >= '0' && s[i] <= '9'))) i++;
      if (json_int_token_bad(s + j, i - j)) return true;
    } else i++;
  }
  return false;
}

}  // namespace etl_bq
