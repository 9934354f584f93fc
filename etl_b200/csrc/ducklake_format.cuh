// ducklake_format.cuh — the SQL-literal formatters of the DuckLake emitter (ducklake_emit.cu) that arrow_format.cuh,
// rowbinary_format.cuh and bigquery_format.cuh do not already have.  Plain device functions: tests/emul/
// host_ducklake.cpp compiles this same file for the host so that the CPU suite can fuzz it against a Python
// restatement (tests/ducklake_ref.py).  crates/etl-destinations/src/ducklake/encoding.rs:28-272:
//   * the shortest round-trip digits of a double (Rust's f64 Display: positional, never an exponent, no ".0", "-0"),
//     by Schubfach (R. Giulietti, "The Schubfach way to render doubles", 2020) over kSchubfachG, which
//     tools/gen_float_tables.py generates; an F32 is printed as `f as f64`.  Rust's shortest digits are taken to be
//     those of Python's repr (both are the shortest string that reads back, the closest one on a tie); no Rust
//     toolchain checked that;
//   * float_literal: NaN / ±Infinity as CAST('…' AS DOUBLE | FLOAT);
//   * pg_escape::quote_literal (third-party, 0.1.1, its source is not in the reference, so parity is unpinned):
//     wrap in ', double every ' and \, prefix E when the text holds a \;
//   * integers in decimal, and the fixed parts of the DATE / TIME / TIMESTAMP / TIMESTAMPTZ / UUID / from_hex literals.
#pragma once
#include <stdint.h>

#include "rowbinary_format.cuh"
#include "bigquery_format.cuh"
#include "float_print_tables.cuh"

namespace etl_dl {

// ------------------------------------------------------------------------------------------------ integers
__device__ __forceinline__ uint32_t dec_len(uint64_t a) {
  uint32_t n = 1;
  while (a >= 10u) { a /= 10u; n++; }
  return n;
}
__device__ __forceinline__ void dec_write(uint64_t a, uint32_t n, uint8_t* out) {
  for (uint32_t k = n; k > 0; k--) { out[k - 1] = (uint8_t)('0' + a % 10u); a /= 10u; }
}
__device__ __forceinline__ uint64_t abs64(int64_t v) { return v < 0 ? 0ull - (uint64_t)v : (uint64_t)v; }
__device__ __forceinline__ uint32_t int_len(int64_t v) { return (v < 0 ? 1u : 0u) + dec_len(abs64(v)); }
__device__ __forceinline__ uint32_t int_write(int64_t v, uint8_t* out) {
  uint32_t o = 0;
  if (v < 0) out[o++] = '-';
  const uint32_t n = dec_len(abs64(v));
  dec_write(abs64(v), n, out + o);
  return o + n;
}

// ------------------------------------------------------------------------------------------------ shortest digits
__device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
__device__ __forceinline__ int flog10pow2(int q) { return (int)(((int64_t)q * 661971961083ll) >> 41); }
__device__ __forceinline__ int flog10three_quarters_pow2(int q) { return (int)(((int64_t)q * 661971961083ll - 274743187321ll) >> 41); }
__device__ __forceinline__ int flog2pow10(int e) { return (int)(((int64_t)e * 913124641741ll) >> 38); }
// round-to-odd of g * cp / 2^126 (g = g1 2^63 + g0)
__device__ __forceinline__ uint64_t rop(uint64_t g1, uint64_t g0, uint64_t cp) {
  constexpr uint64_t kMask63 = 0x7fffffffffffffffull;
  const uint64_t x1 = mulhi64(g0, cp);
  const uint64_t y0 = g1 * cp;
  const uint64_t y1 = mulhi64(g1, cp);
  const uint64_t z = (y0 >> 1) + x1;
  const uint64_t vbp = y1 + (z >> 63);
  return vbp | (((z & kMask63) + kMask63) >> 63);
}
struct Decimal { uint64_t f; int32_t e; };   // f * 10^e, f without trailing zeros
// Schubfach's toDecimal for c * 2^q (dk: a decimal exponent adjustment, 0 here)
__device__ __forceinline__ Decimal schubfach(int q, uint64_t c, int dk) {
  constexpr uint64_t kCMin = 1ull << 52;
  constexpr int kQMin = -1074;
  const uint64_t out = c & 1u;
  const uint64_t cb = c << 2, cbr = cb + 2;
  uint64_t cbl;
  int k;
  if (c != kCMin || q == kQMin) { cbl = cb - 2; k = flog10pow2(q); }
  else { cbl = cb - 1; k = flog10three_quarters_pow2(q); }
  const int h = q + flog2pow10(-k) + 2;
  const uint64_t g1 = etl::kSchubfachG[k - etl::kSchubfachKMin][0], g0 = etl::kSchubfachG[k - etl::kSchubfachKMin][1];
  const uint64_t vb = rop(g1, g0, cb << h), vbl = rop(g1, g0, cbl << h), vbr = rop(g1, g0, cbr << h);
  const uint64_t s = vb >> 2;
  if (s >= 10u) {                       // one digit fewer (Java's guard is s >= 100: it prints at least two digits)
    const uint64_t sp10 = 10u * mulhi64(s, 115292150460684698ull << 4), tp10 = sp10 + 10u;
    const bool upin = vbl + out <= sp10 << 2, wpin = (tp10 << 2) + out <= vbr;
    if (upin != wpin) return Decimal{upin ? sp10 : tp10, k};
  }
  const uint64_t t = s + 1u;
  const bool uin = vbl + out <= s << 2, win = (t << 2) + out <= vbr;
  if (uin != win) return Decimal{uin ? s : t, k + dk};
  const int64_t cmp = (int64_t)(vb - ((s + t) << 1));
  return Decimal{cmp < 0 || (cmp == 0 && (s & 1u) == 0) ? s : t, k + dk};
}
// a finite non-zero double's shortest digits, trailing zeros stripped
__device__ __forceinline__ Decimal shortest(uint64_t bits) {
  const uint64_t t = bits & ((1ull << 52) - 1);
  const int bq = (int)((bits >> 52) & 0x7ffu);
  Decimal d;
  if (bq != 0) {
    const int mq = 1075 - bq;
    const uint64_t c = (1ull << 52) | t;
    if (mq > 0 && mq < 53 && ((c >> mq) << mq) == c) d = Decimal{c >> mq, 0};   // an integer below 2^53
    else d = schubfach(-mq, c, 0);
  } else {
    d = schubfach(-1074, t, 0);   // (Java scales c < 3 by 10 to print two digits; the shortest is one)
  }
  while (d.f % 10u == 0) { d.f /= 10u; d.e++; }
  return d;
}
// Rust's Display of a finite double: the digits laid out around the decimal point, zeros added as needed
__device__ __forceinline__ uint32_t f64_display_len(uint64_t bits) {
  const uint32_t neg = (uint32_t)(bits >> 63);
  if ((bits << 1) == 0) return 1u + neg;
  const Decimal d = shortest(bits);
  const int n = (int)dec_len(d.f), p = n + d.e;
  if (p <= 0) return neg + 2u + (uint32_t)(-p) + (uint32_t)n;
  if (p >= n) return neg + (uint32_t)p;
  return neg + (uint32_t)n + 1u;
}
__device__ __forceinline__ uint32_t f64_display_write(uint64_t bits, uint8_t* out) {
  uint32_t o = 0;
  if (bits >> 63) out[o++] = '-';
  if ((bits << 1) == 0) { out[o] = '0'; return o + 1u; }
  const Decimal d = shortest(bits);
  const int n = (int)dec_len(d.f), p = n + d.e;
  if (p <= 0) {
    out[o++] = '0'; out[o++] = '.';
    for (int k = 0; k < -p; k++) out[o++] = '0';
    dec_write(d.f, (uint32_t)n, out + o);
    return o + (uint32_t)n;
  }
  if (p >= n) {
    dec_write(d.f, (uint32_t)n, out + o);
    o += (uint32_t)n;
    for (int k = n; k < p; k++) out[o++] = '0';
    return o;
  }
  uint8_t* w = out + o;                 // digits, then open the point after p of them
  dec_write(d.f, (uint32_t)n, w);
  for (int k = n; k > p; k--) w[k] = w[k - 1];
  w[p] = '.';
  return o + (uint32_t)n + 1u;
}
__device__ __forceinline__ uint64_t f32_bits_as_f64(uint32_t b) {
  union { uint32_t u; float f; } x;
  x.u = b;
  union { double d; uint64_t u; } y;
  y.d = (double)x.f;
  return y.u;
}
// float_literal: NaN / ±Infinity as a CAST of the text, any other value its Display
__device__ __forceinline__ bool f64_special(uint64_t bits) { return ((bits >> 52) & 0x7ffu) == 0x7ffu; }
__device__ __forceinline__ const char* special_text(uint64_t bits, bool is_double) {
  const bool nan = (bits & ((1ull << 52) - 1)) != 0, neg = bits >> 63;
  if (is_double) return nan ? "CAST('NaN' AS DOUBLE)" : (neg ? "CAST('-Infinity' AS DOUBLE)" : "CAST('Infinity' AS DOUBLE)");
  return nan ? "CAST('NaN' AS FLOAT)" : (neg ? "CAST('-Infinity' AS FLOAT)" : "CAST('Infinity' AS FLOAT)");
}
__device__ __forceinline__ uint32_t cstr_len(const char* s) { uint32_t n = 0; while (s[n]) n++; return n; }
__device__ __forceinline__ uint32_t cstr_write(const char* s, uint8_t* out) { uint32_t n = 0; while (s[n]) { out[n] = (uint8_t)s[n]; n++; } return n; }
__device__ __forceinline__ uint32_t float_lit_len(uint64_t bits, bool is_double) {
  return f64_special(bits) ? cstr_len(special_text(bits, is_double)) : f64_display_len(bits);
}
__device__ __forceinline__ uint32_t float_lit_write(uint64_t bits, bool is_double, uint8_t* out) {
  return f64_special(bits) ? cstr_write(special_text(bits, is_double), out) : f64_display_write(bits, out);
}

// ------------------------------------------------------------------------------------------------ quote_literal
__device__ __forceinline__ bool quote_esc(uint8_t b) { return b == '\'' || b == '\\'; }
// its length; *bs = the text holds a backslash
__device__ __forceinline__ uint32_t quote_len(const uint8_t* s, uint32_t n, bool* bs) {
  uint32_t extra = 0;
  bool b = false;
  for (uint32_t k = 0; k < n; k++) { extra += quote_esc(s[k]) ? 1u : 0u; b = b || s[k] == '\\'; }
  *bs = b;
  return n + extra + 2u + (b ? 1u : 0u);
}
__device__ __forceinline__ uint32_t quote_write(const uint8_t* s, uint32_t n, uint8_t* out) {
  bool b = false;
  for (uint32_t k = 0; k < n && !b; k++) b = s[k] == '\\';
  uint32_t o = 0;
  if (b) out[o++] = 'E';
  out[o++] = '\'';
  for (uint32_t k = 0; k < n; k++) {
    out[o++] = s[k];
    if (quote_esc(s[k])) out[o++] = s[k];
  }
  out[o++] = '\'';
  return o;
}

// ------------------------------------------------------------------------------------------------ fixed literal parts
// DATE 'Y-m-d'
__device__ __forceinline__ uint32_t date_lit_len(int64_t days) { return 7u + etl_bq::date_len(days); }
__device__ __forceinline__ uint32_t date_lit_write(int64_t days, uint8_t* out) {
  uint32_t o = cstr_write("DATE '", out);
  o += etl_bq::date_write(days, out + o);
  out[o++] = '\'';
  return o;
}
// TIME 'HH:MM:SS.ffffff'
constexpr uint32_t kTimeLitLen = 7u + etl_rb::kTime6Len;
__device__ __forceinline__ uint32_t time_lit_write(uint64_t secs, uint32_t nanos, uint8_t* out) {
  uint32_t o = cstr_write("TIME '", out);
  o += etl_rb::time6_write(secs, nanos, out + o);
  out[o++] = '\'';
  return o;
}
// TIMESTAMP 'Y-m-d HH:MM:SS.ffffff' / TIMESTAMPTZ '…+00:00'
__device__ __forceinline__ uint32_t ts_lit_len(int64_t secs, bool tz) {
  return (tz ? 13u : 11u) + etl_bq::date_len(etl_bq::floor_div(secs, 86400)) + 1u + etl_rb::kTime6Len + (tz ? 6u : 0u) + 1u;
}
__device__ __forceinline__ uint32_t ts_lit_write(int64_t secs, uint32_t nanos, bool tz, uint8_t* out) {
  uint32_t o = cstr_write(tz ? "TIMESTAMPTZ '" : "TIMESTAMP '", out);
  const int64_t days = etl_bq::floor_div(secs, 86400);
  o += etl_bq::date_write(days, out + o);
  out[o++] = ' ';
  o += etl_rb::time6_write((uint64_t)(secs - days * 86400), nanos, out + o);
  if (tz) o += cstr_write("+00:00", out + o);
  out[o++] = '\'';
  return o;
}
// CAST('<uuid>' AS UUID)
constexpr uint32_t kUuidLitLen = 16u + etl_bq::kUuidLen;
__device__ __forceinline__ uint32_t uuid_lit_write(const uint8_t* be, uint8_t* out) {
  uint32_t o = cstr_write("CAST('", out);
  etl_bq::uuid_text_write(be, out + o);
  o += etl_bq::kUuidLen;
  return o + cstr_write("' AS UUID)", out + o);
}
// from_hex('<UPPERCASE hex>')
__device__ __forceinline__ uint64_t bytes_lit_len(uint32_t n) { return 12ull + 2ull * n; }
__device__ __forceinline__ uint32_t bytes_lit_write(const uint8_t* s, uint32_t n, uint8_t* out) {
  uint32_t o = cstr_write("from_hex('", out);
  for (uint32_t k = 0; k < n; k++) etl_rb::hex_byte_upper(s[k], out + o + 2 * k);
  o += 2 * n;
  return o + cstr_write("')", out + o);
}

// ------------------------------------------------------------------------------------------------ FNV-1a 64 (BatchIdHasher)
constexpr uint64_t kFnvBasis = 0xcbf29ce484222325ull, kFnvPrime = 0x100000001b3ull;
__device__ __forceinline__ uint64_t fnv_byte(uint64_t h, uint8_t b) { return (h ^ b) * kFnvPrime; }
__device__ __forceinline__ uint64_t fnv_bytes(uint64_t h, const uint8_t* p, uint64_t n) {
  uint64_t k = 0;
  for (; k < n && ((uintptr_t)(p + k) & 7u); k++) h = fnv_byte(h, p[k]);
  for (; k + 8 <= n; k += 8) {                       // aligned 8-byte loads
    uint64_t w = *reinterpret_cast<const uint64_t*>(p + k);
    for (int j = 0; j < 8; j++) { h = fnv_byte(h, (uint8_t)w); w >>= 8; }
  }
  for (; k < n; k++) h = fnv_byte(h, p[k]);
  return h;
}
// Hash for str: the bytes, then 0xff; for u64 / usize: 8 bytes little-endian
__device__ __forceinline__ uint64_t fnv_str(uint64_t h, const uint8_t* p, uint64_t n) { return fnv_byte(fnv_bytes(h, p, n), 0xffu); }
__device__ __forceinline__ uint64_t fnv_u64(uint64_t h, uint64_t v) {
  for (int j = 0; j < 8; j++) { h = fnv_byte(h, (uint8_t)v); v >>= 8; }
  return h;
}
__device__ __forceinline__ uint64_t fnv_cstr(uint64_t h, const char* s) { return fnv_str(h, reinterpret_cast<const uint8_t*>(s), cstr_len(s)); }

}  // namespace etl_dl
