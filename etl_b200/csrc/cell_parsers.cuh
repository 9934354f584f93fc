// cell_parsers.cuh — device-side Postgres text → typed Cell parsers (sm_90a).
//
// Each parser is the GPU counterpart of one arm of parse_cell_from_postgres_text
// (crates/etl/src/conversions/text.rs:28-173) and takes the cell's bytes through a generic pointer
// (shared-memory tile window or global memory for oversize frames).  Integer / byte arithmetic
// only; results must be bit-identical to the reference (the CPU oracle checks that in tests/).
#pragma once
#include <stdint.h>

#include "etl_decode.h"

#include "json_tables.cuh"
namespace etl {

struct CellOut {
  uint64_t val;
  uint32_t aux;
  uint32_t tag;
};

// bump allocator over the frame's pre-sized heap slice
struct HeapCursor {
  uint8_t* heap;   // batch heap base (global)
  uint64_t pos;    // next free byte (8-aligned)
  __device__ __forceinline__ uint64_t alloc(uint32_t nbytes) {
    uint64_t off = pos;
    pos += (uint64_t)((nbytes + 7u) & ~7u);
    return off;
  }
};

__device__ __forceinline__ bool is_digit(uint32_t c) { return (c - '0') <= 9u; }
__device__ __forceinline__ uint32_t lower(uint32_t c) { return (c - 'A') <= 25u ? c + 32u : c; }
__device__ __forceinline__ int hexval(uint32_t c) {
  if ((c - '0') <= 9u) return (int)(c - '0');
  c = lower(c);
  if ((c - 'a') <= 5u) return (int)(c - 'a' + 10);
  return -1;
}
__device__ __forceinline__ bool ieq(const uint8_t* s, uint32_t n, const char* lit, uint32_t m) {
  if (n != m) return false;
  for (uint32_t i = 0; i < n; i++)
    if (lower(s[i]) != (uint32_t)(uint8_t)lit[i]) return false;
  return true;
}

// ------------------------------------------------------------------------------------------------
// UTF-8 validation (core::str::from_utf8, event.rs:972).  Position-local formulation: byte i is
// checked against its three predecessors, so any chunking of a cell gives the same verdict; the
// block-cooperative path for large cells uses the same function on 16-byte chunks.
__device__ __forceinline__ bool utf8_step_bad(uint32_t b, uint32_t p1, uint32_t p2, uint32_t p3) {
  bool must_cont = (p1 >= 0xC0u) || (p2 >= 0xE0u) || (p3 >= 0xF0u);
  bool is_cont = (b & 0xC0u) == 0x80u;
  if (must_cont != is_cont) return true;
  if (p1 >= 0xC0u) {  // b is the first continuation byte of a sequence: range restrictions
    if (p1 < 0xC2u) return true;                  // overlong 2-byte
    if (p1 == 0xE0u && b < 0xA0u) return true;    // overlong 3-byte
    if (p1 == 0xEDu && b >= 0xA0u) return true;   // surrogates
    if (p1 == 0xF0u && b < 0x90u) return true;    // overlong 4-byte
    if (p1 == 0xF4u && b >= 0x90u) return true;   // > U+10FFFF
    if (p1 > 0xF4u) return true;
  }
  return false;
}
// validate bytes [lo, hi) of a cell of n bytes (lo..hi chunk; predecessors read from the cell)
__device__ __forceinline__ bool utf8_chunk_valid(const uint8_t* s, uint32_t n, uint32_t lo, uint32_t hi) {
  uint32_t p1 = lo >= 1 ? s[lo - 1] : 0, p2 = lo >= 2 ? s[lo - 2] : 0, p3 = lo >= 3 ? s[lo - 3] : 0;
  bool bad = false;
  for (uint32_t i = lo; i < hi; i++) {
    uint32_t b = s[i];
    bad |= utf8_step_bad(b, p1, p2, p3);
    p3 = p2; p2 = p1; p1 = b;
  }
  if (hi == n) bad |= (p1 >= 0xC0u) || (p2 >= 0xE0u) || (p3 >= 0xF0u);  // truncated tail sequence
  return !bad;
}
// the same over stream positions [lo, hi) with 64-bit offsets (k_utf8_lines: the "cell" is the whole stream)
__device__ __forceinline__ bool utf8_chunk_valid_at(const uint8_t* s, uint64_t n, uint64_t lo, uint64_t hi) {
  uint32_t p1 = lo >= 1 ? s[lo - 1] : 0, p2 = lo >= 2 ? s[lo - 2] : 0, p3 = lo >= 3 ? s[lo - 3] : 0;
  bool bad = false;
  for (uint64_t i = lo; i < hi; i++) {
    uint32_t b = s[i];
    bad |= utf8_step_bad(b, p1, p2, p3);
    p3 = p2; p2 = p1; p1 = b;
  }
  if (hi == n) bad |= (p1 >= 0xC0u) || (p2 >= 0xE0u) || (p3 >= 0xF0u);
  return !bad;
}
__device__ __forceinline__ bool utf8_valid(const uint8_t* s, uint32_t n) {
  // ASCII fast path per byte; multi-byte handled by the local rule
  uint32_t p1 = 0, p2 = 0, p3 = 0;
  bool bad = false;
  for (uint32_t i = 0; i < n; i++) {
    uint32_t b = s[i];
    if ((b | p1 | p2 | p3) >= 0x80u) bad |= utf8_step_bad(b, p1, p2, p3);
    p3 = p2; p2 = p1; p1 = b;
  }
  bad |= (p1 >= 0xC0u) || (p2 >= 0xE0u) || (p3 >= 0xF0u);
  return !bad;
}

// Unicode White_Space (char::is_whitespace) byte length at s, 0 if none. Input is valid UTF-8.
__device__ __forceinline__ uint32_t ws_len(const uint8_t* s, uint32_t n) {
  if (n == 0) return 0;
  uint32_t b = s[0];
  if (b == ' ' || (b - 9u) <= 4u) return 1;
  if (b < 0xC2u) return 0;
  if (b == 0xC2u && n >= 2 && (s[1] == 0x85 || s[1] == 0xA0)) return 2;
  if (n >= 3) {
    uint32_t c1 = s[1], c2 = s[2];
    if (b == 0xE1u && c1 == 0x9A && c2 == 0x80) return 3;
    if (b == 0xE2u && c1 == 0x80 && ((c2 - 0x80u) <= 0x0Au || c2 == 0xA8 || c2 == 0xA9 || c2 == 0xAF)) return 3;
    if (b == 0xE2u && c1 == 0x81 && c2 == 0x9F) return 3;
    if (b == 0xE3u && c1 == 0x80 && c2 == 0x80) return 3;
  }
  return 0;
}
struct Cur {
  const uint8_t* s;
  uint32_t n;
  __device__ __forceinline__ void trim_start() {
    uint32_t w;
    while ((w = ws_len(s, n)) != 0) { s += w; n -= w; }
  }
  __device__ __forceinline__ bool lit(uint32_t ch) {
    if (n < 1 || s[0] != ch) return false;
    s++; n--; return true;
  }
};

// ------------------------------------------------------------------------------------------------
// integers: Rust FromStr (text.rs:49-60,159-161)
__device__ __forceinline__ uint32_t parse_int(const uint8_t* s, uint32_t n, bool is_signed, uint64_t pos_limit,
                                              uint64_t neg_limit, int64_t* out) {
  if (n == 0) return ETL_E_PARSE_INT;
  bool neg = false;
  uint32_t i = 0;
  uint32_t c0 = s[0];
  if (c0 == '+') i = 1;
  else if (c0 == '-') { if (!is_signed) return ETL_E_PARSE_INT; neg = true; i = 1; }
  if (i == n) return ETL_E_PARSE_INT;
  uint64_t limit = neg ? neg_limit : pos_limit;
  uint64_t acc = 0;
  for (; i < n; i++) {
    uint32_t d = (uint32_t)s[i] - '0';
    if (d > 9u) return ETL_E_PARSE_INT;
    if (acc > (limit - d) / 10u) return ETL_E_PARSE_INT;
    acc = acc * 10u + d;
  }
  *out = neg ? (int64_t)(0ull - acc) : (int64_t)acc;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// chrono 0.4 parse_from_str (formats etl-postgres/src/types/time.rs:7-21)
__device__ __forceinline__ bool scan_number(Cur& c, uint32_t minw, uint32_t maxw, int64_t* out) {
  uint32_t k = 0;
  int64_t v = 0;
  while (k < c.n && k < maxw && is_digit(c.s[k])) {
    int d = c.s[k] - '0';
    if (v > (INT64_MAX - d) / 10) return false;
    v = v * 10 + d;
    k++;
  }
  if (k < minw) return false;
  c.s += k; c.n -= k; *out = v;
  return true;
}
__device__ __forceinline__ bool num_field(Cur& c, uint32_t width, bool is_signed, int64_t* out) {
  c.trim_start();
  if (is_signed && c.n > 0 && c.s[0] == '-') {
    c.s++; c.n--;
    int64_t v;
    if (!scan_number(c, 1, 0xFFFFFFFFu, &v)) return false;
    *out = -v; return true;
  }
  if (is_signed && c.n > 0 && c.s[0] == '+') {
    c.s++; c.n--;
    return scan_number(c, 1, 0xFFFFFFFFu, out);
  }
  return scan_number(c, 1, width, out);
}
__device__ __forceinline__ int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {
  y -= m <= 2;
  int64_t era = (y >= 0 ? y : y - 399) / 400;
  int64_t yoe = y - era * 400;
  int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}
__device__ __forceinline__ bool parse_date_part(Cur& c, int64_t* days) {
  int64_t y, m, d;
  if (!num_field(c, 4, true, &y)) return false;
  if (y < INT32_MIN || y > INT32_MAX) return false;
  if (!c.lit('-')) return false;
  if (!num_field(c, 2, false, &m) || m < 1 || m > 12) return false;
  if (!c.lit('-')) return false;
  if (!num_field(c, 2, false, &d) || d < 1 || d > 31) return false;
  if (y < -262143 || y > 262142) return false;
  int dim = (m == 2) ? (((y % 4 == 0 && y % 100 != 0) || y % 400 == 0) ? 29 : 28)
                     : ((m == 4 || m == 6 || m == 9 || m == 11) ? 30 : 31);
  if (d > dim) return false;
  *days = days_from_civil(y, m, d);
  return true;
}
__device__ __forceinline__ bool parse_time_part(Cur& c, int64_t* secs, uint32_t* nanos) {
  int64_t h, mi, se;
  if (!num_field(c, 2, false, &h) || h > 23) return false;
  if (!c.lit(':')) return false;
  if (!num_field(c, 2, false, &mi) || mi > 59) return false;
  if (!c.lit(':')) return false;
  if (!num_field(c, 2, false, &se) || se > 60) return false;
  uint32_t ns = 0;
  if (c.n > 0 && c.s[0] == '.') {
    c.s++; c.n--;
    uint32_t before = c.n;
    int64_t v;
    if (!scan_number(c, 1, 9, &v)) return false;
    uint32_t consumed = before - c.n;
    for (uint32_t k = consumed; k < 9; k++) v *= 10;
    while (c.n > 0 && is_digit(c.s[0])) { c.s++; c.n--; }
    ns = (uint32_t)v;
  }
  if (se == 60) { se = 59; ns += 1000000000u; }
  *secs = h * 3600 + mi * 60 + se;
  *nanos = ns;
  return true;
}
__device__ __forceinline__ bool parse_tz(Cur& c, bool allow_zulu, bool allow_missing_minutes, int32_t* off) {
  c.trim_start();
  if (allow_zulu && c.n > 0 && (c.s[0] == 'Z' || c.s[0] == 'z')) { c.s++; c.n--; *off = 0; return true; }
  if (c.n == 0) return false;
  bool neg;
  if (c.s[0] == '+') { neg = false; c.s++; c.n--; }
  else if (c.s[0] == '-') { neg = true; c.s++; c.n--; }
  else if (c.n >= 3 && c.s[0] == 0xE2 && c.s[1] == 0x88 && c.s[2] == 0x92) { neg = true; c.s += 3; c.n -= 3; }
  else return false;
  if (c.n < 2 || !is_digit(c.s[0]) || !is_digit(c.s[1])) return false;
  int32_t hours = (c.s[0] - '0') * 10 + (c.s[1] - '0');
  c.s += 2; c.n -= 2;
  for (;;) {
    if (c.n > 0 && c.s[0] == ':') { c.s++; c.n--; continue; }
    uint32_t w = ws_len(c.s, c.n);
    if (w) { c.s += w; c.n -= w; continue; }
    break;
  }
  int32_t minutes;
  if (c.n >= 2) {
    uint32_t m1 = c.s[0], m2 = c.s[1];
    if ((m1 - '0') <= 5u && is_digit(m2)) minutes = (int32_t)((m1 - '0') * 10 + (m2 - '0'));
    else return false;
  } else if (allow_missing_minutes) minutes = 0;
  else return false;
  if (c.n >= 2) { c.s += 2; c.n -= 2; }
  else if (c.n != 0) return false;
  int32_t secs = hours * 3600 + minutes * 60;
  *off = neg ? -secs : secs;
  return true;
}
__device__ __forceinline__ bool parse_ts_prefix(Cur& c, int64_t* days, int64_t* secs, uint32_t* ns) {
  if (!parse_date_part(c, days)) return false;
  c.trim_start();
  return parse_time_part(c, secs, ns);
}
__device__ __noinline__ bool parse_timestamptz_fmt(const uint8_t* s, uint32_t n, bool permissive, CellOut& o) {
  Cur c{s, n};
  int64_t days, secs;
  uint32_t ns;
  int32_t off;
  if (!parse_ts_prefix(c, &days, &secs, &ns)) return false;
  if (!parse_tz(c, permissive, permissive, &off)) return false;
  if (c.n != 0) return false;
  if (off <= -86400 || off >= 86400) return false;
  int64_t utc = days * 86400 + secs - off;
  const int64_t lo = -8334601228800LL;  // days_from_civil(-262143,1,1)*86400
  const int64_t hi = 8210266876800LL;   // (days_from_civil(262142,12,31)+1)*86400
  if (utc < lo || utc >= hi) return false;
  o.tag = ETL_CELL_TIMESTAMPTZ; o.val = (uint64_t)utc; o.aux = ns;
  return true;
}

// ------------------------------------------------------------------------------------------------
// numeric.rs:99-472.  Two passes over the text: grammar + shape, then base-10000 grouping straight
// into the heap slice (no temporaries).
__device__ __noinline__ uint32_t parse_numeric(const uint8_t* s, uint32_t n, HeapCursor& hc, CellOut& o) {
  Cur c{s, n};
  c.trim_start();
  if (c.n == 0) return ETL_E_NUMERIC;
  bool neg = false, explicit_sign = false;
  if (c.s[0] == '+') { explicit_sign = true; c.s++; c.n--; }
  else if (c.s[0] == '-') { neg = true; explicit_sign = true; c.s++; c.n--; }
  etl_numeric_hdr hdr;
  hdr.kind = 0; hdr.sign = 0; hdr.weight = 0; hdr.scale = 0; hdr.pushed_groups = 0;
  const uint8_t* p = c.s;
  uint32_t rem = c.n;
  if (!(rem > 0 && (is_digit(p[0]) || p[0] == '.'))) {
    uint32_t e = rem;
    for (;;) {  // trim_end by Unicode whitespace
      bool trimmed = false;
      for (uint32_t w = 1; w <= 3 && w <= e; w++)
        if (ws_len(p + e - w, w) == w) { e -= w; trimmed = true; break; }
      if (!trimmed) break;
    }
    if (ieq(p, e, "nan", 3)) { if (explicit_sign) return ETL_E_NUMERIC; hdr.kind = 1; }
    else if (ieq(p, e, "infinity", 8) || ieq(p, e, "inf", 3)) hdr.kind = neg ? 3 : 2;
    else return ETL_E_NUMERIC;
    uint64_t off = hc.alloc(8);
    *reinterpret_cast<etl_numeric_hdr*>(hc.heap + off) = hdr;
    o.tag = ETL_CELL_NUMERIC; o.val = off; o.aux = 0;
    return 0;
  }
  // pass 1: grammar (numeric.rs:285-401)
  uint32_t i = 0, ndec = 0;
  bool have_dp = false;
  int64_t dweight = -1, dscale = 0;
  if (p[0] == '.') { have_dp = true; i = 1; }
  if (!(i < rem && is_digit(p[i]))) return ETL_E_NUMERIC;
  uint32_t mant_begin = 0, mant_end;
  while (i < rem) {
    uint32_t ch = p[i];
    if (is_digit(ch)) { i++; ndec++; if (!have_dp) dweight++; else dscale++; }
    else if (ch == '.') {
      if (have_dp) return ETL_E_NUMERIC;
      have_dp = true; i++;
      if (i < rem && p[i] == '_') return ETL_E_NUMERIC;
    } else if (ch == '_') {
      i++;
      if (!(i < rem && is_digit(p[i]))) return ETL_E_NUMERIC;
    } else break;
  }
  mant_end = i;
  if (i < rem && (p[i] == 'e' || p[i] == 'E')) {
    i++;
    int64_t exponent = 0;
    bool eneg = false;
    if (i < rem && p[i] == '+') i++;
    else if (i < rem && p[i] == '-') { eneg = true; i++; }
    if (!(i < rem && is_digit(p[i]))) return ETL_E_NUMERIC;
    while (i < rem) {
      uint32_t ch = p[i];
      if (is_digit(ch)) {
        i++; exponent = exponent * 10 + (int64_t)(ch - '0');
        if (exponent > 2147483647LL / 2) return ETL_E_NUMERIC;
      } else if (ch == '_') {
        i++;
        if (!(i < rem && is_digit(p[i]))) return ETL_E_NUMERIC;
      } else break;
    }
    if (eneg) exponent = -exponent;
    dweight += exponent;
    dscale = (dscale - exponent) < 0 ? 0 : (dscale - exponent);
  }
  { Cur t{p + i, rem - i}; t.trim_start(); if (t.n != 0) return ETL_E_NUMERIC; }
  if (dscale > 16383) return ETL_E_NUMERIC;
  hdr.scale = (uint16_t)dscale;
  // pass 2: convert_to_base_10000 (numeric.rs:409-472)
  int64_t weight = dweight >= 0 ? (dweight + 4) / 4 - 1 : -((-dweight - 1) / 4 + 1);
  int64_t offset = (weight + 1) * 4 - (dweight + 1);
  uint32_t ndig = (uint32_t)(((int64_t)ndec + offset + 3) / 4);
  uint64_t off = hc.alloc(8 + 2 * ndig);
  int16_t* dg = reinterpret_cast<int16_t*>(hc.heap + off + 8);
  uint32_t lead = 0, written = 0, last_nz = 0;
  bool seen_nz = false;
  int v = 0;
  uint32_t pos_in_group = (uint32_t)offset;  // leading pad zeros
  for (uint32_t k = mant_begin; k < mant_end; k++) {
    uint32_t ch = p[k];
    if (!is_digit(ch)) continue;
    v = v * 10 + (int)(ch - '0');
    if (++pos_in_group == 4) {
      if (!seen_nz) { if (v == 0) lead++; else { seen_nz = true; dg[0] = (int16_t)v; written = 1; last_nz = 1; } }
      else { dg[written++] = (int16_t)v; if (v) last_nz = written; }
      v = 0; pos_in_group = 0;
    }
  }
  if (pos_in_group != 0) {
    for (; pos_in_group < 4; pos_in_group++) v *= 10;
    if (!seen_nz) { if (v == 0) lead++; else { seen_nz = true; dg[0] = (int16_t)v; written = 1; last_nz = 1; } }
    else { dg[written++] = (int16_t)v; if (v) last_nz = written; }
  }
  uint32_t nd = 0;
  if (seen_nz) {
    int64_t fw = weight - (int64_t)lead;
    if (fw < -32768 || fw > 32767) return ETL_E_NUMERIC;
    hdr.sign = neg ? 1 : 0;
    hdr.weight = (int16_t)fw;
    nd = last_nz;
    hdr.pushed_groups = (uint16_t)min(ndig, 0xFFFFu);   // groups pushed before the zero strips (Vec capacity, size hints)
  }
  *reinterpret_cast<etl_numeric_hdr*>(hc.heap + off) = hdr;
  o.tag = ETL_CELL_NUMERIC | ((uint32_t)hdr.pushed_groups << 16); o.val = off; o.aux = nd;
  return 0;
}
// heap bytes reserved for a numeric cell of n text bytes (upper bound on 8 + 2*ndigits, 8-aligned)
__device__ __forceinline__ uint32_t numeric_heap_bound(uint32_t n) { return (8u + 2u * (n / 4u + 2u) + 7u) & ~7u; }

// ------------------------------------------------------------------------------------------------
// hex.rs:11-37
__device__ __noinline__ uint32_t parse_bytea(const uint8_t* s, uint32_t n, HeapCursor& hc, CellOut& o) {
  if (n < 2 || s[0] != '\\' || s[1] != 'x') return ETL_E_BYTEA;
  s += 2; n -= 2;
  if (n & 1u) return ETL_E_BYTEA;
  uint64_t off = hc.alloc(n / 2);
  uint8_t* d = hc.heap + off;
  for (uint32_t i = 0; i < n; i += 2) {
    int a, b;
    if (s[i] == '+') { b = hexval(s[i + 1]); if (b < 0) return ETL_E_PARSE_INT; d[i >> 1] = (uint8_t)b; continue; }
    a = hexval(s[i]); b = hexval(s[i + 1]);
    if ((a | b) < 0) return ETL_E_PARSE_INT;
    d[i >> 1] = (uint8_t)(a * 16 + b);
  }
  o.tag = ETL_CELL_BYTES; o.val = off; o.aux = n / 2;
  return 0;
}
__device__ __forceinline__ uint32_t bytea_heap_bound(uint32_t n) { return n >= 2 ? (((n - 2u) / 2u + 7u) & ~7u) : 0u; }

// uuid 1.x Uuid::parse_str (text.rs:141-149)
__device__ __noinline__ uint32_t parse_uuid(const uint8_t* s, uint32_t n, HeapCursor& hc, CellOut& o) {
  uint8_t out[16];
  if (n == 38 && s[0] == '{' && s[37] == '}') { s++; n = 36; }
  else if (n == 45 && s[0] == 'u' && s[1] == 'r' && s[2] == 'n' && s[3] == ':' && s[4] == 'u' && s[5] == 'u' &&
           s[6] == 'i' && s[7] == 'd' && s[8] == ':') { s += 9; n = 36; }
  if (n == 32) {
    for (int i = 0; i < 16; i++) {
      int a = hexval(s[2 * i]), b = hexval(s[2 * i + 1]);
      if ((a | b) < 0) return ETL_E_UUID;
      out[i] = (uint8_t)(a * 16 + b);
    }
  } else if (n == 36) {
    if (s[8] != '-' || s[13] != '-' || s[18] != '-' || s[23] != '-') return ETL_E_UUID;
    int k = 0;
    for (int i = 0; i < 36;) {
      if (i == 8 || i == 13 || i == 18 || i == 23) { i++; continue; }
      int a = hexval(s[i]), b = hexval(s[i + 1]);
      if ((a | b) < 0) return ETL_E_UUID;
      out[k++] = (uint8_t)(a * 16 + b);
      i += 2;
    }
  } else return ETL_E_UUID;
  uint64_t off = hc.alloc(16);
  for (int i = 0; i < 16; i++) hc.heap[off + i] = out[i];
  o.tag = ETL_CELL_UUID; o.val = off; o.aux = 16;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// serde_json::from_str::<Value> acceptance (text.rs:150-153): iterative validator with an explicit
// container stack (1 bit per level, 128 levels = serde_json's recursion limit).
__device__ __noinline__ bool json_valid(const uint8_t* s, uint32_t n) {
  uint32_t stack[4] = {0, 0, 0, 0};  // bit = 1 → object, 0 → array
  int depth = 0;
  uint32_t i = 0;
  // state: 0 expect value, 1 after value, 2 expect key or '}', 3 expect key, 4 expect ':', 5 expect value or ']'
  int st = 0;
  for (;;) {
    while (i < n && (s[i] == ' ' || s[i] == '\t' || s[i] == '\n' || s[i] == '\r')) i++;
    if (st == 1 && depth == 0) return i == n;
    if (i >= n) return false;
    uint32_t ch = s[i];
    if (st == 1) {
      bool is_obj = (stack[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1u;
      if (ch == ',') { i++; st = is_obj ? 3 : 0; continue; }
      if (ch == (is_obj ? '}' : ']')) { i++; depth--; st = 1; continue; }
      return false;
    }
    if (st == 4) { if (ch != ':') return false; i++; st = 0; continue; }
    if (st == 2 || st == 3) {
      if (st == 2 && ch == '}') { i++; depth--; st = 1; continue; }
      if (ch != '"') return false;
      // fallthrough to string parse, then expect ':'
    } else if (st == 5) {
      if (ch == ']') { i++; depth--; st = 1; continue; }
      st = 0;
    }
    if (ch == '"') {
      i++;
      for (;;) {
        if (i >= n) return false;
        uint32_t c = s[i];
        if (c == '"') { i++; break; }
        if (c < 0x20u) return false;
        if (c == '\\') {
          i++;
          if (i >= n) return false;
          uint32_t e = s[i++];
          if (e == 'u') {
            if (i + 4 > n) return false;
            uint32_t u = 0;
            for (int k = 0; k < 4; k++) { int h = hexval(s[i + k]); if (h < 0) return false; u = u * 16 + (uint32_t)h; }
            i += 4;
            if (u >= 0xDC00u && u <= 0xDFFFu) return false;
            if (u >= 0xD800u && u <= 0xDBFFu) {
              if (i + 6 > n || s[i] != '\\' || s[i + 1] != 'u') return false;
              i += 2;
              uint32_t u2 = 0;
              for (int k = 0; k < 4; k++) { int h = hexval(s[i + k]); if (h < 0) return false; u2 = u2 * 16 + (uint32_t)h; }
              i += 4;
              if (u2 < 0xDC00u || u2 > 0xDFFFu) return false;
            }
          } else if (!(e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't')) return false;
          continue;
        }
        i++;
      }
      st = (st == 2 || st == 3) ? 4 : 1;
      continue;
    }
    // st == 0 here: a value
    if (ch == '{' || ch == '[') {
      if (depth >= 127) return false;  // remaining_depth reaches 0 on the 128th nested container
      if (ch == '{') stack[depth >> 5] |= (1u << (depth & 31)); else stack[depth >> 5] &= ~(1u << (depth & 31));
      depth++; i++;
      st = (ch == '{') ? 2 : 5;
      continue;
    }
    if (ch == 't') { if (i + 4 > n || s[i + 1] != 'r' || s[i + 2] != 'u' || s[i + 3] != 'e') return false; i += 4; st = 1; continue; }
    if (ch == 'f') { if (i + 5 > n || s[i + 1] != 'a' || s[i + 2] != 'l' || s[i + 3] != 's' || s[i + 4] != 'e') return false; i += 5; st = 1; continue; }
    if (ch == 'n') { if (i + 4 > n || s[i + 1] != 'u' || s[i + 2] != 'l' || s[i + 3] != 'l') return false; i += 4; st = 1; continue; }
    if (ch == '-' || is_digit(ch)) {
      if (ch == '-') { i++; if (i >= n) return false; }
      if (s[i] == '0') { i++; if (i < n && is_digit(s[i])) return false; }
      else if ((uint32_t)(s[i] - '1') <= 8u) { while (i < n && is_digit(s[i])) i++; }
      else return false;
      if (i < n && s[i] == '.') { i++; if (!(i < n && is_digit(s[i]))) return false; while (i < n && is_digit(s[i])) i++; }
      if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        i++;
        if (i < n && (s[i] == '+' || s[i] == '-')) i++;
        if (!(i < n && is_digit(s[i]))) return false;
        while (i < n && is_digit(s[i])) i++;
      }
      st = 1;
      continue;
    }
    return false;
  }
}


// ================================================================================================
// Warp-synchronous fast paths.  Independent thread scheduling does not reconverge a warp after
// loops that exit through break / return, so the hot parsers are written as loops whose trip is
// voted with __any_sync(mask, ...) (one convergence point per iteration) or as loop-free SWAR
// code.  `mask` = lanes of the warp that execute the same parser together.  Anything outside the
// spellings Postgres itself emits falls back to the exact (divergent, rare) parsers above.

__device__ __forceinline__ uint64_t ldu64(const uint8_t* p) {  // unaligned LE load from aligned words
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(a & 3u) * 8u;
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
  return ((uint64_t)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
}
// 8 ASCII digits (first char in the low byte) → value; valid only if swar_all_digits(x)
__device__ __forceinline__ uint32_t swar_parse8(uint64_t x) {
  x -= 0x3030303030303030ull;
  x = (x * 10ull) + (x >> 8);
  return (uint32_t)((((x & 0x000000FF000000FFull) * 0x000F424000000064ull) +
                     (((x >> 16) & 0x000000FF000000FFull) * 0x0000271000000001ull)) >> 32);
}
__device__ __forceinline__ bool swar_all_digits(uint64_t x) {
  return (((x + 0x4646464646464646ull) | (x - 0x3030303030303030ull)) & 0x8080808080808080ull) == 0ull;
}
// a table in global memory: a local array would be re-materialised (18 stores) by every thread of the cell kernels
__device__ const uint64_t kPow10[9] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull};
__device__ __forceinline__ uint64_t pow10_u64(uint32_t k) { return kPow10[k]; }  // k in 0..8

// Rust FromStr for integers (text.rs:49-60,159-161), 8 digits per step.
__device__ __forceinline__ uint32_t parse_int_sync(unsigned mask, const uint8_t* s, uint32_t n, bool is_signed,
                                                   uint64_t pos_limit, uint64_t neg_limit, int64_t* out) {
  bool bad = n == 0;
  bool neg = false;
  uint32_t i = 0;
  if (n) {
    const uint32_t c0 = s[0];
    if (c0 == '+') i = 1;
    else if (c0 == '-') { if (!is_signed) bad = true; neg = true; i = 1; }
    if (i == n) bad = true;
  }
  uint64_t acc = 0;
  bool ovf = false;
  while (__any_sync(mask, !bad && i < n)) {
    if (!bad && i < n) {
      const uint32_t k = min(8u, n - i);
      uint64_t x = ldu64(s + i);
      // keep the k chars in the high bytes, pad the low bytes with '0' (leading zeros)
      if (k < 8) x = (x << (8u * (8u - k))) | (0x3030303030303030ull >> (8u * k));
      if (!swar_all_digits(x)) bad = true;
      else {
        const uint64_t p10 = pow10_u64(k);
        const uint64_t hi = __umul64hi(acc, p10);
        const uint64_t lo = acc * p10;
        const uint64_t v = (uint64_t)swar_parse8(x);
        const uint64_t sum = lo + v;
        if (hi != 0 || sum < lo) ovf = true;
        acc = sum;
        i += k;
      }
    }
  }
  if (bad || ovf || acc > (neg ? neg_limit : pos_limit)) return ETL_E_PARSE_INT;
  *out = neg ? (int64_t)(0ull - acc) : (int64_t)acc;
  return 0;
}

// "YYYY-MM-DD HH:MM:SS" at s[0..19) → days / seconds of day; false unless it is exactly that shape
__device__ __forceinline__ bool fast_ymd_hms(const uint8_t* s, int64_t* days, int64_t* sod) {
  const uint64_t a = ldu64(s), b = ldu64(s + 8);
  const uint32_t c = (uint32_t)ldu64(s + 16);
  // separators: s[4]='-' s[7]='-' s[10]=' ' s[13]=':' s[16]=':'
  if (((a >> 32) & 0xFFu) != '-' || ((a >> 56) & 0xFFu) != '-' || ((b >> 16) & 0xFFu) != ' ' || ((b >> 40) & 0xFFu) != ':' || (c & 0xFFu) != ':') return false;
  // digits: replace separators by '0' and test all 19 positions
  const uint64_t da = (a & 0x00FFFF00FFFFFFFFull) | 0x3000003000000000ull;
  const uint64_t db = (b & 0xFFFF00FFFF00FFFFull) | 0x0000300000300000ull;
  const uint64_t dc = ((uint64_t)(c & 0x00FFFF00u) | 0x30000030u) | 0x3030303000000000ull;
  if (!swar_all_digits(da) || !swar_all_digits(db) || !swar_all_digits(dc)) return false;
  const uint32_t y = ((uint32_t)(a & 0xF)) * 1000 + ((uint32_t)(a >> 8) & 0xF) * 100 + ((uint32_t)(a >> 16) & 0xF) * 10 + ((uint32_t)(a >> 24) & 0xF);
  const uint32_t mo = ((uint32_t)(a >> 40) & 0xF) * 10 + ((uint32_t)(a >> 48) & 0xF);
  const uint32_t d = ((uint32_t)b & 0xF) * 10 + ((uint32_t)(b >> 8) & 0xF);
  const uint32_t hh = ((uint32_t)(b >> 24) & 0xF) * 10 + ((uint32_t)(b >> 32) & 0xF);
  const uint32_t mi = ((uint32_t)(b >> 48) & 0xF) * 10 + ((uint32_t)(b >> 56) & 0xF);
  const uint32_t ss = ((c >> 8) & 0xF) * 10 + ((c >> 16) & 0xF);
  if (mo < 1 || mo > 12 || d < 1 || hh > 23 || mi > 59 || ss > 59) return false;  // :60 → exact path
  const uint32_t dim = (mo == 2) ? (((y % 4 == 0 && y % 100 != 0) || y % 400 == 0) ? 29u : 28u)
                                 : ((mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30u : 31u);
  if (d > dim) return false;
  *days = days_from_civil((int64_t)y, (int64_t)mo, (int64_t)d);
  *sod = (int64_t)(hh * 3600u + mi * 60u + ss);
  return true;
}
// optional ".f{1,9}" at s[i..): returns nanoseconds and advances i; false on ".": exact path decides
__device__ __forceinline__ bool fast_fraction(const uint8_t* s, uint32_t n, uint32_t* i, uint32_t* ns) {
  *ns = 0;
  if (*i >= n || s[*i] != '.') return true;
  uint32_t k = *i + 1, v = 0, nd = 0;
  while (k < n && nd < 9 && is_digit(s[k])) { v = v * 10 + (s[k] - '0'); k++; nd++; }
  if (nd == 0 || (k < n && is_digit(s[k]))) return false;   // ≥ 10 digits → exact path (drops extras)
  for (; nd < 9; nd++) v *= 10;
  *ns = v; *i = k;
  return true;
}
// timestamptz in the spellings the pinned session produces ("…+00", "…+HH", "…+HH:MM", "…+HHMM")
__device__ __forceinline__ bool fast_timestamptz(const uint8_t* s, uint32_t n, CellOut& o) {
  if (n < 22) return false;
  int64_t days, sod;
  if (!fast_ymd_hms(s, &days, &sod)) return false;
  uint32_t i = 19, ns;
  if (!fast_fraction(s, n, &i, &ns)) return false;
  if (i + 3 > n) return false;
  const uint32_t sg = s[i];
  if (sg != '+' && sg != '-') return false;
  if (!is_digit(s[i + 1]) || !is_digit(s[i + 2])) return false;
  int32_t off = (int32_t)((s[i + 1] - '0') * 10 + (s[i + 2] - '0')) * 3600;
  i += 3;
  if (i < n) {
    if (s[i] == ':') i++;
    if (i + 2 != n || !is_digit(s[i]) || !is_digit(s[i + 1]) || s[i] > '5') return false;
    off += (int32_t)((s[i] - '0') * 10 + (s[i + 1] - '0')) * 60;
  }
  if (off >= 86400) return false;
  if (sg == '-') off = -off;
  o.tag = ETL_CELL_TIMESTAMPTZ; o.val = (uint64_t)(days * 86400 + sod - off); o.aux = ns;
  return true;
}
__device__ __forceinline__ bool fast_timestamp(const uint8_t* s, uint32_t n, CellOut& o) {
  if (n < 19) return false;
  int64_t days, sod;
  if (!fast_ymd_hms(s, &days, &sod)) return false;
  uint32_t i = 19, ns;
  if (!fast_fraction(s, n, &i, &ns) || i != n) return false;
  o.tag = ETL_CELL_TIMESTAMP; o.val = (uint64_t)(days * 86400 + sod); o.aux = ns;
  return true;
}

// "YYYY-MM-DD" exactly (what the pinned session's DateStyle ISO produces), years 0001-9999; else the exact path
__device__ __forceinline__ bool fast_date(const uint8_t* s, uint32_t n, CellOut& o) {
  if (n != 10) return false;
  const uint64_t a = ldu64(s);
  const uint32_t b = (uint32_t)ldu64(s + 8) & 0xFFFFu;
  if (((a >> 32) & 0xFFu) != '-' || ((a >> 56) & 0xFFu) != '-') return false;
  const uint64_t da = (a & 0x00FFFF00FFFFFFFFull) | 0x3000003000000000ull;
  const uint64_t db = (uint64_t)b | 0x3030303030300000ull;
  if (!swar_all_digits(da) || !swar_all_digits(db)) return false;
  const uint32_t y = ((uint32_t)(a & 0xF)) * 1000 + ((uint32_t)(a >> 8) & 0xF) * 100 + ((uint32_t)(a >> 16) & 0xF) * 10 + ((uint32_t)(a >> 24) & 0xF);
  const uint32_t mo = ((uint32_t)(a >> 40) & 0xF) * 10 + ((uint32_t)(a >> 48) & 0xF);
  const uint32_t d = (b & 0xF) * 10 + ((b >> 8) & 0xF);
  if (y < 1 || mo < 1 || mo > 12 || d < 1) return false;
  const uint32_t dim = (mo == 2) ? (((y % 4 == 0 && y % 100 != 0) || y % 400 == 0) ? 29u : 28u)
                                 : ((mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30u : 31u);
  if (d > dim) return false;
  o.tag = ETL_CELL_DATE; o.val = (uint64_t)days_from_civil((int64_t)y, (int64_t)mo, (int64_t)d); o.aux = 0;
  return true;
}
// 8 hex characters (memory order) → 4 bytes (memory order); *ok cleared on any non-hex character
__device__ __forceinline__ uint32_t swar_hex8(uint64_t x, bool* ok) {
  const uint64_t HI = 0x8080808080808080ull, ONES = 0x0101010101010101ull;
  if (x & HI) { *ok = false; return 0; }
  const uint64_t lo = x | 0x2020202020202020ull;
  const uint64_t digit = ((x + 0x50ull * ONES) & HI) & ~((x + 0x46ull * ONES) & HI);      // x >= '0' and not x > '9'
  const uint64_t alpha = ((lo + 0x1Full * ONES) & HI) & ~((lo + 0x19ull * ONES) & HI);    // lo >= 'a' and not lo > 'f'
  if ((digit | alpha) != HI) { *ok = false; return 0; }
  const uint64_t nib = (x & 0x0F0F0F0F0F0F0F0Full) + (alpha >> 7) * 9ull;
  const uint64_t pairs = ((nib << 4) | (nib >> 8)) & 0x00FF00FF00FF00FFull;
  return __byte_perm((uint32_t)pairs, (uint32_t)(pairs >> 32), 0x6420);
}
// the hyphenated 36-character spelling (uuid text output); everything else (braces, urn:, simple) → exact path
__device__ __forceinline__ bool fast_uuid(const uint8_t* s, uint32_t n, uint8_t* heap, uint64_t hpos, CellOut& o) {
  if (n != 36) return false;
  const uint64_t g0 = ldu64(s), g1 = ldu64(s + 8), g2 = ldu64(s + 16), g3 = ldu64(s + 24);
  const uint32_t g4 = (uint32_t)ldu64(s + 32);
  // '-' at 8, 13, 18, 23
  if ((g1 & 0xFFu) != '-' || ((g1 >> 40) & 0xFFu) != '-' || ((g2 >> 16) & 0xFFu) != '-' || ((g2 >> 56) & 0xFFu) != '-') return false;
  bool ok = true;
  const uint32_t o0 = swar_hex8(g0, &ok);                                                                    // chars 0-7
  const uint32_t o1 = swar_hex8(((g1 >> 8) & 0xFFFFFFFFull) | ((((g1 >> 48) | (g2 << 16)) & 0xFFFFFFFFull) << 32), &ok);   // 9-12, 14-17
  const uint32_t o2 = swar_hex8(((g2 >> 24) & 0xFFFFFFFFull) | ((g3 & 0xFFFFFFFFull) << 32), &ok);               // 19-22, 24-27
  const uint32_t o3 = swar_hex8((g3 >> 32) | ((uint64_t)g4 << 32), &ok);                                       // 28-35
  if (!ok) return false;
  uint64_t* dst = reinterpret_cast<uint64_t*>(heap + hpos);      // heap reservations are 8-byte aligned
  dst[0] = (uint64_t)o0 | ((uint64_t)o1 << 32);
  dst[1] = (uint64_t)o2 | ((uint64_t)o3 << 32);
  o.tag = ETL_CELL_UUID; o.val = hpos; o.aux = 16;
  return true;
}

// numeric: [+-]digits[.digits] (what Postgres emits) with warp-synchronous loops; everything else
// (NaN, Infinity, exponents, '_' separators, whitespace) goes to parse_numeric.
__device__ __forceinline__ uint32_t parse_numeric_sync(unsigned mask, const uint8_t* s, uint32_t n, uint8_t* heap, uint64_t hpos, CellOut& o) {
  HeapCursor hc{heap, hpos};
  bool simple = n > 0 && n <= 4096;
  uint32_t i0 = 0;
  bool neg = false;
  if (simple) { const uint32_t c0 = s[0]; if (c0 == '-') { neg = true; i0 = 1; } else if (c0 == '+') i0 = 1; }
  uint32_t code = 0xFFFFFFFFu;   // sentinel: not handled by the fast path
  // the specials as Postgres spells them (numeric.rs:256-278): NaN (unsigned), [+-]Infinity, [+-]inf — one lane with a
  // NaN would otherwise send its whole row of 32 through the exact, lane-serial parser
  if (simple && n - i0 >= 3u && n - i0 <= 8u) {
    const uint32_t m = n - i0;
    uint64_t wv = ldu64(s + i0);
    if (m < 8u) wv &= (1ull << (8u * m)) - 1ull;
    const uint64_t lw = wv | 0x2020202020202020ull;                       // ASCII letters → lower case (other bytes cannot become these words)
    const uint64_t lmask = m < 8u ? (1ull << (8u * m)) - 1ull : ~0ull;
    uint32_t kind = 0;
    if (m == 3u && (lw & lmask) == 0x6E616Eull && i0 == 0u) kind = 1;                     // "nan"
    else if ((m == 3u && (lw & lmask) == 0x666E69ull) || (m == 8u && lw == 0x7974696E69666E69ull)) kind = neg ? 3u : 2u;   // "inf" / "infinity"
    if (kind) {
      etl_numeric_hdr hdr;
      hdr.kind = (uint8_t)kind; hdr.sign = 0; hdr.weight = 0; hdr.scale = 0; hdr.pushed_groups = 0;
      const uint64_t off = hc.alloc(8);
      *reinterpret_cast<etl_numeric_hdr*>(hc.heap + off) = hdr;
      o.tag = ETL_CELL_NUMERIC; o.val = off; o.aux = 0;
      code = 0; simple = false;
    }
  }
  // pass 1: shape
  uint32_t nint = 0, nfrac = 0, ndot = 0;
  uint32_t i = i0;
  while (__any_sync(mask, simple && i < n)) {
    if (simple && i < n) {
      const uint32_t k = min(8u, n - i);
      const uint64_t x = ldu64(s + i);
      // per-byte classes, 8 bytes at a time: 0x80 in a byte of `dig` / `dot` = that byte is a digit / a '.'
      const uint64_t HI = 0x8080808080808080ull, L7 = 0x7F7F7F7F7F7F7F7Full;
      const uint64_t vm = k < 8u ? ((1ull << (8u * k)) - 1ull) & HI : HI;
      const uint64_t t = x ^ 0x3030303030303030ull;                       // digits → 0..9
      const uint64_t dig = ~(((t & L7) + 0x7676767676767676ull) | t) & vm;
      const uint64_t u = x ^ 0x2E2E2E2E2E2E2E2Eull;                       // '.' → 0
      const uint64_t dot = ~(((u & L7) + L7) | u) & vm;
      if ((dig | dot) != vm) simple = false;
      const uint64_t before = dot ? ((dot & (0ull - dot)) - 1ull) : ~0ull;   // bytes below the first '.' of this word
      const uint32_t nd_all = (uint32_t)__popcll(dig), nd_before = (uint32_t)__popcll(dig & before);
      if (ndot) nfrac += nd_all; else { nint += nd_before; nfrac += nd_all - nd_before; }
      ndot += (uint32_t)__popcll(dot);
      i += k;
    }
  }
  simple = simple && ndot <= 1 && (nint + nfrac) > 0;
  // numeric.rs:409-472 on the digit string D = int digits ++ frac digits
  const uint32_t ndec = nint + nfrac;
  const int64_t dweight = (int64_t)nint - 1;
  const int64_t weight = dweight >= 0 ? (dweight + 4) / 4 - 1 : -1;   // nint == 0 → dweight = -1 → weight -1
  const uint32_t offset = (uint32_t)((weight + 1) * 4 - (dweight + 1));
  const uint32_t ndig = simple ? (ndec + offset + 3u) / 4u : 0u;
  uint64_t off = 0;
  int16_t* dg = nullptr;
  if (simple) { off = hc.alloc(8 + 2 * ndig); dg = reinterpret_cast<int16_t*>(hc.heap + off + 8); }
  const uint8_t* dp = s + i0;                       // digit j lives at dp[j] (j < nint) or dp[j+1]
  uint32_t lead = 0, written = 0, last_nz = 0;
  bool seen_nz = false;
  uint32_t g = 0;
  while (__any_sync(mask, g < ndig)) {                // every lane of `mask` votes; non-simple lanes have ndig = 0
    if (g < ndig) {
      uint32_t v = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int32_t j = (int32_t)(g * 4u + (uint32_t)k) - (int32_t)offset;
        uint32_t d = 0;
        if (j >= 0 && (uint32_t)j < ndec) d = (uint32_t)dp[(uint32_t)j + (((uint32_t)j >= nint) ? ndot : 0u)] - '0';
        v = v * 10u + d;
      }
      if (!seen_nz) { if (v == 0) lead++; else { seen_nz = true; dg[0] = (int16_t)v; written = 1; last_nz = 1; } }
      else { dg[written++] = (int16_t)v; if (v) last_nz = written; }
      g++;
    }
  }
  if (simple) {
    etl_numeric_hdr hdr;
    hdr.kind = 0; hdr.sign = 0; hdr.weight = 0; hdr.scale = (uint16_t)nfrac; hdr.pushed_groups = 0;
    uint32_t nd = 0;
    code = 0;
    if (nfrac > 16383u) code = ETL_E_NUMERIC;
    else if (seen_nz) {
      const int64_t fw = weight - (int64_t)lead;
      if (fw < -32768 || fw > 32767) code = ETL_E_NUMERIC;
      hdr.sign = neg ? 1 : 0; hdr.weight = (int16_t)fw; nd = last_nz;
      hdr.pushed_groups = (uint16_t)ndig;            // n ≤ 4096 here
    }
    *reinterpret_cast<etl_numeric_hdr*>(hc.heap + off) = hdr;
    o.tag = ETL_CELL_NUMERIC | ((uint32_t)hdr.pushed_groups << 16); o.val = off; o.aux = nd;
  }
  if (code == 0xFFFFFFFFu) {                          // own copies: `o` must not have its address taken (see parse_heavy_sync)
    HeapCursor h2{heap, hpos};
    CellOut t; t.tag = 0; t.val = 0; t.aux = 0;
    code = parse_numeric(s, n, h2, t);
    o = t;
  }
  return code;
}

// serde_json acceptance, table-driven so that every lane executes the same instructions per byte
// (a switch over the state serialises the warp: the first version spent ~225 warp instructions per
// byte step on it).  Tables: tools/gen_json_tables.py (fuzzed against the oracle in
// tests/test_json_tables.py); T2 = kJsonT2 (state << 8 | byte → next | action << 5), in shared memory.
// One load per byte (the class lookup is folded into the table), eight bytes between two warp votes, and the
// container stack is a 128-bit shift register (bit 0 = innermost level, 1 = object) so that brackets and commas
// are handled by predicated straight-line code: with 32 documents in flight some lane sits on a structural
// byte at almost every step, and a divergent action block was a third of this function's issue slots (ncu, C3).
__device__ __forceinline__ bool json_valid_sync(unsigned mask, const uint8_t* s, uint32_t n, const uint8_t* T2) {
  uint32_t st = JT_VALUE, depth = 0, aux = 0, hexn = 0;
  bool key = false, low_sur = false;
  uint64_t lo = 0, hi = 0;
  uint64_t next = n ? ldu64(s) : 0ull;                // one word ahead: the load overlaps the 8 DFA steps before it
  uint32_t i = 0;
  while (__any_sync(mask, i < n && st != JT_BAD)) {   // i is a multiple of 8 for every lane that is still running
    const uint64_t word = next;
    if (i + 8u < n) next = ldu64(s + i + 8u);
#pragma unroll
    for (int k = 0; k < 8; k++) {
      if (i < n && st != JT_BAD) {
        const uint32_t c = (uint32_t)(word >> (8 * k)) & 0xFFu;
        i++;
        if (st - JT_ESC <= 3u) {                      // inside an escape: rare
          if (st == JT_ESC) {
            if (c == 'u') { st = JT_HEX; hexn = 4; aux = 0; }
            else if (c == '"' || c == '\\' || c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't') st = low_sur ? JT_BAD : JT_STR;
            else st = JT_BAD;
          } else if (st == JT_HEX) {
            const int h = hexval(c);
            if (h < 0) st = JT_BAD;
            else {
              aux = aux * 16u + (uint32_t)h;
              if (--hexn == 0) {
                if (low_sur) { st = (aux >= 0xDC00u && aux <= 0xDFFFu) ? JT_STR : JT_BAD; low_sur = false; }
                else if (aux >= 0xDC00u && aux <= 0xDFFFu) st = JT_BAD;
                else if (aux >= 0xD800u && aux <= 0xDBFFu) st = JT_SUR_BS;
                else st = JT_STR;
              }
            }
          } else if (st == JT_SUR_BS) st = (c == '\\') ? JT_SUR_U : JT_BAD;
          else { if (c == 'u') { st = JT_HEX; hexn = 4; aux = 0; low_sur = true; } else st = JT_BAD; }
        } else {
          const uint32_t e = T2[(st << 8) | c];
          uint32_t nst = e & 31u;
          const uint32_t act = e >> 5;
          const bool top_obj = (lo & 1ull) != 0ull;
          if ((act - JA_PUSH_OBJ) < 2u) {             // '{' '[': serde_json's recursion limit is 128 levels
            nst = depth < 127u ? nst : (uint32_t)JT_BAD;
            hi = (hi << 1) | (lo >> 63); lo = (lo << 1) | (act == JA_PUSH_OBJ ? 1ull : 0ull);
            depth++;
          }
          if ((act - JA_POP_OBJ) < 2u) {              // '}' ']' must close the innermost container of its kind
            nst = (depth > 0u && top_obj == (act == JA_POP_OBJ)) ? nst : (uint32_t)JT_BAD;
            lo = (lo >> 1) | (hi << 63); hi >>= 1;
            depth--;
          }
          if (act == JA_COMMA) nst = depth == 0u ? (uint32_t)JT_BAD : (top_obj ? (uint32_t)JT_KEY : (uint32_t)JT_VALUE);
          if (act >= JA_KEYSTR) { key = act == JA_KEYSTR; low_sur = false; }
          if (nst == JT_STR_END) nst = key ? JT_COLON : JT_AFTER;
          st = nst;
        }
      }
    }
  }
  return depth == 0 && (st == JT_AFTER || st == JT_ZERO || st == JT_INT || st == JT_FRAC || st == JT_EXP);
}

}  // namespace etl
