/*
 * oracle_cells.c — CPU restatement of crates/etl/src/conversions/{text,numeric,hex,bool}.rs.
 * TEST INFRASTRUCTURE ONLY (see oracle.h). Each function cites the reference lines it follows.
 *
 * Library behaviour restated here because the crates are not part of the reference tree:
 *   Rust core str::parse (ints, floats)      — toolchain 1.93.1 (rust-toolchain.toml)
 *   chrono 0.4.44 parse_from_str             — Cargo.lock:1122-1123   (leniency: parity unpinned)
 *   uuid 1.23.1 Uuid::parse_str              — Cargo.lock:6946-6947   (alt spellings: parity unpinned)
 *   serde_json 1.0.149 + arbitrary_precision — Cargo.lock:5622-5623   (depth limit: parity unpinned)
 */
#define _GNU_SOURCE
#include <errno.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "oracle_internal.h"

/* ------------------------------------------------------------------ heap */
uint64_t orc_heap_alloc(orc_heap* h, uint64_t n, uint64_t align) {
  uint64_t off = (h->len + (align - 1)) & ~(align - 1);
  uint64_t need = off + n;
  if (need > h->cap) {
    uint64_t nc = h->cap ? h->cap * 2 : 4096;
    while (nc < need) nc *= 2;
    h->data = (uint8_t*)realloc(h->data, nc);
    memset(h->data + h->cap, 0, nc - h->cap);
    h->cap = nc;
  }
  /* zero alignment padding so heaps compare deterministically */
  if (off > h->len) memset(h->data + h->len, 0, off - h->len);
  h->len = need;
  return off;
}

/* ------------------------------------------------------------------ oid → decode class
 * text.rs:28-173 match arms; array detection utils.rs:12-16 (builtin array types whose name
 * starts with '_'); unknown oids fall back to TEXT (utils.rs:7-9) → String. */
static const uint32_t BUILTIN_OTHER_ARRAY_OIDS[] = {
    /* builtin array types (pg_type.dat) that text.rs does not name → ArrayCell::String (text.rs:166-170).
       int2vector[] (1006) and oidvector[] (1013) are genuine array types named _int2vector/_oidvector. */
    143 /*_xml*/, 199 /*handled*/, 271 /*_xid8*/, 629 /*_line*/, 651 /*_cidr*/, 719 /*_circle*/,
    775 /*_macaddr8*/, 1006, 1008 /*_regproc*/, 1010 /*_tid*/, 1011 /*_xid*/, 1012 /*_cid*/, 1013,
    1017 /*_point*/, 1018 /*_lseg*/, 1019 /*_path*/, 1020 /*_box*/, 1027 /*_polygon*/,
    1034 /*_aclitem*/, 1040 /*_macaddr*/, 1041 /*_inet*/, 1187 /*_interval*/, 1263 /*_cstring*/,
    1270 /*_timetz*/, 1561 /*_bit*/, 1563 /*_varbit*/, 2201 /*_refcursor*/, 2207 /*_regprocedure*/,
    2208 /*_regoper*/, 2209 /*_regoperator*/, 2210 /*_regclass*/, 2211 /*_regtype*/,
    2949 /*_txid_snapshot*/, 3221 /*_pg_lsn*/, 3643 /*_tsvector*/, 3644 /*_gtsvector*/,
    3645 /*_tsquery*/, 3735 /*_regconfig*/, 3770 /*_regdictionary*/, 3905 /*_int4range*/,
    3907 /*_numrange*/, 3909 /*_tsrange*/, 3911 /*_tstzrange*/, 3913 /*_daterange*/,
    3927 /*_int8range*/, 4073 /*_jsonpath*/, 4090 /*_regnamespace*/, 4097 /*_regrole*/,
    4192 /*_regcollation*/, 5039 /*_pg_snapshot*/, 6150 /*_int4multirange*/,
    6151 /*_nummultirange*/, 6152 /*_tsmultirange*/, 6153 /*_tstzmultirange*/,
    6155 /*_datemultirange*/, 6157 /*_int8multirange*/, 12052, 12057, 12062, 12067 /* information_schema domains' arrays vary by version: not matched */
};

uint32_t orc_kind_for_oid(uint32_t oid) {
  switch (oid) {
    case 16: return ETL_K_BOOL;
    case 1000: return ETL_K_ARRAY | ETL_K_BOOL;
    case 18: case 1042: case 1043: case 19: case 25: case 790: return ETL_K_STRING;
    case 1002: case 1014: case 1015: case 1003: case 1009: case 791: return ETL_K_ARRAY | ETL_K_STRING;
    case 21: return ETL_K_I16;
    case 1005: return ETL_K_ARRAY | ETL_K_I16;
    case 23: return ETL_K_I32;
    case 1007: return ETL_K_ARRAY | ETL_K_I32;
    case 20: return ETL_K_I64;
    case 1016: return ETL_K_ARRAY | ETL_K_I64;
    case 700: return ETL_K_F32;
    case 1021: return ETL_K_ARRAY | ETL_K_F32;
    case 701: return ETL_K_F64;
    case 1022: return ETL_K_ARRAY | ETL_K_F64;
    case 1700: return ETL_K_NUMERIC;
    case 1231: return ETL_K_ARRAY | ETL_K_NUMERIC;
    case 17: return ETL_K_BYTES;
    case 1001: return ETL_K_ARRAY | ETL_K_BYTES;
    case 1082: return ETL_K_DATE;
    case 1182: return ETL_K_ARRAY | ETL_K_DATE;
    case 1083: return ETL_K_TIME;
    case 1183: return ETL_K_ARRAY | ETL_K_TIME;
    case 1114: return ETL_K_TIMESTAMP;
    case 1115: return ETL_K_ARRAY | ETL_K_TIMESTAMP;
    case 1184: return ETL_K_TIMESTAMPTZ;
    case 1185: return ETL_K_ARRAY | ETL_K_TIMESTAMPTZ;
    case 2950: return ETL_K_UUID;
    case 2951: return ETL_K_ARRAY | ETL_K_UUID;
    case 114: case 3802: return ETL_K_JSON;
    case 199: case 3807: return ETL_K_ARRAY | ETL_K_JSON;
    case 26: return ETL_K_U32;
    case 1028: return ETL_K_ARRAY | ETL_K_U32;
    default: break;
  }
  for (size_t i = 0; i < sizeof(BUILTIN_OTHER_ARRAY_OIDS) / sizeof(uint32_t); i++)
    if (BUILTIN_OTHER_ARRAY_OIDS[i] == oid) return ETL_K_ARRAY | ETL_K_STRING;
  return ETL_K_STRING;
}

uint32_t orc_error_kind(uint32_t code) {
  switch (code) {
    case ETL_E_NONE: return ETL_EK_NONE;
    case ETL_E_UUID: case ETL_E_BOOL: case ETL_E_NOT_NULL: return ETL_EK_INVALID_DATA;
    case ETL_E_JSON: return ETL_EK_DESERIALIZATION_ERROR;
    case ETL_E_TX_STATE: case ETL_E_MISSING_TABLE_STATE: return ETL_EK_INVALID_STATE;
    case ETL_E_COMMIT_LSN: return ETL_EK_VALIDATION_ERROR;
    case ETL_E_UNKNOWN_COLUMNS: return ETL_EK_CORRUPTED_TABLE_SCHEMA;
    case ETL_E_MISSING_TABLE_SCHEMA: return ETL_EK_MISSING_TABLE_SCHEMA;
    case ETL_E_MALFORMED_FRAME: return ETL_EK_SOURCE_ERROR;
    default: return ETL_EK_CONVERSION_ERROR;
  }
}

/* ------------------------------------------------------------------ UTF-8 (core::str::from_utf8)
 * event.rs:972. Well-formed UTF-8 per Unicode Table 3-7: no overlongs, no surrogates, ≤ U+10FFFF. */
int orc_utf8_valid(const uint8_t* s, uint64_t n) {
  uint64_t i = 0;
  while (i < n) {
    uint8_t b = s[i];
    if (b < 0x80) { i++; continue; }
    if (b >= 0xC2 && b <= 0xDF) {
      if (i + 1 >= n || (s[i + 1] & 0xC0) != 0x80) return 0;
      i += 2;
    } else if (b >= 0xE0 && b <= 0xEF) {
      if (i + 2 >= n) return 0;
      uint8_t c1 = s[i + 1], c2 = s[i + 2];
      uint8_t lo = 0x80, hi = 0xBF;
      if (b == 0xE0) lo = 0xA0;
      if (b == 0xED) hi = 0x9F;
      if (c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80) return 0;
      i += 3;
    } else if (b >= 0xF0 && b <= 0xF4) {
      if (i + 3 >= n) return 0;
      uint8_t c1 = s[i + 1], c2 = s[i + 2], c3 = s[i + 3];
      uint8_t lo = 0x80, hi = 0xBF;
      if (b == 0xF0) lo = 0x90;
      if (b == 0xF4) hi = 0x8F;
      if (c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80 || (c3 & 0xC0) != 0x80) return 0;
      i += 4;
    } else {
      return 0;
    }
  }
  return 1;
}

/* byte length of the Unicode White_Space char at s (char::is_whitespace), 0 if not whitespace.
 * Input is already valid UTF-8. */
static uint32_t ws_len(const uint8_t* s, uint64_t n) {
  if (n == 0) return 0;
  uint8_t b = s[0];
  if (b == ' ' || (b >= 0x09 && b <= 0x0D)) return 1;
  if (b == 0xC2 && n >= 2 && (s[1] == 0x85 || s[1] == 0xA0)) return 2;
  if (n >= 3) {
    if (b == 0xE1 && s[1] == 0x9A && s[2] == 0x80) return 3;                      /* U+1680 */
    if (b == 0xE2 && s[1] == 0x80 && ((s[2] >= 0x80 && s[2] <= 0x8A) ||           /* U+2000-200A */
                                      s[2] == 0xA8 || s[2] == 0xA9 || s[2] == 0xAF)) return 3;
    if (b == 0xE2 && s[1] == 0x81 && s[2] == 0x9F) return 3;                      /* U+205F */
    if (b == 0xE3 && s[1] == 0x80 && s[2] == 0x80) return 3;                      /* U+3000 */
  }
  return 0;
}
static void trim_start_ws(const uint8_t** s, uint64_t* n) {
  uint32_t w;
  while ((w = ws_len(*s, *n)) != 0) { *s += w; *n -= w; }
}

static int is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
static uint8_t lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }
static int ieq(const uint8_t* s, uint64_t n, const char* lit) {
  uint64_t m = strlen(lit);
  if (n != m) return 0;
  for (uint64_t i = 0; i < n; i++) if (lower(s[i]) != (uint8_t)lit[i]) return 0;
  return 1;
}

/* ------------------------------------------------------------------ bool.rs:11-19 */
static uint32_t parse_bool(const uint8_t* s, uint64_t n, orc_cell* c) {
  if (n == 1 && s[0] == 't') { c->tag = ETL_CELL_BOOL; c->val = 1; return 0; }
  if (n == 1 && s[0] == 'f') { c->tag = ETL_CELL_BOOL; c->val = 0; return 0; }
  return ETL_E_BOOL;
}

/* ------------------------------------------------------------------ integers: Rust core::num
 * FromStr for i16/i32/i64/u32 (text.rs:49-60,159-161). Optional single sign ('-' only for signed),
 * ASCII digits only, at least one digit, overflow is an error. */
static uint32_t parse_int(const uint8_t* s, uint64_t n, int is_signed, int64_t lo, uint64_t hi,
                          int64_t* out) {
  if (n == 0) return ETL_E_PARSE_INT;
  int neg = 0;
  uint64_t i = 0;
  if (s[0] == '+') i = 1;
  else if (s[0] == '-') { if (!is_signed) return ETL_E_PARSE_INT; neg = 1; i = 1; }
  if (i == n) return ETL_E_PARSE_INT;
  /* limit is at most 2^63, digits accumulate in u64 with an exact overflow test */
  uint64_t limit = neg ? (uint64_t)(-(lo + 1)) + 1u : hi;
  uint64_t acc = 0;
  for (; i < n; i++) {
    if (!is_digit(s[i])) return ETL_E_PARSE_INT;
    uint64_t d = (uint64_t)(s[i] - '0');
    if (acc > (limit - d) / 10) return ETL_E_PARSE_INT; /* acc*10+d > limit */
    acc = acc * 10 + d;
  }
  *out = neg ? (int64_t)(0 - acc) : (int64_t)acc;
  return 0;
}

/* ------------------------------------------------------------------ floats: Rust core::num::dec2flt
 * (text.rs:61-68). Grammar: [+-] ( digits [. digits] | . digits ) [ (e|E) [+-] digits ] with at
 * least one mantissa digit, or case-insensitive inf / infinity / nan. Result is the correctly
 * rounded nearest-even value; glibc strtod/strtof are correctly rounded, so they serve as the
 * independent evaluator once the grammar has been checked. */
static int float_grammar(const uint8_t* s, uint64_t n, int* special /*1 inf, 2 nan*/, int* neg) {
  *special = 0; *neg = 0;
  if (n == 0) return 0;
  uint64_t i = 0;
  if (s[0] == '+' || s[0] == '-') { *neg = s[0] == '-'; i = 1; }
  if (i == n) return 0;
  uint64_t nd = 0, j = i;
  while (j < n && is_digit(s[j])) { j++; nd++; }
  if (j < n && s[j] == '.') { j++; while (j < n && is_digit(s[j])) { j++; nd++; } }
  if (nd > 0) {
    if (j < n && (s[j] == 'e' || s[j] == 'E')) {
      j++;
      if (j < n && (s[j] == '+' || s[j] == '-')) j++;
      if (j >= n || !is_digit(s[j])) return 0;
      while (j < n && is_digit(s[j])) j++;
    }
    if (j == n) return 1;
  }
  if (ieq(s + i, n - i, "inf") || ieq(s + i, n - i, "infinity")) { *special = 1; return 1; }
  if (ieq(s + i, n - i, "nan")) { *special = 2; return 1; }
  return 0;
}
static uint32_t parse_f64(const uint8_t* s, uint64_t n, orc_cell* c) {
  int special, neg;
  if (!float_grammar(s, n, &special, &neg)) return ETL_E_PARSE_FLOAT;
  uint64_t bits;
  if (special == 1) bits = 0x7ff0000000000000ull | ((uint64_t)neg << 63);
  else if (special == 2) bits = 0x7ff8000000000000ull | ((uint64_t)neg << 63);
  else {
    char* tmp = (char*)malloc(n + 1);
    memcpy(tmp, s, n); tmp[n] = 0;
    double d = strtod(tmp, NULL);
    free(tmp);
    memcpy(&bits, &d, 8);
  }
  c->tag = ETL_CELL_F64; c->val = bits; c->aux = 0;
  return 0;
}
static uint32_t parse_f32(const uint8_t* s, uint64_t n, orc_cell* c) {
  int special, neg;
  if (!float_grammar(s, n, &special, &neg)) return ETL_E_PARSE_FLOAT;
  uint32_t bits;
  if (special == 1) bits = 0x7f800000u | ((uint32_t)neg << 31);
  else if (special == 2) bits = 0x7fc00000u | ((uint32_t)neg << 31);
  else {
    char* tmp = (char*)malloc(n + 1);
    memcpy(tmp, s, n); tmp[n] = 0;
    float f = strtof(tmp, NULL);
    free(tmp);
    memcpy(&bits, &f, 4);
  }
  c->tag = ETL_CELL_F32; c->val = bits; c->aux = 0;
  return 0;
}

/* ------------------------------------------------------------------ numeric.rs:99-472 */
static uint32_t parse_numeric(const uint8_t* s, uint64_t n, orc_heap* heap, orc_cell* c) {
  const uint8_t* p = s;
  uint64_t rem = n;
  trim_start_ws(&p, &rem);                                   /* numeric.rs:106 */
  if (rem == 0) return ETL_E_NUMERIC;                        /* :108 */
  int neg = 0, explicit_sign = 0;
  if (p[0] == '+') { explicit_sign = 1; p++; rem--; }        /* :113-123 */
  else if (p[0] == '-') { neg = 1; explicit_sign = 1; p++; rem--; }
  etl_numeric_hdr hdr;
  memset(&hdr, 0, sizeof hdr);
  if (!(rem > 0 && (is_digit(p[0]) || p[0] == '.'))) {       /* :126 → parse_special_value :256-278 */
    /* remaining.trim_end().to_lowercase(): only ASCII letters can lowercase to these words */
    uint64_t e = rem;
    for (;;) { /* trim_end by Unicode whitespace */
      int trimmed = 0;
      for (uint32_t w = 1; w <= 3 && w <= e; w++) {
        if (ws_len(p + e - w, w) == w) { e -= w; trimmed = 1; break; }
      }
      if (!trimmed) break;
    }
    if (ieq(p, e, "nan")) { if (explicit_sign) return ETL_E_NUMERIC; hdr.kind = 1; }
    else if (ieq(p, e, "infinity") || ieq(p, e, "inf")) hdr.kind = neg ? 3 : 2;
    else return ETL_E_NUMERIC;
    uint64_t off = orc_heap_alloc(heap, sizeof hdr, 8);
    memcpy(heap->data + off, &hdr, sizeof hdr);
    c->tag = ETL_CELL_NUMERIC; c->val = off; c->aux = 0;
    return 0;
  }
  /* parse_numeric_value :285-401 */
  uint8_t* dec = (uint8_t*)malloc(rem + 8);
  uint64_t ndec = 0;
  int have_dp = 0;
  int64_t dweight = -1;
  int64_t dscale = 0;
  uint64_t i = 0;
#define PEEK(k) ((i + (k)) < rem ? p[i + (k)] : 0)
  if (PEEK(0) == '.') { have_dp = 1; i++; }                  /* :295-298 */
  if (!is_digit(PEEK(0)) || i >= rem) { free(dec); return ETL_E_NUMERIC; } /* :301 */
  while (i < rem) {                                          /* :306-337 */
    uint8_t ch = p[i];
    if (is_digit(ch)) { i++; dec[ndec++] = (uint8_t)(ch - '0'); if (!have_dp) dweight++; else dscale++; }
    else if (ch == '.') {
      if (have_dp) { free(dec); return ETL_E_NUMERIC; }
      have_dp = 1; i++;
      if (i < rem && p[i] == '_') { free(dec); return ETL_E_NUMERIC; }
    } else if (ch == '_') {
      i++;
      if (!(i < rem && is_digit(p[i]))) { free(dec); return ETL_E_NUMERIC; }
    } else break;
  }
  int out_of_range = 0;
  if (i < rem && (p[i] == 'e' || p[i] == 'E')) {             /* :340-387 */
    i++;
    int64_t exponent = 0; int eneg = 0;
    if (i < rem && p[i] == '+') i++;
    else if (i < rem && p[i] == '-') { eneg = 1; i++; }
    if (!(i < rem && is_digit(p[i]))) { free(dec); return ETL_E_NUMERIC; }
    while (i < rem) {
      uint8_t ch = p[i];
      if (is_digit(ch)) {
        i++; exponent = exponent * 10 + (ch - '0');
        if (exponent > 2147483647LL / 2) { out_of_range = 1; break; } /* :367 ValueOutOfRange */
      } else if (ch == '_') {
        i++;
        if (!(i < rem && is_digit(p[i]))) { free(dec); return ETL_E_NUMERIC; }
      } else break;
    }
    if (out_of_range) { free(dec); return ETL_E_NUMERIC; }
    if (eneg) exponent = -exponent;
    dweight += (int64_t)(int32_t)exponent;                   /* :385 (i32 arithmetic, cannot overflow here) */
    dscale = (dscale - exponent) < 0 ? 0 : (dscale - exponent);
  }
#undef PEEK
  { const uint8_t* q = p + i; uint64_t r = rem - i; trim_start_ws(&q, &r); if (r != 0) { free(dec); return ETL_E_NUMERIC; } } /* :390-393 */
  if (dscale > 16383) { free(dec); return ETL_E_NUMERIC; }   /* :395 */
  /* convert_to_base_10000 :409-472 */
  hdr.scale = (uint16_t)dscale;
  int16_t* digits = NULL; uint64_t nd = 0; int64_t final_weight = 0;
  if (ndec > 0) {
    int64_t weight = dweight >= 0 ? (dweight + 4) / 4 - 1 : -((-dweight - 1) / 4 + 1);
    int64_t offset = (weight + 1) * 4 - (dweight + 1);
    int64_t total = (int64_t)ndec + offset;
    int64_t ndig = (total + 3) / 4;
    digits = (int16_t*)calloc((size_t)ndig + 1, sizeof(int16_t));
    int allzero = 1;
    for (int64_t g = 0; g < ndig; g++) {
      int v = 0;
      for (int k = 0; k < 4; k++) {
        int64_t idx = g * 4 + k - offset;
        int d = (idx >= 0 && idx < (int64_t)ndec) ? dec[idx] : 0;
        v = v * 10 + d;
      }
      digits[g] = (int16_t)v;
      if (v) allzero = 0;
    }
    if (!allzero) {                                          /* :452-471 */
      int64_t lead = 0;
      while (lead < ndig && digits[lead] == 0) lead++;
      int64_t end = ndig;
      while (end > lead + 1 && digits[end - 1] == 0) end--;
      final_weight = weight - lead;
      if (final_weight < -32768 || final_weight > 32767) { free(dec); free(digits); return ETL_E_NUMERIC; }
      nd = (uint64_t)(end - lead);
      memmove(digits, digits + lead, nd * sizeof(int16_t));
      hdr.sign = (uint8_t)neg;
      hdr.weight = (int16_t)final_weight;
      hdr.pushed_groups = (uint16_t)(ndig > 65535 ? 65535 : ndig);   /* base_10000_digits.push per group, numeric.rs:441-448 */
    } else {
      nd = 0; hdr.sign = 0; hdr.weight = 0;                  /* canonical zero keeps scale */
    }
  }
  uint64_t off = orc_heap_alloc(heap, sizeof hdr + nd * 2, 8);
  memcpy(heap->data + off, &hdr, sizeof hdr);
  if (nd) memcpy(heap->data + off + sizeof hdr, digits, nd * 2);
  free(dec); free(digits);
  c->tag = ETL_CELL_NUMERIC; c->val = off; c->aux = (uint32_t)nd;
  return 0;
}

/* ------------------------------------------------------------------ hex.rs:11-37 */
static int hexval(uint8_t c) {
  if (c >= '0' && c <= '9') return c - '0';
  if (c >= 'a' && c <= 'f') return c - 'a' + 10;
  if (c >= 'A' && c <= 'F') return c - 'A' + 10;
  return -1;
}
static uint32_t parse_bytea(const uint8_t* s, uint64_t n, orc_heap* heap, orc_cell* c) {
  if (n < 2 || s[0] != '\\' || s[1] != 'x') return ETL_E_BYTEA;      /* :12 */
  s += 2; n -= 2;
  if (n % 2 != 0) return ETL_E_BYTEA;                                /* :23 */
  uint64_t off = orc_heap_alloc(heap, n / 2, 8);
  for (uint64_t i = 0; i < n; i += 2) {
    /* u8::from_str_radix(&value[i..i+2], 16): optional leading '+', then ≥1 hex digit (hex.rs:32).
       A multi-byte char straddling the slice makes the reference panic; reported as ParseInt here. */
    int a, b;
    if (s[i] == '+') { b = hexval(s[i + 1]); if (b < 0) return ETL_E_PARSE_INT; heap->data[off + i / 2] = (uint8_t)b; continue; }
    a = hexval(s[i]); b = hexval(s[i + 1]);
    if (a < 0 || b < 0) return ETL_E_PARSE_INT;
    heap->data[off + i / 2] = (uint8_t)(a * 16 + b);
  }
  c->tag = ETL_CELL_BYTES; c->val = off; c->aux = (uint32_t)(n / 2);
  return 0;
}

/* ------------------------------------------------------------------ chrono 0.4 parse_from_str
 * formats: etl-postgres/src/types/time.rs:7-21. Restates chrono::format::parse::parse_internal
 * and format::scan::{number,nanosecond,timezone_offset,colon_or_space}. parity unpinned beyond
 * text.rs:538-592. */
typedef struct { const uint8_t* s; uint64_t n; } cur_t;

/* scan::number(s, min, max): 1..=max ASCII digits, i64 overflow is an error */
static int scan_number(cur_t* c, uint64_t min, uint64_t max, int64_t* out) {
  uint64_t k = 0; int64_t v = 0;
  while (k < c->n && k < max && is_digit(c->s[k])) {
    int d = c->s[k] - '0';
    if (v > (INT64_MAX - d) / 10) return 0;
    v = v * 10 + d; k++;
  }
  if (k < min) return 0;
  c->s += k; c->n -= k; *out = v;
  return 1;
}
/* Item::Numeric: leading whitespace skipped; signed (year) accepts +/- with unbounded digits */
static int num_field(cur_t* c, uint64_t width, int is_signed, int64_t* out) {
  trim_start_ws(&c->s, &c->n);
  if (is_signed && c->n > 0 && c->s[0] == '-') {
    c->s++; c->n--;
    int64_t v; if (!scan_number(c, 1, UINT64_MAX, &v)) return 0;
    *out = -v; return 1;
  }
  if (is_signed && c->n > 0 && c->s[0] == '+') {
    c->s++; c->n--;
    return scan_number(c, 1, UINT64_MAX, out);
  }
  return scan_number(c, 1, width, out);
}
static int lit(cur_t* c, uint8_t ch) {
  if (c->n < 1 || c->s[0] != ch) return 0;
  c->s++; c->n--; return 1;
}
static int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {
  y -= m <= 2;
  int64_t era = (y >= 0 ? y : y - 399) / 400;
  int64_t yoe = y - era * 400;
  int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}
static int days_in_month(int64_t y, int64_t m) {
  static const int dm[] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  if (m == 2) return ((y % 4 == 0 && y % 100 != 0) || y % 400 == 0) ? 29 : 28;
  return dm[m - 1];
}
/* %Y-%m-%d → days; NaiveDate::from_ymd_opt range is [-262143, 262142] (chrono MIN/MAX year) */
static int parse_date_part(cur_t* c, int64_t* days) {
  int64_t y, m, d;
  if (!num_field(c, 4, 1, &y)) return 0;
  if (y < INT32_MIN || y > INT32_MAX) return 0;
  if (!lit(c, '-')) return 0;
  if (!num_field(c, 2, 0, &m)) return 0;
  if (m < 1 || m > 12) return 0;
  if (!lit(c, '-')) return 0;
  if (!num_field(c, 2, 0, &d)) return 0;
  if (d < 1 || d > 31) return 0;
  if (y < -262143 || y > 262142) return 0;
  if (d > days_in_month(y, m)) return 0;
  *days = days_from_civil(y, m, d);
  return 1;
}
/* %H:%M:%S%.f → secs of day + nanos (second 60 → 59 + 1e9 nanos, Parsed::to_naive_time) */
static int parse_time_part(cur_t* c, int64_t* secs, uint32_t* nanos) {
  int64_t h, mi, se;
  if (!num_field(c, 2, 0, &h) || h > 23) return 0;
  if (!lit(c, ':')) return 0;
  if (!num_field(c, 2, 0, &mi) || mi > 59) return 0;
  if (!lit(c, ':')) return 0;
  if (!num_field(c, 2, 0, &se) || se > 60) return 0;
  uint32_t ns = 0;
  if (c->n > 0 && c->s[0] == '.') {                        /* Fixed::Nanosecond → scan::nanosecond */
    c->s++; c->n--;
    uint64_t before = c->n; int64_t v;
    if (!scan_number(c, 1, 9, &v)) return 0;
    uint64_t consumed = before - c->n;
    static const int64_t scale[] = {0, 100000000, 10000000, 1000000, 100000, 10000, 1000, 100, 10, 1};
    v *= scale[consumed];
    while (c->n > 0 && is_digit(c->s[0])) { c->s++; c->n--; } /* extra digits are dropped */
    ns = (uint32_t)v;
  }
  if (se == 60) { se = 59; ns += 1000000000u; }
  *secs = h * 3600 + mi * 60 + se; *nanos = ns;
  return 1;
}
/* scan::timezone_offset(s, colon_or_space, allow_zulu, allow_missing_minutes, allow_tz_minus_sign=true) */
static int parse_tz(cur_t* c, int allow_zulu, int allow_missing_minutes, int32_t* off) {
  trim_start_ws(&c->s, &c->n);
  if (allow_zulu && c->n > 0 && (c->s[0] == 'Z' || c->s[0] == 'z')) { c->s++; c->n--; *off = 0; return 1; }
  int neg;
  if (c->n == 0) return 0;
  if (c->s[0] == '+') { neg = 0; c->s++; c->n--; }
  else if (c->s[0] == '-') { neg = 1; c->s++; c->n--; }
  else if (c->n >= 3 && c->s[0] == 0xE2 && c->s[1] == 0x88 && c->s[2] == 0x92) { neg = 1; c->s += 3; c->n -= 3; } /* U+2212 */
  else return 0;
  if (c->n < 2) return 0;
  if (!is_digit(c->s[0]) || !is_digit(c->s[1])) return 0;
  int32_t hours = (c->s[0] - '0') * 10 + (c->s[1] - '0');
  c->s += 2; c->n -= 2;
  for (;;) { /* colon_or_space: trim_start_matches(':' | whitespace) */
    if (c->n > 0 && c->s[0] == ':') { c->s++; c->n--; continue; }
    uint32_t w = ws_len(c->s, c->n);
    if (w) { c->s += w; c->n -= w; continue; }
    break;
  }
  int32_t minutes;
  if (c->n >= 2) {
    uint8_t m1 = c->s[0], m2 = c->s[1];
    if (m1 >= '0' && m1 <= '5' && is_digit(m2)) minutes = (m1 - '0') * 10 + (m2 - '0');
    else return 0; /* OUT_OF_RANGE or INVALID */
  } else if (allow_missing_minutes) minutes = 0;
  else return 0;
  if (c->n >= 2) { c->s += 2; c->n -= 2; }
  else if (c->n != 0) return 0;
  int32_t secs = hours * 3600 + minutes * 60;
  *off = neg ? -secs : secs;
  return 1;
}
static uint32_t parse_date(const uint8_t* s, uint64_t n, orc_cell* c) {
  cur_t cu = {s, n}; int64_t days;
  if (!parse_date_part(&cu, &days) || cu.n != 0) return ETL_E_DATETIME;
  c->tag = ETL_CELL_DATE; c->val = (uint64_t)days; c->aux = 0; return 0;
}
static uint32_t parse_time(const uint8_t* s, uint64_t n, orc_cell* c) {
  cur_t cu = {s, n}; int64_t secs; uint32_t ns;
  if (!parse_time_part(&cu, &secs, &ns) || cu.n != 0) return ETL_E_DATETIME;
  c->tag = ETL_CELL_TIME; c->val = (uint64_t)secs; c->aux = ns; return 0;
}
static int parse_ts_prefix(cur_t* cu, int64_t* days, int64_t* secs, uint32_t* ns) {
  if (!parse_date_part(cu, days)) return 0;
  trim_start_ws(&cu->s, &cu->n);                           /* Item::Space */
  return parse_time_part(cu, secs, ns);
}
static uint32_t parse_timestamp(const uint8_t* s, uint64_t n, orc_cell* c) {
  cur_t cu = {s, n}; int64_t days, secs; uint32_t ns;
  if (!parse_ts_prefix(&cu, &days, &secs, &ns) || cu.n != 0) return ETL_E_DATETIME;
  c->tag = ETL_CELL_TIMESTAMP; c->val = (uint64_t)(days * 86400 + secs); c->aux = ns; return 0;
}
static int parse_timestamptz_fmt(const uint8_t* s, uint64_t n, int permissive, orc_cell* c) {
  cur_t cu = {s, n}; int64_t days, secs; uint32_t ns; int32_t off;
  if (!parse_ts_prefix(&cu, &days, &secs, &ns)) return 0;
  if (!parse_tz(&cu, permissive, permissive, &off)) return 0;
  if (cu.n != 0) return 0;
  if (off <= -86400 || off >= 86400) return 0;            /* FixedOffset::east_opt */
  int64_t utc = days * 86400 + secs - off;
  /* from_local_datetime → checked_sub_offset must stay inside NaiveDate::{MIN,MAX} */
  int64_t lo = days_from_civil(-262143, 1, 1) * 86400, hi = (days_from_civil(262142, 12, 31) + 1) * 86400;
  if (utc < lo || utc >= hi) return 0;
  c->tag = ETL_CELL_TIMESTAMPTZ; c->val = (uint64_t)utc; c->aux = ns;
  return 1;
}
static uint32_t parse_timestamptz(const uint8_t* s, uint64_t n, orc_cell* c) {
  if (parse_timestamptz_fmt(s, n, 1, c)) return 0;        /* text.rs:111 %#z */
  if (parse_timestamptz_fmt(s, n, 0, c)) return 0;        /* text.rs:113 %:z */
  return ETL_E_DATETIME;
}

/* ------------------------------------------------------------------ uuid 1.x Uuid::parse_str
 * text.rs:141-149. simple (32), hyphenated (36), braced hyphenated (38), urn:uuid: (45). */
static uint32_t parse_uuid(const uint8_t* s, uint64_t n, orc_heap* heap, orc_cell* c) {
  uint8_t out[16];
  if (n == 38 && s[0] == '{' && s[37] == '}') { s++; n = 36; }
  else if (n == 45 && memcmp(s, "urn:uuid:", 9) == 0) { s += 9; n = 36; }
  if (n == 32) {
    for (int i = 0; i < 16; i++) {
      int a = hexval(s[2 * i]), b = hexval(s[2 * i + 1]);
      if (a < 0 || b < 0) return ETL_E_UUID;
      out[i] = (uint8_t)(a * 16 + b);
    }
  } else if (n == 36) {
    if (s[8] != '-' || s[13] != '-' || s[18] != '-' || s[23] != '-') return ETL_E_UUID;
    int k = 0;
    for (int i = 0; i < 36;) {
      if (i == 8 || i == 13 || i == 18 || i == 23) { i++; continue; }
      int a = hexval(s[i]), b = hexval(s[i + 1]);
      if (a < 0 || b < 0) return ETL_E_UUID;
      out[k++] = (uint8_t)(a * 16 + b); i += 2;
    }
  } else return ETL_E_UUID;
  uint64_t off = orc_heap_alloc(heap, 16, 8);
  memcpy(heap->data + off, out, 16);
  c->tag = ETL_CELL_UUID; c->val = off; c->aux = 16;
  return 0;
}

/* ------------------------------------------------------------------ serde_json::from_str::<Value>
 * text.rs:150-153. RFC 8259 grammar; numbers unrestricted in magnitude (arbitrary_precision);
 * strings: no raw control chars, escapes validated incl. surrogate pairing; whitespace = SP HT LF CR;
 * recursion limit 128 (remaining_depth hits 0 on the 128th nested container). */
typedef struct { const uint8_t* s; uint64_t n, i; int depth; } js_t;
static void js_ws(js_t* j) { while (j->i < j->n && (j->s[j->i] == ' ' || j->s[j->i] == '\t' || j->s[j->i] == '\n' || j->s[j->i] == '\r')) j->i++; }
static int js_hex4(js_t* j, uint32_t* out) {
  if (j->i + 4 > j->n) return 0;
  uint32_t v = 0;
  for (int k = 0; k < 4; k++) { int h = hexval(j->s[j->i + k]); if (h < 0) return 0; v = v * 16 + (uint32_t)h; }
  j->i += 4; *out = v; return 1;
}
static int js_string(js_t* j) { /* at opening quote */
  j->i++;
  for (;;) {
    if (j->i >= j->n) return 0;
    uint8_t ch = j->s[j->i];
    if (ch == '"') { j->i++; return 1; }
    if (ch < 0x20) return 0;
    if (ch == '\\') {
      j->i++;
      if (j->i >= j->n) return 0;
      uint8_t e = j->s[j->i++];
      switch (e) {
        case '"': case '\\': case '/': case 'b': case 'f': case 'n': case 'r': case 't': break;
        case 'u': {
          uint32_t u;
          if (!js_hex4(j, &u)) return 0;
          if (u >= 0xDC00 && u <= 0xDFFF) return 0;         /* lone trailing surrogate */
          if (u >= 0xD800 && u <= 0xDBFF) {
            if (j->i + 2 > j->n || j->s[j->i] != '\\' || j->s[j->i + 1] != 'u') return 0;
            j->i += 2;
            uint32_t u2;
            if (!js_hex4(j, &u2)) return 0;
            if (u2 < 0xDC00 || u2 > 0xDFFF) return 0;
          }
          break;
        }
        default: return 0;
      }
      continue;
    }
    j->i++;
  }
}
static int js_number(js_t* j) {
  if (j->i < j->n && j->s[j->i] == '-') j->i++;
  if (j->i >= j->n) return 0;
  if (j->s[j->i] == '0') { j->i++; if (j->i < j->n && is_digit(j->s[j->i])) return 0; }
  else if (j->s[j->i] >= '1' && j->s[j->i] <= '9') { while (j->i < j->n && is_digit(j->s[j->i])) j->i++; }
  else return 0;
  if (j->i < j->n && j->s[j->i] == '.') {
    j->i++;
    if (!(j->i < j->n && is_digit(j->s[j->i]))) return 0;
    while (j->i < j->n && is_digit(j->s[j->i])) j->i++;
  }
  if (j->i < j->n && (j->s[j->i] == 'e' || j->s[j->i] == 'E')) {
    j->i++;
    if (j->i < j->n && (j->s[j->i] == '+' || j->s[j->i] == '-')) j->i++;
    if (!(j->i < j->n && is_digit(j->s[j->i]))) return 0;
    while (j->i < j->n && is_digit(j->s[j->i])) j->i++;
  }
  return 1;
}
static int js_lit(js_t* j, const char* w) {
  uint64_t m = strlen(w);
  if (j->i + m > j->n || memcmp(j->s + j->i, w, m) != 0) return 0;
  j->i += m; return 1;
}
static int js_value(js_t* j) {
  js_ws(j);
  if (j->i >= j->n) return 0;
  uint8_t ch = j->s[j->i];
  switch (ch) {
    case 'n': return js_lit(j, "null");
    case 't': return js_lit(j, "true");
    case 'f': return js_lit(j, "false");
    case '"': return js_string(j);
    case '[': {
      if (--j->depth == 0) return 0;
      j->i++; js_ws(j);
      if (j->i < j->n && j->s[j->i] == ']') { j->i++; j->depth++; return 1; }
      for (;;) {
        if (!js_value(j)) return 0;
        js_ws(j);
        if (j->i >= j->n) return 0;
        if (j->s[j->i] == ',') { j->i++; continue; }
        if (j->s[j->i] == ']') { j->i++; j->depth++; return 1; }
        return 0;
      }
    }
    case '{': {
      if (--j->depth == 0) return 0;
      j->i++; js_ws(j);
      if (j->i < j->n && j->s[j->i] == '}') { j->i++; j->depth++; return 1; }
      for (;;) {
        js_ws(j);
        if (j->i >= j->n || j->s[j->i] != '"') return 0;
        if (!js_string(j)) return 0;
        js_ws(j);
        if (j->i >= j->n || j->s[j->i] != ':') return 0;
        j->i++;
        if (!js_value(j)) return 0;
        js_ws(j);
        if (j->i >= j->n) return 0;
        if (j->s[j->i] == ',') { j->i++; continue; }
        if (j->s[j->i] == '}') { j->i++; j->depth++; return 1; }
        return 0;
      }
    }
    default:
      if (ch == '-' || is_digit(ch)) return js_number(j);
      return 0;
  }
}
int orc_json_valid(const uint8_t* s, uint64_t n) {
  js_t j = {s, n, 0, 128};
  if (!js_value(&j)) return 0;
  js_ws(&j);
  return j.i == n;
}

/* ------------------------------------------------------------------ scalar dispatch text.rs:28-173 */
static uint32_t parse_scalar(uint32_t kind, const uint8_t* s, uint64_t n, uint64_t stream_off,
                             orc_heap* heap, orc_cell* c, int in_array) {
  int64_t iv;
  uint32_t e;
  c->aux = 0;
  switch (kind) {
    case ETL_K_BOOL: return parse_bool(s, n, c);
    case ETL_K_STRING:
      c->tag = ETL_CELL_STRING;
      if (in_array) { uint64_t off = orc_heap_alloc(heap, n, 8); if (n) memcpy(heap->data + off, s, n); c->val = off; }
      else c->val = stream_off;
      c->aux = (uint32_t)n; return 0;
    case ETL_K_I16: e = parse_int(s, n, 1, INT16_MIN, INT16_MAX, &iv); if (e) return e; c->tag = ETL_CELL_I16; c->val = (uint64_t)iv; return 0;
    case ETL_K_I32: e = parse_int(s, n, 1, INT32_MIN, INT32_MAX, &iv); if (e) return e; c->tag = ETL_CELL_I32; c->val = (uint64_t)iv; return 0;
    case ETL_K_I64: e = parse_int(s, n, 1, INT64_MIN, INT64_MAX, &iv); if (e) return e; c->tag = ETL_CELL_I64; c->val = (uint64_t)iv; return 0;
    case ETL_K_U32: e = parse_int(s, n, 0, 0, UINT32_MAX, &iv); if (e) return e; c->tag = ETL_CELL_U32; c->val = (uint64_t)iv; return 0;
    case ETL_K_F32: return parse_f32(s, n, c);
    case ETL_K_F64: return parse_f64(s, n, c);
    case ETL_K_NUMERIC: return parse_numeric(s, n, heap, c);
    case ETL_K_BYTES: return parse_bytea(s, n, heap, c);
    case ETL_K_DATE: return parse_date(s, n, c);
    case ETL_K_TIME: return parse_time(s, n, c);
    case ETL_K_TIMESTAMP: return parse_timestamp(s, n, c);
    case ETL_K_TIMESTAMPTZ: return parse_timestamptz(s, n, c);
    case ETL_K_UUID: return parse_uuid(s, n, heap, c);
    case ETL_K_JSON:
      if (!orc_json_valid(s, n)) return ETL_E_JSON;
      c->tag = ETL_CELL_JSON;
      if (in_array) { uint64_t off = orc_heap_alloc(heap, n, 8); if (n) memcpy(heap->data + off, s, n); c->val = off; }
      else c->val = stream_off;
      c->aux = (uint32_t)n; return 0;
    default: return ETL_E_MALFORMED_FRAME;
  }
}

/* ------------------------------------------------------------------ arrays text.rs:184-249
 * One-dimensional split; `"` toggles quoting, `\` escapes the next char, `,` splits outside
 * quotes, unquoted case-insensitive NULL is a null element. TIMESTAMPTZ arrays are retried whole
 * with the second format (text.rs:117-140). */
static uint32_t parse_array_once(uint32_t ekind, const uint8_t* s, uint64_t n, orc_heap* heap,
                                 orc_cell* c, int tz_fmt /*0 both-per-elem n/a; 1 permissive; 2 colon*/) {
  if (n < 2) return ETL_E_ARRAY_SHORT;
  if (s[0] != '{' || s[n - 1] != '}') return ETL_E_ARRAY_BRACES;
  const uint8_t* p = s + 1;
  uint64_t m = n - 2;
  /* elements are collected first (heap may move) */
  uint64_t cap = 8, cnt = 0;
  orc_cell* elems = (orc_cell*)malloc(cap * sizeof(orc_cell));
  uint8_t* val = (uint8_t*)malloc(m + 1);
  uint64_t vl = 0;
  int in_quotes = 0, in_escape = 0, val_quoted = 0;
  int done = (m == 0);
  uint64_t i = 0;
  uint32_t err = 0;
  while (!done) {
    for (;;) {
      if (i >= m) { done = 1; break; }
      /* chars(): copy a whole UTF-8 scalar at a time; only ASCII chars are structural */
      uint8_t ch = p[i];
      uint32_t clen = ch < 0x80 ? 1 : (ch >= 0xF0 ? 4 : (ch >= 0xE0 ? 3 : 2));
      if (in_escape) { memcpy(val + vl, p + i, clen); vl += clen; i += clen; in_escape = 0; continue; }
      if (ch == '"') { if (!in_quotes) val_quoted = 1; in_quotes = !in_quotes; i++; continue; }
      if (ch == '\\') { in_escape = 1; i++; continue; }
      if (ch == ',' && !in_quotes) { i++; break; }
      memcpy(val + vl, p + i, clen); vl += clen; i += clen;
    }
    orc_cell e; memset(&e, 0, sizeof e);
    if (!val_quoted && ieq(val, vl, "null")) { e.tag = ETL_CELL_NULL; }
    else {
      if (ekind == ETL_K_TIMESTAMPTZ) {
        if (!parse_timestamptz_fmt(val, vl, tz_fmt == 1, &e)) err = ETL_E_DATETIME;
      } else err = parse_scalar(ekind, val, vl, 0, heap, &e, 1);
      if (err) break;
    }
    if (cnt == cap) { cap *= 2; elems = (orc_cell*)realloc(elems, cap * sizeof(orc_cell)); }
    elems[cnt++] = e;
    vl = 0; val_quoted = 0;
  }
  free(val);
  if (err) { free(elems); return err; }
  uint64_t off = orc_heap_alloc(heap, sizeof(etl_array_hdr) + cnt * sizeof(etl_array_elem), 8);
  etl_array_hdr h; memset(&h, 0, sizeof h);
  h.elem_kind = (uint8_t)ekind; h.n_elems = (uint32_t)cnt;
  memcpy(heap->data + off, &h, sizeof h);
  for (uint64_t k = 0; k < cnt; k++) {
    etl_array_elem ae; memset(&ae, 0, sizeof ae);
    ae.val = elems[k].val; ae.aux = elems[k].aux; ae.tag = elems[k].tag;
    memcpy(heap->data + off + sizeof h + k * sizeof ae, &ae, sizeof ae);
  }
  free(elems);
  c->tag = ETL_CELL_ARRAY; c->val = off; c->aux = (uint32_t)cnt;
  return 0;
}

uint32_t orc_parse_text(uint32_t kind, const uint8_t* s, uint64_t n, uint64_t stream_off,
                        orc_heap* heap, orc_cell* c) {
  if (kind & ETL_K_ARRAY) {
    uint32_t ek = kind & ~(uint32_t)ETL_K_ARRAY;
    if (ek == ETL_K_TIMESTAMPTZ) {
      uint64_t mark = heap->len;
      uint32_t e = parse_array_once(ek, s, n, heap, c, 1);
      if (!e) return 0;
      heap->len = mark;
      return parse_array_once(ek, s, n, heap, c, 2);
    }
    return parse_array_once(ek, s, n, heap, c, 0);
  }
  return parse_scalar(kind, s, n, stream_off, heap, c, 0);
}

uint32_t orc_parse_cell(uint32_t type_oid, const uint8_t* text, uint32_t len, uint8_t* tag,
                        uint64_t* val, uint32_t* aux, uint8_t* heap_out, uint32_t heap_cap,
                        uint32_t* heap_len) {
  orc_heap h = {0, 0, 0};
  orc_cell c; memset(&c, 0, sizeof c);
  uint32_t e;
  if (!orc_utf8_valid(text, len)) e = ETL_E_UTF8;          /* event.rs:972 */
  else e = orc_parse_text(orc_kind_for_oid(type_oid), text, len, 0, &h, &c);
  *tag = c.tag; *val = c.val; *aux = c.aux;
  uint64_t nl = h.len < heap_cap ? h.len : heap_cap;
  if (nl && heap_out) memcpy(heap_out, h.data, nl);
  if (heap_len) *heap_len = (uint32_t)h.len;
  free(h.data);
  return e;
}
