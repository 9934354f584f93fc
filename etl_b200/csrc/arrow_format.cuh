// arrow_format.cuh — device formatters of the columnar emitter (arrow_emit.cu) for the column types whose Arrow value is
// text the reference formats on the host (crates/etl-destinations/src/iceberg/encoding.rs cell_to_string and the string
// list builders):
//   * Numeric → PgNumeric's Display (crates/etl/src/conversions/numeric.rs:503-590): numeric_len / numeric_write over
//     the heap's etl_numeric_hdr and its base-10000 digits;
//   * Json → serde_json::Value's Display (`to_string`) as the etl crate builds serde_json (arbitrary_precision, no
//     preserve_order): compact, object keys sorted by their unescaped UTF-8 bytes, the last of duplicate keys wins,
//     numbers verbatim, strings unescaped and escaped again the serde_json way.  json_canon; the same model as json_dump
//     in shim_materialise.cpp (third-party behaviour: parity unpinned, DESIGN §5).
// Plain functions over (pointer, length), one thread each, no warp intrinsics: tests/emul/host_format.cpp compiles this
// very file for the host and fuzzes it against Python restatements.
#pragma once
#include <stdint.h>

#include "etl_decode.h"

namespace etl_fmt {

// ------------------------------------------------------------------------------------------------ Numeric
__device__ __forceinline__ uint32_t numeric_group(const uint8_t* num, uint32_t nd, int32_t d) {
  if (d < 0 || (uint32_t)d >= nd) return 0u;     // a group past the digits (or before the first) counts as 0000
  return (uint32_t)reinterpret_cast<const int16_t*>(num + sizeof(etl_numeric_hdr))[d];
}
__device__ __forceinline__ uint32_t dec_width(uint32_t g) { return g >= 1000u ? 4u : (g >= 100u ? 3u : (g >= 10u ? 2u : 1u)); }

// bytes of the Display text of the numeric at `num` (heap, 8-byte aligned) with `nd` base-10000 digits; from the header
// and the first group only
__device__ __forceinline__ uint32_t numeric_len(const uint8_t* num, uint32_t nd) {
  const etl_numeric_hdr h = *reinterpret_cast<const etl_numeric_hdr*>(num);
  if (h.kind == 1) return 3u;                    // NaN
  if (h.kind == 2) return 8u;                    // Infinity
  if (h.kind == 3) return 9u;                    // -Infinity
  if (nd == 0) return 1u;                        // "0" whatever the sign and scale
  uint32_t n = h.sign ? 1u : 0u;
  if (h.weight < 0) n += 1u;
  else n += dec_width(numeric_group(num, nd, 0)) + 4u * (uint32_t)h.weight;
  if (h.scale) n += 1u + h.scale;
  return n;
}
// writes exactly numeric_len(num, nd) bytes
__device__ __forceinline__ uint32_t numeric_write(const uint8_t* num, uint32_t nd, uint8_t* out) {
  const etl_numeric_hdr h = *reinterpret_cast<const etl_numeric_hdr*>(num);
  const char* lit = h.kind == 1 ? "NaN" : (h.kind == 2 ? "Infinity" : (h.kind == 3 ? "-Infinity" : nullptr));
  if (lit) { uint32_t o = 0; while (lit[o]) { out[o] = (uint8_t)lit[o]; o++; } return o; }
  if (nd == 0) { out[0] = '0'; return 1u; }
  uint32_t o = 0;
  if (h.sign) out[o++] = '-';
  if (h.weight < 0) out[o++] = '0';
  else {
    const uint32_t g0 = numeric_group(num, nd, 0), w0 = dec_width(g0);   // the first group without its leading zeros
    uint32_t t = g0;
    for (uint32_t k = w0; k-- > 0;) { out[o + k] = (uint8_t)('0' + t % 10u); t /= 10u; }
    o += w0;
    for (int32_t d = 1; d <= h.weight; d++) {
      uint32_t g = numeric_group(num, nd, d);
      for (int k = 3; k >= 0; k--) { out[o + k] = (uint8_t)('0' + g % 10u); g /= 10u; }
      o += 4u;
    }
  }
  if (h.scale) {
    out[o++] = '.';
    uint32_t rem = h.scale;
    for (int32_t d = (int32_t)h.weight + 1; rem > 0; d++) {
      const uint32_t g = numeric_group(num, nd, d);
      const uint32_t take = rem < 4u ? rem : 4u;
      const uint32_t pw[4] = {1000u, 100u, 10u, 1u};
      for (uint32_t k = 0; k < take; k++) out[o++] = (uint8_t)('0' + (g / pw[k]) % 10u);
      rem -= take;
    }
  }
  return o;
}

// ------------------------------------------------------------------------------------------------ Json
// The canonical text is never longer than the input (whitespace and duplicate members are dropped, `\/` becomes `/`,
// `\uXXXX` becomes at most 4 bytes, a control character's escape gets no longer), so the output buffer has n bytes.
// `work` holds json_canon_work_words(n) 32-bit words: the value nodes of the document in pre-order (start offset,
// index of the node after its subtree, offset of its key when it is an object member), the member lists of the open
// objects and a 128-frame stack.  Returns the output length, or kJsonCanonBad for input json_valid would have rejected.
constexpr uint32_t kJsonCanonBad = 0xFFFFFFFFu;
constexpr uint32_t kJsonMaxDepth = 128u;
constexpr uint32_t kNoKey = 0xFFFFFFFFu;
__device__ __forceinline__ uint64_t json_canon_node_cap(uint64_t n) { return n / 2u + 2u; }   // a value takes >= 1 byte and a separator
// nodes (3 words each), member lists (1 word per node), 4 words per stack frame: <= 4n + 16 words
__device__ __forceinline__ uint64_t json_canon_work_words(uint64_t n) {
  const uint64_t cap = json_canon_node_cap(n);
  return 4u * cap + 4u * (cap < kJsonMaxDepth ? cap : kJsonMaxDepth);
}

__device__ __forceinline__ bool json_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool json_num_char(uint8_t c) { return (c >= '0' && c <= '9') || c == '-' || c == '+' || c == '.' || c == 'e' || c == 'E'; }
__device__ __forceinline__ bool json_scalar_char(uint8_t c) { return json_num_char(c) || (c >= 'a' && c <= 'z'); }   // numbers, true / false / null
__device__ __forceinline__ int json_hex4(const uint8_t* q) {
  int v = 0;
  for (int k = 0; k < 4; k++) {
    const uint32_t c = q[k];
    int h;
    if (c - '0' <= 9u) h = (int)(c - '0');
    else if ((c | 32u) - 'a' <= 5u) h = (int)((c | 32u) - 'a' + 10u);
    else return -1;
    v = v * 16 + h;
  }
  return v;
}
// code point of the \u escape at s[i] ('\\' 'u' already consumed up to i = first hex digit); advances i; -1 = bad
__device__ __forceinline__ int32_t json_u_escape(const uint8_t* s, uint32_t n, uint32_t* i) {
  if (*i + 4u > n) return -1;
  int32_t u = json_hex4(s + *i);
  *i += 4u;
  if (u < 0 || (u >= 0xDC00 && u <= 0xDFFF)) return -1;
  if (u >= 0xD800 && u <= 0xDBFF) {
    if (*i + 6u > n || s[*i] != '\\' || s[*i + 1] != 'u') return -1;
    const int32_t lo = json_hex4(s + *i + 2);
    if (lo < 0xDC00 || lo > 0xDFFF) return -1;
    *i += 6u;
    u = 0x10000 + ((u - 0xD800) << 10) + (lo - 0xDC00);
  }
  return u;
}
__device__ __forceinline__ uint32_t json_utf8(uint32_t c, uint8_t* b) {
  if (c < 0x80u) { b[0] = (uint8_t)c; return 1; }
  if (c < 0x800u) { b[0] = (uint8_t)(0xC0u | (c >> 6)); b[1] = (uint8_t)(0x80u | (c & 63u)); return 2; }
  if (c < 0x10000u) { b[0] = (uint8_t)(0xE0u | (c >> 12)); b[1] = (uint8_t)(0x80u | ((c >> 6) & 63u)); b[2] = (uint8_t)(0x80u | (c & 63u)); return 3; }
  b[0] = (uint8_t)(0xF0u | (c >> 18)); b[1] = (uint8_t)(0x80u | ((c >> 12) & 63u)); b[2] = (uint8_t)(0x80u | ((c >> 6) & 63u)); b[3] = (uint8_t)(0x80u | (c & 63u));
  return 4;
}
// skips the string whose opening quote is at s[*i]
__device__ __forceinline__ bool json_skip_string(const uint8_t* s, uint32_t n, uint32_t* i) {
  uint32_t j = *i + 1u;
  while (j < n) {
    const uint8_t c = s[j];
    if (c == '"') { *i = j + 1u; return true; }
    if (c == '\\') { j += 2u; continue; }
    if (c < 0x20u) return false;
    j++;
  }
  return false;
}

// unescaped bytes of a key, one at a time; -1 at the closing quote (or at malformed input: emission flags that)
struct JsonKeyCursor {
  uint32_t i;
  uint8_t buf[4];
  uint32_t bl, bp;
};
__device__ __forceinline__ int json_key_next(const uint8_t* s, uint32_t n, JsonKeyCursor& k) {
  if (k.bp < k.bl) return k.buf[k.bp++];
  if (k.i >= n) return -1;
  const uint8_t c = s[k.i];
  if (c == '"') return -1;
  if (c != '\\') { k.i++; return c; }
  if (k.i + 1u >= n) return -1;
  const uint8_t e = s[k.i + 1];
  k.i += 2u;
  switch (e) {
    case 'b': return '\b';
    case 'f': return '\f';
    case 'n': return '\n';
    case 'r': return '\r';
    case 't': return '\t';
    case 'u': {
      const int32_t u = json_u_escape(s, n, &k.i);
      if (u < 0) return -1;
      k.bl = json_utf8((uint32_t)u, k.buf);
      k.bp = 1;
      return k.buf[0];
    }
    default: return e;              // '"', '\\', '/'
  }
}
// order of two keys (offsets of their opening quotes) by unescaped UTF-8 bytes: raw bytes while neither has reached a
// backslash, the decoding cursor from there on (the bytes before it were equal and literal in both)
__device__ __forceinline__ int json_key_cmp(const uint8_t* s, uint32_t n, uint32_t a, uint32_t b) {
  uint32_t i = a + 1u, j = b + 1u;
  for (;;) {
    const uint8_t ca = i < n ? s[i] : (uint8_t)'"', cb = j < n ? s[j] : (uint8_t)'"';
    if (ca == '\\' || cb == '\\') break;
    if (ca == '"' || cb == '"') return ca == '"' ? (cb == '"' ? 0 : -1) : 1;
    if (ca != cb) return ca < cb ? -1 : 1;
    i++; j++;
  }
  JsonKeyCursor x{i, {0, 0, 0, 0}, 0, 0}, y{j, {0, 0, 0, 0}, 0, 0};
  for (;;) {
    const int p = json_key_next(s, n, x), q = json_key_next(s, n, y);
    if (p != q) return p < q ? -1 : 1;
    if (p < 0) return 0;
  }
}
// members sorted by (key, node index): equal keys end with the last one written, which is the one kept
__device__ __forceinline__ bool json_member_less(const uint8_t* s, uint32_t n, const uint32_t* N, uint32_t a, uint32_t b) {
  const int c = json_key_cmp(s, n, N[3u * a + 2u], N[3u * b + 2u]);
  return c < 0 || (c == 0 && a < b);
}
__device__ __forceinline__ void json_sort_members(const uint8_t* s, uint32_t n, const uint32_t* N, uint32_t* M, uint32_t cnt) {
  // heap sort: O(m log m) and no extra memory, for objects of any width
  auto sift = [&](uint32_t root, uint32_t end) {
    for (;;) {
      uint32_t c = 2u * root + 1u;
      if (c >= end) return;
      if (c + 1u < end && json_member_less(s, n, N, M[c], M[c + 1u])) c++;
      if (!json_member_less(s, n, N, M[root], M[c])) return;
      const uint32_t t = M[root]; M[root] = M[c]; M[c] = t;
      root = c;
    }
  };
  for (uint32_t r = cnt / 2u; r-- > 0;) sift(r, cnt);
  for (uint32_t end = cnt; end > 1u; end--) {
    const uint32_t t = M[0]; M[0] = M[end - 1u]; M[end - 1u] = t;
    sift(0, end - 1u);
  }
}

__device__ inline uint32_t json_canon(const uint8_t* s, uint32_t n, uint8_t* out, uint32_t* work) {
  const uint32_t cap = (uint32_t)json_canon_node_cap(n);
  uint32_t* N = work;                 // 3 words per node
  uint32_t* M = work + 3u * cap;      // member lists of the open objects
  uint32_t* F = M + cap;              // stack: 4 words per frame, at most min(cap, 127) frames
  uint32_t i = 0, nn = 0, sp = 0;
  // ---- pass 1: nodes in pre-order
  auto ws = [&]() { while (i < n && json_ws(s[i])) i++; };
  auto key = [&](uint32_t* k) -> bool {     // key, ':' and the whitespace around them
    if (i >= n || s[i] != '"') return false;
    *k = i;
    if (!json_skip_string(s, n, &i)) return false;
    ws();
    if (i >= n || s[i] != ':') return false;
    i++;
    ws();
    return true;
  };
  uint32_t pending = kNoKey;
  ws();
  for (;;) {
    // a value starts at i
    if (i >= n || nn >= cap) return kJsonCanonBad;
    const uint32_t v = nn++;
    N[3u * v] = i; N[3u * v + 2u] = pending; pending = kNoKey;
    const uint8_t c = s[i];
    bool closed = true;
    if (c == '{' || c == '[') {
      if (sp >= kJsonMaxDepth - 1u || sp + 1u >= cap) return kJsonCanonBad;
      i++;
      ws();
      if (i < n && s[i] == (c == '{' ? '}' : ']')) i++;
      else {
        F[sp++] = v;
        if (c == '{' && !key(&pending)) return kJsonCanonBad;
        closed = false;
      }
    } else if (c == '"') {
      if (!json_skip_string(s, n, &i)) return kJsonCanonBad;
    } else if (c == 't' || c == 'f' || c == 'n') {
      const char* lit = c == 't' ? "true" : (c == 'f' ? "false" : "null");
      for (uint32_t k = 0; lit[k]; k++, i++) if (i >= n || s[i] != (uint8_t)lit[k]) return kJsonCanonBad;
    } else {
      const uint32_t j = i;
      while (i < n && json_num_char(s[i])) i++;
      if (i == j) return kJsonCanonBad;
    }
    if (!closed) continue;
    N[3u * v + 1u] = nn;
    // after a complete value: separators and closing brackets
    bool more = false;
    for (;;) {
      ws();
      if (sp == 0) { if (i != n) return kJsonCanonBad; break; }
      const uint32_t t = F[sp - 1u];
      const bool obj = s[N[3u * t]] == '{';
      if (i < n && s[i] == ',') {
        i++;
        ws();
        if (obj && !key(&pending)) return kJsonCanonBad;
        more = true;
        break;
      }
      if (i < n && s[i] == (obj ? '}' : ']')) { i++; sp--; N[3u * t + 1u] = nn; continue; }
      return kJsonCanonBad;
    }
    if (!more) break;
  }
  // ---- pass 2: emit, members of each object in key order
  uint32_t o = 0, mtop = 0, v = 0;
#define JPUT(b) do { if (o >= n) return kJsonCanonBad; out[o++] = (uint8_t)(b); } while (0)
  auto put_esc = [&](uint32_t c) -> bool {         // one byte < 0x80 of an unescaped string, escaped the serde_json way
    const char* sh = c == '"' ? "\\\"" : c == '\\' ? "\\\\" : c == '\n' ? "\\n" : c == '\r' ? "\\r" : c == '\t' ? "\\t" :
                     c == '\b' ? "\\b" : c == '\f' ? "\\f" : nullptr;
    if (sh) { if (o + 2u > n) return false; out[o++] = (uint8_t)sh[0]; out[o++] = (uint8_t)sh[1]; return true; }
    if (c < 0x20u) {
      if (o + 6u > n) return false;
      const char* hx = "0123456789abcdef";
      out[o++] = '\\'; out[o++] = 'u'; out[o++] = '0'; out[o++] = '0'; out[o++] = (uint8_t)hx[c >> 4]; out[o++] = (uint8_t)hx[c & 15u];
      return true;
    }
    if (o >= n) return false;
    out[o++] = (uint8_t)c;
    return true;
  };
  auto put_string = [&](uint32_t at) -> bool {     // the string whose opening quote is at s[at]
    uint32_t j = at + 1u;
    if (o >= n) return false;
    out[o++] = '"';
    for (;;) {
      if (j >= n) return false;
      const uint8_t c = s[j];
      if (c == '"') break;
      if (c < 0x20u) return false;
      if (c != '\\') { if (o >= n) return false; out[o++] = c; j++; continue; }
      if (j + 1u >= n) return false;
      const uint8_t e = s[j + 1];
      j += 2u;
      uint32_t u;
      switch (e) {
        case '"': u = '"'; break;
        case '\\': u = '\\'; break;
        case '/': u = '/'; break;
        case 'b': u = '\b'; break;
        case 'f': u = '\f'; break;
        case 'n': u = '\n'; break;
        case 'r': u = '\r'; break;
        case 't': u = '\t'; break;
        case 'u': { const int32_t x = json_u_escape(s, n, &j); if (x < 0) return false; u = (uint32_t)x; break; }
        default: return false;
      }
      if (u < 0x80u) { if (!put_esc(u)) return false; }
      else {
        uint8_t b[4];
        const uint32_t k = json_utf8(u, b);
        if (o + k > n) return false;
        for (uint32_t q = 0; q < k; q++) out[o++] = b[q];
      }
    }
    if (o >= n) return false;
    out[o++] = '"';
    return true;
  };
  for (;;) {
    const uint32_t at = N[3u * v];
    const uint8_t c = s[at];
    if (c == '{') {
      JPUT('{');
      const uint32_t mb = mtop;
      for (uint32_t ch = v + 1u; ch < N[3u * v + 1u]; ch = N[3u * ch + 1u]) M[mtop++] = ch;
      json_sort_members(s, n, N, M + mb, mtop - mb);
      F[4u * sp] = v; F[4u * sp + 1u] = mb; F[4u * sp + 2u] = mtop; F[4u * sp + 3u] = mb;
      sp++;
    } else if (c == '[') {
      JPUT('[');
      F[4u * sp] = v; F[4u * sp + 1u] = v + 1u; F[4u * sp + 2u] = N[3u * v + 1u]; F[4u * sp + 3u] = 0;
      sp++;
    } else if (c == '"') {
      if (!put_string(at)) return kJsonCanonBad;
    } else {
      for (uint32_t j = at; j < n && json_scalar_char(s[j]); j++) JPUT(s[j]);
    }
    // the next value to emit, closing the containers that are done
    for (;;) {
      if (sp == 0) return o;
      uint32_t* fr = F + 4u * (sp - 1u);
      if (s[N[3u * fr[0]]] == '[') {
        if (fr[1] < fr[2]) {
          if (out[o - 1u] != '[') JPUT(',');
          v = fr[1];
          fr[1] = N[3u * v + 1u];
          break;
        }
        JPUT(']');
        sp--;
      } else {
        while (fr[1] + 1u < fr[2] && json_key_cmp(s, n, N[3u * M[fr[1]] + 2u], N[3u * M[fr[1] + 1u] + 2u]) == 0) fr[1]++;
        if (fr[1] < fr[2]) {
          if (out[o - 1u] != '{') JPUT(',');
          v = M[fr[1]++];
          if (!put_string(N[3u * v + 2u])) return kJsonCanonBad;
          JPUT(':');
          break;
        }
        JPUT('}');
        mtop = fr[3];
        sp--;
      }
    }
  }
#undef JPUT
}

// ------------------------------------------------------------------------------------------------ CDC columns
// EventSequenceKey's Display (crates/etl/src/types/event.rs:331-336): "{commit_lsn:016x}/{tx_ordinal:016x}", always
// kSeqKeyLen bytes; generate_sequence_number(0, 0) of a table-copy row (etl-postgres/src/types/utils.rs:119-139) is the
// key of (0, 0).  Every cdc_operation name ("INSERT" / "UPDATE" / "DELETE") is kCdcOpLen bytes.
constexpr uint32_t kSeqKeyLen = 33, kCdcOpLen = 6;
__device__ __forceinline__ void hex16_write(uint64_t v, uint8_t* out) {
  for (int k = 15; k >= 0; k--) {
    const uint32_t d = (uint32_t)(v & 15u);
    out[k] = (uint8_t)(d < 10u ? '0' + d : 'a' - 10u + d);
    v >>= 4;
  }
}
__device__ __forceinline__ void seq_key_write(uint64_t commit_lsn, uint64_t tx_ordinal, uint8_t* out) {
  hex16_write(commit_lsn, out);
  out[16] = '/';
  hex16_write(tx_ordinal, out + 17);
}
// the cdc_operation of a record kind: 'U' → UPDATE, 'D' → DELETE, anything else (an insert, a COPY row) → INSERT
__device__ __forceinline__ void cdc_op_write(uint32_t rec_kind, uint8_t* out) {
  const char* s = rec_kind == 'U' ? "UPDATE" : (rec_kind == 'D' ? "DELETE" : "INSERT");
  for (uint32_t k = 0; k < kCdcOpLen; k++) out[k] = (uint8_t)s[k];
}

}  // namespace etl_fmt
