// parquet_format.cuh — the byte-level pieces of the Parquet writer (parquet_write.cu) that a host harness can compile too
// (tests/emul/host_parquet.cpp and host_parquet_dict.cpp build this same file with g++, so the CPU suite checks it against
// tests/parquet_ref.py and tests/parquet_dict_ref.py):
//   * a Thrift compact-protocol writer (Parquet's footer and page headers): fields in ascending id order, i32 / i64 as
//     zigzag varints, binary as varint length + bytes, lists with the size in the header nibble below 15;
//   * the data page header (PageHeader {type DATA_PAGE, uncompressed_page_size, compressed_page_size, data_page_header
//     {num_values, encoding PLAIN, definition / repetition level encoding RLE}});
//   * the RLE / bit-packed hybrid level encoder with the deterministic run rule of include/etl_decode.h: entries cut into
//     groups of 8, a group is uniform when its present entries are equal, consecutive uniform groups of one value are one
//     RLE run of their exact entry count, every other stretch is bit-packed runs of at most 63 groups;
//   * the Snappy compressor of one fragment of at most 64 KiB: 4-byte hash match finder over a 4096-entry table,
//     literal / copy-1 / copy-2 elements; copies never reach outside the fragment, so fragments compress independently
//     and their element streams concatenate into one valid stream;
//   * the dictionary pieces (ETL_PQ_DICTIONARY): the DICTIONARY_PAGE header, the RLE_DICTIONARY data page header, and
//     the RLE / bit-packed hybrid of dictionary indices (bit width 1..18) under the same run rule as the levels, split
//     into the run classification and the writing of one run, so that the CTA-parallel encoder of parquet_write.cu and
//     the serial indices_encode below share them;
//   * the page index pieces (ETL_PQ_PAGE_INDEX): the 64-byte truncation of byte-array ColumnIndex bounds, the
//     PageLocation of the OffsetIndex and the header of a list field;
//   * the bloom filter pieces (etl_dec_parquet_write_bloom): XXH64 (seed 0) of a value's PLAIN bytes, the block and bit
//     masks of a split-block insert, the BloomFilterHeader, and (host only) the bitset size from ndv and fpp;
//   * the footer: FileMetaData with the schema, row groups, column chunks, statistics and column orders, for a
//     dictionary chunk its dictionary_page_offset and encoding_stats, with a page index the ColumnChunk's offset and
//     length of its OffsetIndex and ColumnIndex, and with a bloom filter its offset and length.  The schema prefix is
//     host only (the same for every file); the tail behind it (num_rows, row groups, created_by, column orders) is host
//     and device, so that etl_dec_parquet_write_files serialises every file's tail on the device;
//   * (host only) the row-group table of a multi-file write.
#pragma once
#include <stdint.h>
#include <string.h>

#include <cmath>
#include <string>
#include <vector>

namespace etl_pq {

// Parquet physical types / converted types / repetition / codecs / encodings (parquet.thrift)
enum { PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_FLOAT = 4, PT_DOUBLE = 5, PT_BYTE_ARRAY = 6, PT_FLBA = 7 };
enum { CT_UTF8 = 0, CT_LIST = 3, CT_DATE = 6, CT_TIMESTAMP_MICROS = 10, CT_NONE = -1 };
enum { REP_REQUIRED = 0, REP_OPTIONAL = 1, REP_REPEATED = 2 };
enum { ENC_PLAIN = 0, ENC_RLE = 3, ENC_RLE_DICTIONARY = 8 };
enum { PAGE_DATA = 0, PAGE_DICTIONARY = 2 };
constexpr uint32_t kPageRows = 20000;                 // a page ends after the row that brings it to this many rows
constexpr uint64_t kPageBytes = 1ull << 20;           // … or to this many PLAIN value bytes
constexpr uint64_t kRowGroupRows = 1ull << 20;
constexpr uint32_t kFragment = 65536;                 // compressed independently (Snappy, Zstandard)
constexpr uint32_t kSnappyHashBits = 12;
constexpr uint32_t kStatMax = 64;                     // a longer byte-array min / max is not written
constexpr uint32_t kPageHeaderMax = 48;               // 4 fields + a 4-field struct of i32 varints: at most 41 bytes
constexpr uint64_t kDictBytes = 1ull << 20;           // a chunk is dictionary-encoded while its entries' PLAIN size fits

__host__ __device__ inline uint32_t snappy_bound(uint32_t n) { return 32u + n + n / 6u; }
// level section bound (4-byte length prefix, runs): every group costs at most w bytes + 1 header byte of its bit-packed
// run, or 2 bytes as (part of) an RLE run; the constant covers one RLE header of up to 5 bytes
__host__ __device__ inline uint64_t levels_bound(uint64_t n, uint32_t w) { return 14u + ((n + 7u) / 8u) * (w + 2u); }
__host__ __device__ inline uint32_t bit_width(uint32_t max_level) { uint32_t w = 0; while (max_level >> w) w++; return w; }

// ------------------------------------------------------------------------------------------------ Thrift compact
__host__ __device__ inline uint32_t varint(uint64_t v, uint8_t* out) {
  uint32_t n = 0;
  while (v >= 0x80u) { if (out) out[n] = (uint8_t)(v | 0x80u); n++; v >>= 7; }
  if (out) out[n] = (uint8_t)v;
  return n + 1;
}
__host__ __device__ inline uint64_t zigzag(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }

enum { TT_TRUE = 1, TT_FALSE = 2, TT_I16 = 4, TT_I32 = 5, TT_I64 = 6, TT_BINARY = 8, TT_LIST = 9, TT_STRUCT = 12 };
// out == nullptr counts only
struct TWriter {
  uint8_t* out; uint64_t n; int16_t last[8]; int depth;
  __host__ __device__ explicit TWriter(uint8_t* o) : out(o), n(0), depth(0) { last[0] = 0; }
  __host__ __device__ void byte(uint8_t b) { if (out) out[n] = b; n++; }
  __host__ __device__ void var(uint64_t v) { n += varint(v, out ? out + n : nullptr); }
  __host__ __device__ void field(int16_t id, uint8_t type) {
    const int16_t d = id - last[depth];
    if (d > 0 && d <= 15) byte((uint8_t)((d << 4) | type));
    else { byte(type); var(zigzag(id)); }
    last[depth] = id;
  }
  __host__ __device__ void i32(int16_t id, int32_t v) { field(id, TT_I32); var(zigzag(v)); }
  __host__ __device__ void i64(int16_t id, int64_t v) { field(id, TT_I64); var(zigzag(v)); }
  __host__ __device__ void boolean(int16_t id, bool v) { field(id, v ? TT_TRUE : TT_FALSE); }
  __host__ __device__ void bin(int16_t id, const uint8_t* p, uint32_t len) {
    field(id, TT_BINARY); var(len);
    if (out && len) memcpy(out + n, p, len);
    n += len;
  }
  __host__ __device__ void begin(int16_t id) { field(id, TT_STRUCT); last[++depth] = 0; }   // nested struct
  __host__ __device__ void end() { byte(0); if (depth) depth--; }
  __host__ __device__ void list(int16_t id, uint8_t elem_type, uint32_t size) {
    field(id, TT_LIST);
    if (size < 15) byte((uint8_t)((size << 4) | elem_type));
    else { byte((uint8_t)(0xF0 | elem_type)); var(size); }
  }
  __host__ __device__ void list_struct_begin() { last[++depth] = 0; }   // one struct element of a list
};

// DATA_PAGE header (values PLAIN, or RLE_DICTIONARY indices); returns its length (at most kPageHeaderMax)
__host__ __device__ inline uint32_t page_header(uint8_t* out, uint32_t usize, uint32_t csize, uint32_t num_values,
                                                uint32_t encoding = ENC_PLAIN) {
  TWriter w(out);
  w.i32(1, PAGE_DATA);
  w.i32(2, (int32_t)usize);
  w.i32(3, (int32_t)csize);
  w.begin(5);                // data_page_header
  w.i32(1, (int32_t)num_values);
  w.i32(2, (int32_t)encoding);
  w.i32(3, ENC_RLE);
  w.i32(4, ENC_RLE);
  w.end();
  w.end();
  return (uint32_t)w.n;
}

// DICTIONARY_PAGE header {type, sizes, dictionary_page_header {num_values, encoding PLAIN}}; at most 25 bytes
__host__ __device__ inline uint32_t dict_page_header(uint8_t* out, uint32_t usize, uint32_t csize, uint32_t entries) {
  TWriter w(out);
  w.i32(1, PAGE_DICTIONARY);
  w.i32(2, (int32_t)usize);
  w.i32(3, (int32_t)csize);
  w.begin(7);                // dictionary_page_header
  w.i32(1, (int32_t)entries);
  w.i32(2, ENC_PLAIN);
  w.end();
  w.end();
  return (uint32_t)w.n;
}

// ------------------------------------------------------------------------------------------------ levels
// RLE / bit-packed hybrid of n level bytes (values < 2^w, w in 1..2), without the length prefix; returns the bytes
// written.  PRECONDITION: lv is 8-byte aligned and 8 bytes past n are readable (whole groups are loaded at once).
__host__ __device__ inline uint64_t levels_encode(const uint8_t* lv, uint64_t n, uint32_t w, uint8_t* out) {
  const uint64_t ng = (n + 7) / 8;
  uint64_t o = 0, g = 0;
  // uniform value of group g, or -1
  auto cls = [&](uint64_t k) -> int {
    const uint32_t m = (uint32_t)(n - k * 8 < 8 ? n - k * 8 : 8);
    const uint64_t x = reinterpret_cast<const uint64_t*>(lv)[k];
    const uint64_t mask = m == 8 ? ~0ull : ((1ull << (8 * m)) - 1);
    const uint64_t v = x & 0xFFu;
    return ((x ^ (v * 0x0101010101010101ull)) & mask) == 0 ? (int)v : -1;
  };
  while (g < ng) {
    const int c = cls(g);
    if (c >= 0) {                                       // RLE run: every following uniform group of the same value
      uint64_t h = g + 1;
      while (h < ng && cls(h) == c) h++;
      const uint64_t cnt = (h == ng ? n : h * 8) - g * 8;
      o += varint(cnt << 1, out + o);
      out[o++] = (uint8_t)c;
      g = h;
    } else {                                            // bit-packed: the stretch of non-uniform groups, 63 at most
      uint64_t h = g + 1;
      while (h < ng && h - g < 63 && cls(h) < 0) h++;
      out[o++] = (uint8_t)(((h - g) << 1) | 1u);
      for (uint64_t k = g; k < h; k++) {                // 8 entries → w bytes, LSB first
        uint32_t acc = 0;
        for (uint32_t j = 0; j < 8; j++) {
          const uint64_t e = k * 8 + j;
          acc |= (e < n ? (uint32_t)lv[e] : 0u) << (j * w);
        }
        for (uint32_t b = 0; b < w; b++) out[o++] = (uint8_t)(acc >> (8 * b));
      }
      g = h;
    }
  }
  return o;
}

// ------------------------------------------------------------------------------------------------ dictionary indices
// The hybrid of n indices x (bit width w = max(1, bits(entries - 1)) <= 18), without the bit-width byte or a length
// prefix, under the run rule of the levels: groups of 8; the uniform value of a group (its present entries equal) or -1.
__host__ __device__ inline int64_t idx_cls(const uint32_t* x, uint64_t n, uint64_t g) {
  const uint64_t a = g * 8, m = n - a < 8 ? n - a : 8;
  const uint32_t v = x[a];
  for (uint64_t j = 1; j < m; j++) if (x[a + j] != v) return -1;
  return v;
}
// run of groups [g, h): an RLE run when group g is uniform (then every group of the run is), else bit-packed (h - g <= 63)
__host__ __device__ inline uint64_t idx_run_bytes(const uint32_t* x, uint64_t n, uint32_t w, uint64_t g, uint64_t h) {
  if (idx_cls(x, n, g) >= 0) {
    const uint64_t cnt = ((h * 8 < n ? h * 8 : n)) - g * 8;
    return varint(cnt << 1, nullptr) + (w + 7) / 8;
  }
  return 1 + (h - g) * w;
}
__host__ __device__ inline void idx_write_run(const uint32_t* x, uint64_t n, uint32_t w, uint64_t g, uint64_t h, uint8_t* out) {
  const int64_t c = idx_cls(x, n, g);
  if (c >= 0) {
    const uint64_t cnt = ((h * 8 < n ? h * 8 : n)) - g * 8;
    const uint32_t o = varint(cnt << 1, out);
    for (uint32_t b = 0; b < (w + 7) / 8; b++) out[o + b] = (uint8_t)((uint64_t)c >> (8 * b));
    return;
  }
  out[0] = (uint8_t)(((h - g) << 1) | 1u);
  uint64_t o = 1, acc = 0;
  uint32_t bits = 0;
  for (uint64_t e = g * 8; e < h * 8; e++) {          // LSB first, the last group zero-padded
    acc |= (uint64_t)(e < n ? x[e] : 0u) << bits;
    bits += w;
    while (bits >= 8) { out[o++] = (uint8_t)acc; acc >>= 8; bits -= 8; }
  }
}
// serial encoder (the host harness; the device encodes the same runs in parallel); returns the bytes written
__host__ __device__ inline uint64_t indices_encode(const uint32_t* x, uint64_t n, uint32_t w, uint8_t* out) {
  const uint64_t ng = (n + 7) / 8;
  uint64_t o = 0, g = 0;
  while (g < ng) {
    const int64_t c = idx_cls(x, n, g);
    uint64_t h = g + 1;
    if (c >= 0) while (h < ng && idx_cls(x, n, h) == c) h++;
    else while (h < ng && h - g < 63 && idx_cls(x, n, h) < 0) h++;
    idx_write_run(x, n, w, g, h, out + o);
    o += idx_run_bytes(x, n, w, g, h);
    g = h;
  }
  return o;
}
// bound of an RLE_DICTIONARY payload's index part (bit-width byte + runs): a group costs at most w + 1 bytes bit-packed
// or 4 as (part of) an RLE run
__host__ __device__ inline uint64_t indices_bound(uint64_t n) { return 1 + ((n + 7) / 8) * 19; }

// ------------------------------------------------------------------------------------------------ page index
// ColumnIndex bounds of a byte-array value v[0, len) (arrow-rs's truncate_min_value / truncate_max_value with
// column_index_truncate_length 64; utf8: v is valid UTF-8).  Each writes the bound to out unless it is nullptr and
// returns its length.  A value of at most 64 bytes is its own bound.
constexpr uint32_t kIndexTruncate = 64;
// minimum: the first 64 bytes; Utf8: the longest prefix of at most 64 bytes that ends on a character boundary
__host__ __device__ inline uint64_t index_min(const uint8_t* v, uint64_t len, bool utf8, uint8_t* out) {
  uint64_t k = len;
  if (len > kIndexTruncate) {
    k = kIndexTruncate;
    if (utf8) while (k > 1 && (v[k] & 0xC0u) == 0x80u) k--;   // v[k] starts the character after the prefix
  }
  if (out) for (uint64_t i = 0; i < k; i++) out[i] = v[i];
  return k;
}
// maximum: the first 64 bytes with the last byte incremented, 0xFF carrying into the byte before it as 0x00; Utf8: the
// prefix up to the last character boundary at most 64, cut after its last character whose code point + 1 is a Unicode
// scalar value of the same UTF-8 length, that character incremented.  Nothing to increment: the value itself.
__host__ __device__ inline uint64_t index_max(const uint8_t* v, uint64_t len, bool utf8, uint8_t* out) {
  if (len > kIndexTruncate && !utf8) {
    int64_t j = kIndexTruncate - 1;
    while (j >= 0 && v[j] == 0xFFu) j--;
    if (j >= 0) {
      if (out) {
        for (int64_t i = 0; i < j; i++) out[i] = v[i];
        out[j] = (uint8_t)(v[j] + 1);
        for (uint32_t i = (uint32_t)j + 1; i < kIndexTruncate; i++) out[i] = 0;
      }
      return kIndexTruncate;
    }
  } else if (len > kIndexTruncate) {
    uint64_t end = kIndexTruncate;
    while (end > 0 && (v[end] & 0xC0u) == 0x80u) end--;
    while (end > 0) {                                   // the characters of v[0, end), last first
      uint64_t s = end - 1;
      while (s > 0 && (v[s] & 0xC0u) == 0x80u) s--;
      const uint32_t l = (uint32_t)(end - s);
      uint32_t cp = l == 1 ? v[s] : v[s] & (0x7Fu >> l);
      for (uint32_t i = 1; i < l; i++) cp = (cp << 6) | (v[s + i] & 0x3Fu);
      const uint32_t nx = cp + 1;
      const uint32_t nl = nx < 0x80u ? 1 : nx < 0x800u ? 2 : nx < 0x10000u ? 3 : 4;
      if (nx <= 0x10FFFFu && (nx < 0xD800u || nx > 0xDFFFu) && nl == l) {
        if (out) {
          for (uint64_t i = 0; i < s; i++) out[i] = v[i];
          if (l == 1) out[s] = (uint8_t)nx;
          else {
            out[s] = (uint8_t)((0xF00u >> l) | (nx >> (6 * (l - 1))));   // 110xxxxx / 1110xxxx / 11110xxx
            for (uint32_t i = 1; i < l; i++) out[s + i] = (uint8_t)(0x80u | ((nx >> (6 * (l - 1 - i))) & 0x3Fu));
          }
        }
        return end;
      }
      end = s;
    }
  }
  if (out) for (uint64_t i = 0; i < len; i++) out[i] = v[i];
  return len;
}
// PageLocation {1 offset: i64, 2 compressed_page_size: i32, 3 first_row_index: i64}; at most 29 bytes
__host__ __device__ inline uint32_t page_location(uint8_t* out, uint64_t offset, uint32_t size, uint64_t first_row) {
  TWriter w(out);
  w.i64(1, (int64_t)offset);
  w.i32(2, (int32_t)size);
  w.i64(3, (int64_t)first_row);
  w.end();
  return (uint32_t)w.n;
}
// the header of a list field whose id follows the previous field's (one byte) and its size; returns its length
__host__ __device__ inline uint32_t list_field(uint8_t* out, uint8_t elem_type, uint32_t size) {
  TWriter w(out);
  w.list(1, elem_type, size);
  return (uint32_t)w.n;
}

// ------------------------------------------------------------------------------------------------ bloom filters
// Parquet's split-block bloom filter (BloomFilter.md): XXH64 of the value's PLAIN bytes without a length prefix; the
// block ((h >> 32) * blocks) >> 32 of 32 bytes; in it, word i gets bit (uint32)((uint32)h * kBloomSalt[i]) >> 27.
constexpr uint64_t kBloomMinBytes = 32, kBloomMaxBytes = 128ull << 20;
constexpr uint64_t kBloomDefaultBytes = 1ull << 20;   // max_bytes 0 (Iceberg's write.parquet.bloom-filter-max-bytes)
constexpr uint64_t kXxP1 = 0x9E3779B185EBCA87ull, kXxP2 = 0xC2B2AE3D27D4EB4Full, kXxP3 = 0x165667B19E3779F9ull,
                   kXxP4 = 0x85EBCA77C2B2AE63ull, kXxP5 = 0x27D4EB2F165667C5ull;
__host__ __device__ inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__host__ __device__ inline uint32_t load32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
__host__ __device__ inline uint64_t load64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
__host__ __device__ inline uint64_t xxh64_round(uint64_t acc, uint64_t lane) { return rotl64(acc + lane * kXxP2, 31) * kXxP1; }
__host__ __device__ inline uint64_t xxh64_merge(uint64_t h, uint64_t v) { return (h ^ xxh64_round(0, v)) * kXxP1 + kXxP4; }
__host__ __device__ inline uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33; h *= kXxP2; h ^= h >> 29; h *= kXxP3; h ^= h >> 32;
  return h;
}
// XXH64, seed 0, of p[0, len)
__host__ __device__ inline uint64_t xxh64(const uint8_t* p, uint64_t len) {
  uint64_t h, k = 0;
  if (len >= 32) {
    uint64_t v1 = kXxP1 + kXxP2, v2 = kXxP2, v3 = 0, v4 = 0 - kXxP1;
    for (; k + 32 <= len; k += 32) {
      v1 = xxh64_round(v1, load64(p + k)); v2 = xxh64_round(v2, load64(p + k + 8));
      v3 = xxh64_round(v3, load64(p + k + 16)); v4 = xxh64_round(v4, load64(p + k + 24));
    }
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = xxh64_merge(h, v1); h = xxh64_merge(h, v2); h = xxh64_merge(h, v3); h = xxh64_merge(h, v4);
  } else h = kXxP5;
  h += len;
  for (; k + 8 <= len; k += 8) h = rotl64(h ^ xxh64_round(0, load64(p + k)), 27) * kXxP1 + kXxP4;
  if (k + 4 <= len) { h = rotl64(h ^ (uint64_t)load32(p + k) * kXxP1, 23) * kXxP2 + kXxP3; k += 4; }
  for (; k < len; k++) h = rotl64(h ^ (uint64_t)p[k] * kXxP5, 11) * kXxP1;
  return xxh64_avalanche(h);
}
// the same hash of a 4- / 8-byte little-endian value
__host__ __device__ inline uint64_t xxh64_u32(uint32_t v) {
  return xxh64_avalanche(rotl64((kXxP5 + 4) ^ (uint64_t)v * kXxP1, 23) * kXxP2 + kXxP3);
}
__host__ __device__ inline uint64_t xxh64_u64(uint64_t v) {
  return xxh64_avalanche(rotl64((kXxP5 + 8) ^ xxh64_round(0, v), 27) * kXxP1 + kXxP4);
}
// the block of hash h in a bitset of blocks 32-byte blocks, and the bit of its word i
__host__ __device__ inline uint32_t bloom_block(uint64_t h, uint32_t blocks) { return (uint32_t)(((h >> 32) * blocks) >> 32); }
__host__ __device__ inline uint32_t bloom_mask(uint64_t h, int i) {
  const uint32_t salt[8] = {0x47b6137bu, 0x44974d91u, 0x8824ad5bu, 0xa2b7289du, 0x705495c7u, 0x2df1424bu, 0x9efc4947u, 0x5c6bfb31u};
  return 1u << (((uint32_t)h * salt[i]) >> 27);
}
// BloomFilterHeader {1 numBytes, 2 algorithm {1 BLOCK {}}, 3 hash {1 XXHASH {}}, 4 compression {1 UNCOMPRESSED {}}};
// out == nullptr counts.  Returns its length (at most 19 bytes).
__host__ __device__ inline uint32_t bloom_header(uint8_t* out, uint32_t num_bytes) {
  TWriter w(out);
  w.i32(1, (int32_t)num_bytes);
  for (int16_t f = 2; f <= 4; f++) { w.begin(f); w.begin(1); w.end(); w.end(); }
  w.end();
  return (uint32_t)w.n;
}
// (host) bitset bytes for ndv distinct values at false-positive probability fpp, as Arrow C++'s OptimalNumOfBits:
// bits = -8 ndv / ln(1 - fpp^(1/8)) truncated, clamped to [8 × 32, 8 × 128 MiB], rounded up to a power of two; then
// at most max_bytes (a power of two in [32, 128 MiB])
inline uint64_t bloom_bytes(uint64_t ndv, double fpp, uint64_t max_bytes) {
  const double m = -8.0 * (double)ndv / std::log(1.0 - std::pow(fpp, 1.0 / 8));
  uint64_t bits = !(m >= 0) || m > 8.0 * kBloomMaxBytes ? 8 * kBloomMaxBytes : (uint64_t)m;
  if (bits < 8 * kBloomMinBytes) bits = 8 * kBloomMinBytes;
  uint64_t p = 1;
  while (p < bits) p <<= 1;
  const uint64_t bytes = p / 8;
  return bytes < max_bytes ? bytes : max_bytes;
}

// ------------------------------------------------------------------------------------------------ Snappy
__host__ __device__ inline uint32_t snappy_hash(uint32_t v) { return (v * 0x1e35a7bdu) >> (32 - kSnappyHashBits); }
__host__ __device__ inline uint32_t snappy_literal(const uint8_t* src, uint32_t len, uint8_t* out) {
  uint32_t o = 0;
  const uint32_t l = len - 1;
  if (l < 60) out[o++] = (uint8_t)(l << 2);
  else {
    const uint32_t nb = l < 0x100u ? 1 : l < 0x10000u ? 2 : l < 0x1000000u ? 3 : 4;
    out[o++] = (uint8_t)((59 + nb) << 2);
    for (uint32_t b = 0; b < nb; b++) out[o++] = (uint8_t)(l >> (8 * b));
  }
  memcpy(out + o, src, len);
  return o + len;
}
__host__ __device__ inline uint32_t snappy_copy(uint32_t off, uint32_t len, uint8_t* out) {
  uint32_t o = 0;
  while (len > 0) {
    // split as the reference compressor does: 64-byte copies, 60 when that would leave fewer than 4
    const uint32_t take = len >= 68 ? 64 : len > 64 ? 60 : len;
    if (take >= 4 && take <= 11 && off < 2048) {
      out[o++] = (uint8_t)(1u | ((take - 4) << 2) | ((off >> 8) << 5));
      out[o++] = (uint8_t)off;
    } else {
      out[o++] = (uint8_t)(2u | ((take - 1) << 2));
      out[o++] = (uint8_t)off;
      out[o++] = (uint8_t)(off >> 8);
    }
    len -= take;
  }
  return o;
}
// the elements of one fragment (n <= kFragment; no length preamble) into out (snappy_bound(n) bytes); table has
// 1 << kSnappyHashBits entries of scratch.  Returns the bytes written.
__host__ __device__ inline uint32_t snappy_fragment(const uint8_t* in, uint32_t n, uint8_t* out, uint16_t* table) {
  uint32_t o = 0, lit = 0, ip = 0;
  if (n >= 15) {
    for (uint32_t k = 0; k < (1u << kSnappyHashBits); k++) table[k] = 0;
    const uint32_t limit = n - 4;                        // a 4-byte load at ip stays inside the fragment
    uint32_t skip = 32;
    ip = 1;
    while (ip <= limit) {
      const uint32_t cur = load32(in + ip);
      const uint32_t h = snappy_hash(cur);
      const uint32_t cand = table[h];
      table[h] = (uint16_t)ip;
      if (cand < ip && load32(in + cand) == cur) {
        uint32_t len = 4;
        while (ip + len < n && in[cand + len] == in[ip + len]) len++;
        if (ip > lit) o += snappy_literal(in + lit, ip - lit, out + o);
        o += snappy_copy(ip - cand, len, out + o);
        ip += len;
        lit = ip;
        skip = 32;
        if (ip - 1 <= limit) table[snappy_hash(load32(in + ip - 1))] = (uint16_t)(ip - 1);
      } else {
        ip += skip >> 5;                                 // incompressible stretches are skipped faster and faster
        skip++;
      }
    }
  }
  if (n > lit) o += snappy_literal(in + lit, n - lit, out + o);
  return o;
}

// ------------------------------------------------------------------------------------------------ footer (host)
struct Leaf {                       // one column of the file: a flat leaf, or a list and its element
  std::string name;
  int32_t field_id, element_field_id;
  uint32_t ptype;                   // PT_*
  int32_t converted;                // CT_* of the leaf (CT_NONE)
  uint32_t logical;                 // 0 none, 1 STRING, 6 DATE, 7 TIME(µs, utc=false), 8 TIMESTAMP(µs), 14 UUID
  bool utc;                         // TIMESTAMP: isAdjustedToUTC
  bool required, is_list;
};
struct Chunk {
  uint64_t offset, num_values, usize, csize, null_count;   // offset: the chunk's first page (a dictionary chunk: its dictionary page)
  bool has_minmax;
  std::string min, max;
  bool dict = false;                // dictionary chunk: its data pages are RLE_DICTIONARY
  uint64_t data_offset = 0;         // dictionary chunk: the first data page
  uint64_t data_pages = 0;          // dictionary chunk: its data pages
  bool page_index = false;          // ETL_PQ_PAGE_INDEX: the chunk's OffsetIndex and, when ci_len, its ColumnIndex
  uint64_t ci_offset = 0, oi_offset = 0;
  uint32_t ci_len = 0, oi_len = 0;
  uint64_t bloom_offset = 0;        // a bloom filter: its header's file offset, header + bitset bytes (0: none)
  uint32_t bloom_len = 0;
};

inline void schema_element(TWriter& w, const Leaf& L, bool element) {
  w.list_struct_begin();
  w.i32(1, (int32_t)L.ptype);
  if (L.ptype == PT_FLBA) w.i32(2, 16);
  w.i32(3, element ? REP_OPTIONAL : L.required ? REP_REQUIRED : REP_OPTIONAL);
  const std::string& nm = element ? std::string("element") : L.name;
  w.bin(4, (const uint8_t*)nm.data(), (uint32_t)nm.size());
  if (L.converted != CT_NONE) w.i32(6, L.converted);
  w.i32(9, element ? L.element_field_id : L.field_id);
  if (L.logical) {
    w.begin(10);
    w.begin((int16_t)L.logical);
    if (L.logical == 7 || L.logical == 8) {
      w.boolean(1, L.logical == 8 && L.utc);
      w.begin(2); w.begin(2); w.end(); w.end();    // unit: MICROS
    }
    w.end();
    w.end();
  }
  w.end();
}

// the footer fields of one column chunk, as the tail serialiser below reads them (the device's chunk records and the
// host's Chunk both give one); min / max point at their statistic bytes
struct ChunkMeta {
  uint64_t offset, num_values, usize, csize, null_count, data_offset, data_pages, ci_offset, oi_offset, bloom_offset;
  uint32_t ci_len, oi_len, bloom_len, min_len, max_len;
  bool has_minmax, dict, page_index;
  const uint8_t* min;
  const uint8_t* max;
};
// what the tail needs of a leaf: its Parquet type, whether it has levels or is a list, its column name
struct LeafMeta {
  const uint8_t* name;
  uint32_t name_len, ptype;
  bool levels, is_list;
};

// FileMetaData fields 1 (version) and 2 (schema): the same for every file of one schema, serialised once on the host.
// The writer is left where the tail continues (field 2 was the last of the top-level struct).
inline void footer_prefix(TWriter& w, const std::vector<Leaf>& leaves) {
  uint32_t n_elems = 1;
  for (const Leaf& L : leaves) n_elems += L.is_list ? 3 : 1;
  w.i32(1, 1);
  w.list(2, TT_STRUCT, n_elems);
  w.list_struct_begin();
  w.bin(4, (const uint8_t*)"schema", 6);
  w.i32(5, (int32_t)leaves.size());
  w.end();
  for (const Leaf& L : leaves) {
    if (!L.is_list) { schema_element(w, L, false); continue; }
    w.list_struct_begin();                           // <rep> group name (LIST)
    w.i32(3, L.required ? REP_REQUIRED : REP_OPTIONAL);
    w.bin(4, (const uint8_t*)L.name.data(), (uint32_t)L.name.size());
    w.i32(5, 1);
    w.i32(6, CT_LIST);
    w.i32(9, L.field_id);
    w.begin(10); w.begin(3); w.end(); w.end();
    w.end();
    w.list_struct_begin();                           // repeated group list
    w.i32(3, REP_REPEATED);
    w.bin(4, (const uint8_t*)"list", 4);
    w.i32(5, 1);
    w.end();
    schema_element(w, L, true);
  }
}
// one ColumnChunk of a RowGroup's columns list (the writer inside that list: depth 1)
__host__ __device__ inline void column_chunk(TWriter& w, const LeafMeta& L, const ChunkMeta& C, uint32_t codec) {
  w.list_struct_begin();
  w.i64(2, (int64_t)C.offset);
  w.begin(3);
  w.i32(1, (int32_t)L.ptype);
  w.list(2, TT_I32, (L.levels ? 2 : 1) + (C.dict ? 1 : 0));
  w.var(zigzag(ENC_PLAIN));
  if (L.levels) w.var(zigzag(ENC_RLE));
  if (C.dict) w.var(zigzag(ENC_RLE_DICTIONARY));
  w.list(3, TT_BINARY, L.is_list ? 3 : 1);
  w.var(L.name_len);
  for (uint32_t k = 0; k < L.name_len; k++) w.byte(L.name[k]);
  if (L.is_list) { w.var(4); for (const char* s = "list"; *s; s++) w.byte((uint8_t)*s); w.var(7); for (const char* s = "element"; *s; s++) w.byte((uint8_t)*s); }
  w.i32(4, (int32_t)(codec & 0xFFu));            // the compression codec, without the ETL_PQ_DICTIONARY bit
  w.i64(5, (int64_t)C.num_values);
  w.i64(6, (int64_t)C.usize);
  w.i64(7, (int64_t)C.csize);
  w.i64(9, (int64_t)(C.dict ? C.data_offset : C.offset));
  if (C.dict) w.i64(11, (int64_t)C.offset);
  w.begin(12);
  w.i64(3, (int64_t)C.null_count);
  if (C.has_minmax) {
    w.bin(5, C.max, C.max_len);
    w.bin(6, C.min, C.min_len);
  }
  w.end();
  if (C.dict) {                                      // PageEncodingStats {page_type, encoding, count}
    w.list(13, TT_STRUCT, 2);
    w.list_struct_begin(); w.i32(1, PAGE_DICTIONARY); w.i32(2, ENC_PLAIN); w.i32(3, 1); w.end();
    w.list_struct_begin(); w.i32(1, PAGE_DATA); w.i32(2, ENC_RLE_DICTIONARY); w.i32(3, (int32_t)C.data_pages); w.end();
  }
  if (C.bloom_len) { w.i64(14, (int64_t)C.bloom_offset); w.i32(15, (int32_t)C.bloom_len); }
  w.end();
  if (C.page_index) {                                // ColumnChunk offset_index_offset / _length, column_index_*
    w.i64(4, (int64_t)C.oi_offset);
    w.i32(5, (int32_t)C.oi_len);
    if (C.ci_len) { w.i64(6, (int64_t)C.ci_offset); w.i32(7, (int32_t)C.ci_len); }
  }
  w.end();
}

// FileMetaData fields 3 (num_rows), 4 (row_groups), 6 (created_by), 7 (column_orders) and the struct's end, the part
// of a footer behind footer_prefix, cut into independent units: with n_rg row groups of n_leaves chunks (row group g
// is rows [rg_start[g], rg_start[g + 1]), any origin; its chunks chunk(g * n_leaves + l)), unit 0 is num_rows and the
// row_groups list header, unit 1 + c is chunk c's ColumnChunk (the first of a row group with the RowGroup's opening
// and its columns list header, the last with the RowGroup's closing fields), unit n_rg * n_leaves + 1 is created_by,
// column_orders and the end.  Each unit starts from a writer in the state the whole tail has there, so the units
// written back to back are the tail; the device sizes and writes them a lane per unit.  Returns its bytes (out ==
// nullptr counts).
template <class GetChunk>
__host__ __device__ inline uint64_t tail_unit(uint8_t* out, uint64_t u, const LeafMeta* leaves, uint32_t n_leaves, const uint64_t* rg_start,
                                              uint32_t n_rg, GetChunk chunk, uint32_t codec, const uint8_t* created_by, uint32_t cb_len) {
  TWriter w(out);
  const uint64_t nc = (uint64_t)n_rg * n_leaves;
  if (u == 0) {
    w.last[0] = 2;                                   // behind field 2 (schema)
    w.i64(3, (int64_t)(n_rg ? rg_start[n_rg] - rg_start[0] : 0));
    w.list(4, TT_STRUCT, n_rg);
    return w.n;
  }
  if (u == nc + 1) {
    w.last[0] = 4;                                   // behind field 4 (row_groups)
    w.bin(6, created_by, cb_len);
    w.list(7, TT_STRUCT, n_leaves);
    for (uint32_t l = 0; l < n_leaves; l++) {        // ColumnOrder { 1: TypeDefinedOrder {} }
      w.list_struct_begin();
      w.begin(1); w.end();
      w.end();
    }
    w.end();
    return w.n;
  }
  const uint64_t c = u - 1, g = c / n_leaves;
  const uint32_t l = (uint32_t)(c % n_leaves);
  if (l == 0) {                                      // the RowGroup's struct and its columns list (field 1)
    w.list_struct_begin();
    w.list(1, TT_STRUCT, n_leaves);
  } else {
    w.depth = 1; w.last[1] = 1;
  }
  column_chunk(w, leaves[l], chunk(c), codec);
  if (l + 1 == n_leaves) {                           // the RowGroup's totals, rows, file_offset, ordinal
    uint64_t tu = 0, tc = 0;
    for (uint32_t k = 0; k < n_leaves; k++) { const ChunkMeta C = chunk(g * n_leaves + k); tu += C.usize; tc += C.csize; }
    w.i64(2, (int64_t)tu);
    w.i64(3, (int64_t)(rg_start[g + 1] - rg_start[g]));
    w.i64(5, (int64_t)chunk(g * n_leaves).offset);
    w.i64(6, (int64_t)tc);
    w.field(7, TT_I16); w.var(zigzag((int64_t)g));
    w.end();
  }
  return w.n;
}
// the whole tail, its units in order (the host's footer; out == nullptr counts)
template <class GetChunk>
__host__ __device__ inline uint64_t footer_tail(uint8_t* out, const LeafMeta* leaves, uint32_t n_leaves, const uint64_t* rg_start,
                                                uint32_t n_rg, GetChunk chunk, uint32_t codec, const uint8_t* created_by,
                                                uint32_t cb_len) {
  uint64_t n = 0;
  for (uint64_t u = 0; u < (uint64_t)n_rg * n_leaves + 2; u++)
    n += tail_unit(out ? out + n : nullptr, u, leaves, n_leaves, rg_start, n_rg, chunk, codec, created_by, cb_len);
  return n;
}

// (host) the tail's leaves: names point into leaves
inline std::vector<LeafMeta> leaf_meta(const std::vector<Leaf>& leaves) {
  std::vector<LeafMeta> m(leaves.size());
  for (size_t l = 0; l < leaves.size(); l++)
    m[l] = LeafMeta{(const uint8_t*)leaves[l].name.data(), (uint32_t)leaves[l].name.size(), leaves[l].ptype,
                    leaves[l].is_list || !leaves[l].required, leaves[l].is_list};
  return m;
}
inline ChunkMeta chunk_meta(const Chunk& C) {
  return ChunkMeta{C.offset, C.num_values, C.usize, C.csize, C.null_count, C.data_offset, C.data_pages, C.ci_offset, C.oi_offset,
                   C.bloom_offset, C.ci_len, C.oi_len, C.bloom_len, (uint32_t)C.min.size(), (uint32_t)C.max.size(), C.has_minmax,
                   C.dict, C.page_index, (const uint8_t*)C.min.data(), (const uint8_t*)C.max.data()};
}

// FileMetaData {1 version, 2 schema, 3 num_rows, 4 row_groups, 6 created_by, 7 column_orders}; chunks row-group major.
// The schema prefix, then the tail.
inline std::vector<uint8_t> footer(const std::vector<Leaf>& leaves, const std::vector<uint64_t>& rg_rows,
                                   const std::vector<Chunk>& chunks, uint32_t codec, const char* created_by) {
  TWriter pw(nullptr);
  footer_prefix(pw, leaves);
  std::vector<uint8_t> buf(pw.n);
  TWriter w(buf.data());
  footer_prefix(w, leaves);
  std::vector<uint64_t> rg_start(rg_rows.size() + 1, 0);
  for (size_t g = 0; g < rg_rows.size(); g++) rg_start[g + 1] = rg_start[g] + rg_rows[g];
  const std::vector<LeafMeta> lm = leaf_meta(leaves);
  auto get = [&](uint64_t c) { return chunk_meta(chunks[c]); };
  const uint32_t cb = (uint32_t)strlen(created_by);
  const uint64_t t = footer_tail(nullptr, lm.data(), (uint32_t)lm.size(), rg_start.data(), (uint32_t)rg_rows.size(), get, codec,
                                 (const uint8_t*)created_by, cb);
  buf.resize(w.n + t);
  footer_tail(buf.data() + w.n, lm.data(), (uint32_t)lm.size(), rg_start.data(), (uint32_t)rg_rows.size(), get, codec,
              (const uint8_t*)created_by, cb);
  return buf;
}

// ------------------------------------------------------------------------------------------------ files (host)
// etl_dec_parquet_write_files: the row groups of K files, file k rows [ro[k], ro[k + 1]).  Row groups restart in every
// file (at most kRowGroupRows rows each, an empty file has none) and are numbered across the files in order; row0 is
// relative to ro[0], so the row groups tile [0, ro[K] - ro[0]).  first[k] is file k's first row group (first[K]: all).
struct RowGroup { uint64_t row0, rows; uint64_t file; };
inline std::vector<RowGroup> row_group_table(const uint64_t* ro, uint64_t K, std::vector<uint64_t>& first) {
  std::vector<RowGroup> t;
  first.assign(K + 1, 0);
  for (uint64_t k = 0; k < K; k++) {
    first[k] = t.size();
    for (uint64_t r = ro[k]; r < ro[k + 1]; r += kRowGroupRows)
      t.push_back(RowGroup{r - ro[0], ro[k + 1] - r < kRowGroupRows ? ro[k + 1] - r : kRowGroupRows, k});
  }
  first[K] = t.size();
  return t;
}

}  // namespace etl_pq
