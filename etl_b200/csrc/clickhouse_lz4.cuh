// clickhouse_lz4.cuh — the byte-level pieces of the ClickHouse INSERT-body compressor (clickhouse_lz4.cu) that a host
// harness can compile too (tests/emul/host_ch_lz4.cpp builds this same file with g++, so the CPU suite checks it against
// tests/clickhouse_lz4_ref.py):
//   * the block size, the LZ4 end-of-block limits and the compressed slot bound;
//   * the LZ4 sequence writer: token, literal-length and match-length extension bytes, the 2-byte offset;
//   * the ClickHouse compressed block header (method 0x82, u32 LE compressed size = 9 + payload, u32 LE decompressed
//     size) and its 16-byte checksum, CityHash128 v1.0.2 of header and payload, written low64 then high64, each LE
//     (the order CompressedReadBufferBase reads it).
// CityHash128 here is v1.0.2, the version ClickHouse bundles for its checksums, not 1.1: the two differ in the seed
// CityHash128 derives from the first 16 bytes, in HashLen0to16 / HashLen17to32 and in the long-input loop and tail.
#pragma once
#include <stdint.h>
#include <string.h>

#ifndef ETL_CH_LZ4_BLOCK
#define ETL_CH_LZ4_BLOCK 16384
#endif

namespace etl_ch {

constexpr uint32_t kBlock = ETL_CH_LZ4_BLOCK;   // uncompressed bytes per compressed block (the last of a body: fewer)
constexpr uint32_t kHeader = 25;                // checksum 16 + method 1 + compressed size 4 + decompressed size 4
constexpr uint8_t kMethodLz4 = 0x82;
constexpr uint32_t kMfLimit = 12;               // a match starts more than this many bytes before the block's end
constexpr uint32_t kLastLiterals = 5;           // ... and ends at least this many bytes before it
constexpr uint32_t kMinMatch = 4;
static_assert(kBlock == 16384 || kBlock == 32768 || kBlock == 65536, "ETL_CH_LZ4_BLOCK: 16, 32 or 64 KiB");

// LZ4_COMPRESSBOUND of n input bytes
__host__ __device__ inline uint32_t lz4_bound(uint32_t n) { return n + n / 255u + 16u; }

// ------------------------------------------------------------------------------------------------ LZ4 sequences
// bytes of the token and literal-length extension of a sequence with `lit` literals
__host__ __device__ inline uint32_t lz4_lit_header_len(uint32_t lit) { return 1u + (lit >= 15u ? (lit - 15u) / 255u + 1u : 0u); }
// the token and literal-length extension (match_len 0: the last sequence, literals only); returns its length
__host__ __device__ inline uint32_t lz4_lit_header(uint32_t lit, uint32_t match_len, uint8_t* out) {
  const uint32_t ml = match_len ? match_len - kMinMatch : 0u;
  out[0] = (uint8_t)((lit < 15u ? lit : 15u) << 4 | (ml < 15u ? ml : 15u));
  uint32_t o = 1;
  if (lit >= 15u) {
    uint32_t r = lit - 15u;
    for (; r >= 255u; r -= 255u) out[o++] = 255;
    out[o++] = (uint8_t)r;
  }
  return o;
}
// the offset and match-length extension that follow the literals; returns its length
__host__ __device__ inline uint32_t lz4_match_tail(uint32_t offset, uint32_t match_len, uint8_t* out) {
  out[0] = (uint8_t)offset;
  out[1] = (uint8_t)(offset >> 8);
  uint32_t o = 2;
  const uint32_t ml = match_len - kMinMatch;
  if (ml >= 15u) {
    uint32_t r = ml - 15u;
    for (; r >= 255u; r -= 255u) out[o++] = 255;
    out[o++] = (uint8_t)r;
  }
  return o;
}
// one whole sequence: header, literals, and (match_len > 0) the match; returns its length
__host__ __device__ inline uint32_t lz4_sequence(const uint8_t* lit, uint32_t lit_len, uint32_t offset, uint32_t match_len, uint8_t* out) {
  uint32_t o = lz4_lit_header(lit_len, match_len, out);
  for (uint32_t k = 0; k < lit_len; k++) out[o + k] = lit[k];
  o += lit_len;
  if (match_len) o += lz4_match_tail(offset, match_len, out + o);
  return o;
}

// ------------------------------------------------------------------------------------------------ block header
// method, compressed size (9 + payload) and decompressed size at out[16 .. 25)
__host__ __device__ inline void block_header(uint32_t payload, uint32_t raw, uint8_t* out) {
  out[16] = kMethodLz4;
  const uint32_t c = 9u + payload;
  for (int k = 0; k < 4; k++) { out[17 + k] = (uint8_t)(c >> (8 * k)); out[21 + k] = (uint8_t)(raw >> (8 * k)); }
}

// ------------------------------------------------------------------------------------------------ CityHash128 v1.0.2
struct U128 { uint64_t first, second; };   // first = low64, second = high64

constexpr uint64_t kK0 = 0xc3a5c85c97cb3127ull, kK1 = 0xb492b66fbe98f273ull, kK2 = 0x9ae16a3b2f90404full,
                   kK3 = 0xc949d7c7509e6557ull;

__host__ __device__ inline uint64_t fetch64(const uint8_t* p) {
  uint64_t v;
  if (((uintptr_t)p & 7u) == 0) v = *reinterpret_cast<const uint64_t*>(p);
  else memcpy(&v, p, 8);
  return v;
}
__host__ __device__ inline uint64_t fetch32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
__host__ __device__ inline uint64_t rot(uint64_t v, int s) { return s == 0 ? v : (v >> s) | (v << (64 - s)); }
__host__ __device__ inline uint64_t rot1(uint64_t v, int s) { return (v >> s) | (v << (64 - s)); }
__host__ __device__ inline uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }
__host__ __device__ inline uint64_t hash_len16(uint64_t u, uint64_t v) {
  const uint64_t kMul = 0x9ddfea08eb382d69ull;
  uint64_t a = (u ^ v) * kMul;
  a ^= a >> 47;
  uint64_t b = (v ^ a) * kMul;
  b ^= b >> 47;
  return b * kMul;
}
__host__ __device__ inline uint64_t hash_len0to16(const uint8_t* s, uint64_t len) {
  if (len > 8) {
    const uint64_t a = fetch64(s), b = fetch64(s + len - 8);
    return hash_len16(a, rot1(b + len, (int)len)) ^ b;
  }
  if (len >= 4) {
    const uint64_t a = fetch32(s);
    return hash_len16(len + (a << 3), fetch32(s + len - 4));
  }
  if (len > 0) {
    const uint32_t y = (uint32_t)s[0] + ((uint32_t)s[len >> 1] << 8);
    const uint32_t z = (uint32_t)len + ((uint32_t)s[len - 1] << 2);
    return shift_mix((uint64_t)y * kK2 ^ (uint64_t)z * kK3) * kK2;
  }
  return kK2;
}
__host__ __device__ inline void weak32(const uint8_t* s, uint64_t a, uint64_t b, uint64_t* o1, uint64_t* o2) {
  const uint64_t w = fetch64(s), x = fetch64(s + 8), y = fetch64(s + 16), z = fetch64(s + 24);
  a += w;
  b = rot(b + a + z, 21);
  const uint64_t c = a;
  a += x;
  a += y;
  b += rot(a, 44);
  *o1 = a + z;
  *o2 = b + c;
}
__host__ __device__ inline U128 city_murmur(const uint8_t* s, uint64_t len, U128 seed) {
  uint64_t a = seed.first, b = seed.second, c = 0, d = 0;
  if (len <= 16) {
    a = shift_mix(a * kK1) * kK1;
    c = b * kK1 + hash_len0to16(s, len);
    d = shift_mix(a + (len >= 8 ? fetch64(s) : c));
  } else {
    c = hash_len16(fetch64(s + len - 8) + kK1, a);
    d = hash_len16(b + len, c + fetch64(s + len - 16));
    a += d;
    int64_t l = (int64_t)len - 16;
    do {
      a ^= shift_mix(fetch64(s) * kK1) * kK1;
      a *= kK1;
      b ^= a;
      c ^= shift_mix(fetch64(s + 8) * kK1) * kK1;
      c *= kK1;
      d ^= c;
      s += 16;
      l -= 16;
    } while (l > 0);
  }
  a = hash_len16(a, c);
  b = hash_len16(d, b);
  return U128{a ^ b, hash_len16(b, a)};
}
__host__ __device__ inline U128 city128_seed(const uint8_t* s, uint64_t len, U128 seed) {
  if (len < 128) return city_murmur(s, len, seed);
  uint64_t v1, v2, w1, w2;
  uint64_t x = seed.first, y = seed.second, z = len * kK1;
  v1 = rot(y ^ kK1, 49) * kK1 + fetch64(s);
  v2 = rot(v1, 42) * kK1 + fetch64(s + 8);
  w1 = rot(y + z, 35) * kK1 + x;
  w2 = rot(x + fetch64(s + 88), 53) * kK1;
  do {
    for (int half = 0; half < 2; half++) {
      x = rot(x + y + v1 + fetch64(s + 16), 37) * kK1;
      y = rot(y + v2 + fetch64(s + 48), 42) * kK1;
      x ^= w2;
      y ^= v1;
      z = rot(z ^ w1, 33);
      weak32(s, v2 * kK1, x + w1, &v1, &v2);
      weak32(s + 32, z + w2, y, &w1, &w2);
      const uint64_t t = z; z = x; x = t;
      s += 64;
    }
    len -= 128;
  } while (len >= 128);
  y += rot(w1, 37) * kK0 + z;
  x += rot(v1 + z, 49) * kK0;
  for (uint64_t done = 0; done < len;) {
    done += 32;
    y = rot(y - x, 42) * kK0 + v2;
    w1 += fetch64(s + len - done + 16);
    x = rot(x, 49) * kK0 + w1;
    w1 += v1;
    weak32(s + len - done, v1, v2, &v1, &v2);
  }
  x = hash_len16(x, v1);
  y = hash_len16(y, w1);
  return U128{hash_len16(x + v2, w2) + y, hash_len16(x + w2, y + v2)};
}
__host__ __device__ inline U128 city128(const uint8_t* s, uint64_t len) {
  if (len >= 16) return city128_seed(s + 16, len - 16, U128{fetch64(s) ^ kK3, fetch64(s + 8)});
  if (len >= 8) return city128_seed(nullptr, 0, U128{fetch64(s) ^ (len * kK0), fetch64(s + len - 8) ^ kK1});
  return city128_seed(s, len, U128{kK0, kK1});
}
// the checksum of a block at `blk` (header at blk[16 .. 25), payload after it) into blk[0 .. 16)
__host__ __device__ inline void block_checksum(uint8_t* blk, uint32_t payload) {
  const U128 h = city128(blk + 16, 9u + payload);
  for (int k = 0; k < 8; k++) { blk[k] = (uint8_t)(h.first >> (8 * k)); blk[8 + k] = (uint8_t)(h.second >> (8 * k)); }
}

}  // namespace etl_ch
