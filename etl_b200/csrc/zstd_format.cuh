// zstd_format.cuh — a Zstandard (RFC 8878) block compressor for one fragment of at most 64 KiB, written as host + device
// code so that a host harness compiles the very same source (tests/emul/host_parquet_zstd.cpp, checked against pyarrow's
// libzstd in tests/test_parquet_zstd_cpu.py).  One thread compresses one fragment; the output depends only on the
// fragment's bytes.
//   * frame header: magic, Frame_Header_Descriptor 0xA0 (Single_Segment, 4-byte Frame_Content_Size, no checksum, no
//     dictionary id), the content size: 9 bytes;
//   * one block per fragment, self-contained: matches stay inside the fragment, every offset is written in full (no
//     repeat-offset codes), Huffman literals carry their own table (never Treeless) and sequence tables are Predefined,
//     RLE or FSE_Compressed (never Repeat).  So fragments compress independently and their blocks concatenate;
//   * a Compressed block only when strictly smaller than the fragment, otherwise RLE (all bytes equal) or Raw;
//   * match finder: 4-byte hash over a 2^kHashBits table of u16 positions (the Snappy finder's pattern, with backward
//     extension into the pending literals);
//   * literals: Raw, RLE or Huffman, whichever is smallest; the Huffman code is limited to kHufMaxBits, its weights are
//     written directly (at most 128) or FSE-compressed (accuracy log 6), one stream below 1 024 literals, else four;
//   * sequences: for each of literal lengths, offsets and match lengths the cheaper of the predefined distribution and a
//     table normalised from the block's own codes (counted exactly by running the state machine), RLE for one code.
#pragma once
#include <stdint.h>
#include <string.h>

namespace etl_zstd {

constexpr uint32_t kFrameHeader = 9;
constexpr uint32_t kHashBits = 13;
constexpr uint32_t kMinMatch = 4;
constexpr uint32_t kHufMaxBits = 11;
constexpr uint32_t kWeightLog = 6;                    // accuracy log of the FSE-compressed Huffman weights
enum { BLOCK_RAW = 0, BLOCK_RLE = 1, BLOCK_COMPRESSED = 2 };
enum { LIT_RAW = 0, LIT_RLE = 1, LIT_HUFFMAN = 2 };
enum { MODE_PREDEFINED = 0, MODE_RLE = 1, MODE_FSE = 2 };

// a block slot: the 3-byte block header and at most n content bytes (a Raw block)
__host__ __device__ inline uint32_t zstd_bound(uint32_t n) { return n + 3u; }
// scratch of one fragment of n bytes: n literal bytes and zstd_seqs(n) sequences of 8 bytes
__host__ __device__ inline uint32_t zstd_seqs(uint32_t n) { return n / kMinMatch + 1u; }

__host__ __device__ inline uint32_t ld32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
__host__ __device__ inline uint64_t ld64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
__host__ __device__ inline uint32_t highbit(uint32_t v) {   // v > 0
#ifdef __CUDA_ARCH__
  return 31u - (uint32_t)__clz(v);
#else
  return 31u - (uint32_t)__builtin_clz(v);
#endif
}
__host__ __device__ inline uint32_t ctz64(uint64_t v) {   // v > 0
#ifdef __CUDA_ARCH__
  return (uint32_t)__ffsll((long long)v) - 1u;
#else
  return (uint32_t)__builtin_ctzll(v);
#endif
}

// frame header of a frame of `content` bytes; returns kFrameHeader
__host__ __device__ inline uint32_t frame_header(uint32_t content, uint8_t* out) {
  out[0] = 0x28; out[1] = 0xB5; out[2] = 0x2F; out[3] = 0xFD; out[4] = 0xA0;
  for (int b = 0; b < 4; b++) out[5 + b] = (uint8_t)(content >> (8 * b));
  return kFrameHeader;
}
__host__ __device__ inline void block_header(uint8_t* out, bool last, uint32_t type, uint32_t size) {
  const uint32_t v = (last ? 1u : 0u) | (type << 1) | (size << 3);
  out[0] = (uint8_t)v; out[1] = (uint8_t)(v >> 8); out[2] = (uint8_t)(v >> 16);
}

// little-endian bit writer into [p, end): a write past end sets bad and stops storing
struct BitOut {
  uint8_t* p; uint8_t* end; uint64_t acc; uint32_t pos, bad;
  __host__ __device__ BitOut(uint8_t* o, uint8_t* e) : p(o), end(e), acc(0), pos(0), bad(0) {}
  __host__ __device__ void put(uint32_t k) {
    for (uint32_t b = 0; b < k; b++) {
      if (p < end) *p++ = (uint8_t)(acc >> (8 * b));
      else bad = 1;
    }
  }
  __host__ __device__ void add(uint32_t v, uint32_t nb) {   // nb <= 25
    acc |= (uint64_t)(v & ((1u << nb) - 1u)) << pos;
    pos += nb;
    if (pos >= 32) { put(4); acc >>= 32; pos -= 32; }
  }
  // the last bits (a backward stream first adds its end mark); returns one past the last byte
  __host__ __device__ uint8_t* finish(bool mark) {
    if (mark) add(1, 1);
    put((pos + 7) / 8);
    acc = 0; pos = 0;
    return p;
  }
};

// FSE encoding table of one distribution (state values in [L, 2L))
struct FseTable {
  uint16_t state[512];
  uint32_t dnb[64];          // deltaNbBits
  int32_t dfs[64];           // deltaFindState
  uint32_t log;              // accuracy log; 0: RLE (no state, no bits)
};

// the work space of one fragment (shared memory on the device)
struct Work {
  uint16_t hash[1u << kHashBits];
  uint32_t cnt[256];         // literal histogram; then the sequence codes' (LL at 0, OF at 64, ML at 128)
  uint32_t nw[512];          // Huffman node weights (leaves first)
  uint16_t parent[512];
  uint16_t order[256];       // present literal symbols, ascending by count
  uint16_t code[256];
  uint8_t nbits[256], weight[256];
  uint8_t spread[512];       // FSE symbol spread; Huffman node depths
  uint16_t cumul[65];
  int16_t norm[64];
  uint32_t wcnt[16];
  FseTable t[3];             // LL, OF, ML
  uint8_t nc[3][96];         // FSE_Compressed table descriptions
  uint32_t ncl[3];
};

// ------------------------------------------------------------------------------------------------ FSE
// predefined distributions (RFC 8878 §3.1.1.3.2.2), 4 bits per symbol holding norm + 1
__host__ __device__ inline int16_t predefined(uint32_t t, uint32_t s) {
  uint64_t w;
  if (t == 0) w = s < 16 ? 0x2223333333333345ull : s < 32 ? 0x2222234333333333ull : 0;
  else if (t == 1) w = s < 16 ? 0x2222222333222222ull : 0x0000000022222222ull;
  else w = s < 16 ? 0x2222222333333452ull : s < 32 ? 0x2222222222222222ull : s < 48 ? 0x0022222222222222ull : 0;
  return (int16_t)((w >> (4 * (s & 15))) & 15) - 1;
}
// per stream t (0 literal lengths, 1 offsets, 2 match lengths): the predefined accuracy log and largest code, and the
// largest accuracy log of a table of the block's own codes
__host__ __device__ inline uint32_t predef_log(uint32_t t) { return t == 1 ? 5u : 6u; }
__host__ __device__ inline uint32_t predef_max(uint32_t t) { return t == 0 ? 35u : t == 1 ? 28u : 52u; }
__host__ __device__ inline uint32_t max_log(uint32_t t) { return t == 1 ? 8u : 9u; }

// the encoding table of norm[0..max_sym] (-1: a less-than-one probability) at accuracy log al
__host__ __device__ inline void fse_build(FseTable& T, const int16_t* norm, uint32_t max_sym, uint32_t al, Work& W) {
  const uint32_t L = 1u << al, mask = L - 1, step = (L >> 1) + (L >> 3) + 3;
  uint32_t high = L - 1;
  W.cumul[0] = 0;
  for (uint32_t u = 1; u <= max_sym + 1; u++) {
    if (norm[u - 1] == -1) { W.cumul[u] = (uint16_t)(W.cumul[u - 1] + 1); W.spread[high--] = (uint8_t)(u - 1); }
    else W.cumul[u] = (uint16_t)(W.cumul[u - 1] + norm[u - 1]);
  }
  uint32_t pos = 0;
  for (uint32_t s = 0; s <= max_sym; s++)
    for (int i = 0; i < norm[s]; i++) {
      W.spread[pos] = (uint8_t)s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  for (uint32_t u = 0; u < L; u++) T.state[W.cumul[W.spread[u]]++] = (uint16_t)(L + u);
  int32_t total = 0;
  for (uint32_t s = 0; s <= max_sym; s++) {
    const int n = norm[s];
    if (n == 0) { T.dnb[s] = ((al + 1) << 16) - L; T.dfs[s] = 0; }
    else if (n == 1 || n == -1) { T.dnb[s] = (al << 16) - L; T.dfs[s] = total - 1; total++; }
    else {
      const uint32_t mbo = al - highbit((uint32_t)n - 1), msp = (uint32_t)n << mbo;
      T.dnb[s] = (mbo << 16) - msp; T.dfs[s] = total - n; total += n;
    }
  }
  T.log = al;
}
__host__ __device__ inline uint32_t fse_init(const FseTable& T, uint32_t s) {
  const uint32_t nb = (T.dnb[s] + (1u << 15)) >> 16;
  const uint32_t v = (nb << 16) - T.dnb[s];
  return T.state[(v >> nb) + T.dfs[s]];
}
__host__ __device__ inline uint32_t fse_step(const FseTable& T, uint32_t v, uint32_t s, uint32_t* nb) {
  *nb = (v + T.dnb[s]) >> 16;
  return T.state[(v >> *nb) + T.dfs[s]];
}
__host__ __device__ inline void fse_encode(const FseTable& T, uint32_t& v, uint32_t s, BitOut& b) {
  if (!T.log) return;
  uint32_t nb;
  const uint32_t nv = fse_step(T, v, s, &nb);
  b.add(v, nb);
  v = nv;
}

// counts c[0..max_sym] of `total` symbols (at least two distinct) normalised to sum 2^al, every present symbol >= 1 and
// none above cap: floors first, then one at a time to the most under-represented / from the least costly
__host__ __device__ inline void normalize(const uint32_t* c, uint32_t max_sym, uint32_t total, uint32_t al, uint32_t cap, int16_t* norm) {
  const uint32_t L = 1u << al;
  uint32_t sum = 0;
  for (uint32_t s = 0; s <= max_sym; s++) {
    uint32_t v = 0;
    if (c[s]) {
      v = (uint32_t)((uint64_t)c[s] * L / total);
      v = v < 1 ? 1 : v > cap ? cap : v;
    }
    norm[s] = (int16_t)v;
    sum += v;
  }
  while (sum < L) {
    int best = -1;
    for (uint32_t s = 0; s <= max_sym; s++)
      if (norm[s] > 0 && (uint32_t)norm[s] < cap &&
          (best < 0 || (uint64_t)c[s] * (uint32_t)norm[best] > (uint64_t)c[best] * (uint32_t)norm[s]))
        best = (int)s;
    norm[best]++; sum++;
  }
  while (sum > L) {
    int best = -1;
    for (uint32_t s = 0; s <= max_sym; s++)
      if (norm[s] > 1 && (best < 0 || (uint64_t)c[s] * (uint32_t)norm[best] < (uint64_t)c[best] * (uint32_t)norm[s]))
        best = (int)s;
    norm[best]--; sum--;
  }
}

// the FSE table description (RFC 8878 §4.1.1) of norm[0..max_sym] at accuracy log al into [o, end); 0 if it does not fit
__host__ __device__ inline uint32_t write_ncount(const int16_t* norm, uint32_t max_sym, uint32_t al, uint8_t* o, uint8_t* end) {
  BitOut b(o, end);
  b.add(al - 5, 4);
  int remaining = (1 << al) + 1, threshold = 1 << al;
  uint32_t nbits = al + 1, s = 0;
  bool prev0 = false;
  while (s <= max_sym && remaining > 1) {
    if (prev0) {
      uint32_t start = s;
      while (s <= max_sym && !norm[s]) s++;
      while (s >= start + 3) { start += 3; b.add(3, 2); }
      b.add(s - start, 2);
    }
    int count = norm[s++];
    const int mx = 2 * threshold - 1 - remaining;
    remaining -= count < 0 ? -count : count;
    count++;
    if (count >= threshold) count += mx;
    b.add((uint32_t)count, nbits - (count < mx ? 1u : 0u));
    prev0 = count == 1;
    while (remaining < threshold) { nbits--; threshold >>= 1; }
  }
  const uint8_t* e = b.finish(false);
  return b.bad ? 0 : (uint32_t)(e - o);
}

// ------------------------------------------------------------------------------------------------ Huffman literals
// code lengths (W.nbits) of the literal histogram W.cnt[0..max_sym]: Huffman by two queues over the symbols sorted by
// count, then limited to kHufMaxBits and made complete again.  Returns the longest length.
__host__ __device__ inline uint32_t huf_lengths(Work& W, uint32_t max_sym) {
  uint32_t m = 0;
  for (uint32_t s = 0; s <= max_sym; s++) {
    W.nbits[s] = 0;
    if (!W.cnt[s]) continue;
    uint32_t j = m++;                                    // insertion by count, stable in symbol order
    while (j > 0 && W.cnt[W.order[j - 1]] > W.cnt[s]) { W.order[j] = W.order[j - 1]; j--; }
    W.order[j] = (uint16_t)s;
  }
  if (m < 2) return 0;                                   // the callers pass at least two symbols
  for (uint32_t i = 0; i < m; i++) W.nw[i] = W.cnt[W.order[i]];
  uint32_t li = 0, ni = m, nn = m;
  for (uint32_t k = 0; k + 1 < m; k++) {
    uint32_t pick[2];
    for (int q = 0; q < 2; q++) pick[q] = (li < m && (ni >= nn || W.nw[li] <= W.nw[ni])) ? li++ : ni++;
    W.nw[nn] = W.nw[pick[0]] + W.nw[pick[1]];
    W.parent[pick[0]] = W.parent[pick[1]] = (uint16_t)nn;
    nn++;
  }
  W.spread[nn - 1] = 0;
  for (int i = (int)nn - 2; i >= 0; i--) W.spread[i] = (uint8_t)(W.spread[W.parent[i]] + 1);
  int32_t K = 0;                                         // Kraft sum in units of 2^-kHufMaxBits
  for (uint32_t i = 0; i < m; i++) {
    const uint32_t l = W.spread[i] > kHufMaxBits ? kHufMaxBits : W.spread[i];
    W.nbits[W.order[i]] = (uint8_t)l;
    K += 1 << (kHufMaxBits - l);
  }
  const int32_t full = 1 << kHufMaxBits;
  while (K > full) {                                     // lengthen the deepest code below the limit, rarest first
    int best = -1;
    for (uint32_t i = 0; i < m; i++) {
      const uint32_t l = W.nbits[W.order[i]];
      if (l < kHufMaxBits && (best < 0 || l > W.nbits[W.order[best]])) best = (int)i;
    }
    const uint32_t l = W.nbits[W.order[best]]++;
    K -= 1 << (kHufMaxBits - l - 1);
  }
  while (K < full) {                                     // shorten the deepest code, most frequent first
    int best = -1;
    for (int i = (int)m - 1; i >= 0; i--) {
      const uint32_t l = W.nbits[W.order[i]];
      if (l > 1 && (best < 0 || l > W.nbits[W.order[best]])) best = i;
    }
    const uint32_t l = W.nbits[W.order[best]]--;
    K += 1 << (kHufMaxBits - l);
  }
  uint32_t mx = 0;
  for (uint32_t s = 0; s <= max_sym; s++) mx = W.nbits[s] > mx ? W.nbits[s] : mx;
  return mx;
}

// the FSE-compressed weights W.weight[0..n) (n >= 2) into [o, end): description + two interleaved states; 0 if the
// weights cannot be written so (one distinct weight, or no room)
__host__ __device__ inline uint32_t huf_weights_fse(Work& W, uint32_t n, uint8_t* o, uint8_t* end) {
  for (int k = 0; k < 16; k++) W.wcnt[k] = 0;
  uint32_t mx = 0, distinct = 0;
  for (uint32_t i = 0; i < n; i++) { distinct += W.wcnt[W.weight[i]]++ == 0; mx = W.weight[i] > mx ? W.weight[i] : mx; }
  if (distinct < 2) return 0;
  // no probability above one half: every state then reads at least one bit, which is how the decoder finds the end
  normalize(W.wcnt, mx, n, kWeightLog, 1u << (kWeightLog - 1), W.norm);
  const uint32_t h = write_ncount(W.norm, mx, kWeightLog, o, end);
  if (!h) return 0;
  FseTable& T = W.t[0];
  fse_build(T, W.norm, mx, kWeightLog, W);
  BitOut b(o + h, end);
  uint32_t i = n, s1, s2;
  if (n & 1) { s1 = fse_init(T, W.weight[--i]); s2 = fse_init(T, W.weight[--i]); fse_encode(T, s1, W.weight[--i], b); }
  else { s2 = fse_init(T, W.weight[--i]); s1 = fse_init(T, W.weight[--i]); }
  while (i > 0) { fse_encode(T, s2, W.weight[--i], b); fse_encode(T, s1, W.weight[--i], b); }
  b.add(s2, kWeightLog);
  b.add(s1, kWeightLog);
  const uint8_t* e = b.finish(true);
  return b.bad ? 0 : (uint32_t)(e - o);
}

// one backward Huffman stream of lit[0..n) into [o, end); returns its end
__host__ __device__ inline uint8_t* huf_stream(const Work& W, const uint8_t* lit, uint32_t n, uint8_t* o, uint8_t* end, uint32_t* bad) {
  BitOut b(o, end);
  for (uint32_t i = n; i-- > 0;) b.add(W.code[lit[i]], W.nbits[lit[i]]);
  uint8_t* e = b.finish(true);
  *bad |= b.bad;
  return e;
}

__host__ __device__ inline uint32_t lit_header_len(uint32_t n) { return n < 32 ? 1u : n < 4096 ? 2u : 3u; }
// the header of a Raw / RLE literals section of n literals
__host__ __device__ inline uint32_t lit_header(uint8_t* o, uint32_t type, uint32_t n) {
  const uint32_t k = lit_header_len(n);
  const uint32_t v = k == 1 ? type | (n << 3) : k == 2 ? type | (1u << 2) | (n << 4) : type | (3u << 2) | (n << 4);
  for (uint32_t b = 0; b < k; b++) o[b] = (uint8_t)(v >> (8 * b));
  return k;
}

// the Huffman literals section of lit[0..n) (W.cnt its histogram, max_sym its largest symbol, at least two distinct)
// into [o, end); 0 when the code cannot be described or the section does not fit
__host__ __device__ inline uint32_t huf_literals(Work& W, const uint8_t* lit, uint32_t n, uint32_t max_sym, uint8_t* o, uint8_t* end) {
  const uint32_t hsz = n < 1024 ? 3u : n < 16384 ? 4u : 5u;
  if (o + hsz + 2 > end) return 0;
  const uint32_t maxb = huf_lengths(W, max_sym);
  for (uint32_t s = 0; s <= max_sym; s++) W.weight[s] = W.nbits[s] ? (uint8_t)(maxb + 1 - W.nbits[s]) : 0;
  uint8_t* p = o + hsz;
  if (max_sym <= 128) {                                  // direct: 4 bits per weight, the last symbol's implied
    const uint32_t nb = (max_sym + 1) / 2;
    if (p + 1 + nb > end) return 0;
    p[0] = (uint8_t)(127 + max_sym);
    for (uint32_t i = 0; i < nb; i++)
      p[1 + i] = (uint8_t)((W.weight[2 * i] << 4) | (2 * i + 1 < max_sym ? W.weight[2 * i + 1] : 0));
    p += 1 + nb;
  } else {
    const uint32_t f = huf_weights_fse(W, max_sym, p + 1, end);
    if (!f || f >= 128) return 0;
    p[0] = (uint8_t)f;
    p += 1 + f;
  }
  // canonical codes: longest first, symbols in order within a length
  uint32_t per[kHufMaxBits + 2] = {0}, val[kHufMaxBits + 2] = {0};
  for (uint32_t s = 0; s <= max_sym; s++) per[W.nbits[s]]++;
  uint32_t mn = 0;
  for (uint32_t l = maxb; l > 0; l--) { val[l] = mn; mn += per[l]; mn >>= 1; }
  for (uint32_t s = 0; s <= max_sym; s++) if (W.nbits[s]) W.code[s] = (uint16_t)val[W.nbits[s]]++;
  uint32_t bad = 0;
  if (n < 1024) p = huf_stream(W, lit, n, p, end, &bad);
  else {
    if (p + 6 > end) return 0;
    uint8_t* jump = p;
    p += 6;
    const uint32_t seg = (n + 3) / 4;
    for (uint32_t k = 0; k < 4; k++) {
      const uint32_t a = k * seg, e = k == 3 ? n : a + seg;
      uint8_t* q = huf_stream(W, lit + a, e - a, p, end, &bad);
      if (k < 3) { jump[2 * k] = (uint8_t)(q - p); jump[2 * k + 1] = (uint8_t)((q - p) >> 8); }
      p = q;
    }
  }
  if (bad) return 0;
  const uint64_t comp = (uint64_t)(p - o) - hsz;
  const uint64_t v = hsz == 3 ? LIT_HUFFMAN | ((uint64_t)n << 4) | (comp << 14)
                   : hsz == 4 ? LIT_HUFFMAN | (2u << 2) | ((uint64_t)n << 4) | (comp << 18)
                              : LIT_HUFFMAN | (3u << 2) | ((uint64_t)n << 4) | (comp << 22);
  for (uint32_t b = 0; b < hsz; b++) o[b] = (uint8_t)(v >> (8 * b));
  return (uint32_t)(p - o);
}

// the literals section of lit[0..n) into [o, end): RLE for one distinct byte, else the smaller of Huffman and Raw;
// 0 if it does not fit
__host__ __device__ inline uint32_t literals(Work& W, const uint8_t* lit, uint32_t n, uint8_t* o, uint8_t* end) {
  for (int s = 0; s < 256; s++) W.cnt[s] = 0;
  uint32_t max_sym = 0, distinct = 0;
  for (uint32_t i = 0; i < n; i++) { distinct += W.cnt[lit[i]]++ == 0; max_sym = lit[i] > max_sym ? lit[i] : max_sym; }
  const uint32_t raw = lit_header_len(n) + n;
  if (distinct == 1) {
    if (o + lit_header_len(n) + 1 > end) return 0;
    const uint32_t h = lit_header(o, LIT_RLE, n);
    o[h] = lit[0];
    return h + 1;
  }
  if (distinct >= 2) {
    const uint32_t h = huf_literals(W, lit, n, max_sym, o, end);
    if (h && h < raw) return h;
  }
  if (o + raw > end) return 0;
  const uint32_t h = lit_header(o, LIT_RAW, n);
  memcpy(o + h, lit, n);
  return raw;
}

// ------------------------------------------------------------------------------------------------ sequences
// a sequence: literal length (bits 0-20), match length (21-41), offset (42-63)
__host__ __device__ inline uint64_t seq_pack(uint32_t ll, uint32_t ml, uint32_t off) {
  return (uint64_t)ll | ((uint64_t)ml << 21) | ((uint64_t)off << 42);
}
__host__ __device__ inline uint32_t seq_ll(uint64_t q) { return (uint32_t)(q & 0x1FFFFF); }
__host__ __device__ inline uint32_t seq_ml(uint64_t q) { return (uint32_t)((q >> 21) & 0x1FFFFF); }
__host__ __device__ inline uint32_t seq_of(uint64_t q) { return (uint32_t)(q >> 42); }

__host__ __device__ inline uint32_t ll_code(uint32_t ll) {
  if (ll < 16) return ll;
  if (ll < 24) return 16 + ((ll - 16) >> 1);
  if (ll < 32) return 20 + ((ll - 24) >> 2);
  if (ll < 48) return 22 + ((ll - 32) >> 3);
  if (ll < 64) return 24;
  return highbit(ll) + 19;
}
__host__ __device__ inline uint32_t ll_bits(uint32_t c) { return c < 16 ? 0 : c < 20 ? 1 : c < 22 ? 2 : c < 24 ? 3 : c == 24 ? 4 : c - 19; }
__host__ __device__ inline uint32_t ll_base(uint32_t c) {
  return c < 16 ? c : c < 20 ? 16 + 2 * (c - 16) : c < 22 ? 24 + 4 * (c - 20) : c < 24 ? 32 + 8 * (c - 22) : c == 24 ? 48 : 1u << (c - 19);
}
// match length codes of m = match length - 3
__host__ __device__ inline uint32_t ml_code(uint32_t m) {
  if (m < 32) return m;
  if (m < 40) return 32 + ((m - 32) >> 1);
  if (m < 48) return 36 + ((m - 40) >> 2);
  if (m < 64) return 38 + ((m - 48) >> 3);
  if (m < 96) return 40 + ((m - 64) >> 4);
  if (m < 128) return 42;
  return highbit(m) + 36;
}
__host__ __device__ inline uint32_t ml_bits(uint32_t c) { return c < 32 ? 0 : c < 36 ? 1 : c < 38 ? 2 : c < 40 ? 3 : c < 42 ? 4 : c == 42 ? 5 : c - 36; }
__host__ __device__ inline uint32_t ml_base(uint32_t c) {
  return c < 32 ? c : c < 36 ? 32 + 2 * (c - 32) : c < 38 ? 40 + 4 * (c - 36) : c < 40 ? 48 + 8 * (c - 38) : c < 42 ? 64 + 16 * (c - 40)
       : c == 42 ? 96 : 1u << (c - 36);
}
// the code of stream t (0 literal length, 1 offset, 2 match length) of sequence q
__host__ __device__ inline uint32_t seq_code(uint64_t q, uint32_t t) {
  return t == 0 ? ll_code(seq_ll(q)) : t == 1 ? highbit(seq_of(q) + 3) : ml_code(seq_ml(q) - 3);
}

// the state bits of stream t's codes under table T (the extra bits are the same under every table)
__host__ __device__ inline uint64_t fse_cost(const FseTable& T, const uint64_t* seq, uint32_t ns, uint32_t t) {
  uint32_t v = fse_init(T, seq_code(seq[ns - 1], t));
  uint64_t bits = T.log;
  for (uint32_t i = ns - 1; i-- > 0;) {
    uint32_t nb;
    v = fse_step(T, v, seq_code(seq[i], t), &nb);
    bits += nb;
  }
  return bits;
}

// stream t's mode and table into W.t[t] (FSE_Compressed: its description in W.nc[t]); returns the mode, *sym the RLE code
__host__ __device__ inline uint32_t seq_table(Work& W, const uint64_t* seq, uint32_t ns, uint32_t t, uint32_t* sym) {
  const uint32_t* c = W.cnt + 64 * t;
  uint32_t max_sym = 0, distinct = 0;
  for (uint32_t s = 0; s < 64; s++) if (c[s]) { max_sym = s; distinct++; }
  FseTable& T = W.t[t];
  if (distinct == 1) { T.log = 0; *sym = max_sym; return MODE_RLE; }
  int16_t pre[64];
  for (uint32_t s = 0; s <= predef_max(t); s++) pre[s] = predefined(t, s);
  uint64_t best = ~0ull;
  if (max_sym <= predef_max(t)) { fse_build(T, pre, predef_max(t), predef_log(t), W); best = fse_cost(T, seq, ns, t); }
  // a table of the block's own codes, its accuracy log from the sequence count and the alphabet
  uint32_t al = max_log(t);
  const uint32_t lo = highbit(ns - 1) > 2 ? highbit(ns - 1) - 2 : 0;
  if (lo < al) al = lo;
  uint32_t mn = highbit(ns) + 1, ms = highbit(max_sym) + 2;
  mn = ms < mn ? ms : mn;
  al = mn > al ? mn : al;
  al = al < 5 ? 5 : al > max_log(t) ? max_log(t) : al;
  while ((1u << al) < 2 * distinct && al < max_log(t)) al++;
  normalize(c, max_sym, ns, al, 1u << al, W.norm);
  W.ncl[t] = write_ncount(W.norm, max_sym, al, W.nc[t], W.nc[t] + sizeof W.nc[t]);
  if (W.ncl[t]) {
    fse_build(T, W.norm, max_sym, al, W);
    if (fse_cost(T, seq, ns, t) + 8ull * W.ncl[t] < best) return MODE_FSE;
  }
  fse_build(T, pre, predef_max(t), predef_log(t), W);   // the predefined table won (or the only one that fits)
  return MODE_PREDEFINED;
}

// the sequences section of seq[0..ns) into [o, end); 0 if it does not fit
__host__ __device__ inline uint32_t sequences(Work& W, const uint64_t* seq, uint32_t ns, uint8_t* o, uint8_t* end) {
  if (o + 4 > end) return 0;
  uint32_t p = 0;
  if (ns < 128) o[p++] = (uint8_t)ns;
  else { o[p++] = (uint8_t)((ns >> 8) + 128); o[p++] = (uint8_t)ns; }   // ns <= 16 385 < 0x7F00
  if (!ns) return p;
  for (int s = 0; s < 192; s++) W.cnt[s] = 0;
  for (uint32_t i = 0; i < ns; i++)
    for (uint32_t t = 0; t < 3; t++) W.cnt[64 * t + seq_code(seq[i], t)]++;
  uint32_t mode[3], sym[3] = {0, 0, 0};
  for (uint32_t t = 0; t < 3; t++) mode[t] = seq_table(W, seq, ns, t, &sym[t]);
  o[p++] = (uint8_t)((mode[0] << 6) | (mode[1] << 4) | (mode[2] << 2));
  for (uint32_t t = 0; t < 3; t++) {
    if (mode[t] == MODE_RLE) { if (o + p + 1 > end) return 0; o[p++] = (uint8_t)sym[t]; }
    else if (mode[t] == MODE_FSE) {
      if (o + p + W.ncl[t] > end) return 0;
      memcpy(o + p, W.nc[t], W.ncl[t]);
      p += W.ncl[t];
    }
  }
  const FseTable &LL = W.t[0], &OF = W.t[1], &ML = W.t[2];
  BitOut b(o + p, end);
  const uint64_t z = seq[ns - 1];
  uint32_t cl = seq_code(z, 0), co = seq_code(z, 1), cm = seq_code(z, 2);
  uint32_t sml = ML.log ? fse_init(ML, cm) : 0, sof = OF.log ? fse_init(OF, co) : 0, sll = LL.log ? fse_init(LL, cl) : 0;
  b.add(seq_ll(z) - ll_base(cl), ll_bits(cl));
  b.add(seq_ml(z) - 3 - ml_base(cm), ml_bits(cm));
  b.add(seq_of(z) + 3 - (1u << co), co);
  for (uint32_t i = ns - 1; i-- > 0;) {
    const uint64_t q = seq[i];
    cl = seq_code(q, 0); co = seq_code(q, 1); cm = seq_code(q, 2);
    fse_encode(OF, sof, co, b);
    fse_encode(ML, sml, cm, b);
    fse_encode(LL, sll, cl, b);
    b.add(seq_ll(q) - ll_base(cl), ll_bits(cl));
    b.add(seq_ml(q) - 3 - ml_base(cm), ml_bits(cm));
    b.add(seq_of(q) + 3 - (1u << co), co);
  }
  if (ML.log) b.add(sml, ML.log);
  if (OF.log) b.add(sof, OF.log);
  if (LL.log) b.add(sll, LL.log);
  const uint8_t* e = b.finish(true);
  return b.bad ? 0 : (uint32_t)(e - o);
}

// ------------------------------------------------------------------------------------------------ match finder
__host__ __device__ inline uint32_t zhash(uint32_t v) { return (v * 2654435761u) >> (32 - kHashBits); }

// the greedy parse of in[0..n): sequences into seq, literals into lit; returns the sequence count, *nlit the literals
__host__ __device__ inline uint32_t parse(const uint8_t* in, uint32_t n, Work& W, uint8_t* lit, uint64_t* seq, uint32_t* nlit) {
  uint32_t ns = 0, nl = 0, anchor = 0;
  if (n >= 16) {
    for (uint32_t k = 0; k < (1u << kHashBits); k++) W.hash[k] = 0;
    const uint32_t limit = n - 4;                        // a 4-byte load at ip stays inside the fragment
    uint32_t ip = 1, skip = 32;
    while (ip <= limit) {
      const uint32_t cur = ld32(in + ip), h = zhash(cur);
      uint32_t cand = W.hash[h];
      W.hash[h] = (uint16_t)ip;
      if (cand < ip && ld32(in + cand) == cur) {
        uint32_t len = kMinMatch;
        for (;;) {
          if (ip + len + 8 <= n) {
            const uint64_t x = ld64(in + cand + len) ^ ld64(in + ip + len);
            if (x) { len += ctz64(x) >> 3; break; }
            len += 8;
          } else {
            while (ip + len < n && in[cand + len] == in[ip + len]) len++;
            break;
          }
        }
        while (ip > anchor && cand > 0 && in[ip - 1] == in[cand - 1]) { ip--; cand--; len++; }
        for (uint32_t k = anchor; k < ip; k++) lit[nl++] = in[k];
        seq[ns++] = seq_pack(ip - anchor, len, ip - cand);
        ip += len;
        anchor = ip;
        skip = 32;
        if (ip - 2 <= limit) W.hash[zhash(ld32(in + ip - 2))] = (uint16_t)(ip - 2);
        if (ip - 1 <= limit) W.hash[zhash(ld32(in + ip - 1))] = (uint16_t)(ip - 1);
      } else {
        ip += skip >> 5;                                 // incompressible stretches are skipped faster and faster
        skip++;
      }
    }
  }
  for (uint32_t k = anchor; k < n; k++) lit[nl++] = in[k];
  *nlit = nl;
  return ns;
}

// ------------------------------------------------------------------------------------------------ block
// one block of in[0..n) (n <= 65536) into out (zstd_bound(n) bytes): RLE when every byte is equal, Compressed when
// strictly smaller than n, else Raw; n == 0 is an empty Raw block.  Scratch: lit n bytes, seq zstd_seqs(n) entries.
// Returns the bytes written, block header included.
__host__ __device__ inline uint32_t zstd_block(const uint8_t* in, uint32_t n, bool last, uint8_t* out, Work& W, uint8_t* lit,
                                               uint64_t* seq) {
  bool same = n > 0;
  for (uint32_t i = 1; i < n && same; i++) same = in[i] == in[0];
  if (same) { block_header(out, last, BLOCK_RLE, n); out[3] = in[0]; return 4; }
  if (n > 0) {
    uint32_t nl;
    const uint32_t ns = parse(in, n, W, lit, seq, &nl);
    uint8_t* c = out + 3;
    uint8_t* end = c + n;
    const uint32_t a = literals(W, lit, nl, c, end);
    const uint32_t s = a ? sequences(W, seq, ns, c + a, end) : 0;
    if (a && s && a + s < n) { block_header(out, last, BLOCK_COMPRESSED, a + s); return 3 + a + s; }
  }
  block_header(out, last, BLOCK_RAW, n);
  memcpy(out + 3, in, n);
  return 3 + n;
}

}  // namespace etl_zstd
