// utf8.cuh — the word-wise UTF-8 range validator shared by k_rows, k_long_cells and k_copy_rows (sm_90a).
//
// Built on the position-local rule of cell_parsers.cuh (utf8_step_bad / utf8_chunk_valid).  Kept apart from
// wal_kernels.cuh so that the same source also compiles for the host (tests/emul/host_utf8.cpp), where the suite checks
// it against Python's strict decoder.
#pragma once
#include <stdint.h>

#include "cell_parsers.cuh"
namespace etl {

// UTF-8 check of a short/medium cell with word loads: all-ASCII words pass immediately
// any byte >= 0x80 in [s, s+n)?  Aligned 8-byte loads with the edges masked off (the bytes around a cell are
// readable: frame header before, padding after) — one load per word instead of the three of ld64u.
__device__ __forceinline__ bool has_high_bits(const uint8_t* s, uint32_t n) {
  if (n == 0) return false;
  const uintptr_t a = reinterpret_cast<uintptr_t>(s);
  const uint64_t* w = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  const uint32_t lead = (uint32_t)(a & 7u);
  const uint32_t nw = (lead + n + 7u) >> 3;          // words touched
  const uint32_t tail = (lead + n) & 7u;
  // every load is independent of the others: issue them in groups of four so that a 60-byte cell costs two
  // memory round trips instead of eight (a load-OR-load chain was the longest stall of the round-1 cell kernel)
  const uint64_t first = w[0], last = w[nw - 1];
  uint64_t acc = 0;
  for (uint32_t i = 1; i + 1 < nw; i += 4) {
    const uint64_t a0 = w[i];
    const uint64_t a1 = i + 2 < nw ? w[i + 1] : 0ull;
    const uint64_t a2 = i + 3 < nw ? w[i + 2] : 0ull;
    const uint64_t a3 = i + 4 < nw ? w[i + 3] : 0ull;
    acc |= a0 | a1 | a2 | a3;
  }
  const uint64_t lo_mask = ~0ull << (8u * lead);
  const uint64_t hi_mask = tail ? (1ull << (8u * tail)) - 1ull : ~0ull;
  if (nw == 1) acc = first & lo_mask & hi_mask;
  else acc |= (first & lo_mask) | (last & hi_mask);
  return (acc & 0x8080808080808080ull) != 0;
}

// UTF-8 validation of bytes [lo, hi) of one text cell by `nthreads` cooperating threads (one thread, a warp,
// or a half-warp of k_long_cells): 16-byte aligned chunks, 4 independent loads in flight per thread.
// An all-ASCII chunk costs one load + one test; a chunk with high bits is checked with the
// position-local rule over [clo, chi+3) so the following chunk never has to look back; the first 16
// bytes of the range are always checked with look-back (a range may start in the middle of a cell).
__device__ __forceinline__ bool utf8_range_bad(const uint8_t* cell, uint32_t cell_len, uint32_t lo, uint32_t hi, uint32_t t, uint32_t nthreads) {
  bool bad = false;
  if (hi <= lo) return false;
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(cell + lo);
  const uint32_t headn = min(hi - lo, (uint32_t)((16u - (uint32_t)(a0 & 15u)) & 15u));
  if (t == 0) {                                       // head: byte-serial only when it (or its look-back) has high bits
    const uint32_t hhi = min(lo + headn + 19u, hi), hlo = lo >= 3u ? lo - 3u : 0u;
    if (has_high_bits(cell + hlo, hhi - hlo)) bad |= !utf8_chunk_valid(cell, cell_len, lo, hhi);
  }
  const uint32_t body0 = lo + headn;
  const uint32_t nchunks = (hi - body0) / 16u;
  const uint4* body = reinterpret_cast<const uint4*>(cell + body0);
  uint32_t c = t;
  for (; c + 3 * nthreads < nchunks; c += 4 * nthreads) {
    const uint4 x0 = body[c], x1 = body[c + nthreads], x2 = body[c + 2 * nthreads], x3 = body[c + 3 * nthreads];
    const uint32_t h0 = (x0.x | x0.y | x0.z | x0.w), h1 = (x1.x | x1.y | x1.z | x1.w), h2 = (x2.x | x2.y | x2.z | x2.w), h3 = (x3.x | x3.y | x3.z | x3.w);
    if ((h0 | h1 | h2 | h3) & 0x80808080u) {
      if (h0 & 0x80808080u) { const uint32_t cl = body0 + c * 16u; bad |= !utf8_chunk_valid(cell, cell_len, cl, min(cl + 19u, hi)); }
      if (h1 & 0x80808080u) { const uint32_t cl = body0 + (c + nthreads) * 16u; bad |= !utf8_chunk_valid(cell, cell_len, cl, min(cl + 19u, hi)); }
      if (h2 & 0x80808080u) { const uint32_t cl = body0 + (c + 2 * nthreads) * 16u; bad |= !utf8_chunk_valid(cell, cell_len, cl, min(cl + 19u, hi)); }
      if (h3 & 0x80808080u) { const uint32_t cl = body0 + (c + 3 * nthreads) * 16u; bad |= !utf8_chunk_valid(cell, cell_len, cl, min(cl + 19u, hi)); }
    }
  }
  for (; c < nchunks; c += nthreads) {
    const uint4 x = body[c];
    if ((x.x | x.y | x.z | x.w) & 0x80808080u) {
      const uint32_t cl = body0 + c * 16u;
      bad |= !utf8_chunk_valid(cell, cell_len, cl, min(cl + 19u, hi));
    }
  }
  const uint32_t tail0 = body0 + nchunks * 16u;
  if (t == nthreads - 1 && tail0 < hi) {
    const uint32_t tlo = tail0 >= 3u ? tail0 - 3u : 0u;
    if (has_high_bits(cell + tlo, hi - tlo)) bad |= !utf8_chunk_valid(cell, cell_len, tail0, hi);
  }
  return bad;
}

}  // namespace etl
