// host_utf8.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE UTF-8 validators (etl_b200/csrc/cell_parsers.cuh and utf8.cuh — the very sources nvcc compiles for
// sm_90a) for the host with one-lane stand-ins, so that tests/test_utf8_paths_cpu.py can check millions of cells against
// Python's strict decoder.  Batch entry points: one ctypes call runs a whole arena of cells.  Nothing outside tests/
// loads it: the product has no CPU fallback.
//
// Every cell is copied into a scratch buffer at the requested alignment mod 16 with 64 bytes on each side filled with
// 0xFF: has_high_bits reads whole aligned words around a cell, and a byte outside the cell must never reach a verdict.
#include <stdint.h>
#include <string.h>

#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
template <typename T> static inline T min(T a, T b) { return a < b ? a : b; }
template <typename T> static inline T max(T a, T b) { return a > b ? a : b; }
static inline bool __any_sync(unsigned, bool p) { return p; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
#define __align__(n) __attribute__((aligned(n)))
static inline uint64_t __umul64hi(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
  const uint64_t src = ((uint64_t)b << 32) | a;
  uint32_t out = 0;
  for (int i = 0; i < 4; i++) out |= (uint32_t)((src >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
  return out;
}
struct __attribute__((aligned(16))) uint4 { uint32_t x, y, z, w; };

#include "cell_parsers.cuh"
#include "utf8.cuh"

using namespace etl;

namespace {
constexpr uint32_t kPad = 64;
constexpr uint32_t kMaxCell = 1u << 16;
alignas(64) uint8_t g_scratch[kPad + 16 + kMaxCell + kPad];

const uint8_t* place(const uint8_t* src, uint32_t n, uint32_t align) {
  memset(g_scratch, 0xFF, sizeof g_scratch);
  uint8_t* cell = g_scratch + kPad + (align & 15u);
  memcpy(cell, src, n);
  return cell;
}
}  // namespace

// out[i] = 1 when utf8_valid accepts cell i: bytes [off[i], off[i + 1]) of the arena
extern "C" void emu_utf8_valid_batch(const uint8_t* arena, const uint64_t* off, uint64_t n_cells, uint8_t* out) {
  for (uint64_t i = 0; i < n_cells; i++) out[i] = utf8_valid(arena + off[i], (uint32_t)(off[i + 1] - off[i])) ? 1 : 0;
}

// Range checks over cells of the arena (cell c = bytes [off[c], off[c + 1])).  Range r asks about bytes [lo[r], hi[r]) of
// cell cell_of[r]; consecutive ranges of one cell reuse its placement.  mode:
//   0  utf8_range_bad for every t in [0, nthreads): out[r] = bit t set when thread t reports a violation
//   1  out[r] = !utf8_chunk_valid(cell, n, lo, hi)
//   2  utf8_chunk_valid_at on a stream: stream_lead[r] ASCII bytes, the cell, stream_tail[r] ASCII bytes; the range is moved
//      by the lead, and a range that ends at the cell's end runs on to the stream's end (what the dead-segment pass sees)
extern "C" void emu_utf8_ranges(int mode, const uint8_t* arena, const uint64_t* off, const uint32_t* cell_of, const uint32_t* lo,
                                const uint32_t* hi, uint64_t n_ranges, uint32_t align, uint32_t nthreads, const uint8_t* stream_lead,
                                const uint8_t* stream_tail, uint32_t* out) {
  uint32_t placed = 0xFFFFFFFFu, placed_lead = 0, placed_tail = 0;
  const uint8_t* cell = nullptr;
  for (uint64_t r = 0; r < n_ranges; r++) {
    const uint32_t c = cell_of[r];
    const uint32_t n = (uint32_t)(off[c + 1] - off[c]);
    if (n > kMaxCell) { out[r] = 0xFFFFFFFFu; continue; }
    if (mode == 2) {
      const uint32_t lead = stream_lead[r], tail = stream_tail[r];
      if (c != placed || lead != placed_lead || tail != placed_tail) {
        memset(g_scratch, 0xFF, sizeof g_scratch);
        uint8_t* s = g_scratch + kPad + (align & 15u);
        memset(s, 'a', lead);
        memcpy(s + lead, arena + off[c], n);
        memset(s + lead + n, 'z', tail);
        cell = s;
        placed = c; placed_lead = lead; placed_tail = tail;
      }
      const uint64_t sn = (uint64_t)lead + n + tail;
      const uint64_t slo = lead + lo[r], shi = hi[r] == n ? sn : lead + hi[r];
      out[r] = utf8_chunk_valid_at(cell, sn, slo, shi) ? 0u : 1u;
      continue;
    }
    if (c != placed) { cell = place(arena + off[c], n, align); placed = c; }
    if (mode == 1) { out[r] = utf8_chunk_valid(cell, n, lo[r], hi[r]) ? 0u : 1u; continue; }
    uint32_t m = 0;
    for (uint32_t t = 0; t < nthreads; t++)
      if (utf8_range_bad(cell, n, lo[r], hi[r], t, nthreads)) m |= 1u << t;
    out[r] = m;
  }
}

// has_high_bits on bytes [lo, hi) of each cell, placed as above: out[r] = 1 when a byte >= 0x80 lies in the range
extern "C" void emu_has_high_bits(const uint8_t* arena, const uint64_t* off, const uint32_t* cell_of, const uint32_t* lo,
                                  const uint32_t* hi, uint64_t n_ranges, uint32_t align, uint8_t* out) {
  for (uint64_t r = 0; r < n_ranges; r++) {
    const uint32_t c = cell_of[r];
    const uint8_t* cell = place(arena + off[c], (uint32_t)(off[c + 1] - off[c]), align);
    out[r] = has_high_bits(cell + lo[r], hi[r] - lo[r]) ? 1 : 0;
  }
}
