// host_parsers.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE cell parsers (etl_b200/csrc/cell_parsers.cuh, float_parse.cuh — the very sources nvcc
// compiles for sm_90a) for the host with one-lane stand-ins for the warp intrinsics, so that the CPU suite can
// fuzz them against the oracle with millions of spellings (tests/test_device_parsers_on_host.py).  It is not a
// product path and nothing outside tests/ loads it: the product has no CPU fallback.
//
// emu_parse_cell mirrors what k_rows / k_heavy do for one cell (rows_kernel.cuh: UTF-8, then the per-kind fast path with
// the exact parser as fallback); with fast=0 it takes only the exact parsers (what parse_text_cell_impl does).
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

static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p = o + v; return o; }

#include "cell_parsers.cuh"
#include "float_parse.cuh"
#include "array_parse.cuh"

using namespace etl;

// the exact path: parse_text_cell_impl itself (array_parse.cuh); arrays through parse_array_any with a private heap region
static uint32_t exact(uint32_t kind, const uint8_t* s, uint32_t n, uint64_t soff, HeapCursor& hc, CellOut& o) {
  if (kind & ETL_K_ARRAY) {
    static thread_local unsigned long long arr_top;
    arr_top = 0;
    const uint32_t e = parse_array_any(ArrHeap{hc.heap, &arr_top, 0, 1ull << 16}, kind, s, n, o);
    return e == 0xFFFFFFFEu ? 0xFFFFFFFEu : e;
  }
  return parse_text_cell_impl(kind, s, n, soff, hc, o);
}

extern "C" uint32_t emu_parse_cell(uint32_t kind, const uint8_t* text, uint32_t n, int fast, uint8_t* tag, uint64_t* val,
                                   uint32_t* aux, uint8_t* heap, uint32_t heap_cap, uint32_t* heap_len) {
  // the device reads up to 16 bytes past a value (padded stream) and a few before it: give the copy the same slack
  static thread_local uint8_t buf[1 << 16];
  if (n > sizeof(buf) - 64) return 0xFFFFFFFFu;
  memset(buf, 0, 32); memcpy(buf + 32, text, n); memset(buf + 32 + n, 0, 32);
  const uint8_t* s = buf + 32;
  memset(heap, 0, heap_cap);
  CellOut o; o.tag = 0; o.val = 0; o.aux = 0;
  HeapCursor hc{heap, 0};
  uint32_t code = 0;
  if (!utf8_valid(s, n)) code = ETL_E_UTF8;      // event.rs:972 (k_rows: has_high_bits + the position-local rule)
  else if (!fast) code = exact(kind, s, n, 0, hc, o);
  else {
    const unsigned mask = 1u;
    int64_t iv = 0;
    switch (kind) {                                // parse_light_sync / parse_heavy_sync
      case ETL_K_STRING: o.tag = ETL_CELL_STRING; o.val = 0; o.aux = n; break;
      case ETL_K_I32: case ETL_K_I64: case ETL_K_I16: case ETL_K_U32: {
        const uint64_t pos_limit = kind == ETL_K_I32 ? 2147483647ull : (kind == ETL_K_I64 ? 9223372036854775807ull : (kind == ETL_K_I16 ? 32767ull : 4294967295ull));
        const uint64_t neg_limit = kind == ETL_K_U32 ? 0ull : pos_limit + 1ull;
        code = parse_int_sync(mask, s, n, kind != ETL_K_U32, pos_limit, neg_limit, &iv);
        o.tag = kind == ETL_K_I32 ? ETL_CELL_I32 : (kind == ETL_K_I64 ? ETL_CELL_I64 : (kind == ETL_K_I16 ? ETL_CELL_I16 : ETL_CELL_U32));
        o.val = (uint64_t)iv;
        break;
      }
      case ETL_K_NUMERIC: code = parse_numeric_sync(mask, s, n, heap, 0, o); break;
      case ETL_K_JSON:
        if (json_valid_sync(mask, s, n, kJsonT2)) { o.tag = ETL_CELL_JSON; o.val = 0; o.aux = n; } else code = ETL_E_JSON;
        break;
      case ETL_K_TIMESTAMPTZ: if (!fast_timestamptz(s, n, o)) code = exact(kind, s, n, 0, hc, o); break;
      case ETL_K_TIMESTAMP: if (!fast_timestamp(s, n, o)) code = exact(kind, s, n, 0, hc, o); break;
      case ETL_K_DATE: if (!fast_date(s, n, o)) code = exact(kind, s, n, 0, hc, o); break;
      case ETL_K_UUID: if (!fast_uuid(s, n, heap, 0, o)) code = exact(kind, s, n, 0, hc, o); break;
      case ETL_K_BOOL:
        if (n == 1 && (s[0] == 't' || s[0] == 'f')) { o.tag = ETL_CELL_BOOL; o.val = s[0] == 't'; } else code = ETL_E_BOOL;
        break;
      default: code = exact(kind, s, n, 0, hc, o); break;
    }
  }
  *tag = (uint8_t)o.tag; *val = o.val; *aux = o.aux;
  *heap_len = heap_cap;
  return code;
}
