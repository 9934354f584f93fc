// host_parquet_bloom.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the bloom filter pieces of the Parquet writer (etl_b200/csrc/parquet_format.cuh — the very source nvcc
// compiles for sm_90a) for the host, so that the CPU suite can check XXH64, the split-block insert, the
// BloomFilterHeader and the bitset sizing against the Python restatement (tests/parquet_bloom_ref.py,
// tests/test_parquet_bloom_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "parquet_format.cuh"

extern "C" uint64_t emu_xxh64(const uint8_t* p, uint64_t len) { return etl_pq::xxh64(p, len); }
extern "C" uint64_t emu_xxh64_u32(uint32_t v) { return etl_pq::xxh64_u32(v); }
extern "C" uint64_t emu_xxh64_u64(uint64_t v) { return etl_pq::xxh64_u64(v); }
// insert n hashes into a bitset of bytes bytes (u32 words), as k_bloom does without the atomics
extern "C" void emu_bloom_insert(uint32_t* words, uint32_t bytes, const uint64_t* h, uint64_t n) {
  for (uint64_t k = 0; k < n; k++) {
    uint32_t* w = words + 8ull * etl_pq::bloom_block(h[k], bytes / 32);
    for (int i = 0; i < 8; i++) w[i] |= etl_pq::bloom_mask(h[k], i);
  }
}
extern "C" uint32_t emu_bloom_header(uint8_t* out, uint32_t bytes) { return etl_pq::bloom_header(out, bytes); }
extern "C" uint64_t emu_bloom_bytes(uint64_t ndv, double fpp, uint64_t max_bytes) { return etl_pq::bloom_bytes(ndv, fpp, max_bytes); }
