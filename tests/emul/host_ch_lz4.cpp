// host_ch_lz4.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the DEVICE helpers of the ClickHouse INSERT-body compressor (etl_b200/csrc/clickhouse_lz4.cuh — the very
// source nvcc compiles for sm_90a) for the host, so that the CPU suite can check them against the Python restatement
// (tests/clickhouse_lz4_ref.py, tests/test_clickhouse_lz4_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "clickhouse_lz4.cuh"

extern "C" uint32_t emu_block_size(void) { return etl_ch::kBlock; }
// CityHash128 v1.0.2 of s[0 .. n) into out[0] = low64, out[1] = high64
extern "C" void emu_city128(const uint8_t* s, uint64_t n, uint64_t* out) {
  const etl_ch::U128 h = etl_ch::city128(s, n);
  out[0] = h.first;
  out[1] = h.second;
}
// one LZ4 sequence (match_len 0: the last, literals only); returns its length
extern "C" uint32_t emu_sequence(const uint8_t* lit, uint32_t lit_len, uint32_t offset, uint32_t match_len, uint8_t* out) {
  return etl_ch::lz4_sequence(lit, lit_len, offset, match_len, out);
}
// a whole block around a payload: header, then the checksum over header + payload (blk holds 25 + payload bytes, the
// payload already at blk + 25)
extern "C" void emu_frame(uint8_t* blk, uint32_t payload, uint32_t raw) {
  etl_ch::block_header(payload, raw, blk);
  etl_ch::block_checksum(blk, payload);
}
// the token + extension length the warp compressor reserves before it copies the literals
extern "C" uint32_t emu_lit_header_len(uint32_t lit) { return etl_ch::lz4_lit_header_len(lit); }
