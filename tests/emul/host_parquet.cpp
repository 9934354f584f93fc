// host_parquet.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the byte-level pieces of the Parquet writer (etl_b200/csrc/parquet_format.cuh — the very source nvcc compiles
// for sm_90a) for the host, so that the CPU suite can check the Snappy fragment compressor against pyarrow's Snappy and
// the level encoder, page header and footer against the Python restatement (tests/parquet_ref.py,
// tests/test_parquet_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "parquet_format.cuh"

// one Snappy stream of n bytes: the varint length, then the elements of independent 64 KiB fragments; out has room for
// 10 + Σ snappy_bound(fragment).  Returns its length.
extern "C" uint64_t emu_snappy(const uint8_t* in, uint64_t n, uint8_t* out) {
  uint16_t table[1u << etl_pq::kSnappyHashBits];
  uint64_t o = etl_pq::varint(n, out);
  for (uint64_t off = 0; off < n; off += etl_pq::kFragment) {
    const uint32_t len = (uint32_t)(n - off < etl_pq::kFragment ? n - off : etl_pq::kFragment);
    o += etl_pq::snappy_fragment(in + off, len, out + o, table);
  }
  return o;
}
// the level encoder over n level bytes (copied to an aligned, padded buffer as the kernel's scratch is)
extern "C" uint64_t emu_levels(const uint8_t* lv, uint64_t n, uint32_t w, uint8_t* out) {
  uint64_t* buf = (uint64_t*)calloc(n / 8 + 2, 8);
  memcpy(buf, lv, n);
  const uint64_t len = etl_pq::levels_encode((const uint8_t*)buf, n, w, out);
  free(buf);
  return len;
}
extern "C" uint32_t emu_page_header(uint32_t usize, uint32_t csize, uint32_t num_values, uint8_t* out) {
  return etl_pq::page_header(out, usize, csize, num_values);
}
// the footer of a file described by flat arrays: per leaf its name, ids, Parquet type, converted / logical type,
// flags (bit 0 required, bit 1 list, bit 2 utc); per chunk (row-group major) offset, num_values, usize, csize,
// null_count and min / max (min_len == UINT32_MAX: none).  Returns the length written to out (cap bytes), 0 if short.
struct EmuLeaf { const char* name; int32_t field_id, element_field_id; uint32_t ptype; int32_t converted; uint32_t logical, flags; };
struct EmuChunk { uint64_t offset, num_values, usize, csize, null_count; const uint8_t* min; const uint8_t* max; uint32_t min_len, max_len; };
extern "C" uint64_t emu_footer(const EmuLeaf* leaves, uint32_t n_leaves, const uint64_t* rg_rows, uint32_t n_rg,
                               const EmuChunk* chunks, uint32_t codec, uint8_t* out, uint64_t cap) {
  std::vector<etl_pq::Leaf> L(n_leaves);
  for (uint32_t i = 0; i < n_leaves; i++)
    L[i] = etl_pq::Leaf{leaves[i].name, leaves[i].field_id, leaves[i].element_field_id, leaves[i].ptype, leaves[i].converted,
                        leaves[i].logical, (leaves[i].flags & 4) != 0, (leaves[i].flags & 1) != 0, (leaves[i].flags & 2) != 0};
  std::vector<etl_pq::Chunk> K(n_leaves * n_rg);
  for (size_t c = 0; c < K.size(); c++) {
    const EmuChunk& e = chunks[c];
    const bool has = e.min_len != UINT32_MAX;
    K[c] = etl_pq::Chunk{e.offset, e.num_values, e.usize, e.csize, e.null_count, has,
                         has ? std::string((const char*)e.min, e.min_len) : std::string(),
                         has ? std::string((const char*)e.max, e.max_len) : std::string()};
  }
  const std::vector<uint8_t> f = etl_pq::footer(L, std::vector<uint64_t>(rg_rows, rg_rows + n_rg), K, codec, "etl-b200 parquet writer");
  if (f.size() > cap) return 0;
  memcpy(out, f.data(), f.size());
  return f.size();
}
