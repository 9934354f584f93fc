// host_parquet_dict.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the dictionary pieces of the Parquet writer (etl_b200/csrc/parquet_format.cuh — the very source nvcc compiles
// for sm_90a) for the host, so that the CPU suite can check the index hybrid, the page headers and the footer of
// ETL_PQ_DICTIONARY against the Python restatement (tests/parquet_dict_ref.py, tests/test_parquet_dict_cpu.py).
// Nothing outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "parquet_format.cuh"

// the layouts of tests/emul/host_parquet.cpp's footer arguments: per leaf its name, ids, Parquet type, converted /
// logical type, flags (bit 0 required, bit 1 list, bit 2 utc); per chunk offset, num_values, usize, csize, null_count and
// min / max (min_len == UINT32_MAX: none)
struct EmuLeaf { const char* name; int32_t field_id, element_field_id; uint32_t ptype; int32_t converted; uint32_t logical, flags; };
struct EmuChunk { uint64_t offset, num_values, usize, csize, null_count; const uint8_t* min; const uint8_t* max; uint32_t min_len, max_len; };

// ETL_PQ_DICTIONARY pieces: the serial index hybrid over n indices at bit width w, the dictionary page header, the
// data page header with an encoding, and the footer with per-chunk dictionary fields (dict[c]: 0 / 1, data_offset[c],
// data_pages[c]) beside the chunks of emu_footer
extern "C" uint64_t emu_indices(const uint32_t* x, uint64_t n, uint32_t w, uint8_t* out) {
  return etl_pq::indices_encode(x, n, w, out);
}
extern "C" uint32_t emu_dict_page_header(uint32_t usize, uint32_t csize, uint32_t entries, uint8_t* out) {
  return etl_pq::dict_page_header(out, usize, csize, entries);
}
extern "C" uint32_t emu_page_header_enc(uint32_t usize, uint32_t csize, uint32_t num_values, uint32_t encoding, uint8_t* out) {
  return etl_pq::page_header(out, usize, csize, num_values, encoding);
}
extern "C" uint64_t emu_footer_dict(const EmuLeaf* leaves, uint32_t n_leaves, const uint64_t* rg_rows, uint32_t n_rg,
                                    const EmuChunk* chunks, const uint8_t* dict, const uint64_t* data_offset,
                                    const uint64_t* data_pages, uint32_t codec, uint8_t* out, uint64_t cap) {
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
                         has ? std::string((const char*)e.max, e.max_len) : std::string(),
                         dict[c] != 0, data_offset[c], data_pages[c]};
  }
  const std::vector<uint8_t> f = etl_pq::footer(L, std::vector<uint64_t>(rg_rows, rg_rows + n_rg), K, codec, "etl-b200 parquet writer");
  if (f.size() > cap) return 0;
  memcpy(out, f.data(), f.size());
  return f.size();
}
