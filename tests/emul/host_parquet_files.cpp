// host_parquet_files.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles the multi-file pieces of the Parquet writer (etl_b200/csrc/parquet_format.cuh — the very source nvcc compiles
// for sm_90a) for the host, so that the CPU suite can check the row-group table of etl_dec_parquet_write_files against
// a Python restatement and the footer tail the device serialises per file (schema prefix + footer_tail over flat chunk
// records, as k_footer reads them) against footer() (tests/test_parquet_files_cpu.py).  Nothing outside tests/ loads it.
#include <stdint.h>
#include <stdlib.h>

#define __device__
#define __host__
#define __forceinline__ inline

#include "parquet_format.cuh"

// the row-group table of K files (ro: K + 1 row offsets): row0 / rows / file per row group (room for cap), first: K + 1
// entries.  Returns the row groups, or UINT64_MAX when cap is short.
extern "C" uint64_t emu_row_groups(const uint64_t* ro, uint64_t K, uint64_t* row0, uint64_t* rows, uint64_t* file, uint64_t cap,
                                   uint64_t* first) {
  std::vector<uint64_t> f;
  const std::vector<etl_pq::RowGroup> t = etl_pq::row_group_table(ro, K, f);
  if (t.size() > cap) return UINT64_MAX;
  for (size_t g = 0; g < t.size(); g++) { row0[g] = t[g].row0; rows[g] = t[g].rows; file[g] = t[g].file; }
  for (uint64_t k = 0; k <= K; k++) first[k] = f[k];
  return t.size();
}

// a leaf as tests/emul/host_parquet.cpp passes it; a chunk record with every footer field and its statistic bytes
// inline (the device's record)
struct EmuLeaf { const char* name; int32_t field_id, element_field_id; uint32_t ptype; int32_t converted; uint32_t logical, flags; };
struct EmuRec {
  uint64_t offset, num_values, usize, csize, null_count, data_offset, data_pages, ci_offset, oi_offset, bloom_offset;
  uint32_t ci_len, oi_len, bloom_len, min_len, max_len, has, dict, page_index;
  uint8_t min[etl_pq::kStatMax], max[etl_pq::kStatMax];
};

static std::vector<etl_pq::Leaf> leaves_of(const EmuLeaf* leaves, uint32_t n_leaves) {
  std::vector<etl_pq::Leaf> L(n_leaves);
  for (uint32_t i = 0; i < n_leaves; i++)
    L[i] = etl_pq::Leaf{leaves[i].name, leaves[i].field_id, leaves[i].element_field_id, leaves[i].ptype, leaves[i].converted,
                        leaves[i].logical, (leaves[i].flags & 4) != 0, (leaves[i].flags & 1) != 0, (leaves[i].flags & 2) != 0};
  return L;
}

// footer() of the records (converted to the host's Chunk).  Returns its length (0 if cap is short).
extern "C" uint64_t emu_footer_host(const EmuLeaf* leaves, uint32_t n_leaves, const uint64_t* rg_rows, uint32_t n_rg,
                                    const EmuRec* recs, uint32_t codec, uint8_t* out, uint64_t cap) {
  std::vector<etl_pq::Chunk> K(n_leaves * (uint64_t)n_rg);
  for (size_t c = 0; c < K.size(); c++) {
    const EmuRec& e = recs[c];
    K[c] = etl_pq::Chunk{e.offset, e.num_values, e.usize, e.csize, e.null_count, e.has != 0,
                         e.has ? std::string((const char*)e.min, e.min_len) : std::string(),
                         e.has ? std::string((const char*)e.max, e.max_len) : std::string(),
                         e.dict != 0, e.data_offset, e.data_pages, e.page_index != 0, e.ci_offset, e.oi_offset, e.ci_len, e.oi_len,
                         e.bloom_offset, e.bloom_len};
  }
  const std::vector<uint8_t> f = etl_pq::footer(leaves_of(leaves, n_leaves), std::vector<uint64_t>(rg_rows, rg_rows + n_rg), K,
                                                codec, "etl-b200 parquet writer");
  if (f.size() > cap) return 0;
  memcpy(out, f.data(), f.size());
  return f.size();
}

// the schema prefix, then footer_tail over the records (row-group starts from rg0 on: any origin), sized by a counting
// pass as k_footer<false> does.  Returns the length (0 if cap is short).
extern "C" uint64_t emu_footer_split(const EmuLeaf* leaves, uint32_t n_leaves, const uint64_t* rg_rows, uint32_t n_rg, uint64_t rg0,
                                     const EmuRec* recs, uint32_t codec, uint8_t* out, uint64_t cap) {
  const std::vector<etl_pq::Leaf> L = leaves_of(leaves, n_leaves);
  etl_pq::TWriter pw(nullptr);
  etl_pq::footer_prefix(pw, L);
  std::vector<uint64_t> start(n_rg + 1, rg0);
  for (uint32_t g = 0; g < n_rg; g++) start[g + 1] = start[g] + rg_rows[g];
  const std::vector<etl_pq::LeafMeta> lm = etl_pq::leaf_meta(L);
  auto get = [&](uint64_t c) {
    const EmuRec& e = recs[c];
    return etl_pq::ChunkMeta{e.offset, e.num_values, e.usize, e.csize, e.null_count, e.data_offset, e.data_pages, e.ci_offset,
                             e.oi_offset, e.bloom_offset, e.ci_len, e.oi_len, e.bloom_len, e.min_len, e.max_len, e.has != 0,
                             e.dict != 0, e.page_index != 0, e.min, e.max};
  };
  const char* cb = "etl-b200 parquet writer";
  const uint64_t t = etl_pq::footer_tail(nullptr, lm.data(), n_leaves, start.data(), n_rg, get, codec, (const uint8_t*)cb,
                                         (uint32_t)strlen(cb));
  if (pw.n + t > cap) return 0;
  etl_pq::TWriter w(out);
  etl_pq::footer_prefix(w, L);
  const uint64_t t2 = etl_pq::footer_tail(out + w.n, lm.data(), n_leaves, start.data(), n_rg, get, codec, (const uint8_t*)cb,
                                          (uint32_t)strlen(cb));
  return t2 == t ? w.n + t : 0;
}
