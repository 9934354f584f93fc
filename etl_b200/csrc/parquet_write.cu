// parquet_write.cu — the Iceberg destination's Parquet data file, written on the device from an Arrow emit
// (etl_dec_arrow_emit with ETL_ARROW_ALL_COLUMNS [| ETL_ARROW_CDC_COLUMNS]).  Replaces what iceberg-rust's ParquetWriter
// does on the host for IcebergClient::write_record_batch (crates/etl-destinations/src/iceberg/client.rs:324-379):
// encode every value again, build the levels, Snappy-compress the pages and compute the column statistics behind the
// DataFile metrics.  The format rules are in include/etl_decode.h; the byte-level pieces are in parquet_format.cuh.
//
// One engine writes K files, file k the rows [ro[k], ro[k + 1]) (etl_dec_parquet_write_files; the single-file calls are
// K = 1).  The plan runs once over [ro[0], ro[K]); the row-group table (row_group_table of parquet_format.cuh: row groups
// restart in every file) replaces uniform cuts, so a chunk is (row group, leaf) of the whole call and each file's chunks,
// pages and filters are contiguous ranges of the call's (FileRec).  Every offset a file holds is relative to the file.
// Stages (one leaf per column: a flat column, or the element of a List column):
//   1. Plan.  k_plan, a thread per (row, leaf): level entries (1, or max(1, list length)), non-null values and PLAIN
//      value bytes (Boolean: bits) of the row, and a required column's first null row (atomicMin).  Three scans per leaf
//      (emit_scan.cuh) give their prefix sums.  k_cut, a thread per (leaf, row group), walks the greedy page rule with a
//      binary search over the value prefix sums; it runs twice, counting and then writing the pages.  SYNC 1 (the page
//      counts, the totals and the required-null rows) sizes every buffer from bounds, so no later step waits for sizes.
//   1'. Dictionaries (ETL_PQ_DICTIONARY).  k_cut puts a dictionary slot (a Page of kind 1) in front of the data pages of
//      every chunk of a non-Boolean leaf.  k_dict_setup sizes each chunk's open-addressing table from its non-null count
//      (the NN prefix sums), a scan places the tables; k_dict_insert (per leaf, grid-stride) inserts every non-null item,
//      a slot keeping the smallest chunk-relative item of its value by atomicMin, and adds each new entry's PLAIN size to
//      its chunk, marking it for fallback past 1 MiB (exact whatever the order: the entries are a set); k_dict_mark flags
//      the first occurrences (an item equal to its slot's value) and the scans of emit_scan.cuh turn the flags into
//      entry ids in item order and, for byte arrays, the entry sizes into PLAIN offsets; k_dict_finish decides each chunk
//      and its bit width; k_dict_page writes the entries into the dictionary slot.  k_encode<true> writes a dictionary
//      chunk's compacted entry ids and encodes their runs with the whole CTA (encode_indices); k_page gives a slot the
//      DICTIONARY_PAGE header, or no bytes when its chunk is PLAIN, so a fallen-back chunk is the PLAIN chunk.
//   2. Encode.  k_encode, a CTA per page: the page's level bytes into scratch (thread per row), the RLE hybrid by one
//      thread per section over whole 8-entry groups (one u64 load per group), then the non-null values compacted with a
//      block scan over the validity: fixed width at rank * width, Booleans by atomicOr into a zeroed bit scratch, byte
//      arrays as length + bytes with every value copied by the whole warp.  The same pass reduces the page's statistics
//      (min / max as item indices, NaN count).  The payload goes to a slot sized by the bound of the page.
//   3. Compress (ETL_PQ_SNAPPY).  k_snappy, a CTA per 64 KiB fragment slot of every page, runs the fragment compressor
//      of parquet_format.cuh on one thread, its hash table in shared memory, into a slot of snappy_bound bytes.
//      (ETL_PQ_ZSTD) k_zstd, in the same place and shape, runs the block compressor of zstd_format.cuh: each fragment
//      one self-contained Zstandard block (header included) in a slot of zstd_bound bytes, its work space in shared
//      memory, its literals and sequences in scratch placed by the fragment's payload position.  k_page writes the
//      preamble (Snappy's length varint, or the 9-byte Zstandard frame header) and the page header (its varint widths
//      depend on the sizes) and the page's file bytes; a scan gives the pages' offsets (a file's: minus its first
//      page's); k_gather (stage 6), a CTA per page, copies header + payload (+ preamble and fragments) to its place in
//      the output, whose size is the sum of the bounds.  The dictionary slot, the page index and the bloom filters
//      follow csize / hlen, so they need nothing per codec.
//   4. Statistics.  k_chunk, a thread per (leaf, row group), folds the page candidates and sizes of its chunk, k_leaf the
//      chunks of a leaf; both write the PLAIN bytes of min / max (−0.0 / +0.0 for a zero float, none above 64 bytes).
//   4b. Page index (ETL_PQ_PAGE_INDEX).  k_index<false>, a warp per chunk with lanes over its data pages: each page's
//      ColumnIndex entry (null flag, bounds truncated by index_min / index_max, null count) and PageLocation sizes, the
//      boundary order from adjacent non-null pages' untruncated bounds, the chunk's ColumnIndex / OffsetIndex lengths;
//      one k_blk_scan over the 2 × chunks lengths (laid out per file: its ColumnIndexes, then its OffsetIndexes) places
//      them; k_index_place puts each file-relative offset and length into the chunk record, behind the file's pages and
//      filters; k_index<true> (stage 6) writes them.  k_row_max (before SYNC 1) bounds an untruncated byte-array
//      maximum by the leaf's longest row.
//   4c. Bloom filters (etl_dec_parquet_write_bloom).  k_chunk_nn (before SYNC 1) gives each chunk's non-null values, from
//      which the host sizes every bitset and places the filters (row-group major) in each file's region behind its
//      pages, in front of its page index (k_chunk puts the file-relative offset into the chunk record).  One memset
//      zeroes the bitsets' scratch; k_bloom, per filtered leaf and grid-stride over its items, hashes each non-null value
//      (XXH64 of its PLAIN bytes, a byte array serially by its thread) and sets its 8 bits by atomicOr; k_bloom_write
//      (stage 6) copies each header and bitset into its file.  A dictionary chunk's filter is built from its values like
//      any other, so it equals its PLAIN form's.
//   5. Footers, on the device: the schema prefix (the same for every file) is serialised once on the host; k_footer<false>,
//      a warp per file, lanes over its tail's units (tail_unit of parquet_format.cuh: a ColumnChunk each), sizes the
//      tail and the file (4 + pages + filters + index + footer + 8); a scan over the sizes places the files.
//   6. Bytes, each written once at base[file] + its relative offset: k_gather, k_bloom_write, k_index<true>, and
//      k_footer<true> (both magics, prefix, tail, length).  k_leaf, a thread per (file, leaf), folds the metrics.
//      SYNC 2 copies the files' offsets and the (file, leaf) records back; SYNC 3 only with to_host (the pinned copy).
// Per file, beside the scratch of one call over the whole range: a 72 B FileRec, 8 B of size / place and a ChunkOut
// (248 B) per leaf; per row group 12 B of table; once the schema prefix, names and created_by.  Per page (a file has
// at least one per leaf): a 216 B Page, 32 B of slot scans, 64 B of level scratch, a compressed slot sized by its own
// payload (8 B + the bound of each fragment, 32 B + 7/6 of its bytes), and 48 B of header room in the output.
// Scratch: two cudaMalloc blocks, what the plan needs and then the rest once sized, cut into the named regions of
// Call::regions, each 256-aligned with 64 B of slack behind it: at most 16 KiB per call on top of the terms here.
// Per (row, leaf) 3 × 4 B lengths + 3 × 8 B prefix sums; per level entry 2 B (+ 64 B per page of the leaf);
// Boolean leaves 1 bit per item (+ 4 B per page of the leaf); per page a bounded payload slot (the PLAIN value bytes + levels_bound per section) and,
// with Snappy, a compressed slot of snappy_bound per fragment; with ETL_PQ_ZSTD, one of zstd_bound (64 KiB + 3 B) per
// fragment, and 1 B of literal + 2 B of sequence scratch per payload byte (+ 8 B per fragment).  ETL_PQ_DICTIONARY adds, per item of an eligible leaf
// (bounded by its level entries), 4 B slot + 4 B flag + 4 B entry size / index + 2 × 8 B prefix sums and 0.5 B of run
// heads (+ 12 B per page), the chunks' tables (4 B × pow2 >= 2 × non-null values: at most 16 B per value), a dictionary
// slot per chunk (at most 1 MiB, at most the chunk's PLAIN bytes) and 32 B more per data page slot.  ETL_PQ_PAGE_INDEX
// adds 4 B per leaf, 40 B of IndexChunk + 16 B of lengths per chunk, and in the file's buffer 189 B per page + 64 B per
// chunk (+ for a byte-array leaf with a row over 64 bytes, its longest row per page, at most its value bytes).  Bloom
// filters add 8 B of non-null count + 24 B of BloomChunk per chunk, each filtered chunk's bitset in scratch, and in the
// file's buffer its header (at most 19 B) and bitset.
// ptxas -v (sm_90a, CUDA 12.9): see the comment at the end of this file.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "etl_decode.h"
#include "emit_scan.cuh"
#include "parquet_format.cuh"
#include "zstd_format.cuh"

namespace {

using namespace etl_pq;

struct LeafDev {
  uint32_t atype;            // ETL_ARROW_* of the values (a List: of its child)
  uint32_t is_list, required, max_def, max_rep, w;   // w: bit width of the definition level
  uint32_t fixed;            // PLAIN width of a fixed-width value (Boolean: 0)
  uint32_t off64;            // LargeBinary offsets
  uint64_t bscr;             // Boolean: first word of the leaf's bit scratch
  const uint8_t* lvalid;     // List: validity of the lists
  const int32_t* loffs;      // List: offsets of the lists
  const uint8_t* valid;      // validity of the values (the column, or the List's child)
  const uint8_t* values;     // fixed width / Boolean bits
  const void* offs;          // byte arrays
  const uint8_t* data;
  uint64_t dscr, hscr;       // ETL_PQ_DICTIONARY: first item slot of the leaf's dictionary scratch / of its run heads
};
struct Page {
  uint32_t leaf, chunk;
  uint64_t lp;               // index of the page among the pages of its leaf (places its level and bit scratch)
  uint64_t row0, row1;       // local rows [row0, row1)
  uint64_t e0, e1;           // level entries (prefix of the leaf)
  uint64_t it0, it1;         // items of the value column
  uint64_t nn, vbytes, ubound, lscr;   // non-null values, PLAIN value bytes, payload bound, level scratch offset
  uint64_t usize, csize;
  uint32_t hlen, plen;       // page header / preamble bytes (Snappy's length varint, Zstandard's frame header)
  uint64_t min_it, max_it, nan;
  uint32_t kind, _pad;       // 0 data page; 1 the dictionary slot in front of a chunk's data pages (ETL_PQ_DICTIONARY)
  uint8_t hdr[kPageHeaderMax];
  uint8_t pre[12];           // at most 10 (a varint of a 32-bit size) or 9 (etl_zstd::kFrameHeader) bytes
};
struct ChunkOut {
  uint64_t offset, num_values, usize, csize, null_count, nan_count;
  uint64_t data_offset, data_pages;   // the first data page and the data pages (they differ from offset with a dictionary)
  uint32_t has, min_len, max_len, dict;
  uint8_t min[kStatMax], max[kStatMax];
  uint64_t ci_offset, oi_offset;      // ETL_PQ_PAGE_INDEX: file offsets of the chunk's ColumnIndex (ci_len 0: none) and
  uint32_t ci_len, oi_len;            // OffsetIndex
  uint64_t bloom_offset;              // bloom filter: file offset of its header, header + bitset bytes (0: none)
  uint32_t bloom_len, page_index;     // page_index: the call has ETL_PQ_PAGE_INDEX
};
// bloom filters (etl_dec_parquet_write_bloom): one record per chunk (row-group major); bytes 0: no filter
struct BloomChunk {
  uint64_t word;             // first u32 word of the chunk's bitset in the bloom scratch (32-byte aligned)
  uint64_t off;              // the filter's offset (its header) among the call's filters (FileRec.bloom0: its file's first)
  uint32_t bytes, hlen;      // bitset bytes, header bytes
};
// one file of the call (etl_dec_parquet_write_files; the single-file calls are one of it).  Host: its row groups, pages
// and bloom-filter bytes as ranges of the call's (chunks row-group major, so each file's are contiguous); device: the
// sizes of its parts.  Every offset inside a file is relative to the file.
struct FileRec {
  uint64_t rg0, rg1, page0, page1, bloom0, bloom1;
  uint64_t data, index, footer;       // the pages' bytes, the page index's, the footer's (without length and magic)
};
constexpr uint64_t kNone = ~0ull;
// ETL_PQ_DICTIONARY: one record per chunk (Boolean chunks have none: dict stays 0)
struct DictChunk {
  unsigned long long bytes;  // PLAIN size of the entries claimed so far
  uint64_t it0, it1;         // the chunk's items
  uint64_t tab;              // its table's first slot
  uint64_t page;             // its dictionary slot
  uint64_t entries;
  uint32_t mask;             // table slots - 1
  uint32_t fallback;         // the entries passed kDictBytes (or filled the table, which implies it): PLAIN chunk
  uint32_t dict, width;      // k_dict_finish: dictionary-encoded, index bit width
};
constexpr uint32_t kEmpty = 0xffffffffu;
constexpr uint32_t kInsBlocks = 1024, kInsThreads = 256;   // k_dict_insert's grid-stride launch
// entries a table must hold: every entry up to the first past kDictBytes (each entry is >= 4 PLAIN bytes), plus one
// insert in flight per thread of k_dict_insert when the fallback mark is set; a table that fills anyway also proves it
constexpr uint64_t kDictCap = kDictBytes / 4 + 1 + (uint64_t)kInsBlocks * kInsThreads;
constexpr uint32_t kLongBytes = 32;   // longer byte arrays are hashed and compared by the whole warp

__device__ __forceinline__ bool bit(const uint8_t* v, uint64_t i) { return (v[i >> 3] >> (i & 7)) & 1u; }
__device__ __forceinline__ uint64_t byte_off(const LeafDev& L, uint64_t i) {
  return L.off64 ? (uint64_t)((const int64_t*)L.offs)[i] : (uint64_t)(uint32_t)((const int32_t*)L.offs)[i];
}
__device__ __forceinline__ bool is_bytes(const LeafDev& L) { return L.atype == ETL_ARROW_UTF8 || L.atype == ETL_ARROW_LARGE_BINARY; }
__device__ __forceinline__ bool is_float(const LeafDev& L) { return L.atype == ETL_ARROW_FLOAT32 || L.atype == ETL_ARROW_FLOAT64; }
__device__ __forceinline__ bool is_nan(const LeafDev& L, uint64_t i) {
  if (L.atype == ETL_ARROW_FLOAT32) { const float f = ((const float*)L.values)[i]; return f != f; }
  if (L.atype == ETL_ARROW_FLOAT64) { const double d = ((const double*)L.values)[i]; return d != d; }
  return false;
}
// the type-defined order of two present, non-NaN items: < 0, 0, > 0
__device__ int cmp_items(const LeafDev& L, uint64_t a, uint64_t b) {
  switch (L.atype) {
    case ETL_ARROW_BOOLEAN: return (int)bit(L.values, a) - (int)bit(L.values, b);
    case ETL_ARROW_INT32: case ETL_ARROW_DATE32: { const int32_t x = ((const int32_t*)L.values)[a], y = ((const int32_t*)L.values)[b]; return x < y ? -1 : x > y; }
    case ETL_ARROW_FLOAT32: { const float x = ((const float*)L.values)[a], y = ((const float*)L.values)[b]; return x < y ? -1 : x > y; }
    case ETL_ARROW_FLOAT64: { const double x = ((const double*)L.values)[a], y = ((const double*)L.values)[b]; return x < y ? -1 : x > y; }
    case ETL_ARROW_UUID: {
      const uint8_t* x = L.values + a * 16; const uint8_t* y = L.values + b * 16;
      for (int k = 0; k < 16; k++) if (x[k] != y[k]) return x[k] < y[k] ? -1 : 1;
      return 0;
    }
    case ETL_ARROW_UTF8: case ETL_ARROW_LARGE_BINARY: {
      const uint64_t a0 = byte_off(L, a), al = byte_off(L, a + 1) - a0, b0 = byte_off(L, b), bl = byte_off(L, b + 1) - b0;
      const uint64_t m = al < bl ? al : bl;
      for (uint64_t k = 0; k < m; k++) if (L.data[a0 + k] != L.data[b0 + k]) return L.data[a0 + k] < L.data[b0 + k] ? -1 : 1;
      return al < bl ? -1 : al > bl;
    }
    default: { const int64_t x = ((const int64_t*)L.values)[a], y = ((const int64_t*)L.values)[b]; return x < y ? -1 : x > y; }
  }
}
// fold candidate c into (mn, mx); kNone = no candidate
__device__ __forceinline__ void fold(const LeafDev& L, uint64_t c_min, uint64_t c_max, uint64_t& mn, uint64_t& mx) {
  if (c_min != kNone && (mn == kNone || cmp_items(L, c_min, mn) < 0)) mn = c_min;
  if (c_max != kNone && (mx == kNone || cmp_items(L, c_max, mx) > 0)) mx = c_max;
}

// 1. per (row, leaf): entries, non-null values, PLAIN value bytes (Boolean: bits); a required column's first null
__global__ void __launch_bounds__(256) k_plan(const LeafDev* leaves, uint64_t rb, uint64_t n, uint32_t* ent, uint32_t* nn,
                                              uint32_t* vb, unsigned long long* req_null) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const LeafDev L = leaves[blockIdx.y];
  const uint64_t r = rb + i, at = (uint64_t)blockIdx.y * (n + 1) + i;
  uint64_t it0 = r, it1 = r + 1;
  uint32_t e = 1;
  if (L.is_list) {
    const bool present = bit(L.lvalid, r);
    if (!present && L.required) atomicMin(req_null + blockIdx.y, (unsigned long long)r);
    it0 = present ? (uint64_t)L.loffs[r] : 0; it1 = present ? (uint64_t)L.loffs[r + 1] : 0;
    e = it1 > it0 ? (uint32_t)(it1 - it0) : 1u;
  } else if (L.required && !bit(L.valid, r)) atomicMin(req_null + blockIdx.y, (unsigned long long)r);
  uint32_t c = 0;
  uint64_t b = 0;
  for (uint64_t k = it0; k < it1; k++) {
    if (!bit(L.valid, k)) continue;
    c++;
    b += is_bytes(L) ? 4 + byte_off(L, k + 1) - byte_off(L, k) : L.fixed;
  }
  ent[at] = e; nn[at] = c; vb[at] = (uint32_t)(L.atype == ETL_ARROW_BOOLEAN ? c : b);
}

// 1'. ETL_PQ_PAGE_INDEX, per (row, leaf) of a byte-array leaf: the largest PLAIN row bytes of the leaf, which bound an
// untruncated ColumnIndex maximum
__global__ void __launch_bounds__(256) k_row_max(const LeafDev* leaves, uint64_t n, const uint32_t* vb, unsigned int* vmax) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!is_bytes(leaves[blockIdx.y])) return;
  const unsigned m = __reduce_max_sync(0xffffffffu, i < n ? vb[(uint64_t)blockIdx.y * (n + 1) + i] : 0u);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(vmax + blockIdx.y, m);
}

// 1b. a thread per (leaf, row group; rgb: the n_rg + 1 row-group starts): greedy page cuts.  pages == nullptr: count into n_pages[chunk]
__global__ void k_cut(const LeafDev* leaves, uint32_t n_leaves, uint32_t n_rg, uint64_t rb, const uint64_t* rgb, uint64_t n, const uint64_t* E,
                      const uint64_t* NN, const uint64_t* V, uint32_t* n_pages, const uint64_t* page_base, const uint64_t* leaf_page_base,
                      const uint64_t* lscr_base,
                      Page* pages, int dict) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_leaves * n_rg) return;
  const uint32_t g = t / n_leaves, l = t % n_leaves;
  const LeafDev L = leaves[l];
  const uint64_t* e = E + (uint64_t)l * (n + 1); const uint64_t* nv = NN + (uint64_t)l * (n + 1); const uint64_t* v = V + (uint64_t)l * (n + 1);
  const uint64_t g0 = rgb[g], g1 = rgb[g + 1];             // the row group's local rows (row_group_table)
  const bool boolean = L.atype == ETL_ARROW_BOOLEAN;
  const uint64_t thresh = boolean ? 8 * kPageBytes - 7 : kPageBytes;   // ceil(bits / 8) >= 1 MiB
  const uint32_t slot = dict && !boolean ? 1 : 0;          // the dictionary slot in front of the data pages
  if (pages && slot) {
    Page& P = pages[page_base[t]];
    memset(&P, 0, sizeof P);
    P.leaf = l; P.chunk = t; P.kind = 1; P.row0 = P.row1 = g0; P.e0 = P.e1 = e[g0];
    P.it0 = L.is_list ? (uint64_t)L.loffs[rb + g0] : rb + g0;
    P.it1 = L.is_list ? (uint64_t)L.loffs[rb + g1] : rb + g1;
    P.ubound = min(v[g1] - v[g0], kDictBytes);           // the entries are distinct values of the chunk
    P.min_it = P.max_it = kNone;
  }
  uint32_t np = 0;
  for (uint64_t s = g0; s < g1; np++) {
    uint64_t hi = min(g1 - 1, s + kPageRows - 1);
    if (v[hi + 1] - v[s] >= thresh) {                    // the first row that brings the page to the byte limit
      uint64_t lo = s;
      while (lo < hi) { const uint64_t m = (lo + hi) / 2; if (v[m + 1] - v[s] >= thresh) hi = m; else lo = m + 1; }
    }
    const uint64_t end = hi + 1;
    if (pages) {
      Page& P = pages[page_base[t] + slot + np];
      P.leaf = l; P.chunk = t; P.lp = leaf_page_base[t] + np; P.row0 = s; P.row1 = end; P.e0 = e[s]; P.e1 = e[end];
      P.it0 = L.is_list ? (uint64_t)L.loffs[rb + s] : rb + s;
      P.it1 = L.is_list ? (uint64_t)L.loffs[rb + end] : rb + end;
      P.nn = nv[end] - nv[s];
      P.vbytes = boolean ? (P.nn + 7) / 8 : v[end] - v[s];
      const uint64_t ne = P.e1 - P.e0;
      P.ubound = P.vbytes + (L.max_def ? levels_bound(ne, L.w) : 0) + (L.max_rep ? levels_bound(ne, 1) : 0);
      if (slot) P.ubound += 32;                          // bit-width byte + index runs <= PLAIN values + 20 (indices_bound)
      // level scratch: 8-aligned per page, two sections (rep | def)
      P.lscr = lscr_base[l] + 2 * ((P.e0 + 7) & ~7ull) + 64ull * P.lp;
      P.usize = P.csize = 0; P.hlen = P.plen = 0; P.min_it = P.max_it = kNone; P.nan = 0; P.kind = 0;
    }
    s = end;
  }
  if (!pages) n_pages[t] = np;
}

// block-wide scans of kEncThreads threads (every thread calls them): inclusive sum, inclusive max
__device__ uint64_t block_sum(uint64_t x, uint64_t* s_warp, uint64_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  uint64_t before = 0, t = 0;
  for (int k = 0; k < (int)(blockDim.x / 32); k++) { if (k < wid) before += s_warp[k]; t += s_warp[k]; }
  __syncthreads();
  *total = t;
  return before + x;
}
__device__ int64_t block_max(int64_t x, int64_t* s_warp, int64_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int d = 1; d < 32; d <<= 1) { const int64_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d && y > x) x = y; }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  int64_t before = -1, t = -1;
  for (int k = 0; k < (int)(blockDim.x / 32); k++) { if (k < wid && s_warp[k] > before) before = s_warp[k]; if (s_warp[k] > t) t = s_warp[k]; }
  __syncthreads();
  *total = t;
  return before > x ? before : x;
}

// the index hybrid of a page by the whole CTA (idx_cls / idx_run_bytes / idx_write_run of parquet_format.cuh, so the
// runs are those of the serial indices_encode): 1. classify the groups of 8 tile by tile and keep the run heads (a
// uniform group whose predecessor is not the same uniform value; a non-uniform group 63k groups after the start of its
// stretch, found by a max scan of the last uniform group); 2. the heads' byte sizes, their scan, and one thread per run
// writes it.  x: the page's nn indices; heads: room for ng + 1; returns the bytes written to out
__device__ uint64_t encode_indices(const uint32_t* x, uint64_t nn, uint32_t w, uint32_t* heads, uint8_t* out, uint64_t* s_warp,
                                   int64_t* s_cls) {
  __shared__ uint64_t s_carry[3];                         // runs so far, last uniform group, class of the tile's last group
  const uint64_t ng = (nn + 7) / 8;
  if (threadIdx.x == 0) { s_carry[0] = 0; s_carry[1] = (uint64_t)-1; s_carry[2] = (uint64_t)-2; }
  __syncthreads();
  for (uint64_t t0 = 0; t0 < ng; t0 += blockDim.x) {
    const uint64_t g = t0 + threadIdx.x;
    const int64_t c = g < ng ? idx_cls(x, nn, g) : -2;
    s_cls[threadIdx.x] = c;
    const int64_t prev_tile_cls = (int64_t)s_carry[2], last_u = (int64_t)s_carry[1];
    __syncthreads();
    const int64_t prev = threadIdx.x ? s_cls[threadIdx.x - 1] : prev_tile_cls;
    int64_t tmax;
    int64_t u = block_max(c >= 0 ? (int64_t)g : -1, (int64_t*)s_warp, &tmax);
    if (last_u > u) u = last_u;
    const bool head = g < ng && (c >= 0 ? (g == 0 || prev != c) : (g - (uint64_t)(u + 1)) % 63 == 0);
    uint64_t cnt;
    const uint64_t incl = block_sum(head, s_warp, &cnt);
    const uint64_t base = s_carry[0];
    if (head) heads[base + incl - 1] = (uint32_t)g;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_carry[0] = base + cnt;
      if (tmax > last_u) s_carry[1] = (uint64_t)tmax;
      const uint64_t last = min((uint64_t)blockDim.x, ng - t0) - 1;
      s_carry[2] = (uint64_t)s_cls[last];
    }
    __syncthreads();
  }
  const uint64_t R = s_carry[0];
  if (threadIdx.x == 0) heads[R] = (uint32_t)ng;
  __syncthreads();
  uint64_t o = 0;
  for (uint64_t r0 = 0; r0 < R; r0 += blockDim.x) {
    const uint64_t r = r0 + threadIdx.x;
    const uint64_t g = r < R ? heads[r] : 0, h = r < R ? heads[r + 1] : 0;
    const uint64_t b = r < R ? idx_run_bytes(x, nn, w, g, h) : 0;
    uint64_t tot;
    const uint64_t incl = block_sum(b, s_warp, &tot);
    if (r < R) idx_write_run(x, nn, w, g, h, out + o + incl - b);
    o += tot;
  }
  return o;
}

// dictionary state handed to k_encode<true> (ETL_PQ_DICTIONARY)
struct DictArgs {
  const DictChunk* chunks;
  const uint32_t* tab;       // the chunks' tables: chunk-relative item of each entry's first occurrence
  const uint32_t* pos;       // per item: its slot
  const uint64_t* first;     // per item: exclusive scan of the first-occurrence flags (the entry ids)
  uint32_t* idx;             // per item: the pages' compacted indices
  uint32_t* heads;           // run heads
};

// 2. a CTA per page: levels, PLAIN values (kDict: the dictionary indices of a dictionary chunk), statistics
constexpr int kEncThreads = 256;
template <bool kDict>
__global__ void __launch_bounds__(kEncThreads) k_encode(const LeafDev* leaves, Page* pages, uint64_t rb, const uint64_t* E,
                                                        uint64_t n, uint8_t* lscr, uint8_t* uslot_base, const uint64_t* uslot,
                                                        uint32_t* bool_scr, DictArgs D) {
  __shared__ uint64_t s_lv, s_warp[kEncThreads / 32], s_min[kEncThreads], s_max[kEncThreads];
  __shared__ unsigned long long s_nan;
  const uint32_t p = blockIdx.x;
  Page& P = pages[p];
  if (kDict && P.kind) return;                          // a dictionary slot: k_dict_page
  const LeafDev L = leaves[P.leaf];
  const bool dict = kDict && D.chunks[P.chunk].dict;
  uint64_t i0 = 0, c0 = 0;                              // the leaf's first item, the chunk's first entry id
  if (dict) {
    i0 = L.is_list ? (uint64_t)L.loffs[rb] : rb;
    c0 = D.first[L.dscr + D.chunks[P.chunk].it0 - i0];
  }
  const uint64_t ne = P.e1 - P.e0;
  uint8_t* rep = lscr + P.lscr;
  uint8_t* def = rep + ((ne + 15) & ~7ull);
  const uint64_t* e = E + (uint64_t)P.leaf * (n + 1);
  // levels of each row's entries
  if (L.max_def) {
    for (uint64_t i = P.row0 + threadIdx.x; i < P.row1; i += blockDim.x) {
      const uint64_t r = rb + i, at = e[i] - P.e0;
      if (!L.is_list) { def[at] = bit(L.valid, r); continue; }
      if (!bit(L.lvalid, r)) { def[at] = 0; rep[at] = 0; continue; }
      const uint64_t a = (uint64_t)L.loffs[r], b = (uint64_t)L.loffs[r + 1];
      if (a == b) { def[at] = (uint8_t)(L.max_def - 2); rep[at] = 0; continue; }
      for (uint64_t k = a; k < b; k++) {
        def[at + k - a] = (uint8_t)(bit(L.valid, k) ? L.max_def : L.max_def - 1);
        rep[at + k - a] = k == a ? 0 : 1;
      }
    }
  }
  __syncthreads();
  uint8_t* out = uslot_base + uslot[p];
  if (threadIdx.x == 0) {
    uint64_t o = 0;
    for (int s = 0; s < 2; s++) {
      const bool is_rep = s == 0;
      if (is_rep ? !L.max_rep : !L.max_def) continue;
      const uint64_t len = levels_encode(is_rep ? rep : def, ne, is_rep ? 1u : L.w, out + o + 4);
      for (int b = 0; b < 4; b++) out[o + b] = (uint8_t)(len >> (8 * b));
      o += 4 + len;
    }
    s_lv = o;
    s_nan = 0;
  }
  __syncthreads();
  uint8_t* val = out + s_lv;
  // values: compact the non-null items of [it0, it1) in order, tile by tile
  uint64_t base = 0;          // values (Boolean / fixed) or bytes (byte arrays) before this tile
  uint64_t mn = kNone, mx = kNone, nan = 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t bw = L.bscr + (P.it0 >> 5) + P.lp;    // Boolean scratch: first word of this page
  for (uint64_t t0 = P.it0; t0 < P.it1; t0 += blockDim.x) {
    const uint64_t it = t0 + threadIdx.x;
    const bool v = it < P.it1 && bit(L.valid, it);
    uint64_t sz = 0, boff = 0, blen = 0;
    if (v && is_bytes(L) && !dict) { boff = byte_off(L, it); blen = byte_off(L, it + 1) - boff; sz = 4 + blen; }
    else if (v) sz = 1;
    // block exclusive scan of sz
    uint64_t x = sz;
    for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    uint64_t before = 0, tile = 0;
    for (int k = 0; k < kEncThreads / 32; k++) { if (k < wid) before += s_warp[k]; tile += s_warp[k]; }
    const uint64_t rank = base + before + x - sz;
    if (v) {
      if (dict) {                                       // the entry id of the item's value
        const DictChunk& K = D.chunks[P.chunk];
        const uint64_t j = L.dscr + it - i0;
        const uint64_t fo = D.tab[K.tab + D.pos[j]];    // chunk-relative first occurrence
        D.idx[L.dscr + P.it0 - i0 + rank] = (uint32_t)(D.first[L.dscr + K.it0 + fo - i0] - c0);
      } else if (L.atype == ETL_ARROW_BOOLEAN) {
        if (bit(L.values, it)) atomicOr(bool_scr + bw + (rank >> 5), 1u << (rank & 31));
      } else if (!is_bytes(L)) {
        for (uint32_t k = 0; k < L.fixed; k++) val[rank * L.fixed + k] = L.values[it * L.fixed + k];
      } else {
        for (int b = 0; b < 4; b++) val[rank + b] = (uint8_t)(blen >> (8 * b));
      }
      if (is_nan(L, it)) nan++;
      else fold(L, it, it, mn, mx);
    }
    if (is_bytes(L) && !dict) {                         // every value of the warp copied by the whole warp
      unsigned todo = __ballot_sync(0xffffffffu, v && blen);
      while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint64_t so = __shfl_sync(0xffffffffu, boff, src), sl = __shfl_sync(0xffffffffu, blen, src);
        const uint64_t dst = __shfl_sync(0xffffffffu, rank, src) + 4;
        for (uint64_t k = lane; k < sl; k += 32) val[dst + k] = L.data[so + k];
      }
    }
    base += tile;
    __syncthreads();
  }
  // statistics: block reduction of the candidates
  s_min[threadIdx.x] = mn; s_max[threadIdx.x] = mx;
  if (nan) atomicAdd(&s_nan, (unsigned long long)nan);
  __syncthreads();
  for (int d = kEncThreads / 2; d > 0; d >>= 1) {
    if ((int)threadIdx.x < d) {
      uint64_t a = s_min[threadIdx.x], b = s_max[threadIdx.x];
      fold(L, s_min[threadIdx.x + d], s_max[threadIdx.x + d], a, b);
      s_min[threadIdx.x] = a; s_max[threadIdx.x] = b;
    }
    __syncthreads();
  }
  if (L.atype == ETL_ARROW_BOOLEAN) {                   // the page's bits, from the word-aligned scratch
    for (uint64_t k = threadIdx.x; k < P.vbytes; k += blockDim.x) val[k] = (uint8_t)(bool_scr[bw + (k >> 2)] >> (8 * (k & 3)));
  }
  if (dict) {                                           // bit width, then the index runs
    const uint64_t mn0 = s_min[0], mx0 = s_max[0];
    const unsigned long long nan0 = s_nan;
    const uint32_t w = D.chunks[P.chunk].width;
    if (threadIdx.x == 0) val[0] = (uint8_t)w;
    const uint64_t len = encode_indices(D.idx + L.dscr + P.it0 - i0, P.nn, w, D.heads + L.hscr + (P.it0 - i0) / 8 + 3 * P.lp,
                                        val + 1, s_warp, (int64_t*)s_min);
    if (threadIdx.x == 0) {
      P.usize = s_lv + 1 + len;
      P.min_it = mn0; P.max_it = mx0; P.nan = nan0;
    }
    return;
  }
  if (threadIdx.x == 0) {
    P.usize = s_lv + P.vbytes;
    P.min_it = s_min[0]; P.max_it = s_max[0]; P.nan = s_nan;
  }
}

// 1c. ETL_PQ_DICTIONARY, a thread per chunk: its items, and its table sized from its non-null values (pow2 >= 2 ×
// min(nn, kDictCap); Boolean chunks none) into tab_n, whose exclusive scan places the tables
__global__ void k_dict_setup(const LeafDev* leaves, uint32_t n_leaves, uint32_t n_chunks, uint64_t rb, const uint64_t* rgb, uint64_t n, const uint64_t* NN,
                             const uint64_t* page_base, DictChunk* D, unsigned long long* tab_n) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_chunks) return;
  if (t == n_chunks) { tab_n[t] = 0; return; }
  const uint32_t g = t / n_leaves, l = t % n_leaves;
  const LeafDev L = leaves[l];
  const uint64_t g0 = rgb[g], g1 = rgb[g + 1];
  DictChunk K;
  memset(&K, 0, sizeof K);
  K.it0 = L.is_list ? (uint64_t)L.loffs[rb + g0] : rb + g0;
  K.it1 = L.is_list ? (uint64_t)L.loffs[rb + g1] : rb + g1;
  K.page = page_base[t];
  uint64_t slots = 0;
  if (L.atype != ETL_ARROW_BOOLEAN) {
    const uint64_t* nv = NN + (uint64_t)l * (n + 1);
    const uint64_t m = min(nv[g1] - nv[g0], kDictCap);
    slots = 1;
    while (slots < 2 * m) slots <<= 1;
  }
  K.mask = (uint32_t)(slots - 1);
  D[t] = K;
  tab_n[t] = slots;
}

__device__ __forceinline__ uint64_t mix64(uint64_t h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
  return h;
}
// hash of bytes [k, len) step 32 of p (a lane's share of a long value, or k = 0 step 1 for a short one)
__device__ __forceinline__ uint64_t hash_bytes(const uint8_t* p, uint64_t len, uint64_t k, uint64_t step) {
  uint64_t h = 0x9e3779b97f4a7c15ull;
  for (; k < len; k += step) h = (h ^ p[k]) * 0x100000001b3ull;
  return h;
}
// the PLAIN bytes of present items a and b are equal (byte arrays of at most kLongBytes, or fixed width)
__device__ bool same_value(const LeafDev& L, uint64_t a, uint64_t b) {
  if (is_bytes(L)) {
    const uint64_t a0 = byte_off(L, a), al = byte_off(L, a + 1) - a0, b0 = byte_off(L, b), bl = byte_off(L, b + 1) - b0;
    if (al != bl) return false;
    for (uint64_t k = 0; k < al; k++) if (L.data[a0 + k] != L.data[b0 + k]) return false;
    return true;
  }
  switch (L.fixed) {
    case 4: return ((const uint32_t*)L.values)[a] == ((const uint32_t*)L.values)[b];
    case 8: return ((const uint64_t*)L.values)[a] == ((const uint64_t*)L.values)[b];
    default: return ((const uint64_t*)L.values)[2 * a] == ((const uint64_t*)L.values)[2 * b] &&
                    ((const uint64_t*)L.values)[2 * a + 1] == ((const uint64_t*)L.values)[2 * b + 1];
  }
}
__device__ __forceinline__ uint64_t plain_size(const LeafDev& L, uint64_t it) {
  return is_bytes(L) ? 4 + byte_off(L, it + 1) - byte_off(L, it) : L.fixed;
}
// the chunk of leaf l that holds item it: the last row group whose first item is <= it (a binary search, since one call
// can have thousands of row groups)
__device__ __forceinline__ uint32_t chunk_of(const DictChunk* D, uint32_t l, uint32_t n_leaves, uint32_t n_rg, uint64_t it) {
  uint32_t lo = 0, hi = n_rg - 1;
  while (lo < hi) { const uint32_t m = (lo + hi + 1) / 2; if (D[(uint64_t)m * n_leaves + l].it0 <= it) lo = m; else hi = m - 1; }
  return lo * n_leaves + l;
}
// a slot claimed for a new entry: its PLAIN size joins the chunk's total; past kDictBytes the chunk falls back
__device__ __forceinline__ void claimed(DictChunk& K, uint64_t sz) {
  if (atomicAdd(&K.bytes, (unsigned long long)sz) + sz > kDictBytes) atomicExch(&K.fallback, 1u);
}

// a thread per chunk: its table's first slot, from the exclusive scan of the table sizes
__global__ void k_dict_place(uint32_t n_chunks, const unsigned long long* tab_off, DictChunk* D) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n_chunks) D[c].tab = tab_off[c];
}

// 1d. ETL_PQ_DICTIONARY, one leaf, grid-stride over its items (warp-uniform): each non-null item of a chunk that has
// not fallen back goes into the chunk's open-addressing table (linear probing).  A slot keeps the smallest
// chunk-relative item of its value (atomicMin), so after the pass an item is a first occurrence iff it is its slot's
// value, whatever the order of the inserts.  Byte arrays longer than kLongBytes are hashed and compared by the warp.
__global__ void __launch_bounds__(kInsThreads) k_dict_insert(const LeafDev* leaves, uint32_t l, uint32_t n_leaves, uint32_t n_rg,
                                                             uint64_t rb, DictChunk* D, uint32_t* tab, uint32_t* pos) {
  const LeafDev L = leaves[l];
  const uint64_t i0 = L.is_list ? (uint64_t)L.loffs[rb] : rb, i1 = D[(n_rg - 1) * n_leaves + l].it1;
  const int lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = i0 + (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < i1; base += stride) {
    const uint64_t it = base + lane;
    bool v = it < i1 && bit(L.valid, it);
    uint32_t c = 0;
    if (v) {
      c = chunk_of(D, l, n_leaves, n_rg, it);
      v = !*(volatile uint32_t*)&D[c].fallback;          // inserts into a marked chunk stop
    }
    uint64_t len = 0;
    if (v && is_bytes(L)) len = byte_off(L, it + 1) - byte_off(L, it);
    const bool lng = v && len > kLongBytes;
    uint64_t h = 0;
    if (v && !lng) h = is_bytes(L) ? hash_bytes(L.data + byte_off(L, it), len, 0, 1) ^ len
                                   : mix64(L.fixed == 16 ? ((const uint64_t*)L.values)[2 * it] ^ mix64(((const uint64_t*)L.values)[2 * it + 1])
                                                         : L.fixed == 8 ? ((const uint64_t*)L.values)[it] : ((const uint32_t*)L.values)[it]);
    if (v && !lng) {
      DictChunk& K = D[c];
      const uint32_t rel = (uint32_t)(it - K.it0);
      uint32_t* T = tab + K.tab;
      uint32_t s = (uint32_t)h & K.mask;
      for (uint64_t probe = 0;; probe++, s = (s + 1) & K.mask) {
        if (probe > K.mask) { atomicExch(&K.fallback, 1u); break; }   // full: more than kDictCap entries
        uint32_t cur = *(volatile uint32_t*)&T[s];
        if (cur == kEmpty) {
          cur = atomicCAS(&T[s], kEmpty, rel);
          if (cur == kEmpty) { pos[L.dscr + it - i0] = s; claimed(K, plain_size(L, it)); break; }
        }
        if (same_value(L, K.it0 + cur, it)) { atomicMin(&T[s], rel); pos[L.dscr + it - i0] = s; break; }
      }
    }
    unsigned todo = __ballot_sync(0xffffffffu, lng);
    while (todo) {                                       // one long value at a time, by the whole warp
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint64_t sit = __shfl_sync(0xffffffffu, it, src), slen = __shfl_sync(0xffffffffu, len, src);
      const uint32_t sc = __shfl_sync(0xffffffffu, c, src);
      const uint8_t* sp = L.data + byte_off(L, sit);
      uint64_t hh = mix64(hash_bytes(sp, slen, lane, 32) + lane);
      for (int d = 16; d > 0; d >>= 1) hh ^= __shfl_xor_sync(0xffffffffu, hh, d);
      DictChunk& K = D[sc];
      const uint32_t rel = (uint32_t)(sit - K.it0);
      uint32_t* T = tab + K.tab;
      uint32_t s = (uint32_t)(hh ^ slen) & K.mask;
      for (uint64_t probe = 0;; probe++, s = (s + 1) & K.mask) {
        if (probe > K.mask) { if (lane == 0) atomicExch(&K.fallback, 1u); break; }
        uint32_t cur = 0;
        int won = 0;
        if (lane == 0) {
          cur = *(volatile uint32_t*)&T[s];
          if (cur == kEmpty) { cur = atomicCAS(&T[s], kEmpty, rel); won = cur == kEmpty; }
        }
        cur = __shfl_sync(0xffffffffu, cur, 0);
        if (__shfl_sync(0xffffffffu, won, 0)) {
          if (lane == 0) { pos[L.dscr + sit - i0] = s; claimed(K, 4 + slen); }
          break;
        }
        const uint64_t o = K.it0 + cur, o0 = byte_off(L, o);   // a slot lost to another insert holds its claimant
        bool eq = byte_off(L, o + 1) - o0 == slen;
        if (eq) {
          bool mine = true;
          for (uint64_t k = lane; k < slen; k += 32) if (L.data[o0 + k] != sp[k]) { mine = false; break; }
          eq = __all_sync(0xffffffffu, mine);
        }
        if (eq) {
          if (lane == 0) { atomicMin(&T[s], rel); pos[L.dscr + sit - i0] = s; }
          break;
        }
      }
    }
  }
}

// 1e. ETL_PQ_DICTIONARY, one leaf, a thread per item bound: first-occurrence flags (and, byte arrays, entry sizes) of
// the items of chunks that have not fallen back, 0 elsewhere; their scans give entry ids and PLAIN offsets
__global__ void __launch_bounds__(256) k_dict_mark(const LeafDev* leaves, uint32_t l, uint32_t n_leaves, uint32_t n_rg, uint64_t rb,
                                                   uint64_t bound, const DictChunk* D, const uint32_t* tab, const uint32_t* pos,
                                                   uint32_t* flag, uint32_t* esize) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= bound) return;
  const LeafDev L = leaves[l];
  const uint64_t i0 = L.is_list ? (uint64_t)L.loffs[rb] : rb, it = i0 + j;
  uint32_t f = 0, sz = 0;
  if (it < D[(n_rg - 1) * n_leaves + l].it1 && bit(L.valid, it)) {
    const DictChunk& K = D[chunk_of(D, l, n_leaves, n_rg, it)];
    if (!K.fallback && tab[K.tab + pos[L.dscr + j]] == (uint32_t)(it - K.it0)) { f = 1; sz = (uint32_t)plain_size(L, it); }
  }
  flag[L.dscr + j] = f;
  if (esize) esize[L.dscr + j] = sz;
}

// 1f. ETL_PQ_DICTIONARY, a thread per chunk: entries, PLAIN size, decision, bit width; the dictionary slot's payload size
__global__ void k_dict_finish(const LeafDev* leaves, uint32_t n_leaves, uint32_t n_chunks, uint64_t rb, const uint64_t* first,
                              const uint64_t* esum, DictChunk* D, Page* pages) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const LeafDev L = leaves[c % n_leaves];
  DictChunk& K = D[c];
  if (L.atype == ETL_ARROW_BOOLEAN) return;
  const uint64_t i0 = L.is_list ? (uint64_t)L.loffs[rb] : rb, a = L.dscr + K.it0 - i0, b = L.dscr + K.it1 - i0;
  K.entries = K.fallback ? 0 : first[b] - first[a];
  K.dict = K.entries > 0;                                 // no fallback: every entry is in, and their total <= kDictBytes
  uint32_t w = 1;
  while (K.entries > 1 && (K.entries - 1) >> w) w++;
  K.width = w;
  if (K.dict) pages[K.page].usize = is_bytes(L) ? esum[b] - esum[a] : K.entries * L.fixed;
}

// 1g. ETL_PQ_DICTIONARY, one leaf, a thread per item bound: each first occurrence of a dictionary chunk writes its
// entry, PLAIN, at its offset in the chunk's dictionary slot (byte arrays: the bytes copied by the whole warp)
__global__ void __launch_bounds__(256) k_dict_page(const LeafDev* leaves, uint32_t l, uint32_t n_leaves, uint32_t n_rg, uint64_t rb,
                                                   uint64_t bound, const DictChunk* D, const uint64_t* first, const uint64_t* esum,
                                                   uint8_t* uslot_base, const uint64_t* uslot) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const LeafDev L = leaves[l];
  const uint64_t i0 = L.is_list ? (uint64_t)L.loffs[rb] : rb, it = i0 + j;
  const int lane = threadIdx.x & 31;
  bool v = j < bound && first[L.dscr + j + 1] != first[L.dscr + j];   // a first occurrence (only of non-fallback chunks)
  uint64_t dst = 0, boff = 0, blen = 0;
  if (v) {
    const DictChunk& K = D[chunk_of(D, l, n_leaves, n_rg, it)];
    v = K.dict;
    const uint64_t a = L.dscr + K.it0 - i0;
    uint8_t* out = uslot_base + uslot[K.page];
    if (v && is_bytes(L)) {
      dst = uslot[K.page] + esum[L.dscr + j] - esum[a];
      boff = byte_off(L, it); blen = byte_off(L, it + 1) - boff;
      for (int b = 0; b < 4; b++) out[dst - uslot[K.page] + b] = (uint8_t)(blen >> (8 * b));
      dst += 4;
    } else if (v) {
      const uint64_t o = (first[L.dscr + j] - first[a]) * L.fixed;
      for (uint32_t k = 0; k < L.fixed; k++) out[o + k] = L.values[it * L.fixed + k];
    }
  }
  if (!is_bytes(L)) return;
  unsigned todo = __ballot_sync(0xffffffffu, v && blen);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const uint64_t so = __shfl_sync(0xffffffffu, boff, src), sl = __shfl_sync(0xffffffffu, blen, src), d = __shfl_sync(0xffffffffu, dst, src);
    for (uint64_t k = lane; k < sl; k += 32) uslot_base[d + k] = L.data[so + k];
  }
}

// 3. a CTA per fragment slot of every page (fbase: exclusive scan of the slots per page); one thread compresses, with the
// hash table in shared memory: the match finder is a chain of dependent table lookups, so their latency is the cost
__global__ void __launch_bounds__(32) k_snappy(const Page* pages, uint32_t n_pages, const uint64_t* fbase, const uint8_t* uslot_base,
                                               const uint64_t* uslot, uint8_t* cslot_base, const uint64_t* cslot, uint32_t* fsize) {
  __shared__ uint16_t table[1u << kSnappyHashBits];
  const uint64_t f = blockIdx.x;
  if (threadIdx.x) return;
  uint32_t lo = 0, hi = n_pages - 1;                      // the page: last fbase <= f
  while (lo < hi) { const uint32_t m = (lo + hi + 1) / 2; if (fbase[m] <= f) lo = m; else hi = m - 1; }
  const Page& P = pages[lo];
  const uint64_t k = f - fbase[lo], off = k * kFragment;
  if (off >= P.usize) { fsize[f] = 0; return; }
  const uint32_t len = (uint32_t)(P.usize - off < kFragment ? P.usize - off : kFragment);
  fsize[f] = snappy_fragment(uslot_base + uslot[lo] + off, len, cslot_base + cslot[lo] + 8 + k * snappy_bound(kFragment), table);
}

// 3'. ETL_PQ_ZSTD: a CTA per fragment slot, as k_snappy; one thread writes the fragment's block (a page of no bytes
// gets one empty block), the work space in shared memory.  Its literals and sequences go to scratch placed by the
// fragment's bytes in the payload slots: literal byte i of payload position u at lit[u], the sequences of fragment f
// from seq[u0 / 4 + f] (u0 its first position), so no two fragments overlap.
__global__ void __launch_bounds__(32) k_zstd(const Page* pages, uint32_t n_pages, const uint64_t* fbase, const uint8_t* uslot_base,
                                             const uint64_t* uslot, uint8_t* cslot_base, const uint64_t* cslot, uint32_t* fsize,
                                             uint8_t* lit, uint64_t* seq) {
  __shared__ etl_zstd::Work W;
  const uint64_t f = blockIdx.x;
  if (threadIdx.x) return;
  uint32_t lo = 0, hi = n_pages - 1;                      // the page: last fbase <= f
  while (lo < hi) { const uint32_t m = (lo + hi + 1) / 2; if (fbase[m] <= f) lo = m; else hi = m - 1; }
  const Page& P = pages[lo];
  const uint64_t k = f - fbase[lo], off = k * kFragment;
  if (off >= P.usize && off) { fsize[f] = 0; return; }
  const uint32_t len = (uint32_t)(P.usize - off < kFragment ? P.usize - off : kFragment);
  const uint64_t u = uslot[lo] + off;
  fsize[f] = etl_zstd::zstd_block(uslot_base + u, len, off + len >= P.usize, cslot_base + cslot[lo] + 8 + k * etl_zstd::zstd_bound(kFragment),
                                  W, lit + u, seq + u / 4 + f);
}

// the compressed bound of a fragment of n bytes (comp: the codec, ETL_PQ_SNAPPY or ETL_PQ_ZSTD): at most 32 + 7n / 6
__host__ __device__ inline uint32_t frag_bound(uint32_t comp, uint32_t n) {
  return comp == ETL_PQ_ZSTD ? etl_zstd::zstd_bound(n) : snappy_bound(n);
}
// the stride of the fragments in a page's compressed slot: every fragment but the last is a whole kFragment
__host__ __device__ inline uint32_t frag_slot(uint32_t comp) { return frag_bound(comp, kFragment); }

// a thread per page + 1: what the slot scans add up (0 payload bound, 1 compressed slot, 2 fragment slots); entry
// n_pages is 0, so that the exclusive scan leaves the total there.  The compressed slot (after k_encode) is sized by
// the page's payload: 8 B, whole fragments at the stride, then the bound of its last fragment, so a page of a few
// bytes takes a few dozen, not a whole 64 KiB fragment's bound
__global__ void k_fill(const Page* pages, uint32_t n_pages, int which, uint32_t comp, uint64_t* dst) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > n_pages) return;
  if (p == n_pages) { dst[p] = 0; return; }
  const Page& P = pages[p];
  if (which == 1) {
    const uint64_t nu = P.usize ? (P.usize + kFragment - 1) / kFragment : 1;
    dst[p] = 8 + (nu - 1) * frag_slot(comp) + frag_bound(comp, (uint32_t)(P.usize - (nu - 1) * kFragment));
    return;
  }
  const uint64_t nf = P.ubound ? (P.ubound + kFragment - 1) / kFragment : 1;
  dst[p] = which == 0 ? P.ubound : nf;
}

// a thread per page: compressed size, preamble, header, file bytes of the page (comp: the codec; D: ETL_PQ_DICTIONARY;
// the dictionary slot of a chunk that is not dictionary-encoded has no bytes)
__global__ void k_page(Page* pages, uint32_t n_pages, uint32_t comp, const uint64_t* fbase, const uint32_t* fsize, uint64_t* fbytes,
                       const DictChunk* D) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pages) return;
  Page& P = pages[p];
  const bool dict = D && D[P.chunk].dict;
  if (P.kind && !dict) { P.hlen = P.plen = 0; P.csize = 0; fbytes[p] = 0; return; }
  if (comp != ETL_PQ_UNCOMPRESSED) {
    P.plen = comp == ETL_PQ_ZSTD ? etl_zstd::frame_header((uint32_t)P.usize, P.pre) : varint(P.usize, P.pre);
    uint64_t c = P.plen;
    for (uint64_t f = fbase[p]; f < fbase[p + 1]; f++) c += fsize[f];
    P.csize = c;
  } else P.csize = P.usize;
  if (P.kind) P.hlen = dict_page_header(P.hdr, (uint32_t)P.usize, (uint32_t)P.csize, (uint32_t)D[P.chunk].entries);
  else P.hlen = page_header(P.hdr, (uint32_t)P.usize, (uint32_t)P.csize, (uint32_t)(P.e1 - P.e0), dict ? ENC_RLE_DICTIONARY : ENC_PLAIN);
  fbytes[p] = P.hlen + P.csize;
}

// a CTA per page: header, preamble and payload (or its fragments) at the page's place in its file (base: the files'
// places in the output; rgf: the file of each row group)
__global__ void __launch_bounds__(256) k_gather(const Page* pages, uint32_t comp, const uint64_t* foff, const uint8_t* uslot_base,
                                                const uint64_t* uslot, const uint8_t* cslot_base, const uint64_t* cslot,
                                                const uint64_t* fbase, const uint32_t* fsize, uint32_t n_leaves, const uint32_t* rgf,
                                                const FileRec* files, const uint64_t* base, uint8_t* out) {
  const uint32_t p = blockIdx.x;
  const Page& P = pages[p];
  if (!P.hlen) return;                                   // a dictionary slot without a dictionary has no bytes (k_zstd
  const uint32_t f = rgf[P.chunk / n_leaves];            // still wrote an empty block for it)
  uint8_t* dst = out + base[f] + 4 + foff[p] - foff[files[f].page0];
  for (uint32_t k = threadIdx.x; k < P.hlen; k += blockDim.x) dst[k] = P.hdr[k];
  dst += P.hlen;
  if (comp == ETL_PQ_UNCOMPRESSED) {
    const uint8_t* src = uslot_base + uslot[p];
    for (uint64_t k = threadIdx.x; k < P.usize; k += blockDim.x) dst[k] = src[k];
    return;
  }
  for (uint32_t k = threadIdx.x; k < P.plen; k += blockDim.x) dst[k] = P.pre[k];
  dst += P.plen;
  for (uint64_t f = fbase[p]; f < fbase[p + 1]; f++) {
    const uint8_t* src = cslot_base + cslot[p] + 8 + (f - fbase[p]) * frag_slot(comp);
    for (uint32_t k = threadIdx.x; k < fsize[f]; k += blockDim.x) dst[k] = src[k];
    dst += fsize[f];
  }
}

// PLAIN statistic bytes of item it (a zero float minimum as −0.0, maximum as +0.0); false when longer than kStatMax
__device__ bool stat_bytes(const LeafDev& L, uint64_t it, bool is_max, uint8_t* out, uint32_t* len) {
  if (is_bytes(L)) {
    const uint64_t a = byte_off(L, it), l = byte_off(L, it + 1) - a;
    if (l > kStatMax) return false;
    for (uint64_t k = 0; k < l; k++) out[k] = L.data[a + k];
    *len = (uint32_t)l;
    return true;
  }
  if (L.atype == ETL_ARROW_BOOLEAN) { out[0] = bit(L.values, it); *len = 1; return true; }
  const uint32_t w = L.fixed;
  for (uint32_t k = 0; k < w; k++) out[k] = L.values[it * w + k];
  if (is_float(L)) {
    const bool zero = w == 4 ? ((const float*)L.values)[it] == 0.0f : ((const double*)L.values)[it] == 0.0;
    if (zero) out[w - 1] = is_max ? 0x00 : 0x80;        // the sign bit is the top bit of the last byte
  }
  *len = w;
  return true;
}
__device__ void write_stats(const LeafDev& L, uint64_t mn, uint64_t mx, ChunkOut& C) {
  C.has = 0; C.min_len = C.max_len = 0;
  if (mn == kNone) return;
  if (stat_bytes(L, mn, false, C.min, &C.min_len) && stat_bytes(L, mx, true, C.max, &C.max_len)) C.has = 1;
  else C.min_len = C.max_len = 0;
}

// 4. a thread per chunk (row-group major): sizes, counts, statistics of its pages; its offsets relative to its file (the
// bloom filter's: the file's filters follow its pages, B nullable)
__global__ void k_chunk(const LeafDev* leaves, const Page* pages, const uint64_t* page_base, uint32_t n_chunks, uint32_t n_leaves,
                        const uint64_t* foff, const uint32_t* rgf, const FileRec* files, const BloomChunk* B, uint32_t pidx,
                        ChunkOut* out, const DictChunk* D) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const Page& P0 = pages[page_base[c]];
  const LeafDev L = leaves[P0.leaf];
  const FileRec& F = files[rgf[c / n_leaves]];
  const uint64_t f0 = foff[F.page0];                    // the file's first page
  ChunkOut C{};
  C.offset = 4 + foff[page_base[c]] - f0;
  const uint64_t p0 = page_base[c] + P0.kind;          // the first data page
  C.data_offset = 4 + foff[p0] - f0; C.data_pages = page_base[c + 1] - p0;
  C.dict = D ? D[c].dict : 0;
  C.page_index = pidx;
  if (B && B[c].bytes) {
    C.bloom_offset = 4 + (foff[F.page1] - f0) + B[c].off - F.bloom0;
    C.bloom_len = B[c].hlen + B[c].bytes;
  }
  uint64_t mn = kNone, mx = kNone;
  for (uint64_t p = page_base[c]; p < page_base[c + 1]; p++) {
    const Page& P = pages[p];
    C.num_values += P.e1 - P.e0; C.null_count += (P.e1 - P.e0) - P.nn; C.nan_count += P.nan;
    C.usize += P.hlen + P.usize; C.csize += P.hlen + P.csize;
    fold(L, P.min_it, P.max_it, mn, mx);
  }
  write_stats(L, mn, mx, C);
  out[c] = C;
  // the candidates themselves, for the file-level fold
  reinterpret_cast<uint64_t*>(out + n_chunks)[2 * c] = mn;
  reinterpret_cast<uint64_t*>(out + n_chunks)[2 * c + 1] = mx;
}
// a thread per (file, leaf): the file's statistics of the leaf over its chunks, into out[file * n_leaves + leaf]
__global__ void k_leaf(const LeafDev* leaves, uint32_t n_leaves, uint64_t n_files, uint32_t n_chunks, const FileRec* files,
                       ChunkOut* chunks, ChunkOut* out) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_files * n_leaves) return;
  const uint32_t l = (uint32_t)(t % n_leaves);
  const FileRec& F = files[t / n_leaves];
  const LeafDev L = leaves[l];
  const uint64_t* cand = reinterpret_cast<const uint64_t*>(chunks + n_chunks);
  ChunkOut C{};
  uint64_t mn = kNone, mx = kNone;
  for (uint64_t g = F.rg0; g < F.rg1; g++) {
    const ChunkOut& K = chunks[g * n_leaves + l];
    C.num_values += K.num_values; C.null_count += K.null_count; C.nan_count += K.nan_count;
    C.usize += K.usize; C.csize += K.csize;
    fold(L, cand[2 * (g * n_leaves + l)], cand[2 * (g * n_leaves + l) + 1], mn, mx);
  }
  write_stats(L, mn, mx, C);
  out[t] = C;
}

// ETL_PQ_PAGE_INDEX: the ColumnIndex bound of present, non-NaN item it: its statistic bytes, a byte array's truncated
// to 64 bytes (index_min / index_max); out == nullptr counts.  Returns its length.
__device__ uint64_t index_bound(const LeafDev& L, uint64_t it, bool is_max, uint8_t* out) {
  if (is_bytes(L)) {
    const uint64_t a = byte_off(L, it), len = byte_off(L, it + 1) - a;
    const bool utf8 = L.atype == ETL_ARROW_UTF8;
    return is_max ? index_max(L.data + a, len, utf8, out) : index_min(L.data + a, len, utf8, out);
  }
  uint8_t b[16];
  uint32_t len = 0;
  stat_bytes(L, it, is_max, b, &len);
  if (out) for (uint32_t k = 0; k < len; k++) out[k] = b[k];
  return len;
}
__device__ __forceinline__ uint64_t warp_excl(uint64_t x, uint64_t* total) {
  const int lane = threadIdx.x & 31;
  uint64_t s = x;
  for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += y; }
  *total = __shfl_sync(0xffffffffu, s, 31);
  return s - x;
}
// ETL_PQ_PAGE_INDEX: one record per chunk, from k_index<false> to k_index<true>
struct IndexChunk {
  uint64_t s_min, s_max, s_nc, s_loc;   // bytes of the min_values / max_values / null_counts entries, of the PageLocations
  uint32_t order, has_ci;               // BoundaryOrder; a ColumnIndex (no page with values that are all NaN)
};
constexpr uint32_t kIdxWarps = 4;
// 4b. ETL_PQ_PAGE_INDEX, a warp per chunk (row-group major), lanes over its data pages (the dictionary page is not
// listed).  kWrite false: each page's entry sizes, the boundary order (each non-null page against the previous one, on
// the untruncated bounds) and the lengths of the chunk's ColumnIndex (lens[c], 0 when it has none) and OffsetIndex
// (lens[c1 + c]), where the chunk's file has chunks [c0, c1): a file's ColumnIndexes, then its OffsetIndexes, files in
// order; lens[2 n_chunks] = 0, so that their exclusive scan places every file's index as one run (k_index_place).
// kWrite true: both structures at the offsets k_index_place put into the chunk's record, in its file at base.
template <bool kWrite>
__global__ void __maxnreg__(96) k_index(const LeafDev* leaves, const Page* pages, const uint64_t* page_base,
                                                         uint32_t n_chunks, uint32_t n_leaves, const uint64_t* rgb, const uint32_t* rgf,
                                                         const FileRec* files, const uint64_t* base, const uint64_t* foff,
                                                         IndexChunk* X, unsigned long long* lens, uint8_t* out_file, ChunkOut* out) {
  const uint32_t c = blockIdx.x * kIdxWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= n_chunks) {
    if (!kWrite && c == n_chunks && lane == 0) lens[2 * n_chunks] = 0;
    return;
  }
  const uint64_t pb = page_base[c];
  const LeafDev L = leaves[pages[pb].leaf];
  const uint64_t p0 = pb + pages[pb].kind, k = page_base[c + 1] - p0;
  const uint32_t f = rgf[c / n_leaves];
  const uint64_t g0 = rgb[c / n_leaves], f0 = foff[files[f].page0];
  const uint32_t lk = list_field(nullptr, TT_BINARY, (uint32_t)k);   // a list field's header
  IndexChunk I{};
  uint8_t* ci = nullptr;
  uint8_t* oi = nullptr;
  uint64_t o_min = 0, o_max = 0, o_nc = 0;                // kWrite: where the sections' entries start
  if (kWrite) {
    I = X[c];
    const ChunkOut& C = out[c];
    ci = out_file + base[f] + C.ci_offset;
    oi = out_file + base[f] + C.oi_offset;
    o_min = lk + k + lk; o_max = o_min + I.s_min + lk; o_nc = o_max + I.s_max + 2 + lk;
    if (lane == 0) {
      if (I.has_ci) {
        list_field(ci, TT_TRUE, (uint32_t)k);             // null_pages: list<bool>, one byte per element
        list_field(ci + lk + k, TT_BINARY, (uint32_t)k);  // min_values
        list_field(ci + o_min + I.s_min, TT_BINARY, (uint32_t)k);   // max_values
        ci[o_max + I.s_max] = (1u << 4) | TT_I32;         // boundary_order
        ci[o_max + I.s_max + 1] = (uint8_t)zigzag(I.order);
        list_field(ci + o_max + I.s_max + 2, TT_I64, (uint32_t)k);  // null_counts
        ci[o_nc + I.s_nc] = 0;
      }
      list_field(oi, TT_STRUCT, (uint32_t)k);             // page_locations
      oi[lk + I.s_loc] = 0;
    }
  }
  bool asc = true, desc = true, nan_only = false;
  uint64_t s_min = 0, s_max = 0, s_nc = 0, s_loc = 0, prev = kNone;
  for (uint64_t j0 = 0; j0 < k; j0 += 32) {
    const uint64_t j = j0 + lane, p = p0 + (j < k ? j : 0);
    const bool in = j < k;
    const Page& P = pages[p];
    const bool nonnull = in && P.nn;
    const bool bounded = nonnull && P.min_it != kNone;
    if (nonnull && !bounded) nan_only = true;
    // the previous non-null page: a lane below in this tile, or the last one before it
    const unsigned m = __ballot_sync(0xffffffffu, bounded), below = m & ((1u << lane) - 1u);
    const uint64_t q = below ? p0 + j0 + (31 - __clz(below)) : prev;
    if (bounded && q != kNone) {
      const Page& Q = pages[q];
      const int a = cmp_items(L, P.min_it, Q.min_it), b = cmp_items(L, P.max_it, Q.max_it);
      if (a < 0 || b < 0) asc = false;
      if (a > 0 || b > 0) desc = false;
    }
    if (m) prev = p0 + j0 + (31 - __clz(m));
    const uint64_t mnl = bounded ? index_bound(L, P.min_it, false, nullptr) : 0;
    const uint64_t mxl = bounded ? index_bound(L, P.max_it, true, nullptr) : 0;
    const uint64_t nc = in ? (P.e1 - P.e0) - P.nn : 0;
    const uint64_t off = 4 + foff[p] - f0, first = P.row0 - g0;
    const uint32_t fsz = (uint32_t)(foff[p + 1] - foff[p]);
    uint64_t t_min, t_max, t_nc, t_loc;
    const uint64_t x_min = warp_excl(in ? varint(mnl, nullptr) + mnl : 0, &t_min);
    const uint64_t x_max = warp_excl(in ? varint(mxl, nullptr) + mxl : 0, &t_max);
    const uint64_t x_nc = warp_excl(in ? varint(zigzag((int64_t)nc), nullptr) : 0, &t_nc);
    const uint64_t x_loc = warp_excl(in ? page_location(nullptr, off, fsz, first) : 0, &t_loc);
    if (kWrite && in) {
      if (I.has_ci) {
        ci[lk + j] = nonnull ? TT_FALSE : TT_TRUE;         // null_pages[j]: 0x01 true, 0x02 false
        uint8_t* d = ci + o_min + s_min + x_min;
        d += varint(mnl, d);
        if (bounded) index_bound(L, P.min_it, false, d);
        d = ci + o_max + s_max + x_max;
        d += varint(mxl, d);
        if (bounded) index_bound(L, P.max_it, true, d);
        varint(zigzag((int64_t)nc), ci + o_nc + s_nc + x_nc);
      }
      page_location(oi + lk + s_loc + x_loc, off, fsz, first);
    }
    s_min += t_min; s_max += t_max; s_nc += t_nc; s_loc += t_loc;
  }
  if (kWrite) return;
  asc = __all_sync(0xffffffffu, asc); desc = __all_sync(0xffffffffu, desc); nan_only = __any_sync(0xffffffffu, nan_only);
  if (lane == 0) {
    I.s_min = s_min; I.s_max = s_max; I.s_nc = s_nc; I.s_loc = s_loc;
    I.order = asc ? 1 : desc ? 2 : 0;                       // ASCENDING, DESCENDING, UNORDERED
    I.has_ci = !nan_only;
    X[c] = I;
    const FileRec& F = files[f];
    lens[F.rg0 * n_leaves + c] = I.has_ci ? (lk + k) + (lk + s_min) + (lk + s_max) + 2 + (lk + s_nc) + 1 : 0;
    lens[F.rg1 * n_leaves + c] = lk + s_loc + 1;
  }
}
// ETL_PQ_PAGE_INDEX, a thread per chunk, after the scan of k_index<false>'s lengths: the offsets and lengths of the
// chunk's ColumnIndex and OffsetIndex in its file, whose index follows its pages and bloom filters
__global__ void k_index_place(uint32_t n_chunks, uint32_t n_leaves, const uint32_t* rgf, const FileRec* files, const uint64_t* foff,
                              const IndexChunk* X, const unsigned long long* lens, ChunkOut* out) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const FileRec& F = files[rgf[c / n_leaves]];
  const uint64_t c0 = F.rg0 * n_leaves, c1 = F.rg1 * n_leaves;
  const uint64_t at = 4 + foff[F.page1] - foff[F.page0] + (F.bloom1 - F.bloom0) - lens[2 * c0];
  ChunkOut& C = out[c];
  const bool has_ci = X[c].has_ci;
  C.ci_len = has_ci ? (uint32_t)(lens[c0 + c + 1] - lens[c0 + c]) : 0;
  C.ci_offset = has_ci ? at + lens[c0 + c] : 0;
  C.oi_offset = at + lens[c1 + c];
  C.oi_len = (uint32_t)(lens[c1 + c + 1] - lens[c1 + c]);
}

// a thread per chunk: the non-null values of the chunk (NN prefix sums at its row-group bounds), which size its bitset
__global__ void k_chunk_nn(uint32_t n_leaves, uint32_t n_chunks, uint64_t n, const uint64_t* rgb, const uint64_t* NN, unsigned long long* cnn) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const uint64_t* nv = NN + (uint64_t)(c % n_leaves) * (n + 1);
  const uint64_t g0 = rgb[c / n_leaves], g1 = rgb[c / n_leaves + 1];
  cnn[c] = nv[g1] - nv[g0];
}
// XXH64 of present item it's PLAIN bytes (byte arrays without the length prefix, hashed serially by this thread)
__device__ __forceinline__ uint64_t item_hash(const LeafDev& L, uint64_t it) {
  if (is_bytes(L)) { const uint64_t a = byte_off(L, it); return xxh64(L.data + a, byte_off(L, it + 1) - a); }
  switch (L.fixed) {
    case 4: return xxh64_u32(((const uint32_t*)L.values)[it]);
    case 8: return xxh64_u64(((const uint64_t*)L.values)[it]);
    default: return xxh64(L.values + 16 * it, 16);
  }
}
// the first item of row group g of a leaf (g == n_rg: the end of its items)
__device__ __forceinline__ uint64_t group_item(const LeafDev& L, uint64_t rb, const uint64_t* rgb, uint32_t g) {
  const uint64_t r = rb + rgb[g];
  return L.is_list ? (uint64_t)L.loffs[r] : r;
}
// 4c. bloom filters, one filtered leaf, grid-stride over its items: each non-null item's hash sets 8 bits of one block
// of its chunk's bitset (atomicOr into the zeroed scratch; the bits are a set, so any order gives the same bitset)
__global__ void __launch_bounds__(kInsThreads) k_bloom(const LeafDev* leaves, uint32_t l, uint32_t n_leaves, uint32_t n_rg,
                                                       uint64_t rb, const uint64_t* rgb, const BloomChunk* B, uint32_t* words) {
  const LeafDev L = leaves[l];
  const uint64_t i0 = group_item(L, rb, rgb, 0), i1 = group_item(L, rb, rgb, n_rg);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t it = i0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; it < i1; it += stride) {
    if (!bit(L.valid, it)) continue;
    uint32_t g = 0, hi = n_rg - 1;                       // the last row group whose first item is <= it
    while (g < hi) { const uint32_t m = (g + hi + 1) / 2; if (group_item(L, rb, rgb, m) <= it) g = m; else hi = m - 1; }
    const BloomChunk K = B[g * n_leaves + l];
    const uint64_t h = item_hash(L, it);
    uint32_t* w = words + K.word + 8ull * bloom_block(h, K.bytes / 32);
#pragma unroll
    for (int i = 0; i < 8; i++) atomicOr(w + i, bloom_mask(h, i));
  }
}
// 4d. CTAs (chunk, slice): the chunk's header and bitset in its file, behind the file's pages (ETL_PQ_PAGE_INDEX comes
// after), at the offset k_chunk put into its record
__global__ void __launch_bounds__(256) k_bloom_write(const BloomChunk* B, const uint32_t* words, uint32_t n_leaves, const uint32_t* rgf,
                                                     const uint64_t* base, const ChunkOut* chunks, uint8_t* out) {
  const BloomChunk K = B[blockIdx.x];
  if (!K.bytes) return;
  uint8_t* dst = out + base[rgf[blockIdx.x / n_leaves]] + chunks[blockIdx.x].bloom_offset;
  if (blockIdx.y == 0 && threadIdx.x == 0) bloom_header(dst, K.bytes);
  const uint8_t* src = (const uint8_t*)(words + K.word);
  dst += K.hlen;
  for (uint64_t k = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; k < K.bytes; k += (uint64_t)gridDim.y * blockDim.x) dst[k] = src[k];
}

// 5. footers, a warp per file, its lanes over the footer's units (tail_unit of parquet_format.cuh: a ColumnChunk each,
// so a file of many row groups or leaves is written by the whole warp).  The schema prefix (the same for every file) is
// serialised once on the host.  kWrite false: the footer's length and the file's size (4 + pages + filters + index +
// footer + 8) into size[f], whose exclusive scan places the files (size[K] = 0); kWrite true: both magics, the prefix,
// the units at their scanned places, and the footer's length, at the file's place.
struct FooterArgs {
  const LeafMeta* leaves;
  const uint8_t* prefix;
  const uint8_t* created_by;
  uint32_t n_leaves, prefix_len, cb_len, codec;
};
__device__ __forceinline__ ChunkMeta out_meta(const ChunkOut& K) {
  return ChunkMeta{K.offset, K.num_values, K.usize, K.csize, K.null_count, K.data_offset, K.data_pages, K.ci_offset, K.oi_offset,
                   K.bloom_offset, K.ci_len, K.oi_len, K.bloom_len, K.min_len, K.max_len, K.has != 0, K.dict != 0,
                   K.page_index != 0, K.min, K.max};
}
constexpr uint32_t kFootWarps = 4;
template <bool kWrite>
__global__ void __maxnreg__(96) k_footer(FooterArgs A, uint64_t n_files, const uint64_t* rgb, FileRec* files,
                                                           const uint64_t* foff, const unsigned long long* lens,
                                                           const ChunkOut* chunks, uint64_t* size, uint8_t* out) {
  const uint64_t f = (uint64_t)blockIdx.x * kFootWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (f > n_files) return;
  if (f == n_files) { if (!kWrite && lane == 0) size[f] = 0; return; }
  FileRec& F = files[f];
  const ChunkOut* C = chunks + F.rg0 * A.n_leaves;
  auto get = [&](uint64_t c) { return out_meta(C[c]); };
  const uint32_t n_rg = (uint32_t)(F.rg1 - F.rg0);
  const uint64_t n_units = (uint64_t)n_rg * A.n_leaves + 2;
  if (!kWrite) {
    uint64_t t = 0;
    for (uint64_t u = lane; u < n_units; u += 32)
      t += tail_unit(nullptr, u, A.leaves, A.n_leaves, rgb + F.rg0, n_rg, get, A.codec, A.created_by, A.cb_len);
    for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(0xffffffffu, t, d);
    if (lane == 0) {
      F.data = foff[F.page1] - foff[F.page0];
      F.index = lens ? lens[2 * F.rg1 * A.n_leaves] - lens[2 * F.rg0 * A.n_leaves] : 0;
      F.footer = A.prefix_len + t;
      size[f] = 4 + F.data + (F.bloom1 - F.bloom0) + F.index + F.footer + 8;
    }
    return;
  }
  uint8_t* o = out + size[f];                             // the scan: the file's place
  const uint8_t magic[4] = {'P', 'A', 'R', '1'};
  uint8_t* t = o + 4 + F.data + (F.bloom1 - F.bloom0) + F.index;
  for (uint32_t k = lane; k < A.prefix_len; k += 32) t[k] = A.prefix[k];
  uint64_t at = A.prefix_len;
  for (uint64_t u0 = 0; u0 < n_units; u0 += 32) {
    const uint64_t u = u0 + lane;
    const uint64_t n = u < n_units ? tail_unit(nullptr, u, A.leaves, A.n_leaves, rgb + F.rg0, n_rg, get, A.codec, A.created_by, A.cb_len) : 0;
    uint64_t tile;
    const uint64_t x = warp_excl(n, &tile);
    if (u < n_units) tail_unit(t + at + x, u, A.leaves, A.n_leaves, rgb + F.rg0, n_rg, get, A.codec, A.created_by, A.cb_len);
    at += tile;
  }
  if (lane == 0) {
    for (int k = 0; k < 4; k++) o[k] = magic[k];
    uint8_t* e = t + F.footer;
    for (int k = 0; k < 4; k++) e[k] = (uint8_t)(F.footer >> (8 * k));
    for (int k = 0; k < 4; k++) e[4 + k] = magic[k];
  }
}

uint32_t parquet_type(uint32_t at) {
  switch (at) {
    case ETL_ARROW_BOOLEAN: return PT_BOOLEAN;
    case ETL_ARROW_INT32: case ETL_ARROW_DATE32: return PT_INT32;
    case ETL_ARROW_FLOAT32: return PT_FLOAT;
    case ETL_ARROW_FLOAT64: return PT_DOUBLE;
    case ETL_ARROW_UTF8: case ETL_ARROW_LARGE_BINARY: return PT_BYTE_ARRAY;
    case ETL_ARROW_UUID: return PT_FLBA;
    default: return PT_INT64;
  }
}
uint32_t plain_width(uint32_t at) {
  switch (at) {
    case ETL_ARROW_INT32: case ETL_ARROW_DATE32: case ETL_ARROW_FLOAT32: return 4;
    case ETL_ARROW_INT64: case ETL_ARROW_FLOAT64: case ETL_ARROW_TIME64_US: case ETL_ARROW_TIMESTAMP_US: case ETL_ARROW_TIMESTAMPTZ_US: return 8;
    case ETL_ARROW_UUID: return 16;
    default: return 0;
  }
}

}  // namespace

struct etl_parquet_files {
  uint8_t *dev = nullptr, *host = nullptr;
  uint64_t n_files = 0;
  uint32_t n_leaves = 0;
  std::vector<uint64_t> offs;                       // n_files + 1 byte offsets of the files in dev / host
  std::vector<etl_parquet_metrics> metrics;         // file-major, n_leaves per file (none after a required null)
  std::vector<uint8_t> stats;                       // min / max bytes of the metrics
  uint32_t null_column = UINT32_MAX;
  uint64_t null_row = UINT64_MAX;
  ~etl_parquet_files() { if (dev) cudaFree(dev); if (host) cudaFreeHost(host); }
};
struct etl_parquet_file : etl_parquet_files {};     // etl_dec_parquet_write(_bloom): the K = 1 result

namespace {

// the slot of each scan's total (k_fill's `which` is its scan's slot; every dictionary scan shares kTotDict)
enum TotSlot : uint32_t { kTotUslot, kTotCslot, kTotFbase, kTotFoff, kTotDict, kTotIndex, kTotFiles, kTotSlots };
// places regions one after another (from 0 to size a block, then from the block), each 256-aligned as a cudaMalloc of
// its own, with kSlack bytes + its extra behind it: a zero-count region is still a valid, distinct pointer
constexpr uint64_t kAlign = 256, kSlack = 64;
struct Carve {
  uintptr_t base;
  uint64_t at = 0;
  template <class T> void operator()(T*& p, uint64_t count, uint64_t extra = 0) {
    p = reinterpret_cast<T*>(base + at);
    at = (at + sizeof(T) * count + extra + kSlack + kAlign - 1) / kAlign * kAlign;
  }
};
struct Totals {                                     // the plan's results (SYNC 1): per chunk the data pages and
  std::vector<uint32_t> np;                         // (bloom filters) the non-null values; per leaf the level entries |
  std::vector<unsigned long long> cnn, tot, req;    // non-null values | PLAIN bytes, a required column's first null row
  std::vector<unsigned int> vmax;                   // (kNone: none) and (ETL_PQ_PAGE_INDEX) its longest row's PLAIN bytes
};
struct Sizes {                                      // every bound and host table, from the description and the totals
  std::vector<LeafDev> hl;                          // the leaves with their scratch offsets (bscr, dscr, hscr)
  std::vector<uint64_t> page_base, leaf_page_base, pages_of, lscr_base;
  uint64_t P, U, n_frag_bound, C_bound, bool_words, d_items, d_heads, d_slots, d_maxI, bloom_total, bloom_words;
  std::vector<BloomChunk> hb; std::vector<FileRec> hf;
  std::vector<uint8_t> prefix; std::vector<LeafMeta> lm;   // the footers' schema prefix and leaves
  uint64_t meta_bytes, data_bound, index_bound, footer_bound;
};
constexpr char kCreatedBy[] = "etl-b200 parquet writer";
constexpr uint32_t kCreatedByLen = sizeof kCreatedBy - 1;

// One writer call: its stages share this record, which owns the scratch blocks until the call returns and the output
// until collect() hands it over.  Aggregate initialisation zeroes every member it does not name.
struct Call {
  const etl_arrow_batch* a; const etl_parquet_field* fields; const etl_parquet_bloom* bloom;
  uint32_t nL; const uint64_t* ro; uint64_t K; uint32_t codec; int to_host;   // nL: the leaves, one per field
  uint32_t cc; int dict, pidx, snappy, zstd; bool any_bloom;   // describe(); snappy: compressed fragments (Snappy or Zstandard)
  std::vector<LeafDev> hl; std::vector<Leaf> meta;
  std::vector<uint64_t> values, frg, rgb;           // items of each leaf's value column; first row group of each file;
  std::vector<uint32_t> rgf;                        // row-group starts (local rows), then n; each row group's file
  uint64_t row_begin, n; uint32_t n_rg, n_chunks;
  Totals t; Sizes s;                                // plan(), size()
  // the device scratch: regions of two cudaMalloc blocks, laid out by regions(); a region of a feature the call does
  // not use stays null (the kernels test for it)
  LeafDev* d_leaves; Page* d_pages; ChunkOut *d_cout, *d_lout; FileRec* d_files; DictChunk* d_dch; IndexChunk* d_ix; BloomChunk* d_bch;
  uint32_t *d_ent, *d_nn, *d_vb, *d_np, *d_rgf, *d_bool, *d_fsz, *d_tab, *d_dpos, *d_dflag, *d_desz, *d_dhead, *d_bwords;
  uint64_t *d_E, *d_NN, *d_V, *d_rgb, *d_pbase, *d_lpbase, *d_lbase, *d_uslot, *d_cslot, *d_fbase, *d_foff, *d_zseq,
      *d_fplace, *d_dfirst, *d_desum;
  unsigned long long *d_blk, *d_tot, *d_req, *d_cnn, *d_stot, *d_tabn, *d_dblk, *d_ixlen; unsigned int* d_vmax;
  uint8_t *d_lscr, *d_u, *d_c, *d_zlit, *d_meta;
  void* blk[2]; uint8_t *dev, *host;
  cudaStream_t st = cudaStreamPerThread;
  ~Call() { for (void* p : blk) if (p) cudaFree(p); if (dev) cudaFree(dev); if (host) cudaFreeHost(host); }
  bool bloomed(uint32_t l) const { return bloom && bloom[l].fpp > 0.0; }
  // ETL_PQ_DICTIONARY: every chunk of a non-Boolean leaf has a dictionary slot in front of its data pages
  bool has_dict(uint32_t l) const { return dict && hl[l].atype != ETL_ARROW_BOOLEAN; }
  void regions(int b, Carve& r); bool carve(int b);
  int describe(); int plan(); Sizes size() const; int launch(); int collect(etl_parquet_files* Fs);   // the stages
};

// block 0 holds what the plan needs (before SYNC 1), block 1 the rest (sized from the totals)
void Call::regions(int b, Carve& r) {
  if (b == 0) {
    const uint64_t nr1 = (uint64_t)nL * (n + 1);    // per (leaf, row): level entries, non-null values, PLAIN value
    r(d_leaves, nL + 1);                            // bytes, and their prefix sums
    r(d_ent, nr1); r(d_nn, nr1); r(d_vb, nr1); r(d_E, nr1); r(d_NN, nr1); r(d_V, nr1);
    r(d_blk, 3ull * nL * (scan_blocks(n) + 1)); r(d_tot, 3ull * nL);
    r(d_req, nL); r(d_vmax, nL); r(d_np, n_chunks);
    if (any_bloom) r(d_cnn, n_chunks);
    r(d_rgb, n_rg + 1ull); r(d_rgf, n_rg + 1ull);
    return;
  }
  const uint64_t P = s.P, nc = n_chunks;
  r(d_pages, P + 1); r(d_pbase, nc + 1); r(d_lpbase, nc + 1); r(d_lbase, nL + 1ull); r(d_lscr, s.lscr_base[nL], 16);
  r(d_uslot, P + 1); r(d_cslot, P + 1); r(d_fbase, P + 1); r(d_foff, P + 1); r(d_stot, kTotSlots);
  r(d_u, s.U, 16); r(d_bool, s.bool_words, 8);
  if (snappy) { r(d_c, s.C_bound, 16); r(d_fsz, s.n_frag_bound + 1); }
  if (zstd) { r(d_zlit, s.U, 16); r(d_zseq, s.U / 4 + s.n_frag_bound + 1); }   // k_zstd's literals and sequences
  r(d_cout, nc, 16 * nc);                           // + the chunks' (min, max) candidates k_leaf reads at cout + nc
  r(d_lout, K * nL); r(d_files, K); r(d_fplace, K + 1); r(d_meta, s.meta_bytes);
  if (s.d_items && P) {
    r(d_dch, nc); r(d_tabn, nc + 1); r(d_dblk, scan_blocks(s.d_maxI) + 2ull); r(d_tab, s.d_slots); r(d_dhead, s.d_heads);
    r(d_dpos, s.d_items); r(d_dflag, s.d_items); r(d_desz, s.d_items); r(d_dfirst, s.d_items); r(d_desum, s.d_items);
  }
  if (pidx && P) { r(d_ix, nc); r(d_ixlen, 2 * nc + 1); }
  if (s.bloom_total) { r(d_bch, nc); r(d_bwords, s.bloom_words); }
}
// sizes block b, allocates it and places its regions
bool Call::carve(int b) {
  Carve r{0};
  regions(b, r);
  if (cudaMalloc(&blk[b], r.at) != cudaSuccess) { blk[b] = nullptr; return false; }
  r = Carve{(uintptr_t)blk[b]};
  regions(b, r);
  return true;
}

#define CK(call) do { if ((call) != cudaSuccess) return ETL_ERR_CUDA; } while (0)

// Describe: check the arguments, build the leaves, their schema and the row-group table (no CUDA call)
int Call::describe() {
  // a file needs at least one column (an emit of a zero-column table without ETL_ARROW_CDC_COLUMNS has none)
  if (!a || !ro || !nL || !fields || nL != etl_dec_arrow_cols(a)) return ETL_ERR_INVALID_ARG;
  cc = codec & 0xFFu;                               // the compression codec; the flag bits are ETL_PQ_DICTIONARY and
  if ((codec & ~(0xFFu | ETL_PQ_DICTIONARY | ETL_PQ_PAGE_INDEX)) ||   // ETL_PQ_PAGE_INDEX
      (cc != ETL_PQ_UNCOMPRESSED && cc != ETL_PQ_SNAPPY && cc != ETL_PQ_ZSTD))
    return ETL_ERR_INVALID_ARG;
  if (K >= UINT32_MAX) return ETL_ERR_INVALID_ARG;
  for (uint64_t k = 0; k < K; k++) if (ro[k + 1] < ro[k]) return ETL_ERR_INVALID_ARG;
  if (ro[K] > etl_dec_arrow_rows(a)) return ETL_ERR_INVALID_ARG;
  dict = (codec & ETL_PQ_DICTIONARY) != 0; pidx = (codec & ETL_PQ_PAGE_INDEX) != 0;
  snappy = cc != ETL_PQ_UNCOMPRESSED; zstd = cc == ETL_PQ_ZSTD;
  hl.resize(nL); meta.resize(nL); values.resize(nL);
  for (uint32_t c = 0; c < nL; c++) {
    const etl_parquet_field& F = fields[c];
    if (!F.name) return ETL_ERR_INVALID_ARG;
    const size_t nl = strnlen(F.name, 1025);
    if (nl == 0 || nl > 1024) return ETL_ERR_INVALID_ARG;
    etl_arrow_column col;
    if (etl_dec_arrow_column(a, c, 0, &col) != ETL_OK || col.arrow_type == ETL_ARROW_UNSUPPORTED) return ETL_ERR_INVALID_ARG;
    LeafDev& L = hl[c];
    memset(&L, 0, sizeof L);
    L.is_list = col.arrow_type == ETL_ARROW_LIST;
    L.required = F.required != 0;
    values[c] = etl_dec_arrow_rows(a);
    if (L.is_list) {
      etl_arrow_column kid;
      if (etl_dec_arrow_list_child(a, c, 0, &kid, &values[c]) != ETL_OK) return ETL_ERR_INVALID_ARG;
      L.lvalid = col.validity; L.loffs = (const int32_t*)col.offsets;
      col = kid;
    }
    L.atype = col.arrow_type;
    L.max_def = L.is_list ? (L.required ? 2 : 3) : (L.required ? 0 : 1);
    L.max_rep = L.is_list ? 1 : 0;
    L.w = bit_width(L.max_def);
    L.fixed = plain_width(L.atype);
    L.off64 = L.atype == ETL_ARROW_LARGE_BINARY;
    L.valid = col.validity; L.values = (const uint8_t*)col.values; L.offs = col.offsets; L.data = col.data;
    if (bloom) {
      const etl_parquet_bloom& Bf = bloom[c];
      const uint32_t mb = Bf.max_bytes;
      if (!(Bf.fpp >= 0.0 && Bf.fpp < 1.0) || (mb && (mb < kBloomMinBytes || mb > kBloomMaxBytes || (mb & (mb - 1)))) ||
          (Bf.fpp > 0.0 && L.atype == ETL_ARROW_BOOLEAN))
        return ETL_ERR_INVALID_ARG;
    }
    any_bloom |= bloomed(c);
    Leaf& M = meta[c];
    M.name.assign(F.name, nl);
    M.field_id = F.field_id; M.element_field_id = F.element_field_id;
    M.ptype = parquet_type(L.atype);
    M.required = L.required; M.is_list = L.is_list;
    M.converted = CT_NONE; M.logical = 0; M.utc = false;
    switch (L.atype) {
      case ETL_ARROW_UTF8: M.converted = CT_UTF8; M.logical = 1; break;
      case ETL_ARROW_DATE32: M.converted = CT_DATE; M.logical = 6; break;
      case ETL_ARROW_TIME64_US: M.logical = 7; break;
      case ETL_ARROW_TIMESTAMP_US: M.logical = 8; break;
      case ETL_ARROW_TIMESTAMPTZ_US: M.logical = 8; M.utc = true; M.converted = CT_TIMESTAMP_MICROS; break;
      case ETL_ARROW_UUID: M.logical = 14; break;
      default: break;
    }
  }
  // the row-group table: row groups restart in every file; chunk indices are 32-bit, and the page index's length scan
  // runs over 2 × chunks + 1 entries in 32 bits, so at most 2^31 - 1 chunks
  const std::vector<RowGroup> rgt = row_group_table(ro, K, frg);
  if ((uint64_t)rgt.size() * nL >= (1ull << 31)) return ETL_ERR_INVALID_ARG;
  if (!K) return ETL_OK;
  row_begin = ro[0]; n = ro[K] - ro[0];
  n_rg = (uint32_t)rgt.size(); n_chunks = n_rg * nL;
  rgb.assign(n_rg + 1, n); rgf.assign(n_rg + 1, 0);
  for (uint32_t g = 0; g < n_rg; g++) { rgb[g] = rgt[g].row0; rgf[g] = (uint32_t)rgt[g].file; }
  return ETL_OK;
}

// Plan (block 0): k_plan and the length scans, the counting k_cut, k_row_max, k_chunk_nn; SYNC 1 reads the totals
int Call::plan() {
  if (!carve(0)) return ETL_ERR_ALLOC;
  const uint32_t lb = scan_blocks(n);
  CK(cudaMemcpyAsync(d_leaves, hl.data(), sizeof(LeafDev) * nL, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_rgb, rgb.data(), 8ull * (n_rg + 1), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_rgf, rgf.data(), 4ull * (n_rg + 1), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_req, 0xff, nL * 8ull, st));
  if (pidx) CK(cudaMemsetAsync(d_vmax, 0, 4ull * nL, st));
  CK(cudaMemsetAsync(d_tot, 0, 3ull * nL * 8, st));
  uint32_t* lens[3] = {d_ent, d_nn, d_vb}; uint64_t* pre[3] = {d_E, d_NN, d_V};
  for (uint64_t* p : pre) CK(cudaMemsetAsync(p, 0, 8ull * nL * (n + 1), st));
  if (n) {
    k_plan<<<dim3((uint32_t)((n + 255) / 256), nL), 256, 0, st>>>(d_leaves, row_begin, n, d_ent, d_nn, d_vb, d_req);
    for (uint32_t s = 0; s < 3; s++)
      for (uint32_t l = 0; l < nL; l++) {
        const uint64_t at = (uint64_t)(s * nL + l);
        scan_lengths(lens[s] + (uint64_t)l * (n + 1), n, d_blk + at * (lb + 1), d_tot + at, pre[s] + (uint64_t)l * (n + 1), st);
      }
    k_cut<<<(n_chunks + 63) / 64, 64, 0, st>>>(d_leaves, nL, n_rg, row_begin, d_rgb, n, d_E, d_NN, d_V, d_np, nullptr, nullptr, nullptr, nullptr, 0);
    if (pidx) k_row_max<<<dim3((uint32_t)((n + 255) / 256), nL), 256, 0, st>>>(d_leaves, n, d_vb, d_vmax);
    if (any_bloom) k_chunk_nn<<<(n_chunks + 255) / 256, 256, 0, st>>>(nL, n_chunks, n, d_rgb, d_NN, d_cnn);
  }
  // SYNC 1: page counts, totals, required-column nulls (bloom filters: the chunks' non-null values)
  t.np.assign(n_chunks, 0); t.cnn.assign(n_chunks, 0); t.tot.assign(3ull * nL, 0); t.req.assign(nL, 0); t.vmax.assign(nL, 0);
  if (any_bloom && n_chunks) CK(cudaMemcpyAsync(t.cnn.data(), d_cnn, n_chunks * 8ull, cudaMemcpyDeviceToHost, st));
  if (n_chunks) CK(cudaMemcpyAsync(t.np.data(), d_np, n_chunks * 4ull, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(t.tot.data(), d_tot, 3ull * nL * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(t.req.data(), d_req, nL * 8ull, cudaMemcpyDeviceToHost, st));
  if (pidx) CK(cudaMemcpyAsync(t.vmax.data(), d_vmax, 4ull * nL, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ETL_OK;
}

// Size: every bound and host table, a function of the description and the totals
Sizes Call::size() const {
  const std::vector<unsigned long long>& tot = t.tot;
  Sizes o{};
  o.hl = hl;
  o.page_base.assign(n_chunks + 1, 0);
  for (uint32_t c = 0; c < n_chunks; c++) o.page_base[c + 1] = o.page_base[c] + t.np[c] + (has_dict(c % nL) ? 1 : 0);
  o.P = o.page_base[n_chunks];
  // bounds of every buffer from the totals
  o.pages_of.assign(nL, 0);
  for (uint32_t c = 0; c < n_chunks; c++) o.pages_of[c % nL] += t.np[c];
  for (uint32_t l = 0; l < nL; l++) {
    const uint64_t El = tot[l], NNl = tot[nL + l], Vl = tot[2 * nL + l], Pl = o.pages_of[l];
    const uint64_t lev = 14 * Pl + (El / 8 + Pl) * (hl[l].w + 2);
    o.U += (hl[l].atype == ETL_ARROW_BOOLEAN ? NNl / 8 + Pl : Vl) + (hl[l].max_def ? lev : 0) + (hl[l].max_rep ? 14 * Pl + (El / 8 + Pl) * 3 : 0);
    if (has_dict(l)) o.U += std::min<uint64_t>(Vl, n_rg * kDictBytes) + 32 * Pl;   // the dictionary slots, the index runs
  }
  // dictionary scratch: per item bound (a leaf's level entries) slot, flag, entry size / index, two prefix sums; run
  // heads per 8 items + 3 per page; the chunks' tables of at most 4 × non-null values (+ 1) slots
  for (uint32_t l = 0; l < nL; l++) {
    if (!has_dict(l)) continue;
    o.hl[l].dscr = o.d_items; o.hl[l].hscr = o.d_heads;
    o.d_items += tot[l] + 1;
    o.d_heads += tot[l] / 8 + 3 * (o.pages_of[l] + 1) + 8;
    o.d_slots += 4 * tot[nL + l] + n_rg;
    o.d_maxI = std::max<uint64_t>(o.d_maxI, tot[l]);
  }
  // level scratch of a leaf: rep | def of each page, 8-aligned, at 2 * align8(e0) + 64 * (page index within the leaf)
  o.lscr_base.assign(nL + 1, 0);
  for (uint32_t l = 0; l < nL; l++) o.lscr_base[l + 1] = o.lscr_base[l] + 2 * ((tot[l] + 7) & ~7ull) + 64 * (o.pages_of[l] + 1) + 64;
  o.leaf_page_base.assign(n_chunks + 1, 0);         // pages of the chunk's leaf in the row groups before it
  for (uint32_t c = nL; c < n_chunks; c++) o.leaf_page_base[c] = o.leaf_page_base[c - nL] + t.np[c - nL];
  o.n_frag_bound = snappy ? o.U / kFragment + o.P + 1 : 0;
  // compressed slots: 8 B per page and each fragment's bound (affine in its bytes: 32 + 7 n / 6 at most), the
  // fragments' bytes adding up to at most U
  o.C_bound = snappy ? 8 * o.P + 32 * o.n_frag_bound + o.U + o.U / 6 : 0;
  // bit scratch: page lp of a Boolean leaf starts at word bscr + it0 / 32 + lp
  for (uint32_t l = 0; l < nL; l++)
    if (hl[l].atype == ETL_ARROW_BOOLEAN) {
      o.hl[l].bscr = o.bool_words;
      o.bool_words += values[l] / 32 + o.pages_of[l] + 2;
    }
  // bloom filters: each filtered chunk's bitset size from its ndv (or non-null count), its header, its place among the
  // call's filters (row-group major, column minor: each file's run follows its pages) and its bitset's place in the
  // zeroed scratch
  o.hb.assign(n_chunks, BloomChunk{0, 0, 0, 0});
  std::vector<uint64_t> bloom_at(n_chunks + 1, 0);
  for (uint32_t c = 0; c < n_chunks; c++) {
    const uint32_t l = c % nL;
    bloom_at[c] = o.bloom_total;
    if (!bloomed(l)) continue;
    const etl_parquet_bloom& Bf = bloom[l];
    const uint64_t ndv = Bf.ndv ? Bf.ndv : std::max<uint64_t>(1, t.cnn[c]);
    BloomChunk& Kb = o.hb[c];
    Kb.bytes = (uint32_t)bloom_bytes(ndv, Bf.fpp, Bf.max_bytes ? Bf.max_bytes : kBloomDefaultBytes);
    Kb.hlen = bloom_header(nullptr, Kb.bytes);
    Kb.off = o.bloom_total; Kb.word = o.bloom_words;
    o.bloom_total += Kb.hlen + Kb.bytes; o.bloom_words += Kb.bytes / 4;
  }
  bloom_at[n_chunks] = o.bloom_total;
  o.hf.resize(K);
  for (uint64_t k = 0; k < K; k++) {
    const uint64_t c0 = frg[k] * nL, c1 = frg[k + 1] * nL;
    o.hf[k] = FileRec{frg[k], frg[k + 1], o.page_base[c0], o.page_base[c1], bloom_at[c0], bloom_at[c1], 0, 0, 0};
  }
  // footers: the schema prefix once; the tail's bound from one file of no row group and one of a row group whose every
  // field is at its widest (sizes and offsets 2^62, statistics of kStatMax bytes), with room for the varints that
  // grow with the row count and the row-group ordinal
  TWriter pw(nullptr);
  footer_prefix(pw, meta);
  o.prefix.resize(pw.n);
  { TWriter w(o.prefix.data()); footer_prefix(w, meta); }
  o.lm = leaf_meta(meta);
  const std::string stat_x(kStatMax, 'x');
  auto wide = [&](uint64_t c) {
    const uint32_t l = (uint32_t)(c % nL);
    const uint64_t x = 1ull << 62;
    return ChunkMeta{x, x, x, x, x, x, INT32_MAX, x, x, x, INT32_MAX, INT32_MAX, bloomed(l) ? INT32_MAX : 0u, kStatMax, kStatMax,
                     true, has_dict(l), pidx != 0, (const uint8_t*)stat_x.data(), (const uint8_t*)stat_x.data()};
  };
  const uint64_t wide_rg[2] = {0, 1ull << 62};
  const uint64_t tail0 = footer_tail(nullptr, o.lm.data(), nL, wide_rg, 0, wide, cc, (const uint8_t*)kCreatedBy, kCreatedByLen);
  const uint64_t tail1 = footer_tail(nullptr, o.lm.data(), nL, wide_rg, 1, wide, cc, (const uint8_t*)kCreatedBy, kCreatedByLen);
  o.footer_bound = K * (o.prefix.size() + tail0 + 20 + 8) + (uint64_t)n_rg * (tail1 - tail0 + 40);
  o.data_bound = 4 * K + o.P * kPageHeaderMax + (snappy ? o.C_bound : o.U);
  // ETL_PQ_PAGE_INDEX: per page a ColumnIndex entry (null flag, two bounds of at most 64 bytes + a 10-byte length, a
  // null count) and a PageLocation, per chunk the fields' and lists' headers; a byte-array maximum that cannot be
  // incremented stays whole, at most its page's longest row (bounded by the leaf's rows or its value bytes)
  if (pidx) {
    o.index_bound = o.P * (1 + 2 * (10 + kIndexTruncate) + 10 + 30) + 64ull * n_chunks;
    for (uint32_t l = 0; l < nL; l++)
      if (t.vmax[l] > kIndexTruncate) o.index_bound += std::min<uint64_t>(tot[2 * nL + l], (o.pages_of[l] + n_rg) * (uint64_t)t.vmax[l]);
  }
  // the footers' leaves, names, created_by and schema prefix, in one device block
  o.meta_bytes = sizeof(LeafMeta) * nL + kCreatedByLen + o.prefix.size();
  for (const Leaf& M : meta) o.meta_bytes += M.name.size();
  return o;
}

// Launch (block 1 and the output buffer): the uploads, then every stage's kernels in order
int Call::launch() {
  if (!carve(1)) return ETL_ERR_ALLOC;
  const uint64_t P = s.P;
  if (cudaMalloc(&dev, s.data_bound + s.bloom_total + s.index_bound + s.footer_bound + 64) != cudaSuccess) { dev = nullptr; return ETL_ERR_ALLOC; }
  // the footers' device block: the leaves (their names pointing into it), the names, created_by, the schema prefix
  const uint64_t lm_bytes = sizeof(LeafMeta) * nL;
  std::vector<uint8_t> hmeta(s.meta_bytes);
  std::vector<LeafMeta> dm = s.lm;
  uint64_t o = lm_bytes;
  for (uint32_t l = 0; l < nL; l++) {
    memcpy(hmeta.data() + o, meta[l].name.data(), meta[l].name.size());
    dm[l].name = d_meta + o;
    o += meta[l].name.size();
  }
  memcpy(hmeta.data(), dm.data(), lm_bytes);
  memcpy(hmeta.data() + o, kCreatedBy, kCreatedByLen);
  memcpy(hmeta.data() + o + kCreatedByLen, s.prefix.data(), s.prefix.size());
  const FooterArgs fa{(const LeafMeta*)d_meta, d_meta + s.meta_bytes - s.prefix.size(), d_meta + s.meta_bytes - s.prefix.size() - kCreatedByLen,
                      nL, (uint32_t)s.prefix.size(), kCreatedByLen, cc};
  CK(cudaMemcpyAsync(d_leaves, s.hl.data(), sizeof(LeafDev) * nL, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_pbase, s.page_base.data(), 8 * (n_chunks + 1ull), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_lpbase, s.leaf_page_base.data(), 8 * (n_chunks + 1ull), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_lbase, s.lscr_base.data(), 8 * (nL + 1ull), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_files, s.hf.data(), sizeof(FileRec) * K, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_meta, hmeta.data(), s.meta_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_bool, 0, s.bool_words * 4 + 8, st));
  CK(cudaMemsetAsync(d_lscr, 0, s.lscr_base[nL] + 16, st));
  CK(cudaMemsetAsync(d_foff + P, 0, 8, st));
  if (s.bloom_total) {
    CK(cudaMemcpyAsync(d_bch, s.hb.data(), sizeof(BloomChunk) * n_chunks, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_bwords, 0, 4 * s.bloom_words, st));
  }
  const uint32_t kb = (uint32_t)((K + 1 + kFootWarps - 1) / kFootWarps);   // a warp per file (+ the scan's last entry)
  const uint32_t xb = (n_chunks + kIdxWarps) / kIdxWarps;            // k_index: a warp per chunk
  if (P) {
    k_cut<<<(n_chunks + 63) / 64, 64, 0, st>>>(d_leaves, nL, n_rg, row_begin, d_rgb, n, d_E, d_NN, d_V, d_np, d_pbase, d_lpbase, d_lbase, d_pages, dict);
    // payload slots: exclusive scan of the page bounds (and, with Snappy, of the fragment slots)
    auto fill_scan = [&](TotSlot which, uint64_t* dst) {
      k_fill<<<(uint32_t)((P + 256) / 256), 256, 0, st>>>(d_pages, (uint32_t)P, which, cc, dst);
      k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>((unsigned long long*)dst, (uint32_t)(P + 1), d_stot + which);
    };
    fill_scan(kTotUslot, d_uslot);
    if (d_dch) {
      // dictionaries: tables, inserts, first-occurrence flags and their scans, decisions, dictionary pages
      k_dict_setup<<<(n_chunks + 256) / 256, 256, 0, st>>>(d_leaves, nL, n_chunks, row_begin, d_rgb, n, d_NN, d_pbase, d_dch, d_tabn);
      k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>(d_tabn, n_chunks + 1, d_stot + kTotDict);
      k_dict_place<<<(n_chunks + 255) / 256, 256, 0, st>>>(n_chunks, d_tabn, d_dch);
      CK(cudaMemsetAsync(d_tab, 0xff, 4 * s.d_slots, st));
      for (uint32_t l = 0; l < nL; l++) {
        if (!has_dict(l)) continue;
        const uint64_t I = t.tot[l], at = s.hl[l].dscr;
        const uint32_t ib = (uint32_t)((I + 255) / 256);
        k_dict_insert<<<std::min<uint32_t>(kInsBlocks, ib), kInsThreads, 0, st>>>(d_leaves, l, nL, n_rg, row_begin, d_dch, d_tab, d_dpos);
        const bool bytes = hl[l].atype == ETL_ARROW_UTF8 || hl[l].atype == ETL_ARROW_LARGE_BINARY;
        k_dict_mark<<<ib, 256, 0, st>>>(d_leaves, l, nL, n_rg, row_begin, I, d_dch, d_tab, d_dpos, d_dflag, bytes ? d_desz : nullptr);
        scan_lengths(d_dflag + at, I, d_dblk, d_stot + kTotDict, d_dfirst + at, st);
        if (bytes) scan_lengths(d_desz + at, I, d_dblk, d_stot + kTotDict, d_desum + at, st);
      }
      k_dict_finish<<<(n_chunks + 255) / 256, 256, 0, st>>>(d_leaves, nL, n_chunks, row_begin, d_dfirst, d_desum, d_dch, d_pages);
      for (uint32_t l = 0; l < nL; l++)
        if (has_dict(l))
          k_dict_page<<<(uint32_t)((t.tot[l] + 255) / 256), 256, 0, st>>>(d_leaves, l, nL, n_rg, row_begin, t.tot[l], d_dch, d_dfirst, d_desum, d_u, d_uslot);
      const DictArgs da{d_dch, d_tab, d_dpos, d_dfirst, d_desz, d_dhead};
      k_encode<true><<<(uint32_t)P, kEncThreads, 0, st>>>(d_leaves, d_pages, row_begin, d_E, n, d_lscr, d_u, d_uslot, d_bool, da);
    } else {
      k_encode<false><<<(uint32_t)P, kEncThreads, 0, st>>>(d_leaves, d_pages, row_begin, d_E, n, d_lscr, d_u, d_uslot, d_bool, DictArgs{});
    }
    if (snappy) {
      fill_scan(kTotCslot, d_cslot);
      fill_scan(kTotFbase, d_fbase);
      if (zstd) k_zstd<<<(uint32_t)s.n_frag_bound, 32, 0, st>>>(d_pages, (uint32_t)P, d_fbase, d_u, d_uslot, d_c, d_cslot, d_fsz, d_zlit, d_zseq);
      else k_snappy<<<(uint32_t)s.n_frag_bound, 32, 0, st>>>(d_pages, (uint32_t)P, d_fbase, d_u, d_uslot, d_c, d_cslot, d_fsz);
    }
    k_page<<<(uint32_t)((P + 255) / 256), 256, 0, st>>>(d_pages, (uint32_t)P, cc, d_fbase, d_fsz, d_foff, d_dch);
    k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>((unsigned long long*)d_foff, (uint32_t)(P + 1), d_stot + kTotFoff);
    k_chunk<<<(n_chunks + 63) / 64, 64, 0, st>>>(d_leaves, d_pages, d_pbase, n_chunks, nL, d_foff, d_rgf, d_files, d_bch, pidx, d_cout, d_dch);
    if (d_ix) {
      // page index: sizes and boundary orders, their places in each file behind its pages and filters
      k_index<false><<<xb, 32 * kIdxWarps, 0, st>>>(d_leaves, d_pages, d_pbase, n_chunks, nL, d_rgb, d_rgf, d_files, d_fplace, d_foff, d_ix, d_ixlen, dev, d_cout);
      k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>(d_ixlen, 2 * n_chunks + 1, d_stot + kTotIndex);
      k_index_place<<<(n_chunks + 63) / 64, 64, 0, st>>>(n_chunks, nL, d_rgf, d_files, d_foff, d_ix, d_ixlen, d_cout);
    }
  }
  // every file's footer length and size, their scan (the files' places), then every byte at its place
  k_footer<false><<<kb, 32 * kFootWarps, 0, st>>>(fa, K, d_rgb, d_files, d_foff, d_ixlen, d_cout, d_fplace, dev);
  k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>((unsigned long long*)d_fplace, (uint32_t)(K + 1), d_stot + kTotFiles);
  if (P) {
    k_gather<<<(uint32_t)P, 256, 0, st>>>(d_pages, cc, d_foff, d_u, d_uslot, d_c, d_cslot, d_fbase, d_fsz, nL, d_rgf, d_files, d_fplace, dev);
    if (s.bloom_total) {
      // bloom filters: the bitsets in scratch, then headers and bitsets behind each file's pages
      for (uint32_t l = 0; l < nL; l++)
        if (bloomed(l))
          k_bloom<<<std::min<uint32_t>(kInsBlocks, (uint32_t)((t.tot[l] + kInsThreads - 1) / kInsThreads) + 1), kInsThreads, 0, st>>>(
              d_leaves, l, nL, n_rg, row_begin, d_rgb, d_bch, d_bwords);
      k_bloom_write<<<dim3(n_chunks, 16), 256, 0, st>>>(d_bch, d_bwords, nL, d_rgf, d_fplace, d_cout, dev);
    }
    if (d_ix)
      k_index<true><<<xb, 32 * kIdxWarps, 0, st>>>(d_leaves, d_pages, d_pbase, n_chunks, nL, d_rgb, d_rgf, d_files, d_fplace, d_foff, d_ix, d_ixlen, dev, d_cout);
  }
  k_footer<true><<<kb, 32 * kFootWarps, 0, st>>>(fa, K, d_rgb, d_files, d_foff, d_ixlen, d_cout, d_fplace, dev);
  k_leaf<<<(uint32_t)((K * nL + 63) / 64), 64, 0, st>>>(d_leaves, nL, K, n_chunks, d_files, d_cout, d_lout);
  return ETL_OK;
}

// Collect: SYNC 2 (the files' places and every (file, leaf) record), SYNC 3 with to_host (the pinned image) and the
// metrics; the output moves to Fs
int Call::collect(etl_parquet_files* Fs) {
  std::vector<ChunkOut> hlo(K * nL);
  CK(cudaMemcpyAsync(Fs->offs.data(), d_fplace, 8 * (K + 1), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(hlo.data(), d_lout, sizeof(ChunkOut) * K * nL, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  const uint64_t total = Fs->offs[K];
  if (to_host) {
    if (cudaHostAlloc((void**)&host, total + 1, cudaHostAllocDefault) != cudaSuccess) { host = nullptr; return ETL_ERR_ALLOC; }
    CK(cudaMemcpyAsync(host, dev, total, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));                  // SYNC 3
  }
  // metrics: one record per (file, leaf); their statistic bytes in one block
  uint64_t sb = 0;
  for (const ChunkOut& R : hlo) if (R.has) sb += R.min_len + R.max_len;
  Fs->stats.resize(sb);
  Fs->metrics.resize(K * nL);
  uint64_t so = 0;
  for (uint64_t i = 0; i < K * nL; i++) {
    const ChunkOut& R = hlo[i];
    const uint32_t l = (uint32_t)(i % nL);
    etl_parquet_metrics& M = Fs->metrics[i];           // zeroed by resize
    M.field_id = hl[l].is_list ? fields[l].element_field_id : fields[l].field_id;
    M.flags = R.has ? ETL_PQ_HAS_MIN_MAX : 0;
    M.num_values = R.num_values; M.null_count = R.null_count; M.nan_count = R.nan_count;
    M.compressed_bytes = R.csize; M.uncompressed_bytes = R.usize;
    if (R.has) {
      memcpy(Fs->stats.data() + so, R.min, R.min_len); M.min = Fs->stats.data() + so; M.min_len = R.min_len; so += R.min_len;
      memcpy(Fs->stats.data() + so, R.max, R.max_len); M.max = Fs->stats.data() + so; M.max_len = R.max_len; so += R.max_len;
    }
  }
  Fs->dev = dev; Fs->host = host;
  dev = host = nullptr;
  return ETL_OK;
}
#undef CK

// The writer: files k < K, file k the rows [ro[k], ro[k + 1]) of the emit, in one device buffer (and with to_host one
// pinned image), packed in order.  etl_dec_parquet_write(_bloom) is K = 1.  Fs is filled on ETL_OK; on an error
// everything the call allocated is freed (Fs owns nothing yet).
int write_files(const etl_arrow_batch* a, const etl_parquet_field* fields, const etl_parquet_bloom* bloom, uint32_t n_fields,
                const uint64_t* ro, uint64_t K, uint32_t codec, int to_host, etl_parquet_files* Fs) {
  Call c{a, fields, bloom, n_fields, ro, K, codec, to_host};
  int rc = c.describe();
  if (rc != ETL_OK) return rc;
  Fs->n_files = K; Fs->n_leaves = n_fields; Fs->offs.assign(K + 1, 0);
  if (!K) return ETL_OK;
  rc = c.plan();
  if (rc == ETL_OK) {
    for (uint32_t l = 0; l < n_fields; l++)           // RecordBatch::try_new fails before anything is written
      if (c.t.req[l] != kNone) { Fs->null_column = l; Fs->null_row = c.t.req[l]; return ETL_OK; }
    c.s = c.size();
    rc = c.launch();
    if (rc == ETL_OK) rc = c.collect(Fs);
  }
  if (rc != ETL_OK) cudaGetLastError();             // a failed call leaves no CUDA error behind for the next
  return rc;
}

}  // namespace

extern "C" {

int etl_dec_parquet_write(const etl_arrow_batch* a, const etl_parquet_field* fields, uint32_t n_fields, uint64_t row_begin,
                          uint64_t row_end, uint32_t codec, int to_host, etl_parquet_file** out) {
  return etl_dec_parquet_write_bloom(a, fields, nullptr, n_fields, row_begin, row_end, codec, to_host, out);
}

int etl_dec_parquet_write_bloom(const etl_arrow_batch* a, const etl_parquet_field* fields, const etl_parquet_bloom* bloom,
                                uint32_t n_fields, uint64_t row_begin, uint64_t row_end, uint32_t codec, int to_host,
                                etl_parquet_file** out) {
  if (!out) return ETL_ERR_INVALID_ARG;
  const uint64_t ro[2] = {row_begin, row_end};
  std::unique_ptr<etl_parquet_file> f(new etl_parquet_file());
  const int rc = write_files(a, fields, bloom, n_fields, ro, 1, codec, to_host, f.get());
  if (rc == ETL_OK) *out = f.release();
  return rc;
}
// file 0 of its etl_parquet_files (offs[1]: its size, 0 after a required null)
uint64_t etl_dec_parquet_size(const etl_parquet_file* f) { return f ? etl_dec_parquet_files_offsets(f)[1] : 0; }
const uint8_t* etl_dec_parquet_bytes(const etl_parquet_file* f, int host) { return etl_dec_parquet_files_bytes(f, host); }
int etl_dec_parquet_metrics(const etl_parquet_file* f, uint32_t leaf, etl_parquet_metrics* out) { return etl_dec_parquet_files_metrics(f, 0, leaf, out); }
int etl_dec_parquet_required_null(const etl_parquet_file* f, uint32_t* column, uint64_t* row) { return etl_dec_parquet_files_required_null(f, column, row); }
void etl_dec_parquet_free(etl_parquet_file* f) { delete f; }

int etl_dec_parquet_write_files(const etl_arrow_batch* a, const etl_parquet_field* fields, const etl_parquet_bloom* bloom,
                                uint32_t n_fields, const uint64_t* row_offsets, uint64_t n_files, uint32_t codec, int to_host,
                                etl_parquet_files** out) {
  if (!out) return ETL_ERR_INVALID_ARG;
  std::unique_ptr<etl_parquet_files> Fs(new etl_parquet_files());
  const int rc = write_files(a, fields, bloom, n_fields, row_offsets, n_files, codec, to_host, Fs.get());
  if (rc == ETL_OK) *out = Fs.release();
  return rc;
}
uint64_t etl_dec_parquet_files_count(const etl_parquet_files* fs) { return fs ? fs->n_files : 0; }
const uint64_t* etl_dec_parquet_files_offsets(const etl_parquet_files* fs) { return fs ? fs->offs.data() : nullptr; }
const uint8_t* etl_dec_parquet_files_bytes(const etl_parquet_files* fs, int host) { return fs ? (host ? fs->host : fs->dev) : nullptr; }
int etl_dec_parquet_files_metrics(const etl_parquet_files* fs, uint64_t file, uint32_t leaf, etl_parquet_metrics* out) {
  if (!fs || !out || file >= fs->n_files || leaf >= fs->n_leaves || fs->metrics.empty()) return ETL_ERR_INVALID_ARG;
  *out = fs->metrics[file * fs->n_leaves + leaf];
  return ETL_OK;
}
int etl_dec_parquet_files_required_null(const etl_parquet_files* fs, uint32_t* column, uint64_t* row) {
  if (!fs) return ETL_ERR_INVALID_ARG;
  if (column) *column = fs->null_column;
  if (row) *row = fs->null_row;
  return ETL_OK;
}
void etl_dec_parquet_files_free(etl_parquet_files* fs) { delete fs; }

}  // extern "C"

// ptxas -v, sm_90a, CUDA 12.9 (registers / shared memory / stack):
//   k_plan 32 / 0 / 0      k_cut 53 / 0 / 0       k_encode<false> 48 / 4176 B / 8 B (one 8-byte spill)    k_fill 16 / 0 / 0
//   k_encode<true> 64 / 4200 B / 16 B (two 8-byte spills)
//   k_snappy 50 / 8192 B / 0                      k_page 29 / 0 / 40 B (the header bytes)   k_gather 22 / 0 / 0 (+ a load
//   of its file's place)
//   k_zstd 88 / 27772 B / 104 B, no spills (the stack is the canonical-code rank counters of the Huffman table)
//   k_dict_setup 23 / 0 / 0   k_dict_place 10 / 0 / 0   k_dict_insert 46 / 0 / 0   k_dict_mark 24 / 0 / 0
//   k_dict_finish 22 / 0 / 0  k_dict_page 32 / 0 / 0
//   k_chunk 56 / 0 / 248 B and k_leaf 56 / 0 / 248 B (the ChunkOut record built in local memory, written once)
//   k_row_max 12 / 0 / 0   k_index<false> 89 / 0 / 40 B and k_index<true> 96 / 0 / 48 B (a fixed-width bound's bytes;
//   no spills: __maxnreg__(96) instead of the launch bound, which left ptxas at 64 registers and spilling)
//   k_index_place 30 / 0 / 0   k_footer<false> 96 / 0 / 40 B and k_footer<true> 96 / 0 / 40 B (the Thrift writer;
//   __maxnreg__(96), as k_index: a 128-thread launch bound left them at 64 registers, one spilling)
//   k_chunk_nn 14 / 0 / 0   k_bloom 55 / 0 / 0   k_bloom_write 29 / 0 / 40 B (the header's Thrift writer)
//   the shared scans of emit_scan.cuh: k_len_blocks 22 / 256 B, k_blk_scan<unsigned long long> 32 / 8192 B,
//   k_offsets<uint64_t> 18 / 8192 B, k_copy_sel 12 / 0 / 0
