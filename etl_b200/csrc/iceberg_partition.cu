// iceberg_partition.cu — Iceberg partitioning of an Arrow emit on the device (etl_dec_iceberg_partition): the partition
// transforms per (row, field), the grouping of the rows by partition tuple, and a permuted copy of the emit in which
// every partition is a contiguous row range that etl_dec_parquet_write(_bloom) writes as one data file.
//
// Stages (the header comment states the semantics):
//   k_ice_transform  thread per row: every field's result (an integer, or a span of the source's bytes: identity and
//                    truncate of Utf8 / LargeBinary / UUID copy nothing) and a 64-bit tuple hash;
//   k_ice_group      thread per row: insert into an open-addressing table of 2n+ slots keyed by tuple (hash, then a
//                    full compare against the slot's first claimant), atomicMin of the row into the slot's first row;
//   k_ice_heads      a row is its partition's head when it is the slot's first row; the scan of the head flags ranks
//                    the partitions by first row, the scans of the heads' byte lengths size the representative values;
//   k_ice_slice      the slice's byte and element counts of every variable-width column (for the output layout);
//   — sync: partition count, representative bytes, slice sizes —
//   k_ice_keys       rank of each row's partition; a stable CUB radix sort of (rank, row) is the permutation;
//   k_ice_bounds     partition row offsets from the sorted ranks;  k_ice_reps  the representative values (warp each);
//   k_ice_gather_*   every column through the permutation: validity / Boolean bits by ballot, fixed-width values,
//                    lengths → offsets (emit_scan.cuh's scan_lengths) → bytes a warp per row; a List expands its rows'
//                    element indices and its child goes through the same flat gathers.
// The output's sizes are those of the source slice, so nothing but the one sync above sizes a buffer.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <vector>

#include "etl_decode.h"
#include "arrow_internal.h"
#include "emit_scan.cuh"
#include "iceberg_partition.cuh"

using etl_arrow::Col;

namespace {

constexpr uint32_t kEmpty = 0xFFFFFFFFu;

struct FieldDesc {
  const uint8_t* validity; const uint8_t* values; const uint8_t* data; const void* offsets;
  const uint64_t* rep_off;        // span results: offsets of the heads' bytes (scan over rows)
  uint64_t rep_base;              // span results: where this field's representative bytes start
  uint32_t arrow_type, transform, param, span;   // span: the result is a span of base() (Utf8 / LargeBinary / UUID)
};
struct TParams {
  FieldDesc f[ETL_ICE_MAX_FIELDS];
  uint32_t n_fields;
  uint64_t rb, n;                 // source rows [rb, rb + n)
  int64_t* val; uint32_t* len; uint8_t* nul;    // per (field, row), field-major: value or span offset, span length, null
  uint64_t* hash;                 // per row
};
__host__ __device__ __forceinline__ const uint8_t* base_of(const FieldDesc& F) { return F.arrow_type == ETL_ARROW_UUID ? F.values : F.data; }
__device__ __forceinline__ bool bit_at(const uint8_t* b, uint64_t i) { return (b[i >> 3] >> (i & 7)) & 1u; }
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// thread per row: the result of every field and the tuple hash
__global__ void __launch_bounds__(256) k_ice_transform(TParams T) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T.n) return;
  const uint64_t s = T.rb + i;
  uint64_t h = 0x9e3779b97f4a7c15ull;
  for (uint32_t k = 0; k < T.n_fields; k++) {
    const FieldDesc& F = T.f[k];
    const bool nul = F.transform == ETL_ICE_VOID || !bit_at(F.validity, s);
    int64_t v = 0;
    uint32_t ln = 0;
    if (!nul) {
      switch (F.arrow_type) {
        case ETL_ARROW_BOOLEAN: v = bit_at(F.values, s); break;
        case ETL_ARROW_INT32: case ETL_ARROW_DATE32: v = reinterpret_cast<const int32_t*>(F.values)[s]; break;
        case ETL_ARROW_UTF8: { const int32_t* o = static_cast<const int32_t*>(F.offsets); v = o[s]; ln = (uint32_t)(o[s + 1] - o[s]); break; }
        case ETL_ARROW_LARGE_BINARY: { const int64_t* o = static_cast<const int64_t*>(F.offsets); v = o[s]; ln = (uint32_t)(o[s + 1] - o[s]); break; }
        case ETL_ARROW_UUID: v = (int64_t)(16 * s); ln = 16; break;
        default: v = reinterpret_cast<const int64_t*>(F.values)[s]; break;      // Int64, Time64, Timestamp(tz)
      }
      const bool bytes_src = F.arrow_type == ETL_ARROW_UTF8 || F.arrow_type == ETL_ARROW_LARGE_BINARY || F.arrow_type == ETL_ARROW_UUID;
      const bool date = F.arrow_type == ETL_ARROW_DATE32;
      switch (F.transform) {
        case ETL_ICE_BUCKET:
          v = etl_ice::bucket_of(bytes_src ? etl_ice::murmur3_32(base_of(F) + v, ln, 0) : etl_ice::murmur3_i64(v), F.param);
          ln = 0;
          break;
        case ETL_ICE_TRUNCATE:
          if (F.arrow_type == ETL_ARROW_INT32) v = etl_ice::truncate_i32((int32_t)v, F.param);
          else if (F.arrow_type == ETL_ARROW_INT64) v = etl_ice::truncate_i64(v, F.param);
          else if (F.arrow_type == ETL_ARROW_UTF8) ln = etl_ice::utf8_prefix(F.data + v, ln, F.param);
          else ln = min(ln, F.param);
          break;
        case ETL_ICE_YEAR: v = etl_ice::years_of_days(date ? v : etl_ice::days_of_micros(v)); break;
        case ETL_ICE_MONTH: v = etl_ice::months_of_days(date ? v : etl_ice::days_of_micros(v)); break;
        case ETL_ICE_DAY: if (!date) v = etl_ice::days_of_micros(v); break;
        case ETL_ICE_HOUR: v = etl_ice::hours_of_micros(v); break;
        default: break;                                    // identity
      }
    }
    const uint64_t at = (uint64_t)k * T.n + i;
    T.val[at] = v; T.len[at] = ln; T.nul[at] = nul;
    const uint64_t x = nul ? 0x6e756c6cull : F.span ? ((uint64_t)etl_ice::murmur3_32(base_of(F) + v, ln, k) << 32 | ln) : (uint64_t)v;
    h = mix64(h ^ (x + 0x9e3779b97f4a7c15ull * (k + 1)));
  }
  T.hash[i] = h;
}
__device__ bool same_tuple(const TParams& T, uint64_t a, uint64_t b) {
  if (T.hash[a] != T.hash[b]) return false;
  for (uint32_t k = 0; k < T.n_fields; k++) {
    const uint64_t ia = (uint64_t)k * T.n + a, ib = (uint64_t)k * T.n + b;
    if (T.nul[ia] != T.nul[ib]) return false;
    if (T.nul[ia]) continue;
    if (!T.f[k].span) { if (T.val[ia] != T.val[ib]) return false; continue; }
    const uint32_t ln = T.len[ia];
    if (ln != T.len[ib]) return false;
    const uint8_t* pa = base_of(T.f[k]) + T.val[ia];
    const uint8_t* pb = base_of(T.f[k]) + T.val[ib];
    for (uint32_t j = 0; j < ln; j++) if (pa[j] != pb[j]) return false;
  }
  return true;
}
// thread per row: find or claim the tuple's slot (linear probing; the table has at least twice as many slots as rows)
__global__ void __launch_bounds__(256) k_ice_group(TParams T, uint32_t* slot_row, uint32_t* slot_first, uint32_t mask, uint32_t* row_slot) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T.n) return;
  uint32_t s = (uint32_t)(T.hash[i] ^ (T.hash[i] >> 32)) & mask;
  for (;;) {
    uint32_t cur = slot_row[s];
    if (cur == kEmpty) {
      cur = atomicCAS(slot_row + s, kEmpty, (uint32_t)i);
      if (cur == kEmpty) break;
    }
    if (same_tuple(T, cur, i)) break;
    s = (s + 1) & mask;
  }
  atomicMin(slot_first + s, (uint32_t)i);
  row_slot[i] = s;
}
// thread per row: head flag (the row is its partition's first) and, per span field, the head's byte length
__global__ void __launch_bounds__(256) k_ice_heads(TParams T, const uint32_t* slot_first, const uint32_t* row_slot, uint32_t* head, uint32_t* rep_len) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T.n) return;
  const bool hd = slot_first[row_slot[i]] == (uint32_t)i;
  head[i] = hd;
  uint32_t b = 0;
  for (uint32_t k = 0; k < T.n_fields; k++) {
    if (!T.f[k].span) continue;
    const uint64_t at = (uint64_t)k * T.n + i;
    rep_len[(uint64_t)b++ * (T.n + 1) + i] = hd && !T.nul[at] ? T.len[at] : 0u;
  }
}
// the slice [rb, re) of each variable-width column: data bytes (Utf8 / LargeBinary) or elements and the child's data
// bytes (List)
struct SliceDesc { const void* offs; const void* kid_offs; uint32_t arrow_type, kid_type; };
__global__ void k_ice_slice(const SliceDesc* d, uint32_t n_cols, uint64_t rb, uint64_t re, unsigned long long* out) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  const SliceDesc D = d[c];
  auto span = [](uint32_t at, const void* o, uint64_t a, uint64_t b) -> unsigned long long {
    if (at == ETL_ARROW_LARGE_BINARY) return (unsigned long long)(static_cast<const int64_t*>(o)[b] - static_cast<const int64_t*>(o)[a]);
    return (unsigned long long)(uint32_t)(static_cast<const int32_t*>(o)[b] - static_cast<const int32_t*>(o)[a]);
  };
  unsigned long long a = 0, b = 0;
  if (D.offs) a = span(D.arrow_type, D.offs, rb, re);
  if (D.kid_offs) {
    const int32_t* lo = static_cast<const int32_t*>(D.offs);
    b = span(D.kid_type, D.kid_offs, (uint32_t)lo[rb], (uint32_t)lo[re]);
  }
  out[2 * c] = a; out[2 * c + 1] = b;
}
// thread per row: rank of the row's partition (the scan of the head flags at its first row) and the row itself
__global__ void __launch_bounds__(256) k_ice_keys(const uint32_t* slot_first, const uint32_t* row_slot, const uint32_t* head_rank, uint64_t n, uint32_t* keys, uint32_t* rows) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = head_rank[slot_first[row_slot[i]]];
  rows[i] = (uint32_t)i;
}
__global__ void __launch_bounds__(256) k_ice_bounds(const uint32_t* keys, uint64_t n, uint64_t n_parts, uint64_t* prow) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (j == 0 || keys[j] != keys[j - 1]) prow[keys[j]] = j;
  if (j == 0) prow[n_parts] = n;
}
struct Rep { int64_t value; uint64_t off; uint32_t len, is_null; };
// warp per partition: its first row's results; span results copied into the representative bytes
__global__ void __launch_bounds__(256) k_ice_reps(TParams T, const uint32_t* perm, const uint64_t* prow, uint64_t n_parts, Rep* reps, uint8_t* bytes) {
  const uint64_t p = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (p >= n_parts) return;
  const uint64_t h = perm[prow[p]];
  for (uint32_t k = 0; k < T.n_fields; k++) {
    const FieldDesc& F = T.f[k];
    const uint64_t at = (uint64_t)k * T.n + h;
    const bool nul = T.nul[at];
    const uint32_t ln = nul ? 0u : T.len[at];
    const uint64_t off = F.span ? F.rep_base + F.rep_off[h] : 0;
    if (lane == 0) reps[p * T.n_fields + k] = Rep{F.span || nul ? 0 : T.val[at], off, F.span ? ln : 0u, nul ? 1u : 0u};
    if (F.span && !nul) {
      const uint8_t* src = base_of(F) + T.val[at];
      for (uint32_t j = lane; j < ln; j += 32) bytes[off + j] = src[j];
    }
  }
}

// ---------------------------------------------------------------- gathers: output item j is source item base + idx[j]
__global__ void __launch_bounds__(256) k_ice_gather_bits(const uint8_t* sv, const uint8_t* sb, const uint32_t* idx, uint64_t base, uint64_t n, uint32_t* dv, uint32_t* db) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool v = false, b = false;
  if (j < n) {
    const uint64_t s = base + idx[j];
    v = bit_at(sv, s);
    if (sb) b = bit_at(sb, s);
  }
  const unsigned vw = __ballot_sync(0xffffffffu, v), bw = __ballot_sync(0xffffffffu, b);
  if ((threadIdx.x & 31) == 0 && j < n) { dv[j >> 5] = vw; if (db) db[j >> 5] = bw; }
}
template <typename T>
__global__ void __launch_bounds__(256) k_ice_gather_fixed(const T* src, const uint32_t* idx, uint64_t base, uint64_t n, T* dst) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) dst[j] = src[base + idx[j]];
}
template <typename OffT>
__global__ void __launch_bounds__(256) k_ice_gather_lens(const OffT* so, const uint32_t* idx, uint64_t base, uint64_t n, uint32_t* lens) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t s = base + idx[j];
  lens[j] = (uint32_t)(so[s + 1] - so[s]);
}
// warp per item: its bytes to their place in the output
template <typename OffT>
__global__ void __launch_bounds__(256) k_ice_gather_bytes(const OffT* so, const uint8_t* sd, const uint32_t* idx, uint64_t base, uint64_t n, const OffT* dof, uint8_t* dd) {
  const uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (j >= n) return;
  const uint64_t s = base + idx[j];
  const uint8_t* src = sd + (uint64_t)so[s];
  uint8_t* dst = dd + (uint64_t)dof[j];
  const uint64_t len = (uint64_t)(so[s + 1] - so[s]);
  for (uint64_t k = lane; k < len; k += 32) dst[k] = src[k];
}
// thread per List row: the source element index of each of its output elements
__global__ void __launch_bounds__(256) k_ice_gather_items(const int32_t* so, const uint32_t* idx, uint64_t base, uint64_t n, const int32_t* dof, uint32_t* items) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t s = base + idx[j];
  const uint32_t first = (uint32_t)so[s], cnt = (uint32_t)(so[s + 1] - so[s]);
  uint32_t* out = items + (uint32_t)dof[j];
  for (uint32_t k = 0; k < cnt; k++) out[k] = first + k;
}

uint32_t grid_of(uint64_t threads) { return (uint32_t)((threads + 255) / 256); }

// which transforms a source type accepts (the header's table)
bool accepts(uint32_t at, uint32_t tr) {
  if (at == ETL_ARROW_UNSUPPORTED || at == ETL_ARROW_LIST) return false;
  const bool flt = at == ETL_ARROW_FLOAT32 || at == ETL_ARROW_FLOAT64;
  switch (tr) {
    case ETL_ICE_VOID: return true;
    case ETL_ICE_IDENTITY: return !flt;
    case ETL_ICE_BUCKET: return !flt && at != ETL_ARROW_BOOLEAN;
    case ETL_ICE_TRUNCATE: return at == ETL_ARROW_INT32 || at == ETL_ARROW_INT64 || at == ETL_ARROW_UTF8 || at == ETL_ARROW_LARGE_BINARY;
    case ETL_ICE_YEAR: case ETL_ICE_MONTH: case ETL_ICE_DAY:
      return at == ETL_ARROW_DATE32 || at == ETL_ARROW_TIMESTAMP_US || at == ETL_ARROW_TIMESTAMPTZ_US;
    case ETL_ICE_HOUR: return at == ETL_ARROW_TIMESTAMP_US || at == ETL_ARROW_TIMESTAMPTZ_US;
    default: return false;
  }
}

}  // namespace

struct etl_iceberg_partitioned {
  etl_arrow_batch* arrow = nullptr;
  uint32_t n_fields = 0;
  uint64_t n_parts = 0;
  uint64_t* dev_rows = nullptr;            // n_parts + 1 partition row offsets on the device
  uint8_t* host = nullptr;                 // pinned: the row offsets | n_parts × n_fields Rep | representative bytes
  uint64_t* rows = nullptr;
  Rep* reps = nullptr;
  uint8_t* rep_bytes = nullptr;
  std::vector<uint32_t> span;              // per field: the result is bytes
};

extern "C" {

void etl_dec_iceberg_partition_free(etl_iceberg_partitioned* r) {
  if (!r) return;
  if (r->arrow) {
    if (r->arrow->dev) cudaFree(r->arrow->dev);
    if (r->arrow->host) cudaFreeHost(r->arrow->host);
    delete r->arrow;
  }
  if (r->dev_rows) cudaFree(r->dev_rows);
  if (r->host) cudaFreeHost(r->host);
  delete r;
}

int etl_dec_iceberg_partition(const etl_arrow_batch* a, const etl_iceberg_partition_field* spec, uint32_t n_fields,
                              uint64_t row_begin, uint64_t row_end, int to_host, etl_iceberg_partitioned** out) {
  if (!a || !spec || !out || !n_fields || n_fields > ETL_ICE_MAX_FIELDS) return ETL_ERR_INVALID_ARG;
  if (row_begin > row_end || row_end > a->n_rows || row_end - row_begin >= 0xFFFFFFFFull) return ETL_ERR_INVALID_ARG;
  for (uint32_t k = 0; k < n_fields; k++) {
    const etl_iceberg_partition_field& f = spec[k];
    if (f.source_column >= a->cols.size() || !accepts(a->cols[f.source_column].arrow_type, f.transform)) return ETL_ERR_INVALID_ARG;
    const bool param = f.transform == ETL_ICE_BUCKET || f.transform == ETL_ICE_TRUNCATE;
    if (param ? (f.param == 0 || f.param > 0x7FFFFFFFu) : f.param != 0) return ETL_ERR_INVALID_ARG;
  }
  const uint64_t n = row_end - row_begin, rb = row_begin;
  const uint32_t n_cols = (uint32_t)a->cols.size();
  cudaStream_t st = cudaStreamPerThread;
  etl_iceberg_partitioned* R = new etl_iceberg_partitioned();
  R->n_fields = n_fields;
  etl_arrow_batch* A = R->arrow = new etl_arrow_batch();
  A->n_rows = n;
  A->first_skipped = a->first_skipped;
  Scratch scratch(st);
  auto fail = [&](int rc) { scratch.release(); cudaStreamSynchronize(st); cudaGetLastError(); etl_dec_iceberg_partition_free(R); return rc; };
  const uint8_t* sd = a->dev;

  // ---- fields
  TParams T{};
  T.n_fields = n_fields; T.rb = rb; T.n = n;
  uint32_t n_span = 0;
  R->span.resize(n_fields);
  for (uint32_t k = 0; k < n_fields; k++) {
    const Col& c = a->cols[spec[k].source_column];
    FieldDesc& F = T.f[k];
    F.arrow_type = c.arrow_type; F.transform = spec[k].transform; F.param = spec[k].param;
    F.validity = sd + c.validity_off;
    F.values = c.values_bytes ? sd + c.values_off : nullptr;
    F.offsets = c.offsets_bytes ? sd + c.offsets_off : nullptr;
    F.data = c.offsets_bytes ? sd + c.data_off : nullptr;
    const bool bytes = c.arrow_type == ETL_ARROW_UTF8 || c.arrow_type == ETL_ARROW_LARGE_BINARY || c.arrow_type == ETL_ARROW_UUID;
    F.span = bytes && (F.transform == ETL_ICE_IDENTITY || F.transform == ETL_ICE_TRUNCATE);
    R->span[k] = F.span;
    n_span += F.span;
  }

  // ---- transform, group, rank (then one sync)
  std::vector<unsigned long long> tot(1 + n_span, 0), sizes(2ull * n_cols, 0);
  uint32_t* perm = nullptr;
  std::vector<uint64_t*> rep_off(n_span, nullptr);
  uint32_t *row_slot = nullptr, *slot_first = nullptr, *head_rank = nullptr;
  if (n) {
    uint64_t slots = 64;
    while (slots < 2 * n) slots <<= 1;
    T.val = (int64_t*)scratch(8 * n * n_fields); T.len = (uint32_t*)scratch(4 * n * n_fields); T.nul = (uint8_t*)scratch(n * n_fields);
    T.hash = (uint64_t*)scratch(8 * n);
    uint32_t* slot_row = (uint32_t*)scratch(4 * slots);
    slot_first = (uint32_t*)scratch(4 * slots);
    row_slot = (uint32_t*)scratch(4 * n);
    uint32_t* head = (uint32_t*)scratch(4 * (n + 1));
    head_rank = (uint32_t*)scratch(4 * (n + 1));
    uint32_t* rep_len = (uint32_t*)scratch(4 * (n + 1) * std::max(n_span, 1u));
    unsigned long long* blk = (unsigned long long*)scratch(8ull * (scan_blocks(n) + 1) * (1 + n_span));
    unsigned long long* d_tot = (unsigned long long*)scratch(8ull * (1 + n_span + 2ull * n_cols));
    SliceDesc* d_slice = (SliceDesc*)scratch(sizeof(SliceDesc) * std::max(n_cols, 1u));
    bool ok = T.val && T.len && T.nul && T.hash && slot_row && slot_first && row_slot && head && head_rank && rep_len && blk && d_tot && d_slice;
    for (uint32_t b = 0; ok && b < n_span; b++) ok = (rep_off[b] = (uint64_t*)scratch(8 * (n + 1))) != nullptr;
    if (!ok) return fail(ETL_ERR_ALLOC);
    std::vector<SliceDesc> slice(n_cols);
    for (uint32_t c = 0; c < n_cols; c++) {
      const Col& col = a->cols[c];
      slice[c] = SliceDesc{nullptr, nullptr, col.arrow_type, 0};
      if (col.offsets_bytes) slice[c].offs = sd + col.offsets_off;
      if (col.arrow_type == ETL_ARROW_LIST && col.child >= 0) {
        const Col& kid = a->kids[(size_t)col.child];
        slice[c].kid_type = kid.arrow_type;
        if (kid.offsets_bytes) slice[c].kid_offs = sd + kid.offsets_off;
      }
    }
    ok = cudaMemsetAsync(slot_row, 0xff, 4 * slots, st) == cudaSuccess && cudaMemsetAsync(slot_first, 0xff, 4 * slots, st) == cudaSuccess &&
         cudaMemsetAsync(d_tot, 0, 8ull * (1 + n_span + 2ull * n_cols), st) == cudaSuccess &&
         cudaMemcpyAsync(d_slice, slice.data(), sizeof(SliceDesc) * n_cols, cudaMemcpyHostToDevice, st) == cudaSuccess;
    if (!ok) return fail(ETL_ERR_CUDA);
    k_ice_transform<<<grid_of(n), 256, 0, st>>>(T);
    k_ice_group<<<grid_of(n), 256, 0, st>>>(T, slot_row, slot_first, (uint32_t)(slots - 1), row_slot);
    k_ice_heads<<<grid_of(n), 256, 0, st>>>(T, slot_first, row_slot, head, rep_len);
    const uint32_t nb = scan_blocks(n) + 1;
    scan_lengths(head, n, blk, d_tot, head_rank, st);
    for (uint32_t b = 0; b < n_span; b++) scan_lengths(rep_len + (uint64_t)b * (n + 1), n, blk + (uint64_t)(b + 1) * nb, d_tot + 1 + b, rep_off[b], st);
    if (n_cols) k_ice_slice<<<(n_cols + 127) / 128, 128, 0, st>>>(d_slice, n_cols, rb, row_end, d_tot + 1 + n_span);
    if (cudaMemcpyAsync(tot.data(), d_tot, 8ull * (1 + n_span), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (n_cols && cudaMemcpyAsync(sizes.data(), d_tot + 1 + n_span, 16ull * n_cols, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaStreamSynchronize(st) != cudaSuccess)
      return fail(ETL_ERR_CUDA);
  }
  const uint64_t P = tot[0];
  R->n_parts = P;

  // ---- output layout: row_rec | per column validity | values or offsets | data | per List child the same
  uint64_t cur = (n * 8 + 63) & ~63ull;
  A->row_rec_off = 0;
  A->cols.resize(n_cols);
  auto place = [&](Col& o, const Col& s, uint64_t items, uint64_t data_bytes) {
    o.arrow_type = s.arrow_type; o.kind = s.kind; o.text = s.text; o.n_items = items;
    if (s.arrow_type == ETL_ARROW_UNSUPPORTED) return;
    o.validity_off = cur; cur += ((items + 31) / 32 * 4 + 63) & ~63ull;
    if (s.arrow_type == ETL_ARROW_BOOLEAN) { o.values_off = cur; o.values_bytes = ((items + 31) / 32 * 4 + 63) & ~63ull; cur += o.values_bytes; }
    else if (etl_arrow::value_width(s.arrow_type)) { o.values_off = cur; o.values_bytes = (items * etl_arrow::value_width(s.arrow_type) + 63) & ~63ull; cur += o.values_bytes; }
    else if (etl_arrow::is_var(s.arrow_type)) {
      o.offsets_off = cur; o.offsets_bytes = ((items + 1) * (s.arrow_type == ETL_ARROW_LARGE_BINARY ? 8 : 4) + 63) & ~63ull; cur += o.offsets_bytes;
      if (s.arrow_type != ETL_ARROW_LIST) { o.data_off = cur; o.data_bytes = data_bytes; cur += (data_bytes + 63) & ~63ull; }
    }
  };
  for (uint32_t c = 0; c < n_cols; c++) {
    const Col& s = a->cols[c];
    Col& o = A->cols[c];
    place(o, s, n, s.arrow_type == ETL_ARROW_LIST ? 0 : sizes[2 * c]);
    o.n_items = 0;
    if (s.arrow_type == ETL_ARROW_LIST && s.child >= 0 && n) {
      Col kid;
      place(kid, a->kids[(size_t)s.child], sizes[2 * c], sizes[2 * c + 1]);
      o.child = (int32_t)A->kids.size();
      A->kids.push_back(kid);
    }
  }
  A->bytes = cur + 64;
  uint64_t rep_total = 0;
  for (uint32_t k = 0, b = 0; k < n_fields; k++) if (T.f[k].span) { T.f[k].rep_off = rep_off[b]; T.f[k].rep_base = rep_total; rep_total += tot[1 + b]; b++; }
  const uint64_t reps_at = 8 * (P + 1), bytes_at = reps_at + sizeof(Rep) * P * n_fields;
  if (cudaMalloc(&A->dev, A->bytes) != cudaSuccess || cudaMalloc(&R->dev_rows, 8 * (P + 1)) != cudaSuccess ||
      cudaHostAlloc((void**)&R->host, bytes_at + rep_total + 1, cudaHostAllocDefault) != cudaSuccess)
    return fail(ETL_ERR_ALLOC);
  R->rows = reinterpret_cast<uint64_t*>(R->host);
  R->reps = reinterpret_cast<Rep*>(R->host + reps_at);
  R->rep_bytes = R->host + bytes_at;
  if (cudaMemsetAsync(R->dev_rows, 0, 8, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  if (!n) {
    if (cudaMemsetAsync(A->dev, 0, A->bytes, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  } else {
    // ---- permutation, partition offsets, representative values
    uint32_t* keys = (uint32_t*)scratch(4 * n);
    uint32_t* keys_out = (uint32_t*)scratch(4 * n);
    uint32_t* rows = (uint32_t*)scratch(4 * n);
    perm = (uint32_t*)scratch(4 * n);
    Rep* d_reps = (Rep*)scratch(sizeof(Rep) * P * n_fields);
    uint8_t* d_rep_bytes = (uint8_t*)scratch(rep_total);
    int end_bit = 1;
    while (end_bit < 32 && (P - 1) >> end_bit) end_bit++;
    size_t temp_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys, keys_out, rows, perm, (uint32_t)n, 0, end_bit, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    void* temp = scratch(temp_bytes);
    if (!keys || !keys_out || !rows || !perm || !d_reps || !d_rep_bytes || !temp) return fail(ETL_ERR_ALLOC);
    k_ice_keys<<<grid_of(n), 256, 0, st>>>(slot_first, row_slot, head_rank, n, keys, rows);
    if (cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_out, rows, perm, (uint32_t)n, 0, end_bit, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    k_ice_bounds<<<grid_of(n), 256, 0, st>>>(keys_out, n, P, R->dev_rows);
    k_ice_reps<<<grid_of(P * 32), 256, 0, st>>>(T, perm, R->dev_rows, P, d_reps, d_rep_bytes);
    if (cudaMemcpyAsync(R->reps, d_reps, sizeof(Rep) * P * n_fields, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (rep_total && cudaMemcpyAsync(R->rep_bytes, d_rep_bytes, rep_total, cudaMemcpyDeviceToHost, st) != cudaSuccess))
      return fail(ETL_ERR_CUDA);

    // ---- gathers
    uint8_t* od = A->dev;
    unsigned long long* d_tot = (unsigned long long*)scratch(8);
    if (!d_tot) return fail(ETL_ERR_ALLOC);
    // one column (or List child) of `items` items, output item j = source item base + idx[j]
    auto gather = [&](const Col& s, const Col& o, const uint32_t* idx, uint64_t base, uint64_t items, auto& self) -> int {
      if (s.arrow_type == ETL_ARROW_UNSUPPORTED || !items) return ETL_OK;
      const uint32_t g = grid_of(items);
      if (cudaMemsetAsync(od + o.validity_off, 0, ((items + 31) / 32 * 4 + 63) & ~63ull, st) != cudaSuccess) return ETL_ERR_CUDA;
      const bool boolean = s.arrow_type == ETL_ARROW_BOOLEAN;
      if (boolean && cudaMemsetAsync(od + o.values_off, 0, o.values_bytes, st) != cudaSuccess) return ETL_ERR_CUDA;
      k_ice_gather_bits<<<g, 256, 0, st>>>(sd + s.validity_off, boolean ? sd + s.values_off : nullptr, idx, base, items,
                                          (uint32_t*)(od + o.validity_off), boolean ? (uint32_t*)(od + o.values_off) : nullptr);
      switch (etl_arrow::value_width(s.arrow_type)) {
        case 4: k_ice_gather_fixed<uint32_t><<<g, 256, 0, st>>>((const uint32_t*)(sd + s.values_off), idx, base, items, (uint32_t*)(od + o.values_off)); return ETL_OK;
        case 8: k_ice_gather_fixed<uint64_t><<<g, 256, 0, st>>>((const uint64_t*)(sd + s.values_off), idx, base, items, (uint64_t*)(od + o.values_off)); return ETL_OK;
        case 16: k_ice_gather_fixed<uint4><<<g, 256, 0, st>>>((const uint4*)(sd + s.values_off), idx, base, items, (uint4*)(od + o.values_off)); return ETL_OK;
        default: break;
      }
      if (!etl_arrow::is_var(s.arrow_type)) return ETL_OK;
      uint32_t* lens = (uint32_t*)scratch(4 * (items + 1));
      unsigned long long* blk = (unsigned long long*)scratch(8ull * (scan_blocks(items) + 1));
      if (!lens || !blk) return ETL_ERR_ALLOC;
      if (s.arrow_type == ETL_ARROW_LARGE_BINARY) {
        const int64_t* so = (const int64_t*)(sd + s.offsets_off);
        int64_t* dof = (int64_t*)(od + o.offsets_off);
        k_ice_gather_lens<int64_t><<<g, 256, 0, st>>>(so, idx, base, items, lens);
        scan_lengths(lens, items, blk, d_tot, dof, st);
        k_ice_gather_bytes<int64_t><<<grid_of(items * 32), 256, 0, st>>>(so, sd + s.data_off, idx, base, items, dof, od + o.data_off);
        return ETL_OK;
      }
      const int32_t* so = (const int32_t*)(sd + s.offsets_off);
      int32_t* dof = (int32_t*)(od + o.offsets_off);
      k_ice_gather_lens<int32_t><<<g, 256, 0, st>>>(so, idx, base, items, lens);
      scan_lengths(lens, items, blk, d_tot, dof, st);
      if (s.arrow_type == ETL_ARROW_UTF8) {
        k_ice_gather_bytes<int32_t><<<grid_of(items * 32), 256, 0, st>>>(so, sd + s.data_off, idx, base, items, dof, od + o.data_off);
        return ETL_OK;
      }
      if (o.child < 0) return ETL_OK;                      // List
      const Col& sk = a->kids[(size_t)s.child];
      const Col& ko = A->kids[(size_t)o.child];
      if (!ko.n_items) return ETL_OK;
      uint32_t* item_idx = (uint32_t*)scratch(4 * ko.n_items);
      if (!item_idx) return ETL_ERR_ALLOC;
      k_ice_gather_items<<<g, 256, 0, st>>>(so, idx, base, items, dof, item_idx);
      return self(sk, ko, item_idx, 0, ko.n_items, self);
    };
    int rc = ETL_OK;
    if (cudaMemsetAsync(od, 0, A->row_rec_off + ((n * 8 + 63) & ~63ull), st) != cudaSuccess) return fail(ETL_ERR_CUDA);
    k_ice_gather_fixed<uint64_t><<<grid_of(n), 256, 0, st>>>((const uint64_t*)(sd + a->row_rec_off), perm, rb, n, (uint64_t*)(od + A->row_rec_off));
    for (uint32_t c = 0; rc == ETL_OK && c < n_cols; c++) rc = gather(a->cols[c], A->cols[c], perm, rb, n, gather);
    if (rc != ETL_OK) return fail(rc);
  }
  if (cudaMemcpyAsync(R->rows, R->dev_rows, 8 * (P + 1), cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  if (to_host) {
    if (cudaHostAlloc((void**)&A->host, A->bytes, cudaHostAllocDefault) != cudaSuccess) return fail(ETL_ERR_ALLOC);
    if (cudaMemcpyAsync(A->host, A->dev, A->bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  }
  scratch.release();
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ETL_ERR_CUDA);
  *out = R;
  return ETL_OK;
}

uint64_t etl_dec_iceberg_partitions(const etl_iceberg_partitioned* r) { return r ? r->n_parts : 0; }
const uint64_t* etl_dec_iceberg_partition_rows(const etl_iceberg_partitioned* r, int host) {
  if (!r) return nullptr;
  return host ? r->rows : r->dev_rows;
}
int etl_dec_iceberg_partition_value(const etl_iceberg_partitioned* r, uint64_t partition, uint32_t field, etl_iceberg_partition_value* out) {
  if (!r || !out || partition >= r->n_parts || field >= r->n_fields) return ETL_ERR_INVALID_ARG;
  const Rep& p = r->reps[partition * r->n_fields + field];
  out->is_null = p.is_null;
  out->len = p.len;
  out->value = p.value;
  out->data = r->span[field] && !p.is_null ? r->rep_bytes + p.off : nullptr;
  return ETL_OK;
}
const etl_arrow_batch* etl_dec_iceberg_partitioned_arrow(const etl_iceberg_partitioned* r) { return r ? r->arrow : nullptr; }

}  // extern "C"
