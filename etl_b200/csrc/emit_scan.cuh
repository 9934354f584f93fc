// emit_scan.cuh — the row selection and length → offsets kernels shared by the destination emitters (arrow_emit.cu,
// rowbinary_emit.cu).  Each emitter includes it once; the kernels have internal linkage, so every translation unit gets
// its own copy.
//
// Selection: k_sel_count / k_blk_scan / k_sel_scatter turn the records of one schema version into the emit's rows, in
// record order.  The emitter's row rule is the template parameter Rule: a default-constructible functor with
//   __device__ int operator()(const SelParams&, uint64_t r, uint64_t* cell0) const
// that returns kRow (and the first cell of the image that becomes the row), kSkipped for a record the destination
// would reject (the smallest such record is reported through n_rows[1]) or kNotRow.
// Scans: k_len_blocks / k_blk_scan64 / k_offsets turn uint32 lengths into n + 1 exclusive offsets and their total.
#pragma once
#include <stdint.h>

#include "etl_decode.h"

namespace {

constexpr int kSelThreads = 1024;

struct SelParams {
  const uint8_t* rec_kind; const uint8_t* rec_flags; const int32_t* rec_schema; const uint64_t* rec_cell_base;
  uint64_t n_records;
  int32_t schema; uint32_t row_kinds; uint32_t n_cols;
  uint32_t* blk;          // per-block counts → exclusive offsets
  uint64_t* row_cell0;    // out: first cell of the row's image, per selected row
  uint64_t* row_rec;      // out: record index per selected row
  unsigned long long* n_rows;   // [0] rows, [1] first skipped record (UINT64_MAX = none)
};
enum { kNotRow = 0, kRow = 1, kSkipped = 2 };

template <class Rule>
__global__ void __launch_bounds__(kSelThreads) k_sel_count(SelParams S) {
  uint64_t c0;
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int sel = Rule()(S, r, &c0);
  const int c = __syncthreads_count(sel == kRow);
  // record indices of a batch are 32-bit: one min per warp, one atomicMin per warp that has a skipped record
  const unsigned skip = __reduce_min_sync(0xffffffffu, sel == kSkipped ? (unsigned)r : 0xffffffffu);
  if ((threadIdx.x & 31) == 0 && skip != 0xffffffffu) atomicMin(S.n_rows + 1, (unsigned long long)skip);
  if (threadIdx.x == 0) S.blk[blockIdx.x] = (uint32_t)c;
}
__global__ void __launch_bounds__(kSelThreads) k_blk_scan(uint32_t* blk, uint32_t nb, unsigned long long* total) {
  __shared__ uint32_t sh[kSelThreads];
  const uint32_t per = (nb + blockDim.x - 1) / blockDim.x;
  const uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
  uint32_t acc = 0;
  for (uint32_t i = lo; i < hi; i++) acc += blk[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (uint32_t d = 1; d < blockDim.x; d <<= 1) {
    uint32_t v = sh[threadIdx.x];
    if (threadIdx.x >= d) v += sh[threadIdx.x - d];
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  uint32_t run = threadIdx.x ? sh[threadIdx.x - 1] : 0u;
  for (uint32_t i = lo; i < hi; i++) { const uint32_t c = blk[i]; blk[i] = run; run += c; }
  if (threadIdx.x == blockDim.x - 1) *total = sh[blockDim.x - 1];
}
template <class Rule>
__global__ void __launch_bounds__(kSelThreads) k_sel_scatter(SelParams S) {
  __shared__ uint32_t warp_cnt[kSelThreads / 32];
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t c0 = 0;
  const bool sel = Rule()(S, r, &c0) == kRow;
  const unsigned bal = __ballot_sync(0xffffffffu, sel);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) warp_cnt[wid] = __popc(bal);
  __syncthreads();
  uint32_t before = 0;
  for (int k = 0; k < wid; k++) before += warp_cnt[k];
  if (sel) {
    const uint64_t at = (uint64_t)S.blk[blockIdx.x] + before + __popc(bal & ((1u << lane) - 1u));
    S.row_cell0[at] = c0; S.row_rec[at] = r;
  }
}
// COPY rows (etl_dec_copy_decode): every row of the valid prefix is an insert image, row r's cells are r * n_cols + c
__global__ void __launch_bounds__(256) k_copy_sel(uint64_t n_rows, uint32_t n_cols, uint64_t* row_cell0, uint64_t* row_rec) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_rows) { row_cell0[r] = r * n_cols; row_rec[r] = r; }
}

// exclusive scan of lens → int32 / int64 offsets (n + 1 entries): block sums, scan of the sums, final pass
__global__ void __launch_bounds__(1024) k_len_blocks(const uint32_t* lens, uint64_t n, unsigned long long* blk) {
  __shared__ unsigned long long sh[32];
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v = i < n ? lens[i] : 0ull;
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = sh[threadIdx.x];
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    if (threadIdx.x == 0) blk[blockIdx.x] = v;
  }
}
__global__ void __launch_bounds__(1024) k_blk_scan64(unsigned long long* blk, uint32_t nb, unsigned long long* total) {
  __shared__ unsigned long long sh[1024];
  const uint32_t per = (nb + blockDim.x - 1) / blockDim.x;
  const uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
  unsigned long long acc = 0;
  for (uint32_t i = lo; i < hi; i++) acc += blk[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (uint32_t d = 1; d < blockDim.x; d <<= 1) {
    unsigned long long v = sh[threadIdx.x];
    if (threadIdx.x >= d) v += sh[threadIdx.x - d];
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  unsigned long long run = threadIdx.x ? sh[threadIdx.x - 1] : 0ull;
  for (uint32_t i = lo; i < hi; i++) { const unsigned long long c = blk[i]; blk[i] = run; run += c; }
  if (threadIdx.x == blockDim.x - 1) *total = sh[blockDim.x - 1];
}
template <typename OffT>
__global__ void __launch_bounds__(1024) k_offsets(const uint32_t* lens, uint64_t n, const unsigned long long* blk, OffT* offs) {
  __shared__ unsigned long long sh[1024];
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long mine = i < n ? lens[i] : 0ull;
  sh[threadIdx.x] = mine;
  __syncthreads();
  for (uint32_t d = 1; d < blockDim.x; d <<= 1) {
    unsigned long long v = sh[threadIdx.x];
    if (threadIdx.x >= d) v += sh[threadIdx.x - d];
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  const unsigned long long excl = blk[blockIdx.x] + sh[threadIdx.x] - mine;
  if (i < n) offs[i] = (OffT)excl;
  if (i + 1 == n) offs[n] = (OffT)(excl + mine);
}

}  // namespace
