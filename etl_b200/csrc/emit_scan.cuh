// emit_scan.cuh — the row selection and length → offsets kernels shared by the destination emitters, with the host
// steps that launch them (select_rows, scan_lengths) and the emitters' stream-ordered scratch (Scratch).  Each emitter
// includes it once; the kernels have internal linkage, so every translation unit gets its own copy.
//
// Selection: k_sel_count / k_blk_scan / k_sel_scatter turn the records of one schema version into the emit's rows, in
// record order.  The emitter's row rule is the template parameter Rule: a default-constructible functor with
//   __device__ int operator()(const SelParams&, uint64_t r, uint64_t* cell0) const
// that returns kRow (and the first cell of the image that becomes the row), kSkipped for a record the destination
// would reject (the smallest such record is reported through n_rows[1]) or kNotRow.
// Scans: k_len_blocks / k_blk_scan / k_offsets turn uint32 lengths into n + 1 exclusive offsets and their total.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

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
// exclusive scan of nb block sums in place (one CTA of 1024 threads), their total into *total
template <typename T>
__global__ void __launch_bounds__(1024) k_blk_scan(T* blk, uint32_t nb, unsigned long long* total) {
  __shared__ T sh[1024];
  const uint32_t per = (nb + blockDim.x - 1) / blockDim.x;
  const uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
  T acc = 0;
  for (uint32_t i = lo; i < hi; i++) acc += blk[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (uint32_t d = 1; d < blockDim.x; d <<= 1) {
    T v = sh[threadIdx.x];
    if (threadIdx.x >= d) v += sh[threadIdx.x - d];
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  T run = threadIdx.x ? sh[threadIdx.x - 1] : (T)0;
  for (uint32_t i = lo; i < hi; i++) { const T c = blk[i]; blk[i] = run; run += c; }
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

// stream-ordered scratch of one emit: blocks of bytes + 64 (nullptr when the allocation fails), all released by
// release() with cudaFreeAsync on the stream, before the emit's final sync or on a failure path
class Scratch {
 public:
  explicit Scratch(cudaStream_t st) : st_(st) {}
  ~Scratch() { release(); }
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  void* operator()(uint64_t bytes) {
    void* p = nullptr;
    if (cudaMallocAsync(&p, bytes + 64, st_) != cudaSuccess) return nullptr;
    blocks_.push_back(p);
    return p;
  }
  void release() {
    for (void* p : blocks_) cudaFreeAsync(p, st_);
    blocks_.clear();
  }
 private:
  cudaStream_t st_;
  std::vector<void*> blocks_;
};

// blocks of the length scan of n items: blk holds scan_blocks(n) sums
uint32_t scan_blocks(uint64_t n) { return (uint32_t)((n + 1023) / 1024); }
// lens[0, n) → offs[0, n] and their total into *total
template <typename OffT>
void scan_lengths(const uint32_t* lens, uint64_t n, unsigned long long* blk, unsigned long long* total, OffT* offs, cudaStream_t st) {
  const uint32_t nb = scan_blocks(n);
  k_len_blocks<<<nb, 1024, 0, st>>>(lens, n, blk);
  k_blk_scan<unsigned long long><<<1, 1024, 0, st>>>(blk, nb, total);
  k_offsets<OffT><<<nb, 1024, 0, st>>>(lens, n, blk, offs);
}

// the emit's rows.  COPY (copy): rows are the first n_copy records, no sync.  Otherwise the records [0, S.n_records)
// through Rule, then (sync) sel = {rows, first skipped record}; sel is left alone when there is no record.  The caller
// allocates S's buffers and initialises S.n_rows[1] to UINT64_MAX
template <class Rule>
int select_rows(const SelParams& S, bool copy, uint64_t n_copy, cudaStream_t st, unsigned long long sel[2]) {
  if (copy) {
    sel[0] = n_copy;
    if (n_copy) k_copy_sel<<<(uint32_t)((n_copy + 255) / 256), 256, 0, st>>>(n_copy, S.n_cols, S.row_cell0, S.row_rec);
    return ETL_OK;
  }
  const uint32_t nb = (uint32_t)((S.n_records + kSelThreads - 1) / kSelThreads);
  if (!nb) return ETL_OK;
  k_sel_count<Rule><<<nb, kSelThreads, 0, st>>>(S);
  k_blk_scan<uint32_t><<<1, kSelThreads, 0, st>>>(S.blk, nb, S.n_rows);
  k_sel_scatter<Rule><<<nb, kSelThreads, 0, st>>>(S);
  if (cudaMemcpyAsync(sel, S.n_rows, 16, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
    return ETL_ERR_CUDA;
  return ETL_OK;
}

}  // namespace
