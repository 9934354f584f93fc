// clickhouse_lz4.cu — the INSERT bodies of the ClickHouse destination, compressed on the device: rows [row_begin,
// row_end) of a RowBinary emit (rowbinary_emit.cu) cut into INSERTs by insert_rows's greedy rule, each body a sequence
// of ClickHouse compressed blocks (LZ4, method 0x82, CityHash128 v1.0.2 checksum) that the shim posts with
// decompress=1.  The byte-level pieces are in clickhouse_lz4.cuh.
//
// Passes (one CUDA stream, three syncs: the cuts, the output size, the end of the call):
//   1. k_cut, one thread: from row_begin, each INSERT's end row by a galloping then binary search over the emit's row
//      offsets (the first row r with off[r] - off[start] >= max_bytes_per_insert, or row_end), the running block count
//      (ceil(bytes / kBlock) per INSERT) as the block base of each INSERT.  (sync: INSERTs, blocks, byte range)
//   2. k_blocks, a thread per block: its INSERT by binary search over the block bases, its first byte; the blocks tile
//      the byte range, so block b is [bstart[b], bstart[b + 1]).
//   3. k_lz4, a warp (CTA) per block: the block is staged into shared memory by one bulk async copy (cp.async.bulk,
//      completion on an mbarrier; the 16-byte aligned window around it), the hash table of positions (u16, 1 <<
//      kHashBits) lives in shared memory.  Each step the lanes hash 32 consecutive positions; a lane's candidate is the
//      nearest lower lane with the same hash (__match_any_sync) or else the table's entry, so matches inside the 32
//      positions (runs, offset 1) are found too.  The lowest lane whose candidate holds the same 4 bytes starts the
//      match (greedy, first match wins); the warp extends it 32 bytes per step with one ballot.  The lanes up to the
//      match (every lane when there is none) enter their positions, the highest lane of each hash writes, so the
//      table, and the output, do not depend on scheduling.  The warp writes each sequence into the block's slot at
//      slot_off(b) + 25; the slot holds lz4_bound(n) bytes.  No match starts within the last 12 bytes of the block or
//      ends within its last 5, and the last sequence is literals only.  Lane 0 writes the 9-byte header.
//   4. k_checksum, a thread per block: CityHash128 v1.0.2 of header + payload, a serial chain over the slot the
//      compressor just wrote, into the slot's first 16 bytes.
//   5. k_len_blocks / k_blk_scan64 / k_offsets (emit_scan.cuh) over the block sizes (25 + payload) → block offsets
//      in the output (sync: total), k_ins_off takes each INSERT's offset from its first block, k_gather (a warp per
//      block) copies the slots into place.
// Slots: block b whose first byte lies u bytes into the range starts at round_up_16(u + u / 255 + 56 b), which leaves
// each block 25 + lz4_bound(n) bytes and aligns the checksum input (slot + 16) for the hash's 8-byte loads.
// Scratch: 16 B per INSERT (+ 16), 16 B per block (+ 24), the slots (range bytes * 256 / 255 + 56 B per block + 32).
// Output: (n_inserts + 1) * 16 B of insert rows and offsets, and the bodies.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "etl_decode.h"
#include "clickhouse_lz4.cuh"
#include "emit_scan.cuh"

using namespace etl_ch;

namespace {

constexpr uint32_t kHashBits = 12;
constexpr uint32_t kStage = kBlock + 32;       // staged window: 15 bytes of alignment head, the block, word-read slack
constexpr uint32_t kSmem = kStage + (2u << kHashBits) + 16;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ uint64_t slot_off(uint64_t u, uint64_t b) { return (u + u / 255u + 56u * b + 15u) & ~15ull; }

// 1. the INSERT cuts and block bases (one thread); res: INSERTs, blocks, off[row_begin], off[row_end]
__global__ void k_cut(const uint64_t* off, uint64_t row_begin, uint64_t row_end, uint64_t max_bytes, uint64_t* ins_rows,
                      uint64_t* blk_base, unsigned long long* res) {
  uint64_t s = row_begin, k = 0, nb = 0;
  while (s < row_end) {
    const uint64_t o0 = off[s];
    uint64_t lo = s, hi = s + 1, step = 1;          // off[lo] - o0 < max; the end is in (lo, hi]
    while (hi < row_end && off[hi] - o0 < max_bytes) { lo = hi; step <<= 1; hi = s + step; }
    if (hi > row_end) hi = row_end;
    while (hi - lo > 1) { const uint64_t m = lo + (hi - lo) / 2; if (off[m] - o0 < max_bytes) lo = m; else hi = m; }
    ins_rows[k] = s;
    blk_base[k] = nb;
    nb += (off[hi] - o0 + kBlock - 1) / kBlock;
    k++;
    s = hi;
  }
  ins_rows[k] = row_end;
  blk_base[k] = nb;
  res[0] = k;
  res[1] = nb;
  res[2] = off[row_begin];
  res[3] = off[row_end];
}

// 2. the first byte of every block (bstart[n_blocks] = off[row_end])
__global__ void k_blocks(const uint64_t* off, const uint64_t* ins_rows, const uint64_t* blk_base, uint64_t n_ins, uint64_t n_blocks,
                         uint64_t* bstart) {
  const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b > n_blocks) return;
  if (b == n_blocks) { bstart[b] = off[ins_rows[n_ins]]; return; }
  uint64_t lo = 0, hi = n_ins - 1;                   // the INSERT: last blk_base <= b
  while (lo < hi) { const uint64_t m = (lo + hi + 1) / 2; if (blk_base[m] <= b) lo = m; else hi = m - 1; }
  bstart[b] = off[ins_rows[lo]] + (b - blk_base[lo]) * kBlock;
}

// ---- mbarrier / bulk-copy primitives (PTX ISA 8.x)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LZ4_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@!p bra LZ4_WAIT;\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// the 4 bytes at p of the staged window (word-aligned loads and a funnel shift)
__device__ __forceinline__ uint32_t rd32(const uint32_t* w, uint32_t p) {
  return __funnelshift_r(w[p >> 2], w[(p >> 2) + 1], (p & 3u) * 8u);
}
__device__ __forceinline__ uint32_t lz4_hash(uint32_t v) { return (v * 2654435761u) >> (32 - kHashBits); }

// 3. a warp per block: LZ4 into the block's slot; csize[b] = 25 + payload
__global__ void __launch_bounds__(32) k_lz4(const uint8_t* data, const uint64_t* bstart, uint8_t* slots, uint32_t* csize) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* stage = smem;
  uint16_t* table = reinterpret_cast<uint16_t*>(smem + kStage);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kStage + (2u << kHashBits));
  const uint32_t lane = threadIdx.x;
  const uint64_t b = blockIdx.x;
  const uint64_t s0 = bstart[b], u = s0 - bstart[0];
  const uint32_t n = (uint32_t)(bstart[b + 1] - s0);
  const uint64_t a0 = s0 & ~15ull;                  // the emit's data is 256-aligned with 64 bytes of slack
  const uint32_t head = (uint32_t)(s0 - a0), win = (head + n + 15u) & ~15u;
  const uint32_t sbar = smem_u32(bar);
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sbar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sbar), "r"(win) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(stage)), "l"(data + a0), "r"(win), "r"(sbar) : "memory");
  }
  for (uint32_t k = lane; k < (1u << kHashBits) / 2; k += 32) reinterpret_cast<uint32_t*>(table)[k] = 0;
  __syncwarp();
  mbar_wait(sbar, 0);
  const uint32_t* words = reinterpret_cast<const uint32_t*>(stage);
  const uint8_t* in = stage + head;
  uint8_t* out = slots + slot_off(u, b);
  uint8_t* pay = out + kHeader;
  const uint32_t lim = n > kMfLimit ? n - kMfLimit : 0;   // a match starts before lim …
  const uint32_t mend = n - kLastLiterals;                // … and ends by mend
  const unsigned below = (1u << lane) - 1u;
  uint32_t ip = 0, anchor = 0, o = 0;
  while (ip < lim) {
    const uint32_t p = ip + lane;
    const bool act = p < lim;
    const uint32_t v = act ? rd32(words, head + p) : 0u;
    const uint32_t h = act ? lz4_hash(v) : 0x80000000u | lane;   // inactive lanes: a group of their own
    const unsigned grp = __match_any_sync(kFull, h);
    const unsigned lower = grp & below;
    const uint32_t cand = lower ? ip + 31u - __clz(lower) : act ? table[h] : 0u;
    const bool m = act && cand < p && p - cand <= 65535u && rd32(words, head + cand) == v;
    const unsigned mb = __ballot_sync(kFull, m);
    const uint32_t f = mb ? __ffs(mb) - 1u : 32u;
    const unsigned ins = __ballot_sync(kFull, act && lane <= f);
    __syncwarp();
    if (((ins >> lane) & 1u) && !(grp & ins & ~(below | (1u << lane)))) table[h] = (uint16_t)p;
    __syncwarp();
    if (!mb) { ip += 32; continue; }
    const uint32_t q = ip + f, c = __shfl_sync(kFull, cand, f);
    uint32_t len = kMinMatch;
    for (;;) {                                            // 32 bytes per step; q + 4 <= mend
      const uint32_t a = q + len + lane;
      const bool eq = a < mend && in[a] == in[c + len + lane];
      const unsigned ne = __ballot_sync(kFull, !eq);
      if (ne) { len += __ffs(ne) - 1u; break; }
      len += 32;
    }
    const uint32_t lit = q - anchor, hl = lz4_lit_header_len(lit);
    if (lane == 0) lz4_lit_header(lit, len, pay + o);
    for (uint32_t k = lane; k < lit; k += 32) pay[o + hl + k] = in[anchor + k];
    o += hl + lit;
    if (lane == 0) lz4_match_tail(q - c, len, pay + o);
    o += 2u + (len - kMinMatch >= 15u ? (len - kMinMatch - 15u) / 255u + 1u : 0u);
    ip = anchor = q + len;
  }
  const uint32_t lit = n - anchor, hl = lz4_lit_header_len(lit);   // the last sequence: literals only
  if (lane == 0) { lz4_lit_header(lit, 0, pay + o); block_header(o + hl + lit, n, out); }
  for (uint32_t k = lane; k < lit; k += 32) pay[o + hl + k] = in[anchor + k];
  o += hl + lit;
  if (lane == 0) csize[b] = kHeader + o;
}

// 4. a thread per block: the checksum
__global__ void __launch_bounds__(128) k_checksum(const uint64_t* bstart, uint64_t n_blocks, uint8_t* slots, const uint32_t* csize) {
  const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  block_checksum(slots + slot_off(bstart[b] - bstart[0], b), csize[b] - kHeader);
}

// 5. INSERT offsets from their first block; a warp per block copies its slot into place
__global__ void k_ins_off(const uint64_t* blk_base, uint64_t n_ins, const uint64_t* boff, uint64_t* ins_off) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k <= n_ins) ins_off[k] = boff[blk_base[k]];
}
__global__ void __launch_bounds__(128) k_gather(const uint64_t* bstart, uint64_t n_blocks, const uint8_t* slots, const uint32_t* csize,
                                                const uint64_t* boff, uint8_t* out) {
  const uint64_t b = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (b >= n_blocks) return;
  const uint32_t lane = threadIdx.x & 31u, len = csize[b];
  const uint8_t* src = slots + slot_off(bstart[b] - bstart[0], b);
  uint8_t* dst = out + boff[b];
  for (uint32_t k = lane; k < len; k += 32) dst[k] = src[k];
}

}  // namespace

struct etl_rowbinary_lz4 {
  uint64_t n_inserts = 0, bytes = 0;
  uint8_t* meta = nullptr;    // device: n_inserts + 1 insert rows | n_inserts + 1 insert offsets
  uint8_t* data = nullptr;    // device: the bodies
  uint8_t* host = nullptr;    // pinned: meta | data (to_host)
};

extern "C" {

int etl_dec_rowbinary_lz4(const etl_rowbinary_batch* rb, uint64_t row_begin, uint64_t row_end, uint64_t max_bytes_per_insert,
                          int to_host, etl_rowbinary_lz4** out) {
  if (!rb || !out || max_bytes_per_insert == 0) return ETL_ERR_INVALID_ARG;
  const uint64_t n_rows = etl_dec_rowbinary_rows(rb), emit_bytes = etl_dec_rowbinary_bytes(rb);
  if (row_begin > row_end || row_end > n_rows) return ETL_ERR_INVALID_ARG;
  const uint64_t* d_off = etl_dec_rowbinary_row_offsets(rb, 0);
  const uint8_t* d_data = etl_dec_rowbinary_data(rb, 0);

  cudaStream_t st = cudaStreamPerThread;
  etl_rowbinary_lz4* Z = new etl_rowbinary_lz4();
  std::vector<void*> scratch;                           // stream-ordered, released on every exit
  auto salloc = [&](uint64_t bytes) -> void* {
    void* p = nullptr;
    if (cudaMallocAsync(&p, bytes + 64, st) != cudaSuccess) return nullptr;
    scratch.push_back(p);
    return p;
  };
  auto fail = [&](int rc) {
    for (void* p : scratch) cudaFreeAsync(p, st);
    cudaStreamSynchronize(st);
    cudaGetLastError();
    etl_dec_rowbinary_lz4_free(Z);
    return rc;
  };
  // 1. cuts: at most one INSERT per row, and every INSERT but the last holds max_bytes_per_insert bytes or more
  const uint64_t ins_bound = std::min<uint64_t>(row_end - row_begin, emit_bytes / max_bytes_per_insert + 1);
  uint64_t* d_ins_rows = (uint64_t*)salloc((ins_bound + 1) * 8);
  uint64_t* d_blk_base = (uint64_t*)salloc((ins_bound + 1) * 8);
  unsigned long long* d_res = (unsigned long long*)salloc(32);
  if (!d_ins_rows || !d_blk_base || !d_res) return fail(ETL_ERR_ALLOC);
  unsigned long long res[4] = {0, 0, 0, 0};            // INSERTs, blocks, off[row_begin], off[row_end]
  k_cut<<<1, 1, 0, st>>>(d_off, row_begin, row_end, max_bytes_per_insert, d_ins_rows, d_blk_base, d_res);
  if (cudaMemcpyAsync(res, d_res, sizeof res, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
    return fail(ETL_ERR_CUDA);
  const uint64_t n_ins = res[0], nb = res[1], range = res[3] - res[2];
  Z->n_inserts = n_ins;
  const uint64_t meta_bytes = (2 * n_ins + 2) * 8;
  if (cudaMalloc(&Z->meta, meta_bytes) != cudaSuccess) { Z->meta = nullptr; return fail(ETL_ERR_ALLOC); }
  uint64_t* ins_off = reinterpret_cast<uint64_t*>(Z->meta) + n_ins + 1;
  if (cudaMemcpyAsync(Z->meta, d_ins_rows, (n_ins + 1) * 8, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return fail(ETL_ERR_CUDA);

  unsigned long long total = 0;
  uint64_t* d_bstart = nullptr; uint8_t* d_slots = nullptr; uint32_t* d_csize = nullptr; uint64_t* d_boff = nullptr;
  if (nb) {
    // 2-4. block table, compression, checksums
    d_bstart = (uint64_t*)salloc((nb + 1) * 8);
    d_csize = (uint32_t*)salloc(nb * 4);
    d_boff = (uint64_t*)salloc((nb + 1) * 8);
    d_slots = (uint8_t*)salloc(range + range / 255 + 56 * nb + 32);
    const uint32_t sb = (uint32_t)((nb + 1023) / 1024);
    unsigned long long* d_sblk = (unsigned long long*)salloc((sb + 1) * 8ull);
    if (!d_bstart || !d_csize || !d_boff || !d_slots || !d_sblk) return fail(ETL_ERR_ALLOC);
    if (cudaFuncSetAttribute(k_lz4, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem) != cudaSuccess) return fail(ETL_ERR_CUDA);
    k_blocks<<<(uint32_t)((nb + 256) / 256), 256, 0, st>>>(d_off, d_ins_rows, d_blk_base, n_ins, nb, d_bstart);
    k_lz4<<<(uint32_t)nb, 32, kSmem, st>>>(d_data, d_bstart, d_slots, d_csize);
    k_checksum<<<(uint32_t)((nb + 127) / 128), 128, 0, st>>>(d_bstart, nb, d_slots, d_csize);
    // 5. block offsets (sync: the output size)
    k_len_blocks<<<sb, 1024, 0, st>>>(d_csize, nb, d_sblk);
    k_blk_scan64<<<1, 1024, 0, st>>>(d_sblk, sb, d_sblk + sb);
    k_offsets<uint64_t><<<sb, 1024, 0, st>>>(d_csize, nb, d_sblk, d_boff);
    k_ins_off<<<(uint32_t)((n_ins + 256) / 256), 256, 0, st>>>(d_blk_base, n_ins, d_boff, ins_off);
    if (cudaMemcpyAsync(&total, d_sblk + sb, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
      return fail(ETL_ERR_CUDA);
  } else if (cudaMemsetAsync(ins_off, 0, (n_ins + 1) * 8, st) != cudaSuccess) {
    return fail(ETL_ERR_CUDA);
  }
  Z->bytes = total;
  if (cudaMalloc(&Z->data, total + 64) != cudaSuccess) { Z->data = nullptr; return fail(ETL_ERR_ALLOC); }
  if (nb) k_gather<<<(uint32_t)((nb * 32 + 127) / 128), 128, 0, st>>>(d_bstart, nb, d_slots, d_csize, d_boff, Z->data);
  if (to_host) {
    if (cudaHostAlloc((void**)&Z->host, meta_bytes + total + 64, cudaHostAllocDefault) != cudaSuccess) { Z->host = nullptr; return fail(ETL_ERR_ALLOC); }
    if (cudaMemcpyAsync(Z->host, Z->meta, meta_bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(Z->host + meta_bytes, Z->data, total, cudaMemcpyDeviceToHost, st) != cudaSuccess) return fail(ETL_ERR_CUDA);
  }
  for (void* p : scratch) cudaFreeAsync(p, st);
  scratch.clear();
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ETL_ERR_CUDA);
  *out = Z;
  return ETL_OK;
}
uint64_t etl_dec_rowbinary_lz4_inserts(const etl_rowbinary_lz4* z) { return z ? z->n_inserts : 0; }
const uint64_t* etl_dec_rowbinary_lz4_insert_rows(const etl_rowbinary_lz4* z, int host) {
  if (!z) return nullptr;
  const uint8_t* base = host ? z->host : z->meta;
  return base ? reinterpret_cast<const uint64_t*>(base) : nullptr;
}
const uint64_t* etl_dec_rowbinary_lz4_insert_offsets(const etl_rowbinary_lz4* z, int host) {
  if (!z) return nullptr;
  const uint8_t* base = host ? z->host : z->meta;
  return base ? reinterpret_cast<const uint64_t*>(base) + z->n_inserts + 1 : nullptr;
}
uint64_t etl_dec_rowbinary_lz4_bytes(const etl_rowbinary_lz4* z) { return z ? z->bytes : 0; }
const uint8_t* etl_dec_rowbinary_lz4_data(const etl_rowbinary_lz4* z, int host) {
  if (!z) return nullptr;
  if (!host) return z->data;
  return z->host ? z->host + (2 * z->n_inserts + 2) * 8 : nullptr;
}
void etl_dec_rowbinary_lz4_free(etl_rowbinary_lz4* z) {
  if (!z) return;
  if (z->meta) cudaFree(z->meta);
  if (z->data) cudaFree(z->data);
  if (z->host) cudaFreeHost(z->host);
  delete z;
}

}  // extern "C"
