// wal_kernels.cuh — sm_90a kernels of the batched pgoutput decode path (launch order):
//
//   k_act_count/scan/scatter  list the anchor segments that contain a frame start (`act`) and those that do
//                       not (`dead`): TOAST-heavy streams leave most segments empty.
//   k_chase   (pass A)  one thread per live segment chases the 'd'+len32 frame chain (only the length fields are
//                       read), the frame counts are scanned in the same launch and every frame's offset is written
//                       in stream order: everything after this pass is record-parallel.
//   k_records (pass B + C1)  one thread per frame: head → element of the stream-state transformer {records, cells,
//                       Begin / Commit effect}; CTA scan + decoupled look-back give every frame the state the apply
//                       loop has when it reaches it (the transformer is associative, so commit_lsn / tx_ordinal are
//                       a scan); writes the record plane, coalesced, and counts the frame shapes.  A totals-only
//                       variant runs first when the plane sizes or the carry-in are not known yet.
//   k_utf8_dead         structure-blind UTF-8 pass over the dead segments (the inside of TOAST-sized values) at HBM
//                       speed: one bit per 128-byte line, "some position in this line breaks the position-local rule".
//   k_bin_scan, k_perm  counting sort of the DML records by frame shape (column layout, op, old-image kind).
//   k_rows, k_heavy, k_fix (pass C2, rows_kernel.cuh)  tuples → rows.
//   k_long_cells        the verdict of every long text cell: interior from the line bitmap, edges validated here.
//
// Reference semantics: apply.rs:1687-2248 (state machine), event.rs:376-979 (tuples → rows),
// text.rs:28-173 (cells).  HBM-bound integer/byte work — no tensor cores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cell_parsers.cuh"
#include "float_parse.cuh"

namespace etl {

constexpr int kIndexThreads = 256;
constexpr int kMaxBins = 4096;         // 16 frame shapes x 256 schema versions (more versions share the last bins)
#ifndef ETL_BIN_TILE
#define ETL_BIN_TILE 16384
#endif
// Records per shape-bin tile at least (bin_tile = max(this, 1024 · n_bins)); a multiple of the k_perm and k_records CTAs
constexpr uint32_t kBinTileMin = ETL_BIN_TILE;
static_assert(kBinTileMin % 1024 == 0, "a shape-bin tile holds whole k_perm / k_records CTAs");

struct ScanSlot;
struct LongCell { uint32_t rec_local, seq; uint64_t soff; uint32_t len, edges; };   // a text cell of ≥ kCoopLen bytes; edges: its head and tail are still to be validated

// ---- stream-state transformer (apply.rs:600-626, 1927-2006) + counters; associative under fold()
struct Summ {
  uint64_t lsn;      // final_lsn of the last Begin (valid if HAS_B)
  uint64_t ord;      // HAS_B: next ordinal after the span; else number of ordinal consumers in the span
  uint64_t n_cells;
  uint32_t n_rec;
  uint32_t flags;    // 1 HAS_B, 2 CLOSED (a Commit follows the last Begin / any Commit if no Begin)
};
constexpr uint32_t S_HAS_B = 1, S_CLOSED = 2;

__host__ __device__ __forceinline__ Summ summ_identity() { return Summ{0, 0, 0, 0, 0}; }
__host__ __device__ __forceinline__ Summ fold(const Summ& a, const Summ& b) {
  Summ r;
  r.n_rec = a.n_rec + b.n_rec;
  r.n_cells = a.n_cells + b.n_cells;
  if (b.flags & S_HAS_B) { r.flags = b.flags; r.lsn = b.lsn; r.ord = b.ord; }
  else {
    r.flags = (a.flags & S_HAS_B) | ((b.flags & S_CLOSED) ? S_CLOSED : (a.flags & S_CLOSED));
    r.lsn = a.lsn;
    r.ord = a.ord + b.ord;
  }
  return r;
}

struct DevSchema {
  uint32_t table_id;
  uint32_t n_cols;
  uint32_t n_ident;
  uint32_t col_base;      // into col_kind / col_flags
  uint64_t effective_off; // stream offset from which this version applies
  uint32_t batch_index;   // index reported in rec_schema
  uint32_t has_heap;      // any numeric / bytea / uuid / array column
  uint32_t layout;        // versions with identical (kind, flags) columns share a layout: the shape bins are keyed by it
  uint32_t _pad;
};

// carry-in of the shard, resident on the device (single GPU: uploaded with the batch scalars; multi-GPU: written
// by k_seam_fold from the all-gathered seam summaries — no host round trip between the index and record passes)
struct DevCarry {
  Summ carry;                  // stream state at the shard's first record
  uint64_t record_index_base;  // global index of the shard's first record
};
// what one rank contributes to the seam all-gather (64 bytes)
struct SeamBlock { Summ total; uint64_t _pad[4]; };


struct DecodeParams {
  const uint8_t* buf;
  uint64_t len;
  const uint64_t* anchors;   // n_anchors + 1 entries (last = len)
  uint32_t n_anchors;
  uint32_t anchor_stride;
  const DevSchema* schemas;  // sorted by (table_id, effective_off)
  uint32_t n_schemas;
  const uint8_t* col_kind;
  const uint8_t* col_flags;  // bit0 nullable, bit1 identity
  // pass A (k_chase): frame offsets in stream order + the scan state of the two single-pass scans
  uint64_t* frame_off;       // offset of frame r (scratch of the context: k_records copies it into the rec_off plane)
  uint64_t frame_cap;        // entries frame_off can hold
  uint32_t* seg_rec_base;    // per live segment: index of its first frame
  unsigned int* n_frames;    // frames (= records) of the batch
  unsigned long long* chase_status;   // k_chase look-back words (zero-initialised once; epochs tell launches apart)
  uint32_t* scan_status;     // k_records look-back words
  struct ScanSlot* scan_slots;
  uint32_t scan_epoch;       // changes with every launch of a scanning kernel
  Summ* chase_summ;          // multi-GPU: per-CTA state aggregates of k_chase (the seam block is their fold)
  unsigned int* chase_done;  // ... and the count of CTAs that have published theirs
  Summ* total;               // [0] = fold of everything (shard seam summary)
  // grouping of the DML records by frame shape within tiles of bin_tile consecutive records (k_records counts,
  // k_bin_scan lays out, k_perm fills); entry (tile, bin) of bin_count / bin_cursor is tile * n_bins + bin
  uint32_t* bin_count; uint32_t* bin_cursor; uint32_t n_bins; uint32_t* perm; unsigned int* perm_len;
  uint32_t bin_tile, n_bin_tiles;
  uint32_t n_batch_schemas;
  uint32_t* rec_flen;               // CopyData length + 1 of every record's frame (k_records → k_rows: sizes the staged window)
  unsigned int* abort_flag;         // ABORT_* bits: the batch does not fit the planes / scratch the host reserved (k_chase, k_records)
  unsigned int* copy_count;         // unchanged-TOAST cells left for k_fix
  uint32_t copy_cols;               // COPY-row decode (copy_kernel.cuh): columns per row; 0 on the replication path
  uint64_t cap_records, cap_cells;  // capacity of the record / cell planes
  uint32_t* line_bad;               // k_utf8_dead: bit l set = line l (128 bytes) holds a UTF-8 rule violation (zeroed per batch)
  uint32_t* dead;                   // segments without a frame start (ascending); n_dead = n_anchors - *n_act
  struct LongCell* long_cells; unsigned int* long_count; uint32_t long_cap;   // text cells spanning whole dead segments
  // carry-in (device resident; valid when pass C runs)
  const DevCarry* dc;
  SeamBlock* seam_send;        // this rank's block (k_records writes it); NULL on a single GPU
  const SeamBlock* seam_all;   // n_ranks blocks after the all-gather
  DevCarry* dc_out;            // = dc, writable (k_seam_fold)
  uint32_t rank, n_ranks;
  Summ host_carry;             // carry-in of the whole (unsharded) stream
  const uint32_t* schema_by_batch;  // batch schema index → position in `schemas`
  // outputs
  uint64_t* rec_off; uint8_t* rec_kind; uint8_t* rec_flags; uint32_t* rec_rel; int32_t* rec_schema;
  uint64_t* rec_start_lsn; uint64_t* rec_commit_lsn; uint64_t* rec_tx_ordinal; uint64_t* rec_cell_base;
  uint32_t* rec_tuple_bytes; uint32_t* rec_heap_hint;
  uint8_t* cell_tag; uint64_t* cell_val; uint32_t* cell_aux;
  uint8_t* heap;
  uint32_t* act;                    // compacted list of the segments that contain a frame start (ascending)
  uint32_t* act_blk;                // per-1024-segment block: count, then exclusive offset
  unsigned int* n_act;              // length of `act` (device scalar: no host round trip)
  unsigned long long* heap_top;     // bump pointer of the heap plane
  unsigned long long* arr_top;      // bump pointer of the array region, relative to arr_base
  uint64_t arr_base;
  unsigned int* heap_overflow;      // set when an array reservation did not fit (host retries with a larger heap)
  uint64_t heap_cap;                // 0 when no schema of the batch has a heap-kind column
  unsigned long long* first_error;  // atomicMin key: rec_index << 24 | seq << 6 | code
  unsigned long long* metrics;      // [0] insert bytes [1] update bytes [2] delete bytes [3] events
  // Relation frames rejected on the host (missing stored schema / unknown columns / malformed)
  const uint64_t* rel_error_off; const uint32_t* rel_error_code; const uint32_t* rel_error_seq; uint32_t n_rel_errors;
};

// ---- big-endian readers on byte-addressed (unaligned) generic pointers
__device__ __forceinline__ uint32_t be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}
__device__ __forceinline__ uint64_t be64(const uint8_t* p) { return ((uint64_t)be32(p) << 32) | be32(p + 4); }
__device__ __forceinline__ uint32_t be16(const uint8_t* p) { return ((uint32_t)p[0] << 8) | (uint32_t)p[1]; }

// error sequencing inside one record (same numbering as the oracle)
constexpr uint32_t SEQ_MALFORMED = 0, SEQ_STATE = 1, SEQ_TABLE = 2, SEQ_OLD_SHAPE = 0x10000, SEQ_NEW_SHAPE = 0x20000;
__device__ __forceinline__ uint32_t seq_old_cell(uint32_t i) { return 0x10001u + i; }
__device__ __forceinline__ uint32_t seq_new_cell(uint32_t i) { return 0x20001u + i; }
__device__ __forceinline__ void report_error(const DecodeParams& P, uint64_t rec_index, uint32_t seq, uint32_t code) {
  unsigned long long key = ((unsigned long long)rec_index << 24) | ((unsigned long long)(seq & 0x3FFFFu) << 6) | (code & 63u);
  atomicMin(P.first_error, key);
}

// schema version for (table_id, frame offset): last entry with that table and effective_off <= off
__device__ __forceinline__ const DevSchema* find_schema(const DecodeParams& P, uint32_t table_id, uint64_t off) {
  int lo = 0, hi = (int)P.n_schemas;  // upper_bound on (table_id, off)
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    const DevSchema& s = P.schemas[mid];
    bool le = (s.table_id < table_id) || (s.table_id == table_id && s.effective_off <= off);
    if (le) lo = mid + 1; else hi = mid;
  }
  if (lo == 0) return nullptr;
  const DevSchema* s = &P.schemas[lo - 1];
  return s->table_id == table_id ? s : nullptr;
}

// ---- frame head: everything the index pass and the emit pass agree on
struct FrameHead {
  uint32_t flen;       // CopyData length field (counts itself)
  uint32_t kind;       // pgoutput tag, 'k' for keepalive, 0 when malformed at the frame level
  uint32_t rel;        // relation id (R/I/U/D), relation count (T)
  uint32_t old_tag;    // 'O' | 'K' | 0 for U/D
  bool malformed;
};
// p points at the frame's 'd'; avail = bytes from p to the end of the stream
__device__ __forceinline__ FrameHead read_head(const uint8_t* p, uint64_t avail) {
  FrameHead h;
  h.kind = 0; h.rel = 0; h.old_tag = 0; h.malformed = true; h.flen = 4;
  if (avail < 5 || p[0] != 'd') { h.flen = (uint32_t)(avail > 0 ? avail - 1 : 0); return h; }
  uint32_t flen = be32(p + 1);
  if (flen < 4 || 1ull + flen > avail) { h.flen = (uint32_t)(avail - 1); return h; }  // chain ends here
  h.flen = flen;
  uint32_t blen = flen - 4;
  if (blen < 1) return h;
  uint32_t t = p[5];
  if (t == 'k') { if (blen < 18) return h; h.kind = 'k'; h.malformed = false; return h; }
  if (t != 'w' || blen < 26) return h;
  uint32_t tag = p[30];
  uint32_t mlen = blen - 26;  // message bytes after the tag
  h.kind = tag;
  switch (tag) {
    case 'B': if (mlen < 20) return h; break;
    case 'C': if (mlen < 25) return h; break;
    case 'R': case 'I': case 'U': case 'D':
      if (mlen < 5) return h;
      h.rel = be32(p + 31);
      if (tag == 'U' || tag == 'D') { uint32_t tt = p[35]; if (tt == 'O' || tt == 'K') h.old_tag = tt; }
      break;
    case 'T': {
      if (mlen < 5) return h;
      int32_t n = (int32_t)be32(p + 31);
      if (n > 0 && (uint64_t)n * 4 > (uint64_t)mlen - 5) return h;
      h.rel = n > 0 ? (uint32_t)n : 0u;
      break;
    }
    case 'O': case 'Y': case 'M': break;
    default: return h;  // unknown tag
  }
  h.malformed = false;
  return h;
}

// The first 36 bytes of a frame as little-endian words aligned to the frame start: ten aligned 4-byte loads and nine
// funnel shifts instead of ~25 byte loads with their shifts and ORs (the byte loads were 12 % of k_records'
// instructions).  The stream is padded, so the loads may run past a short frame.
struct HeadW { uint32_t a[9]; };
__device__ __forceinline__ HeadW load_head_words(const uint8_t* p) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u) * 8u;
  uint32_t x[10];
#pragma unroll
  for (int k = 0; k < 10; k++) x[k] = w[k];
  HeadW H;
#pragma unroll
  for (int k = 0; k < 9; k++) H.a[k] = __funnelshift_r(x[k], x[k + 1], sh);
  return H;
}
template <int I> __device__ __forceinline__ uint32_t hw_u8(const HeadW& H) { return (H.a[I >> 2] >> (8 * (I & 3))) & 0xFFu; }
template <int I> __device__ __forceinline__ uint32_t hw_be32(const HeadW& H) {
  static_assert(I + 4 <= 36, "inside the loaded head");
  const uint32_t v = (I & 3) ? __funnelshift_r(H.a[I >> 2], H.a[(I >> 2) + ((I & 3) ? 1 : 0)], 8 * (I & 3)) : H.a[I >> 2];
  return __byte_perm(v, 0, 0x0123);
}
template <int I> __device__ __forceinline__ uint64_t hw_be64(const HeadW& H) { return ((uint64_t)hw_be32<I>(H) << 32) | hw_be32<I + 4>(H); }
// read_head on the loaded words (same rules, same order)
__device__ __forceinline__ FrameHead read_head_w(const HeadW& H, uint64_t avail) {
  FrameHead h;
  h.kind = 0; h.rel = 0; h.old_tag = 0; h.malformed = true; h.flen = 4;
  if (avail < 5 || hw_u8<0>(H) != 'd') { h.flen = (uint32_t)(avail > 0 ? avail - 1 : 0); return h; }
  const uint32_t flen = hw_be32<1>(H);
  if (flen < 4 || 1ull + flen > avail) { h.flen = (uint32_t)(avail - 1); return h; }  // chain ends here
  h.flen = flen;
  const uint32_t blen = flen - 4;
  if (blen < 1) return h;
  const uint32_t t = hw_u8<5>(H);
  if (t == 'k') { if (blen < 18) return h; h.kind = 'k'; h.malformed = false; return h; }
  if (t != 'w' || blen < 26) return h;
  const uint32_t tag = hw_u8<30>(H);
  const uint32_t mlen = blen - 26;  // message bytes after the tag
  h.kind = tag;
  switch (tag) {
    case 'B': if (mlen < 20) return h; break;
    case 'C': if (mlen < 25) return h; break;
    case 'R': case 'I': case 'U': case 'D':
      if (mlen < 5) return h;
      h.rel = hw_be32<31>(H);
      if (tag == 'U' || tag == 'D') { const uint32_t tt = hw_u8<35>(H); if (tt == 'O' || tt == 'K') h.old_tag = tt; }
      break;
    case 'T': {
      if (mlen < 5) return h;
      const int32_t n = (int32_t)hw_be32<31>(H);
      if (n > 0 && (uint64_t)n * 4 > (uint64_t)mlen - 5) return h;
      h.rel = n > 0 ? (uint32_t)n : 0u;
      break;
    }
    case 'O': case 'Y': case 'M': break;
    default: return h;  // unknown tag
  }
  h.malformed = false;
  return h;
}

// output cells of a frame (depends only on kind / old tag / schema — never on the tuple contents)
__device__ __forceinline__ uint32_t frame_out_cells(const FrameHead& h, const DevSchema* s) {
  switch (h.kind) {
    case 'B': return 2;
    case 'C': return 3;
    case 'T': return 1 + h.rel;
    case 'I': return s ? s->n_cols : 0;
    case 'U': return s ? (s->n_cols + (h.old_tag == 'O' ? s->n_cols : (h.old_tag == 'K' ? s->n_ident : 0))) : 0;
    case 'D': return s ? (h.old_tag == 'O' ? s->n_cols : (h.old_tag == 'K' ? s->n_ident : 0)) : 0;
    default: return 0;
  }
}
__device__ __forceinline__ Summ frame_state_elem(const FrameHead& h, const uint8_t* p) {
  Summ e = summ_identity();
  e.n_rec = 1;
  if (h.malformed) return e;
  switch (h.kind) {
    case 'B': e.flags = S_HAS_B; e.lsn = be64(p + 31); e.ord = 1; break;
    case 'C': e.flags = S_CLOSED; e.ord = 1; break;
    case 'R': case 'I': case 'U': case 'D': case 'T': e.ord = 1; break;
    default: break;
  }
  return e;
}

// heap bytes a text cell of `kind` and length n may need (upper bound; identical in passes A and C)
__device__ __forceinline__ uint32_t cell_heap_bound(uint32_t kind, uint32_t n) {
  switch (kind) {
    case ETL_K_NUMERIC: return numeric_heap_bound(n);
    case ETL_K_BYTES: return bytea_heap_bound(n);
    case ETL_K_UUID: return 16;
    default: return 0;
  }
}

// Walk one TupleData, calling f(col_index, tag, value_ptr, len) per cell. Returns bytes consumed
// or 0 if the tuple runs past `end` / has an unknown cell tag (malformed frame).
template <typename F>
__device__ __forceinline__ uint32_t walk_tuple(const uint8_t* p, const uint8_t* end, int32_t* ncols_out, F&& f) {
  if (p + 2 > end) return 0;
  int32_t n = (int32_t)(int16_t)be16(p);
  if (n < 0) n = 0;
  *ncols_out = n;
  const uint8_t* q = p + 2;
  for (int32_t i = 0; i < n; i++) {
    if (q + 1 > end) return 0;
    uint32_t tag = *q++;
    if (tag == 'n' || tag == 'u') { f(i, tag, q, 0u); continue; }
    if (tag != 't' && tag != 'b') return 0;
    if (q + 4 > end) return 0;
    int32_t l = (int32_t)be32(q);
    q += 4;
    if (l < 0 || (uint64_t)l > (uint64_t)(end - q)) return 0;
    f(i, tag, q, (uint32_t)l);
    q += l;
  }
  return (uint32_t)(q - p);
}

// structure of a DML message body (what LogicalReplicationMessage::parse would reject) + Σ text lengths
__device__ __noinline__ bool dml_structure_ok(const FrameHead& h, const uint8_t* p, unsigned long long* tbytes) {
  const uint8_t* end = p + 1 + h.flen;
  const uint8_t* t = p + 35;
  unsigned long long tb = 0;
  int32_t nc;
  auto count = [&](int32_t, uint32_t tag, const uint8_t*, uint32_t l) { if (tag == 't' || tag == 'b') tb += l; };
  if (t >= end) return false;
  uint32_t tt = *t++;
  if (h.kind == 'I') { if (tt != 'N') return false; }
  else if (h.kind == 'U') {
    if (tt == 'O' || tt == 'K') {
      uint32_t used = walk_tuple(t, end, &nc, count);
      if (!used) return false;
      t += used;
      if (t >= end || *t != 'N') return false;
      t++;
    } else if (tt != 'N') return false;
  } else if (tt != 'O' && tt != 'K') return false;
  if (!walk_tuple(t, end, &nc, count)) return false;
  *tbytes = tb;
  return true;
}
__device__ __forceinline__ const uint8_t* cstr_end(const uint8_t* q, const uint8_t* end) {
  while (q < end && *q) q++;
  return q < end ? q + 1 : nullptr;
}

// ================================================================================================
// pass A0: compaction.  A segment is a thread's unit of work in k_chase; a stream with large
// values (TOAST) leaves most segments without a frame start, and a warp whose 32 segments hold three
// live ones still issues every instruction (the round-1 index pass ran at 2.9 active lanes on C5).  Listing the live
// segments first packs them 32 to a warp.  Empty segments fold as the identity, so the scans are
// unchanged in the compacted index space.
constexpr int kActThreads = 1024;
__device__ __forceinline__ bool seg_live(const DecodeParams& P, uint32_t seg) {
  // anchors are caller data: clamp to the stream, a non-ascending pair is an empty segment
  return seg < P.n_anchors && P.anchors[seg] < min(P.anchors[seg + 1], P.len);
}
__global__ void __launch_bounds__(kActThreads) k_act_count(DecodeParams P) {
  const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = __syncthreads_count(seg_live(P, seg));
  if (threadIdx.x == 0) P.act_blk[blockIdx.x] = (uint32_t)c;
}
__global__ void __launch_bounds__(kActThreads) k_act_scan(DecodeParams P, uint32_t nb) {
  __shared__ uint32_t sh[kActThreads];
  const uint32_t per = (nb + blockDim.x - 1) / blockDim.x;
  const uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
  uint32_t acc = 0;
  for (uint32_t i = lo; i < hi; i++) acc += P.act_blk[i];
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
  for (uint32_t i = lo; i < hi; i++) { const uint32_t c = P.act_blk[i]; P.act_blk[i] = run; run += c; }
  if (threadIdx.x == blockDim.x - 1) *P.n_act = sh[blockDim.x - 1];
}
__global__ void __launch_bounds__(kActThreads) k_act_scatter(DecodeParams P) {
  __shared__ uint32_t warp_cnt[kActThreads / 32];
  const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = seg_live(P, seg);
  const unsigned bal = __ballot_sync(0xffffffffu, live);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) warp_cnt[wid] = __popc(bal);
  __syncthreads();
  uint32_t before = 0;
  for (int k = 0; k < wid; k++) before += warp_cnt[k];
  const uint32_t live_rank = P.act_blk[blockIdx.x] + before + __popc(bal & ((1u << lane) - 1u));   // live segments before this one
  if (live) P.act[live_rank] = seg;
  else if (seg < P.n_anchors) P.dead[seg - live_rank] = seg;
}
// the three steps in one launch for a batch of up to kActSmallSegs segments (the reference's 8 MiB batch has 4096):
// a small batch is bound by the number of dependent launches, not by their work
constexpr uint32_t kActSmallPer = 8, kActSmallSegs = kActThreads * kActSmallPer;
__global__ void __launch_bounds__(kActThreads) k_act_small(DecodeParams P) {
  __shared__ uint32_t wsum[kActThreads / 32];
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const uint32_t seg0 = threadIdx.x * kActSmallPer;
  uint32_t livem = 0;
#pragma unroll
  for (uint32_t i = 0; i < kActSmallPer; i++) if (seg_live(P, seg0 + i)) livem |= 1u << i;
  const uint32_t c = (uint32_t)__popc(livem);
  uint32_t inc = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += up; }
  if (lane == 31u) wsum[wid] = inc;
  __syncthreads();
  uint32_t before = 0, total = 0;
#pragma unroll
  for (uint32_t k = 0; k < kActThreads / 32; k++) { const uint32_t v = wsum[k]; if (k < wid) before += v; total += v; }
  uint32_t rank = before + inc - c;                   // live segments before seg0
#pragma unroll
  for (uint32_t i = 0; i < kActSmallPer; i++) {
    const uint32_t seg = seg0 + i;
    if ((livem >> i) & 1u) P.act[rank++] = seg;
    else if (seg < P.n_anchors) P.dead[seg - rank] = seg;
  }
  if (threadIdx.x == 0) *P.n_act = total;
}

// ================================================================================================
// pass A: frame offsets.  One thread per live segment chases the 'd'+len32 chain of the frames that start in its
// 2 KiB (ONE dependent 8-byte read per hop: nothing of a frame but its length field is looked at), the counts are
// scanned in the same launch (decoupled look-back over the CTAs: a CTA publishes its count, then sums the
// counts of its predecessors), and a second walk over the now cached length fields writes every frame's offset
// into `frame_off` in stream order.  Everything after this pass is record-parallel: one thread per frame, coalesced.
// (Round 1/2a walked the chain twice with the whole per-frame state machine inside the walk — k_index, k_frames:
// 10 serial hops for a 2 KiB segment of 200-byte frames, most of the time of an 8 MiB batch.)
__device__ __forceinline__ Summ ld_summ_cg(const Summ* p) {      // L2 (another CTA wrote it)
  const uint4 a = __ldcg(reinterpret_cast<const uint4*>(p)), b = __ldcg(reinterpret_cast<const uint4*>(p) + 1);
  Summ r;
  r.lsn = ((uint64_t)a.y << 32) | a.x; r.ord = ((uint64_t)a.w << 32) | a.z; r.n_cells = ((uint64_t)b.y << 32) | b.x; r.n_rec = b.z; r.flags = b.w;
  return r;
}
constexpr int kChaseThreads = 256;
constexpr int kChaseKeep = 12;
constexpr uint32_t ABORT_RECORDS = 1u, ABORT_SCRATCH = 2u, ABORT_CELLS = 4u;   // bits of *P.abort_flag
// status word of the count scan: [0,2) state (1 = CTA count, 2 = inclusive prefix), [2,34) value, [34,64) launch epoch
__device__ __forceinline__ unsigned long long chase_word(uint32_t epoch, uint32_t value, uint32_t state) {
  return ((unsigned long long)epoch << 34) | ((unsigned long long)value << 2) | state;
}
// CopyData length of the frame at `pos` under read_head's rules: a chain that cannot continue runs to the end of the stream
__device__ __forceinline__ uint32_t chase_flen(const uint8_t* buf, uint64_t pos, uint64_t len) {
  const uint64_t avail = len - pos;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(buf + (pos & ~3ull));   // the stream is 16-byte aligned and padded
  const uint32_t w0 = w[0], w1 = w[1];
  const uint64_t v = (((uint64_t)w1 << 32) | w0) >> ((uint32_t)(pos & 3u) * 8u);   // bytes pos .. pos+4
  if (avail < 5 || (uint32_t)(v & 0xFFu) != 'd') return (uint32_t)(avail > 0 ? avail - 1 : 0);
  const uint32_t flen = __byte_perm((uint32_t)(v >> 8), 0, 0x0123);
  if (flen < 4 || 1ull + flen > avail) return (uint32_t)(avail - 1);
  return flen;
}
// mode bit 0: count + scan (writes seg_rec_base, n_frames, the abort bits); bit 1: write frame_off (needs seg_rec_base)
// SEAM (a multi-GPU shard, counting): the walk also looks at every frame's head and folds its effect on the stream state
// (Begin / Commit / ordinal consumers — no schema needed); the last CTA to finish folds the CTA aggregates in order and
// writes the shard's seam block, so that the exchange can start without a separate totals pass over the frames.
template <bool SEAM>
__global__ void __launch_bounds__(kChaseThreads) k_chase(DecodeParams P, uint32_t mode) {
  __shared__ uint32_t wsum[kChaseThreads / 32];
  __shared__ uint32_t blk_prefix;
  __shared__ Summ wagg[SEAM ? kChaseThreads / 32 : 1];
  __shared__ uint32_t is_last;
  const uint32_t n_act = *P.n_act;
  const uint32_t n_blocks = (n_act + kChaseThreads - 1) / kChaseThreads;
  if (SEAM && n_blocks == 0u && blockIdx.x == 0 && threadIdx.x == 0 && (mode & 1u) && P.seam_send) {   // no frame starts in this range
    SeamBlock sb; sb.total = summ_identity(); sb._pad[0] = sb._pad[1] = sb._pad[2] = sb._pad[3] = 0;
    *P.seam_send = sb;
  }
  if (blockIdx.x >= n_blocks) return;                 // the grid is sized for a stream with every segment live
  const uint32_t j = blockIdx.x * kChaseThreads + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const bool live = j < n_act;
  uint64_t pos0 = 0, stop = 0;
  if (live) { const uint32_t seg = P.act[j]; pos0 = P.anchors[seg]; stop = min(P.anchors[seg + 1], P.len); }
  uint32_t base = 0;
  // the first kChaseKeep frame starts of the segment stay in registers (16-bit distances from the anchor: a segment is at
  // most 32 KiB), so that segments of up to that many frames are not walked a second time for the write
  uint32_t dd[kChaseKeep / 2];
#pragma unroll
  for (int k = 0; k < kChaseKeep / 2; k++) dd[k] = 0;
  uint32_t count = 0, kept = 0;
  uint64_t pos_keep = pos0;                           // position after the kept frames
  Summ acc = summ_identity();                         // SEAM: fold of this segment's frames (n_cells stays 0: a shard's cells are its own)
  auto flen_at = [&](uint64_t pos) -> uint32_t {
    if (!SEAM) return chase_flen(P.buf, pos, P.len);
    const HeadW H = load_head_words(P.buf + pos);
    const FrameHead h = read_head_w(H, P.len - pos);
    acc = fold(acc, frame_state_elem(h, P.buf + pos));
    return h.flen;
  };
  if (mode & 1u) {
#pragma unroll
    for (int k = 0; k < kChaseKeep; k++)
      if (pos_keep < stop && pos_keep - pos0 < 65536ull && kept == (uint32_t)k) {   // (anchors are caller data: a "segment" may be longer than a stride)
        dd[k >> 1] |= (uint32_t)(pos_keep - pos0) << (16 * (k & 1));
        kept++;
        pos_keep += 1ull + flen_at(pos_keep);
      }
    count = kept;
    for (uint64_t pos = pos_keep; pos < stop; count++) pos += 1ull + flen_at(pos);
    uint32_t inc = count;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += up; }
    if (lane == 31u) wsum[wid] = inc;
    __syncthreads();
    uint32_t before = 0, blk_total = 0;
#pragma unroll
    for (uint32_t k = 0; k < kChaseThreads / 32; k++) { const uint32_t c = wsum[k]; if (k < wid) before += c; blk_total += c; }
    if (wid == 0) {
      volatile unsigned long long* status = P.chase_status;
      const uint32_t ep = P.scan_epoch;
      if (lane == 0) status[blockIdx.x] = chase_word(ep, blk_total, blockIdx.x == 0 ? 2u : 1u);
      uint32_t prefix = 0;
      for (int hi = (int)blockIdx.x - 1; hi >= 0; hi -= 32) {
        const int idx = hi - (int)lane;
        unsigned long long sw = chase_word(ep, 0u, 2u);            // before the first CTA: an inclusive prefix of 0
        if (idx >= 0) do { sw = status[idx]; } while ((uint32_t)(sw >> 34) != ep || (sw & 3ull) == 0ull);
        const unsigned incl = __ballot_sync(0xffffffffu, (sw & 3ull) == 2ull);
        const uint32_t last = incl ? (uint32_t)__ffs(incl) - 1u : 32u;   // nearest predecessor that already knows its inclusive prefix
        uint32_t v = lane <= last ? (uint32_t)(sw >> 2) : 0u;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
        prefix += __shfl_sync(0xffffffffu, v, 0);
        if (incl) break;
      }
      if (lane == 0) {
        blk_prefix = prefix;
        const uint32_t total = prefix + blk_total;
        if (blockIdx.x) status[blockIdx.x] = chase_word(ep, total, 2u);
        if (blockIdx.x == n_blocks - 1u) {
          *P.n_frames = total;
          // sizes were guessed from earlier batches: record planes too small → pass C is re-run with exact sizes;
          // offset scratch too small → nothing after this kernel can run
          *P.abort_flag = ((uint64_t)total > P.cap_records ? ABORT_RECORDS : 0u) | ((uint64_t)total > P.frame_cap ? ABORT_SCRATCH : 0u);
        }
      }
    }
    __syncthreads();
    base = blk_prefix + before + (inc - count);
    if (live) P.seg_rec_base[j] = base;
    if (SEAM) {
      // ordered fold of the CTA's segments (thread order = stream order), published for the last CTA
      Summ v = acc;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        Summ later;
        later.lsn = __shfl_down_sync(0xffffffffu, v.lsn, d); later.ord = __shfl_down_sync(0xffffffffu, v.ord, d);
        later.n_cells = 0; later.n_rec = __shfl_down_sync(0xffffffffu, v.n_rec, d); later.flags = __shfl_down_sync(0xffffffffu, v.flags, d);
        if (lane + (uint32_t)d < 32u) v = fold(v, later);
      }
      if (lane == 0) wagg[wid] = v;
      __syncthreads();
      if (threadIdx.x == 0) {
        Summ a = wagg[0];
#pragma unroll
        for (uint32_t k = 1; k < kChaseThreads / 32; k++) a = fold(a, wagg[k]);
        P.chase_summ[blockIdx.x] = a;
        __threadfence();
        is_last = atomicAdd(P.chase_done, 1u) == n_blocks - 1u ? 1u : 0u;
      }
      __syncthreads();
      if (is_last && wid == 0) {                      // every CTA has published its aggregate (and the frame count is final)
        __threadfence();
        Summ total = summ_identity();
        for (uint32_t b0 = 0; b0 < n_blocks; b0 += 32u) {
          Summ w = b0 + lane < n_blocks ? ld_summ_cg(&P.chase_summ[b0 + lane]) : summ_identity();
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            Summ later;
            later.lsn = __shfl_down_sync(0xffffffffu, w.lsn, d); later.ord = __shfl_down_sync(0xffffffffu, w.ord, d);
            later.n_cells = 0; later.n_rec = __shfl_down_sync(0xffffffffu, w.n_rec, d); later.flags = __shfl_down_sync(0xffffffffu, w.flags, d);
            if (lane + (uint32_t)d < 32u) w = fold(w, later);
          }
          total = fold(total, w);                     // lane 0 holds the window's fold
        }
        if (lane == 0 && P.seam_send) {
          SeamBlock sb; sb.total = total; sb._pad[0] = sb._pad[1] = sb._pad[2] = sb._pad[3] = 0;
          if (*reinterpret_cast<volatile unsigned int*>(P.abort_flag) & ABORT_SCRATCH) sb.total.flags |= 0x80000000u;   // offsets missing: every rank starts over
          *P.seam_send = sb;
        }
      }
    }
  } else if (live) base = P.seg_rec_base[j];
  if ((mode & 2u) && live) {
    uint64_t k = base, pos = pos0;
    if (mode & 1u) {
#pragma unroll
      for (int i = 0; i < kChaseKeep; i++)
        if ((uint32_t)i < kept && k + i < P.frame_cap) P.frame_off[k + i] = pos0 + ((dd[i >> 1] >> (16 * (i & 1))) & 0xFFFFu);
      k += kept;
      pos = pos_keep;
    }
    for (; pos < stop; k++) {
      if (k < P.frame_cap) P.frame_off[k] = pos;
      pos += 1ull + chase_flen(P.buf, pos, P.len);
    }
  }
}

// multi-GPU: fold the seam summaries of the ranks before this one into the carry-in and the record-index base
// (apply.rs:600-626: the state transformer is associative, so a shard's effect on the stream state is its Summ)
__global__ void k_seam_fold(DecodeParams P) {
  if (threadIdx.x || blockIdx.x) return;
  Summ c = P.host_carry;
  uint64_t base = 0;
  for (uint32_t r = 0; r < P.rank; r++) { c = fold(c, P.seam_all[r].total); base += P.seam_all[r].total.n_rec; }
  c.n_rec = 0; c.n_cells = 0;                          // the planes are this rank's own: only the stream state carries over
  DevCarry d; d.carry = c; d.record_index_base = base;
  *P.dc_out = d;
}

// ================================================================================================
// helpers shared by the pass C kernels
// unaligned little-endian 8-byte load built from aligned 32-bit words (works on the shared window
// and on global memory; may touch up to 3 bytes before and 11 after p — buffers are padded)
__device__ __forceinline__ uint64_t ld64u(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(a & 3u) * 8u;
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
  return ((uint64_t)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
}
__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__device__ __forceinline__ uint64_t bswap64(uint64_t v) { return ((uint64_t)bswap32((uint32_t)v) << 32) | bswap32((uint32_t)(v >> 32)); }

}  // namespace etl
#include "utf8.cuh"         // has_high_bits, utf8_range_bad
#include "array_parse.cuh"   // parse_text_cell_impl, parse_text_cell, parse_array_cell / parse_array_any
namespace etl {

__device__ __forceinline__ void put_cell(const DecodeParams& P, uint64_t idx, uint32_t tag, uint64_t val, uint32_t aux) {
  P.cell_tag[idx] = (uint8_t)tag; P.cell_val[idx] = val; P.cell_aux[idx] = aux;
}
constexpr int kWideLen = 96;     // text cells at least this long are validated with 16-byte loads
constexpr int kCoopLen = 512;    // ... these by the whole warp; the part that covers whole dead segments by k_utf8_dead
// Structure-blind UTF-8 pass.  The position-local rule (utf8_step_bad) needs only the three preceding
// bytes, so the verdict for position i of a cell is the verdict for stream position a+i whenever the
// three predecessors lie inside the cell.  A segment without a frame start lies inside one frame; the
// segments that lie inside one text cell are what k_long_cells asks about.  One warp per dead segment, 2 KiB
// (4 coalesced 16-byte loads per lane) per pass; the bitmap is written only where a violation is found.
// Short-lived CTAs (a warp takes kDeadSegsPerWarp consecutive dead segments and retires): the pass runs on a low-priority
// side stream underneath latency-bound kernels, and a persistent grid would sit on every SM's thread slots until it is
// done — k_bin_scan / k_perm waited for a slot behind it (round-2 sweep).  The grid is sized for "every segment dead".
constexpr uint32_t kDeadSegsPerWarp = 4;
// Work item i of the dead-segment pass = 2 KiB pass (i % ppseg) of dead segment (i / ppseg), ppseg = passes per segment.
// The verdict of one lane's 64 bytes [off, off + 64) of a dead-segment item that ends at s1: x = the four 16-byte chunks,
// pw = the word before them.  Sets the line bits of the item (two lanes per 128-byte line) — all lanes of the warp call it.
__device__ __forceinline__ void utf8_dead_verdict(const DecodeParams& P, const uint4 (&x)[4], uint32_t pw, uint64_t off, uint64_t s1, uint32_t lane) {
  bool bad = false;
  uint32_t prev = pw;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint32_t h = x[k].x | x[k].y | x[k].z | x[k].w;
    if ((h & 0x80808080u) | (prev & 0x80808000u)) {           // high bits here or in the three bytes before
      const uint64_t o = off + 16ull * k;
      if (o < s1) bad |= !utf8_chunk_valid_at(P.buf, P.len, o, o + 16ull < P.len ? o + 16ull : P.len);
    }
    prev = x[k].w;
  }
  // two lanes per 128-byte line, 16 lines per item: bit m = line m holds a violation
  unsigned bal = __ballot_sync(0xffffffffu, bad);
  if (bal) {
    bal = (bal | (bal >> 1)) & 0x55555555u;
    bal = (bal | (bal >> 1)) & 0x33333333u; bal = (bal | (bal >> 2)) & 0x0F0F0F0Fu;
    bal = (bal | (bal >> 4)) & 0x00FF00FFu; bal = (bal | (bal >> 8)) & 0x0000FFFFu;
    const uint64_t base = off - (uint64_t)lane * 64ull;     // a multiple of min(stride, 2048): the bits stay inside one word
    if (lane == 0) atomicOr(&P.line_bad[(base >> 7) >> 5], bal << ((base >> 7) & 31u));
  }
}
// One item per warp step: every lane owns 64 contiguous bytes (half a 128-byte line), four 16-byte loads in flight before the
// first byte is looked at; the three bytes before a lane's first chunk come from one 4-byte load that hits L1 — no shuffles
// (round 1 paid three __shfl per 16 bytes).  Measured: 4 items (16 loads) per lane cost 102 registers and a quarter of the
// warps, and the pass was slower on C5.
__device__ __forceinline__ void utf8_dead_items(const DecodeParams& P, uint32_t it, uint32_t n_items, uint32_t ppseg, uint32_t lane) {
  uint4 x[4];
  uint32_t pw = 0;
  uint64_t off = 0, s1 = 0;
  if (it < n_items) {
    const uint64_t seg0 = (uint64_t)P.dead[it / ppseg] * P.anchor_stride;
    const uint64_t base = seg0 + (uint64_t)(it % ppseg) * 2048ull;
    const uint64_t e = seg0 + P.anchor_stride < P.len ? seg0 + P.anchor_stride : P.len;
    s1 = base < e ? e : 0;
    off = base + (uint64_t)lane * 64ull;
  }
#pragma unroll
  for (int k = 0; k < 4; k++)
    x[k] = off + 16ull * k < s1 ? *reinterpret_cast<const uint4*>(P.buf + off + 16ull * k) : make_uint4(0, 0, 0, 0);   // +64 bytes of padding are readable
  if (off >= 4 && off < s1) pw = *reinterpret_cast<const uint32_t*>(P.buf + off - 4);   // last word before the lane's bytes
  utf8_dead_verdict(P, x, pw, off, s1, lane);
}
__device__ __forceinline__ uint32_t dead_ppseg(const DecodeParams& P) { return P.anchor_stride > 2048u ? P.anchor_stride / 2048u : 1u; }
__global__ void __launch_bounds__(256) k_utf8_dead(DecodeParams P) {
  const uint32_t ppseg = dead_ppseg(P);
  const uint32_t n_items = (P.n_anchors - *P.n_act) * ppseg;
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;      // warp w: items [w * kDeadSegsPerWarp, +kDeadSegsPerWarp)
  for (uint32_t it = w * kDeadSegsPerWarp; it < min(n_items, (w + 1u) * kDeadSegsPerWarp); it++)
    utf8_dead_items(P, it, min(n_items, (w + 1u) * kDeadSegsPerWarp), ppseg, threadIdx.x & 31u);
}
// any flagged line in [l0, l1)?  One bitmap word per lane and step (a 64 KiB value spans 16 words: a single lane
// testing them one after the other was a chain of 16 dependent-by-branch loads per cell)
__device__ __forceinline__ bool lines_any_bad(const uint32_t* bm, uint64_t l0, uint64_t l1, uint32_t lane) {
  const uint64_t w0 = l0 >> 5, w1 = (l1 - 1) >> 5;
  bool bad = false;
  for (uint64_t w = w0 + lane; w <= w1; w += 32u) {
    uint32_t m = 0xFFFFFFFFu;
    if (w == w0) m &= 0xFFFFFFFFu << (l0 & 31);
    if (w == w1 && (l1 & 31)) m &= (1u << (l1 & 31)) - 1u;
    bad = bad || (bm[w] & m) != 0u;
  }
  return bad;
}
// One warp per listed long cell, after the dead-segment pass has joined: the part of the cell that covers whole
// dead segments is judged from the line bitmap; head and tail (up to a segment each) are validated here when k_rows
// deferred them (text columns) — four 16-byte loads in flight per lane, enough warps to hide the latency.
__global__ void __launch_bounds__(256) k_long_cells(DecodeParams P) {
  if (*P.abort_flag) return;
  const uint32_t n = min(*P.long_count, P.long_cap);
  const uint32_t lane = threadIdx.x & 31u, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n; e += nwarps) {
    const LongCell c = P.long_cells[e];
    const uint64_t cb = c.soff + c.len;
    const uint64_t S0 = (c.soff + 3ull + P.anchor_stride - 1ull) & ~(uint64_t)(P.anchor_stride - 1u), S1 = cb & ~(uint64_t)(P.anchor_stride - 1u);
    bool bad = false;
    if (S0 < S1) {
      bad = lines_any_bad(P.line_bad, S0 >> 7, S1 >> 7, lane);
      if (c.edges) {                                     // head on lanes 0-15, tail on lanes 16-31: one latency chain, not two
        const bool tail = lane >= 16u;
        // a cell that ends on a boundary keeps its last byte in the tail: a sequence left open at the end of the interior
        // is a violation only past the cell's end, which the bitmap does not cover
        const uint32_t t0 = min((uint32_t)(S1 - c.soff), c.len - 1u);
        bad |= utf8_range_bad(P.buf + c.soff, c.len, tail ? t0 : 0u, tail ? c.len : (uint32_t)(S0 - c.soff), lane & 15u, 16u);
      }
    } else if (c.edges) bad = utf8_range_bad(P.buf + c.soff, c.len, 0u, c.len, lane, 32u);
    if (__any_sync(0xffffffffu, bad) && lane == 0) report_error(P, P.dc->record_index_base + c.rec_local, c.seq, ETL_E_UTF8);
  }
}
// out of line: cold (an oversize cell just below the warp-cooperative threshold)
__device__ __noinline__ bool utf8_medium_bad(const uint8_t* cell, uint32_t len) { return utf8_range_bad(cell, len, 0, len, 0, 1); }


// ================================================================================================
// Shape bins.  A warp of k_rows is fastest when its 32 records have the same frame shape (column layout,
// operation, old-image kind): wire cell i is then the same column for every lane and one parser runs for
// all of them.  Output positions are fixed by the scan, so records can be walked in any order: k_records
// histograms the shapes, k_bin_scan lays the bins out (each padded to a whole warp), k_perm writes the
// record indices bin by bin, and k_rows thread t walks record perm[t].  Schema versions with identical
// columns share a layout (a table whose Relation is re-sent keeps its bins); a batch with more layouts
// than bins shares the last 16 bins, whose warps then hold mixed shapes (k_rows handles that per lane).
// The records are binned within tiles of P.bin_tile consecutive records, tile after tile: the k_rows CTAs that
// are resident together then read a narrow band of the stream and can finish each sector of the record and cell planes
// while it is in L2 (bins over the whole batch scattered every warp's frames and plane writes over all of it).
__device__ __forceinline__ uint32_t walk_bin(const DecodeParams& P, uint32_t layout, uint32_t kind, uint32_t rflags) {
  const uint32_t b = (layout << 4) | (kind == 'I' ? 0u : (kind == 'U' ? 4u : 8u)) | (rflags & 3u);
  return b < P.n_bins ? b : P.n_bins - 16u + (b & 15u);
}
// Exclusive scan of the warp-padded counts in (tile, bin) order.  bin_cursor ← the bin's start, bin_count ← the end of
// its records: k_perm writes the padding lanes behind them.
__global__ void __launch_bounds__(1024) k_bin_scan(DecodeParams P) {
  __shared__ uint32_t sh[1024];
  if (*P.abort_flag) return;
  const uint32_t n = P.n_bins * P.n_bin_tiles;
  const uint32_t per = (n + 1023u) / 1024u;
  const uint32_t lo = threadIdx.x * per, hi = min(lo + per, n);
  uint32_t acc = 0;
  for (uint32_t i = lo; i < hi; i++) acc += (P.bin_count[i] + 31u) & ~31u;
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (uint32_t d = 1; d < 1024; d <<= 1) {
    uint32_t v = sh[threadIdx.x];
    if (threadIdx.x >= d) v += sh[threadIdx.x - d];
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  uint32_t run = threadIdx.x ? sh[threadIdx.x - 1] : 0u;
  for (uint32_t i = lo; i < hi; i++) {
    const uint32_t c = P.bin_count[i];
    P.bin_cursor[i] = run;
    P.bin_count[i] = run + c;
    run += (c + 31u) & ~31u;
  }
  if (threadIdx.x == 1023) *P.perm_len = sh[1023];
}
// k_perm: CTA-local counting first (shared-memory histogram), then ONE global atomic per occupied bin per CTA.
// (Round 1 issued one global atomic per bin per WARP: a single-table stream has ~8 occupied bins, so 75 k warps
// queued on 8 addresses, a visible cost for what is a 10 MB permutation.)
constexpr int kPermThreads = 1024;
__global__ void __launch_bounds__(kPermThreads) k_perm(DecodeParams P) {
  __shared__ uint32_t hist[kMaxBins];                 // count of the CTA's records per bin, then the CTA's base in the bin
  if (*P.abort_flag) return;
  const uint64_t n_rec = P.total[0].n_rec;
  if ((uint64_t)blockIdx.x * blockDim.x >= n_rec) return;
  const uint32_t tile_bins = (uint32_t)((uint64_t)blockIdx.x * kPermThreads / P.bin_tile) * P.n_bins;
  for (uint32_t i = threadIdx.x; i < P.n_bins; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  bool dml = false;
  uint32_t bin = 0, local = 0;
  if (r < n_rec) {
    const uint32_t kind = P.rec_kind[r];
    const int32_t sc = P.rec_schema[r];
    if ((kind == 'I' || kind == 'U' || kind == 'D') && sc >= 0) { dml = true; bin = walk_bin(P, P.schemas[P.schema_by_batch[sc]].layout, kind, P.rec_flags[r]); }
  }
  const unsigned vm = __ballot_sync(0xffffffffu, dml);
  if (dml) {                                          // one shared-memory atomic per bin per warp
    const unsigned mask = __match_any_sync(vm, bin);
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(&hist[bin], (uint32_t)__popc(mask));
    base = __shfl_sync(mask, base, leader);
    local = base + __popc(mask & ((1u << lane) - 1u));
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < P.n_bins; i += blockDim.x) {
    const uint32_t c = hist[i];
    if (!c) continue;
    const uint32_t at = atomicAdd(&P.bin_cursor[tile_bins + i], c), end = at + c;
    hist[i] = at;
    if (end == P.bin_count[tile_bins + i])            // the bin's last records: its padding lanes follow them
      for (uint32_t k = end; k & 31u; k++) P.perm[k] = 0xFFFFFFFFu;
  }
  __syncthreads();
  if (dml) P.perm[hist[bin] + local] = (uint32_t)r;
}

// ================================================================================================
// pass B + C1: records.  One THREAD per frame (offsets from k_chase), 256 consecutive frames per CTA.  Every thread
// reads its frame head and forms the frame's element of the stream-state transformer {records, cells, Begin / Commit
// effect} (apply.rs:600-626, 1927-2006: associative, so commit_lsn / tx_ordinal / "inside a transaction" are a scan);
// the CTA scans its 256 elements, publishes the aggregate and obtains its exclusive prefix from its predecessors in the
// same launch (decoupled look-back with an ORDERED fold: the transformer does not commute).  With the prefix every
// thread holds exactly the state the reference's apply loop has when it reaches that message (apply.rs:1687-2248),
// and writes the record plane — consecutive records from consecutive lanes — plus the cells of Begin / Commit /
// Truncate, and counts the frame shapes for k_perm.
//   FULL = false: totals only (P.total, the seam block, the cells-overflow bit) — first batch (plane sizes unknown),
//                 multi-GPU shards (the carry-in arrives through the seam exchange after this pass).
#ifndef ETL_REC_THREADS
#define ETL_REC_THREADS 512
#endif
// Records per CTA, one thread each.  The look-back chain advances one window of 32 CTAs per L2 round trip (with the
// fold): with 256 records per CTA that alone capped the pass on every workload (ncu: a third of the samples at the
// barrier behind the look-back warp).
constexpr int kRecThreads = ETL_REC_THREADS;
static_assert(1024 % kRecThreads == 0, "a shape-bin tile holds whole k_records CTAs");
constexpr int kRecCtaThreads = kRecThreads + 32;      // + the look-back warp
struct ScanSlot { Summ aggr; Summ incl; };
#define SUMM_SHFL(dst, src, fn, arg)                                                                     \
  do {                                                                                                    \
    (dst).lsn = fn(0xffffffffu, (src).lsn, arg); (dst).ord = fn(0xffffffffu, (src).ord, arg);             \
    (dst).n_cells = fn(0xffffffffu, (src).n_cells, arg); (dst).n_rec = fn(0xffffffffu, (src).n_rec, arg); \
    (dst).flags = fn(0xffffffffu, (src).flags, arg);                                                      \
  } while (0)
template <bool FULL>
__global__ void __launch_bounds__(kRecCtaThreads, kRecThreads >= 512 ? 2 : 4) k_records(DecodeParams P) {
  __shared__ Summ wtot[kRecThreads / 32];
  __shared__ Summ blk_excl_sh;
  __shared__ uint32_t hist[FULL ? kMaxBins : 1];     // frame shapes of the CTA's DML records
  {
    const uint32_t ab = *P.abort_flag;               // RECORDS / SCRATCH: set by k_chase, before this launch
    if (ab & ABORT_SCRATCH) {                        // offsets are missing: no totals.  A shard says so in its seam block
      if (!FULL && blockIdx.x == 0 && threadIdx.x == 0 && P.seam_send) {
        SeamBlock sb; sb.total = summ_identity(); sb.total.flags = 0x80000000u; sb._pad[0] = sb._pad[1] = sb._pad[2] = sb._pad[3] = 0;
        *P.seam_send = sb;
      }
      return;
    }
    if (FULL && (ab & ABORT_RECORDS)) return;
  }
  const uint32_t n_rec = *P.n_frames;
  const uint32_t n_blocks = (n_rec + kRecThreads - 1) / kRecThreads;
  if (n_rec == 0) {                                  // a batch without frames: the totals are the identity
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      P.total[0] = summ_identity();
      if (FULL && P.rec_cell_base) P.rec_cell_base[0] = 0;
      if (P.seam_send) { SeamBlock sb; sb.total = summ_identity(); sb._pad[0] = sb._pad[1] = sb._pad[2] = sb._pad[3] = 0; *P.seam_send = sb; }
    }
    return;
  }
  if (blockIdx.x >= n_blocks) return;                // the grid is sized for the capacity of the planes
  if (FULL) { for (uint32_t i = threadIdx.x; i < P.n_bins; i += blockDim.x) hist[i] = 0; }
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const bool lb_warp = wid == kRecThreads / 32;      // the last warp holds no records: it looks back while the others read their heads
  const uint32_t r = blockIdx.x * kRecThreads + threadIdx.x;
  const bool live = !lb_warp && r < n_rec;
  volatile uint32_t* const status = P.scan_status;
  const uint32_t ep = P.scan_epoch << 2;
  ScanSlot* const slots = P.scan_slots;
  uint64_t pos = 0;
  HeadW H;
#pragma unroll
  for (int k = 0; k < 9; k++) H.a[k] = 0;
  FrameHead h;
  h.kind = 0; h.rel = 0; h.old_tag = 0; h.malformed = true; h.flen = 4;
  const DevSchema* s = nullptr;
  Summ ex = summ_identity(), wpre = summ_identity();
  if (lb_warp) {
    // ---- exclusive prefix of the CTA (carry not included): look back over the predecessors, 32 at a time.  Nothing
    // here depends on this CTA's own records, so it overlaps their head reads; predecessors are usually done by then.
    Summ prefix = summ_identity();                   // fold of the predecessors examined so far (the nearest ones)
    for (int hi = (int)blockIdx.x - 1; hi >= 0; hi -= 32) {
      const int idx = hi - (int)lane;
      uint32_t sw = ep | 2u;                          // before the first CTA: an inclusive prefix equal to the identity
      if (idx >= 0) do { sw = status[idx]; } while ((sw & ~3u) != ep || (sw & 3u) == 0u);
      __threadfence();
      const unsigned incl = __ballot_sync(0xffffffffu, (sw & 3u) == 2u);
      const uint32_t last = incl ? (uint32_t)__ffs(incl) - 1u : 32u;
      Summ v = summ_identity();
      if (idx >= 0 && lane <= last) v = ld_summ_cg((sw & 3u) == 2u ? &slots[idx].incl : &slots[idx].aggr);
      // ordered: lane 0 is the nearest predecessor, so the fold runs from the highest lane down
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        Summ older;
        SUMM_SHFL(older, v, __shfl_down_sync, d);
        if (lane + (uint32_t)d < 32u) v = fold(older, v);
      }
      Summ window;
      SUMM_SHFL(window, v, __shfl_sync, 0);
      prefix = fold(window, prefix);
      if (incl) break;
    }
    if (lane == 0) blk_excl_sh = prefix;
  } else {
    Summ e = summ_identity();
    if (live) {
      pos = P.frame_off[r];
      H = load_head_words(P.buf + pos);
      h = read_head_w(H, P.len - pos);
      e = frame_state_elem(h, P.buf + pos);
      if (!h.malformed) {
        if (h.kind == 'I' || h.kind == 'U' || h.kind == 'D') s = find_schema(P, h.rel, pos);
        e.n_cells = frame_out_cells(h, s);
      }
    }
    // ---- scan of the CTA's elements: inclusive inside each warp, then across the warps
    Summ inc = e;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      Summ up;
      SUMM_SHFL(up, inc, __shfl_up_sync, d);
      if (lane >= (uint32_t)d) inc = fold(up, inc);
    }
    SUMM_SHFL(ex, inc, __shfl_up_sync, 1);
    if (lane == 0) ex = summ_identity();
    if (lane == 31u) wtot[wid] = inc;
    asm volatile("bar.sync 1, %0;" ::"n"(kRecThreads) : "memory");      // the record warps only
    if (threadIdx.x == 0) {                           // publish the aggregate at once: the successors wait for it
      Summ aggr = wtot[0];
#pragma unroll
      for (uint32_t k = 1; k < kRecThreads / 32; k++) aggr = fold(aggr, wtot[k]);
      if (blockIdx.x == 0) slots[0].incl = aggr; else slots[blockIdx.x].aggr = aggr;
      __threadfence();
      status[blockIdx.x] = ep | (blockIdx.x == 0 ? 2u : 1u);
    }
    for (uint32_t k = 0; k < wid; k++) wpre = fold(wpre, wtot[k]);
  }
  __syncthreads();                                    // the prefix is known
  uint64_t blk_cells = blk_excl_sh.n_cells;
#pragma unroll
  for (uint32_t k = 0; k < kRecThreads / 32; k++) blk_cells += wtot[k].n_cells;
  const bool blk_fits = blk_cells <= P.cap_cells;     // prefixes grow: every CTA after the first overflow sees it too
  if (lb_warp) {
    if (lane == 0) {
      Summ aggr = wtot[0];
#pragma unroll
      for (uint32_t k = 1; k < kRecThreads / 32; k++) aggr = fold(aggr, wtot[k]);
      const Summ incl_total = fold(blk_excl_sh, aggr);
      if (blockIdx.x) { slots[blockIdx.x].incl = incl_total; __threadfence(); status[blockIdx.x] = ep | 2u; }
      if (!blk_fits) atomicOr(P.abort_flag, ABORT_CELLS);
      if (blockIdx.x == n_blocks - 1u) {
        P.total[0] = incl_total;
        if (FULL && blk_fits && P.rec_cell_base) P.rec_cell_base[incl_total.n_rec] = incl_total.n_cells;
        if (P.seam_send) { SeamBlock sb; sb.total = incl_total; sb._pad[0] = sb._pad[1] = sb._pad[2] = sb._pad[3] = 0; *P.seam_send = sb; }
      }
    }
  }
  if (!FULL) return;
  uint32_t events = 0;
  if (live && blk_fits) {
    const uint8_t* const fp = P.buf + pos;
    const Summ st = fold(fold(P.dc->carry, blk_excl_sh), fold(wpre, ex));
    const uint64_t ridx = st.n_rec;
    const uint64_t gidx = P.dc->record_index_base + ridx;
    const uint64_t my_cell0 = st.n_cells;
    const bool in_tx = (st.flags & S_HAS_B) && !(st.flags & S_CLOSED);
    uint64_t commit_lsn = 0, ordinal = 0, start_lsn = 0;
    uint32_t rflags = 0;
    int32_t rschema = -1;
    uint32_t rrel = h.rel;
    bool ok = true;
    bool wellformed = !h.malformed;
    if (wellformed && h.kind == 'O') wellformed = (h.flen >= 4 + 26 + 8) && cstr_end(fp + 39, fp + 1 + h.flen) != nullptr;
    if (wellformed && h.kind == 'Y') {
      const uint8_t* fe = fp + 1 + h.flen;
      const uint8_t* q1 = (h.flen >= 4 + 26 + 4) ? cstr_end(fp + 35, fe) : nullptr;
      wellformed = q1 != nullptr && cstr_end(q1, fe) != nullptr;
    }
    if (wellformed && (h.kind == 'I' || h.kind == 'U' || h.kind == 'D')) {
      const uint32_t tt = hw_u8<35>(H);  // tuple marker (mlen >= 5 is guaranteed by read_head)
      if (h.kind == 'I') wellformed = tt == 'N';
      else if (h.kind == 'U') wellformed = tt == 'N' || tt == 'O' || tt == 'K';
      else wellformed = tt == 'O' || tt == 'K';
    }
    if (!wellformed) { report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); ok = false; }
    else if (h.kind == 'k') { start_lsn = hw_be64<6>(H); rrel = hw_u8<22>(H); }
    else {
      start_lsn = hw_be64<6>(H);                     // wal_start apply.rs:1700
      const uint8_t* m = fp + 31;                    // message body after the tag
      switch (h.kind) {
        case 'B':                                    // apply.rs:1927-1943
          commit_lsn = be64(m); ordinal = 0; rflags = ETL_RF_EVENT;
          put_cell(P, my_cell0, ETL_CELL_I64, be64(m + 8), 0);
          put_cell(P, my_cell0 + 1, ETL_CELL_U32, be32(m + 16), 0);
          break;
        case 'C': {                                  // apply.rs:1946-2006
          if (!in_tx) { report_error(P, gidx, SEQ_STATE, ETL_E_TX_STATE); ok = false; break; }
          const uint64_t cl = be64(m + 1);
          if (cl != st.lsn) { report_error(P, gidx, SEQ_STATE, ETL_E_COMMIT_LSN); ok = false; break; }
          commit_lsn = cl; ordinal = st.ord; rflags = ETL_RF_EVENT;
          put_cell(P, my_cell0, ETL_CELL_I32, (uint64_t)(int64_t)(int8_t)m[0], 0);
          put_cell(P, my_cell0 + 1, ETL_CELL_I64, be64(m + 9), 0);
          put_cell(P, my_cell0 + 2, ETL_CELL_I64, be64(m + 17), 0);
          break;
        }
        case 'R':                                    // apply.rs:2012-2089 (masks are built on the host)
          for (uint32_t k = 0; k < P.n_rel_errors; k++)
            if (P.rel_error_off[k] == pos) { report_error(P, gidx, P.rel_error_seq[k], P.rel_error_code[k]); ok = false; }
          if (!in_tx) { report_error(P, gidx, SEQ_STATE, ETL_E_TX_STATE); ok = false; break; }
          commit_lsn = st.lsn; ordinal = st.ord; rflags = ETL_RF_EVENT;
          { const DevSchema* rs = find_schema(P, h.rel, pos); if (rs && rs->effective_off == pos) rschema = (int32_t)rs->batch_index; }
          break;
        case 'I': case 'U': case 'D': {              // apply.rs:2092-2203
          // the tuple structure is validated by k_rows (a malformed frame outranks state errors)
          if (!in_tx) report_error(P, gidx, SEQ_STATE, ETL_E_TX_STATE);
          commit_lsn = st.lsn; ordinal = st.ord;
          if (!s) {                                  // no schema to walk with: structure check only
            unsigned long long ignored;
            if (!dml_structure_ok(h, fp, &ignored)) report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME);
            report_error(P, gidx, SEQ_TABLE, ETL_E_MISSING_TABLE_STATE); ok = false; break;
          }
          rschema = (int32_t)s->batch_index; rflags = ETL_RF_EVENT;
          if (h.old_tag == 'O') rflags |= ETL_RF_OLD_FULL; else if (h.old_tag == 'K') rflags |= ETL_RF_OLD_KEY;
          break;
        }
        case 'T': {                                  // apply.rs:2206-2248
          if (!in_tx) { report_error(P, gidx, SEQ_STATE, ETL_E_TX_STATE); ok = false; break; }
          commit_lsn = st.lsn; ordinal = st.ord;
          put_cell(P, my_cell0, ETL_CELL_I32, (uint64_t)(int64_t)(int8_t)m[4], 0);
          for (uint32_t i = 0; i < h.rel; i++) {
            const uint32_t rid = be32(m + 5 + 4 * i);
            const DevSchema* ts = find_schema(P, rid, pos);
            if (!ts) { report_error(P, gidx, SEQ_TABLE, ETL_E_MISSING_TABLE_STATE); ok = false; break; }
            put_cell(P, my_cell0 + 1 + i, ETL_CELL_U32, rid, ts->batch_index);
          }
          if (h.rel > 0) rflags = ETL_RF_EVENT;
          break;
        }
        case 'M': {                                  // apply.rs:1808-1924
          const uint8_t* end = fp + 1 + h.flen;
          const uint8_t* q = m + 9;
          const char* ddl = "supabase_etl_ddl";
          bool is_ddl = true; uint32_t k = 0; bool term = false;
          if (q > end) { report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); ok = false; break; }
          for (; q + k < end; k++) { uint32_t ch = q[k]; if (!ch) { term = true; break; } if (k >= 16 || ch != (uint32_t)(uint8_t)ddl[k]) is_ddl = false; }
          if (!term || !utf8_valid(q, k)) { report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); ok = false; break; }
          is_ddl = is_ddl && k == 16;
          const uint8_t* cq = q + k + 1;
          if (cq + 4 > end) { report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); ok = false; break; }
          const int32_t cl = (int32_t)be32(cq);
          if (cl < 0 || (uint64_t)cl > (uint64_t)(end - cq - 4)) { report_error(P, gidx, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); ok = false; break; }
          if (is_ddl) { rflags |= ETL_RF_DDL_MESSAGE; if (!in_tx) { report_error(P, gidx, SEQ_STATE, ETL_E_TX_STATE); ok = false; } }
          break;
        }
        default: break;                              // Origin / Type: structure only
      }
    }
    // a record k_rows must not touch keeps schema = -1 only when it failed before conversion
    if (h.kind == 'I' || h.kind == 'U' || h.kind == 'D') {
      if (!ok) rschema = -1;
      else if (rschema >= 0) atomicAdd(&hist[walk_bin(P, s->layout, h.kind, rflags)], 1u);
    }
    P.rec_off[ridx] = pos; P.rec_kind[ridx] = (uint8_t)h.kind; P.rec_flags[ridx] = (uint8_t)rflags;
    P.rec_rel[ridx] = rrel; P.rec_schema[ridx] = rschema; P.rec_start_lsn[ridx] = start_lsn;
    P.rec_commit_lsn[ridx] = commit_lsn; P.rec_tx_ordinal[ridx] = ordinal; P.rec_cell_base[ridx] = my_cell0;
    P.rec_flen[ridx] = 1u + h.flen; P.rec_tuple_bytes[ridx] = 0; P.rec_heap_hint[ridx] = 0;   // k_rows fills the DML records
    if (ok && (rflags & ETL_RF_EVENT)) events++;
  }
  // events: warp reduce, one atomic per warp
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) events += __shfl_down_sync(0xffffffffu, events, d);
  if (lane == 0 && events) atomicAdd(&P.metrics[3], (unsigned long long)events);
  __syncthreads();
  // the CTA's records are frames [blockIdx.x · kRecThreads, …) (one record per frame): all of them in one tile
  const uint32_t tile_bins = (uint32_t)((uint64_t)blockIdx.x * kRecThreads / P.bin_tile) * P.n_bins;
  for (uint32_t i = threadIdx.x; i < P.n_bins; i += blockDim.x) if (hist[i]) atomicAdd(&P.bin_count[tile_bins + i], hist[i]);
}
#undef SUMM_SHFL

// ================================================================================================
// size hints (types/table_row.rs:250-345): heap bytes a decoded cell owns.  String / Bytes: the Vec's capacity =
// its length (to_owned, with_capacity).  Numeric: the digit vector is pushed group by group onto Vec::new()
// (numeric.rs:441-448), so its capacity follows RawVec's amortised growth 0 → 4 → 8 → 16 …; the parsers leave the
// number of pushed groups in bits [16,32) of CellOut.tag.  Json / Array payloads are estimated by whoever builds
// the serde_json::Value / ArrayCell (the shim has to run that parser anyway) and are NOT part of rec_heap_hint.
__device__ __forceinline__ uint32_t vec_cap_after_pushes(uint32_t n) { return n == 0 ? 0u : (n <= 4u ? 4u : 1u << (32 - __clz(n - 1u))); }
__device__ __forceinline__ uint32_t cell_heap_hint(uint32_t tag32, uint32_t aux) {
  const uint32_t tag = tag32 & 0xFFu;
  if (tag == ETL_CELL_STRING || tag == ETL_CELL_BYTES) return aux;
  if (tag == ETL_CELL_NUMERIC) return 2u * vec_cap_after_pushes(tag32 >> 16);
  return 0u;
}
// a cloned cell (unchanged TOAST taken from the old image, event.rs:958-970): Clone allocates exactly len
__device__ __forceinline__ uint32_t cell_clone_hint(uint32_t tag, uint32_t aux) {
  if (tag == ETL_CELL_STRING || tag == ETL_CELL_BYTES) return aux;
  if (tag == ETL_CELL_NUMERIC) return 2u * aux;
  return 0u;
}

}  // namespace etl
#include "rows_kernel.cuh"
#include "copy_kernel.cuh"
namespace etl {

}  // namespace etl
