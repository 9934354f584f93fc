// rows_kernel.cuh — pass C2: tuples → rows, fused (replaces the round-1 k_walk → descriptors → k_cells → k_copy chain).
//
//   k_rows   one THREAD per DML record in shape-bin order (bins per tile of consecutive records, tile after
//            tile), one WARP per 32 structurally identical records.
//            Every pass each lane stages a window of its record's frame into shared memory with one 1-D bulk
//            async copy (cp.async.bulk → UBLKCP, completion on a per-warp mbarrier), then the 32 lanes walk
//            their tuples in lockstep: wire cell i is the same column in every lane, so one parser runs for
//            the whole warp on bytes that sit in shared memory.  The cell-header hop chain and the value bytes
//            are read from HBM exactly once (by the copy engine); there is no descriptor round trip, and an
//            unchanged-TOAST cell takes the value the same lane decoded for the old image a few steps earlier.
//            A lane's output cells go to its warp's stage in shared memory, not to the planes: at every step the 32
//            lanes write 32 different records' cells, which straight to the planes touched ~60 lines per step.  The
//            warp flushes the stage as runs of consecutive cells of one record (stage_flush).
//            k_rows itself parses the LIGHT decode classes (text, bool, integers, date / timestamp(tz), uuid in the
//            spellings Postgres emits): ~100 registers, no stack, 20+ warps per SM.  Every other cell (json, numeric,
//            floats, bytea, time, arrays, and any spelling the fast paths decline) is left in the cell plane as a
//            PENDING placeholder {kind, record, frame offset, length}.
//   k_heavy  second pass over the cell plane: a CTA takes a tile of 4096 cells, gathers the pending ones per decode
//            class in shared memory and parses them 32 at a time (one class per warp row, so the warp-synchronous
//            parsers run full width), each lane's bytes staged from global memory with all its 16-byte loads in flight.
//   k_fix    resolves unchanged-TOAST cells whose source was still pending when k_rows met them.
//
// Reference semantics: event.rs:376-979 (tuples → rows), text.rs:28-173 (cells), event.rs:260-270 (tuple bytes),
// types/table_row.rs + types/event.rs:288-312 (size hints).
#pragma once

namespace etl {

// k_rows: the window and the cell stage share the shared memory of 5 CTAs per SM.  A 4-cell stage per lane (1.6 KB per
// warp) is paid for by a 240-byte window instead of 304; 240 is the largest window that still fits 5 CTAs next to a
// 4-cell stage (256 fits, 272 misses by ~0.5 KB), and a 16-cell stage (6.5 KB per warp) would leave under 160 bytes.
// Measured on C5 / C2 (H100 SXM, 700 W), k_rows + k_heavy + k_fix: no stage, 304 B 2.05 / 0.53 ms; 4 cells, 240 B
// 1.41 / 0.46 ms; 8 cells, 208 B 1.59 / 0.54 ms; 8 cells, 176 B 1.74 / 0.58 ms: the window's restages cost more than
// the longer runs save.
#ifndef ETL_TUPLE_WIN
#define ETL_TUPLE_WIN 240                // k_rows: bytes of one record's frame staged per pass (multiple of 16)
#endif
// k_copy_rows has no cell stage and keeps the whole window
#ifndef ETL_ROWS_WIN
#define ETL_ROWS_WIN 304                 // k_copy_rows: bytes of one COPY row staged per pass (multiple of 16)
#endif
#ifndef ETL_ROWS_STAGE
#define ETL_ROWS_STAGE 4                 // output cells per lane staged in shared memory between flushes (power of 2, ≤ 16)
#endif
#ifndef ETL_ROWS_CTAS
#define ETL_ROWS_CTAS 5                  // resident CTAs per SM the register budget is set for
#endif
#ifndef ETL_ROWS_WARPS
#define ETL_ROWS_WARPS 4
#endif
constexpr uint32_t kRowsWarps = ETL_ROWS_WARPS;
constexpr uint32_t kRowsThreads = kRowsWarps * 32;
constexpr uint32_t kRowsWin = ETL_TUPLE_WIN;
constexpr uint32_t kRowsSlot = kRowsWin + 16;                      // slot stride: 16-byte aligned, skews the banks
constexpr uint32_t kRowsBarOff = 0;                                // one mbarrier per warp
constexpr uint32_t kRowsColsOff = kRowsBarOff + 128;               // per warp: 256 column kinds + 256 column flags of its schema
constexpr uint32_t kRowsColsCached = 256;
// per warp: the cell stage, kRowsStage rows of 32 entries as planes val (u64), aux (u32), tag (u8)
constexpr uint32_t kRowsStage = ETL_ROWS_STAGE;
constexpr uint32_t kRowsStageRuns = 32 / kRowsStage;               // lanes' runs stored per round of a flush
constexpr uint32_t kRowsStageBytes = kRowsStage * 32 * 13;
constexpr uint32_t kRowsStageOff = kRowsColsOff + kRowsWarps * 2 * kRowsColsCached;
constexpr uint32_t kRowsSlotsOff = kRowsStageOff + kRowsWarps * kRowsStageBytes;
constexpr uint32_t kRowsSmemBytes = kRowsSlotsOff + kRowsWarps * 32 * kRowsSlot + 64;   // + tail padding for word reads
constexpr uint32_t kRowsMaxInWin = kRowsWin - 24;                  // a text cell up to this long always fits a fresh window
static_assert(kRowsWarps <= 15 && kRowsWin % 16 == 0, "k_rows geometry");
static_assert(kRowsStage >= 2 && kRowsStage <= 16 && (kRowsStage & (kRowsStage - 1)) == 0 && kRowsStageBytes % 16 == 0, "k_rows stage");
// k_copy_rows: the same barriers and column cache, no stage, its own window
constexpr uint32_t kCopyWin = ETL_ROWS_WIN;
constexpr uint32_t kCopySlot = kCopyWin + 16;
constexpr uint32_t kCopySlotsOff = kRowsStageOff;
constexpr uint32_t kCopySmemBytes = kCopySlotsOff + kRowsWarps * 32 * kCopySlot + 64;
static_assert(kCopyWin % 16 == 0, "k_copy_rows geometry");
static_assert((size_t)ETL_ROWS_CTAS * (kRowsSmemBytes + 1024) <= 228u * 1024u, "k_rows: the CTAs per SM must fit the shared memory");
static_assert((size_t)ETL_ROWS_CTAS * (kCopySmemBytes + 1024) <= 228u * 1024u, "k_copy_rows: the CTAs per SM must fit the shared memory");

// ---- mbarrier / bulk-copy primitives (PTX ISA 8.x; SASS: SYNCS.*, UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
// global → shared, 16-byte aligned on both sides, size a multiple of 16; completion is signalled on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// Cells k_rows leaves for k_heavy: tag = ETL_CELL_PENDING | decode class (ETL_K_*, 6 bits), val = record << 32 | offset
// of the value bytes inside the record's frame, aux = length.  ETL_CELL_PENDING_COPY: an unchanged-TOAST cell whose
// source (val = its cell index, aux = record) was itself pending.  Internal: no placeholder survives a decode.
constexpr uint32_t ETL_CELL_PENDING = 0x80u, ETL_CELL_PENDING_MASK = 0xC0u, ETL_CELL_PENDING_COPY = 0xF0u;
__device__ __forceinline__ bool kind_is_light(uint32_t kind) {
  return kind == ETL_K_STRING || kind == ETL_K_BOOL || (kind - ETL_K_I16) <= (ETL_K_I64 - ETL_K_I16) || kind == ETL_K_DATE ||
         kind == ETL_K_TIMESTAMP || kind == ETL_K_TIMESTAMPTZ || kind == ETL_K_UUID;
}
// text.rs:28-173, the light classes, for the lanes of `mask` (same class): warp-synchronous / SWAR fast paths for the
// spellings Postgres emits.  Returns 0 (o filled), an error code, or 0xFFFFFFFF = "not this spelling": the cell is
// left to k_heavy's exact parsers.  `hpos` = this lane's 16 bytes in the heap (uuid).
__device__ __forceinline__ uint32_t parse_light_sync(unsigned mask, uint32_t kind, const uint8_t* tv, uint32_t len, uint8_t* heap, uint64_t hpos, CellOut& o) {
  switch (kind) {
    case ETL_K_I32: case ETL_K_I64: case ETL_K_I16: case ETL_K_U32: {   // one copy of the parser, limits by kind
      const uint64_t pos_limit = kind == ETL_K_I32 ? 2147483647ull : (kind == ETL_K_I64 ? 9223372036854775807ull : (kind == ETL_K_I16 ? 32767ull : 4294967295ull));
      const uint64_t neg_limit = kind == ETL_K_U32 ? 0ull : pos_limit + 1ull;
      int64_t iv = 0;
      const uint32_t code = parse_int_sync(mask, tv, len, kind != ETL_K_U32, pos_limit, neg_limit, &iv);
      o.tag = kind == ETL_K_I32 ? ETL_CELL_I32 : (kind == ETL_K_I64 ? ETL_CELL_I64 : (kind == ETL_K_I16 ? ETL_CELL_I16 : ETL_CELL_U32));
      o.val = (uint64_t)iv;
      return code;
    }
    case ETL_K_TIMESTAMPTZ: return fast_timestamptz(tv, len, o) ? 0u : 0xFFFFFFFFu;
    case ETL_K_TIMESTAMP: return fast_timestamp(tv, len, o) ? 0u : 0xFFFFFFFFu;
    case ETL_K_DATE: return fast_date(tv, len, o) ? 0u : 0xFFFFFFFFu;
    case ETL_K_UUID: return fast_uuid(tv, len, heap, hpos, o) ? 0u : 0xFFFFFFFFu;
    case ETL_K_BOOL:                                  // bool.rs: exactly "t" / "f"
      if (len == 1 && (tv[0] == 't' || tv[0] == 'f')) { o.tag = ETL_CELL_BOOL; o.val = tv[0] == 't'; return 0u; }
      return ETL_E_BOOL;
    default: return 0xFFFFFFFFu;
  }
}
// ... and every class, exactly, for k_heavy (the exact parsers are out of line; json / numeric have warp-synchronous paths)
struct CellHeaps { uint8_t* heap; unsigned long long* arr_top; uint64_t arr_base, heap_cap; unsigned int* heap_overflow; };
__device__ __forceinline__ uint32_t parse_heavy_sync(unsigned mask, uint32_t kind, const uint8_t* tv, uint32_t len, uint64_t soff,
                                                     const CellHeaps H, uint64_t hpos, const uint8_t* JT, CellOut& o) {
  uint32_t code = 0;
  if (kind == ETL_K_JSON) {
    if (json_valid_sync(mask, tv, len, JT)) { o.tag = ETL_CELL_JSON; o.val = soff; o.aux = len; } else code = ETL_E_JSON;
  } else if (kind == ETL_K_NUMERIC) code = parse_numeric_sync(mask, tv, len, H.heap, hpos, o);
  else {
    CellOut tt; tt.tag = 0; tt.val = 0; tt.aux = 0;     // out-of-line parsers get their own CellOut so that `o` never has its address taken
    if (kind & ETL_K_ARRAY) {
      code = parse_array_any(ArrHeap{H.heap, H.arr_top, H.arr_base, H.heap_cap}, kind, tv, len, tt);
      if (code == 0xFFFFFFFEu) { atomicExch(H.heap_overflow, 1u); code = 0; tt.tag = ETL_CELL_NULL; }
    } else code = parse_text_cell(kind, tv, len, soff, H.heap, hpos, tt);
    o = tt;
  }
  return code;
}

// Walker state of one record.
struct Wk {
  const uint8_t* base;   // frame start (global)
  uint32_t pos, end;     // frame-relative: next byte to read / frame end
  uint32_t col_base;
  uint32_t nc_ni;        // n_cols | n_ident << 16   (both ≤ 32767: int16 on the wire)
  uint64_t cell0;        // first output cell of the record
  uint32_t rec_local;
  uint32_t rem_wire;     // remaining | wire_i << 16
  uint32_t cmap_kout;    // cmap | k_out << 16
  uint32_t keyi_nold;    // key_i | n_old << 16
  uint32_t bits;         // stage[0:3) kind[3:5) old[5:7) dense[7] partial[8] emit[9]
  uint32_t tb;           // Σ text lengths (calculate_tuple_bytes event.rs:260-270)
  uint32_t hint;         // Σ heap capacities of the decoded cells (size hints, types/table_row.rs:138-175)
};
enum : uint32_t { W_OLD_HDR = 0, W_OLD_CELLS = 1, W_NEW_HDR = 2, W_NEW_CELLS = 3, W_DONE = 4 };
enum : uint32_t { WK_I = 1, WK_U = 2, WK_D = 3, WO_FULL = 1, WO_KEY = 2, WB_DENSE = 1u << 7, WB_PARTIAL = 1u << 8,
                  WB_EMIT = 1u << 9 };   // emit clears after the first data error: structure-only walk (a malformed
                                         // frame, i.e. a parser error in the reference, outranks every conversion error)
struct TextCell { uint32_t voff, len, kind, dest, seq; };   // voff frame-relative, dest relative to cell0
#define W_SET_STAGE(s_) (w.bits = (w.bits & ~7u) | (s_))
#define W_DATA_ERROR(seq_, code_) do { report_error(P, P.dc->record_index_base + w.rec_local, (seq_), (code_)); w.bits &= ~WB_EMIT; } while (0)
#define W_MALFORMED() do { report_error(P, P.dc->record_index_base + w.rec_local, SEQ_MALFORMED, ETL_E_MALFORMED_FRAME); W_SET_STAGE(W_DONE); } while (0)

// The dest of the next cell `w` can write (the start of a fresh run).
__device__ __forceinline__ uint32_t rk_next_dest(const Wk& w) {
  const uint32_t stage = w.bits & 7u, n_old = w.keyi_nold >> 16;
  if (stage == W_OLD_CELLS) return ((w.bits >> 5) & 3u) == WO_KEY ? (w.cmap_kout >> 16) : (w.rem_wire >> 16);
  if (stage == W_NEW_CELLS) return n_old + (w.rem_wire >> 16);
  return stage == W_NEW_HDR ? n_old : 0u;
}

// The staged window of a lane: frame-relative bytes [max(delta,0), w1) live at win[pos - delta].
struct RowWin { const uint8_t* win; int32_t delta; uint32_t w1; };
__device__ __forceinline__ bool win_has(const RowWin& W, uint32_t pos, uint32_t n, uint32_t end) {
  return (int32_t)pos >= W.delta && (pos + n <= W.w1 || W.w1 >= end);
}

// Does the next step of `w` need bytes that are not in the window?  (No state is changed: when any lane says
// yes, the warp restages every lane at its current position and asks again, so the lanes stay in lockstep.)
// *hdr receives the 8 bytes at w.pos when they are readable.
__device__ __forceinline__ bool rk_peek(const Wk& w, const RowWin& W, uint64_t* hdr) {
  const uint32_t stage = w.bits & 7u;
  *hdr = 0;
  if (stage == W_DONE) return false;
  const bool is_hdr = stage == W_OLD_HDR || stage == W_NEW_HDR;
  if (!is_hdr && (w.rem_wire & 0xFFFFu) == 0) return false;            // end of a tuple: no bytes needed
  if (w.pos >= w.end) return false;                                    // malformed: the step reports it
  if (!win_has(W, w.pos, 5u, w.end)) return true;
  const uint64_t x = ld64u(W.win + ((int32_t)w.pos - W.delta));
  *hdr = x;
  if (is_hdr) return false;
  const uint32_t tag = (uint32_t)(x & 0xFFu);
  if (tag != 't' && tag != 'b') return false;
  const uint32_t len = bswap32((uint32_t)(x >> 8));
  if ((uint64_t)w.pos + 5 > w.end || (int32_t)len < 0 || (uint64_t)len > (uint64_t)(w.end - w.pos - 5)) return false;   // malformed
  if (len > kRowsMaxInWin) return false;                               // oversize cell: parsed from global memory
  return w.pos + 5u + len > W.w1;
}

// ---- the cell stage.  Neighbouring lanes walk different records, so a cell stored straight to the planes at every step
// touches ~60 lines per warp for 13 useful bytes per lane.  Instead each lane writes its cells into its warp's stage, at
// dest − rb (rb = the dest its current run starts at), and the warp flushes the stage as runs: S lanes store S
// consecutive cells of one record, a few lines per run.  Within one tuple the dests a lane writes are consecutive (a
// skipped or failed cell ends the writes of its tuple), so a run is full when its entry S − 1 is written; the old
// image is flushed before the new tuple starts (an unchanged-TOAST cell reads its source from the planes).
// sg = rb | valid entries << 16.  Entry (j, lane) sits at row j, column lane ^ (j · runs per round): the lanes of one
// step write one row, and the lanes of one flush round read 32 distinct banks.
__device__ __forceinline__ uint32_t stage_entry(uint32_t j, uint32_t lane) { return j * 32u + (lane ^ ((j * kRowsStageRuns) & 31u)); }
__device__ __forceinline__ void stage_put(const DecodeParams& P, uint8_t* st, uint32_t& sg, uint64_t cell0, uint32_t dest, uint32_t tag, uint64_t val, uint32_t aux) {
  const uint32_t j = dest - (sg & 0xFFFFu);
  // Unreachable while the run invariants hold (consecutive dests within a tuple, a flush when a run is full and before
  // a new tuple starts elsewhere).  A store that missed the stage still lands in the plane, so a broken invariant
  // would cost coalescing, not correctness; tests/test_gpu_rows_stage.py covers the run edges.
  if (j >= kRowsStage) { put_cell(P, cell0 + dest, tag, val, aux); return; }
  const uint32_t e = stage_entry(j, threadIdx.x & 31u);
  reinterpret_cast<uint64_t*>(st)[e] = val;
  reinterpret_cast<uint32_t*>(st + kRowsStage * 256u)[e] = aux;
  st[kRowsStage * 384u + e] = (uint8_t)tag;
  sg |= 1u << (16u + j);
}
// Warp-wide: every lane's staged entries to the planes, run after run; the next run of each lane starts at rb_next.
__device__ __forceinline__ void stage_flush(const DecodeParams& P, const uint8_t* st, uint32_t& sg, uint64_t cell0, uint32_t rb_next) {
  const uint32_t lane = threadIdx.x & 31u, j = lane & (kRowsStage - 1u);
  const uint32_t vm = sg >> 16;
  const unsigned have = __ballot_sync(0xffffffffu, vm != 0u);
  if (have) {
    __syncwarp();
    const uint64_t base = cell0 + (sg & 0xFFFFu);
    for (uint32_t r = 0; r < 32u; r += kRowsStageRuns) {
      if (!((have >> r) & ((1u << kRowsStageRuns) - 1u))) continue;
      const uint32_t src = r + lane / kRowsStage;
      const uint32_t vs = __shfl_sync(0xffffffffu, vm, src);
      const uint64_t bs = __shfl_sync(0xffffffffu, base, src);
      if ((vs >> j) & 1u) {
        const uint32_t e = stage_entry(j, src);
        put_cell(P, bs + j, st[kRowsStage * 384u + e], reinterpret_cast<const uint64_t*>(st)[e], reinterpret_cast<const uint32_t*>(st + kRowsStage * 256u)[e]);
      }
    }
    __syncwarp();
  }
  sg = rb_next;
}

// One step: a tuple header or ONE wire cell (event.rs:550-919).  Returns 0 when no wire cell was consumed
// (header, end of a tuple, malformed), 1 when one was consumed and needs no parsing, 2 when it is a text cell.
__device__ __forceinline__ uint32_t rk_step(const DecodeParams& P, Wk& w, TextCell& tc, const uint64_t x, const uint8_t* kinds, const uint8_t* flags,
                                           uint8_t* st, uint32_t& sg) {
  const uint32_t stage = w.bits & 7u, kind = (w.bits >> 3) & 3u, old = (w.bits >> 5) & 3u;
  const bool emit = (w.bits & WB_EMIT) != 0;
  const uint32_t n_cols = w.nc_ni & 0xFFFFu, n_ident = w.nc_ni >> 16;
  uint32_t ret = 0;
  do {
    if (stage == W_OLD_HDR || stage == W_NEW_HDR) {
      const bool is_new = stage == W_NEW_HDR;
      if ((uint64_t)w.pos + (is_new ? 3u : 2u) > w.end) { W_MALFORMED(); break; }
      uint32_t hdr = (uint32_t)x;
      if (is_new) {
        if ((hdr & 0xFFu) != 'N') { W_MALFORMED(); break; }
        hdr >>= 8; w.pos++;
      }
      int32_t nci = (int32_t)(int16_t)(((hdr & 0xFFu) << 8) | ((hdr >> 8) & 0xFFu));
      const uint32_t nc = nci < 0 ? 0u : (uint32_t)nci;
      w.pos += 2;
      w.rem_wire = nc; w.cmap_kout = 0;
      if (!is_new) {
        if (old == WO_KEY) {                        // normalize_key_tuple_to_row event.rs:879-919
          w.keyi_nold = (w.keyi_nold & 0xFFFFu) | (n_ident << 16);
          const bool dense = nc == n_ident;
          if (dense) w.bits |= WB_DENSE;
          if (emit) {
            if (n_ident == 0) W_DATA_ERROR(SEQ_OLD_SHAPE, ETL_E_KEY_NO_COLUMNS);
            else if (!dense && nc != n_cols) W_DATA_ERROR(SEQ_OLD_SHAPE, ETL_E_KEY_SHAPE);
          }
        } else {                                    // convert_tuple_to_row event.rs:550-583
          w.keyi_nold = (w.keyi_nold & 0xFFFFu) | (n_cols << 16);
          if (emit && nc != n_cols) W_DATA_ERROR(SEQ_OLD_SHAPE, ETL_E_FIELD_COUNT);
        }
        W_SET_STAGE(W_OLD_CELLS);
      } else {
        if (emit && nc != n_cols) W_DATA_ERROR(SEQ_NEW_SHAPE, ETL_E_FIELD_COUNT);
        W_SET_STAGE(W_NEW_CELLS);
      }
      break;
    }
    if ((w.rem_wire & 0xFFFFu) == 0) {
      W_SET_STAGE((stage == W_OLD_CELLS && kind != WK_D) ? W_NEW_HDR : W_DONE);
      break;
    }
    if (w.pos >= w.end) { W_MALFORMED(); break; }
    const uint32_t tag = (uint32_t)(x & 0xFFu);
    const uint32_t len = bswap32((uint32_t)(x >> 8));
    const uint32_t voff = w.pos + 5u;
    if (tag == 't' || tag == 'b') {
      if ((uint64_t)w.pos + 5 > w.end || (int32_t)len < 0 || (uint64_t)len > (uint64_t)(w.end - w.pos - 5)) { W_MALFORMED(); break; }
      w.tb += len;
      w.pos += 5u + len;
    } else if (tag == 'n' || tag == 'u') w.pos += 1;
    else { W_MALFORMED(); break; }
    const uint32_t i = w.rem_wire >> 16;
    w.rem_wire += 0x10000u - 1u;                    // wire_i++, remaining--
    ret = 1;
    if (!emit) break;                               // structure-only after a data error
    const bool is_new = stage == W_NEW_CELLS;
    uint32_t col = i, dest;
    if (!is_new && old == WO_KEY) {
      if (w.bits & WB_DENSE) {
        uint32_t cmap = w.cmap_kout & 0xFFFFu;
        while (cmap < n_cols && !(flags[cmap] & 2)) cmap++;
        col = cmap++;
        w.cmap_kout = (w.cmap_kout & 0xFFFF0000u) | cmap;
      } else if (!(flags[i] & 2)) break;            // full-width key: non-identity entries are not decoded
      dest = w.cmap_kout >> 16;
      w.cmap_kout += 0x10000u;
    } else dest = (is_new ? (w.keyi_nold >> 16) : 0u) + i;
    const uint32_t seq = is_new ? seq_new_cell(i) : seq_old_cell(i);
    const bool upd_key = is_new && kind == WK_U && old == WO_KEY;
    const bool need_flags = tag != 't' || upd_key;
    const uint32_t cflags = need_flags ? (uint32_t)flags[col] : 0u;
    const bool resolver_key = upd_key && (cflags & 2);
    if (tag == 't') {
      if (resolver_key) w.keyi_nold++;
      tc.voff = voff; tc.len = len; tc.kind = kinds[col]; tc.dest = dest; tc.seq = seq;
      return 2;
    }
    if (tag == 'n') {                               // convert_tuple_data_to_cell event.rs:941-957
      if (resolver_key) w.keyi_nold++;
      if (cflags & 1) stage_put(P, st, sg, w.cell0, dest, ETL_CELL_NULL, 0, 0);
      else W_DATA_ERROR(seq, ETL_E_NOT_NULL);
      break;
    }
    if (tag == 'u') {                               // event.rs:958-970 + OldRowResolver :722-762
      if (is_new && kind == WK_U) {
        uint64_t src = ~0ull;
        if (old == WO_FULL) src = w.cell0 + i;
        else if (resolver_key) { src = w.cell0 + (w.keyi_nold & 0xFFFFu); w.keyi_nold++; }
        if (src != ~0ull) {                         // this lane decoded the old image earlier in the same walk
          const uint32_t stag = P.cell_tag[src];
          const uint32_t saux = P.cell_aux[src];
          if ((stag & ETL_CELL_PENDING_MASK) == ETL_CELL_PENDING) {     // the old cell waits for k_heavy: k_fix copies it afterwards
            stage_put(P, st, sg, w.cell0, dest, ETL_CELL_PENDING_COPY, src, w.rec_local);
            atomicAdd(P.copy_count, 1u);
          } else {
            stage_put(P, st, sg, w.cell0, dest, stag, P.cell_val[src], saux);
            w.hint += cell_clone_hint(stag, saux);  // the clone owns its own heap buffer (Cell::clone)
          }
        } else { stage_put(P, st, sg, w.cell0, dest, ETL_CELL_MISSING, 0, 0); w.bits |= WB_PARTIAL; }
      } else W_DATA_ERROR(seq, (!is_new && old == WO_KEY) ? ETL_E_KEY_MISSING_VALUE : ETL_E_FULL_ROW_MISSING);
      break;
    }
    if (resolver_key) w.keyi_nold++;
    W_DATA_ERROR(seq, ETL_E_BINARY_FORMAT);         // 'b'
  } while (0);
  return ret;
}

// pass C2: rows.  grid = chunks of kRowsThreads records of the binned order (+ padding), dynamic smem kRowsSmemBytes.
__device__ __forceinline__ void rows_body(const DecodeParams& P, uint8_t* smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t n_perm = *P.perm_len;
  // chunk of the binned order for this CTA: consecutive CTAs, consecutive chunks.  The bins are per tile of
  // consecutive records, so the CTAs resident together work on a narrow band of the stream, and every tile holds
  // its natural mix of costs per record (an update with a full old image walks twice the cells of an insert).
  // The grid is sized for the worst-case padding.
  const uint32_t chunk = blockIdx.x;
  if ((uint64_t)chunk * blockDim.x >= n_perm) return;
  // CTA set-up: one mbarrier per warp
  if (threadIdx.x == 0) {
    for (uint32_t k = 0; k < kRowsWarps; k++) mbar_init(smem_u32(smem + kRowsBarOff + 8u * k), 32u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t bar = smem_u32(smem + kRowsBarOff + 8u * wid);
  uint8_t* const slot = smem + kRowsSlotsOff + ((uint32_t)wid * 32u + (uint32_t)lane) * kRowsSlot;
  const uint32_t slot_s = smem_u32(slot);
  uint32_t parity = 0;

  const uint32_t t = chunk * blockDim.x + threadIdx.x;
  const uint32_t my_rec = t < n_perm ? P.perm[t] : 0xFFFFFFFFu;   // 0xFFFFFFFF = bin padding
  Wk w;
  w.bits = W_DONE; w.tb = 0; w.hint = 0; w.rec_local = 0; w.base = P.buf; w.pos = 0; w.end = 0; w.col_base = 0; w.nc_ni = 0; w.cell0 = 0;
  w.rem_wire = 0; w.cmap_kout = 0; w.keyi_nold = 0;
  uint64_t frame_goff = 0;
  if (my_rec != 0xFFFFFFFFu) {
    const uint64_t rr = my_rec;
    frame_goff = P.rec_off[rr];
    const int32_t sc = P.rec_schema[rr];
    const DevSchema& s = P.schemas[P.schema_by_batch[sc]];
    w.base = P.buf + frame_goff; w.end = P.rec_flen[rr];
    w.col_base = s.col_base; w.nc_ni = s.n_cols | (s.n_ident << 16);
    w.cell0 = P.rec_cell_base[rr]; w.rec_local = (uint32_t)rr;
    const uint32_t k = P.rec_kind[rr], rf = P.rec_flags[rr];
    const uint32_t kc = k == 'I' ? WK_I : (k == 'U' ? WK_U : WK_D);
    const uint32_t oc = (rf & ETL_RF_OLD_FULL) ? WO_FULL : ((rf & ETL_RF_OLD_KEY) ? WO_KEY : 0u);
    const bool old_first = kc != WK_I && oc;        // old image first; else the 'N' marker, then the new tuple
    w.pos = old_first ? 36u : 35u;
    w.bits = (old_first ? W_OLD_HDR : W_NEW_HDR) | (kc << 3) | (oc << 5) | WB_EMIT;
  }
  const unsigned valid = __ballot_sync(0xffffffffu, my_rec != 0xFFFFFFFFu);
  if (valid == 0) return;
  // the warp's column kinds / flags: one schema per warp in a shape bin → a shared-memory copy (every step reads them);
  // warps of a clamped bin (mixed schemas) and very wide tables read them from global memory
  const uint8_t* kinds = P.col_kind + w.col_base;
  const uint8_t* flags = P.col_flags + w.col_base;
  {
    const int first = __ffs(valid) - 1;
    const uint32_t cb0 = __shfl_sync(0xffffffffu, w.col_base, first), nn0 = __shfl_sync(0xffffffffu, w.nc_ni, first);
    const bool same = __all_sync(0xffffffffu, my_rec == 0xFFFFFFFFu || (w.col_base == cb0 && w.nc_ni == nn0));
    const uint32_t nc0 = nn0 & 0xFFFFu;
    if (same && nc0 <= kRowsColsCached) {
      uint8_t* ck = smem + kRowsColsOff + (uint32_t)wid * 2u * kRowsColsCached;
      for (uint32_t i = (uint32_t)lane; i < nc0; i += 32u) { ck[i] = P.col_kind[cb0 + i]; ck[kRowsColsCached + i] = P.col_flags[cb0 + i]; }
      __syncwarp();
      kinds = ck; flags = ck + kRowsColsCached;
    }
  }
  RowWin W;
  W.win = slot; W.delta = 0x7FFFFFFF; W.w1 = 0;     // empty window: the first peek stages
  uint8_t* const st = smem + kRowsStageOff + (uint32_t)wid * kRowsStageBytes;
  uint32_t sg = 0;                                  // the lane's run: rb | staged entries << 16
  for (;;) {
    const bool act = (w.bits & 7u) != W_DONE;
    if (!__any_sync(0xffffffffu, act)) break;
    // a lane whose run is full, or whose new tuple starts elsewhere than its run (the old image is staged): flush
    const bool flush = ((sg >> (15u + kRowsStage)) & 1u) || ((w.bits & 7u) == W_NEW_HDR && (sg & 0xFFFFu) != (w.keyi_nold >> 16));
    if (__any_sync(0xffffffffu, flush)) stage_flush(P, st, sg, w.cell0, rk_next_dest(w));
    uint64_t hdr;
    const bool need = rk_peek(w, W, &hdr);
    if (__any_sync(0xffffffffu, need)) {
      // restage every live lane at its current position: [g0, g0 + n) with g0 = 16-byte floor of the position
      __syncwarp();                                   // other lanes may still be reading this lane's window (UTF-8 slow path)
      uint32_t n = 0;
      if (act && w.pos < w.end) {
        const uint64_t gpos = frame_goff + w.pos;
        const uint64_t g0 = gpos & ~15ull;
        const uint64_t gend = (frame_goff + w.end + 15ull) & ~15ull;       // ≤ len + 15: the stream has 64 readable bytes of padding
        n = (uint32_t)min((uint64_t)kRowsWin, gend - g0);
        W.delta = (int32_t)((int64_t)g0 - (int64_t)frame_goff);
        W.w1 = (uint32_t)(W.delta + (int32_t)n);
        mbar_arrive_expect_tx(bar, n);
        bulk_g2s(slot_s, P.buf + g0, n, bar);
      } else mbar_arrive(bar);
      mbar_wait(bar, parity);
      parity ^= 1u;
      continue;
    }
    TextCell tc;
    tc.voff = 0; tc.len = 0; tc.kind = 0; tc.dest = 0; tc.seq = 0;
    const uint32_t got = act ? rk_step(P, w, tc, hdr, kinds, flags, st, sg) : 0u;
    const bool is_text = got == 2u;
    if (!__any_sync(0xffffffffu, is_text)) continue;
    // ---- the text cells of this step: UTF-8 (event.rs:972), the per-kind parser, the cell plane and the heap
    const uint32_t kind = tc.kind, len = tc.len;
    const uint64_t soff = frame_goff + tc.voff;
    const bool in_win = is_text && len <= kRowsMaxInWin;              // rk_peek made sure it is resident
    const uint8_t* tv = in_win ? W.win + ((int32_t)tc.voff - W.delta) : P.buf + soff;
    CellOut o;
    o.tag = 0; o.val = 0; o.aux = 0;
    uint32_t code = 0;
    bool need_slow = false;                            // cell with non-ASCII bytes: validated by the whole warp below
    uint32_t r0_hi = 0, r1_lo = 0, r1_hi = 0;          // long cell: byte ranges [0, r0_hi) and [r1_lo, r1_hi) validated by the whole warp
    if (is_text) {
      if (kind == ETL_K_STRING) { o.tag = ETL_CELL_STRING; o.val = soff; o.aux = len; }
      if (in_win) need_slow = has_high_bits(tv, len);
      else if (len >= (uint32_t)kCoopLen) {
        // a long cell is read from global memory.  A text column (the TOAST case) needs nothing but its UTF-8 verdict:
        // listed for k_long_cells, which runs after the join with enough warps to hide the latency.  Other kinds must
        // be validated before they are parsed: whole warp, here.
        const bool defer = kind == ETL_K_STRING;
        const uint64_t cb = soff + len;
        const uint64_t S0 = (soff + 3ull + P.anchor_stride - 1ull) & ~(uint64_t)(P.anchor_stride - 1u), S1 = cb & ~(uint64_t)(P.anchor_stride - 1u);
        r0_hi = defer ? 0u : len;
        if (defer || S0 < S1) {
          const uint32_t at = atomicAdd(P.long_count, 1u);
          if (at < P.long_cap) {
            LongCell lc;
            lc.rec_local = w.rec_local; lc.seq = tc.seq; lc.soff = soff; lc.len = len; lc.edges = defer ? 1u : 0u;
            P.long_cells[at] = lc;
            // the tail keeps at least the last byte (k_long_cells does the same): a sequence left open at the end of the
            // interior is a violation only past the cell's end
            if (!defer) { r0_hi = (uint32_t)(S0 - soff); r1_lo = min((uint32_t)(S1 - soff), len - 1u); r1_hi = len; }
          } else r0_hi = len;                          // cannot happen (the list holds every cell of ≥ kCoopLen bytes)
        }
      } else if (utf8_medium_bad(tv, len)) code = ETL_E_UTF8;
    }
    __syncwarp();
    // position-local UTF-8 rule, one byte position per lane (a lane-serial walk of a 60-byte cell would
    // hold the other 31 lanes for ~1000 issue slots; this costs ~60 for the whole warp)
    for (unsigned sm = __ballot_sync(0xffffffffu, need_slow); sm; sm &= sm - 1) {
      const int src = __ffs(sm) - 1;
      const uint8_t* cp = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(tv), src));
      const uint32_t cn = __shfl_sync(0xffffffffu, len, src);
      bool bad = false;
      for (uint32_t i = lane; i <= cn; i += 32) {        // position cn = a virtual ASCII terminator (catches a truncated tail)
        const uint32_t b = i < cn ? cp[i] : 0u, p1 = i >= 1 ? cp[i - 1] : 0u, p2 = i >= 2 ? cp[i - 2] : 0u, p3 = i >= 3 ? cp[i - 3] : 0u;
        if ((b | p1 | p2 | p3) >= 0x80u) bad |= utf8_step_bad(b, p1, p2, p3);
      }
      bad = __any_sync(0xffffffffu, bad);
      if (lane == src && bad) code = ETL_E_UTF8;
    }
    for (int round = 0; round < 2; round++) {
      const uint32_t my_lo = round ? r1_lo : 0u, my_hi = round ? r1_hi : r0_hi;
      for (unsigned sm = __ballot_sync(0xffffffffu, my_hi > my_lo); sm; sm &= sm - 1) {
        const int src = __ffs(sm) - 1;
        const uint8_t* cp = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(tv), src));
        const uint32_t cn = __shfl_sync(0xffffffffu, len, src), lo = __shfl_sync(0xffffffffu, my_lo, src), hi = __shfl_sync(0xffffffffu, my_hi, src);
        const bool bad = __any_sync(0xffffffffu, utf8_range_bad(cp, cn, lo, hi, (uint32_t)lane, 32u));
        if (lane == src && bad) code = ETL_E_UTF8;
      }
    }
    const bool light = kind_is_light(kind);
    const bool do_parse = is_text && !code && kind != ETL_K_STRING && light;
    const unsigned pm = __ballot_sync(0xffffffffu, do_parse);
    // heap space of this step's uuid cells: one warp-wide exclusive scan, one atomic
    uint64_t hpos = 0;
    {
      const bool heap_kind = do_parse && kind == ETL_K_UUID;
      const unsigned hm = __ballot_sync(0xffffffffu, heap_kind);
      if (hm) {
        unsigned long long hbase = 0;
        if (lane == 0) hbase = atomicAdd(P.heap_top, 16ull * (unsigned long long)__popc(hm));
        hbase = __shfl_sync(0xffffffffu, hbase, 0);
        hpos = hbase + 16ull * (unsigned long long)__popc(hm & ((1u << lane) - 1u));
      }
    }
    bool defer = is_text && !code && !light;
    if (do_parse) {
      // lanes of one shape bin hold the same column here; lanes of a clamped bin (more layouts than bins) may not
      const unsigned mask = __match_any_sync(pm, kind);
      code = parse_light_sync(mask, kind, tv, len, P.heap, hpos, o);
      if (code == 0xFFFFFFFFu) { code = 0; defer = true; }     // not a spelling the fast paths take: k_heavy's exact parser decides
    }
    if (is_text) {
      if (code) { report_error(P, P.dc->record_index_base + w.rec_local, tc.seq, code); w.bits &= ~WB_EMIT; }
      else if (defer) stage_put(P, st, sg, w.cell0, tc.dest, ETL_CELL_PENDING | kind, ((uint64_t)w.rec_local << 32) | tc.voff, len);
      else { stage_put(P, st, sg, w.cell0, tc.dest, o.tag, o.val, o.aux); w.hint += cell_heap_hint(o.tag, o.aux); }
    }
  }
  stage_flush(P, st, sg, w.cell0, 0);
  // ---- per-record epilogue: Partial flag, tuple bytes + size hint planes; tuple-byte metrics (one atomic per warp and op kind)
  if (my_rec != 0xFFFFFFFFu) {
    if (w.bits & WB_PARTIAL) P.rec_flags[w.rec_local] |= ETL_RF_NEW_PARTIAL;
    P.rec_tuple_bytes[w.rec_local] = w.tb;
    P.rec_heap_hint[w.rec_local] = w.hint;
  }
  const uint32_t wkind = (w.bits >> 3) & 3u;
  uint32_t tbi = wkind == WK_I ? w.tb : 0u, tbu = wkind == WK_U ? w.tb : 0u, tbd = wkind == WK_D ? w.tb : 0u;
  unsigned long long si = tbi, su = tbu, sd = tbd;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { si += __shfl_down_sync(0xffffffffu, si, d); su += __shfl_down_sync(0xffffffffu, su, d); sd += __shfl_down_sync(0xffffffffu, sd, d); }
  if (lane == 0) { if (si) atomicAdd(&P.metrics[0], si); if (su) atomicAdd(&P.metrics[1], su); if (sd) atomicAdd(&P.metrics[2], sd); }
}
// The kernel: the rows of this CTA's chunk.
__global__ void __launch_bounds__(kRowsThreads, ETL_ROWS_CTAS) k_rows(DecodeParams P) {
  extern __shared__ __align__(128) uint8_t smem[];
  if (*P.abort_flag) return;
  rows_body(P, smem);
}
#undef W_DATA_ERROR
#undef W_MALFORMED
#undef W_SET_STAGE

// ================================================================================================
// pass C3: the pending cells.
constexpr uint32_t kHeavyThreads = 256, kHeavyWarps = kHeavyThreads / 32, kHeavyTile = 4096, kHeavyStage = 128, kHeavySlot = kHeavyStage + 32;
constexpr uint32_t kHeavyListOff = 32 * 256;                                     // after kJsonT2
constexpr uint32_t kHeavyCntOff = kHeavyListOff + 3 * kHeavyTile * 2;
constexpr uint32_t kHeavySlotsOff = kHeavyCntOff + 64;
constexpr uint32_t kHeavySmemBytes = kHeavySlotsOff + kHeavyWarps * 32 * kHeavySlot + 64;
// (record, evaluation step) → the error key of a cell, recomputed from the planes: only a failing cell pays for it
__device__ __noinline__ uint32_t seq_of_cell(const DecodeParams P, uint32_t rec, uint64_t cell) {
  const uint32_t out_idx = (uint32_t)(cell - P.rec_cell_base[rec]);
  const uint32_t rf = P.rec_flags[rec];
  const DevSchema sc = P.schemas[P.schema_by_batch[P.rec_schema[rec]]];
  const uint32_t n_old = (rf & ETL_RF_OLD_FULL) ? sc.n_cols : ((rf & ETL_RF_OLD_KEY) ? sc.n_ident : 0u);
  if (out_idx >= n_old) return seq_new_cell(out_idx - n_old);
  if (rf & ETL_RF_OLD_FULL) return seq_old_cell(out_idx);
  const uint8_t* fp = P.buf + P.rec_off[rec];              // key tuple: dense (one entry per identity column) or full width
  const int32_t nc = (int32_t)(int16_t)(((uint32_t)fp[36] << 8) | fp[37]);
  if ((uint32_t)(nc < 0 ? 0 : nc) == sc.n_ident) return seq_old_cell(out_idx);
  uint32_t k = 0;
  for (uint32_t i = 0; i < sc.n_cols; i++) if (P.col_flags[sc.col_base + i] & 2) { if (k == out_idx) return seq_old_cell(i); k++; }
  return seq_old_cell(out_idx);
}
__global__ void __launch_bounds__(kHeavyThreads, 3) k_heavy(DecodeParams P) {
  extern __shared__ __align__(128) uint8_t smem[];
  if (*P.abort_flag) return;
  const uint64_t n_cells = P.total[0].n_cells;
  const uint32_t n_tiles = (uint32_t)((n_cells + kHeavyTile - 1) / kHeavyTile);
  if (blockIdx.x >= n_tiles) return;
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  for (uint32_t i = threadIdx.x; i < 32u * 256u / 16u; i += blockDim.x)       // the JSON acceptor's table
    reinterpret_cast<uint4*>(smem)[i] = reinterpret_cast<const uint4*>(kJsonT2)[i];
  uint16_t* const lists = reinterpret_cast<uint16_t*>(smem + kHeavyListOff);
  uint32_t* const cnt = reinterpret_cast<uint32_t*>(smem + kHeavyCntOff);
  uint8_t* const slot = smem + kHeavySlotsOff + (wid * 32u + lane) * kHeavySlot;
  const CellHeaps H{P.heap, P.arr_top, P.arr_base, P.heap_cap, P.heap_overflow};
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint64_t c0 = (uint64_t)tile * kHeavyTile;
    if (threadIdx.x < 4) cnt[threadIdx.x] = 0;           // [0..3) cells per class, [3] the next row to hand out
    __syncthreads();
    {   // gather: 16 tags per thread (one 16-byte load: the cell planes are 256-byte aligned and the tile is a multiple of 16)
      const uint64_t t0 = c0 + (uint64_t)threadIdx.x * 16u;
      uint4 tg = make_uint4(0, 0, 0, 0);
      if (t0 < n_cells) tg = *reinterpret_cast<const uint4*>(P.cell_tag + t0);     // the planes are padded to 256 bytes: the tail reads stay inside
      const uint32_t wv[4] = {tg.x, tg.y, tg.z, tg.w};
#pragma unroll
      for (int k = 0; k < 16; k++) {
        const uint32_t t = (wv[k >> 2] >> (8 * (k & 3))) & 0xFFu;
        if ((t & ETL_CELL_PENDING_MASK) == ETL_CELL_PENDING && t0 + k < n_cells) {
          const uint32_t kind = t & 0x3Fu;
          const uint32_t cls = kind == ETL_K_JSON ? 0u : (kind == ETL_K_NUMERIC ? 1u : 2u);
          const uint32_t at = atomicAdd(&cnt[cls], 1u);
          lists[cls * kHeavyTile + at] = (uint16_t)(threadIdx.x * 16u + k);
        }
      }
    }
    __syncthreads();
    // rows of 32 cells of one class, taken by whichever warp is free (a json row costs many times a float row: a fixed
    // row → warp assignment left warps waiting at the tile's barrier for a quarter of the kernel's samples)
    const uint32_t rows0 = (cnt[0] + 31u) >> 5, rows1 = (cnt[1] + 31u) >> 5, rows2 = (cnt[2] + 31u) >> 5;
    for (;;) {
      uint32_t row = 0;
      if (lane == 0) row = atomicAdd(&cnt[3], 1u);
      row = __shfl_sync(0xffffffffu, row, 0);
      if (row >= rows0 + rows1 + rows2) break;
      const uint32_t cls = row < rows0 ? 0u : (row < rows0 + rows1 ? 1u : 2u);
      const uint32_t n = cnt[cls];
      {
        const uint32_t base = (row - (cls == 0u ? 0u : (cls == 1u ? rows0 : rows0 + rows1))) * 32u;
        const bool have = base + lane < n;
        const uint64_t cell = c0 + (have ? lists[cls * kHeavyTile + base + lane] : 0u);
        uint32_t kind = 0, len = 0, rec = 0;
        uint64_t soff = 0;
        const uint8_t* tv = P.buf;
        if (have) {
          kind = P.cell_tag[cell] & 0x3Fu;
          const uint64_t v = P.cell_val[cell];
          len = P.cell_aux[cell];
          if (P.copy_cols) {                                // COPY rows: val locates the text itself (bit 63: an unescaped copy in the heap)
            rec = (uint32_t)(cell / P.copy_cols);
            soff = v;
            tv = ((v >> 63) ? P.heap : P.buf) + (v & ~(1ull << 63));
          } else {
            rec = (uint32_t)(v >> 32);
            soff = P.rec_off[rec] + (uint32_t)v;
            tv = P.buf + soff;
          }
          if (len <= kHeavyStage) {                         // stage the value: every 16-byte load of the lane in flight at once
            const uintptr_t a0 = reinterpret_cast<uintptr_t>(tv) & ~uintptr_t(15);
            const uint32_t nch = (uint32_t)((reinterpret_cast<uintptr_t>(tv) + len + 15u - a0) >> 4);        // ≤ 9
            const uint4* gp = reinterpret_cast<const uint4*>(a0);
            uint4 ch[9];
#pragma unroll
            for (int k = 0; k < 9; k++) ch[k] = (uint32_t)k < nch ? gp[k] : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int k = 0; k < 9; k++) if ((uint32_t)k < nch) reinterpret_cast<uint4*>(slot)[k] = ch[k];
            tv = slot + (uint32_t)(reinterpret_cast<uintptr_t>(tv) - a0);
          }
        }
        __syncwarp();
        // heap space of this row's numeric / bytea / uuid cells
        uint64_t hpos = 0;
        {
          const bool heap_kind = have && (kind == ETL_K_NUMERIC || kind == ETL_K_BYTES || kind == ETL_K_UUID);
          if (__any_sync(0xffffffffu, heap_kind)) {
            const uint32_t hb = heap_kind ? cell_heap_bound(kind, len) : 0u;
            uint32_t inc = hb;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += up; }
            const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
            unsigned long long hbase = 0;
            if (lane == 0) hbase = atomicAdd(P.heap_top, (unsigned long long)total);
            hbase = __shfl_sync(0xffffffffu, hbase, 0);
            hpos = hbase + (inc - hb);
          }
        }
        const unsigned hm = __ballot_sync(0xffffffffu, have);
        if (have) {
          const unsigned mask = cls == 2u ? __match_any_sync(hm, kind) : hm;      // the json / numeric lists hold one class each
          CellOut o;
          o.tag = 0; o.val = 0; o.aux = 0;
          const uint32_t code = parse_heavy_sync(mask, kind, tv, len, soff, H, hpos, smem, o);
          if (code) report_error(P, P.dc->record_index_base + rec, P.copy_cols ? 1u + (uint32_t)(cell % P.copy_cols) : seq_of_cell(P, rec, cell), code);
          else {
            put_cell(P, cell, o.tag, o.val, o.aux);
            const uint32_t h = P.copy_cols ? 0u : cell_heap_hint(o.tag, o.aux);
            if (h) atomicAdd(&P.rec_heap_hint[rec], h);
          }
        }
        __syncwarp();
      }
    }
    __syncthreads();
  }
}

// pass C4: unchanged-TOAST cells whose source was pending in k_rows take the parsed value now (event.rs:958-970: a clone)
__global__ void __launch_bounds__(256) k_fix(DecodeParams P) {
  if (*P.abort_flag || *P.copy_count == 0u) return;
  const uint64_t n_cells = P.total[0].n_cells;
  for (uint64_t t0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16u; t0 < n_cells; t0 += (uint64_t)gridDim.x * blockDim.x * 16u) {
    const uint4 tg = *reinterpret_cast<const uint4*>(P.cell_tag + t0);
    const uint32_t wv[4] = {tg.x, tg.y, tg.z, tg.w};
    if (!(((tg.x | tg.y | tg.z | tg.w) & 0x80808080u))) continue;
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const uint32_t t = (wv[k >> 2] >> (8 * (k & 3))) & 0xFFu;
      if (t == ETL_CELL_PENDING_COPY && t0 + k < n_cells) {
        const uint64_t src = P.cell_val[t0 + k];
        const uint32_t rec = P.cell_aux[t0 + k];
        const uint32_t stag = P.cell_tag[src], saux = P.cell_aux[src];
        put_cell(P, t0 + k, stag, P.cell_val[src], saux);
        const uint32_t h = cell_clone_hint(stag, saux);
        if (h) atomicAdd(&P.rec_heap_hint[rec], h);
      }
    }
  }
}

}  // namespace etl
