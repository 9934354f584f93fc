// copy_kernel.cuh — initial-sync COPY-text rows on the device (SURVEY §8f N1).
//
//   k_copy_rows   parse_table_row_from_postgres_copy_bytes (crates/etl/src/conversions/table_row.rs:25-165), one
//                 THREAD per row, one warp per 32 rows, the rows staged into shared memory by bulk async copies
//                 exactly like k_rows stages frames.  A row is walked field by field: an 8-byte SWAR scan finds the
//                 next TAB / LF / backslash; a field without a backslash is a zero-copy span of the staged buffer,
//                 `\N` alone is NULL, anything else with an escape is unescaped into the heap (table_row.rs:46-71).
//                 The lanes stay in lockstep by column, so the light decode classes are parsed in place with the
//                 same warp-synchronous parsers as the replication path; the other classes are left as PENDING
//                 cells for k_heavy (rows_kernel.cuh), which serves both paths.
//
// Row-level rules restated from the reference: the whole row must be UTF-8 before anything else is looked at (:33);
// TAB ends a field, LF ends a field and marks the row terminated, and the scan goes on to the end of the input;
// input ending without any LF → "Row data not properly terminated" (:88-96); one field too many → column-count error
// as soon as it is met (:103-113); too few → at the end (:150-160).  Error order inside a row = the order in which
// the reference would raise them: UTF-8 first (step 0), then by field position (step 1 + column).
#pragma once

namespace etl {

constexpr uint64_t COPY_IN_HEAP = 1ull << 63;     // string / json cell: val = heap offset (unescaped copy) instead of a stream offset

__device__ __forceinline__ void copy_error(const DecodeParams& P, uint32_t row, uint32_t step, uint32_t code) {
  report_error(P, P.dc->record_index_base + row, step, code);
}
// bytes of x (8 bytes, little endian) equal to c → 0x80 in that byte
__device__ __forceinline__ uint64_t swar_eq(uint64_t x, uint32_t c) {
  const uint64_t L7 = 0x7F7F7F7F7F7F7F7Full;
  const uint64_t u = x ^ (0x0101010101010101ull * c);
  return ~(((u & L7) + L7) | u) & 0x8080808080808080ull;
}

// P.copy_cols = columns of the table; P.rec_off[r] .. P.rec_off[r + 1] = row r; cells row-major in the cell plane.
__global__ void __launch_bounds__(kRowsThreads, ETL_ROWS_CTAS) k_copy_rows(DecodeParams P) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (uint32_t k = 0; k < kRowsWarps; k++) mbar_init(smem_u32(smem + kRowsBarOff + 8u * k), 32u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t bar = smem_u32(smem + kRowsBarOff + 8u * wid);
  uint8_t* const slot = smem + kCopySlotsOff + ((uint32_t)wid * 32u + (uint32_t)lane) * kCopySlot;
  const uint32_t slot_s = smem_u32(slot);
  uint32_t parity = 0;
  const uint32_t n_rows = (uint32_t)P.total[0].n_rec, n_cols = P.copy_cols;
  const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = row < n_rows;
  if (__ballot_sync(0xffffffffu, valid) == 0) return;
  // column classes: the warp's shared-memory copy (every row of a COPY stream belongs to one table)
  const uint8_t* kinds = P.col_kind;
  if (n_cols <= kRowsColsCached) {
    uint8_t* ck = smem + kRowsColsOff + (uint32_t)wid * 2u * kRowsColsCached;
    for (uint32_t i = (uint32_t)lane; i < n_cols; i += 32u) ck[i] = P.col_kind[i];
    __syncwarp();
    kinds = ck;
  }
  const uint64_t goff = valid ? P.rec_off[row] : 0;
  const uint32_t end = valid ? (uint32_t)(P.rec_off[row + 1] - goff) : 0u;
  const uint64_t cell0 = (uint64_t)row * n_cols;
  uint32_t pos = 0, fstart = 0, col = 0;
  bool done = !valid, terminated = false, has_esc = false, esc = false, emit = true, found = false;
  uint64_t hib = 0;                                   // OR of every byte of the row: any high bit → the row is checked for UTF-8
  RowWin W;
  W.win = slot; W.delta = 0x7FFFFFFF; W.w1 = 0;
  for (;;) {
    if (!__any_sync(0xffffffffu, !done)) break;
    // ---- scan for the end of the current field inside the window (a lane that has found it waits for the others:
    // the fields are processed together, column by column)
    bool need = false;
    if (!done && !found) {
      for (;;) {
        if (pos >= end) break;
        if (!((int32_t)pos >= W.delta && pos < W.w1)) { need = true; break; }
        const uint32_t lim = min(W.w1, end);
        if (esc) {                                    // the character after a backslash is taken whatever it is (:46-71)
          hib |= (uint64_t)W.win[(int32_t)pos - W.delta];
          pos += 1; esc = false;
          continue;
        }
        const uint32_t k = min(8u, lim - pos);
        uint64_t x = ld64u(W.win + ((int32_t)pos - W.delta));
        if (k < 8u) x &= (1ull << (8u * k)) - 1ull;
        const uint64_t m = swar_eq(x, '\t') | swar_eq(x, '\n') | swar_eq(x, '\\');   // zero padding bytes match nothing
        if (!m) { hib |= x; pos += k; continue; }
        const uint32_t p = (uint32_t)(__ffsll((long long)m) - 1) >> 3;
        hib |= x & ((1ull << (8u * p)) - 1ull);
        pos += p;
        if (((uint32_t)(x >> (8u * p)) & 0xFFu) == '\\') { has_esc = true; esc = true; pos += 1; continue; }
        found = true;
        break;
      }
    }
    if (__any_sync(0xffffffffu, need)) {              // some lane ran out of window: restage every live lane
      __syncwarp();
      uint32_t n = 0;
      const uint32_t from = found ? fstart : pos;     // a lane that waits keeps its field in the window when it fits
      if (!done && from < end) {
        const uint64_t g0 = (goff + from) & ~15ull;
        const uint64_t gend = (goff + end + 15ull) & ~15ull;
        n = (uint32_t)min((uint64_t)kCopyWin, gend - g0);
        W.delta = (int32_t)((int64_t)g0 - (int64_t)goff);
        W.w1 = (uint32_t)(W.delta + (int32_t)n);
        mbar_arrive_expect_tx(bar, n);
        bulk_g2s(slot_s, P.buf + g0, n, bar);
      } else mbar_arrive(bar);
      mbar_wait(bar, parity);
      parity ^= 1u;
      continue;
    }
    // ---- end of input without a terminator for this field
    if (!done && !found && pos >= end) {
      if (!terminated) copy_error(P, row, 1u + col, ETL_E_COPY_NOT_TERMINATED);       // table_row.rs:88-92
      else if (col < n_cols) copy_error(P, row, 1u + col, ETL_E_COPY_COLUMN_COUNT);   // :150-160
      done = true;
    }
    // ---- a complete field: [fstart, pos), terminator at pos
    const bool have = !done && found;
    uint32_t kind = 0, flen = 0, mycol = 0;
    uint64_t soff = 0;
    const uint8_t* tv = P.buf;
    bool text_cell = false;
    uint32_t code = 0;
    if (have) {
      // the terminator byte is ASCII: read it from global memory when it fell out of the window
      const uint32_t tch = ((int32_t)pos >= W.delta && pos < W.w1) ? (uint32_t)W.win[(int32_t)pos - W.delta] : (uint32_t)P.buf[goff + pos];
      if (tch == '\n') terminated = true;
      flen = pos - fstart; mycol = col;
      const uint32_t f0 = fstart;
      pos += 1; fstart = pos; col++;
      if (mycol >= n_cols) { copy_error(P, row, 1u + mycol, ETL_E_COPY_COLUMN_COUNT); emit = false; }   // :103-113 (the scan goes on for the UTF-8 verdict)
      else if (emit) {
        kind = kinds[mycol];
        soff = goff + f0;
        const bool in_win = (int32_t)f0 >= W.delta && f0 + flen <= W.w1;
        tv = in_win ? W.win + ((int32_t)f0 - W.delta) : P.buf + soff;
        if (has_esc) {
          if (flen == 2u && tv[0] == '\\' && tv[1] == 'N') put_cell(P, cell0 + mycol, ETL_CELL_NULL, 0, 0);   // :116-121
          else {                                        // unescape into the heap (:46-71); rare, lane-serial
            const uint64_t at = atomicAdd(P.heap_top, (unsigned long long)((flen + 7u) & ~7u));
            uint8_t* d = P.heap + at;
            uint32_t n = 0;
            for (uint32_t i = 0; i < flen; i++) {
              uint32_t c = tv[i];
              if (c == '\\' && i + 1 < flen) {
                c = tv[++i];
                if (c == 'N') { d[n++] = '\\'; }
                else if (c == 'b') c = 8; else if (c == 'f') c = 12; else if (c == 'n') c = '\n';
                else if (c == 'r') c = '\r'; else if (c == 't') c = '\t'; else if (c == 'v') c = 11;
              } else if (c == '\\') continue;           // a trailing lone backslash (the row ended inside an escape)
              d[n++] = (uint8_t)c;
            }
            if (n == 2u && d[0] == '\\' && d[1] == 'N') put_cell(P, cell0 + mycol, ETL_CELL_NULL, 0, 0);
            else if (kind == ETL_K_STRING) put_cell(P, cell0 + mycol, ETL_CELL_STRING, COPY_IN_HEAP | at, n);
            else put_cell(P, cell0 + mycol, ETL_CELL_PENDING | kind, COPY_IN_HEAP | at, n);   // parsed from the heap copy by k_heavy
          }
        } else if (kind == ETL_K_STRING) put_cell(P, cell0 + mycol, ETL_CELL_STRING, soff, flen);
        else text_cell = true;
      }
      has_esc = false; found = false;
    }
    // ---- the light classes in place (lanes are on the same column unless a row needed an extra window)
    const bool light = kind_is_light(kind);
    const bool do_parse = text_cell && light;
    const unsigned pm = __ballot_sync(0xffffffffu, do_parse);
    uint64_t hpos = 0;
    {
      const unsigned hm = __ballot_sync(0xffffffffu, do_parse && kind == ETL_K_UUID);
      if (hm) {
        unsigned long long hbase = 0;
        if (lane == 0) hbase = atomicAdd(P.heap_top, 16ull * (unsigned long long)__popc(hm));
        hbase = __shfl_sync(0xffffffffu, hbase, 0);
        hpos = hbase + 16ull * (unsigned long long)__popc(hm & ((1u << lane) - 1u));
      }
    }
    bool defer = text_cell && !light;
    CellOut o;
    o.tag = 0; o.val = 0; o.aux = 0;
    if (do_parse) {
      const unsigned mask = __match_any_sync(pm, kind);
      code = parse_light_sync(mask, kind, tv, flen, P.heap, hpos, o);
      if (code == 0xFFFFFFFFu) { code = 0; defer = true; }
    }
    if (text_cell) {
      if (code) { copy_error(P, row, 1u + mycol, code); emit = false; }
      else if (defer) put_cell(P, cell0 + mycol, ETL_CELL_PENDING | kind, soff, flen);
      else put_cell(P, cell0 + mycol, o.tag, o.val, o.aux);
    }
  }
  // ---- str::from_utf8(row) (:33): rows with a high bit anywhere are validated whole, by the warp, from global memory
  for (unsigned sm = __ballot_sync(0xffffffffu, valid && (hib & 0x8080808080808080ull) != 0ull); sm; sm &= sm - 1) {
    const int src = __ffs(sm) - 1;
    const uint64_t g = __shfl_sync(0xffffffffu, goff, src);
    const uint32_t n = __shfl_sync(0xffffffffu, end, src);
    const bool bad = __any_sync(0xffffffffu, utf8_range_bad(P.buf + g, n, 0u, n, (uint32_t)lane, 32u));
    if (lane == src && bad) copy_error(P, row, 0u, ETL_E_UTF8);
  }
}

}  // namespace etl
