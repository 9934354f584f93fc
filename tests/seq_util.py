"""Sequences of batches on ONE decode context — the way the library runs in production (one long-lived etl_dec_ctx
that decodes batch after batch) — checked against ONE oracle context driven through the same steps.

A step is one of:
  Decode(stream, ...)      one batch (etl_dec_decode, or decode_begin / decode_finish with two_phase=True)
  PutTableSchema(id, cols) etl_dec_put_table_schema between batches
  ResetRelations()         etl_dec_reset_relations between batches
  CopyDecode(id, rows)     COPY-text rows on the same context (etl_dec_copy_decode)
Each side threads its own carry_out into its next batch; every batch is compared plane by plane.

`stitched_check` compares a sequence of batches cut from one stream with the oracle's decode of the WHOLE stream,
which pins cross-batch semantics to a single decode rather than to the oracle's own sequence behaviour.
"""
from __future__ import annotations

from collections import Counter
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from canon import assert_planes_equal
from shard_util import schema_maps, stitch

SIZING = {"EXACT": 0x01, "OPTIMISTIC": 0x02, "RERUN_RECORDS": 0x04, "RERUN_CELLS": 0x08, "SCRATCH_RESTART": 0x10,
          "ARRAY_HEAP_RETRY": 0x20, "LONG_PASSES_LATE": 0x40}       # etl_dec_summary.sizing (ETL_SIZING_*)
RERUN = SIZING["RERUN_RECORDS"] | SIZING["RERUN_CELLS"]


def sizing_names(bits: int) -> List[str]:
    return [n for n, b in SIZING.items() if bits & b]


@dataclass
class Decode:
    stream: bytes
    stride: int = 2048
    max_frame_len: Optional[int] = None   # None: the stager's own hint; else an override (0 = unknown)
    two_phase: bool = False
    label: str = ""


@dataclass
class PutTableSchema:
    table_id: int
    cols: list


@dataclass
class ResetRelations:
    pass


@dataclass
class CopyDecode:
    table_id: int
    rows: list                            # COPY-text rows, each with its LF


@dataclass
class BatchResult:
    got: object                           # DecodedBatch (device)
    want: object                          # oracle Planes
    stream: bytes
    sizing: int
    label: str = ""


@dataclass
class SequenceResult:
    batches: List[BatchResult] = field(default_factory=list)

    @property
    def sizing(self) -> List[int]:
        return [b.sizing for b in self.batches]

    def histogram(self) -> Counter:
        return Counter(n for b in self.batches for n in sizing_names(b.sizing))


def run_sequence(gpu, oracle_mod, steps: Sequence, tables: Dict[int, list], reuse_stager: bool = False,
                 check: bool = True) -> SequenceResult:
    """Drive one Decoder and one Oracle through `steps`.  reuse_stager: stage every batch through one Stager per
    anchor stride, reset between batches (the stager's production use) instead of a new one per batch."""
    dec = gpu.Decoder(0)
    orc = oracle_mod.Oracle()
    schemas = dict(tables)
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
        orc.put_table_schema(tid, cols)
    cap = max([len(s.stream) for s in steps if isinstance(s, Decode)] + [1])
    stagers = {}
    out = SequenceResult()
    g_carry = w_carry = None
    try:
        for i, s in enumerate(steps):
            if isinstance(s, PutTableSchema):
                dec.put_table_schema(s.table_id, s.cols)
                orc.put_table_schema(s.table_id, s.cols)
                schemas[s.table_id] = s.cols
            elif isinstance(s, ResetRelations):
                dec.reset_relations()
                orc.reset_relations()
            elif isinstance(s, CopyDecode):
                _copy_step(dec, oracle_mod, [c["type_oid"] for c in schemas[s.table_id]], s, i)
            else:
                if reuse_stager:
                    st = stagers.get(s.stride)
                    if st is None:
                        st = stagers[s.stride] = gpu.Stager(cap, s.stride)
                    st.reset()
                else:
                    st = gpu.Stager(max(len(s.stream), 1), s.stride)
                try:
                    st.append_framed(s.stream)
                    inp = st.view()
                    if s.max_frame_len is not None:
                        inp.max_frame_len = int(s.max_frame_len)
                    if s.two_phase:
                        dec.decode_begin(inp, to_host=True)
                        bh = dec.decode_finish(g_carry or (0, 0, 0), 0)
                    else:
                        gpu.Decoder._carry(inp, g_carry)
                        bh = dec.decode_input(inp, to_host=True)
                    with bh:
                        got = bh.to_host()
                finally:
                    if not reuse_stager:
                        st.close()
                want = orc.decode(s.stream, w_carry)
                label = s.label or f"batch {len(out.batches)}"
                if check:
                    try:
                        assert_planes_equal(got, want, s.stream)
                    except AssertionError as e:
                        raise AssertionError(f"step {i} ({label}, {len(s.stream)} bytes, sizing {sizing_names(got.sizing)}): {e}") from e
                out.batches.append(BatchResult(got, want, s.stream, got.sizing, label))
                g_carry, w_carry = got.carry_out, want.carry_out
    finally:
        for st in stagers.values():
            st.close()
        dec.close()
        orc.close()
    return out


def _copy_step(dec, oracle_mod, oids, s: CopyDecode, i: int):
    offs = np.zeros(len(s.rows) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in s.rows])
    buf = np.frombuffer(b"".join(s.rows), dtype=np.uint8)
    want, err = oracle_mod.copy_rows_digest(oids, buf, offs)
    b = dec.copy_decode(s.table_id, buf, offs)
    if err is None:
        assert b.first_error[0] is None, (i, b.first_error)
        n_ok = len(s.rows)
    else:
        n_ok = err[0]
        assert b.first_error[0] == err[0], (i, b.first_error, err)
    got = oracle_mod.copy_planes_digest(b.cell_tag, b.cell_val, b.cell_aux, n_ok, len(oids), b.stream, b.heap)
    assert got == want, f"step {i}: COPY rows differ from the oracle"


# ------------------------------------------------------------------------------------------------ cutting a stream
def record_cuts(full, total_len: int, rng: np.random.Generator, lo: int, hi: int, first_min: int = 0,
                max_parts: Optional[int] = None) -> List[int]:
    """Byte offsets [0, c1, …, end] cutting a stream (decoded as `full`) at record starts into parts of log-uniform
    size in [lo, hi] (the first at least `first_min`).  No part starts with a Relation frame (its effective_off would
    read as "carried in", see shard_util.schema_maps).  With max_parts the stream is truncated after that many parts."""
    starts = np.asarray(full.rec_off[:full.n_records], dtype=np.int64)
    kinds = np.asarray(full.rec_kind[:full.n_records])
    cand = starts[(kinds != ord("R")) & (starts > 0)]
    cuts = [0]
    while max_parts is None or len(cuts) <= max_parts:
        size = float(np.exp(rng.uniform(np.log(lo), np.log(hi))))
        if len(cuts) == 1:
            size = max(size, first_min)
        j = int(np.searchsorted(cand, cuts[-1] + int(size)))
        if j >= len(cand):
            break
        cuts.append(int(cand[j]))
    if max_parts is None or len(cuts) <= max_parts:
        cuts.append(total_len)
    return cuts


def next_cut(full, target: int) -> int:
    """The first record start at or after byte `target` that is not a Relation frame."""
    starts = np.asarray(full.rec_off[:full.n_records], dtype=np.int64)
    kinds = np.asarray(full.rec_kind[:full.n_records])
    j = int(np.searchsorted(starts, target))
    while kinds[j] == ord("R"):
        j += 1
    return int(starts[j])


def stitched_check(oracle_mod, tables: Dict[int, list], raw: bytes, cuts: Sequence[int], parts: Sequence):
    """parts[k] decoded raw[cuts[k]:cuts[k+1]] as the k-th batch of one sequence (carry threaded, relations carried):
    stitched, they must equal a fresh oracle's decode of raw[:cuts[-1]] on every plane, the schema versions and the
    carry-out.  Array cells are not supported (stitch does not rebase element offsets)."""
    whole = bytes(raw[:cuts[-1]])
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        orc.put_table_schema(tid, cols)
    full = orc.decode(whole)
    orc.close()
    assert full.first_error[0] is None, full.first_error
    for k, p in enumerate(parts):
        assert p.first_error[0] is None, (k, p.first_error)
        assert not np.any(np.asarray(p.cell_tag) == 17), "stitch does not rebase array cells"
    got = stitch(parts, cuts, schema_maps(full, parts, cuts))
    got.schemas = full.schemas                          # compared through the mapping
    assert_planes_equal(got, full, whole)
    return full
