"""Helpers for the sharded-decode tests: cut one stream into byte ranges at record starts and stitch the
per-range planes back into one batch that can be compared with the oracle's decode of the whole stream."""
from __future__ import annotations

from types import SimpleNamespace
from typing import List, Sequence

import numpy as np

STREAM_SPAN_TAGS = (2, 15)            # String / Json: val = offset into the staged stream
HEAP_TAGS = (9, 14, 16, 17)           # Numeric / Uuid / Bytes / Array: val = heap offset


def mid_tx_cuts(full, n_parts: int) -> List[int]:
    """Byte offsets cutting the stream decoded as `full` (oracle planes) into n_parts ranges at DML records that
    follow a DML record (i.e. inside a transaction)."""
    kinds = [chr(k) for k in full.rec_kind]
    cuts = [0]
    for f in range(1, n_parts):
        i = next(i for i in range(full.n_records * f // n_parts, full.n_records) if kinds[i] in "IUD" and kinds[i - 1] in "IUD")
        cuts.append(int(full.rec_off[i]))
    return cuts


def schema_maps(full, parts: Sequence, cuts: Sequence[int]) -> List[List[int]]:
    """Per range: local schema index → index in `full.schemas` (the whole-stream decode).  A range numbers its
    schema versions itself: the versions in force at its first byte (effective_off 0), then its own Relation frames
    (effective_off = offset inside the range).  A range must therefore not start with a Relation frame: its
    effective_off would be 0 as well."""
    want_index = {}
    for i, s in enumerate(full.schemas):
        want_index.setdefault(int(s.table_id), []).append((int(s.effective_off), i))
    maps = []
    for k, p in enumerate(parts):
        m = []
        for s in p.schemas:
            off = s.effective_off + cuts[k] if s.effective_off else None      # None: the version in force at the range's first byte
            cands = want_index[s.table_id]
            if off is None:
                prior = [i for (o, i) in cands if o < cuts[k]] or [cands[0][1]]
                m.append(prior[-1])
            else:
                m.append(next(i for (o, i) in cands if o == off))
        maps.append(m)
    return maps


def stitch(parts: Sequence, cuts: Sequence[int], schema_maps=None):
    """Concatenate per-range DecodedBatch objects (range k starts at byte cuts[k]) into one batch in the layout of
    a whole-stream decode.  Array cells are left out of the heap fix-up (not used by these tests).
    schema_maps[k][local index] = index in the whole-stream numbering (default: identity)."""
    rec_off, cell_val, cell_base, heaps, rec_schema = [], [], [], [], []
    cells_before, heap_before = 0, 0
    for k, p in enumerate(parts):
        rec_off.append(p.rec_off + np.uint64(cuts[k]))
        v = p.cell_val.copy()
        span = np.isin(p.cell_tag, STREAM_SPAN_TAGS)
        v[span] += np.uint64(cuts[k])
        hp = np.isin(p.cell_tag, HEAP_TAGS)
        v[hp] += np.uint64(heap_before)
        cell_val.append(v)
        cell_base.append(p.rec_cell_base[:-1] + np.uint64(cells_before))
        sc = p.rec_schema.copy()
        if schema_maps is not None:
            m = np.asarray(schema_maps[k], dtype=np.int32)
            sc = np.where(sc >= 0, m[np.maximum(sc, 0)], sc).astype(np.int32)
        rec_schema.append(sc)
        heaps.append(p.heap)
        cells_before += int(p.rec_cell_base[-1])
        heap_before += int(p.heap.nbytes)
    cat = lambda name: np.concatenate([getattr(p, name) for p in parts])  # noqa: E731
    first_errors = [p.first_error for p in parts if p.first_error[0] is not None]
    fe = min(first_errors, key=lambda e: e[0]) if first_errors else parts[0].first_error
    return SimpleNamespace(
        n_records=sum(p.n_records for p in parts), n_cells=cells_before,
        rec_off=np.concatenate(rec_off), rec_kind=cat("rec_kind"), rec_flags=cat("rec_flags"), rec_rel=cat("rec_rel"),
        rec_schema=np.concatenate(rec_schema), rec_start_lsn=cat("rec_start_lsn"), rec_commit_lsn=cat("rec_commit_lsn"),
        rec_tx_ordinal=cat("rec_tx_ordinal"), rec_tuple_bytes=cat("rec_tuple_bytes"), rec_heap_hint=cat("rec_heap_hint"),
        rec_cell_base=np.concatenate(cell_base + [np.array([cells_before], dtype=np.uint64)]),
        cell_tag=cat("cell_tag"), cell_val=np.concatenate(cell_val), cell_aux=cat("cell_aux"), heap=np.concatenate(heaps),
        first_error=fe, carry_out=parts[-1].carry_out,
        insert_bytes=sum(p.insert_bytes for p in parts), update_bytes=sum(p.update_bytes for p in parts),
        delete_bytes=sum(p.delete_bytes for p in parts), n_events=sum(p.n_events for p in parts), schemas=parts[0].schemas)
