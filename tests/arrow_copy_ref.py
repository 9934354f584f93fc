"""Expected columns of etl_dec_arrow_emit for COPY-row batches and for ETL_ARROW_CDC_COLUMNS, on top of the encoder
restatements of tests/arrow_ref.py.

* expected_row_columns: a per-row entry point — the columns built from rows given as decoded cell values (the oracle's
  per-row COPY parse), with and without ETL_ARROW_ALL_COLUMNS.
* sequence_key / CDC_OP: EventSequenceKey's Display (crates/etl/src/types/event.rs:331-336) and IcebergOperationType's
  Display (crates/etl-destinations/src/iceberg/core.rs:82-90); expected_cdc_columns applies them to a batch's records.
* first_skipped: the record etl_dec_arrow_first_skipped reports (write_events' InvalidState cases,
  iceberg/core.rs:311-322 and :336-357).
"""
from __future__ import annotations

import numpy as np

from arrow_ref import A_LBIN, A_UNSUP, A_UTF8, KIND2ARROW, cell_text, element_value

CDC_COLUMNS = 0x200
CDC_OP = {ord("I"): b"INSERT", ord("U"): b"UPDATE", ord("D"): b"DELETE"}


def sequence_key(commit_lsn: int, tx_ordinal: int) -> bytes:
    """EventSequenceKey's Display; a COPY row's key is that of (0, 0)"""
    return ("%016x/%016x" % (commit_lsn, tx_ordinal)).encode()


def _var_column(chunks):
    """(valid[], offsets[], data) of var-width entries (None = null)"""
    valid = np.array([t is not None for t in chunks], dtype=bool)
    offs = np.zeros(len(chunks) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(t or b"") for t in chunks])
    return valid, offs, b"".join(t or b"" for t in chunks)


def utf8_column(texts):
    """an entry in arrow_ref.expected_formatted_columns' "utf8" form"""
    return ("utf8",) + _var_column(texts)


def list_column(kind, cells):
    """an entry in arrow_ref.expected_formatted_columns' "list" form (build_list_array, encoding.rs:386-776)"""
    ct = KIND2ARROW.get(kind & 0x1F, A_UNSUP)
    is_arr = [isinstance(v, tuple) and v[0] == "array" for v in cells]
    loffs = np.zeros(len(cells) + 1, dtype=np.int64)
    loffs[1:] = np.cumsum([len(v[2]) if a else 0 for v, a in zip(cells, is_arr)])
    ev = [element_value(ct, e) for v, a in zip(cells, is_arr) if a for e in v[2]]
    cvalid = np.array([ok for ok, _ in ev], dtype=bool)
    if ct in (A_UTF8, A_LBIN):
        chunks = [x if ok else b"" for ok, x in ev]
        coffs = np.zeros(len(chunks) + 1, dtype=np.int64)
        coffs[1:] = np.cumsum([len(x) for x in chunks])
        child = (coffs, b"".join(chunks))
    else:
        child = [x if ok else None for ok, x in ev]
    return ("list", np.array(is_arr, dtype=bool), loffs, ct, cvalid, child)


def expected_row_columns(kinds, rows, all_columns: bool):
    """the columns etl_dec_arrow_emit builds from rows given as decoded cell values (canon.decode_cell's form, one list
    per row in column order) of a table whose columns have the ETL_K_* classes `kinds`:
    {column: ("unsupported",) | ("fixed", arrow_type, valid[], values (None for nulls)) | ("lbin", valid[], offsets[], data)
    | "utf8" / "list" entries as above}"""
    out = {}
    for c, kind in enumerate(kinds):
        kind = int(kind)
        cells = [r[c] for r in rows]
        if kind & 0x20:
            out[c] = list_column(kind, cells) if all_columns else ("unsupported",)
            continue
        at = KIND2ARROW.get(kind, A_UNSUP) if all_columns or kind not in (9, 15) else A_UNSUP
        if at == A_UNSUP:
            out[c] = ("unsupported",)
        elif at == A_UTF8:
            out[c] = utf8_column([cell_text(v) for v in cells])
        elif at == A_LBIN:
            out[c] = ("lbin",) + _var_column([v[1] if v is not None else None for v in cells])
        else:
            ev = [element_value(at, v) for v in cells]
            out[c] = ("fixed", at, np.array([ok for ok, _ in ev], dtype=bool), [x if ok else None for ok, x in ev])
    return out


def expected_cdc_columns(p, records):
    """(cdc_operation, sequence_number) as "utf8" entries, for rows of the given records of a decoded batch's planes;
    p = None for COPY rows (INSERT, the key of (0, 0))"""
    if p is None:
        return utf8_column([CDC_OP[ord("I")]] * len(records)), utf8_column([sequence_key(0, 0)] * len(records))
    ops = [CDC_OP[int(p.rec_kind[r])] for r in records]
    keys = [sequence_key(int(p.rec_commit_lsn[r]), int(p.rec_tx_ordinal[r])) for r in records]
    return utf8_column(ops), utf8_column(keys)


def first_skipped(p, schema_index: int, row_kinds: int) -> int:
    """the smallest record of the schema version in the valid prefix that row_kinds selects but that has no full image
    (an Update with a partial new row under bit 1, a Delete without a full old row under bit 2); 2**64 - 1 if none"""
    n = p.n_records if p.first_error[0] is None else p.first_error[0]
    kind, flags = p.rec_kind[:n].astype(np.int64), p.rec_flags[:n].astype(np.int64)
    mine = (p.rec_schema[:n] == schema_index) & ((flags & 0x80) != 0)
    skip = np.zeros(n, dtype=bool)
    if row_kinds & 2:
        skip |= (kind == ord("U")) & ((flags & 4) != 0)
    if row_kinds & 4:
        skip |= (kind == ord("D")) & ((flags & 1) == 0)
    hit = np.flatnonzero(mine & skip)
    return int(hit[0]) if len(hit) else 2**64 - 1
