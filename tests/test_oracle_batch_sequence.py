"""The oracle's own semantics over a sequence of batches on one context (CPU only).

The GPU batch-sequence tests (test_gpu_batch_sequence.py) compare batch N of a device session with batch N of an
oracle session, so the oracle's sequence behaviour is pinned here first: a stream cut into batches at seeded record
boundaries (some inside transactions) and decoded batch after batch, carry threaded, must stitch back to the oracle's
decode of the whole stream — every plane, the schema versions and the carry-out."""
import numpy as np
import pytest

from canon import assert_planes_equal
from etl_b200 import pgoutput as pg
from etl_b200 import workloads as wl
import scenarios as sc
from seq_util import record_cuts, stitched_check


def _oracle_sequence(oracle_mod, tables, raw, cuts):
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        orc.put_table_schema(tid, cols)
    parts, carry = [], None
    for k in range(len(cuts) - 1):
        p = orc.decode(raw[cuts[k]:cuts[k + 1]], carry)
        parts.append(p)
        carry = p.carry_out
    orc.close()
    return parts


@pytest.mark.parametrize("name,scale,seed", [("c2", 0.004, 1), ("c2", 0.004, 2), ("c4", 0.0004, 3), ("c4", 0.0004, 4), ("c5", 0.0003, 5)])
def test_oracle_sequence_equals_whole_stream(oracle_mod, name, scale, seed):
    w = wl.make(name, scale, n_segments=1)
    if name == "c4":
        w.schema_bump_ppm = 3000                         # Relation re-sends with replica-identity flips mid-stream
    stream, _ = w.generate()
    raw = stream.tobytes()
    tables = w.table_schemas()
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        orc.put_table_schema(tid, cols)
    full = orc.decode(raw)
    orc.close()
    cuts = record_cuts(full, len(raw), np.random.default_rng(seed), 512, 256 << 10)
    assert len(cuts) >= 8
    kinds = [chr(k) for k in full.rec_kind]
    starts = {int(o): i for i, o in enumerate(full.rec_off)}
    in_tx = [c for c in cuts[1:-1] if kinds[starts[c]] in "IUD" and kinds[starts[c] - 1] in "IUD"]
    assert in_tx, "no cut falls inside a transaction"
    parts = _oracle_sequence(oracle_mod, tables, raw, cuts)
    assert any(p.carry_out[0] for p in parts[:-1])
    if name == "c4":
        assert sum(len(p.schemas) for p in parts[1:]) > len(parts) - 1   # later batches carry versions in
    stitched_check(oracle_mod, tables, raw, cuts, parts)


def _lifecycle_tables():
    cols = [sc.col("id", sc.INT8, 1), sc.col("a", sc.TEXT, None, True), sc.col("b", sc.INT4, None, True)]
    return {70: cols}, cols


def test_oracle_relation_after_data_error_is_not_installed(oracle_mod):
    """A batch whose data error comes BEFORE a Relation frame: the Relation is not in force in the next batch (the
    reference bails out before caching it), the version before it still is."""
    tables, cols = _lifecycle_tables()
    v2 = pg.relation(70, "public", "t", "d", sc.rel_cols(cols, {"id"}))
    v3 = pg.relation(70, "public", "t", "d", sc.rel_cols(cols[:2], {"id"}))
    b1 = sc.stream_with(None, [v2], [pg.insert(70, ["1", "x", "2"])]).bytes()
    b2 = sc.stream_with(None, [], [pg.insert(70, ["2", "y", "bad"]), v3, pg.insert(70, ["3", "z"])]).bytes()
    b3 = sc.stream_with(None, [], [pg.insert(70, ["4", "w", "5"]), pg.insert(70, ["5", "v"])]).bytes()
    orc = oracle_mod.Oracle()
    orc.put_table_schema(70, cols)
    p1 = orc.decode(b1)
    assert p1.first_error[0] is None
    p2 = orc.decode(b2, p1.carry_out)
    assert p2.first_error[0] == 1 and p2.first_error[2] == 2          # int4 "bad": before v3
    p3 = orc.decode(b3, p2.carry_out)
    assert p3.first_error[0] == 2 and p3.first_error[2] == 12         # a v3-shaped row under v2: field count
    assert len(p3.schemas) == 1 and p3.schemas[0].n_cols == 3 and int(p3.rec_schema[1]) == 0
    # the same three batches without the error: v3 is in force afterwards
    b2ok = sc.stream_with(None, [], [pg.insert(70, ["2", "y", "7"]), v3, pg.insert(70, ["3", "z"])]).bytes()
    orc2 = oracle_mod.Oracle()
    orc2.put_table_schema(70, cols)
    q1 = orc2.decode(b1)
    q2 = orc2.decode(b2ok, q1.carry_out)
    assert q2.first_error[0] is None
    q3 = orc2.decode(b3, q2.carry_out)
    assert q3.first_error[0] == 1 and q3.first_error[2] == 12         # now the v2-shaped row is the wrong one
    assert q3.schemas[0].n_cols == 2
    orc.close()
    orc2.close()


def test_oracle_carried_versions_ascend_by_table_id(oracle_mod):
    """Versions carried into a batch come first and ascend by table id, whatever order the tables were announced in
    (the device numbers them the same way: rec_schema is compared index for index)."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("v", sc.TEXT, None, True)]
    tables = {91: cols, 90: cols}
    rels = [pg.relation(t, "public", f"t{t}", "d", sc.rel_cols(cols, {"id"})) for t in (91, 90)]
    b1 = sc.stream_with(None, rels, [pg.insert(91, ["1", "a"]), pg.insert(90, ["2", "b"])]).bytes()
    b2 = sc.stream_with(None, [], [pg.insert(90, ["3", "c"]), pg.insert(91, ["4", "d"])]).bytes()
    parts = _oracle_sequence(oracle_mod, tables, b1 + b2, [0, len(b1), len(b1) + len(b2)])
    assert [s.table_id for s in parts[0].schemas] == [91, 90]
    assert [s.table_id for s in parts[1].schemas] == [90, 91]
    assert [int(x) for x in parts[1].rec_schema[1:3]] == [0, 1]
