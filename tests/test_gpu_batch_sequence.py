"""Batch after batch on ONE decode context, against one oracle context driven through the same steps.

In production the library runs as one long-lived context, and every batch after the first is sized optimistically from
the history of the earlier ones.  Each test here reaches one sizing branch of run_decode (decode_api.cu) and asserts
it through etl_dec_summary.sizing, or exercises state that outlives a batch (device schema tables, installed Relation
versions, the staged-stream buffer, the stager).  Every batch is compared with the oracle plane by plane; sequences cut
from one stream are also stitched and compared with the oracle's decode of the whole stream.

Plane reservations of an optimistic batch (run_decode): records len·rec_per_byte·1.08 + 4096, cells
len·cells_per_byte·1.08 + 16384, frame offsets 2·records + 65536; the per-byte history is the max of the last batch's
density and 97 % of the previous history.  The tests compute the reservations from the oracle's counts and check that
each batch is on the intended side of them before they look at the sizing bits.
"""
import time

import numpy as np
import pytest

import scenarios as sc
from etl_b200 import pgoutput as pg
from etl_b200 import workloads as wl
from seq_util import (RERUN, SIZING, CopyDecode, Decode, PutTableSchema, ResetRelations, next_cut, record_cuts,
                      run_sequence, sizing_names, stitched_check)

pytestmark = pytest.mark.gpu

EXACT, OPT = SIZING["EXACT"], SIZING["OPTIMISTIC"]
HIST_TABLE = 80
HIST_COLS = [sc.col("id", sc.INT8, 1), sc.col("doc", sc.TEXT, None, True)]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


@pytest.fixture(autouse=True)
def _timed(request):
    t0 = time.time()
    yield
    print(f"\n[{request.node.name}] {time.time() - t0:.1f} s")


def history_batch():
    """A sparse first batch: one transaction of 16 inserts of 60 KiB text (≈2e-5 records/byte, ≈4e-5 cells/byte)."""
    rng = np.random.default_rng(80)
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(HIST_TABLE, "public", "hist", "d", sc.rel_cols(HIST_COLS, {"id"})))
    for i in range(16):
        w.emit(pg.insert(HIST_TABLE, [str(i), rng.integers(97, 123, size=60 << 10, dtype=np.uint8).tobytes()]))
    tx.commit()
    return w.bytes()


def reservations(hist_records, hist_cells, hist_len, n_bytes):
    """(records, cells, frame offsets) reserved for the batch right after the history batch."""
    cap_r = int(n_bytes * (hist_records / hist_len) * 1.08) + 4096
    cap_c = int(n_bytes * (hist_cells / hist_len) * 1.08) + 16384
    return cap_r, cap_c, 2 * cap_r + 65536


def oracle_of(oracle_mod, tables, stream, carry=None):
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        orc.put_table_schema(tid, cols)
    p = orc.decode(stream, carry)
    orc.close()
    return p


def stream_of(name, scale, seed_segment=0, bump=0):
    w = wl.make(name, scale, n_segments=1)
    w.schema_bump_ppm = bump or w.schema_bump_ppm
    s, _ = w.generate(range(seed_segment, seed_segment + 1))
    return w, s.tobytes()


def show(res, title):
    print(f"{title}: " + " | ".join(f"{b.label or i}:{'+'.join(sizing_names(b.sizing))}" for i, b in enumerate(res.batches)))


# ------------------------------------------------------------------------------------------------ 1. steady state
@pytest.mark.parametrize("name,scale,seed", [("c2", 0.06, 11), ("c4", 0.004, 12)])
def test_steady_state_sequence(gpu, oracle_mod, name, scale, seed):
    """~15 batches of log-uniform size (1 KiB – 4 MiB) cut at seeded record boundaries, anchor stride varying per
    batch, one reused stager: every batch after the first is optimistic and fits; stitched = the whole stream."""
    w, raw = stream_of(name, scale, bump=3000 if name == "c4" else 0)
    tables = w.table_schemas()
    full = oracle_of(oracle_mod, tables, raw)
    rng = np.random.default_rng(seed)
    cuts = record_cuts(full, len(raw), rng, 1 << 10, 4 << 20, first_min=256 << 10, max_parts=15)
    assert len(cuts) >= 13, len(cuts)
    strides = [int(x) for x in rng.choice([256, 1024, 2048, 8192, 32768], size=len(cuts) - 1)]
    steps = [Decode(raw[cuts[k]:cuts[k + 1]], stride=strides[k], label=f"{cuts[k + 1] - cuts[k]}B/s{strides[k]}")
             for k in range(len(cuts) - 1)]
    res = run_sequence(gpu, oracle_mod, steps, tables, reuse_stager=True)
    show(res, name)
    assert res.sizing[0] == EXACT
    for b in res.batches[1:]:
        assert b.sizing & OPT and not b.sizing & (EXACT | RERUN), (b.label, sizing_names(b.sizing))
    stitched_check(oracle_mod, tables, raw, cuts, [b.got for b in res.batches])


# ------------------------------------------------------------------------------------------------ 2. planes rerun
def test_rerun_records_after_sparse_history(gpu, oracle_mod):
    """After the sparse history batch, 4 MiB of c2 holds more frames than the record reservation but fewer than the
    offset scratch: the tuple pass runs again with exact sizes (k_records wrote nothing the first time)."""
    hist = history_batch()
    hp = oracle_of(oracle_mod, {HIST_TABLE: HIST_COLS}, hist)
    w, raw = stream_of("c2", 0.03)
    tables = {HIST_TABLE: HIST_COLS, **w.table_schemas()}
    full = oracle_of(oracle_mod, tables, raw)
    end = int(full.rec_off[np.searchsorted(full.rec_off, 4 << 20)])
    batch = raw[:end]
    n_rec = int(np.searchsorted(full.rec_off, end))
    cap_r, _, cap_scratch = reservations(hp.n_records, hp.n_cells, len(hist), len(batch))
    assert cap_r < n_rec < cap_scratch, (cap_r, n_rec, cap_scratch)
    res = run_sequence(gpu, oracle_mod, [Decode(hist, label="hist"), Decode(batch, label="c2"),
                                         Decode(raw[end:], label="c2 rest")], tables)
    show(res, "rerun records")
    assert res.sizing[0] == EXACT
    assert res.sizing[1] & SIZING["RERUN_RECORDS"] and res.sizing[1] & OPT, sizing_names(res.sizing[1])
    assert not res.sizing[1] & SIZING["SCRATCH_RESTART"]


def test_rerun_cells_only_after_sparse_history(gpu, oracle_mod):
    """~100 KiB of c2 then ~1 MiB of c3 (100 columns): under a thousand records fit the record reservation, tens of
    thousands of cells do not.  The first record CTA (512 records of c2) fits and writes its records before the
    overflow; the rerun overwrites them."""
    hist = history_batch()
    hp = oracle_of(oracle_mod, {HIST_TABLE: HIST_COLS}, hist)
    w2, raw2 = stream_of("c2", 0.004)
    w3 = wl.make("c3", 0.002, n_segments=1)
    w3.tables[0].rel_id = 32000
    raw3 = w3.generate()[0].tobytes()
    tables = {HIST_TABLE: HIST_COLS, **w2.table_schemas(), **w3.table_schemas()}
    p2 = oracle_of(oracle_mod, tables, raw2)
    p3 = oracle_of(oracle_mod, tables, raw3)
    c3_rest = int(p3.rec_off[np.searchsorted(p3.rec_off, 1 << 20)])
    batch = raw2[:int(p2.rec_off[600])] + raw3[:c3_rest]
    full = oracle_of(oracle_mod, tables, batch)
    assert full.first_error[0] is None
    cap_r, cap_c, _ = reservations(hp.n_records, hp.n_cells, len(hist), len(batch))
    assert full.n_records < cap_r and full.n_cells > cap_c, (full.n_records, cap_r, full.n_cells, cap_c)
    assert int(full.rec_cell_base[512]) <= cap_c                   # the first CTA of k_records fits
    res = run_sequence(gpu, oracle_mod, [Decode(hist, label="hist"), Decode(batch, label="c2+c3"),
                                         Decode(raw3[c3_rest:], label="c3 rest")], tables)
    show(res, "rerun cells")
    assert res.sizing[1] & SIZING["RERUN_CELLS"] and not res.sizing[1] & SIZING["RERUN_RECORDS"], sizing_names(res.sizing[1])


# ------------------------------------------------------------------------------------------------ 3. scratch restart
def test_scratch_restart_then_normal_batch(gpu, oracle_mod):
    """~4 MiB of keepalives mixed with one-column inserts after the sparse history: far more frames than the offset
    scratch, so the attempt is abandoned and the batch decoded again on the exact path.  Then a normal batch."""
    hist = history_batch()
    hp = oracle_of(oracle_mod, {HIST_TABLE: HIST_COLS}, hist)
    one = [sc.col("id", sc.INT8, 1)]
    tables = {HIST_TABLE: HIST_COLS, 81: one}
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(81, "public", "one", "d", sc.rel_cols(one, {"id"})))
    i = 0
    while w.size < (4 << 20):
        w.emit(pg.insert(81, [str(i)]))
        w.emit_keepalive()
        w.emit_keepalive()
        i += 1
    tx.commit()
    batch = w.bytes()
    n_frames = sum(1 for _ in _frames(batch))
    _, _, cap_scratch = reservations(hp.n_records, hp.n_cells, len(hist), len(batch))
    assert n_frames > cap_scratch + 32768, (n_frames, cap_scratch)
    w2 = pg.StreamWriter()
    tx2 = sc.Tx(w2)
    tx2.begin()
    for j in range(200):
        w2.emit(pg.insert(81, [str(10 ** 6 + j)]))
    tx2.commit()
    res = run_sequence(gpu, oracle_mod, [Decode(hist, label="hist"), Decode(batch, label="keepalives"),
                                         Decode(w2.bytes(), label="normal")], tables)
    show(res, "scratch restart")
    s = res.sizing[1]
    assert s & SIZING["SCRATCH_RESTART"] and s & OPT and s & EXACT, sizing_names(s)
    assert res.sizing[2] & OPT and not res.sizing[2] & (RERUN | SIZING["SCRATCH_RESTART"]), sizing_names(res.sizing[2])


def _frames(raw):
    pos = 0
    while pos < len(raw):
        yield pos
        pos += 1 + int.from_bytes(raw[pos + 1:pos + 5], "big")


# ------------------------------------------------------------------------------------------------ 4. array heap retry
def test_array_heap_retry_with_history(gpu, oracle_mod):
    """Arrays of many empty elements on a primed context: the array heap is enlarged and the tuple pass runs again.
    The next batch is correct."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("a", 1009, None, True)]
    rel = pg.relation(93, "public", "wide", "d", sc.rel_cols(cols, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(64):
        w.emit(pg.insert(93, [str(r), "{" + "," * 3000 + "}"]))
    tx.commit()
    w2 = pg.StreamWriter()
    tx2 = sc.Tx(w2)
    tx2.begin()
    for r in range(300):
        w2.emit(pg.insert(93, [str(r), "{a,NULL,\"b c\"}"]))
        w2.emit(pg.insert(HIST_TABLE, [str(r), "x" * (r % 700)]))
    tx2.commit()
    tables = {HIST_TABLE: HIST_COLS, 93: cols}
    res = run_sequence(gpu, oracle_mod, [Decode(history_batch(), label="hist"), Decode(w.bytes(), label="arrays"),
                                         Decode(w2.bytes(), label="after")], tables)
    show(res, "array heap")
    assert res.sizing[1] & SIZING["ARRAY_HEAP_RETRY"] and res.sizing[1] & OPT, sizing_names(res.sizing[1])
    assert not res.sizing[2] & SIZING["ARRAY_HEAP_RETRY"]


# ------------------------------------------------------------------------------------------------ 5. wrong hint
@pytest.mark.parametrize("poison", [False, True])
def test_wrong_frame_hint_with_history(gpu, oracle_mod, poison):
    """A c5 batch whose frame-length hint wrongly promises short frames, on a primed context: the long-value passes run
    late; the first error (a poisoned byte deep inside a TOAST value) is the oracle's.  Then the stager's own hint."""
    w, raw = stream_of("c5", 0.0004)
    tables = {HIST_TABLE: HIST_COLS, **w.table_schemas()}
    clean = oracle_of(oracle_mod, tables, raw)
    longs = np.flatnonzero((np.asarray(clean.cell_tag) == 2) & (np.asarray(clean.cell_aux) > 8192))
    assert len(longs) > 4
    data = raw
    if poison:
        v = int(longs[len(longs) // 2])
        b = bytearray(raw)
        b[int(clean.cell_val[v]) + int(clean.cell_aux[v]) // 2] = 0xFF
        data = bytes(b)
    _, raw2 = stream_of("c5", 0.0004, seed_segment=1)
    res = run_sequence(gpu, oracle_mod, [Decode(history_batch(), label="hist"), Decode(data, max_frame_len=64, label="hint 64"),
                                         Decode(raw2, label="own hint")], tables)
    show(res, f"wrong hint poison={poison}")
    assert res.sizing[1] & SIZING["LONG_PASSES_LATE"] and res.sizing[1] & OPT, sizing_names(res.sizing[1])
    assert (res.batches[1].want.first_error[0] is not None) == poison
    assert not res.sizing[2] & SIZING["LONG_PASSES_LATE"]


# ------------------------------------------------------------------------------------------------ 6. relation lifecycle
LC_COLS = [sc.col("id", sc.INT8, 1), sc.col("a", sc.TEXT, None, True), sc.col("b", sc.INT4, None, True)]


def _tx(*msgs):
    return sc.stream_with(None, [], list(msgs)).bytes()


def test_relation_lifecycle(gpu, oracle_mod):
    v1 = pg.relation(70, "public", "t", "d", sc.rel_cols(LC_COLS[:2], {"id"}))
    v2 = pg.relation(70, "public", "t", "f", sc.rel_cols(LC_COLS, set()))
    v3 = pg.relation(70, "public", "t", "d", sc.rel_cols([LC_COLS[0], LC_COLS[2]], {"id"}))
    ins1 = lambda i: pg.insert(70, [str(i), f"a{i}"])                   # noqa: E731  v1 / v3 shape: 2 columns
    ins2 = lambda i: pg.insert(70, [str(i), f"a{i}", str(i * 7)])        # noqa: E731  v2 shape: 3 columns
    upd2 = lambda i: pg.update(70, [str(i), "new", "1"], old=[str(i), f"a{i}", str(i * 7)])  # noqa: E731
    b_text = [sc.col("id", sc.INT8, 1), sc.col("a", sc.TEXT, None, True), sc.col("b", sc.TEXT, None, True)]
    steps = [
        Decode(_tx(v1, *[ins1(i) for i in range(50)]), label="v1"),
        Decode(_tx(*[ins1(i) for i in range(50, 90)]), label="v1 dml only"),                     # device tables reused
        Decode(_tx(ins1(90), ins1(91), v2, ins2(92), upd2(92), ins2(93)), label="v2 mid-batch"),
        Decode(_tx(ins2(94), upd2(94), pg.delete(70, old=[str(94), "new", "1"])), label="v2 dml only"),
        Decode(_tx(ins2(95), pg.insert(70, ["96", "x", "notint"]), v3, ins1(97)), label="error before v3"),
        Decode(_tx(ins2(98), ins1(99)), label="still v2"),                                           # v3-shaped row fails
        PutTableSchema(70, b_text),                                                                  # no Relation yet
        Decode(_tx(ins2(100), pg.insert(70, ["101", "x", "notint"])), label="stored changed, v2 in force"),
        Decode(_tx(v2, pg.insert(70, ["102", "x", "notint"])), label="v2 again, text b"),
        Decode(_tx(pg.insert(70, ["103", "y", "alsotext"])), label="text b, dml only"),
        ResetRelations(),
        Decode(_tx(ins2(104)), label="after reset"),
    ]
    res = run_sequence(gpu, oracle_mod, steps, {70: LC_COLS})
    show(res, "relations")
    fe = [b.got.first_error for b in res.batches]
    assert [e[0] for e in fe[:4]] == [None] * 4
    assert (fe[4][0], fe[4][2]) == (2, 2)             # "notint" as int4, before v3
    assert (fe[5][0], fe[5][2]) == (2, 12)            # v2 still in force: the 2-column row has the wrong field count
    assert (fe[6][0], fe[6][2]) == (2, 2)             # put_table_schema alone changes nothing
    assert fe[7][0] is None and fe[8][0] is None      # the next Relation picks the new stored schema up
    assert (fe[9][0], fe[9][2]) == (1, 19)            # missing table state after reset_relations
    assert all(b.sizing & OPT for b in res.batches[1:])


# ------------------------------------------------------------------------------------------------ 7. entry points
def test_interleaved_entry_points(gpu, oracle_mod):
    """Replication batch → COPY rows → replication batch WITHOUT a Relation (device tables rebuilt after the COPY
    decode reused them) → two-phase begin/finish → replication batch; all on one context, stitched."""
    from test_gpu_copy import cols_of, synth_rows
    w, raw = stream_of("c2", 0.01)
    tables = w.table_schemas()
    full = oracle_of(oracle_mod, tables, raw)
    cuts = record_cuts(full, len(raw), np.random.default_rng(7), 64 << 10, 512 << 10, first_min=128 << 10, max_parts=4)
    assert len(cuts) == 5
    oids, rows = synth_rows(3000, 99)
    parts = [raw[cuts[k]:cuts[k + 1]] for k in range(4)]
    steps = [Decode(parts[0], label="repl"), CopyDecode(7, rows), Decode(parts[1], label="repl, no Relation"),
             Decode(parts[2], two_phase=True, label="two-phase"), CopyDecode(7, rows[:17]), Decode(parts[3], label="repl")]
    res = run_sequence(gpu, oracle_mod, steps, {**tables, 7: cols_of(oids)}, reuse_stager=True)
    show(res, "interleaved")
    assert res.sizing[2] == EXACT                      # decode_finish: totals known
    stitched_check(oracle_mod, tables, raw, cuts, [b.got for b in res.batches])


# ------------------------------------------------------------------------------------------------ 8. size swings
def test_size_swings(gpu, oracle_mod):
    """8 MiB of c5 (clean, then poisoned deep inside a long value) → a 300-byte batch (the single-CTA activity pass) →
    an empty batch → keepalives only → long values again.  Stale bytes of the staged-stream buffer, the line bitmap
    or the long-cell list of an earlier, larger batch must not leak into a later one."""
    w, big = stream_of("c5", 0.0008)
    tables = w.table_schemas()
    clean = oracle_of(oracle_mod, tables, big)
    longs = np.flatnonzero((np.asarray(clean.cell_tag) == 2) & (np.asarray(clean.cell_aux) > 8192))
    b = bytearray(big)
    v = int(longs[-1])
    b[int(clean.cell_val[v]) + int(clean.cell_aux[v]) - 100] = 0xC0
    poisoned = bytes(b)
    tid = w.tables[0].rel_id
    small = sc.stream_with(None, [], [pg.insert(tid, ["1", "2", None, "3", "4", "short", None, "x", "y", "z", "doc" * 20])]).bytes()
    assert 250 < len(small) < 350
    kw = pg.StreamWriter()
    for _ in range(40):
        kw.emit_keepalive()
    _, again = stream_of("c5", 0.0003, seed_segment=3)
    steps = [Decode(big, stride=256, label="8MiB clean"), Decode(poisoned, stride=256, label="8MiB poisoned"),
             Decode(small, stride=256, label=f"{len(small)}B"), Decode(b"", stride=256, label="empty"),
             Decode(kw.bytes(), stride=256, label="keepalives"), Decode(again, stride=256, label="long again")]
    for reuse in (False, True):
        res = run_sequence(gpu, oracle_mod, steps, tables, reuse_stager=reuse)
        show(res, f"size swings reuse_stager={reuse}")
        assert res.batches[1].want.first_error[0] is not None
        assert res.batches[3].got.n_records == 0 and res.batches[4].got.n_records == 40


# ------------------------------------------------------------------------------------------------ 9. seeded soak
def test_seeded_soak(gpu, oracle_mod):
    """~30 batches cut at random sizes and strides from one stream of c1–c5 segments (table ids made distinct), sparse
    TOAST segments right before dense ones.  Checked per batch and stitched; prints the histogram of sizing bits."""
    specs = [("c5", 0.0003, 0, 30000), ("c1", 0.5, 0, 31000), ("c3", 0.0008, 0, 32000), ("c5", 0.0003, 1, 33000),
             ("c2", 0.004, 0, 34000), ("c4", 0.0008, 0, 35000), ("c5", 0.0002, 2, 36000), ("c1", 0.3, 1, 37000)]
    tables, chunks = {}, []
    for name, scale, seg, base in specs:
        w = wl.make(name, scale, n_segments=1)
        for k, t in enumerate(w.tables):
            t.rel_id = base + k
        if name == "c4":
            w.schema_bump_ppm = 3000
        s, _ = w.generate(range(seg, seg + 1))
        chunks.append(s.tobytes())
        tables.update(w.table_schemas())
    raw = b"".join(chunks)
    full = oracle_of(oracle_mod, tables, raw)
    assert full.first_error[0] is None
    # the first batch is the whole sparse c5 segment (its history: ≈2e-4 records/byte), the second 1 MiB of the dense c1
    # segment after it (≈9e-3 records/byte); the rest is cut at random
    c2nd = next_cut(full, len(chunks[0]) + (1 << 20))
    rng = np.random.default_rng(2026)
    cuts = [0, len(chunks[0]), c2nd] + [c for c in record_cuts(full, len(raw), rng, 2 << 10, 2 << 20, max_parts=40) if c > c2nd]
    strides = [int(x) for x in rng.choice([256, 512, 2048, 4096, 32768], size=len(cuts) - 1)]
    steps = [Decode(raw[cuts[k]:cuts[k + 1]], stride=strides[k], label=f"{cuts[k + 1] - cuts[k]}B") for k in range(len(cuts) - 1)]
    res = run_sequence(gpu, oracle_mod, steps, tables, reuse_stager=True)
    hist = res.histogram()
    print(f"soak: {len(res.batches)} batches, {len(raw)} bytes, sizing histogram {dict(hist)}")
    show(res, "soak")
    assert len(res.batches) >= 30
    assert hist["EXACT"] >= 1 and hist["OPTIMISTIC"] >= 1 and hist["RERUN_RECORDS"] + hist["RERUN_CELLS"] >= 1
    assert res.sizing[1] & RERUN, sizing_names(res.sizing[1])
    stitched_check(oracle_mod, tables, raw, cuts, [b.got for b in res.batches])


# ------------------------------------------------------------------------------------------------ regressions
def _one_row_tx(first: bool):
    cols = [sc.col("id", sc.INT8, 1)]
    rels = [pg.relation(82, "public", "k", "d", sc.rel_cols(cols, {"id"}))] if first else []
    return {82: cols}, sc.stream_with(None, rels, [pg.insert(82, ["1" if first else "2"])]).bytes()


def test_carry_passes_through_keepalive_batch(gpu, oracle_mod):
    """A batch of keepalives between two transactions hands on the carry it received: final_lsn of the last Begin
    passes through, as in one decode of the joined batches (the device used to report final_lsn 0 after it)."""
    tables, first = _one_row_tx(True)
    _, last = _one_row_tx(False)
    kw = pg.StreamWriter()
    for _ in range(3):
        kw.emit_keepalive()
    res = run_sequence(gpu, oracle_mod, [Decode(first), Decode(kw.bytes()), Decode(last)], tables)
    c0, c1 = res.batches[0].got.carry_out, res.batches[1].got.carry_out
    assert c0[0] == 0 and c0[1] != 0 and c1 == c0, (c0, c1)
    cuts = [0, len(first), len(first) + kw.size, len(first) + kw.size + len(last)]
    stitched_check(oracle_mod, tables, first + kw.bytes() + last, cuts, [b.got for b in res.batches])


def test_empty_batch_on_a_used_context(gpu, oracle_mod):
    """An empty batch after another one: rec_cell_base[0] must be 0 (no record pass runs, and the plane block comes
    from the stream-ordered pool with whatever an earlier batch left there); the carry passes through."""
    tables, first = _one_row_tx(True)
    _, last = _one_row_tx(False)
    res = run_sequence(gpu, oracle_mod, [Decode(first), Decode(b""), Decode(last)], tables)
    e = res.batches[1].got
    assert e.n_records == 0 and e.n_cells == 0 and e.rec_cell_base.tolist() == [0]
    assert e.carry_out == res.batches[0].got.carry_out
